// Index::multi_search_batched with hybrid requests at topster_size 5000. With TSGPU_VEC_DEEP_TOPSTER in the request's vector
// parameters the keyword rounds run at the full Topster size and the fusion keeps the whole Topster: more than TSGPU_MAX_TOPK
// records. Without the bit the same requests return exactly what topster_size 1024 returns. A deep request with diversity
// metrics is re-ranked over its whole fused list before it is cut to `hits`. The records of every request are written to the
// file named by argv[1], so that the run linked against libtsgpu.so can be compared record for record with the run linked
// against the oracle-backed test double (tests/cpp/tsgpu_oracle_double.cpp).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../../typesense_b200/host/tsgpu_host.hpp"
#include "../../oracle/ts_oracle.h"      // test infrastructure: only used to build the HNSW graph

static int failures = 0;
#define CHECK(cond) do { if(!(cond)) { failures++; printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); } } while(0)

using tsgpu::KV;
static bool same_bytes(const std::vector<KV>& a, const std::vector<KV>& b) {
    return a.size() == b.size() && (a.empty() || memcmp(a.data(), b.data(), a.size() * sizeof(KV)) == 0);
}

int main(int argc, char** argv) {
    const uint32_t n = 6000, dim = 16;
    tsgpu::Index index(n);
    tsgpu::field_mirror_t title;
    std::mt19937 rng(11);
    std::unordered_map<uint32_t, int64_t> points;
    for(uint32_t i = 0; i < n; i++) {            // frequent words (alpha: 2/3 of the documents, beta: 1/2) and rare ones
        std::string t = "w" + std::to_string(rng() % 400);
        if(i % 3) t += " alpha";
        if(i % 2) t += " beta";
        if(i % 5 == 0) t += " alpha gamma";
        title.index_plain_string(i, tsgpu::tokenize_ascii(t));
        points[i] = (int64_t) (rng() % 7);
    }
    CHECK(index.add_field("title", title).ok());
    CHECK(index.add_sort_field("points", points).ok());
    std::normal_distribution<float> nd;
    std::vector<float> vecs((size_t) n * dim);
    for(uint32_t i = 0; i < n; i++) {
        float s = 0;
        for(uint32_t d = 0; d < dim; d++) { vecs[(size_t) i * dim + d] = nd(rng); s += vecs[(size_t) i * dim + d] * vecs[(size_t) i * dim + d]; }
        for(uint32_t d = 0; d < dim; d++) vecs[(size_t) i * dim + d] /= std::sqrt(s);
    }
    void* bld = tso_hnsw_build(vecs.data(), n, dim, 16, 100, 100);
    uint32_t max_level = 0, entry = 0; uint64_t n_up = 0;
    tso_hnsw_build_info(bld, &max_level, &entry, &n_up);
    std::vector<uint8_t> levels(n); std::vector<uint32_t> links0((size_t) n * 33), links_up((n_up + 1) * 17); std::vector<uint64_t> upper_off(n + 1);
    tso_hnsw_build_fetch(bld, levels.data(), links0.data(), upper_off.data(), links_up.data());
    tso_hnsw_build_free(bld);
    const tsgpu_hnsw g{n, dim, 16, max_level, entry, 0, vecs.data(), nullptr, levels.data(), links0.data(), upper_off.data(), links_up.data()};
    CHECK(index.add_vector_field(g).ok());

    const std::vector<std::vector<std::string>> queries = {{"alpha"}, {"alpha", "beta"}, {"beta", "gamma"}, {"w17"}, {"alpah"}, {}};
    const std::vector<tsgpu::sort_by> sf = {{tsgpu::sort_by::text_match, "", true}, {tsgpu::sort_by::numeric, "points", true}};
    auto requests = [&](size_t topster_size, uint32_t flags, uint32_t k, float alpha) {
        std::vector<tsgpu::Index::batched_request> rs;
        for(size_t i = 0; i < queries.size(); i++) {
            tsgpu::Index::batched_request b;
            b.r.tokens = queries[i]; b.r.the_fields = {"title"}; b.r.sort_fields = sf;
            b.r.topster_size = topster_size;
            b.query_vector = vecs.data() + (size_t) (31 * i + 5) * dim;
            b.vp = tsgpu_vec_params{k, 10, 0, 3.4e38f, alpha, 100, flags};
            rs.push_back(b);
        }
        return rs;
    };
    FILE* dump = argc > 1 ? fopen(argv[1], "wb") : nullptr;
    auto write = [&](const std::vector<tsgpu::Index::search_response>& r) {
        for(auto& x: r) {
            const uint64_t hdr[2] = {x.found, x.raw_result_kvs.size()};
            if(dump) { fwrite(hdr, 8, 2, dump); fwrite(x.raw_result_kvs.data(), sizeof(KV), x.raw_result_kvs.size(), dump); }
        }
    };
    for(const float alpha: {0.3f, 0.8f}) {
        for(const uint32_t k: {200u, 3000u}) {
            const auto deep = index.multi_search_batched(requests(5000, TSGPU_VEC_DEEP_TOPSTER, k, alpha), 2);
            const auto plain = index.multi_search_batched(requests(5000, 0, std::min(k, 1024u), alpha), 2);
            const auto capped = index.multi_search_batched(requests(1024, 0, std::min(k, 1024u), alpha), 2);
            size_t longest = 0;
            for(size_t i = 0; i < queries.size(); i++) {
                CHECK(deep[i].status.ok() && plain[i].status.ok() && capped[i].status.ok());
                if(!deep[i].status.ok()) printf("request %zu: %s\n", i, deep[i].status.error().c_str());
                longest = std::max(longest, deep[i].raw_result_kvs.size());
                CHECK(deep[i].raw_result_kvs.size() <= 5000);
                // without the bit: what topster_size 1024 returns
                CHECK(plain[i].found == capped[i].found && same_bytes(plain[i].raw_result_kvs, capped[i].raw_result_kvs));
                CHECK(plain[i].raw_result_kvs.size() <= 1024);
            }
            CHECK(longest > 1024);
            write(deep); write(plain);
        }
    }
    // diversity over the whole fused list (where the library has tsgpu_diversify_batch)
    if(tsgpu_diversify_batch) {
        auto whole = requests(5000, TSGPU_VEC_DEEP_TOPSTER, 3000, 0.3f);
        auto with = whole;
        for(auto& b: with) {
            b.hits = 300;
            b.r.opts.diversity = {{"points", TSGPU_DIV_EQUALITY, 1.0f}};
            b.r.opts.diversity_lambda = 0.4f;
        }
        const auto rw = index.multi_search_batched(whole, 2);
        const auto rd = index.multi_search_batched(with, 2);
        std::vector<std::vector<KV>> lists(queries.size());
        std::vector<std::vector<KV>*> lp;
        std::vector<const tsgpu::search_options*> lo;
        for(size_t i = 0; i < queries.size(); i++) {
            CHECK(rw[i].status.ok() && rd[i].status.ok());
            lists[i] = rw[i].raw_result_kvs;
            lp.push_back(&lists[i]); lo.push_back(&with[i].r.opts);
        }
        std::vector<tsgpu::Option<bool>> dst;
        index.diversify_lists(lp, lo, dst);
        size_t longest = 0;
        for(size_t i = 0; i < queries.size(); i++) {
            CHECK(dst[i].ok());
            longest = std::max(longest, rw[i].raw_result_kvs.size());
            std::vector<KV> want(lists[i].begin(), lists[i].begin() + std::min<size_t>(300, lists[i].size()));
            CHECK(rd[i].found == rw[i].found && same_bytes(rd[i].raw_result_kvs, want));
        }
        CHECK(longest > 1024);
        write(rd);
        printf("diversity: re-ranked over fused lists of up to %zu records\n", longest);
    }
    if(dump) fclose(dump);
    printf("%s (%d failures)\n", failures ? "FAILED" : "ok", failures);
    return failures ? 1 : 0;
}
