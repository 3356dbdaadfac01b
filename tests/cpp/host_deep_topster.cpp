// Index::multi_search_batched with topster_size 5000 (deep pagination): a keyword-only q=* and a phrase-only request return every
// match (more than TSGPU_MAX_TOPK), while the same requests with a query vector — whose keyword stage feeds
// tsgpu_hybrid_fuse_batch — return exactly what they return at topster_size 1024. Linked against libtsgpu.so, or against
// tests/cpp/tsgpu_oracle_double.cpp on a machine without a GPU.
#include <cstdio>
#include <cstdlib>
#include <random>
#include <string>
#include <vector>

#include "../../typesense_b200/host/tsgpu_host.hpp"
#include "../../oracle/ts_oracle.h"      // test infrastructure: only used to build the HNSW graph

static int failures = 0;
#define CHECK(cond) do { if(!(cond)) { failures++; printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); } } while(0)

int main() {
    const uint32_t n = 3000, dim = 8;
    tsgpu::Index index(n);
    tsgpu::field_mirror_t title;
    for(uint32_t i = 0; i < n; i++)              // every document holds the phrase "alpha beta"
        title.index_plain_string(i, tsgpu::tokenize_ascii("alpha beta w" + std::to_string(i % 50) + (i % 3 ? " gamma" : "")));
    CHECK(index.add_field("title", title).ok());
    std::mt19937 rng(5);
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
    const std::vector<float> qv(vecs.begin() + 7 * dim, vecs.begin() + 8 * dim);

    // requests: q=*, phrase-only; each keyword-only and with the query vector
    auto requests = [&](size_t topster_size) {
        std::vector<tsgpu::Index::batched_request> rs;
        for(int with_vec = 0; with_vec < 2; with_vec++)
            for(int phrase = 0; phrase < 2; phrase++) {
                tsgpu::Index::batched_request b;
                b.r.the_fields = {"title"};
                b.r.sort_fields = {{tsgpu::sort_by::text_match, "", true}, {tsgpu::sort_by::seq_id, "", true}};
                b.r.topster_size = topster_size;
                if(phrase) b.r.opts.phrases = {{"alpha", "beta"}};
                if(with_vec) { b.query_vector = qv.data(); b.vp = tsgpu_vec_params{0, 20, 0, 3.4e38f, 0.3f, 100, 0}; }
                rs.push_back(b);
            }
        return rs;
    };
    const auto deep = index.multi_search_batched(requests(5000), 2);
    const auto capped = index.multi_search_batched(requests(1024), 2);
    for(size_t i = 0; i < 4; i++) {
        CHECK(deep[i].status.ok() && capped[i].status.ok());
        if(!deep[i].status.ok()) printf("request %zu: %s\n", i, deep[i].status.error().c_str());
    }
    for(size_t i = 0; i < 2; i++) {              // keyword only: every match, beyond 1024
        CHECK(deep[i].found == n && deep[i].raw_result_kvs.size() == n);
        CHECK(capped[i].raw_result_kvs.size() == 1024);
        for(size_t j = 0; j < 1024 && j < deep[i].raw_result_kvs.size(); j++) CHECK(deep[i].raw_result_kvs[j].key == capped[i].raw_result_kvs[j].key);
    }
    for(size_t i = 2; i < 4; i++) {              // with a vector: what topster_size 1024 returns
        CHECK(deep[i].found == capped[i].found && deep[i].raw_result_kvs.size() == capped[i].raw_result_kvs.size());
        CHECK(!deep[i].raw_result_kvs.empty() && deep[i].raw_result_kvs.size() <= 1024 + 100);
        for(size_t j = 0; j < deep[i].raw_result_kvs.size() && j < capped[i].raw_result_kvs.size(); j++) {
            const tsgpu::KV& a = deep[i].raw_result_kvs[j];
            const tsgpu::KV& b = capped[i].raw_result_kvs[j];
            CHECK(a.key == b.key && a.scores[0] == b.scores[0] && a.scores[1] == b.scores[1] && a.scores[2] == b.scores[2]);
        }
    }
    printf("%s (%d failures)\n", failures ? "FAILED" : "ok", failures);
    return failures ? 1 : 0;
}
