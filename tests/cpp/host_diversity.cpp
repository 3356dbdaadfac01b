// The C++ host layer's diversity re-ranking (search_options::diversity, Index::add_facet_field): the reference's DiversityOverride
// scenario through Index::search, the re-ranked list of keyword / q=* / hybrid requests against the oracle's transcription of the
// reference loop (tso_diversify) over the list the request returns without metrics, requests without metrics unchanged next to
// ones with metrics in multi_search_batched, search_grouped ignoring the metrics, and the reference's 400 for an unknown field.
// Linked against libtsgpu.so, or against the oracle-backed test double (tests/cpp/tsgpu_oracle_double_diversity.cpp) on a machine
// without a GPU.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../../typesense_b200/host/tsgpu_host.hpp"
#ifdef WITH_ORACLE_DIVERSIFY
#include "tso_diversify.cpp"           // the test double already carries the oracle
#else
#include "../../oracle/ts_oracle.h"
extern "C" {
typedef struct { const uint64_t* doc_off; const uint32_t* value_ids; const int64_t* sort_col; uint32_t method; float weight; } tso_div_metric;
void tso_diversify(uint32_t n_docs, const tso_div_metric* metrics, uint32_t n_metrics, float lambda, const tso_kv* topster, uint32_t size, tso_kv* out);
}
#endif

static int failures = 0;
#define CHECK(cond) do { if(!(cond)) { failures++; printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); } } while(0)

using tsgpu::KV;
static std::vector<uint64_t> keys_of(const std::vector<KV>& kvs) { std::vector<uint64_t> r; for(auto& kv: kvs) r.push_back(kv.key); return r; }
static bool same_bytes(const std::vector<KV>& a, const std::vector<KV>& b) {
    return a.size() == b.size() && (a.empty() || memcmp(a.data(), b.data(), a.size() * sizeof(KV)) == 0);
}

// TEST_F(CollectionCurationTest, DiversityOverride), test/collection_curation_test.cpp:5591-5691
static void diversity_override() {
    const std::vector<std::vector<std::string>> tags = {{"gold", "silver"}, {"FINE PLATINUM"}, {"bronze", "gold"}, {"silver"},
                                                        {"silver", "gold", "bronze"}, {"silver", "FINE PLATINUM"}};
    tsgpu::Index index(6);
    tsgpu::field_mirror_t m(true);
    std::map<std::string, uint32_t> value_id;
    std::vector<uint64_t> doc_off{0};
    std::vector<uint32_t> vals;
    for(uint32_t d = 0; d < tags.size(); d++) {
        std::vector<std::vector<std::string>> elems;
        for(auto& t: tags[d]) {
            elems.push_back(tsgpu::tokenize_ascii(t));
            auto it = value_id.emplace(t, (uint32_t) value_id.size()).first;
            vals.push_back(it->second);
        }
        m.index_string_array(d, elems);
        doc_off.push_back(vals.size());
    }
    CHECK(index.add_field("tags", m).ok());
    CHECK(index.add_facet_field("tags", doc_off, vals).ok());
    const std::vector<tsgpu::sort_by> by_seq_id = {{tsgpu::sort_by::seq_id, "", true}};
    tsgpu::search_options o;
    std::vector<KV> kvs;
    size_t found = 0;
    CHECK(index.search({}, {"tags"}, by_seq_id, 1, 250, kvs, found, o).ok());
    CHECK(found == 6 && (keys_of(kvs) == std::vector<uint64_t>{5, 4, 3, 2, 1, 0}));
    o.diversity = {{"tags", TSGPU_DIV_JACCARD, 1.0f}};
    CHECK(index.search({}, {"tags"}, by_seq_id, 1, 250, kvs, found, o).ok());
    CHECK(found == 6 && (keys_of(kvs) == std::vector<uint64_t>{5, 2, 0, 3, 1, 4}));
    o.diversity_lambda = 1.0f;                                           // no diversity
    CHECK(index.search({}, {"tags"}, by_seq_id, 1, 250, kvs, found, o).ok());
    CHECK((keys_of(kvs) == std::vector<uint64_t>{5, 4, 3, 2, 1, 0}));
    o.diversity_lambda = 7.0f;                                           // outside [0, 1]: the parameter keeps its default 0.5
    CHECK(index.search({}, {"tags"}, by_seq_id, 1, 250, kvs, found, o).ok());
    CHECK((keys_of(kvs) == std::vector<uint64_t>{5, 2, 0, 3, 1, 4}));
    // a keyword query: "silver" matches 0, 3, 4, 5
    o.diversity_lambda = 0.5f;
    CHECK(index.search({"silver"}, {"tags"}, by_seq_id, 1, 250, kvs, found, o).ok());
    CHECK(found == 4 && kvs.size() == 4);
    printf("diversity override: %zu hits\n", kvs.size());
}

struct Data {
    uint32_t n = 0;
    std::vector<uint64_t> tag_off;
    std::vector<uint32_t> tag_vals;
    std::vector<int64_t> brand, points;
};

static std::vector<KV> oracle_mmr(const Data& d, const std::vector<KV>& list, float lambda, float w_tags, float w_brand) {
    const tso_div_metric m[2] = {{d.tag_off.data(), d.tag_vals.data(), nullptr, TSGPU_DIV_JACCARD, w_tags},
                                 {nullptr, nullptr, d.brand.data(), TSGPU_DIV_EQUALITY, w_brand}};
    std::vector<KV> out(list.size());
    if(!list.empty())
        tso_diversify(d.n, m, 2, lambda, reinterpret_cast<const tso_kv*>(list.data()), (uint32_t) list.size(), reinterpret_cast<tso_kv*>(out.data()));
    return out;
}

static void collection_scenarios() {
    const uint32_t n = 600, dim = 8;
    std::mt19937 rng(11);
    const std::vector<std::string> vocab = {"red", "green", "blue", "shoe", "shirt", "hat", "sock", "bag", "belt", "coat", "scarf", "boot"};
    Data d;
    d.n = n;
    tsgpu::field_mirror_t title;
    d.tag_off.push_back(0);
    std::unordered_map<uint32_t, int64_t> points;
    for(uint32_t i = 0; i < n; i++) {
        std::vector<std::string> toks;
        const uint32_t nt = 2 + rng() % 4;
        for(uint32_t t = 0; t < nt; t++) toks.push_back(vocab[rng() % vocab.size()]);
        title.index_plain_string(i, toks);
        const uint32_t ntags = rng() % 5;                                 // 0..4 tags, repeats allowed (a set compares them once)
        for(uint32_t t = 0; t < ntags; t++) d.tag_vals.push_back(rng() % 9);
        d.tag_off.push_back(d.tag_vals.size());
        d.brand.push_back(rng() % 4 == 0 ? INT64_MIN : (int64_t) (rng() % 6));
        points[i] = (int64_t) (rng() % 7);
    }
    std::vector<float> vecs((size_t) n * dim);
    std::normal_distribution<float> nd;
    for(auto& v: vecs) v = nd(rng);
    void* bld = tso_hnsw_build(vecs.data(), n, dim, 8, 100, 100);
    uint32_t max_level = 0, entry = 0; uint64_t n_up = 0;
    tso_hnsw_build_info(bld, &max_level, &entry, &n_up);
    std::vector<uint8_t> levels(n); std::vector<uint32_t> links0((size_t) n * 17), links_up((n_up + 1) * 9); std::vector<uint64_t> upper_off(n + 1);
    tso_hnsw_build_fetch(bld, levels.data(), links0.data(), upper_off.data(), links_up.data());
    tso_hnsw_build_free(bld);
    const tsgpu_hnsw g{n, dim, 8, max_level, entry, 0, vecs.data(), nullptr, levels.data(), links0.data(), upper_off.data(), links_up.data()};

    tsgpu::Index index(n);
    CHECK(index.add_field("title", title).ok());
    CHECK(index.add_sort_field("points", points).ok());
    CHECK(index.add_sort_field_dense("brand", d.brand.data()).ok());
    CHECK(index.add_facet_field("tags", d.tag_off, d.tag_vals).ok());
    CHECK(index.add_vector_field(g).ok());
    const std::vector<tsgpu::sort_by> sf = {{tsgpu::sort_by::text_match, "", true}, {tsgpu::sort_by::numeric, "points", true}};
    const float w_tags = 0.6f, w_brand = 0.1f;

    // ---- a request list: keyword, q=*, typo and hybrid requests; every other one carries metrics
    std::vector<tsgpu::Index::batched_request> plain, with;
    // (9: phrase-only, "red shoe" as a phrase)
    const std::vector<std::vector<std::string>> queries = {{"red"}, {}, {"shrit"}, {"blue", "shoe"}, {}, {"coat"}, {"green", "hat", "sock"}, {"bag"}, {"hat"}, {}};
    const float lambdas[] = {0.5f, 0.3f, 0.0f, 1.0f};
    for(size_t i = 0; i < queries.size(); i++) {
        tsgpu::Index::batched_request b;
        b.r.tokens = queries[i]; b.r.the_fields = {"title"}; b.r.sort_fields = sf;
        b.r.topster_size = i == 4 ? 40 : 250;
        if(i == 9) b.r.opts.phrases = {{"red", "shoe"}};
        if(i == 5 || i == 7) { b.query_vector = vecs.data() + (size_t) (17 * i) * dim; b.hits = 10; b.vp.k = 60; b.vp.ef = 80; }
        plain.push_back(b);
        if(i % 2 == 1) {
            b.r.opts.diversity = {{"tags", TSGPU_DIV_JACCARD, w_tags}, {"brand", TSGPU_DIV_EQUALITY, w_brand}};
            b.r.opts.diversity_lambda = lambdas[(i / 2) % 4];
        }
        with.push_back(b);
    }
    auto r0 = index.multi_search_batched(plain, 2);
    auto r1 = index.multi_search_batched(with, 2);
    // the hybrid requests' whole fused Topsters, for the MMR the requests with metrics must show
    std::vector<tsgpu::Index::batched_request> whole = plain;
    for(auto& b: whole) b.hits = 0;
    auto rw = index.multi_search_batched(whole, 2);
    for(size_t i = 0; i < queries.size(); i++) {
        CHECK(r0[i].status.ok() && r1[i].status.ok() && rw[i].status.ok());
        CHECK(r0[i].found == r1[i].found);
        if(with[i].r.opts.diversity.empty()) {
            CHECK(same_bytes(r0[i].raw_result_kvs, r1[i].raw_result_kvs));
            continue;
        }
        const auto& base = with[i].query_vector ? rw[i].raw_result_kvs : r0[i].raw_result_kvs;
        auto want = oracle_mmr(d, base, with[i].r.opts.diversity_lambda, w_tags, w_brand);
        if(with[i].query_vector) {
            CHECK(base.size() > with[i].hits);                        // the re-ranking saw more than `hits` records
            if(want.size() > with[i].hits) want.resize(with[i].hits);
        }
        CHECK(same_bytes(r1[i].raw_result_kvs, want));
        printf("request %zu: %zu records re-ranked (%zu before truncation), lambda %.1f\n", i, r1[i].raw_result_kvs.size(), base.size(),
               with[i].r.opts.diversity_lambda);
    }
    // the same lists through Index::search one by one, and through the lock-step multi_search
    std::vector<tsgpu::Index::search_request> sreqs;
    for(size_t i = 0; i < queries.size(); i++) {
        if(with[i].query_vector) continue;
        std::vector<KV> kvs;
        size_t found = 0;
        CHECK(index.search(with[i].r.tokens, with[i].r.the_fields, with[i].r.sort_fields, 1, with[i].r.topster_size, kvs, found, with[i].r.opts).ok());
        CHECK(same_bytes(kvs, r1[i].raw_result_kvs));
        sreqs.push_back(with[i].r);
    }
    auto ls = index.multi_search(sreqs, true);
    for(size_t i = 0, k = 0; i < queries.size(); i++) {
        if(with[i].query_vector) continue;
        CHECK(ls[k].status.ok() && same_bytes(ls[k].raw_result_kvs, r1[i].raw_result_kvs));
        k++;
    }

    // ---- search_grouped ignores the metrics
    {
        tsgpu::search_options o, od;
        od.diversity = {{"tags", TSGPU_DIV_JACCARD, 1.0f}};
        std::vector<std::vector<KV>> ga, gb;
        size_t fa = 0, fb = 0;
        CHECK(index.search_grouped({"red"}, {"title"}, sf, 1, 20, "brand", 3, false, ga, fa, o).ok());
        CHECK(index.search_grouped({"red"}, {"title"}, sf, 1, 20, "brand", 3, false, gb, fb, od).ok());
        CHECK(fa == fb && ga.size() == gb.size() && !ga.empty());
        for(size_t i = 0; i < ga.size() && i < gb.size(); i++) CHECK(same_bytes(ga[i], gb[i]));
    }

    // ---- an unknown field: the reference's 400 once a pair is compared; a single hit compares none
    {
        tsgpu::search_options o;
        o.diversity = {{"tags", TSGPU_DIV_JACCARD, 1.0f}, {"colour", TSGPU_DIV_EQUALITY, 1.0f}};
        std::vector<KV> kvs;
        size_t found = 0;
        auto op = index.search({"red"}, {"title"}, sf, 1, 250, kvs, found, o);
        CHECK(!op.ok() && op.code() == 400 && op.error() == "`colour` field not found in either facet or sort index.");
        CHECK(index.search({"red"}, {"title"}, sf, 1, 1, kvs, found, o).ok() && kvs.size() == 1);
        std::vector<tsgpu::Index::batched_request> bad = {with[1], with[1]};
        bad[1].r.opts = o;
        auto rb = index.multi_search_batched(bad, 1);
        CHECK(rb[0].status.ok() && same_bytes(rb[0].raw_result_kvs, r1[1].raw_result_kvs));
        CHECK(!rb[1].status.ok() && rb[1].status.code() == 400);
    }
}

int main() {
    diversity_override();
    collection_scenarios();
    if(failures) { printf("%d failures\n", failures); return 1; }
    printf("host diversity: all checks passed\n");
    return 0;
}
