// The C++ host layer following a live collection for good: Index::update_field (tsgpu_index_append_lists) after each batch of
// writes, Index::compact_field to free what the batches replaced, Index::reserve_docs when seq_ids reach the capacity. After every
// step Index::search — exact tokens, typo and prefix candidates from the ART mirror rebuilt over the compacted vocabulary, the
// default sorting field — must answer like an Index loaded from the documents as they stand. Linked against libtsgpu.so, or
// against tests/cpp/tsgpu_oracle_double.cpp on a machine without a GPU.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../typesense_b200/host/tsgpu_host.hpp"

static int failures = 0;
#define CHECK(cond) do { if(!(cond)) { failures++; printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); } } while(0)

static tsgpu::search_options opt(uint32_t num_typos, bool prefix) {
    tsgpu::search_options o;
    o.num_typos = num_typos; o.prefix = prefix; o.typo_tokens_threshold = 1;
    o.device_art_walk = getenv("TSGPU_HOST_DEVICE_ART") != nullptr;      // candidate walks through tsgpu_art_walk_batch
    return o;
}

static std::vector<uint64_t> keys_of(const std::vector<tsgpu::KV>& kvs) { std::vector<uint64_t> r; for(auto& kv: kvs) r.push_back(kv.key); return r; }

struct Collection {
    std::map<uint32_t, std::string> titles;       // live documents
    std::map<uint32_t, int64_t> points;
};

// an Index loaded at once from the documents as they stand
static void compare_with_fresh(tsgpu::Index& index, const Collection& c, uint32_t capacity, const char* step) {
    tsgpu::Index fresh(capacity);
    tsgpu::field_mirror_t m;
    std::unordered_map<uint32_t, int64_t> pts;
    for(auto& d: c.titles) m.index_plain_string(d.first, tsgpu::tokenize_ascii(d.second));
    for(auto& p: c.points) pts[p.first] = p.second;
    CHECK(fresh.add_field("title", m).ok());
    CHECK(fresh.add_sort_field("points", pts).ok());
    const std::vector<tsgpu::sort_by> sort_fields = {{tsgpu::sort_by::text_match, "", true}, {tsgpu::sort_by::numeric, "points", true}};
    for(const char* q: {"rocket", "launch", "brown", "quick rocket", "rocket launch", "bears", "rover", "north", "lau", "rokcet", "foxs", "luanch",
                        "guide", "the", "comet", "comte", "nebula", "orbit", "orb", "storm", "northern lights", "ro"}) {
        for(int mode = 0; mode < 2; mode++) {
            const bool prefix = mode == 1;
            std::vector<tsgpu::KV> a, b;
            size_t fa = 0, fb = 0;
            CHECK(index.search(tsgpu::tokenize_ascii(q), {"title"}, sort_fields, 1, 250, a, fa, opt(2, prefix)).ok());
            CHECK(fresh.search(tsgpu::tokenize_ascii(q), {"title"}, sort_fields, 1, 250, b, fb, opt(2, prefix)).ok());
            const bool same = fa == fb && keys_of(a) == keys_of(b);
            CHECK(same);
            if(!same) printf("  %s: query '%s' (prefix %d) differs: %zu vs %zu hits\n", step, q, (int) prefix, fa, fb);
            for(size_t i = 0; i < a.size() && i < b.size(); i++) CHECK(a[i].scores[0] == b[i].scores[0] && a[i].scores[1] == b[i].scores[1]);
        }
    }
}

static void write_doc(Collection& c, tsgpu::field_mirror_t& m, uint32_t id, const std::string& title, int64_t pts) {
    if(c.titles.count(id)) m.remove(id);
    m.index_plain_string(id, tsgpu::tokenize_ascii(title));
    c.titles[id] = title; c.points[id] = pts;
}

int main() {
    if(tsgpu_device_count() == 0) { printf("no CUDA device: nothing to run (the library has no CPU path)\n"); return 99; }
    uint32_t capacity = 8;
    tsgpu::Index index(capacity);
    CHECK(index.ok());
    Collection c;
    tsgpu::field_mirror_t m;
    const char* first[] = {"The quick brown fox", "Rocket launch delayed by weather", "Brown bears of the north", "A rocket science primer",
                           "Launch day for the new rover", "Quick guide to foxes"};
    for(uint32_t i = 0; i < 6; i++) write_doc(c, m, i, first[i], 100 - i);
    CHECK(index.add_field("title", m).ok());
    m.take_delta();
    {
        std::unordered_map<uint32_t, int64_t> pts(c.points.begin(), c.points.end());
        CHECK(index.add_sort_field("points", pts).ok());
    }
    compare_with_fresh(index, c, capacity, "loaded");
    // an unpatched field: compaction changes nothing
    CHECK(index.compact_field("title").ok());
    compare_with_fresh(index, c, capacity, "compacted, unpatched");
    // batch 1: new documents, a rewritten one, a removed one
    write_doc(c, m, 6, "Rocket fuel and brown sugar", 94);
    write_doc(c, m, 7, "Foxes launch a quick rocket", 93);
    write_doc(c, m, 2, "Rocket bears of the north", 98);
    m.remove(4); c.titles.erase(4); c.points.erase(4);
    CHECK(index.update_field("title", m.take_delta()).ok());
    CHECK(index.set_sort_values("points", {6, 7, 2, 4}, {94, 93, 98, INT64_MIN}).ok());
    compare_with_fresh(index, c, capacity, "batch 1");
    CHECK(index.compact_field("title").ok());
    compare_with_fresh(index, c, capacity, "batch 1, compacted");
    // the next seq_ids reach the capacity: grow first, as the binding does when next_seq_id passes it
    capacity = 40;
    CHECK(index.reserve_docs(capacity).ok());
    CHECK(index.capacity() == capacity);
    CHECK(!index.reserve_docs(10).ok());                        // the capacity never shrinks
    const char* more[] = {"Northern lights guide", "Rover lands after long launch", "Comet storm over the north", "Nebula and comet guide",
                          "Orbit of the rover", "Rocket orbit insertion", "Brown storm clouds", "Quick comet facts"};
    for(uint32_t i = 0; i < 8; i++) write_doc(c, m, 8 + 4 * i, more[i], 90 - (int64_t) i);        // ids 8 .. 36
    m.remove(6); c.titles.erase(6); c.points.erase(6);
    CHECK(index.update_field("title", m.take_delta()).ok());
    std::vector<uint32_t> ids;
    std::vector<int64_t> vals;
    for(uint32_t i = 0; i < 8; i++) { ids.push_back(8 + 4 * i); vals.push_back(90 - (int64_t) i); }
    ids.push_back(6); vals.push_back(INT64_MIN);
    CHECK(index.set_sort_values("points", ids, vals).ok());
    compare_with_fresh(index, c, capacity, "grown, batch 2");
    // repeated rewrites with a compaction after each
    for(int round = 0; round < 5; round++) {
        write_doc(c, m, 3, round % 2 ? "A rocket science primer" : "A comet science primer", 97);
        write_doc(c, m, 12, round % 2 ? "Nebula and comet guide" : "Nebula storm guide", 89);
        CHECK(index.update_field("title", m.take_delta()).ok());
        CHECK(index.compact_field("title").ok());
    }
    compare_with_fresh(index, c, capacity, "after rewrite rounds");
    // an erased token leaves the vocabulary and stays gone after compaction: "day" only lived in document 4
    std::vector<tsgpu::KV> kvs;
    size_t found = 0;
    const std::vector<tsgpu::sort_by> sf = {{tsgpu::sort_by::text_match, "", true}, {tsgpu::sort_by::numeric, "points", true}};
    CHECK(index.search(tsgpu::tokenize_ascii("day"), {"title"}, sf, 0, 250, kvs, found, opt(0, false)).ok());
    CHECK(found == 0 && kvs.empty());
    CHECK(!index.compact_field("nope").ok());
    printf("%s: %d failure(s)\n", failures ? "FAILED" : "ok", failures);
    return failures ? 1 : 0;
}
