// TEST INFRASTRUCTURE — the oracle of the diversity re-ranking: a literal transcription of the diversity branch of
// Index::populate_result_kvs (src/index.cpp:9016-9064) and of similarity_t::calculate (src/diversity.cpp), the cubic loop with its
// pair cache, over the data the mirror holds instead of facet_index_t / sort_index:
//   - facet_index_v4->get_facet_hash_index(field)  -> a facet's CSR (doc_off [n_docs + 1], value_ids); facet_it.skip_to(seq_id)
//     lands on the document when its row is not empty, and posting_list_t::get_offsets gives the row's values;
//   - sort_index.at(field)->find(seq_id)            -> a sort column [n_docs]; INT64_MIN (or a seq_id >= n_docs) is no entry.
// Types are the reference's: `lambda * vector_distance` is a float product, `(1 - lambda) * max_similarity` a double one.
// Compiled with -ffp-contract=off. Included by tsgpu_oracle_double_diversity.cpp; never part of the product.
#include <algorithm>
#include <cstdint>
#include <iterator>
#include <limits>
#include <map>
#include <set>
#include <utility>
#include <vector>

#include "../../oracle/ts_oracle.h"

extern "C" {
typedef struct {
    const uint64_t* doc_off;      // facet metric: the facet's CSR; NULL: sort metric
    const uint32_t* value_ids;
    const int64_t* sort_col;      // sort metric: [n_docs], INT64_MIN = no value
    uint32_t method;              // diversity_t::similarity_methods: 0 equality, 1 jaccard
    float weight;
} tso_div_metric;
}

namespace tso_div {

enum similarity_methods : int { equality, jaccard };

struct view_t {
    uint32_t n_docs;
    const tso_div_metric* metrics;
    uint32_t n_metrics;
    // facet_it.skip_to(seq_id); facet_it.valid() && facet_it.id() == seq_id
    bool facet_has(const tso_div_metric& m, uint32_t seq_id) const { return seq_id < n_docs && m.doc_off[seq_id + 1] > m.doc_off[seq_id]; }
    std::vector<uint32_t> facet_offsets(const tso_div_metric& m, uint32_t seq_id) const {
        return std::vector<uint32_t>(m.value_ids + m.doc_off[seq_id], m.value_ids + m.doc_off[seq_id + 1]);
    }
    bool sort_find(const tso_div_metric& m, uint32_t seq_id, int64_t& v) const {
        if(seq_id >= n_docs || m.sort_col[seq_id] == INT64_MIN) return false;
        v = m.sort_col[seq_id];
        return true;
    }
};

struct similarity_t {
    std::map<std::pair<uint32_t, uint32_t>, double> similarity_map{};

    double calculate(uint32_t seq_id_i, uint32_t seq_id_j, const view_t& diversity, bool use_cache = true) {
        // Since similarity(i, j) == similarity(j, i), we use {lower_seq_id, higher_seq_id} as the similarity_map key.
        if (seq_id_j < seq_id_i) {
            std::swap(seq_id_i, seq_id_j);
        }
        if(use_cache) {
            auto sim_it = similarity_map.find(std::make_pair(seq_id_i, seq_id_j));
            if (sim_it != similarity_map.end()) {
                return sim_it->second;
            }
        }

        double similarity = 0;
        for (uint32_t mi = 0; mi < diversity.n_metrics; mi++) {
            const tso_div_metric& metric = diversity.metrics[mi];

            if (metric.doc_off) {
                if (!diversity.facet_has(metric, seq_id_i)) {
                    continue;
                }
                std::set<uint32_t> i_facet_hashes;
                {
                    std::vector<uint32_t> facet_hashes = diversity.facet_offsets(metric, seq_id_i);
                    i_facet_hashes.insert(facet_hashes.begin(), facet_hashes.end());
                }

                if (!diversity.facet_has(metric, seq_id_j)) {
                    continue;
                }
                std::set<uint32_t> j_facet_hashes;
                {
                    std::vector<uint32_t> facet_hashes = diversity.facet_offsets(metric, seq_id_j);
                    j_facet_hashes.insert(facet_hashes.begin(), facet_hashes.end());
                }

                if ((int) metric.method == jaccard) {
                    if (i_facet_hashes.empty() && j_facet_hashes.empty()) {
                        continue;
                    }
                    std::vector<uint32_t> out{};
                    std::set_intersection(i_facet_hashes.begin(), i_facet_hashes.end(),
                                          j_facet_hashes.begin(), j_facet_hashes.end(),
                                          std::back_inserter(out));
                    const auto intersection_size = out.size();
                    out.clear();

                    std::set_union(i_facet_hashes.begin(), i_facet_hashes.end(),
                                   j_facet_hashes.begin(), j_facet_hashes.end(),
                                   std::back_inserter(out));
                    const auto union_size = out.size();

                    similarity += ((double) intersection_size/union_size) * metric.weight;
                } else if ((int) metric.method == equality) {
                    if (i_facet_hashes.size() != j_facet_hashes.size()) {
                        continue;
                    }
                    std::vector<uint32_t> out{};
                    std::set_difference(i_facet_hashes.begin(), i_facet_hashes.end(),
                                        j_facet_hashes.begin(), j_facet_hashes.end(),
                                        std::back_inserter(out));
                    similarity += metric.weight * out.empty();
                }
            }

            else {
                int64_t i_value = 0, j_value = 0;
                if (!diversity.sort_find(metric, seq_id_i, i_value)) {
                    continue;
                }
                if (!diversity.sort_find(metric, seq_id_j, j_value)) {
                    continue;
                }
                if ((int) metric.method == equality && i_value == j_value) {
                    similarity += metric.weight;
                }
            }
        }

        if(use_cache) similarity_map[std::make_pair(seq_id_i, seq_id_j)] = similarity;
        return similarity;
    }
};

}  // namespace tso_div

extern "C" {

// similarity_t::calculate for one pair, without the cache
double tso_div_similarity(uint32_t n_docs, const tso_div_metric* metrics, uint32_t n_metrics, uint32_t seq_id_i, uint32_t seq_id_j) {
    tso_div::similarity_t similarity;
    const tso_div::view_t diversity{n_docs, metrics, n_metrics};
    return similarity.calculate(seq_id_i, seq_id_j, diversity, false);
}

// the diversity branch of Index::populate_result_kvs over one sorted Topster of `size` records: out[0 .. size) in MMR order
void tso_diversify(uint32_t n_docs, const tso_div_metric* metrics, uint32_t n_metrics, float lambda, const tso_kv* topster, uint32_t size,
                   tso_kv* out) {
    if(size == 0) return;
    const tso_div::view_t diversity{n_docs, metrics, n_metrics};
    tso_div::similarity_t similarity;
    std::vector<const tso_kv*> result_kvs;
    result_kvs.push_back(&topster[0]);
    std::set<uint32_t> processed_seq_ids{(uint32_t) topster[0].key};
    while (result_kvs.size() < size) {
        auto mmr = std::numeric_limits<double>::lowest();
        const tso_kv* max_kv = nullptr;

        for (uint32_t i = 1; i < size; i++) {
            auto kv_i = &topster[i];
            const auto& seq_id_i = (uint32_t) kv_i->key;
            if (processed_seq_ids.count(seq_id_i) > 0) {
                continue;
            }

            auto left = lambda * kv_i->vector_distance;
            auto max_similarity = std::numeric_limits<double>::lowest();
            for (const auto& kv_j: result_kvs) {
                const auto& seq_id_j = (uint32_t) kv_j->key;
                auto sim = similarity.calculate(seq_id_i, seq_id_j, diversity);
                max_similarity = std::max(max_similarity, sim);
            }

            auto right = (1 - lambda) * max_similarity;
            auto mr = left - right;
            if (mr > mmr) {
                max_kv = kv_i;
                mmr = mr;
            }
        }

        // The reference dereferences max_kv here. It stays null only when no mr is above lowest() (NaN or -inf everywhere,
        // which no finite distance produces); the first unprocessed record is taken then, as the device does.
        if (!max_kv) {
            for (uint32_t i = 1; i < size && !max_kv; i++) if (processed_seq_ids.count((uint32_t) topster[i].key) == 0) max_kv = &topster[i];
        }
        processed_seq_ids.insert((uint32_t) max_kv->key);
        result_kvs.push_back(max_kv);
    }
    std::vector<tso_kv> tmp;                     // `out` may be `topster`
    for (auto* kv: result_kvs) tmp.push_back(*kv);
    std::copy(tmp.begin(), tmp.end(), out);
}

}  // extern "C"
