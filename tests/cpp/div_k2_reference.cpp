// TEST INFRASTRUCTURE — the K^2 formulation of the diversity re-ranking, serial, from the device's own functions
// (typesense_b200/csrc/diversity.cuh compiled by g++): max_sim per entry updated against the last pick, the pick by (mr, -position).
// The literal transcription (tso_diversify.cpp) compares K^3 / 6 pairs through a map; this answers a Topster of thousands of
// records in a blink, so the device's largest lists are checked against it. tests/test_diversity.py shows it equal to the
// transcription on seeded inputs. Included by tsgpu_oracle_double_diversity.cpp; never part of the product.
#include <vector>

#include "../../typesense_b200/csrc/diversity.cuh"

extern "C" void div_k2_order(uint32_t n_docs, const tso_div_metric* metrics, uint32_t n_metrics, float lambda, const tso_kv* kv, uint32_t K,
                             uint32_t* order) {
    if(K == 0) return;
    std::vector<std::vector<std::vector<uint32_t>>> rows(n_metrics, std::vector<std::vector<uint32_t>>(K));
    std::vector<std::vector<int64_t>> sortv(n_metrics, std::vector<int64_t>(K, INT64_MIN));
    for(uint32_t i = 0; i < n_metrics; i++) for(uint32_t e = 0; e < K; e++) {
        const uint64_t key = kv[e].key;
        if(key >= n_docs) continue;
        if(metrics[i].doc_off) {
            auto& r = rows[i][e];
            r.assign(metrics[i].value_ids + metrics[i].doc_off[key], metrics[i].value_ids + metrics[i].doc_off[key + 1]);
            r.resize(tsdiv::sort_unique(r.data(), (uint32_t) r.size()));
        } else sortv[i][e] = metrics[i].sort_col[key];
    }
    std::vector<double> msim(K, tsdiv::kLowest);
    std::vector<char> picked(K, 0);
    picked[0] = 1; order[0] = 0;
    uint32_t last = 0;
    for(uint32_t s = 1; s < K; s++) {
        double best_mr = 0;
        uint32_t best = tsdiv::kNoPos, first = tsdiv::kNoPos;
        for(uint32_t e = 0; e < K; e++) {
            if(picked[e]) continue;
            if(first == tsdiv::kNoPos) first = e;
            double sim = 0;
            for(uint32_t i = 0; i < n_metrics; i++) {
                const tso_div_metric& m = metrics[i];
                if(m.doc_off) sim = tsdiv::add_facet(sim, m.method, m.weight, rows[i][e].data(), (uint32_t) rows[i][e].size(), rows[i][last].data(), (uint32_t) rows[i][last].size());
                else sim = tsdiv::add_sort(sim, m.method, m.weight, sortv[i][e], sortv[i][last]);
            }
            msim[e] = tsdiv::max_sim(msim[e], sim);
            const double mr = tsdiv::mmr(lambda, kv[e].vector_distance, msim[e]);
            if(tsdiv::beats(mr, e, best_mr, best)) { best_mr = mr; best = e; }
        }
        last = best != tsdiv::kNoPos ? best : first;
        picked[last] = 1;
        order[s] = last;
    }
}
