// The device's pair similarity and MMR expression (typesense_b200/csrc/diversity.cuh, compiled here by g++) against the oracle's
// transcription of similarity_t::calculate (tso_div_similarity), pair for pair and bit for bit, on seeded random facet rows (repeated
// values, empty rows, single values) and sort columns (missing values), with several metric lists and weights.
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "../../typesense_b200/csrc/diversity.cuh"

extern "C" {
typedef struct { const uint64_t* doc_off; const uint32_t* value_ids; const int64_t* sort_col; uint32_t method; float weight; } tso_div_metric;
double tso_div_similarity(uint32_t n_docs, const tso_div_metric* metrics, uint32_t n_metrics, uint32_t seq_id_i, uint32_t seq_id_j);
}

int main() {
    const uint32_t n = 160;
    std::mt19937 rng(5);
    std::vector<uint64_t> off_a{0}, off_b{0};
    std::vector<uint32_t> va, vb;
    std::vector<int64_t> col(n);
    for(uint32_t d = 0; d < n; d++) {
        const uint32_t k = rng() % 6;                      // 0..5 values from 7: repeats and empty rows
        for(uint32_t i = 0; i < k; i++) va.push_back(rng() % 7);
        off_a.push_back(va.size());
        if(rng() % 5) vb.push_back(rng() % 4);             // a single-value facet, some documents without one
        off_b.push_back(vb.size());
        col[d] = rng() % 4 == 0 ? INT64_MIN : (int64_t) (rng() % 3);
    }
    const float weights[] = {1.0f, 0.1f, 0.6f, 0.3f};
    uint64_t pairs = 0, mismatches = 0;
    for(int variant = 0; variant < 8; variant++) {
        const float w0 = weights[variant % 4], w1 = weights[(variant + 1) % 4], w2 = weights[(variant + 2) % 4];
        const uint32_t m0 = variant & 1 ? TSGPU_DIV_EQUALITY : TSGPU_DIV_JACCARD, m1 = variant & 2 ? TSGPU_DIV_EQUALITY : TSGPU_DIV_JACCARD;
        const uint32_t m2 = variant & 4 ? TSGPU_DIV_EQUALITY : TSGPU_DIV_JACCARD;
        const tso_div_metric om[3] = {{off_a.data(), va.data(), nullptr, m0, w0}, {nullptr, nullptr, col.data(), m2, w2}, {off_b.data(), vb.data(), nullptr, m1, w1}};
        // the rows as the device gathers them: sorted and de-duplicated
        std::vector<std::vector<uint32_t>> ra(n), rb(n);
        for(uint32_t d = 0; d < n; d++) {
            ra[d].assign(va.begin() + off_a[d], va.begin() + off_a[d + 1]);
            ra[d].resize(tsdiv::sort_unique(ra[d].data(), (uint32_t) ra[d].size()));
            rb[d].assign(vb.begin() + off_b[d], vb.begin() + off_b[d + 1]);
            rb[d].resize(tsdiv::sort_unique(rb[d].data(), (uint32_t) rb[d].size()));
        }
        for(uint32_t i = 0; i < n; i++) for(uint32_t j = i + 1; j < n; j++) {
            double s = 0;
            s = tsdiv::add_facet(s, m0, w0, ra[i].data(), (uint32_t) ra[i].size(), ra[j].data(), (uint32_t) ra[j].size());
            s = tsdiv::add_sort(s, m2, w2, col[i], col[j]);
            s = tsdiv::add_facet(s, m1, w1, rb[i].data(), (uint32_t) rb[i].size(), rb[j].data(), (uint32_t) rb[j].size());
            const double o = tso_div_similarity(n, om, 3, i, j);
            pairs++;
            if(memcmp(&s, &o, 8) != 0) { if(mismatches++ < 5) printf("pair (%u, %u) variant %d: %.17g vs oracle %.17g\n", i, j, variant, s, o); }
            // mmr as populate_result_kvs types it, at the lambdas a request can carry
            for(float lambda: {0.0f, 0.3f, 0.5f, 1.0f}) for(float vd: {-1.0f, 0.25f, 0.7134f}) {
                const float left = lambda * vd;
                const double want = left - (1 - lambda) * o;
                const double got = tsdiv::mmr(lambda, vd, s);
                if(memcmp(&want, &got, 8) != 0 && mismatches++ < 5) printf("mmr differs: lambda %g vd %g\n", lambda, vd);
            }
        }
    }
    printf("pairs %llu mismatches %llu\n", (unsigned long long) pairs, (unsigned long long) mismatches);
    return mismatches ? 1 : 0;
}
