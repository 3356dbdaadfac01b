// TEST INFRASTRUCTURE — the oracle-backed test double of the C-ABI (tsgpu_oracle_double_mirror.cpp, included whole: the base double
// and the mirror maintenance calls) plus tsgpu_diversify_batch, answered query by query by tso_diversify (tso_diversify.cpp, the
// transcription of the reference's loop); div_k2_reference.cpp rides along for the tests. It checks its arguments as the library does. Built as one library (or linked into one
// program) so that the Python and C++ sides of the diversity tests run on a machine without a GPU. Never part of the product.
#include "tsgpu_oracle_double_mirror.cpp"
#include "tso_diversify.cpp"
#include "div_k2_reference.cpp"

extern "C" {

tsgpu_status tsgpu_diversify_batch(tsgpu_index* idx, const tsgpu_div_metric* metrics, uint32_t n_metrics, uint32_t nq,
                                   const float* lambda, const tsgpu_kv* kv, uint32_t kv_stride, const uint32_t* count,
                                   tsgpu_kv* out_kv) {
    Double* d = D(idx);
    if(n_metrics > TSGPU_MAX_DIV_METRICS) { g_err = "too many diversity metrics"; return TSGPU_ERR_CAPACITY; }
    if(n_metrics == 0) { g_err = "no diversity metric"; return TSGPU_ERR_INVALID; }
    if(!metrics || (nq && (!lambda || !count))) { g_err = "null argument"; return TSGPU_ERR_INVALID; }
    uint64_t n_rec = 0;
    for(uint32_t q = 0; q < nq; q++) {
        if(count[q] > kv_stride) { g_err = "count exceeds kv_stride"; return TSGPU_ERR_INVALID; }
        if(!(lambda[q] >= 0.0f && lambda[q] <= 1.0f)) { g_err = "lambda must be in [0, 1]"; return TSGPU_ERR_INVALID; }
        n_rec += count[q];
    }
    if(n_rec && (!kv || !out_kv)) { g_err = "null argument"; return TSGPU_ERR_INVALID; }
    std::vector<tso_div_metric> m(n_metrics);
    for(uint32_t i = 0; i < n_metrics; i++) {
        const tsgpu_div_metric& a = metrics[i];
        if(a.method != TSGPU_DIV_EQUALITY && a.method != TSGPU_DIV_JACCARD) { g_err = "unknown diversity method"; return TSGPU_ERR_INVALID; }
        m[i] = tso_div_metric{nullptr, nullptr, nullptr, a.method, a.weight};
        if(a.facet != TSGPU_NO_LIST) {
            if(a.facet >= g_facets.size() || g_facet_owner[a.facet] != idx) { g_err = "facet id out of range"; return TSGPU_ERR_INVALID; }
            m[i].doc_off = g_facets[a.facet]->off.data();
            m[i].value_ids = g_facets[a.facet]->vals.data();
        } else {
            if(a.sort_col < 0 || (size_t) a.sort_col >= d->cols.size()) { g_err = "sort column out of range"; return TSGPU_ERR_INVALID; }
            m[i].sort_col = d->cols[a.sort_col]->data();
        }
    }
    for(uint32_t q = 0; q < nq; q++)
        tso_diversify(d->n_docs, m.data(), n_metrics, lambda[q], reinterpret_cast<const tso_kv*>(kv) + (size_t) q * kv_stride, count[q],
                      reinterpret_cast<tso_kv*>(out_kv) + (size_t) q * kv_stride);
    return TSGPU_OK;
}

}  // extern "C"
