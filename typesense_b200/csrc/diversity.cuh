// Diversity re-ranking on sm_90a: the maximal-marginal-relevance order of Index::populate_result_kvs (src/index.cpp:9016-9064)
// with the pair similarity of similarity_t::calculate (src/diversity.cpp).
//
// The reference picks K - 1 times; at each pick every unpicked entry takes the max of its similarity to EVERY entry picked so
// far (about K^3 / 6 pair lookups). A max does not depend on the order it is taken in, so max_sim[i] is kept per entry and
// updated once per pick against the last pick only: K^2 / 2 similarity evaluations, the same values. The pick itself is a
// block argmax of (mr, -position); the reference scans positions upward with a strict `>` against a running max that starts
// at lowest(), which is the same choice (the greatest mr above lowest(), the lowest position among equals).
//
// One CTA per query. Its workspace (below) holds each entry's max_sim, vector distance, sort values and facet rows sorted and
// de-duplicated (the std::set of the reference); it lives in shared memory when it fits, else in a per-call HBM slice sized
// from a counting pass (div_count_kernel) before the re-ranking kernel runs. The arithmetic is the reference's, in its types
// (float products, double sums / quotients) with explicitly rounded operations, so nothing is contracted into an FMA and the
// order is the reference's bit for bit. The functions marked TSDIV_HD compile with g++ too (tests/cpp/diversity_pairs.cpp).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "../../include/tsgpu.h"

#ifdef __CUDACC__
#include <cuda_runtime.h>
#define TSDIV_HD __host__ __device__ __forceinline__
#else
#define TSDIV_HD inline
#endif

namespace tsdiv {

constexpr uint32_t kThreads = 256;
constexpr uint32_t kNoPos = 0xFFFFFFFFu;
constexpr unsigned long long kInShared = ~0ull;           // ws_off of a query whose workspace is in shared memory
constexpr double kLowest = -1.7976931348623157e308;       // std::numeric_limits<double>::lowest()

// round-to-nearest operations, never fused
TSDIV_HD float fmul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
TSDIV_HD float fsub(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}
TSDIV_HD double dmul(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
TSDIV_HD double dadd(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
TSDIV_HD double dsub(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
TSDIV_HD double ddiv(double a, double b) {
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// One facet metric's contribution added to the running sum, as similarity_t::calculate adds it. a / b: the two documents' facet
// values, ascending and distinct; an empty row is a document the facet index does not hold (the metric is skipped).
TSDIV_HD double add_facet(double sim, uint32_t method, float weight, const uint32_t* a, uint32_t na, const uint32_t* b, uint32_t nb) {
    if(na == 0 || nb == 0) return sim;
    uint32_t i = 0, j = 0, inter = 0;
    while(i < na && j < nb) {
        const uint32_t x = a[i], y = b[j];
        if(x < y) i++;
        else if(y < x) j++;
        else { inter++; i++; j++; }
    }
    if(method == TSGPU_DIV_JACCARD)               // ((double) intersection_size / union_size) * metric.weight
        return dadd(sim, dmul(ddiv((double) inter, (double) (na + nb - inter)), (double) weight));
    if(method == TSGPU_DIV_EQUALITY) {            // sizes differ: skipped; else metric.weight * set_difference.empty(), a float product
        if(na != nb) return sim;
        return dadd(sim, (double) fmul(weight, inter == na ? 1.0f : 0.0f));
    }
    return sim;
}

// One sort-field metric: INT64_MIN is a document without a value; only equality contributes (`similarity += metric.weight`).
TSDIV_HD double add_sort(double sim, uint32_t method, float weight, int64_t a, int64_t b) {
    if(a == INT64_MIN || b == INT64_MIN) return sim;
    if(method == TSGPU_DIV_EQUALITY && a == b) return dadd(sim, (double) weight);
    return sim;
}

// std::max(max_similarity, sim)
TSDIV_HD double max_sim(double cur, double sim) { return cur < sim ? sim : cur; }

// mr = lambda * vector_distance (float) - (1 - lambda) (float) * max_similarity (double)
TSDIV_HD double mmr(float lambda, float vector_distance, double max_similarity) {
    const float left = fmul(lambda, vector_distance);
    const double right = dmul((double) fsub(1.0f, lambda), max_similarity);
    return dsub((double) left, right);
}

// does candidate (mr, pos) win over (best_mr, best_pos)? Only an mr above lowest() can be picked; kNoPos = nothing yet.
TSDIV_HD bool beats(double mr, uint32_t pos, double best_mr, uint32_t best_pos) {
    if(pos == kNoPos || !(mr > kLowest)) return false;
    return best_pos == kNoPos || mr > best_mr || (mr == best_mr && pos < best_pos);
}

// sorts v[0..n) ascending and drops repeats; returns the distinct count (rows are a handful of values: insertion sort)
TSDIV_HD uint32_t sort_unique(uint32_t* v, uint32_t n) {
    for(uint32_t i = 1; i < n; i++) {
        const uint32_t x = v[i];
        uint32_t j = i;
        while(j > 0 && v[j - 1] > x) { v[j] = v[j - 1]; j--; }
        v[j] = x;
    }
    uint32_t m = 0;
    for(uint32_t i = 0; i < n; i++) if(m == 0 || v[i] != v[m - 1]) v[m++] = v[i];
    return m;
}

// A query's workspace: K entries, F facet metrics, S sort metrics, T facet values (the entries' raw rows, all facet metrics).
struct Layout { size_t max_sim, sortv, vd, order, row_off, row_len, vals, picked, total; };
TSDIV_HD Layout layout(uint32_t K, uint32_t F, uint32_t S, unsigned long long T) {
    Layout L;
    size_t o = 0;
    L.max_sim = o; o += (size_t) 8 * K;
    L.sortv = o;   o += (size_t) 8 * S * K;
    L.vd = o;      o += (size_t) 4 * K;
    L.order = o;   o += (size_t) 4 * K;
    L.row_off = o; o += (size_t) 4 * F * K;
    L.row_len = o; o += (size_t) 4 * F * K;
    L.vals = o;    o += (size_t) 4 * T;
    L.picked = o;  o += K;
    L.total = (o + 15) & ~size_t(15);
    return L;
}

struct Metric {
    const unsigned long long* doc_off;     // facet metric: the facet's CSR; nullptr: sort metric
    const uint32_t* value_ids;
    const int64_t* sort_col;               // sort metric: the column
    uint32_t method;
    float weight;
    uint32_t slot;                         // index among the facet metrics / among the sort metrics
};

struct Params {
    Metric m[TSGPU_MAX_DIV_METRICS];
    uint32_t n_metrics, n_facet, n_sort, n_docs;
    const tsgpu_kv* kv;                    // [nq * stride]
    tsgpu_kv* out;                         // [nq * stride]
    uint32_t stride;
    const uint32_t* count;                 // [nq]
    const float* lambda;                   // [nq]
    unsigned long long* n_vals;            // [nq] raw facet values of the query's entries (div_count_kernel)
    const unsigned long long* ws_off;      // [nq] byte offset of the query's workspace in `scratch`, or kInShared
    unsigned char* scratch;
};

}  // namespace tsdiv

#if defined(__CUDACC__) && defined(TSDIV_KERNELS)
#include <cub/block/block_scan.cuh>

namespace tsdiv {

__device__ __forceinline__ uint32_t raw_len(const Metric& m, uint64_t key, uint32_t n_docs) {
    return key < n_docs ? (uint32_t) (m.doc_off[key + 1] - m.doc_off[key]) : 0u;
}

// n_vals[q] = facet values the query's entries hold over all facet metrics (before de-duplication): sizes the workspaces
__global__ void __launch_bounds__(kThreads) div_count_kernel(const __grid_constant__ Params P) {
    const uint32_t q = blockIdx.x, K = P.count[q];
    const tsgpu_kv* in = P.kv + (size_t) q * P.stride;
    unsigned long long n = 0;
    for(uint32_t e = threadIdx.x; e < K; e += kThreads) {
        const uint64_t key = in[e].key;
        for(uint32_t i = 0; i < P.n_metrics; i++) if(P.m[i].doc_off) n += raw_len(P.m[i], key, P.n_docs);
    }
    if(n) atomicAdd(P.n_vals + q, n);
}

__global__ void __launch_bounds__(kThreads, 6) div_mmr_kernel(const __grid_constant__ Params P) {
    extern __shared__ __align__(16) unsigned char smem[];
    using Scan = cub::BlockScan<unsigned long long, kThreads>;
    __shared__ typename Scan::TempStorage scan_tmp;
    __shared__ double w_mr[kThreads / 32];
    __shared__ uint32_t w_pos[kThreads / 32], w_first[kThreads / 32];
    __shared__ uint32_t s_last;
    const uint32_t q = blockIdx.x, K = P.count[q], tid = threadIdx.x;
    if(K == 0) return;
    const tsgpu_kv* in = P.kv + (size_t) q * P.stride;
    tsgpu_kv* out = P.out + (size_t) q * P.stride;
    if(K == 1) { if(tid == 0) out[0] = in[0]; return; }
    const uint32_t F = P.n_facet, S = P.n_sort;
    const Layout L = layout(K, F, S, P.n_vals[q]);
    unsigned char* ws = P.ws_off[q] == kInShared ? smem : P.scratch + P.ws_off[q];
    double* msim = reinterpret_cast<double*>(ws + L.max_sim);
    int64_t* sortv = reinterpret_cast<int64_t*>(ws + L.sortv);
    float* vd = reinterpret_cast<float*>(ws + L.vd);
    uint32_t* order = reinterpret_cast<uint32_t*>(ws + L.order);
    uint32_t* row_off = reinterpret_cast<uint32_t*>(ws + L.row_off);
    uint32_t* row_len = reinterpret_cast<uint32_t*>(ws + L.row_len);
    uint32_t* vals = reinterpret_cast<uint32_t*>(ws + L.vals);
    uint8_t* picked = ws + L.picked;

    // ---- gather: per entry its distance, sort values and facet rows (sorted, distinct), the rows packed in entry order
    unsigned long long base = 0;
    for(uint32_t c0 = 0; c0 < K; c0 += kThreads) {
        const uint32_t e = c0 + tid;
        uint64_t key = 0;
        unsigned long long len = 0;
        if(e < K) {
            key = in[e].key;
            vd[e] = in[e].vector_distance;
            msim[e] = kLowest;
            picked[e] = e == 0;
            for(uint32_t i = 0; i < P.n_metrics; i++) {
                const Metric& m = P.m[i];
                if(m.doc_off) len += raw_len(m, key, P.n_docs);
                else sortv[(size_t) m.slot * K + e] = key < P.n_docs ? m.sort_col[key] : INT64_MIN;
            }
        }
        unsigned long long off = 0, agg = 0;
        Scan(scan_tmp).ExclusiveSum(len, off, agg);
        if(e < K) {
            unsigned long long pos = base + off;
            for(uint32_t i = 0; i < P.n_metrics; i++) {
                const Metric& m = P.m[i];
                if(!m.doc_off) continue;
                const uint32_t n = raw_len(m, key, P.n_docs);
                const unsigned long long o0 = n ? m.doc_off[key] : 0;
                for(uint32_t j = 0; j < n; j++) vals[pos + j] = m.value_ids[o0 + j];
                row_off[(size_t) m.slot * K + e] = (uint32_t) pos;
                row_len[(size_t) m.slot * K + e] = sort_unique(vals + pos, n);
                pos += n;
            }
        }
        base += agg;
        __syncthreads();                  // scan_tmp is reused by the next chunk
    }
    if(tid == 0) order[0] = 0;
    const float lambda = P.lambda[q];
    uint32_t last = 0;
    __syncthreads();

    // ---- K - 1 picks
    for(uint32_t s = 1; s < K; s++) {
        double best_mr = 0;
        uint32_t best_pos = kNoPos, first = kNoPos;
        for(uint32_t e = tid; e < K; e += kThreads) {
            if(picked[e]) continue;
            if(first == kNoPos) first = e;
            double sim = 0;
            for(uint32_t i = 0; i < P.n_metrics; i++) {
                const Metric& m = P.m[i];
                if(m.doc_off) {
                    const size_t a = (size_t) m.slot * K + e, b = (size_t) m.slot * K + last;
                    sim = add_facet(sim, m.method, m.weight, vals + row_off[a], row_len[a], vals + row_off[b], row_len[b]);
                } else {
                    sim = add_sort(sim, m.method, m.weight, sortv[(size_t) m.slot * K + e], sortv[(size_t) m.slot * K + last]);
                }
            }
            const double ms = max_sim(msim[e], sim);
            msim[e] = ms;
            const double mr = mmr(lambda, vd[e], ms);
            if(beats(mr, e, best_mr, best_pos)) { best_mr = mr; best_pos = e; }
        }
        for(int o = 16; o > 0; o >>= 1) {
            const double omr = __shfl_xor_sync(0xffffffffu, best_mr, o);
            const uint32_t opos = __shfl_xor_sync(0xffffffffu, best_pos, o);
            const uint32_t ofirst = __shfl_xor_sync(0xffffffffu, first, o);
            if(beats(omr, opos, best_mr, best_pos)) { best_mr = omr; best_pos = opos; }
            first = min(first, ofirst);
        }
        if((tid & 31) == 0) { w_mr[tid >> 5] = best_mr; w_pos[tid >> 5] = best_pos; w_first[tid >> 5] = first; }
        __syncthreads();
        if(tid == 0) {
            for(uint32_t w = 1; w < kThreads / 32; w++) {
                if(beats(w_mr[w], w_pos[w], best_mr, best_pos)) { best_mr = w_mr[w]; best_pos = w_pos[w]; }
                first = min(first, w_first[w]);
            }
            // nothing above lowest() (a NaN or -inf mr everywhere): the reference has no pick there; take the first unpicked
            const uint32_t p = best_pos != kNoPos ? best_pos : first;
            picked[p] = 1;
            order[s] = p;
            s_last = p;
        }
        __syncthreads();
        last = s_last;
    }
    for(uint32_t s = tid; s < K; s += kThreads) out[s] = in[order[s]];
}

}  // namespace tsdiv
#endif
