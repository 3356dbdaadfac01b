// Deep vector assembly and deep hybrid fusion: the vector and hybrid calls for queries whose Topster is larger than
// TSGPU_MAX_TOPK (TSGPU_VEC_DEEP_TOPSTER with TSGPU_QFLAG_DEEP_TOPSTER).
//
// vec_assemble_kernel and hybrid_fuse_kernel (fuse_kernels.cuh) keep the whole Topster in shared memory, so they stop at 1024.
// The kernels below compute the same answer at any K:
//   deep vector assembly (src/index.cpp:3682-3732): every kNN / flat result passing distance_threshold becomes a DeepEntry
//       (deep_topster.cuh's layout; the vector distance rides in the two 16-bit tail fields, which the KV order ignores), the
//       entries are radix-sorted by that order, and the first min(K, n, kv_stride) are written as records;
//   deep hybrid fusion (src/index.cpp:4036-4221), one CTA per query over a workspace that is in shared memory when it fits and
//       in a slice of an HBM buffer otherwise. Everything that does not depend on the order of the reference's loop runs in
//       parallel: the text ranks (two block scans), the threshold cut of the kNN list, the per-result filter bit, sort scores,
//       keyword-match test and all_result_ids OR, and each vector result's keyword Topster slot (binary search over the keyword
//       keys sorted by seq_id). What remains serial is the replay of the loop itself: a rewrite of the slot's scores, or
//       Topster::add on the array as it is after sort() (include/topster.h:321-466), with a per-slot bit that tells whether the
//       keyword entry is still in the Topster's map after earlier evictions. compute_aux_scores' two ranks come from two sorts
//       instead of the O(n^2) counts, and the final sort is a bitonic sort by the KV order.
// The kernels are compiled in deep_fuse.cu (TSDF_KERNELS), so the kernels of tsgpu.cu keep their code generation; the host side
// is deep_fuse_host.inc.
#pragma once
#include "fuse_kernels.cuh"
#include "deep_topster.cuh"
#ifdef TSDF_KERNELS
#include <cub/block/block_scan.cuh>
#endif

namespace tsdf {

using namespace tsk;

constexpr uint32_t kThreads = 256;
constexpr unsigned long long kInShared = ~0ull;     // ws_off of a query whose workspace is in shared memory
constexpr uint32_t kNoSlot = 0xFFFFFFFFu;

// ---- deep vector assembly
struct VecDeepParams {
    const QDesc* qd;
    const float* res_dist; const uint32_t* res_ids; const uint32_t* res_n; uint32_t res_stride;
    const float* flat_dist; const uint32_t* flat_ids; const unsigned long long* res_off; const uint8_t* q_is_flat;
    tsf::VecParams vp;
    const uint32_t* deep_q;               // [n_deep] query of each deep slot
    const unsigned long long* ent_off;    // [n_deep] slice of the deep slot in `ent`
    DeepEntry* ent;
    unsigned long long* ent_n;            // [n_deep] entries kept (zeroed before the pack kernel) = found
};

// ---- deep hybrid fusion
struct HybridDeepParams {
    tsf::HybridParams hp;                 // as for hybrid_fuse_kernel (qd: the batch's real query descriptors)
    const uint32_t* deep_q;               // [n_deep]
    const uint32_t* nv_cap;               // [n_deep] vector results the workspace holds (k, or the flat id count)
    const unsigned long long* ws_off;     // [n_deep] byte offset in `ws`, or kInShared
    unsigned char* ws;
    unsigned long long* timers;           // [n_deep * 5] %globaltimer at the phase boundaries (prep | replay | rerank | sort)
};

// Workspace of one deep query: K Topster slots, NV vector results.
struct HybridWs {
    size_t o_data, o_kvs, o_key, o_slot, o_inmap, o_vid, o_vdist, o_vrank, o_vsc, o_vslot, o_vmsi, o_vflag, bytes;
};
__host__ __device__ inline uint32_t pow2_at_least(uint32_t v) { uint32_t p = 1; while(p < v) p <<= 1; return p; }
__host__ __device__ inline HybridWs hybrid_ws_layout(uint32_t K, uint32_t NV) {
    HybridWs w;
    const size_t PK = pow2_at_least(K), PV = pow2_at_least(NV);
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off = (off + bytes + 15) & ~size_t(15); return o; };
    w.o_data = take((size_t) K * sizeof(KVOut));
    w.o_vsc = take(PV * 24);
    w.o_kvs = take(PK * 4);               // heap position -> slot; the final sort's index array
    w.o_key = take(PK * 4);               // keyword keys sorted by seq_id; rerank: index array
    w.o_slot = take(PK * 4);              // their slots; text-rank increments; rerank: keyword ranks
    w.o_inmap = take(K);
    w.o_vid = take(PV * 4); w.o_vdist = take(PV * 4); w.o_vrank = take(PV * 4); w.o_vslot = take(PV * 4);
    w.o_vmsi = take(PV); w.o_vflag = take(PV);
    w.bytes = off;
    return w;
}

#ifdef TSDF_KERNELS
__device__ __forceinline__ unsigned long long global_ns() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }

__device__ __forceinline__ void vd_store(DeepEntry& e, float v) { const uint32_t b = __float_as_uint(v); e.cmb = (uint16_t) (b & 0xFFFFu); e.pad = (uint16_t) (b >> 16); }
__device__ __forceinline__ float vd_load(const DeepEntry& e) { return __uint_as_float((uint32_t) e.cmb | ((uint32_t) e.pad << 16)); }

// grid (x: result tiles, y: deep slot). Result -> DeepEntry as vec_assemble_kernel computes it (src/index.cpp:3699-3712).
__global__ void __launch_bounds__(256)
vec_deep_pack_kernel(const __grid_constant__ VecDeepParams P) {
    const uint32_t d = blockIdx.y, q = P.deep_q[d];
    const QDesc& qd = P.qd[q];
    SortSpec SS;
    for(int i = 0; i < 3; i++) { SS.type[i] = qd.sort_type[i]; SS.order[i] = qd.sort_order[i]; SS.missing_first[i] = qd.missing_first[i]; SS.col[i] = qd.sort_col[i]; }
    const bool flat = P.q_is_flat && P.q_is_flat[q];
    const float* rd; const uint32_t* ri; unsigned long long n_in;
    if(flat) { rd = P.flat_dist + P.res_off[q]; ri = P.flat_ids + P.res_off[q]; n_in = P.res_off[q + 1] - P.res_off[q]; }
    else { rd = P.res_dist + (size_t) q * P.res_stride; ri = P.res_ids + (size_t) q * P.res_stride; n_in = P.res_n[q]; }
    for(unsigned long long i = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; i < n_in; i += (unsigned long long) gridDim.x * blockDim.x) {
        const uint32_t id = ri[i];
        const float d0 = rd[i];
        const float vds = (P.vp.metric == 1) ? fabsf(d0) : d0;
        if(vds > P.vp.distance_threshold) continue;
        int64_t sc[3];
        compute_sort_scores(SS, id, 0, vds, sc);
        DeepEntry e;
        e.s0 = sc[0]; e.s1 = sc[1]; e.s2 = sc[2]; e.key = id;
        vd_store(e, vds);
        const unsigned long long pos = atomicAdd(P.ent_n + d, 1ull);
        P.ent[P.ent_off[d] + pos] = e;
    }
}

// First n_out entries of the sorted slice -> records of query q (vec_assemble_kernel's record layout).
__global__ void __launch_bounds__(256)
vec_deep_write_kernel(const DeepEntry* __restrict__ in, uint32_t n_out, unsigned long long found, const QDesc* __restrict__ qds, uint32_t q,
                      KVOut* __restrict__ out_kv, uint32_t kv_stride, uint32_t* __restrict__ out_count, uint32_t* __restrict__ out_found) {
    const QDesc& qd = qds[q];
    int msi = -1;
    for(int i = 0; i < 3; i++) if(qd.sort_type[i] == 1) msi = i;
    for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_out; i += gridDim.x * blockDim.x) {
        const DeepEntry e = in[i];
        KVOut kv;
        kv.key = e.key; kv.distinct_key = e.key;
        kv.scores[0] = e.s0; kv.scores[1] = e.s1; kv.scores[2] = e.s2;
        kv.text_match_score = msi >= 0 ? kv.scores[msi] : 0;
        kv.vector_distance = vd_load(e);
        kv.match_score_index = (int8_t) msi; kv.pad0 = 0; kv.query_index = 0;
        out_kv[(size_t) q * kv_stride + i] = kv;
    }
    if(blockIdx.x == 0 && threadIdx.x == 0) { out_count[q] = n_out; out_found[q] = (uint32_t) found; }
}

// Bitonic sort of a[0..P2) (P2 a power of two) into `before` order; kNone entries go last. `before` must be a strict total
// order on the live entries, so the result does not depend on the network.
template <class Before>
__device__ void cta_bitonic(uint32_t* a, uint32_t P2, Before before) {
    for(uint32_t k = 2; k <= P2; k <<= 1) {
        for(uint32_t j = k >> 1; j > 0; j >>= 1) {
            for(uint32_t t = threadIdx.x; t < (P2 >> 1); t += blockDim.x) {
                const uint32_t i = ((t & ~(j - 1)) << 1) | (t & (j - 1)), p = i + j;
                const uint32_t x = a[i], y = a[p];
                const bool y_first = y != kNone && (x == kNone || before(y, x));
                const bool x_first = x != kNone && (y == kNone || before(x, y));
                if((i & k) == 0 ? y_first : x_first) { a[i] = y; a[p] = x; }
            }
            __syncthreads();
        }
    }
}

struct MaxI64 { __device__ long long operator()(long long a, long long b) const { return a > b ? a : b; } };

__global__ void __launch_bounds__(kThreads)
hybrid_deep_kernel(const __grid_constant__ HybridDeepParams D) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    using Scan = cub::BlockScan<long long, kThreads>;
    __shared__ typename Scan::TempStorage s_scan;
    __shared__ long long s_carry;
    __shared__ uint32_t s_size, s_vec_new;
    const tsf::HybridParams& P = D.hp;
    const uint32_t d = blockIdx.x, q = D.deep_q[d], tid = threadIdx.x;
    const QDesc qd = P.qd[q];
    const uint32_t K = qd.topk, NV = D.nv_cap[d];
    unsigned char* ws = D.ws_off[d] == kInShared ? smem_raw : D.ws + D.ws_off[d];
    const HybridWs W = hybrid_ws_layout(K, NV);
    KVOut* data = reinterpret_cast<KVOut*>(ws + W.o_data);
    uint32_t* kvs = reinterpret_cast<uint32_t*>(ws + W.o_kvs);
    uint32_t* kw_key = reinterpret_cast<uint32_t*>(ws + W.o_key);
    uint32_t* kw_slot = reinterpret_cast<uint32_t*>(ws + W.o_slot);
    uint8_t* inmap = ws + W.o_inmap;
    uint32_t* v_id = reinterpret_cast<uint32_t*>(ws + W.o_vid);
    float* v_dist = reinterpret_cast<float*>(ws + W.o_vdist);
    uint32_t* v_rank = reinterpret_cast<uint32_t*>(ws + W.o_vrank);
    int64_t* v_sc = reinterpret_cast<int64_t*>(ws + W.o_vsc);
    uint32_t* v_slot = reinterpret_cast<uint32_t*>(ws + W.o_vslot);
    int8_t* v_msi = reinterpret_cast<int8_t*>(ws + W.o_vmsi);
    uint8_t* v_flag = ws + W.o_vflag;
    const uint32_t PK = pow2_at_least(K), PV = pow2_at_least(NV);
    unsigned long long* tm = D.timers + (size_t) d * 5;
    if(tid == 0) tm[0] = global_ns();

    SortSpec SS;
    for(int i = 0; i < 3; i++) { SS.type[i] = qd.sort_type[i]; SS.order[i] = qd.sort_order[i]; SS.missing_first[i] = qd.missing_first[i]; SS.col[i] = qd.sort_col[i]; }
    const float VECTOR_SEARCH_WEIGHT = P.vp.alpha;
    const float TEXT_MATCH_WEIGHT = (float) (1.0 - (double) VECTOR_SEARCH_WEIGHT);

    // ---- keyword Topster after topster->sort(): slot i at heap position i, every slot in the map
    const uint32_t n_kw = P.kw_count[q];
    for(uint32_t i = tid; i < n_kw; i += kThreads) { data[i] = P.kw_kv[(size_t) q * P.kw_stride + i]; kvs[i] = i; inmap[i] = 1; }
    if(tid == 0) s_carry = -1;
    __syncthreads();

    // ---- text ranks (src/index.cpp:4094-4112): the rank grows when a valid entry's score is below the previous valid one's.
    // Scan 1 (max): the previous valid position of every entry -> increment flags in kw_slot. Scan 2 (sum): the ranks.
    for(uint32_t base = 0; base < n_kw; base += kThreads) {
        const uint32_t i = base + tid;
        bool valid = false;
        if(i < n_kw) { const int m = data[i].match_score_index; valid = m >= 0 && m <= 2; }
        long long prev, agg;
        Scan(s_scan).ExclusiveScan(valid ? (long long) i : -1ll, prev, -1ll, MaxI64{}, agg);
        const long long carry = s_carry;
        prev = prev > carry ? prev : carry;
        if(i < n_kw) {
            uint32_t inc = 0;
            if(valid) {
                const int64_t last = prev >= 0 ? data[prev].scores[data[prev].match_score_index] : INT64_MAX;
                inc = data[i].scores[data[i].match_score_index] < last ? 1u : 0u;
            }
            kw_slot[i] = inc;
        }
        __syncthreads();
        if(tid == 0) s_carry = agg > carry ? agg : carry;
        __syncthreads();
    }
    if(tid == 0) s_carry = 0;
    __syncthreads();
    for(uint32_t base = 0; base < n_kw; base += kThreads) {
        const uint32_t i = base + tid;
        long long rank, agg;
        Scan(s_scan).InclusiveSum(i < n_kw ? (long long) kw_slot[i] : 0ll, rank, agg);
        rank += s_carry;
        if(i < n_kw) {
            KVOut& r = data[i];
            const int m = r.match_score_index;
            if(m >= 0 && m <= 2) {
                r.text_match_score = r.scores[m];
                r.scores[m] = float_to_int64(__double2float_rn((1.0 / (double) rank) * (double) TEXT_MATCH_WEIGHT));
            }
        }
        __syncthreads();
        if(tid == 0) s_carry += agg;
        __syncthreads();
    }

    // ---- vector results: rank = position in the distance-ordered list; iteration order = ascending seq_id (kNN) or the
    // flat path's id order
    const bool flat = P.q_is_flat && P.q_is_flat[q];
    uint32_t n_v;
    if(flat) {
        const float* rd = P.flat_dist + P.res_off[q]; const uint32_t* ri = P.flat_ids + P.res_off[q];
        n_v = (uint32_t) (P.res_off[q + 1] - P.res_off[q]);
        for(uint32_t i = tid; i < n_v; i += kThreads) { v_id[i] = ri[i]; v_dist[i] = rd[i]; v_rank[i] = i; }
    } else {
        // drop > distance_threshold (process_results_hnsw_index, :3419-3428), keeping the (distance, seq_id) order
        const float* rd = P.res_dist + (size_t) q * P.res_stride; const uint32_t* ri = P.res_ids + (size_t) q * P.res_stride;
        const uint32_t n_raw = P.res_n[q];
        if(tid == 0) s_carry = 0;
        __syncthreads();
        for(uint32_t base = 0; base < n_raw; base += kThreads) {
            const uint32_t i = base + tid;
            bool keep = false; float dd = 0.f;
            if(i < n_raw) { dd = rd[i]; const float s = (P.vp.metric == 1) ? fabsf(dd) : dd; keep = !(s > P.vp.distance_threshold); }
            long long pos, agg;
            Scan(s_scan).ExclusiveSum(keep ? 1ll : 0ll, pos, agg);
            pos += s_carry;
            if(keep) { v_id[pos] = ri[i]; v_dist[pos] = dd; v_rank[pos] = (uint32_t) pos; }
            __syncthreads();
            if(tid == 0) s_carry += agg;
            __syncthreads();
        }
        n_v = (uint32_t) s_carry;
        for(uint32_t i = n_v + tid; i < PV; i += kThreads) v_id[i] = kNone;
        __syncthreads();
        // sort by seq_id, the distance and rank travel along
        for(uint32_t k = 2; k <= PV; k <<= 1) {
            for(uint32_t j = k >> 1; j > 0; j >>= 1) {
                for(uint32_t t = tid; t < (PV >> 1); t += kThreads) {
                    const uint32_t i = ((t & ~(j - 1)) << 1) | (t & (j - 1)), p = i + j;
                    const bool up = ((i & k) == 0);
                    if(up ? (v_id[p] < v_id[i]) : (v_id[i] < v_id[p])) {
                        uint32_t a = v_id[i]; v_id[i] = v_id[p]; v_id[p] = a;
                        float b = v_dist[i]; v_dist[i] = v_dist[p]; v_dist[p] = b;
                        uint32_t c = v_rank[i]; v_rank[i] = v_rank[p]; v_rank[p] = c;
                    }
                }
                __syncthreads();
            }
        }
    }
    // keyword keys sorted by seq_id, for the slot look-up of every vector result
    for(uint32_t i = tid; i < PK; i += kThreads) { kw_key[i] = i < n_kw ? (uint32_t) data[i].key : kNone; kw_slot[i] = i; }
    __syncthreads();
    for(uint32_t k = 2; k <= PK; k <<= 1) {
        for(uint32_t j = k >> 1; j > 0; j >>= 1) {
            for(uint32_t t = tid; t < (PK >> 1); t += kThreads) {
                const uint32_t i = ((t & ~(j - 1)) << 1) | (t & (j - 1)), p = i + j;
                const bool up = ((i & k) == 0);
                if(up ? (kw_key[p] < kw_key[i]) : (kw_key[i] < kw_key[p])) {
                    uint32_t a = kw_key[i]; kw_key[i] = kw_key[p]; kw_key[p] = a;
                    uint32_t c = kw_slot[i]; kw_slot[i] = kw_slot[p]; kw_slot[p] = c;
                }
            }
            __syncthreads();
        }
    }

    // ---- the order-independent part of the loop body, one vector result per thread: filter bit, all_result_ids, the
    // vector-only KV's sort scores, whether the id is a keyword match, and its keyword Topster slot
    for(uint32_t vi = tid; vi < n_v; vi += kThreads) {
        const uint32_t seq_id = v_id[vi];
        uint8_t fl = 0;
        bool pass = !qd.filter_empty;
        if(pass && qd.filter_bitmap) pass = (qd.filter_bitmap[seq_id >> 5] >> (seq_id & 31)) & 1;
        uint32_t slot = kNoSlot;
        if(pass) {
            fl = 1;
            if(qd.keep_all && qd.found_bitmap) atomicOr(qd.found_bitmap + (seq_id >> 5), 1u << (seq_id & 31));
            const double vec_part = (1.0 / (double) (v_rank[vi] + 1)) * (double) VECTOR_SEARCH_WEIGHT;
            int64_t sc[3];
            v_msi[vi] = (int8_t) compute_sort_scores(SS, seq_id, float_to_int64(__double2float_rn(vec_part)), v_dist[vi], sc);
            v_sc[3 * vi] = sc[0]; v_sc[3 * vi + 1] = sc[1]; v_sc[3 * vi + 2] = sc[2];
            bool in_kw = true;
            if(qd.n_excl && excluded(qd.excl, qd.n_excl, seq_id)) in_kw = false;
            if(in_kw) in_kw = tsf::is_keyword_match(P, qd, seq_id);
            if(!in_kw) fl |= 2;
            uint32_t lo = 0, hi = n_kw;
            while(lo < hi) { const uint32_t mid = (lo + hi) >> 1; if(kw_key[mid] < seq_id) lo = mid + 1; else hi = mid; }
            if(lo < n_kw && kw_key[lo] == seq_id) slot = kw_slot[lo];
        }
        v_flag[vi] = fl; v_slot[vi] = slot;
    }
    __syncthreads();
    if(tid == 0) tm[1] = global_ns();

    // ---- serial replay of the fusion loop
    if(tid == 0) {
        uint32_t size = n_kw, vec_new = 0;
        for(uint32_t vi = 0; vi < n_v; vi++) {
            const uint8_t fl = v_flag[vi];
            if(!(fl & 1)) continue;
            const uint32_t seq_id = v_id[vi], slot = v_slot[vi];
            const float dist = v_dist[vi];
            if(slot != kNoSlot && inmap[slot]) {               // topster->map.find(seq_id) hit: rewrite the scores in place
                KVOut& fk = data[slot];
                if(!(fk.match_score_index < 0 || fk.match_score_index > 2)) {
                    const double vec_part = (1.0 / (double) (v_rank[vi] + 1)) * (double) VECTOR_SEARCH_WEIGHT;
                    fk.vector_distance = dist;
                    const int64_t match_score = float_to_int64(__double2float_rn((double) int64_to_float(fk.scores[fk.match_score_index]) + vec_part));
                    int64_t sc[3];
                    const int msi = compute_sort_scores(SS, seq_id, match_score, dist, sc);
                    fk.scores[0] = sc[0]; fk.scores[1] = sc[1]; fk.scores[2] = sc[2];
                    fk.match_score_index = (int8_t) msi;
                }
                continue;
            }
            KVOut kv;
            kv.key = seq_id; kv.distinct_key = seq_id;
            kv.scores[0] = v_sc[3 * vi]; kv.scores[1] = v_sc[3 * vi + 1]; kv.scores[2] = v_sc[3 * vi + 2];
            kv.match_score_index = v_msi[vi]; kv.pad0 = 0;
            kv.query_index = (uint16_t) P.kw_searched[q];
            kv.text_match_score = 0;
            kv.vector_distance = dist;
            // Topster::add(&kv) on the (no longer heap-ordered) array
            if(!(size >= K && tsf::kvo_smaller(kv, data[kvs[0]]))) {
                uint32_t hidx;
                if(size < K) {
                    hidx = size; kvs[hidx] = size; size++;
                    data[kvs[hidx]] = kv;
                    while(hidx > 0) {
                        const uint32_t parent = (hidx - 1) / 2;
                        if(tsf::kvo_greater(data[kvs[parent]], data[kvs[hidx]])) { const uint32_t t = kvs[hidx]; kvs[hidx] = kvs[parent]; kvs[parent] = t; hidx = parent; }
                        else break;
                    }
                } else {
                    hidx = 0;
                    inmap[kvs[0]] = 0;                      // the evicted entry leaves the map
                    data[kvs[0]] = kv;
                    while((2 * hidx + 1) < size) {
                        uint32_t next = 2 * hidx + 1;
                        if(next + 1 < size && tsf::kvo_greater(data[kvs[next]], data[kvs[next + 1]])) next++;
                        if(tsf::kvo_greater(data[kvs[hidx]], data[kvs[next]])) { const uint32_t t = kvs[hidx]; kvs[hidx] = kvs[next]; kvs[next] = t; }
                        else break;
                        hidx = next;
                    }
                }
            }
            if(fl & 2) vec_new++;                           // vec_search_ids.push_back whether or not the heap took it
        }
        s_size = size; s_vec_new = vec_new;
        tm[2] = global_ns();
    }
    __syncthreads();
    const uint32_t size = s_size;

    // ---- rerank_hybrid_matches: Index::compute_aux_scores (src/index.cpp:8793-8923); slots 0 .. size-1 hold the entries
    if(qd.rerank && size) {
        for(uint32_t i = tid; i < size; i += kThreads) {
            KVOut& kv = data[i];
            if(kv.text_match_score == 0) kv.text_match_score = tsf::aux_text_score(P, qd, (uint32_t) kv.key);
        }
        __syncthreads();                                   // the distance loop below reads text_match_score
        {   // results only the keyword query found: their vector distance (one warp per result, W128 order as everywhere)
            const uint32_t lane2 = tid & 31, warp2 = tid >> 5;
            const float* qv = P.queries + (size_t) q * P.dim;
            for(uint32_t i = warp2; i < size; i += kThreads / 32) {
                const bool need = data[i].vector_distance == -1.0f && data[i].text_match_score != 0 && (uint32_t) data[i].key < P.n_nodes;
                if(!need) continue;
                const float* v = P.vectors + (size_t) (uint32_t) data[i].key * P.dim;
                float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
                for(uint32_t sgm = 0; sgm * 128 < P.dim; sgm++) {
                    const uint32_t e = sgm * 128 + 4 * lane2;
                    if(e + 0 < P.dim) a0 = __fmaf_rn(qv[e + 0], __ldg(v + e + 0), a0);
                    if(e + 1 < P.dim) a1 = __fmaf_rn(qv[e + 1], __ldg(v + e + 1), a1);
                    if(e + 2 < P.dim) a2 = __fmaf_rn(qv[e + 2], __ldg(v + e + 2), a2);
                    if(e + 3 < P.dim) a3 = __fmaf_rn(qv[e + 3], __ldg(v + e + 3), a3);
                }
                float t = __fadd_rn(__fadd_rn(a0, a1), __fadd_rn(a2, a3));
                for(int off = 16; off >= 1; off >>= 1) t = __fadd_rn(t, __shfl_xor_sync(0xffffffffu, t, off));
                if(lane2 == 0) data[i].vector_distance = 1.0f - t;
            }
        }
        __syncthreads();
        // keyword rank: position in (text_match_score, key) descending
        uint32_t* order = kw_key;
        uint32_t* kr = kw_slot;
        for(uint32_t i = tid; i < PK; i += kThreads) order[i] = i < size ? i : kNone;
        __syncthreads();
        auto kw_before = [&](uint32_t a, uint32_t b) {
            const int64_t ta = data[a].text_match_score, tb = data[b].text_match_score;
            return ta > tb || (ta == tb && (uint32_t) data[a].key > (uint32_t) data[b].key);
        };
        cta_bitonic(order, PK, kw_before);
        for(uint32_t p = tid; p < size; p += kThreads) kr[order[p]] = p + 1;
        __syncthreads();
        // semantic rank: position in distance ascending, ties in keyword-rank order
        for(uint32_t i = tid; i < PK; i += kThreads) order[i] = i < size ? i : kNone;
        __syncthreads();
        auto sem_before = [&](uint32_t a, uint32_t b) {
            const float da = data[a].vector_distance, db = data[b].vector_distance;
            return da < db || (da == db && kr[a] < kr[b]);
        };
        cta_bitonic(order, PK, sem_before);
        const double alpha = (double) P.vp.alpha;
        for(uint32_t p = tid; p < size; p += kThreads) {
            const uint32_t i = order[p];
            const int m = data[i].match_score_index;
            if(m >= 0 && m <= 2) data[i].scores[m] = float_to_int64(__double2float_rn((1.0 / (double) kr[i]) * (1.0 - alpha) + (1.0 / (double) (p + 1)) * alpha));
        }
        __syncthreads();
    }
    if(tid == 0) tm[3] = global_ns();

    // ---- final topster->sort(): by the KV order (a total order: keys are unique)
    for(uint32_t i = tid; i < PK; i += kThreads) kvs[i] = i < size ? i : kNone;
    __syncthreads();
    cta_bitonic(kvs, PK, [&](uint32_t a, uint32_t b) { return tsf::kvo_greater(data[a], data[b]); });
    const uint32_t n_out = size < P.kv_stride ? size : P.kv_stride;
    for(uint32_t i = tid; i < n_out; i += kThreads) P.out_kv[(size_t) q * P.kv_stride + i] = data[kvs[i]];
    if(tid == 0) { P.out_count[q] = n_out; P.out_found[q] = P.kw_found[q] + s_vec_new; }
    __syncthreads();
    if(tid == 0) tm[4] = global_ns();
}
#endif  // TSDF_KERNELS

}  // namespace tsdf
