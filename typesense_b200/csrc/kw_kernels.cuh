// Keyword hot path on sm_90a: block decode + k-way intersection (K1/K2), match scoring (K3), sort-key assembly
// and streaming top-K (K4), phrase check (K5).
//
// Replaces (reference file:line):
//   or_iterator_t::intersect + take_id           include/or_iterator.h:61-181, src/or_iterator.cpp:218-272
//   posting_list_t::iterator_t next/skip_to      src/posting_list.cpp:1954-2061 (FOR decode + std::map skip index)
//   Index::compute_aggregated_score / score_results2 / Match     src/index.cpp:5227-5383, 6966-7098
//   Index::compute_sort_scores, Topster<KV>::add/sort            src/index.cpp:5662-5907, include/topster.h:321-473
//   posting_list_t::intersect / get_phrase_matches               src/posting_list.cpp:708-756, 1791-1825
//
// Execution model (see DESIGN.md §3): a work UNIT is (token combination, run of driver tiles). The driver is the
// required token with the fewest postings; a tile is one 128-id block of one of its field lists. One 128-thread CTA
// per unit, one candidate id per thread:
//   decode   : thread i extracts id i of the packed block (FOR: first + b-bit delta) — coalesced, no neighbours needed
//   filter   : bitmap test (filter_result_iterator_t materialised to bits) + binary search in the exclusion list
//   narrow   : 2 threads per probed list gallop the skip index (blk_first) from the previous tile's position to the
//              blocks covering [tile min id, tile max id]
//   probe    : each live candidate binary-searches those few skip entries, then the b-bit packed block itself
//   compact  : warp ballots -> dense list of matches (so scoring threads are not diverged)
//   score    : score_field()/Match per field from the raw offsets in HBM, sort keys from the dense sort columns
//   select   : CTA-local top-K kept in shared memory: append survivors above the running K-th threshold, bitonic
//              sort + truncate when the 2*KP buffer fills; unit writes <= K entries
// kw_final_kernel then merges a query's units (all combinations), de-duplicates seq_ids keeping the greater KV
// (Topster::add, include/topster.h:392-406) and emits KV records in Topster::sort() order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "postings_device.cuh"

namespace tsk {

using namespace tsdev;

constexpr int kThreads = 128;          // == kBlock: one candidate per thread
constexpr int kMaxFieldSlots = 8;      // TSGPU_MAX_FIELDS
constexpr int kMaxLists = 32;          // rows * fields per combination
constexpr int kMaxIndexFields = 16;
constexpr int kMaxCombosPerQuery = 256;

struct IndexDev {
    DevField fields[kMaxIndexFields];
    uint32_t n_docs;
};

struct QDesc {
    const int64_t* sort_col[3];
    const uint32_t* filter_bitmap;     // nullptr: no filter
    const uint32_t* excl;
    uint32_t* found_bitmap;            // nullptr unless the query has several combinations
    uint32_t n_excl;
    uint32_t topk;
    uint32_t combo_begin, combo_end;
    uint32_t unit_begin, unit_end;
    uint8_t  sort_type[3];
    int8_t   sort_order[3];
    uint8_t  missing_first[3];
    uint8_t  flags, match_type, num_query_tokens;
    uint8_t  field_weight[kMaxFieldSlots];
    uint8_t  filter_empty;             // filter given but matches no doc (src/index.cpp:4823-4826)
    uint8_t  keep_all;                 // found_bitmap is the query's all_result_ids and outlives the call (facets, export)
    uint8_t  rerank;                   // hybrid calls: compute_aux_scores after the fusion (rerank_hybrid_matches)
    uint8_t  pad[1];
};

struct CDesc {
    uint32_t q;
    uint32_t total_cost;
    int32_t  syn_orig, orig;
    uint8_t  n_rows, n_req, driver_row, cflags;
    uint32_t req_mask;                 // rows that are required AND present in at least one field
    uint32_t lists[kMaxLists];         // [row * F + f]
    uint32_t drv_tile_off[kMaxFieldSlots + 1];
    uint8_t  probe_order[16];
    uint32_t mode;                     // 0: driver tiles + per-candidate probes; 1: word-parallel AND of dense bitmaps
    uint32_t w_begin, w_end;           // mode 1: bitmap words [w_begin, w_end) the tiles cover; w_begin is a multiple of 32
};

struct UDesc {
    uint32_t combo;
    uint32_t tile_begin, tile_end;
    uint32_t out_off;                  // first pool slot of this unit
};

struct KwParams {
    const QDesc* qd;
    const CDesc* cd;
    const UDesc* ud;
    int64_t* pool_s0; int64_t* pool_s1; int64_t* pool_s2;
    uint32_t* pool_key;
    uint16_t* pool_cmb;                // combination index local to the query
    uint32_t* unit_cnt;                // [n_units]
    uint32_t* combo_matches;           // [n_combos]
    unsigned long long* stats;         // [0] driver ids, [1] probed block ids, [2] matches
    long long* q_thr;                  // [nq] best "K-th scores[0]" published by any finished top-K of the query
    uint32_t F;
    uint32_t field_ids[kMaxFieldSlots];
    uint32_t KP;                       // power of two >= max topk in the batch
    uint32_t NL;                       // max rows*F in the batch (shared-memory stride)
};

// ---------------------------------------------------------------------------------------------------------------
// shared-memory top-K buffer (structure of arrays, 2*KP slots)
struct TopBuf {
    int64_t* s0; int64_t* s1; int64_t* s2;
    uint32_t* key;
    uint16_t* cmb;     // combination index local to the query (final kernel only; nullptr in the unit kernel)
    float* vd;         // vector distance payload (vector assembly only; nullptr otherwise)
};

__device__ __forceinline__ bool tb_greater(const TopBuf& b, uint32_t i, uint32_t j) {
    const uint32_t ki = b.key[i], kj = b.key[j];
    if(ki == kNone) return false;
    if(kj == kNone) return true;
    const int64_t a0 = b.s0[i], b0 = b.s0[j];
    if(a0 != b0) return a0 > b0;
    const int64_t a1 = b.s1[i], b1 = b.s1[j];
    if(a1 != b1) return a1 > b1;
    const int64_t a2 = b.s2[i], b2 = b.s2[j];
    if(a2 != b2) return a2 > b2;
    if(ki != kj) return ki > kj;
    return b.cmb ? (b.cmb[i] > b.cmb[j]) : false;
}
// order for the de-duplication pass: key ascending, then the KV order descending (best entry of a key first)
__device__ __forceinline__ bool tb_before_bykey(const TopBuf& b, uint32_t i, uint32_t j) {
    const uint32_t ki = b.key[i], kj = b.key[j];
    if(ki != kj) return ki < kj;          // kNone (invalid) sorts last
    if(ki == kNone) return false;
    return tb_greater(b, i, j);
}
__device__ __forceinline__ void tb_swap(const TopBuf& b, uint32_t i, uint32_t j) {
    int64_t t;
    t = b.s0[i]; b.s0[i] = b.s0[j]; b.s0[j] = t;
    t = b.s1[i]; b.s1[i] = b.s1[j]; b.s1[j] = t;
    t = b.s2[i]; b.s2[i] = b.s2[j]; b.s2[j] = t;
    uint32_t k = b.key[i]; b.key[i] = b.key[j]; b.key[j] = k;
    if(b.cmb) { uint16_t c = b.cmb[i]; b.cmb[i] = b.cmb[j]; b.cmb[j] = c; }
    if(b.vd) { float v = b.vd[i]; b.vd[i] = b.vd[j]; b.vd[j] = v; }
}

// bitonic sort of N (power of two) slots; BYKEY selects the de-dup order. All threads of the CTA call it.
template <bool BYKEY>
__device__ void tb_sort(const TopBuf& b, uint32_t N) {
    for(uint32_t k = 2; k <= N; k <<= 1) {
        for(uint32_t j = k >> 1; j > 0; j >>= 1) {
            for(uint32_t t = threadIdx.x; t < (N >> 1); t += blockDim.x) {
                const uint32_t i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                const uint32_t p = i + j;
                const bool up = ((i & k) == 0);
                const uint32_t x = up ? p : i, y = up ? i : p;          // swap when x has to come before y
                if(BYKEY ? tb_before_bykey(b, x, y) : tb_greater(b, x, y)) tb_swap(b, i, p);
            }
            __syncthreads();
        }
    }
}

__device__ __forceinline__ void tb_fill_invalid(const TopBuf& b, uint32_t from, uint32_t N) {
    for(uint32_t i = from + threadIdx.x; i < N; i += blockDim.x) b.key[i] = kNone;
}

// ---------------------------------------------------------------------------------------------------------------
// Last block b in [start, end] with blk_first[b] <= target, galloping from `start`; kNone if blk_first[start] > target.
__device__ __forceinline__ uint32_t gallop_block(const uint32_t* __restrict__ blk_first, uint32_t start, uint32_t end,
                                                 uint32_t target) {
    if(__ldg(blk_first + start) > target) return kNone;
    uint32_t lo = start, step = 1;
    while(lo + step <= end && __ldg(blk_first + lo + step) <= target) { lo += step; step <<= 1; }
    uint32_t hi = lo + step - 1;
    if(hi > end) hi = end;
    return find_block(blk_first, lo, hi, target);
}

__device__ __forceinline__ bool excluded(const uint32_t* __restrict__ excl, uint32_t n, uint32_t id) {
    uint32_t lo = 0, hi = n;
    while(lo < hi) { uint32_t mid = (lo + hi) >> 1; if(excl[mid] < id) lo = mid + 1; else hi = mid; }
    return lo < n && excl[lo] == id;
}

// exclusive prefix of `flag` over the CTA; returns this thread's rank, *total = CTA count. s_warp: >= 4 u32 scratch.
__device__ __forceinline__ uint32_t cta_rank(bool flag, uint32_t* s_warp, uint32_t* total) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t bal = __ballot_sync(0xffffffffu, flag);
    if(lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    uint32_t base = 0, tot = 0;
    const uint32_t nw = blockDim.x >> 5;
    for(uint32_t w = 0; w < nw; w++) { const uint32_t c = s_warp[w]; if(w < warp) base += c; tot += c; }
    __syncthreads();
    *total = tot;
    return base + __popc(bal & ((1u << lane) - 1u));
}

// ---------------------------------------------------------------------------------------------------------------
constexpr int kQCap = 2 * kThreads;        // pending-match queue slots per CTA

// The kernel is latency-bound on dependent HBM loads (gallop -> probe -> offsets), so resident warps matter more than
// registers per thread: cap at 64 registers (no spills at -O3) for 8 CTAs = 32 warps per SM.
#ifndef TSGPU_KW_MIN_CTAS
#define TSGPU_KW_MIN_CTAS 8
#endif
// REGSCORE (the default, TSGPU_REG_SCORE=0 switches it off): plain fields of combinations with at most kSmallTokens
// rows are scored by score_field_plain_small(), which keeps the tokens and the Match window in registers instead of the
// run-time indexed local arrays of score_field_plain(). <false> is the general scorer.
// ONEFIELD (only instantiated next to REGSCORE): the batch searches a single field, so F is the constant 1 and the
// per-row / per-field index arithmetic of narrowing, probing and scoring folds away.
// DEEP (deep_topster.cuh; kw_deep.cu launches it only over the units of deep queries, with KP = 0): no top-K buffer. Every scored match
// goes to the query's slice of the deep buffer, which P.pool_* then address (64-bit index); P.q_thr[q] is the query's
// cursor into it, starting at the slice's first entry. Match counts, found bitmaps and work counters are kept as here.
template <bool REGSCORE, bool ONEFIELD = false, bool DEEP = false>
__global__ void __launch_bounds__(kThreads, TSGPU_KW_MIN_CTAS)
kw_search_kernel(const __grid_constant__ IndexDev ix, const __grid_constant__ KwParams P) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const uint32_t KP = P.KP, N2 = 2 * KP, NL = P.NL, F = ONEFIELD ? 1u : P.F;
    TopBuf tb;
    tb.s0 = reinterpret_cast<int64_t*>(smem_raw);
    tb.s1 = tb.s0 + N2;
    tb.s2 = tb.s1 + N2;
    tb.key = reinterpret_cast<uint32_t*>(tb.s2 + N2);
    tb.cmb = nullptr;
    tb.vd = nullptr;
    uint32_t* hp = tb.key + N2;                       // [NL][128] staging: list-local posting index of candidate in list j
    uint32_t* q_id = hp + NL * kThreads;              // [kQCap] queue of matched docs waiting to be scored
    uint32_t* q_hp = q_id + kQCap;                    // [NL][kQCap]

    __shared__ CDesc cd;
    __shared__ QDesc qd;
    __shared__ uint32_t l_blk0[kMaxLists], l_blk1[kMaxLists], l_dense[kMaxLists];
    __shared__ uint32_t w_gal[kThreads / 32][kMaxLists], w_lo[kThreads / 32][kMaxLists], w_hi[kThreads / 32][kMaxLists];
    __shared__ unsigned long long l_df[kMaxLists], l_base[kMaxLists];
    __shared__ uint32_t s_warp[8];
    __shared__ int64_t thr[3];
    __shared__ uint32_t thr_key;
    __shared__ uint32_t s_n, s_have_thr, s_matches, s_driver_ids, s_probe_blocks, s_qn;

    const uint32_t tid = threadIdx.x;
    const UDesc ud = P.ud[blockIdx.x];
    {   // descriptors -> shared
        const uint32_t* src = reinterpret_cast<const uint32_t*>(P.cd + ud.combo);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&cd);
        for(uint32_t i = tid; i < sizeof(CDesc) / 4; i += kThreads) dst[i] = src[i];
    }
    __syncthreads();
    {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(P.qd + cd.q);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&qd);
        for(uint32_t i = tid; i < sizeof(QDesc) / 4; i += kThreads) dst[i] = src[i];
    }
    const uint32_t n_lists = (uint32_t) cd.n_rows * F;
    if(tid < n_lists) {
        const uint32_t l = cd.lists[tid];
        if(l != kNone) {
            const DevField& fld = ix.fields[P.field_ids[tid % F]];
            const uint32_t b0 = fld.list_blk_off[l], b1 = fld.list_blk_off[l + 1];
            l_blk0[tid] = b0; l_blk1[tid] = b1 - 1;      // lists are never empty
            l_base[tid] = fld.list_off[l];
            l_df[tid] = fld.list_off[l + 1] - fld.list_off[l];
            l_dense[tid] = fld.list_dense ? fld.list_dense[l] : kNone;
        } else { l_blk0[tid] = 0; l_blk1[tid] = 0; l_base[tid] = 0; l_df[tid] = 0; l_dense[tid] = kNone; }
    }
    if(tid == 0) { s_n = 0; s_have_thr = 0; s_matches = 0; s_driver_ids = 0; s_probe_blocks = 0; s_qn = 0; }
    __syncthreads();

    ScoreParams SP;
    SP.total_cost = cd.total_cost;
    SP.num_query_tokens = qd.num_query_tokens;
    SP.syn_orig_num_tokens = cd.syn_orig;
    SP.orig_num_tokens = cd.orig;
    SP.is_synonym_query = cd.cflags & 1;
    SP.demote_synonym_match = (cd.cflags >> 1) & 1;
    SP.prioritize_exact_match = qd.flags & 1;
    SP.prioritize_token_position = (qd.flags >> 1) & 1;
    SP.prioritize_num_matching_fields = (qd.flags >> 2) & 1;
    SP.match_type = qd.match_type;
    SortSpec SS;
    for(int i = 0; i < 3; i++) {
        SS.type[i] = qd.sort_type[i]; SS.order[i] = qd.sort_order[i]; SS.missing_first[i] = qd.missing_first[i];
        SS.col[i] = qd.sort_col[i];
    }
    const uint32_t K = qd.topk;
    const uint32_t drv = cd.driver_row;
    const uint16_t cmb_local = (uint16_t) (ud.combo - qd.combo_begin);
    const uint32_t warp = tid >> 5, lane = tid & 31;
    long long* const gthr_p = P.q_thr + cd.q;
    uint32_t prev_fd = 0xFFFFFFFFu;
    uint32_t qn = 0;                               // queue length, identical in every thread (see the barriers below)

    // Scores queue entries [base, base+cnt) (cnt <= 128) with all threads busy, appends the survivors to the top-K
    // buffer and compacts that buffer when the next batch might not fit.
    auto score_batch = [&](uint32_t base, uint32_t cnt) {
        const long long gthr = DEEP ? 0 : *reinterpret_cast<volatile long long*>(gthr_p);
        bool keep = false;
        int64_t sc[3] = {0, 0, 0};
        uint32_t mid = 0;
        bool valid = tid < cnt;
        if(valid && cd.mode == 1 && qd.n_excl && excluded(qd.excl, qd.n_excl, q_id[base + tid])) valid = false;   // dense mode excludes here
        if(cd.mode == 1) {
            const uint32_t vb = __ballot_sync(0xffffffffu, valid);
            if(lane == 0 && vb) atomicAdd(&s_matches, (uint32_t) __popc(vb));
        }
        if(valid) {
            const uint32_t src = base + tid;
            mid = q_id[src];
            FieldAgg agg; field_agg_init(agg);
            uint32_t query_len = 0;
            for(uint32_t r = 0; r < cd.n_rows; r++) {
                bool any = false;
                for(uint32_t f = 0; f < F; f++) any |= (q_hp[(r * F + f) * kQCap + src] != kNone);
                query_len += any;
            }
            for(uint32_t f = 0; f < F; f++) {
                const DevField& g = ix.fields[P.field_ids[f]];
                if constexpr (REGSCORE) {
                    if(cd.n_rows <= (uint32_t) kSmallTokens && (g.is_array & kFieldPos16)) {
                        const uint32_t* tp[kSmallTokens];
                        uint32_t tn[kSmallTokens], present = 0;
#pragma unroll
                        for(int r = 0; r < kSmallTokens; r++) {
                            tp[r] = g.positions; tn[r] = 0;
                            if((uint32_t) r < cd.n_rows) {
                                const uint32_t j = (uint32_t) r * F + f;
                                const uint32_t h = q_hp[j * kQCap + src];
                                if(h != kNone) {
                                    const unsigned long long p = l_base[j] + h;
                                    const unsigned long long o0 = __ldg(reinterpret_cast<const unsigned long long*>(g.pos_off) + p);
                                    const unsigned long long o1 = __ldg(reinterpret_cast<const unsigned long long*>(g.pos_off) + p + 1);
                                    tp[r] = g.positions + o0; tn[r] = (uint32_t) (o1 - o0); present |= 1u << r;
                                }
                            }
                        }
                        if(!present) continue;
                        const int64_t fs = score_field_plain_small<kSmallTokens>(SP, SP.total_cost == 0 && SP.num_query_tokens == 1, tp, tn, present);
                        field_agg_add(agg, SP.match_type, fs, (int64_t) qd.field_weight[f]);
                        continue;
                    }
                }
                RawTok toks[kMaxTokens];
                int nt = 0;
                for(uint32_t r = 0; r < cd.n_rows; r++) {
                    const uint32_t j = r * F + f;
                    const uint32_t h = q_hp[j * kQCap + src];
                    if(h == kNone) continue;
                    const unsigned long long p = l_base[j] + h;
                    const unsigned long long o0 = __ldg(reinterpret_cast<const unsigned long long*>(g.pos_off) + p);
                    const unsigned long long o1 = __ldg(reinterpret_cast<const unsigned long long*>(g.pos_off) + p + 1);
                    toks[nt].p = g.positions + o0;
                    toks[nt].n = (uint32_t) (o1 - o0);
                    nt++;
                }
                if(nt == 0) continue;
                const bool single_exact = (SP.total_cost == 0 && SP.num_query_tokens == 1);
                const int64_t fs = (g.is_array & kFieldPlainOk) ? score_field_plain(SP, single_exact, toks, nt)
                                                                : score_field(SP, (g.is_array & kFieldIsArray) != 0, single_exact, toks, nt);
                field_agg_add(agg, SP.match_type, fs, (int64_t) qd.field_weight[f]);
            }
            const uint64_t aggs = field_agg_finish(agg, SP, query_len);
            const int msi = compute_sort_scores(SS, mid, (int64_t) aggs, 0.0f, sc);
            if(msi >= 0) sc[msi] = (int64_t) aggs;            // src/index.cpp:5541-5544 (undoes the ASC negation)
            if(qd.found_bitmap) atomicOr(qd.found_bitmap + (mid >> 5), 1u << (mid & 31));
            if constexpr (DEEP) keep = true;
            else {
                keep = sc[0] >= gthr;          // K distinct docs of this query already have scores[0] >= gthr
                if(keep && s_have_thr) keep = kv_greater(sc[0], sc[1], sc[2], mid, thr[0], thr[1], thr[2], thr_key);
            }
        }
        uint32_t a_total;
        const uint32_t arank = cta_rank(keep, s_warp, &a_total);
        if constexpr (DEEP) {
            // one atomic per CTA per batch reserves the batch's entries; thr[0] (unused here) carries the base
            if(tid == 0 && a_total) thr[0] = (int64_t) atomicAdd(reinterpret_cast<unsigned long long*>(gthr_p), (unsigned long long) a_total);
            __syncthreads();
            if(keep) {
                const size_t o = (size_t) thr[0] + arank;
                P.pool_s0[o] = sc[0]; P.pool_s1[o] = sc[1]; P.pool_s2[o] = sc[2]; P.pool_key[o] = mid; P.pool_cmb[o] = cmb_local;
            }
            return;
        }
        const uint32_t n0 = s_n;
        if(keep) {
            const uint32_t slot = n0 + arank;
            tb.s0[slot] = sc[0]; tb.s1[slot] = sc[1]; tb.s2[slot] = sc[2]; tb.key[slot] = mid;
        }
        __syncthreads();
        if(tid == 0) s_n = n0 + a_total;
        __syncthreads();
        if(s_n + kThreads > N2) {                 // the next batch might not fit: sort, keep the best K
            const uint32_t n = s_n;
            tb_fill_invalid(tb, n, N2);
            __syncthreads();
            tb_sort<false>(tb, N2);
            if(tid == 0) {
                const uint32_t nn = n < K ? n : K;
                s_n = nn;
                if(nn == K) {
                    s_have_thr = 1; thr[0] = tb.s0[K - 1]; thr[1] = tb.s1[K - 1]; thr[2] = tb.s2[K - 1]; thr_key = tb.key[K - 1];
                    atomicMax(gthr_p, (long long) tb.s0[K - 1]);
                }
            }
            __syncthreads();
        }
    };

    if(cd.mode == 1) {
        // ---- all required tokens are dense lists: intersect their bitmaps 32 docs per instruction. A tile is 128
        // consecutive bitmap words (4096 docs) of the lists' common id range, one word per thread; set bits are popped one
        // per thread and round into the same scoring queue. Replaces the decode/narrow/probe pipeline for the heaviest
        // combinations.
        for(uint32_t tile = ud.tile_begin; tile < ud.tile_end; tile++) {
            const uint32_t w0 = cd.w_begin + tile * kThreads, wi = w0 + tid;
            uint32_t word = 0;
            if(tid == 0) s_driver_ids += (min(cd.w_end - w0, (uint32_t) kThreads)) << 5;      // documents the tile covers
            if(wi < cd.w_end && !qd.filter_empty) {
                word = 0xFFFFFFFFu;
                for(uint32_t r = 0; r < cd.n_rows; r++) {
                    if(!((cd.req_mask >> r) & 1)) continue;
                    uint32_t rw = 0;
                    for(uint32_t f = 0; f < F; f++) {
                        const uint32_t j = r * F + f;
                        if(cd.lists[j] == kNone) continue;
                        const DevField& g = ix.fields[P.field_ids[f]];
                        rw |= __ldg(g.dense_bits + (size_t) l_dense[j] * g.dense_words + wi);
                    }
                    word &= rw;
                }
                if(qd.filter_bitmap) word &= __ldg(qd.filter_bitmap + wi);
            }
            for(;;) {
                // Every decision below is taken from values that are uniform across the CTA by construction (the barrier's
                // count and the register `qn`), never from shared memory that a faster warp may already be updating.
                const uint32_t cnt = (uint32_t) __syncthreads_count(word != 0);    // also publishes the previous round's queue writes
                if(cnt == 0) break;
                if(qn >= kThreads) {                                   // make room: cnt <= 128 more entries are coming
                    score_batch(qn - kThreads, kThreads);
                    qn -= kThreads;
                    if(tid == 0) s_qn = qn;
                    __syncthreads();
                }
                const bool has = word != 0;
                uint32_t id = 0;
                if(has) {
                    const uint32_t bit = __ffs(word) - 1;
                    word &= word - 1;
                    id = (wi << 5) | bit;
                }
                const uint32_t bal = __ballot_sync(0xffffffffu, has);
                if(bal) {
                    uint32_t qb = 0;
                    if(lane == 0) qb = atomicAdd(&s_qn, (uint32_t) __popc(bal));
                    qb = __shfl_sync(0xffffffffu, qb, 0);
                    if(has) {
                        const uint32_t slot = qb + __popc(bal & ((1u << lane) - 1u));
                        q_id[slot] = id;
                        for(uint32_t j = 0; j < n_lists; j++) {
                            const uint32_t l = cd.lists[j];
                            uint32_t h = kNone;
                            if(l != kNone) {
                                const DevField& g = ix.fields[P.field_ids[j % F]];
                                if(l_dense[j] != kNone) { if(dense_test(g, l_dense[j], id)) h = dense_rank_of(g, l_dense[j], id); }
                                else h = probe_list(g, l, l_blk0[j], l_blk1[j], id);      // sparse list of a dropped token
                            }
                            q_hp[j * kQCap + slot] = h;
                        }
                    }
                }
                qn += cnt;
            }
        }
    } else
    for(uint32_t tile = ud.tile_begin; tile < ud.tile_end; tile++) {
        // ---- which driver field / block
        uint32_t fd = 0;
        while(fd + 1 < F && tile >= cd.drv_tile_off[fd + 1]) fd++;
        const uint32_t jd = drv * F + fd;
        const DevField& dfld = ix.fields[P.field_ids[fd]];
        const uint32_t b = l_blk0[jd] + (tile - cd.drv_tile_off[fd]);
        const uint32_t cnt = block_count(b, l_blk0[jd], l_df[jd]);
        if(fd != prev_fd) {                        // ids restart with a new driver list: reset this warp's gallop cursors
            __syncwarp();
            if(lane < n_lists) w_gal[warp][lane] = l_blk0[lane];
            prev_fd = fd;
            __syncwarp();
        }
        // ---- decode (K2)
        const uint32_t first = __ldg(dfld.blk_first + b);
        const unsigned long long info = __ldg(reinterpret_cast<const unsigned long long*>(dfld.blk_info) + b);
        const uint32_t bits = (uint32_t) (info >> 40) & 0xFF;
        const uint32_t* w = dfld.packed + (info & 0xFFFFFFFFFFull);
        const uint32_t id = first + unpack_at(w, bits, tid < cnt ? tid : 0);
        bool alive = tid < cnt;
        if(alive && qd.filter_bitmap) alive = (__ldg(qd.filter_bitmap + (id >> 5)) >> (id & 31)) & 1;
        if(alive && qd.n_excl) alive = !excluded(qd.excl, qd.n_excl, id);
        if(qd.filter_empty) alive = false;
        if(tid == 0) s_driver_ids += cnt;
        bool enq = false;

        // Everything up to the enqueue is warp-private (no CTA barrier): each warp owns 32 consecutive candidates.
        const uint32_t wbase = warp * 32;
        if(wbase < cnt && __any_sync(0xffffffffu, alive)) {
            // ---- narrow every probed list to the blocks covering this warp's [min id, max id]
            if(n_lists > 1) {
                const uint32_t last_lane = (cnt - wbase) >= 32 ? 31 : (cnt - wbase - 1);
                const uint32_t wmin = __shfl_sync(0xffffffffu, id, 0);
                const uint32_t wmax = __shfl_sync(0xffffffffu, id, last_lane);
                for(uint32_t t = lane; t < 2 * n_lists; t += 32) {
                    const uint32_t j = t >> 1;
                    if(cd.lists[j] != kNone && j != jd && l_dense[j] == kNone) {
                        const uint32_t* bf = ix.fields[P.field_ids[j % F]].blk_first;
                        const uint32_t r = gallop_block(bf, w_gal[warp][j], l_blk1[j], (t & 1) ? wmax : wmin);
                        if(t & 1) w_hi[warp][j] = r; else w_lo[warp][j] = r;
                    }
                }
                __syncwarp();
                if(lane < n_lists && cd.lists[lane] != kNone && lane != jd && l_dense[lane] == kNone) {
                    // lo == kNone: the warp starts before the list's first remaining block -> clamp; hi == kNone: no hit possible
                    if(w_lo[warp][lane] == kNone) w_lo[warp][lane] = w_gal[warp][lane]; else w_gal[warp][lane] = w_lo[warp][lane];
                    if(w_hi[warp][lane] != kNone) atomicAdd(&s_probe_blocks, w_hi[warp][lane] - w_lo[warp][lane] + 1);
                }
                __syncwarp();
            }
            // ---- probe (K1): rows in probe order, all field slots of a row
            for(uint32_t oi = 0; oi < cd.n_rows; oi++) {
                const uint32_t r = cd.probe_order[oi];
                bool any = false;
                for(uint32_t f = 0; f < F; f++) {
                    const uint32_t j = r * F + f;
                    const uint32_t l = cd.lists[j];
                    uint32_t h = kNone;
                    if(l != kNone) {
                        if(j == jd) h = (b - l_blk0[jd]) * kBlock + tid;
                        else if(l_dense[j] != kNone) {          // dense list: one bit test in an L2-resident bitmap
                            if(alive && dense_test(ix.fields[P.field_ids[f]], l_dense[j], id)) h = kDenseHit;
                        }
                        else if(alive && w_hi[warp][j] != kNone) {
                            const DevField& g = ix.fields[P.field_ids[f]];
                            const uint32_t bb = find_block(g.blk_first, w_lo[warp][j], w_hi[warp][j], id);
                            if(bb != kNone) {
                                const uint32_t c2 = block_count(bb, l_blk0[j], l_df[j]);
                                const uint32_t ii = probe_block(g, bb, c2, id);
                                if(ii != kNone) h = (bb - l_blk0[j]) * kBlock + ii;
                            }
                        }
                    }
                    hp[j * kThreads + tid] = h;
                    if(h != kNone) { any = true; if(r == drv && f < fd) alive = false; }   // produced by an earlier field's tile
                }
                if(((cd.req_mask >> r) & 1) && !any) alive = false;
            }
            // ---- enqueue matches: one shared-memory atomic per warp reserves the slots
            enq = alive;
            const uint32_t bal = __ballot_sync(0xffffffffu, alive);
            if(bal) {
                uint32_t qb = 0;
                if(lane == 0) { qb = atomicAdd(&s_qn, (uint32_t) __popc(bal)); atomicAdd(&s_matches, (uint32_t) __popc(bal)); }
                qb = __shfl_sync(0xffffffffu, qb, 0);
                if(alive) {
                    const uint32_t slot = qb + __popc(bal & ((1u << lane) - 1u));
                    q_id[slot] = id;
                    for(uint32_t j = 0; j < n_lists; j++) {
                        uint32_t h = hp[j * kThreads + tid];
                        if(h == kDenseHit) h = dense_rank_of(ix.fields[P.field_ids[j % F]], l_dense[j], id);   // only matches pay for the rank
                        q_hp[j * kQCap + slot] = h;
                    }
                }
            }
        }
        // the only CTA barrier of a tile: queue writes become visible, and its count keeps the queue length `qn` uniform in
        // registers (reading s_qn here would race with the next tile's enqueues of a faster warp)
        qn += (uint32_t) __syncthreads_count(enq);
        if(qn >= kThreads) {                      // scoring happens 128 docs at a time so no lane idles
            score_batch(qn - kThreads, kThreads);
            qn -= kThreads;
            if(tid == 0) s_qn = qn;
            __syncthreads();
        }
    }
    // ---- drain the queue
    __syncthreads();
    while(qn) {
        const uint32_t c = qn < (uint32_t) kThreads ? qn : (uint32_t) kThreads;
        score_batch(qn - c, c);
        qn -= c;
        __syncthreads();
    }

    // ---- unit epilogue: best <= K entries to the pool
    if constexpr (DEEP) {
        if(tid == 0) {
            if(s_matches) atomicAdd(P.combo_matches + ud.combo, s_matches);
            atomicAdd(P.stats + 0, (unsigned long long) s_driver_ids);
            atomicAdd(P.stats + 1, (unsigned long long) s_probe_blocks * kBlock);
            atomicAdd(P.stats + 2, (unsigned long long) s_matches);
        }
    } else {
        const uint32_t n = s_n;
        uint32_t nn = n;
        if(n > 1) {                               // always sorted best-first: the merges read only the heads of their inputs
            uint32_t NS = 2;
            while(NS < n) NS <<= 1;
            tb_fill_invalid(tb, n, NS);
            __syncthreads();
            tb_sort<false>(tb, NS);
            if(n > K) nn = K;
        }
        for(uint32_t i = tid; i < nn; i += kThreads) {
            const uint32_t o = ud.out_off + i;
            P.pool_s0[o] = tb.s0[i]; P.pool_s1[o] = tb.s1[i]; P.pool_s2[o] = tb.s2[i]; P.pool_key[o] = tb.key[i];
            P.pool_cmb[o] = cmb_local;
        }
        if(tid == 0) {
            P.unit_cnt[blockIdx.x] = nn;
            if(s_matches) atomicAdd(P.combo_matches + ud.combo, s_matches);
            atomicAdd(P.stats + 0, (unsigned long long) s_driver_ids);
            atomicAdd(P.stats + 1, (unsigned long long) s_probe_blocks * kBlock);
            atomicAdd(P.stats + 2, (unsigned long long) s_matches);
        }
    }
}

#ifndef TSGPU_KW_SEARCH_ONLY          // kw_regscore.cu compiles kw_search_kernel alone
// ---------------------------------------------------------------------------------------------------------------
// KV record as in include/tsgpu.h (56 bytes)
struct KVOut {
    uint64_t key, distinct_key;
    int64_t  scores[3];
    int64_t  text_match_score;
    float    vector_distance;
    int8_t   match_score_index;
    uint8_t  pad0;
    uint16_t query_index;
};
static_assert(sizeof(KVOut) == 56, "tsgpu_kv layout");

// A merge group: reads the entries of units [in_begin, in_end) of one query, writes its best K (after de-duplication)
// either back to the pool as unit `out_unit` (intermediate level) or as KV records (final level).
struct MDesc {
    uint32_t q;
    uint32_t in_begin, in_end;
    uint32_t out_unit;
};

struct FinalParams {
    const QDesc* qd;
    const UDesc* ud;             // unit table: level-0 units followed by merge outputs
    const MDesc* md;             // intermediate levels only
    int64_t* pool_s0; int64_t* pool_s1; int64_t* pool_s2;
    uint32_t* pool_key;
    uint16_t* pool_cmb;
    uint32_t* unit_cnt;
    const uint32_t* combo_matches;
    KVOut* out_kv;
    uint32_t* out_count;
    uint32_t* out_found;
    uint32_t* out_searched;     // [nq] combinations with results = searched_queries.size() (may be nullptr)
    uint32_t kv_stride;
    uint32_t KP;
};

constexpr int kFinalThreads = 256;
constexpr uint32_t kMergeIn = 32;          // inputs a merge group can interleave (planning uses fan-in 16)

// shared by the intermediate and the final merge: leaves the best <= K de-duplicated entries sorted in tb[0..n)
__device__ uint32_t merge_units(const TopBuf& tb, uint32_t N2, uint32_t K, bool multi, const UDesc* ud, const uint32_t* unit_cnt,
                                uint32_t u_begin, uint32_t u_end, const int64_t* p0, const int64_t* p1, const int64_t* p2,
                                const uint32_t* pk, const uint16_t* pc) {
    const uint32_t tid = threadIdx.x;
    auto reduce = [&](uint32_t n) -> uint32_t {
        uint32_t NS = 64;                          // sort the smallest power of two that covers the n held entries
        while(NS < n) NS <<= 1;
        tb_fill_invalid(tb, n, NS);
        __syncthreads();
        if(multi) {
            tb_sort<true>(tb, NS);
            // entries of one seq_id are adjacent, best first: drop the rest (Topster keeps the greater KV per key)
            bool dup[8];
            int cnt = 0;
            for(uint32_t i = tid; i < NS; i += kFinalThreads) dup[cnt++] = (i > 0 && tb.key[i] != kNone && tb.key[i] == tb.key[i - 1]);
            __syncthreads();
            cnt = 0;
            for(uint32_t i = tid; i < NS; i += kFinalThreads) if(dup[cnt++]) tb.key[i] = kNone;
            __syncthreads();
        }
        tb_sort<false>(tb, NS);
        uint32_t lo = 0, hi = NS;                 // valid entries are in front
        while(lo < hi) { const uint32_t mid = (lo + hi) >> 1; if(tb.key[mid] != kNone) lo = mid + 1; else hi = mid; }
        return lo < K ? lo : K;
    };
    uint32_t n = 0;
    const uint32_t nu = u_end - u_begin;
    if(nu <= kMergeIn) {
        // Inputs are sorted best-first, so only their heads can reach the top K. Rounds: every unit whose next entry is
        // not below the current K-th (or any unit while fewer than K are held) contributes an equal share of the free
        // slots; reduce; repeat until no unit qualifies. An entry left unread is <= its unit's last-read entry <= the
        // K-th of K distinct held keys, so it cannot be in the result; entries EQUAL to the K-th are read (the later
        // combination wins ties). Typically 2-3 reductions instead of one per 256 entries.
        __shared__ uint32_t s_cur[kMergeIn], s_take[kMergeIn], s_base[kMergeIn];
        __shared__ uint32_t s_total;
        if(tid < nu) s_cur[tid] = 0;
        __syncthreads();
        for(;;) {
            bool live = false;
            if(tid < nu) {
                const uint32_t u = u_begin + tid, c = s_cur[tid];
                if(c < unit_cnt[u]) {
                    live = true;
                    if(n >= K) {                     // tb[0..n) is sorted and n == K: compare with the K-th
                        const uint32_t o = ud[u].out_off + c, t = K - 1;
                        const int64_t a0 = p0[o], a1 = p1[o], a2 = p2[o]; const uint32_t ak = pk[o];
                        bool below;
                        if(a0 != tb.s0[t]) below = a0 < tb.s0[t];
                        else if(a1 != tb.s1[t]) below = a1 < tb.s1[t];
                        else if(a2 != tb.s2[t]) below = a2 < tb.s2[t];
                        else below = ak < tb.key[t];
                        live = !below;
                    }
                }
                s_take[tid] = live ? 1u : 0u;
            }
            const uint32_t n_live = (uint32_t) __syncthreads_count(live);
            if(n_live == 0) break;
            if(tid == 0) {
                const uint32_t share = max(1u, (N2 - n) / n_live);
                uint32_t tot = 0;
                for(uint32_t i = 0; i < nu; i++) {
                    uint32_t t = 0;
                    if(s_take[i]) { const uint32_t rem = unit_cnt[u_begin + i] - s_cur[i]; t = rem < share ? rem : share; }
                    s_base[i] = tot; s_take[i] = t; tot += t;
                }
                s_total = tot;
            }
            __syncthreads();
            for(uint32_t i = 0; i < nu; i++) {
                const uint32_t take = s_take[i];
                if(take == 0) continue;
                const uint32_t o0 = ud[u_begin + i].out_off + s_cur[i], d0 = n + s_base[i];
                for(uint32_t j = tid; j < take; j += kFinalThreads) {
                    tb.s0[d0 + j] = p0[o0 + j]; tb.s1[d0 + j] = p1[o0 + j]; tb.s2[d0 + j] = p2[o0 + j];
                    tb.key[d0 + j] = pk[o0 + j]; tb.cmb[d0 + j] = pc[o0 + j];
                }
            }
            __syncthreads();
            if(tid < nu) s_cur[tid] += s_take[tid];
            n = reduce(n + s_total);
            __syncthreads();
        }
        return n;
    }
    for(uint32_t u = u_begin; u < u_end; u++) {
        const uint32_t cnt = unit_cnt[u];
        if(cnt == 0) continue;
        const uint32_t off = ud[u].out_off;
        uint32_t done = 0;
        while(done < cnt) {
            if(n == N2) { n = reduce(n); __syncthreads(); }
            const uint32_t take = min(cnt - done, N2 - n);
            for(uint32_t i = tid; i < take; i += kFinalThreads) {
                const uint32_t o = off + done + i;
                tb.s0[n + i] = p0[o]; tb.s1[n + i] = p1[o]; tb.s2[n + i] = p2[o];
                tb.key[n + i] = pk[o];
                tb.cmb[n + i] = pc[o];
            }
            n += take; done += take;
            __syncthreads();
        }
    }
    n = reduce(n);
    __syncthreads();
    return n;
}

__global__ void __launch_bounds__(kFinalThreads)
kw_merge_kernel(const __grid_constant__ FinalParams P) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const uint32_t KP = P.KP, N2 = 2 * KP;
    TopBuf tb;
    tb.s0 = reinterpret_cast<int64_t*>(smem_raw);
    tb.s1 = tb.s0 + N2;
    tb.s2 = tb.s1 + N2;
    tb.key = reinterpret_cast<uint32_t*>(tb.s2 + N2);
    tb.cmb = reinterpret_cast<uint16_t*>(tb.key + N2);
    tb.vd = nullptr;
    const MDesc md = P.md[blockIdx.x];
    const QDesc& qd = P.qd[md.q];
    const uint32_t K = qd.topk;
    const bool multi = (qd.combo_end - qd.combo_begin) > 1;
    const uint32_t n = merge_units(tb, N2, K, multi, P.ud, P.unit_cnt, md.in_begin, md.in_end, P.pool_s0, P.pool_s1, P.pool_s2,
                                   P.pool_key, P.pool_cmb);
    const uint32_t off = P.ud[md.out_unit].out_off;
    for(uint32_t i = threadIdx.x; i < n; i += kFinalThreads) {
        P.pool_s0[off + i] = tb.s0[i]; P.pool_s1[off + i] = tb.s1[i]; P.pool_s2[off + i] = tb.s2[i];
        P.pool_key[off + i] = tb.key[i]; P.pool_cmb[off + i] = tb.cmb[i];
    }
    if(threadIdx.x == 0) P.unit_cnt[md.out_unit] = n;
}

// One CTA per query: merge the (remaining) units of all its combinations into the final Topster content.
__global__ void __launch_bounds__(kFinalThreads)
kw_final_kernel(const __grid_constant__ FinalParams P) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const uint32_t KP = P.KP, N2 = 2 * KP;
    TopBuf tb;
    tb.s0 = reinterpret_cast<int64_t*>(smem_raw);
    tb.s1 = tb.s0 + N2;
    tb.s2 = tb.s1 + N2;
    tb.key = reinterpret_cast<uint32_t*>(tb.s2 + N2);
    tb.cmb = reinterpret_cast<uint16_t*>(tb.key + N2);
    tb.vd = nullptr;
    __shared__ uint16_t s_qidx[kMaxCombosPerQuery];
    __shared__ uint32_t s_found;

    const uint32_t q = blockIdx.x, tid = threadIdx.x;
    const QDesc qd = P.qd[q];
    const uint32_t K = qd.topk;
    const uint32_t n_combos = qd.combo_end - qd.combo_begin;
    const bool multi = n_combos > 1;
    if(tid == 0) {
        // query_index = searched_queries.size() when the combination ran = number of earlier combinations with
        // results (src/index.cpp:5575-5580)
        uint32_t qi = 0, found = 0;
        for(uint32_t c = 0; c < n_combos; c++) {
            const uint32_t m = P.combo_matches[qd.combo_begin + c];
            if(c < kMaxCombosPerQuery) s_qidx[c] = (uint16_t) qi;
            if(m) qi++;
            found += m;
        }
        s_found = found;
        if(P.out_searched) P.out_searched[q] = qi;
    }
    __syncthreads();
    const uint32_t n = merge_units(tb, N2, K, multi, P.ud, P.unit_cnt, qd.unit_begin, qd.unit_end, P.pool_s0, P.pool_s1, P.pool_s2,
                                   P.pool_key, P.pool_cmb);
    int msi = -1;
    for(int i = 0; i < 3; i++) if(qd.sort_type[i] == 1) msi = i;
    const uint32_t n_out = n < P.kv_stride ? n : P.kv_stride;
    for(uint32_t i = tid; i < n_out; i += kFinalThreads) {
        KVOut kv;
        kv.key = tb.key[i]; kv.distinct_key = tb.key[i];
        kv.scores[0] = tb.s0[i]; kv.scores[1] = tb.s1[i]; kv.scores[2] = tb.s2[i];
        kv.text_match_score = msi >= 0 ? kv.scores[msi] : 0;
        kv.vector_distance = -1.0f;
        kv.match_score_index = (int8_t) msi;
        kv.pad0 = 0;
        const uint16_t c = tb.cmb[i];
        kv.query_index = c < kMaxCombosPerQuery ? s_qidx[c] : 0;
        P.out_kv[(size_t) q * P.kv_stride + i] = kv;
    }
    if(tid == 0) {
        P.out_count[q] = n_out;
        P.out_found[q] = (multi && qd.found_bitmap) ? 0 : s_found;   // multi: found_popcount_kernel adds the union's popcount
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Index::search_wildcard (src/index.cpp:6616-6800): the reference partitions the filter ids over `concurrency` threads,
// each with its own Topster, then aggregates. Here a unit is a run of 128-id tiles of the query's id set (its filter
// ids, or the id range [0, n_docs) when it has no filter); units feed the same pool / merge / final kernels as the
// keyword path (pseudo-combination == query).
struct WcParams {
    const QDesc* qd;
    const UDesc* ud;                   // ud.combo == query index
    const uint32_t* const* q_ids;      // [nq] device id arrays or nullptr (= identity)
    const uint32_t* q_nids;            // [nq]
    const int64_t* const* q_scores;    // [nq] per-id match scores aligned with q_ids (do_phrase_search) or nullptr = the wildcard's 100
    int64_t* pool_s0; int64_t* pool_s1; int64_t* pool_s2;
    uint32_t* pool_key; uint16_t* pool_cmb;
    uint32_t* unit_cnt; uint32_t* combo_matches;
    long long* q_thr;
    uint32_t KP;
};

// DEEP: as kw_search_kernel<.., DEEP>: every matched id goes to the query's slice of the deep buffer (P.pool_*, cursor
// P.q_thr[q]); launched with KP = 0 over the units of deep queries only.
template <bool DEEP = false>
__global__ void __launch_bounds__(kThreads)
wc_unit_kernel(const __grid_constant__ WcParams P) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const uint32_t KP = P.KP, N2 = 2 * KP;
    TopBuf tb;
    tb.s0 = reinterpret_cast<int64_t*>(smem_raw);
    tb.s1 = tb.s0 + N2; tb.s2 = tb.s1 + N2;
    tb.key = reinterpret_cast<uint32_t*>(tb.s2 + N2);
    tb.cmb = nullptr; tb.vd = nullptr;
    __shared__ uint32_t s_warp[8];
    __shared__ int64_t thr[3];
    __shared__ uint32_t thr_key, s_n, s_have_thr, s_matches;
    const uint32_t tid = threadIdx.x;
    const UDesc ud = P.ud[blockIdx.x];
    const uint32_t q = ud.combo;
    const QDesc qd = P.qd[q];
    const uint32_t K = qd.topk;
    const uint32_t* ids = P.q_ids[q];
    const uint32_t n_ids = P.q_nids[q];
    SortSpec SS;
    for(int i = 0; i < 3; i++) { SS.type[i] = qd.sort_type[i]; SS.order[i] = qd.sort_order[i]; SS.missing_first[i] = qd.missing_first[i]; SS.col[i] = qd.sort_col[i]; }
    long long* const gthr_p = P.q_thr + q;
    if(tid == 0) { s_n = 0; s_have_thr = 0; s_matches = 0; }
    __syncthreads();
    for(uint32_t tile = ud.tile_begin; tile < ud.tile_end; tile++) {
        const uint32_t i = tile * kThreads + tid;
        bool keep = i < n_ids;
        uint32_t id = 0;
        int64_t sc[3] = {0, 0, 0};
        if(keep) {
            id = ids ? __ldg(ids + i) : i;
            if(qd.n_excl && excluded(qd.excl, qd.n_excl, id)) keep = false;
        }
        const bool matched = keep;
        if(keep) {
            const int64_t ms = (P.q_scores && P.q_scores[q]) ? __ldg(P.q_scores[q] + i) : 100;      // src/index.cpp:6727-6729; phrase-only: :6045
            compute_sort_scores(SS, id, ms, 0.0f, sc);
            if constexpr (!DEEP) {
                const long long gthr = *reinterpret_cast<volatile long long*>(gthr_p);
                keep = sc[0] >= gthr;
                if(keep && s_have_thr) keep = kv_greater(sc[0], sc[1], sc[2], id, thr[0], thr[1], thr[2], thr_key);
            }
        }
        uint32_t m_total, a_total;
        cta_rank(matched, s_warp, &m_total);
        const uint32_t arank = cta_rank(keep, s_warp, &a_total);
        if constexpr (DEEP) {
            if(tid == 0) { s_matches += m_total; if(a_total) thr[0] = (int64_t) atomicAdd(reinterpret_cast<unsigned long long*>(gthr_p), (unsigned long long) a_total); }
            __syncthreads();
            if(keep) {
                const size_t o = (size_t) thr[0] + arank;
                P.pool_s0[o] = sc[0]; P.pool_s1[o] = sc[1]; P.pool_s2[o] = sc[2]; P.pool_key[o] = id; P.pool_cmb[o] = 0;
            }
            continue;
        }
        const uint32_t n0 = s_n;
        if(keep) { const uint32_t slot = n0 + arank; tb.s0[slot] = sc[0]; tb.s1[slot] = sc[1]; tb.s2[slot] = sc[2]; tb.key[slot] = id; }
        __syncthreads();
        if(tid == 0) { s_n = n0 + a_total; s_matches += m_total; }
        __syncthreads();
        if(s_n + kThreads > N2) {
            const uint32_t n = s_n;
            tb_fill_invalid(tb, n, N2);
            __syncthreads();
            tb_sort<false>(tb, N2);
            if(tid == 0) {
                const uint32_t nn = n < K ? n : K;
                s_n = nn;
                if(nn == K) {
                    s_have_thr = 1; thr[0] = tb.s0[K - 1]; thr[1] = tb.s1[K - 1]; thr[2] = tb.s2[K - 1]; thr_key = tb.key[K - 1];
                    atomicMax(gthr_p, (long long) tb.s0[K - 1]);
                }
            }
            __syncthreads();
        }
    }
    __syncthreads();
    if constexpr (DEEP) {
        if(tid == 0 && s_matches) atomicAdd(P.combo_matches + q, s_matches);
        return;
    }
    const uint32_t n = s_n;
    uint32_t nn = n;
    if(n > 1) {                                   // always sorted best-first (see merge_units)
        uint32_t NS = 2;
        while(NS < n) NS <<= 1;
        tb_fill_invalid(tb, n, NS);
        __syncthreads();
        tb_sort<false>(tb, NS);
        if(n > K) nn = K;
    }
    for(uint32_t i = tid; i < nn; i += kThreads) {
        const uint32_t o = ud.out_off + i;
        P.pool_s0[o] = tb.s0[i]; P.pool_s1[o] = tb.s1[i]; P.pool_s2[o] = tb.s2[i]; P.pool_key[o] = tb.key[i];
        P.pool_cmb[o] = 0;
    }
    if(tid == 0) { P.unit_cnt[blockIdx.x] = nn; if(s_matches) atomicAdd(P.combo_matches + q, s_matches); }
}

// found = |union of result ids| for queries with several combinations (the reference ORs id_buff into
// all_result_ids, src/index.cpp:5081-5090). grid = (queries, splits); 16-byte loads; every word is cleared after it is
// counted, so the bitmaps are all-zero again for the next call and no memset pass is needed. out_found[q] was zeroed by
// kw_final_kernel.
__global__ void __launch_bounds__(256)
found_popcount_kernel(const QDesc* qd, const uint32_t* multi_q, uint32_t n_vec, uint32_t* out_found, int clear) {
    const uint32_t q = multi_q[blockIdx.x];
    uint4* bm = reinterpret_cast<uint4*>(qd[q].found_bitmap);
    const uint32_t per = (n_vec + gridDim.y - 1) / gridDim.y;
    const uint32_t v0 = blockIdx.y * per, v1 = min(n_vec, v0 + per);
    uint32_t c = 0;
    for(uint32_t i = v0 + threadIdx.x; i < v1; i += blockDim.x) {
        const uint4 w = bm[i];
        if(w.x | w.y | w.z | w.w) {
            c += __popc(w.x) + __popc(w.y) + __popc(w.z) + __popc(w.w);
            if(clear) bm[i] = make_uint4(0, 0, 0, 0);
        }
    }
    for(int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    __shared__ uint32_t s[8];
    if((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = c;
    __syncthreads();
    if(threadIdx.x == 0) { uint32_t t = 0; for(int i = 0; i < 8; i++) t += s[i]; if(t) atomicAdd(out_found + q, t); }
}

// sorted ids -> bitmap (filter_result_iterator_t::to_filter_id_array() mirrored as bits)
__global__ void bitmap_from_ids_kernel(const uint32_t* __restrict__ ids, size_t n, uint32_t* __restrict__ bitmap, uint32_t n_docs) {
    const size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if(i < n) { const uint32_t id = ids[i]; if(id < n_docs) atomicOr(bitmap + (id >> 5), 1u << (id & 31)); }
}

// ---------------------------------------------------------------------------------------------------------------
// tsgpu_intersect / tsgpu_phrase_matches: per-tile flags -> (count, compacted ids) -> scan -> gather.
struct IsectParams {
    uint32_t field;          // index field id
    uint32_t k;
    uint32_t lists[kMaxTokens];
    uint32_t driver;         // index into lists (intersect); unused for phrase
    const uint32_t* ids;     // phrase: candidate ids (ascending); nullptr for intersect
    size_t n_ids;
    uint32_t n_tiles;
    uint32_t* tile_cnt;      // [n_tiles]
    uint32_t* tile_ids;      // [n_tiles*128]
    int phrase;              // 0 intersect, 1 phrase, 2 exact (get_exact_matches), 3 prefix (get_prefix_matches)
};

__global__ void __launch_bounds__(kThreads)
isect_tiles_kernel(const __grid_constant__ IndexDev ix, const __grid_constant__ IsectParams P) {
    __shared__ uint32_t l_blk0[kMaxTokens], l_blk1[kMaxTokens], l_lo[kMaxTokens], l_hi[kMaxTokens];
    __shared__ unsigned long long l_df[kMaxTokens], l_base[kMaxTokens];
    __shared__ uint32_t s_warp[8];
    const DevField& g = ix.fields[P.field];
    const uint32_t tid = threadIdx.x, tile = blockIdx.x;
    if(tid < P.k) {
        const uint32_t l = P.lists[tid];
        l_blk0[tid] = g.list_blk_off[l]; l_blk1[tid] = g.list_blk_off[l + 1] - 1;
        l_base[tid] = g.list_off[l]; l_df[tid] = g.list_off[l + 1] - g.list_off[l];
    }
    __syncthreads();
    uint32_t id = 0, first = 0, tmax = 0, cnt = 0;
    uint32_t own = kNone;      // posting index of the candidate in the driver list (intersect)
    if(!P.phrase) {
        const uint32_t d = P.driver;
        const uint32_t b = l_blk0[d] + tile;
        cnt = block_count(b, l_blk0[d], l_df[d]);
        first = __ldg(g.blk_first + b);
        const unsigned long long info = __ldg(reinterpret_cast<const unsigned long long*>(g.blk_info) + b);
        const uint32_t bits = (uint32_t) (info >> 40) & 0xFF;
        const uint32_t* w = g.packed + (info & 0xFFFFFFFFFFull);
        id = first + unpack_at(w, bits, tid < cnt ? tid : 0);
        tmax = first + unpack_at(w, bits, cnt - 1);
        own = tile * kBlock + tid;
    } else {
        const size_t base = (size_t) tile * kBlock;
        cnt = (uint32_t) min((size_t) kBlock, P.n_ids - base);
        id = P.ids[base + (tid < cnt ? tid : 0)];
        first = P.ids[base];
        tmax = P.ids[base + cnt - 1];
    }
    bool alive = tid < cnt;
    if(tid < 2 * P.k) {
        const uint32_t j = tid >> 1;
        const uint32_t r = gallop_block(g.blk_first, l_blk0[j], l_blk1[j], (tid & 1) ? tmax : first);
        if(tid & 1) l_hi[j] = r; else l_lo[j] = (r == kNone ? l_blk0[j] : r);
    }
    __syncthreads();
    uint32_t hidx[kMaxTokens];
    for(uint32_t j = 0; j < P.k; j++) {
        uint32_t h = kNone;
        const uint32_t dslot = g.list_dense ? g.list_dense[P.lists[j]] : kNone;
        if(!P.phrase && j == P.driver) h = own;
        else if(dslot != kNone) { if(alive && dense_test(g, dslot, id)) h = dense_rank_of(g, dslot, id); }
        else if(alive && l_hi[j] != kNone) {
            const uint32_t bb = find_block(g.blk_first, l_lo[j], l_hi[j], id);
            if(bb != kNone) {
                const uint32_t ii = probe_block(g, bb, block_count(bb, l_blk0[j], l_df[j]), id);
                if(ii != kNone) h = (bb - l_blk0[j]) * kBlock + ii;
            }
        }
        hidx[j] = h;
        if(h == kNone) alive = false;
    }
    if(alive && P.phrase) {
        RawTok toks[kMaxTokens];
        for(uint32_t j = 0; j < P.k; j++) {
            const unsigned long long p = l_base[j] + hidx[j];
            const unsigned long long o0 = g.pos_off[p], o1 = g.pos_off[p + 1];
            toks[j].p = g.positions + o0; toks[j].n = (uint32_t) (o1 - o0);
        }
        if(P.phrase == 1) alive = phrase_match_doc(toks, (int) P.k);
        else alive = positional_match_doc(toks, (int) P.k, (g.is_array & kFieldIsArray) != 0, P.phrase == 2);
    }
    uint32_t total;
    const uint32_t rank = cta_rank(alive, s_warp, &total);
    if(alive) P.tile_ids[(size_t) tile * kBlock + rank] = id;
    if(tid == 0) P.tile_cnt[tile] = total;
}

// posting_list_t::contains_atleast_one (src/posting_list.cpp:1090-1112; compact form src/posting.cpp:215): is any of the
// ascending target ids a member of list l? One probe per target id (skip index + packed block, or the dense bitmap).
__global__ void __launch_bounds__(256)
contains_any_kernel(const __grid_constant__ IndexDev ix, uint32_t field, uint32_t l, const uint32_t* __restrict__ ids, size_t n, int* __restrict__ out) {
    const DevField& g = ix.fields[field];
    const uint32_t b0 = g.list_blk_off[l], b1 = g.list_blk_off[l + 1];
    bool hit = false;
    if(b1 > b0)
        for(size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n && !hit; i += (size_t) gridDim.x * blockDim.x)
            hit = probe_list(g, l, b0, b1 - 1, ids[i]) != kNone;
    if(__any_sync(0xffffffffu, hit) && (threadIdx.x & 31) == 0) atomicExch(out, 1);
}

// ---------------------------------------------------------------------------------------------------------------
// filter_by evaluated on the device (SURVEY 8 f-2). A numeric / bool leaf (filter_result_iterator_t over num_tree_t,
// src/filter_result_iterator.cpp:1507-1700, src/num_tree.cpp:35-250) is one pass over the field's dense column: 32 docs per
// thread word, straight into the filter bitmap in HBM — no id list crosses the host. A doc without a value (INT64_MIN, it is not
// in the reference's tree) matches no comparator; `!=` is "every doc minus the equal ones" (apply_not_equals), so it does
// match docs without a value, as in the reference.
enum { kCmpEq = 0, kCmpNe = 1, kCmpLt = 2, kCmpLe = 3, kCmpGt = 4, kCmpGe = 5, kCmpRange = 6 };
__global__ void __launch_bounds__(256)
filter_numeric_kernel(const int64_t* __restrict__ col, uint32_t n_docs, int op, int64_t v1, int64_t v2, uint32_t* __restrict__ bitmap) {
    const uint32_t wi = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t base = wi << 5;
    if(base >= n_docs) return;
    uint32_t w = 0;
    const uint32_t n = min(32u, n_docs - base);
    for(uint32_t k = 0; k < n; k++) {
        const int64_t v = __ldg(col + base + k);
        const bool has = v != INT64_MIN;
        bool m;
        switch(op) {
            case kCmpEq: m = has && v == v1; break;
            case kCmpNe: m = !(has && v == v1); break;
            case kCmpLt: m = has && v < v1; break;
            case kCmpLe: m = has && v <= v1; break;
            case kCmpGt: m = has && v > v1; break;
            case kCmpGe: m = has && v >= v1; break;
            default: m = has && v >= v1 && v <= v2; break;
        }
        w |= (m ? 1u : 0u) << k;
    }
    bitmap[wi] = w;
}
// the AND / OR / AND-NOT nodes of the filter tree (filter_result_iterator_t::and_filter_iterators / or_filter_iterators) on bitmaps
__global__ void __launch_bounds__(256)
filter_combine_kernel(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, uint32_t n_words, int op, uint32_t* __restrict__ out) {
    const uint32_t wi = blockIdx.x * blockDim.x + threadIdx.x;
    if(wi >= n_words) return;
    const uint32_t x = a[wi], y = b[wi];
    out[wi] = op == 0 ? (x & y) : op == 1 ? (x | y) : (x & ~y);
}

// single-CTA exclusive scan of tile counts (n_tiles <= a few hundred thousand)
__global__ void __launch_bounds__(1024)
scan_tiles_kernel(const uint32_t* __restrict__ cnt, uint32_t n, unsigned long long* __restrict__ off, unsigned long long* total) {
    __shared__ unsigned long long s[1024];
    __shared__ unsigned long long carry;
    if(threadIdx.x == 0) carry = 0;
    __syncthreads();
    for(uint32_t base = 0; base < n; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        const unsigned long long v = i < n ? cnt[i] : 0;
        s[threadIdx.x] = v;
        __syncthreads();
        for(uint32_t d = 1; d < 1024; d <<= 1) {
            const unsigned long long t = threadIdx.x >= d ? s[threadIdx.x - d] : 0;
            __syncthreads();
            s[threadIdx.x] += t;
            __syncthreads();
        }
        if(i < n) off[i] = carry + s[threadIdx.x] - v;
        __syncthreads();
        if(threadIdx.x == 0) carry += s[1023];
        __syncthreads();
    }
    if(threadIdx.x == 0) *total = carry;
}

__global__ void __launch_bounds__(kThreads)
gather_tiles_kernel(const uint32_t* __restrict__ cnt, const unsigned long long* __restrict__ off,
                    const uint32_t* __restrict__ tile_ids, uint32_t* __restrict__ out, size_t cap) {
    const uint32_t tile = blockIdx.x;
    const uint32_t c = cnt[tile];
    const unsigned long long o = off[tile];
    if(threadIdx.x < c && o + threadIdx.x < cap) out[o + threadIdx.x] = tile_ids[(size_t) tile * kBlock + threadIdx.x];
}

// ---------------------------------------------------------------------------------------------------------------
// tsgpu_ids_setop: ArrayUtils::and_scalar / or_scalar / exclude_scalar (src/array_utils.cpp:4-170) on strictly
// ascending id arrays, done in the bitmap domain: ids -> bits, one word-parallel pass combines the bitmaps and counts
// the result per 128-word tile, scan, then every thread writes the ids of its own word in place.
__global__ void bitmap_from_sorted_ids_kernel(const uint32_t* __restrict__ ids, size_t n, uint32_t* __restrict__ bitmap,
                                              uint32_t n_docs, uint32_t* __restrict__ bad) {
    const size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= n) return;
    const uint32_t id = ids[i];
    if(id >= n_docs || (i && ids[i - 1] >= id)) { *bad = 1; return; }
    atomicOr(bitmap + (id >> 5), 1u << (id & 31));
}

__global__ void __launch_bounds__(kThreads)
setop_count_kernel(uint32_t* __restrict__ A, const uint32_t* __restrict__ B, uint32_t n_words, int op, uint32_t* __restrict__ tile_cnt) {
    __shared__ uint32_t s_warp[kThreads / 32];
    const uint32_t wi = blockIdx.x * kThreads + threadIdx.x;
    uint32_t w = 0;
    if(wi < n_words) {
        const uint32_t a = A[wi], b = B[wi];
        w = op == 0 ? (a & b) : op == 1 ? (a | b) : (a & ~b);
        A[wi] = w;
    }
    uint32_t c = __popc(w);
    for(int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = c;
    __syncthreads();
    if(threadIdx.x == 0) { uint32_t t = 0; for(int i = 0; i < kThreads / 32; i++) t += s_warp[i]; tile_cnt[blockIdx.x] = t; }
}

__global__ void __launch_bounds__(kThreads)
setop_extract_kernel(const uint32_t* __restrict__ R, uint32_t n_words, const unsigned long long* __restrict__ tile_off,
                     uint32_t* __restrict__ out, size_t cap) {
    __shared__ uint32_t s_warp[kThreads / 32];
    const uint32_t wi = blockIdx.x * kThreads + threadIdx.x, lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    uint32_t w = wi < n_words ? R[wi] : 0;
    const uint32_t c = __popc(w);
    uint32_t incl = c;                                   // inclusive warp scan of the per-word counts
    for(int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if((int) lane >= o) incl += t; }
    if(lane == 31) s_warp[wp] = incl;
    __syncthreads();
    uint32_t before = 0;
    for(uint32_t i = 0; i < wp; i++) before += s_warp[i];
    unsigned long long o = tile_off[blockIdx.x] + before + incl - c;
    while(w) {
        const uint32_t bit = __ffs(w) - 1;
        w &= w - 1;
        if(o < cap) out[o] = (wi << 5) | bit;
        o++;
    }
}

#endif  // TSGPU_KW_SEARCH_ONLY

}  // namespace tsk
