// Deep Topster: selection for a query whose Topster is larger than TSGPU_MAX_TOPK (TSGPU_QFLAG_DEEP_TOPSTER).
//
// The ordinary path keeps each unit's best K in a shared-memory buffer of 2*KP slots and merges the units' heads, so K is
// bounded by shared memory. A deep query instead has kw_search_kernel<.., DEEP = true> / wc_unit_kernel<true> append every
// scored match (s0, s1, s2, key, combination) to the query's slice of a device buffer, and the kernels below turn that
// slice into the Topster's content:
//   de-duplicate (several combinations with matches only): sort by (seq_id ascending, KV order descending, combination
//       descending) and keep the head of every seq_id's run -- Topster::add keeps the greater KV per key
//       (include/topster.h:392-406), and a later combination wins an exact tie as in merge_units;
//   select: sort the (now distinct-key) entries by the KV order (s0, s1, s2, key) descending, a total order, so the result
//       does not depend on the order in which the units emitted their entries;
//   write: the first min(K, entries, kv_stride) as tsgpu_kv records, exactly as kw_final_kernel writes them.
// Both sorts are CUB radix sorts of a 32-byte struct key; the host side is run_deep_select() in tsgpu.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <cuda/std/tuple>
#include "kw_kernels.cuh"

namespace tsk {

struct DeepEntry {
    int64_t  s0, s1, s2;
    uint32_t key;                  // seq_id; ~seq_id while the de-duplication order is in force
    uint16_t cmb;                  // combination index local to the query
    uint16_t pad;
};
static_assert(sizeof(DeepEntry) == 32, "DeepEntry layout");

// Topster::sort() order: scores[0..2] then key, all descending (kv_greater)
struct DeepKvOrder {
    __host__ __device__ ::cuda::std::tuple<int64_t&, int64_t&, int64_t&, uint32_t&> operator()(DeepEntry& e) const {
        return {e.s0, e.s1, e.s2, e.key};
    }
};
// de-duplication order, sorted descending with key = ~seq_id: seq_id ascending, then the best entry of a seq_id first
struct DeepKeyOrder {
    __host__ __device__ ::cuda::std::tuple<uint32_t&, int64_t&, int64_t&, int64_t&, uint16_t&> operator()(DeepEntry& e) const {
        return {e.key, e.s0, e.s1, e.s2, e.cmb};
    }
};

// The emitted SoA slice [0, n) -> DeepEntry; by_key stores ~seq_id for the de-duplication sort.
__global__ void __launch_bounds__(256)
deep_pack_kernel(const int64_t* __restrict__ s0, const int64_t* __restrict__ s1, const int64_t* __restrict__ s2,
                 const uint32_t* __restrict__ key, const uint16_t* __restrict__ cmb, size_t n, int by_key, DeepEntry* __restrict__ out) {
    for(size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
        DeepEntry e;
        e.s0 = s0[i]; e.s1 = s1[i]; e.s2 = s2[i];
        e.key = by_key ? ~key[i] : key[i];
        e.cmb = cmb[i]; e.pad = 0;
        out[i] = e;
    }
}

// After the de-duplication sort: flag the head of every seq_id's run and restore the seq_id (for DeviceSelect::Flagged).
__global__ void __launch_bounds__(256)
deep_heads_kernel(const DeepEntry* __restrict__ in, size_t n, DeepEntry* __restrict__ out, uint8_t* __restrict__ head) {
    for(size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
        DeepEntry e = in[i];
        head[i] = (i == 0 || in[i - 1].key != e.key) ? 1 : 0;
        e.key = ~e.key;
        out[i] = e;
    }
}

// First n_out entries of the sorted slice -> tsgpu_kv records of query q (kw_final_kernel's record layout and query_index).
__global__ void __launch_bounds__(256)
deep_write_kernel(const DeepEntry* __restrict__ in, uint32_t n_out, const QDesc* __restrict__ qds, uint32_t q,
                  const uint32_t* __restrict__ combo_matches, KVOut* __restrict__ out_kv, uint32_t kv_stride, uint32_t* __restrict__ out_count) {
    __shared__ uint16_t s_qidx[kMaxCombosPerQuery];
    const QDesc& qd = qds[q];
    const uint32_t n_combos = qd.combo_end - qd.combo_begin;
    if(threadIdx.x == 0) {
        // query_index = number of earlier combinations with results (src/index.cpp:5575-5580)
        uint32_t qi = 0;
        for(uint32_t c = 0; c < n_combos && c < (uint32_t) kMaxCombosPerQuery; c++) {
            s_qidx[c] = (uint16_t) qi;
            if(combo_matches[qd.combo_begin + c]) qi++;
        }
    }
    __syncthreads();
    int msi = -1;
    for(int i = 0; i < 3; i++) if(qd.sort_type[i] == 1) msi = i;
    for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_out; i += gridDim.x * blockDim.x) {
        const DeepEntry e = in[i];
        KVOut kv;
        kv.key = e.key; kv.distinct_key = e.key;
        kv.scores[0] = e.s0; kv.scores[1] = e.s1; kv.scores[2] = e.s2;
        kv.text_match_score = msi >= 0 ? kv.scores[msi] : 0;
        kv.vector_distance = -1.0f;
        kv.match_score_index = (int8_t) msi;
        kv.pad0 = 0;
        kv.query_index = e.cmb < kMaxCombosPerQuery ? s_qidx[e.cmb] : 0;
        out_kv[(size_t) q * kv_stride + i] = kv;
    }
    if(blockIdx.x == 0 && threadIdx.x == 0) out_count[q] = n_out;
}

}  // namespace tsk
