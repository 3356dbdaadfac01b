// Device side of the mirror's maintenance calls (tsgpu_index_compact_field, tsgpu_index_reserve_docs; host code in
// mirror_host.inc). Compaction never re-encodes a posting: packed blocks are self-contained (word-aligned, relative to their
// blk_first, bit width in blk_info), so a field's live lists are a segmented gather of its arrays with a few offsets rebased.
//
// Work split: one CTA per fixed-size chunk of the OUTPUT array, not one per list — a field holds a few huge lists and a long tail
// of tiny ones. Segment s (a list, or a dense row) occupies output [dst[s], dst[s+1]) and reads input from src[s]; a CTA finds
// the segments overlapping its chunk with two binary searches over dst, then every thread writes 16 contiguous bytes per step
// (and reads them as one 16-byte load when the group lies inside one segment at a 16-byte aligned source). HBM-bound copying.
#pragma once
#include <stdint.h>
#include "postings_device.cuh"

namespace tsmir {

constexpr int kThreads = 256;
constexpr int kGroupsPerThread = 8;                  // 16-byte groups per thread per chunk: a chunk is 32 KB of output
constexpr unsigned long long kWordMask = 0xFFFFFFFFFFull;
enum { kCopy = 0, kRebase = 1, kRebase40 = 2 };     // value as is / + (rb_dst - rb_src) / the same on the low 40 bits

// last i in [lo, hi] with a[i] <= v (a ascending, a[lo] <= v)
__device__ __forceinline__ uint32_t last_le(const unsigned long long* __restrict__ a, uint32_t lo, uint32_t hi, unsigned long long v) {
    while(lo < hi) {
        const uint32_t mid = lo + ((hi - lo + 1) >> 1);
        if(a[mid] <= v) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// Per live list i (old id live[i]): where its blocks, postings, packed words and raw offsets start in the old arrays, and how
// many words / offsets it has (word_cnt[n] = pos_cnt[n] = 0, so an exclusive scan over n + 1 entries ends in the totals).
// Blocks are laid out back to back with cumulative word offsets, appended ones included, so a list's words run from its first
// block's offset to the next block's (n_words after the last block).
__global__ void __launch_bounds__(kThreads)
extents_kernel(const uint32_t* __restrict__ live, uint32_t n, const unsigned long long* __restrict__ list_off, const uint32_t* __restrict__ list_blk_off,
               const unsigned long long* __restrict__ blk_info, uint32_t n_blocks, unsigned long long n_words, const unsigned long long* __restrict__ pos_off,
               const uint32_t* __restrict__ new_blk_off, unsigned long long* __restrict__ blk_src, unsigned long long* __restrict__ blk_dst,
               unsigned long long* __restrict__ post_src, unsigned long long* __restrict__ word_src, unsigned long long* __restrict__ word_cnt,
               unsigned long long* __restrict__ pos_src, unsigned long long* __restrict__ pos_cnt) {
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if(i > n) return;
    blk_dst[i] = new_blk_off[i];
    if(i == n) { word_cnt[n] = 0; pos_cnt[n] = 0; return; }
    const uint32_t l = live[i];
    const uint32_t b0 = list_blk_off[l], b1 = list_blk_off[l + 1];
    const unsigned long long w0 = b0 < n_blocks ? (blk_info[b0] & kWordMask) : n_words;
    const unsigned long long w1 = b1 < n_blocks ? (blk_info[b1] & kWordMask) : n_words;
    const unsigned long long p0 = list_off[l], p1 = list_off[l + 1];
    const unsigned long long q0 = pos_off[p0], q1 = pos_off[p1];
    blk_src[i] = b0; post_src[i] = p0;
    word_src[i] = w0; word_cnt[i] = w1 - w0;
    pos_src[i] = q0; pos_cnt[i] = q1 - q0;
}

// out[0 .. total) = the segments of `in` named by (src, dst), values rebased per MODE
template <class T, int MODE>
__global__ void __launch_bounds__(kThreads)
gather_kernel(const T* __restrict__ in, T* __restrict__ out, unsigned long long total, const unsigned long long* __restrict__ src,
              const unsigned long long* __restrict__ dst, uint32_t n_seg, const unsigned long long* __restrict__ rb_src,
              const unsigned long long* __restrict__ rb_dst) {
    constexpr int V = 16 / sizeof(T);
    constexpr unsigned long long kChunk = (unsigned long long) kThreads * V * kGroupsPerThread;
    __shared__ uint32_t s_lo, s_hi;
    const unsigned long long c0 = (unsigned long long) blockIdx.x * kChunk;
    if(c0 >= total) return;
    const unsigned long long c1 = c0 + kChunk < total ? c0 + kChunk : total;
    if(threadIdx.x == 0) s_lo = last_le(dst, 0, n_seg - 1, c0);
    if(threadIdx.x == 32) s_hi = last_le(dst, 0, n_seg - 1, c1 - 1);
    __syncthreads();
    const uint32_t lo = s_lo, hi = s_hi;
    for(unsigned long long j0 = c0 + (unsigned long long) threadIdx.x * V; j0 < c1; j0 += (unsigned long long) kThreads * V) {
        uint32_t s = lo == hi ? lo : last_le(dst, lo, hi, j0);
        T v[V];
        const unsigned long long from = src[s] + (j0 - dst[s]);
        if(j0 + V <= dst[s + 1] && (from % V) == 0) {      // one segment, 16-byte aligned source (arrays are cudaMalloc'd): one load
            const uint4 x = *reinterpret_cast<const uint4*>(in + from);
            *reinterpret_cast<uint4*>(v) = x;
            if(MODE != kCopy) {
                const unsigned long long d = rb_dst[s] - rb_src[s];
#pragma unroll
                for(int k = 0; k < V; k++) v[k] = MODE == kRebase ? (T) (v[k] + d) : (T) ((((v[k] & kWordMask) + d) & kWordMask) | (v[k] & ~kWordMask));
            }
        } else {
#pragma unroll
            for(int k = 0; k < V; k++) {
                const unsigned long long j = j0 + k;
                if(j >= c1) { v[k] = 0; continue; }
                while(s < hi && dst[s + 1] <= j) s++;
                T x = in[src[s] + (j - dst[s])];
                if(MODE != kCopy) {
                    const unsigned long long d = rb_dst[s] - rb_src[s];
                    x = MODE == kRebase ? (T) (x + d) : (T) ((((x & kWordMask) + d) & kWordMask) | (x & ~kWordMask));
                }
                v[k] = x;
            }
        }
        if(j0 + V <= c1) *reinterpret_cast<uint4*>(out + j0) = *reinterpret_cast<const uint4*>(v);
        else for(int k = 0; j0 + k < c1; k++) out[j0 + k] = v[k];
    }
}

// one gather on `st`; counts its launch in *launches
template <class T, int MODE>
inline cudaError_t launch_gather(cudaStream_t st, unsigned long long* launches, const void* in, void* out, unsigned long long total,
                                 const unsigned long long* src, const unsigned long long* dst, uint32_t n_seg,
                                 const unsigned long long* rb_src = nullptr, const unsigned long long* rb_dst = nullptr) {
    if(total == 0 || n_seg == 0) return cudaSuccess;
    const unsigned long long chunk = (unsigned long long) kThreads * (16 / sizeof(T)) * kGroupsPerThread;
    gather_kernel<T, MODE><<<(unsigned) ((total + chunk - 1) / chunk), kThreads, 0, st>>>(reinterpret_cast<const T*>(in), reinterpret_cast<T*>(out), total,
                                                                                         src, dst, n_seg, rb_src, rb_dst);
    (*launches)++;
    return cudaGetLastError();
}

// kFieldPlainOk / kFieldPos16 over every posting of a (compacted) plain field: bit 1 = a posting's offsets are malformed,
// bit 2 = an offset exceeds 65535 — the per-posting predicates of the loader, as one reduction
__global__ void __launch_bounds__(kThreads)
plain_flags_kernel(const unsigned long long* __restrict__ pos_off, const uint32_t* __restrict__ positions, unsigned long long n_post, uint32_t* __restrict__ bad) {
    uint32_t b = 0;
    for(unsigned long long p = (unsigned long long) blockIdx.x * kThreads + threadIdx.x; p < n_post; p += (unsigned long long) gridDim.x * kThreads) {
        const unsigned long long a = pos_off[p], e = pos_off[p + 1];
        if(!tsdev::offsets_wellformed(positions, a, e)) b |= 1u;
        if(!tsdev::offsets_fit_u16(positions, a, e)) b |= 2u;
    }
    b = __reduce_or_sync(0xFFFFFFFFu, b);
    if((threadIdx.x & 31) == 0 && b) atomicOr(bad, b);
}

__global__ void fill_i64_kernel(long long* __restrict__ p, unsigned long long n, long long v) {
    for(unsigned long long i = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long) gridDim.x * blockDim.x) p[i] = v;
}

// p[begin .. end) = p[begin - 1]: facet doc_off rows of documents that have no values
__global__ void extend_u64_kernel(unsigned long long* __restrict__ p, unsigned long long begin, unsigned long long end) {
    const unsigned long long v = p[begin - 1];
    for(unsigned long long i = begin + (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; i < end; i += (unsigned long long) gridDim.x * blockDim.x) p[i] = v;
}

// rank directory entries [g0, dg) of every dense slot: no bit is set past the old capacity, so each is the list's df
__global__ void rank_tail_kernel(uint32_t* __restrict__ rank, uint32_t n_dense, uint32_t dg, uint32_t g0, const uint32_t* __restrict__ slot_df) {
    const uint32_t w = dg - g0;
    for(unsigned long long i = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; i < (unsigned long long) n_dense * w; i += (unsigned long long) gridDim.x * blockDim.x) {
        const uint32_t s = (uint32_t) (i / w), g = g0 + (uint32_t) (i % w);
        rank[(size_t) s * dg + g] = slot_df[s];
    }
}

}  // namespace tsmir
