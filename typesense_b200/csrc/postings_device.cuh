// Device posting-list layout and block probe, written as __host__ __device__ code (see score_device.cuh for why).
//
// Replaces, for reading: posting_list_t::block_t + iterator_t (include/posting_list.h:56-127,
// src/posting_list.cpp:1954-2061) and the FOR containers behind them (src/sorted_array.cpp, libfor).
//
// Layout per field (all arrays in HBM, built by tsgpu_index_load_field, extended by tsgpu_index_append_lists, rebuilt by
// tsgpu_index_compact_field as a gather of the live lists):
//   list_off[L+1]      u64  posting index range of token list l            (-> pos_off, df = difference)
//   list_blk_off[L+1]  u32  block index range of list l; blocks hold kBlock ids, only the last may be short
//   blk_first[NB]      u32  first (= minimum) id of the block: the skip index (reference: id_block_map keyed by LAST id)
//   blk_info[NB]       u64  bits 0..39 word offset into `packed`, bits 40..47 bit width b
//   packed[]           u32  per block kBlock * b bits, LSB-first: (id - blk_first) in b bits — frame of reference,
//                           the same scheme as the reference's sorted_array (base + fixed bit width), so any id of a
//                           block can be extracted without decoding its neighbours
//   pos_off[P+1]       u64  -> positions
//   positions[]        u32  raw reference offsets
// Dense lists (df >= n_docs/64) additionally get a bitmap over seq_ids plus a rank directory (one running popcount
// per 512 bits): membership of a candidate is ONE bit test in an L2-resident bitmap instead of a skip-index + block
// search, and the posting index of a hit (needed to reach its offsets) is directory + at most 4 popcounts. At the 10 M-doc
// bench shape ~50 tokens are dense (62 MB of bitmaps) and they receive most of the probes, because the driver is
// always the shortest list of a combination.
//   list_dense[L]      u32  dense slot of list l or kNone
//   dense_bits[]       u32  slot s owns words [s*dense_words, (s+1)*dense_words)
//   dense_rank[]       u32  slot s owns [s*dense_groups, ...): number of set bits before 128-bit group g
#pragma once
#include <stdint.h>
#include "score_device.cuh"

namespace tsdev {

constexpr int kBlock = 128;                 // ids per block (reference: posting_t::MAX_BLOCK_ELEMENTS 256)
constexpr uint32_t kNone = 0xFFFFFFFFu;

constexpr uint32_t kFieldIsArray = 1;       // string[] (in-band array protocol in the offsets)
constexpr uint32_t kFieldPlainOk = 2;        // plain string field whose offsets were validated as well formed at load
constexpr uint32_t kFieldPos16 = 4;          // ... and every position fits uint16 (precondition of score_field_plain_small)

struct DevField {
    uint32_t n_lists;
    uint32_t is_array;          // bit flags kField*
    const uint64_t* list_off;
    const uint32_t* list_blk_off;
    const uint32_t* blk_first;
    const uint64_t* blk_info;
    const uint32_t* packed;
    const uint64_t* pos_off;
    const uint32_t* positions;
    const uint32_t* list_dense;
    const uint32_t* dense_bits;
    const uint32_t* dense_rank;
    uint32_t dense_words;       // words per bitmap (multiple of 16)
    uint32_t dense_groups;      // dense_words / 4 (one directory entry per 128 bits)
};

constexpr uint32_t kDenseHit = 0xFFFFFFFEu;   // probe marker: member of a dense list, rank not computed yet

TS_HD bool dense_test(const DevField& f, uint32_t slot, uint32_t id) {
    return (f.dense_bits[(size_t) slot * f.dense_words + (id >> 5)] >> (id & 31)) & 1u;
}
// list-local posting index of a member id of dense slot `slot`: directory entry + popcount of one 16-byte group
TS_HD uint32_t dense_rank_of(const DevField& f, uint32_t slot, uint32_t id) {
    const uint32_t w = id >> 5, g = w >> 2, wi = w & 3;
    const uint32_t* bits = f.dense_bits + (size_t) slot * f.dense_words + ((size_t) g << 2);
    uint32_t r = f.dense_rank[(size_t) slot * f.dense_groups + g];
#if defined(__CUDA_ARCH__)
    const uint4 v = *reinterpret_cast<const uint4*>(bits);
    const uint32_t b0 = v.x, b1 = v.y, b2 = v.z, b3 = v.w;
#define TS_POPC(x) __popc(x)
#else
    const uint32_t b0 = bits[0], b1 = bits[1], b2 = bits[2], b3 = bits[3];
#define TS_POPC(x) ((uint32_t) __builtin_popcount(x))
#endif
    const uint32_t m = (1u << (id & 31)) - 1u;
    r += TS_POPC(wi == 0 ? (b0 & m) : b0);
    if(wi >= 1) r += TS_POPC(wi == 1 ? (b1 & m) : b1);
    if(wi >= 2) r += TS_POPC(wi == 2 ? (b2 & m) : b2);
    if(wi >= 3) r += TS_POPC(b3 & m);
#undef TS_POPC
    return r;
}

// The per-posting halves of kFieldPlainOk / kFieldPos16, shared by the loader (postings_pack.h) and the device-side
// compaction (mirror_kernels.cuh) so the two cannot disagree. Raw offsets positions[a, b) of one posting are well formed
// when they are strictly increasing, non-zero, optionally followed by one trailing 0 (src/index.cpp:1341-1348).
TS_HD bool offsets_wellformed(const uint32_t* positions, uint64_t a, uint64_t b) {
    if(b <= a) return false;
    uint64_t e = b;
    if(positions[b - 1] == 0) e = b - 1;
    if(e <= a) return false;
    uint32_t prev = 0;
    for(uint64_t i = a; i < e; i++) { if(positions[i] == 0 || positions[i] <= prev) return false; prev = positions[i]; }
    return true;
}
// no offset beyond 65535 (Match keeps offsets as uint16: beyond that they wrap)
TS_HD bool offsets_fit_u16(const uint32_t* positions, uint64_t a, uint64_t b) {
    for(uint64_t i = a; i < b; i++) if(positions[i] > 0xFFFFu) return false;
    return true;
}

TS_HD uint32_t bits_required(uint32_t v) {
    uint32_t b = 0;
    while(v) { b++; v >>= 1; }
    return b;
}

TS_HD uint32_t unpack_at(const uint32_t* __restrict__ w, uint32_t bits, uint32_t idx) {
    // w points at the block's first word; one padding word follows the last block so w[wi+1] is always readable
    const uint32_t bitpos = idx * bits;
    const uint32_t wi = bitpos >> 5, sh = bitpos & 31;
    const uint32_t lo = w[wi];
    if(bits == 0) return 0;
    if(sh + bits <= 32) return bits == 32 ? lo : ((lo >> sh) & ((1u << bits) - 1u));
    const uint32_t hi = w[wi + 1];
    const uint64_t both = ((uint64_t) hi << 32) | lo;
    return (uint32_t) (both >> sh) & (bits == 32 ? 0xFFFFFFFFu : ((1u << bits) - 1u));
}

// Last block b in [lo, hi] (absolute block indices, lo <= hi) with blk_first[b] <= id, or kNone if id < blk_first[lo].
TS_HD uint32_t find_block(const uint32_t* __restrict__ blk_first, uint32_t lo, uint32_t hi, uint32_t id) {
    if(blk_first[lo] > id) return kNone;
    while(lo < hi) {
        const uint32_t mid = lo + ((hi - lo + 1) >> 1);
        if(blk_first[mid] <= id) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// Index (0..cnt) of `id` inside block `b`, or kNone. Interpolation on the packed words: ids inside a block are close
// to uniform between the block's first and last id, so one estimate from the block's span lands within a few slots;
// a short gallop brackets the target and a binary search finishes (about 4 probes instead of log2(128)+1 = 8).
TS_HD uint32_t probe_block(const DevField& f, uint32_t b, uint32_t cnt, uint32_t id) {
    const uint32_t first = f.blk_first[b];
    const uint64_t info = f.blk_info[b];
    const uint32_t bits = (uint32_t) (info >> 40) & 0xFF;
    const uint32_t* w = f.packed + (info & 0xFFFFFFFFFFull);
    const uint32_t delta = id - first;
    if(delta == 0) return 0;
    if(bits < 32 && (delta >> bits) != 0) return kNone;        // beyond the block's range: falls between two blocks
    if(cnt <= 1) return kNone;
    const uint32_t vlast = unpack_at(w, bits, cnt - 1);
    if(delta > vlast) return kNone;
    if(delta == vlast) return cnt - 1;
    uint32_t est = (uint32_t) (((uint64_t) delta * (cnt - 1)) / vlast);       // 0 < delta < vlast  =>  est in [0, cnt-2]
    uint32_t v = unpack_at(w, bits, est);
    if(v == delta) return est;
    uint32_t lo, hi;                                            // invariant: value[lo-1] < delta (or lo == 0), value[hi] > delta
    if(v < delta) {
        lo = est + 1; hi = cnt - 1;
        uint32_t step = 2, p = lo + 1;
        while(p < hi) { const uint32_t pv = unpack_at(w, bits, p); if(pv == delta) return p; if(pv > delta) { hi = p; break; } lo = p + 1; p += step; step <<= 1; }
    } else {
        lo = 1; hi = est;
        uint32_t step = 2;
        while(hi - lo >= step) { const uint32_t p = hi - step; const uint32_t pv = unpack_at(w, bits, p); if(pv == delta) return p; if(pv < delta) { lo = p + 1; break; } hi = p; step <<= 1; }
    }
    while(lo < hi) {                                            // first index in [lo, hi) with value >= delta
        const uint32_t mid = (lo + hi) >> 1;
        if(unpack_at(w, bits, mid) < delta) lo = mid + 1; else hi = mid;
    }
    if(lo < cnt && unpack_at(w, bits, lo) == delta) return lo;
    return kNone;
}

// number of ids in block b of a list with df ids whose first block is lb0
TS_HD uint32_t block_count(uint32_t b, uint32_t lb0, uint64_t df) {
    const uint64_t before = (uint64_t) (b - lb0) * kBlock;
    const uint64_t rem = df - before;
    return rem < (uint64_t) kBlock ? (uint32_t) rem : (uint32_t) kBlock;
}

// Membership probe of `id` in list `l` restricted to blocks [b_lo, b_hi] (absolute). Returns the list-local posting
// index (0..df) or kNone.
TS_HD uint32_t probe_list(const DevField& f, uint32_t l, uint32_t b_lo, uint32_t b_hi, uint32_t id) {
    if(f.list_dense) {
        const uint32_t slot = f.list_dense[l];
        if(slot != kNone) return ((id >> 5) < f.dense_words && dense_test(f, slot, id)) ? dense_rank_of(f, slot, id) : kNone;
    }
    const uint32_t lb0 = f.list_blk_off[l];
    const uint32_t b = find_block(f.blk_first, b_lo, b_hi, id);
    if(b == kNone) return kNone;
    const uint64_t df = f.list_off[l + 1] - f.list_off[l];
    const uint32_t cnt = block_count(b, lb0, df);
    const uint32_t idx = probe_block(f, b, cnt, id);
    if(idx == kNone) return kNone;
    return (b - lb0) * kBlock + idx;
}

}  // namespace tsdev
