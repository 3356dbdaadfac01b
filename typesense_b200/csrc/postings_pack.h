// Host-side builder of the device posting layout (postings_device.cuh) from a flattened field (tsgpu_field).
// Runs when a field is loaded or lists are appended (see DESIGN.md §7a), never inside a search call.
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <algorithm>
#include <vector>
#include "postings_device.cuh"

namespace tspack {

struct PackedField {
    std::vector<uint32_t> list_blk_off;   // [L+1]
    std::vector<uint32_t> blk_first;      // [NB]
    std::vector<uint64_t> blk_info;       // [NB]
    std::vector<uint32_t> packed;         // words (+1 padding word)
    // dense lists
    std::vector<uint32_t> list_dense;     // [L] slot or kNone
    std::vector<uint32_t> dense_bits, dense_rank;
    uint32_t dense_words = 0, dense_groups = 0, n_dense = 0;
};

// bitmap + rank directory for every list with df >= min_df (and at most max_lists of them, longest first by id order)
inline void pack_dense(uint32_t n_lists, const uint64_t* list_off, const uint32_t* ids, uint32_t n_docs, uint64_t min_df,
                       PackedField& out) {
    out.list_dense.assign(n_lists ? n_lists : 1, tsdev::kNone);
    out.dense_words = (((n_docs + 31) / 32) + 15) & ~15u;
    out.dense_groups = out.dense_words / 4;
    out.n_dense = 0;
    if(min_df == 0) min_df = 1;
    for(uint32_t l = 0; l < n_lists; l++) if(list_off[l + 1] - list_off[l] >= min_df) out.list_dense[l] = out.n_dense++;
    out.dense_bits.assign((size_t) out.n_dense * out.dense_words + 16, 0);
    out.dense_rank.assign((size_t) out.n_dense * out.dense_groups + 1, 0);
    for(uint32_t l = 0; l < n_lists; l++) {
        const uint32_t s = out.list_dense[l];
        if(s == tsdev::kNone) continue;
        uint32_t* bits = out.dense_bits.data() + (size_t) s * out.dense_words;
        for(uint64_t i = list_off[l]; i < list_off[l + 1]; i++) bits[ids[i] >> 5] |= 1u << (ids[i] & 31);
        uint32_t* rk = out.dense_rank.data() + (size_t) s * out.dense_groups;
        uint32_t run = 0;
        for(uint32_t g = 0; g < out.dense_groups; g++) {
            rk[g] = run;
            for(int i = 0; i < 4; i++) run += (uint32_t) __builtin_popcount(bits[(size_t) g * 4 + i]);
        }
    }
}

inline void pack_field(uint32_t n_lists, const uint64_t* list_off, const uint32_t* ids, PackedField& out) {
    using tsdev::kBlock;
    out.list_blk_off.assign((size_t) n_lists + 1, 0);
    uint64_t nb = 0;
    for(uint32_t l = 0; l < n_lists; l++) {
        out.list_blk_off[l] = (uint32_t) nb;
        const uint64_t df = list_off[l + 1] - list_off[l];
        nb += (df + kBlock - 1) / kBlock;
    }
    out.list_blk_off[n_lists] = (uint32_t) nb;
    out.blk_first.resize(nb);
    out.blk_info.resize(nb);
    // pass 1: widths and word offsets
    uint64_t words = 0;
    for(uint32_t l = 0; l < n_lists; l++) {
        const uint64_t base = list_off[l], df = list_off[l + 1] - base;
        uint32_t b = out.list_blk_off[l];
        for(uint64_t s = 0; s < df; s += kBlock, b++) {
            const uint64_t cnt = (df - s) < (uint64_t) kBlock ? (df - s) : (uint64_t) kBlock;
            const uint32_t first = ids[base + s], last = ids[base + s + cnt - 1];
            const uint32_t bits = tsdev::bits_required(last - first);
            out.blk_first[b] = first;
            out.blk_info[b] = (words & 0xFFFFFFFFFFull) | ((uint64_t) bits << 40);
            words += ((uint64_t) kBlock * bits + 31) / 32;       // fixed kBlock slots keep every block word-aligned
        }
    }
    out.packed.assign(words + 1, 0);
    // pass 2: pack
    for(uint32_t l = 0; l < n_lists; l++) {
        const uint64_t base = list_off[l], df = list_off[l + 1] - base;
        uint32_t b = out.list_blk_off[l];
        for(uint64_t s = 0; s < df; s += kBlock, b++) {
            const uint64_t cnt = (df - s) < (uint64_t) kBlock ? (df - s) : (uint64_t) kBlock;
            const uint32_t first = out.blk_first[b];
            const uint32_t bits = (uint32_t) (out.blk_info[b] >> 40) & 0xFF;
            if(bits == 0) continue;
            uint32_t* w = out.packed.data() + (out.blk_info[b] & 0xFFFFFFFFFFull);
            for(uint64_t i = 0; i < cnt; i++) {
                const uint64_t v = ids[base + s + i] - first;
                const uint64_t bitpos = i * bits;
                const uint64_t wi = bitpos >> 5, sh = bitpos & 31;
                const uint64_t both = v << sh;
                w[wi] |= (uint32_t) both;
                if(sh + bits > 32) w[wi + 1] |= (uint32_t) (both >> 32);
            }
        }
    }
}

// True when every posting of a plain string field has well-formed raw offsets: strictly increasing non-zero
// positions, optionally followed by one trailing 0 (src/index.cpp:1341-1348). Enables score_field_plain().
inline bool plain_wellformed(const uint64_t* pos_off, const uint32_t* positions, uint64_t n_post) {
    for(uint64_t p = 0; p < n_post; p++) if(!tsdev::offsets_wellformed(positions, pos_off[p], pos_off[p + 1])) return false;
    return true;
}

// True when no position exceeds 65535 (Match keeps offsets as uint16: beyond that they wrap).
inline bool positions_fit_u16(const uint32_t* positions, uint64_t n_positions) {
    return tsdev::offsets_fit_u16(positions, 0, n_positions);
}

// The dense-list threshold of a field: lists with at least this many postings get a bitmap. `div` is fixed per field at load
// time (TSGPU_DENSE_DIV, default 64); n_docs is the index's capacity, which only grows.
inline uint64_t dense_min_df(uint32_t n_docs, uint32_t div) { return std::max<uint64_t>(64, n_docs / (uint64_t) std::max<uint32_t>(1, div)); }

}  // namespace tspack
