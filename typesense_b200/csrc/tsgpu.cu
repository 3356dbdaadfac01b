// libtsgpu.so — C-ABI (include/tsgpu.h) over the sm_90a kernels in kw_kernels.cuh / knn_kernels.cuh /
// fuse_kernels.cuh. Host code here only mirrors data into HBM, turns a batch of resolved queries into work
// descriptors, launches kernels on one stream and copies results out. There is no CPU compute path: every entry point
// fails with TSGPU_ERR_NO_DEVICE when no CUDA device is usable.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <cmath>
#include <map>
#include <mutex>
#include <random>
#include <string>
#include <vector>

#include "../../include/tsgpu.h"
#include "fuse_kernels.cuh"
#include "knn_kernels.cuh"
#include "hnsw_build.cuh"
#include "facet_kernels.cuh"
#include "mirror_kernels.cuh"
#include "deep_topster.cuh"
#include "diversity.cuh"
#include "deep_fuse.cuh"
#include "postings_pack.h"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

// flat_tc.cu: the batched flat scan on the tensor cores (wgmma, tf32 x 3)
extern "C" size_t tsgpu_flat_tc_image_bytes_(uint32_t ng, uint32_t dim, uint32_t* n_tile_out, uint32_t* n_qtiles_out);
extern "C" int tsgpu_flat_tc_supported_(uint32_t dim);
extern "C" cudaError_t tsgpu_flat_tc_run_(const float* vectors, uint32_t n_nodes, uint32_t dim, const float* queries, const uint32_t* qsel, uint32_t ng,
                                          const uint32_t* ids, uint32_t n_ids, const unsigned long long* out_off, float* out_dist,
                                          unsigned char* img, int n_sms, cudaStream_t stream, int* launches);

using namespace tsk;

// art_kernels.cu (SURVEY 8 f-1) keeps its state outside tsgpu_index; it frees it through this hook
extern "C" void tsgpu_art_release_(const tsgpu_index* idx);
// kw_regscore.cu: kw_search_kernel<true> lives in its own translation unit (see there)
extern "C" cudaError_t tsgpu_launch_kw_search_regscore(const void* index_dev, const void* kw_params, unsigned n_units, size_t smem, cudaStream_t st);
extern "C" cudaError_t tsgpu_launch_kw_search_deep(const void* index_dev, const void* kw_params, unsigned n_units, size_t smem, cudaStream_t st);
// diversity.cu: the MMR re-ranking kernels (tsgpu_diversify_batch)
extern "C" cudaError_t tsgpu_launch_div_count_(const tsdiv::Params* P, unsigned nq, cudaStream_t st);
extern "C" cudaError_t tsgpu_launch_div_mmr_(const tsdiv::Params* P, unsigned nq, size_t smem, cudaStream_t st);

namespace {

thread_local std::string g_err;
tsgpu_status fail(tsgpu_status s, const std::string& m) { g_err = m; return s; }

#define CU(call)                                                                                              \
    do {                                                                                                      \
        cudaError_t e__ = (call);                                                                             \
        if(e__ != cudaSuccess) {                                                                              \
            return fail(TSGPU_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e__) + " @" + std::to_string(__LINE__)); \
        }                                                                                                     \
    } while(0)

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t bytes, bool zero_new = false) {
        if(bytes <= cap) return cudaSuccess;
        if(p) cudaFree(p);
        p = nullptr;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if(e != cudaSuccess) { cap = 0; return e; }
        cap = want;
        if(zero_new) return cudaMemset(p, 0, cap);
        return cudaSuccess;
    }
    void release() { if(p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct PinBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t bytes) {
        if(bytes <= cap) return cudaSuccess;
        if(p) cudaFreeHost(p);
        p = nullptr;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMallocHost(&p, want);
        if(e != cudaSuccess) { cap = 0; return e; }
        cap = want;
        return cudaSuccess;
    }
    void release() { if(p) cudaFreeHost(p); p = nullptr; cap = 0; }
};

// sequential packer of several arrays into one staging buffer (8-byte aligned pieces)
struct Stager {
    std::vector<unsigned char> host;
    size_t add(const void* src, size_t bytes) {
        size_t off = (host.size() + 15) & ~size_t(15);
        host.resize(off + bytes);
        if(bytes && src) memcpy(host.data() + off, src, bytes);
        return off;
    }
    size_t reserve(size_t bytes) { return add(nullptr, bytes); }
};

struct FieldMirror {
    DevField dev{};
    std::vector<uint64_t> h_list_off;
    std::vector<uint32_t> h_list_blk_off;
    std::vector<uint32_t> h_list_dense;
    std::vector<uint32_t> h_list_first, h_list_last;   // smallest / largest id of each list (the bitmap path's word range)
    void* d_alloc[10] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    // element counts of the device arrays (tsgpu_index_append_lists grows them)
    size_t d_bytes[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};   // bytes allocated per array (tsgpu_index_field_info)
    uint64_t n_post = 0, n_pos = 0, n_words = 0;      // postings, raw offsets, packed words (without the padding word)
    uint32_t n_blocks = 0, n_dense = 0;
    uint64_t dense_min_df = 0;
    uint32_t dense_div = 64;                          // TSGPU_DENSE_DIV at load: the threshold is max(64, n_docs / dense_div)
};

struct Filter {
    uint32_t* d_bitmap = nullptr;
    uint32_t* d_ids = nullptr;
    size_t n = 0;
    bool live = false;
};

}  // namespace

struct tsgpu_index {
    int device = 0;
    uint32_t n_docs = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t stream2 = nullptr;      // vector stage of hybrid calls (overlaps the keyword kernels)
    cudaStream_t vs = nullptr;           // stream the vector stage is issued on for the current call
    cudaEvent_t evA = nullptr, evB = nullptr;
    unsigned knn_blocks_per_sm = 7;
    unsigned long long build_stats[4] = {0, 0, 0, 0}; size_t build_rounds = 0;   // counters of the last tsgpu_index_build_hnsw
    uint32_t* knn_work_dev = nullptr; uint32_t knn_work_n = 0;   // per-walk counters of the last HNSW launch (tsgpu_debug_knn_work)
    unsigned char* knn_misc_dev = nullptr;    // counters of the last HNSW launch (read after the final sync)
    std::vector<unsigned char> knn_tables;   // host copies that must outlive the async uploads
    std::vector<uint8_t> tmp_is_flat; std::vector<unsigned long long> tmp_foff; std::vector<unsigned char> flat_tc_host;
    std::mutex mu;
    std::vector<FieldMirror> fields;
    IndexDev ixdev{};
    std::vector<int64_t*> sort_cols;
    bool has_hnsw = false;
    tsv::HnswDev hnsw{};
    std::vector<void*> hnsw_alloc;
    uint32_t* d_deleted = nullptr; size_t deleted_words = 0;     // markDelete bitmap over labels (lives with the index, survives appends)
    std::vector<Filter> filters;
    struct FacetMirror { tsfc::FacetDev dev{}; void* d_off = nullptr; void* d_vals = nullptr; };
    std::vector<FacetMirror> facets;
    std::vector<const uint32_t*> keep_bitmaps;      // per query of the last search: its all_result_ids bitmap (device) or nullptr
    DevBuf d_keep_bm, d_facet, d_comm, d_flat_tc;
    void* comm = nullptr; int comm_rank = 0, comm_world = 1; float last_comm_ms = 0;       // ncclComm_t of tsgpu_comm_init
    int n_sms = 132;
    // scratch
    DevBuf d_stage, d_pool, d_small, d_bitmaps, d_found_bm, d_out, d_knn_vis, d_knn_retry_vis, d_knn_retry_cand, d_knn_cand, d_knn_out, d_isect, d_kw_out, d_deep;
    PinBuf h_stage;
    size_t knn_slots = 0;
    bool found_dirty = false;            // d_found_bm is all-zero between calls unless a call died before its popcount pass
    cudaEvent_t ev[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t deep_ev[4] = {nullptr, nullptr, nullptr, nullptr};     // emit / de-duplicate / select of deep queries (created on first use)
    DevBuf d_fuse;                       // deep vector assembly / deep hybrid fusion (deep_fuse_host.inc)
    DevBuf d_div, d_div_ws;              // tsgpu_diversify_batch: records, per-query arrays / the workspaces that do not fit in shared memory
    PinBuf h_div;
    tsgpu_stats stats{};
};

namespace {

tsgpu_status check_device(tsgpu_index* idx) {
    if(!idx) return fail(TSGPU_ERR_INVALID, "null index");
    CU(cudaSetDevice(idx->device));
    return TSGPU_OK;
}

constexpr uint32_t kMergeFan = 16;

uint32_t pow2_ceil(uint32_t v) { uint32_t p = 1; while(p < v) p <<= 1; return p; }

// appends the first and last id of lists [0, n) (offsets list_off[] - base into ids[]); an empty list gets first > last
void list_id_range(uint32_t n, const uint64_t* list_off, const uint32_t* ids, uint64_t base, std::vector<uint32_t>& first,
                   std::vector<uint32_t>& last) {
    for(uint32_t l = 0; l < n; l++) {
        const uint64_t a = list_off[l] - base, b = list_off[l + 1] - base;
        first.push_back(b > a ? ids[a] : kNone);
        last.push_back(b > a ? ids[b - 1] : 0);
    }
}

// ------------------------------------------------------------------------------------------------- keyword prep
struct KwPlan {
    uint32_t nq = 0, nc = 0, F = 0, n_units = 0;
    uint32_t KP = 128, NL = 1, KMAX = 1;
    uint32_t field_ids[kMaxFieldSlots] = {0, 0, 0, 0, 0, 0, 0, 0};
    std::vector<QDesc> qd;
    std::vector<CDesc> cd;
    std::vector<UDesc> ud;
    std::vector<uint32_t> multi_q;        // queries whose found count needs the union bitmap (cleared after counting)
    std::vector<uint32_t> multi_keep_q;   // ... and whose bitmap is kept (all_result_ids for facets / export)
    std::vector<uint32_t> keep_q;         // every query that keeps its all_result_ids bitmap
    std::vector<std::vector<MDesc>> levels;   // intermediate merge levels (only queries with many units)
    std::vector<MDesc*> d_levels;
    uint32_t n_units_total = 0;           // level-0 units + merge outputs
    bool wildcard = false;                // units walk the filter ids (Index::search_wildcard) instead of posting lists
    std::vector<uint32_t> q_nids;         // wildcard: ids per query
    std::vector<unsigned long long> q_inline_off;   // wildcard: offset of the query's ids inside the batch's inline filter ids (~0: not inline)
    size_t n_inline_ids = 0;
    const int64_t* id_scores = nullptr;   // scored id sets (host or device, aligned with the batch's inline filter ids) or nullptr
    size_t pool_slots = 0;
    // deep queries (TSGPU_QFLAG_DEEP_TOPSTER with topk > TSGPU_MAX_TOPK): their units, kept apart from everything that sizes the
    // ordinary path, and their slices of the deep buffer, bounded by the entries they can emit
    std::vector<uint32_t> deep_q;
    std::vector<UDesc> deep_ud;
    std::vector<unsigned long long> deep_off;  // [deep_q.size()+1] slice of deep query i in the deep buffer
    unsigned long long deep_max = 0;           // largest slice
    UDesc* d_deep_ud = nullptr; long long* d_deep_cur = nullptr;
    // device views (valid after upload)
    QDesc* d_qd = nullptr; CDesc* d_cd = nullptr; UDesc* d_ud = nullptr; uint32_t* d_multi_q = nullptr; uint32_t* d_multi_keep_q = nullptr;
    uint32_t* d_unit_cnt = nullptr; uint32_t* d_combo_matches = nullptr; unsigned long long* d_stats = nullptr;
    long long* d_q_thr = nullptr;
    std::vector<const uint32_t*> q_bitmap;   // per query filter bitmap (device) or nullptr
    std::vector<const uint32_t*> q_filter_ids; std::vector<size_t> q_filter_n;   // device ids (flat path)
    std::vector<const uint32_t*> q_excl_dev;
};

tsgpu_status build_kw_plan(tsgpu_index* idx, const tsgpu_kw_batch* b, bool with_combos, KwPlan& pl, bool wildcard = false) {
    if(!b) return fail(TSGPU_ERR_INVALID, "null batch");
    const uint32_t nq = b->n_queries, F = b->n_fields;
    if(with_combos && (F == 0 || F > TSGPU_MAX_FIELDS)) return fail(TSGPU_ERR_CAPACITY, "n_fields must be 1.." + std::to_string(TSGPU_MAX_FIELDS));
    for(uint32_t f = 0; f < F; f++) if(b->field_ids[f] >= idx->fields.size()) return fail(TSGPU_ERR_INVALID, "field id out of range");
    pl.nq = nq; pl.F = F; pl.nc = with_combos ? b->n_combos : 0;
    pl.wildcard = wildcard;
    for(uint32_t f = 0; f < F && f < (uint32_t) kMaxFieldSlots; f++) pl.field_ids[f] = b->field_ids[f];
    pl.qd.assign(nq, QDesc{});
    pl.cd.assign(pl.nc, CDesc{});
    pl.q_bitmap.assign(nq, nullptr); pl.q_filter_ids.assign(nq, nullptr); pl.q_filter_n.assign(nq, 0); pl.q_excl_dev.assign(nq, nullptr);
    uint32_t kmax = 1, nl_max = 1;
    auto df_of = [&](uint32_t f, uint32_t l) -> uint64_t {
        const FieldMirror& fm = idx->fields[b->field_ids[f]];
        return fm.h_list_off[l + 1] - fm.h_list_off[l];
    };
    // ---- combos
    const double dense_cost = getenv("TSGPU_DENSE_COST") ? atof(getenv("TSGPU_DENSE_COST")) : 0.5;   // read per call: tools/bench_dense_kw.py sweeps it
    std::vector<uint32_t> combo_tiles(pl.nc, 0);
    uint64_t total_tiles = 0;
    for(uint32_t c = 0; c < pl.nc; c++) {
        CDesc& cd = pl.cd[c];
        const uint32_t r0 = b->c_tok_off[c], n_rows = b->c_tok_off[c + 1] - r0;
        if(n_rows > TSGPU_MAX_TOKENS) return fail(TSGPU_ERR_CAPACITY, "more than TSGPU_MAX_TOKENS token rows in a combination");
        if(n_rows * F > (uint32_t) kMaxLists) return fail(TSGPU_ERR_CAPACITY, "rows*fields exceeds 32 in a combination");
        const uint32_t n_req = std::min<uint32_t>(b->c_n_required[c], n_rows);
        cd.total_cost = b->c_total_cost[c];
        cd.syn_orig = b->c_syn_orig_num_tokens ? b->c_syn_orig_num_tokens[c] : -1;
        cd.orig = b->c_orig_num_tokens ? b->c_orig_num_tokens[c] : -1;
        cd.cflags = b->c_flags ? b->c_flags[c] : 0;
        cd.n_rows = (uint8_t) n_rows; cd.n_req = (uint8_t) n_req;
        nl_max = std::max(nl_max, n_rows * F);
        uint64_t sumdf[TSGPU_MAX_TOKENS];
        for(uint32_t i = 0; i < (uint32_t) kMaxLists; i++) cd.lists[i] = kNone;
        for(uint32_t r = 0; r < n_rows; r++) {
            sumdf[r] = 0;
            for(uint32_t f = 0; f < F; f++) {
                uint32_t l = b->t_list[(size_t) (r0 + r) * F + f];
                if(l != TSGPU_NO_LIST) {
                    const FieldMirror& fm = idx->fields[b->field_ids[f]];
                    if(l >= fm.dev.n_lists) return fail(TSGPU_ERR_INVALID, "posting list id out of range");
                    if(df_of(f, l) == 0) l = TSGPU_NO_LIST;       // empty list == token absent from the field
                }
                cd.lists[r * F + f] = l;
                if(l != TSGPU_NO_LIST) sumdf[r] += df_of(f, l);
            }
        }
        cd.req_mask = 0;
        uint32_t drv = kNone;
        for(uint32_t r = 0; r < n_req; r++) if(sumdf[r]) { cd.req_mask |= 1u << r; if(drv == kNone || sumdf[r] < sumdf[drv]) drv = r; }
        uint32_t tiles = 0;
        for(uint32_t f = 0; f <= (uint32_t) kMaxFieldSlots; f++) cd.drv_tile_off[f] = 0;
        cd.mode = 0; cd.w_begin = cd.w_end = 0;
        // Every required token dense: the bitmap AND reads each word of the id range once per list, the driver tiles probe
        // every driver id. Take the bitmaps when the words are fewer than dense_cost x the driver ids (DESIGN.md §3).
        bool all_dense = drv != kNone;
        uint32_t id_lo = 0, id_hi = idx->n_docs ? idx->n_docs - 1 : 0;     // docs every required row can hold
        for(uint32_t r = 0; r < n_req && all_dense; r++) {
            if(!((cd.req_mask >> r) & 1)) continue;
            uint32_t row_lo = kNone, row_hi = 0;
            for(uint32_t f = 0; f < F; f++) {
                const uint32_t l = cd.lists[r * F + f];
                if(l == TSGPU_NO_LIST) continue;
                const FieldMirror& fm = idx->fields[b->field_ids[f]];
                if(fm.h_list_dense[l] == kNone) { all_dense = false; break; }
                row_lo = std::min(row_lo, fm.h_list_first[l]); row_hi = std::max(row_hi, fm.h_list_last[l]);
            }
            id_lo = std::max(id_lo, row_lo); id_hi = std::min(id_hi, row_hi);
        }
        if(all_dense) {
            cd.w_begin = (id_lo >> 5) & ~31u;                          // 128-byte aligned loads
            cd.w_end = id_lo <= id_hi ? (id_hi >> 5) + 1 : cd.w_begin;
            if((double) (cd.w_end - cd.w_begin) >= dense_cost * (double) sumdf[drv]) all_dense = false;
        }
        if(all_dense) {
            // word-parallel bitmap AND over [w_begin, w_end) (kw_kernels.cuh)
            cd.mode = 1;
            cd.driver_row = (uint8_t) drv;
            tiles = (cd.w_end - cd.w_begin + kThreads - 1) / kThreads;
            for(uint32_t f = 0; f <= (uint32_t) kMaxFieldSlots; f++) cd.drv_tile_off[f] = f == 0 ? 0 : tiles;
            for(uint32_t i = 0; i < 16; i++) cd.probe_order[i] = (uint8_t) (i < n_rows ? i : 0);
        } else if(drv != kNone) {
            cd.driver_row = (uint8_t) drv;
            for(uint32_t f = 0; f < F; f++) {
                cd.drv_tile_off[f] = tiles;
                const uint32_t l = cd.lists[drv * F + f];
                if(l != TSGPU_NO_LIST) tiles += (uint32_t) ((df_of(f, l) + tsdev::kBlock - 1) / tsdev::kBlock);
            }
            for(uint32_t f = F; f <= (uint32_t) kMaxFieldSlots; f++) cd.drv_tile_off[f] = tiles;
            // probe order: driver, other required rows by ascending postings, then the dropped rows
            uint32_t order[TSGPU_MAX_TOKENS + 1], n_order = 0;
            order[n_order++] = drv;
            for(uint32_t r = 0; r < n_req; r++) {            // stable insertion by ascending postings
                if(r == drv) continue;
                uint32_t i = n_order++;
                while(i > 1 && sumdf[order[i - 1]] > sumdf[r]) { order[i] = order[i - 1]; i--; }
                order[i] = r;
            }
            for(uint32_t r = n_req; r < n_rows; r++) order[n_order++] = r;
            for(uint32_t i = 0; i < 16; i++) cd.probe_order[i] = i < n_order ? (uint8_t) order[i] : 0;
        }
        combo_tiles[c] = tiles;
        total_tiles += tiles;
    }
    // ---- queries
    static const uint64_t unit_target = getenv("TSGPU_KW_UNIT_TARGET") ? (uint64_t) std::max(1, atoi(getenv("TSGPU_KW_UNIT_TARGET"))) : 8192;
    uint32_t tpu = (uint32_t) std::min<uint64_t>(256, std::max<uint64_t>(4, total_tiles / unit_target));
    std::vector<std::pair<uint32_t, uint32_t>> q_units0;
    pl.deep_off.assign(1, 0);
    for(uint32_t q = 0; q < nq; q++) {
        QDesc& qd = pl.qd[q];
        const uint32_t K = b->q_topk[q];
        const bool deep_ok = (b->q_flags[q] & TSGPU_QFLAG_DEEP_TOPSTER) != 0;
        if(K == 0 || (K > TSGPU_MAX_TOPK && !deep_ok))
            return fail(TSGPU_ERR_CAPACITY, "topk must be 1.." + std::to_string(TSGPU_MAX_TOPK) + " (larger needs TSGPU_QFLAG_DEEP_TOPSTER)");
        const bool deep = K > TSGPU_MAX_TOPK;
        std::vector<UDesc>& uds = deep ? pl.deep_ud : pl.ud;
        uint64_t deep_bound = 0;                  // entries a deep query can emit: one per matched (id, combination)
        qd.topk = K; if(!deep) kmax = std::max(kmax, K);
        for(int i = 0; i < 3; i++) {
            qd.sort_type[i] = b->q_sort_type[q * 3 + i];
            qd.sort_order[i] = b->q_sort_order[q * 3 + i];
            qd.missing_first[i] = b->q_sort_missing_first ? b->q_sort_missing_first[q * 3 + i] : 0;
            qd.sort_col[i] = nullptr;
            if(qd.sort_type[i] == TSGPU_SORT_NUMERIC) {
                const int32_t col = b->q_sort_col[q * 3 + i];
                if(col < 0 || (size_t) col >= idx->sort_cols.size()) return fail(TSGPU_ERR_INVALID, "sort column out of range");
                qd.sort_col[i] = idx->sort_cols[col];
            }
        }
        qd.flags = b->q_flags[q] & 0x1F; qd.rerank = (b->q_flags[q] & TSGPU_FLAG_RERANK_HYBRID_MATCHES) ? 1 : 0; qd.match_type = b->q_match_type[q]; qd.num_query_tokens = b->q_num_query_tokens[q];
        qd.keep_all = (b->q_flags[q] & TSGPU_QFLAG_KEEP_ALL_IDS) ? 1 : 0;
        for(uint32_t f = 0; f < (uint32_t) kMaxFieldSlots; f++) qd.field_weight[f] = f < F ? b->q_field_weight[(size_t) q * F + f] : 0;
        qd.n_excl = b->q_excl_off[q + 1] - b->q_excl_off[q];
        qd.combo_begin = with_combos ? b->q_combo_off[q] : 0;
        qd.combo_end = with_combos ? b->q_combo_off[q + 1] : 0;
        if(qd.combo_end - qd.combo_begin > (uint32_t) kMaxCombosPerQuery) return fail(TSGPU_ERR_CAPACITY, "more than 256 combinations in a query");
        qd.unit_begin = (uint32_t) pl.ud.size();
        uint32_t combos_with_tiles = 0;
        for(uint32_t c = qd.combo_begin; c < qd.combo_end; c++) {
            pl.cd[c].q = q;
            if(combo_tiles[c]) combos_with_tiles++;
            const uint32_t ctpu = pl.cd[c].mode == 1 ? 64u : tpu;      // a dense tile is 4096 docs of bitmap words
            if(deep) deep_bound += std::min<uint64_t>((uint64_t) combo_tiles[c] * (pl.cd[c].mode == 1 ? 4096u : 128u), idx->n_docs);
            for(uint32_t t = 0; t < combo_tiles[c]; t += ctpu) {
                UDesc u;
                u.combo = c; u.tile_begin = t; u.tile_end = std::min(combo_tiles[c], t + ctpu);
                u.out_off = deep ? 0u : (uint32_t) pl.pool_slots;
                if(!deep) pl.pool_slots += K;
                uds.push_back(u);
            }
        }
        if(wildcard) {
            // id set of the query: its filter ids, or every seq_id when it has no filter (src/index.cpp:3738-3745)
            uint64_t n_ids = idx->n_docs;
            const int32_t wfs = b->q_filter[q];
            if(wfs >= 0 && (uint32_t) wfs < b->n_filters) n_ids = b->filter_off[wfs + 1] - b->filter_off[wfs];
            else if(wfs <= -2 && (size_t) (-(wfs + 2)) < idx->filters.size()) n_ids = idx->filters[(size_t) (-(wfs + 2))].n;
            pl.q_nids.push_back((uint32_t) n_ids);
            pl.q_inline_off.push_back((wfs >= 0 && (uint32_t) wfs < b->n_filters) ? (unsigned long long) b->filter_off[wfs] : ~0ull);
            pl.n_inline_ids = b->n_filters ? (size_t) b->filter_off[b->n_filters] : 0;
            qd.combo_begin = q; qd.combo_end = q + 1;
            const uint32_t tiles = (uint32_t) ((n_ids + kThreads - 1) / kThreads), wtpu = 64;
            if(deep) deep_bound = n_ids;
            for(uint32_t t = 0; t < tiles; t += wtpu) {
                UDesc u;
                u.combo = q; u.tile_begin = t; u.tile_end = std::min(tiles, t + wtpu);
                u.out_off = deep ? 0u : (uint32_t) pl.pool_slots;
                if(!deep) pl.pool_slots += K;
                uds.push_back(u);
            }
        }
        qd.unit_end = (uint32_t) pl.ud.size();
        if(deep) {
            pl.deep_q.push_back(q);
            pl.deep_off.push_back(pl.deep_off.back() + deep_bound);
            pl.deep_max = std::max<unsigned long long>(pl.deep_max, deep_bound);
        }
        q_units0.push_back({qd.unit_begin, qd.unit_end});
        if(qd.keep_all && !wildcard) { pl.keep_q.push_back(q); if(combos_with_tiles > 1) pl.multi_keep_q.push_back(q); }
        else if(combos_with_tiles > 1) pl.multi_q.push_back(q);
        const int32_t fs = b->q_filter[q];
        if(fs >= 0 && (uint32_t) fs >= b->n_filters) return fail(TSGPU_ERR_INVALID, "inline filter slot out of range");
        if(fs <= -2) {
            const size_t h = (size_t) (-(fs + 2));
            if(h >= idx->filters.size() || !idx->filters[h].live) return fail(TSGPU_ERR_INVALID, "unknown filter handle");
        }
    }
    if(wildcard) pl.nc = nq;                // one pseudo-combination per query carries its match count
    pl.n_units = (uint32_t) pl.ud.size();
    // queries with more than kMergeFan units get intermediate merge levels (fan-in kMergeFan) so the per-query final
    // merge stays short and the work of a heavy query is spread over many CTAs
    {
        std::vector<std::pair<uint32_t, uint32_t>> cur = q_units0;
        for(int level = 0; level < 6; level++) {
            std::vector<MDesc> groups;
            bool any = false;
            for(uint32_t q = 0; q < nq; q++) {
                const uint32_t a = cur[q].first, e = cur[q].second;
                if(e - a <= kMergeFan) continue;
                any = true;
                const uint32_t ob = (uint32_t) pl.ud.size();
                for(uint32_t s0 = a; s0 < e; s0 += kMergeFan) {
                    MDesc m; m.q = q; m.in_begin = s0; m.in_end = std::min(e, s0 + kMergeFan); m.out_unit = (uint32_t) pl.ud.size();
                    UDesc u; u.combo = 0; u.tile_begin = u.tile_end = 0; u.out_off = (uint32_t) pl.pool_slots;
                    pl.pool_slots += pl.qd[q].topk;
                    pl.ud.push_back(u);
                    groups.push_back(m);
                }
                cur[q] = {ob, (uint32_t) pl.ud.size()};
            }
            if(!any) break;
            pl.levels.push_back(std::move(groups));
        }
        for(uint32_t q = 0; q < nq; q++) { pl.qd[q].unit_begin = cur[q].first; pl.qd[q].unit_end = cur[q].second; }
    }
    if(pl.pool_slots > 0xFFFFFFF0ull) return fail(TSGPU_ERR_CAPACITY, "result pool too large; split the batch");
    pl.n_units_total = (uint32_t) pl.ud.size();
    pl.KMAX = kmax;
    pl.KP = std::max<uint32_t>(128, pow2_ceil(kmax));
    pl.NL = nl_max;
    return TSGPU_OK;
}

// uploads descriptors, exclusion lists and inline filters; builds filter / found bitmaps
tsgpu_status upload_kw_plan(tsgpu_index* idx, const tsgpu_kw_batch* b, KwPlan& pl) {
    cudaStream_t st = idx->stream;
    const uint32_t nq = pl.nq;
    const size_t words = ((size_t) idx->n_docs + 31) / 32;
    // device bitmaps: [inline filters][found bitmaps]
    const size_t n_inline = b->n_filters;
    if(n_inline) {
        CU(idx->d_bitmaps.reserve(n_inline * words * 4));
        CU(cudaMemsetAsync(idx->d_bitmaps.p, 0, n_inline * words * 4, st));
    }
    uint32_t* bm = idx->d_bitmaps.as<uint32_t>();
    // found bitmaps live in their own buffer that is all-zero between calls (found_popcount_kernel clears what it counts)
    const size_t fwords = (words + 3) & ~size_t(3);
    if(!pl.multi_q.empty()) {
        const size_t old_cap = idx->d_found_bm.cap;
        CU(idx->d_found_bm.reserve(pl.multi_q.size() * fwords * 4));
        if(idx->found_dirty || idx->d_found_bm.cap != old_cap) CU(cudaMemsetAsync(idx->d_found_bm.p, 0, idx->d_found_bm.cap, st));
        idx->found_dirty = true;
    }
    uint32_t* fbm = idx->d_found_bm.as<uint32_t>();
    idx->keep_bitmaps.assign(nq, nullptr);
    if(!pl.keep_q.empty()) {               // all_result_ids that outlive the call: their own buffer, zeroed per call
        CU(idx->d_keep_bm.reserve(pl.keep_q.size() * fwords * 4));
        CU(cudaMemsetAsync(idx->d_keep_bm.p, 0, pl.keep_q.size() * fwords * 4, st));
    }
    Stager sg;
    const size_t n_excl_total = b->q_excl_off[nq];
    const size_t o_excl = sg.add(b->excl_ids, n_excl_total * 4);
    const size_t n_fids = n_inline ? (size_t) b->filter_off[n_inline] : 0;
    const size_t o_fids = sg.add(b->filter_ids, n_fids * 4);
    // descriptor pointers need the device base first: compute offsets, then patch
    const size_t o_qd = sg.reserve(pl.qd.size() * sizeof(QDesc));
    const size_t o_cd = sg.reserve(pl.cd.size() * sizeof(CDesc));
    const size_t o_ud = sg.reserve(pl.ud.size() * sizeof(UDesc));
    const size_t o_mq = sg.reserve(pl.multi_q.size() * 4);
    const size_t o_mk = sg.reserve(pl.multi_keep_q.size() * 4);
    std::vector<size_t> o_lv;
    for(auto& lv: pl.levels) o_lv.push_back(sg.add(lv.data(), lv.size() * sizeof(MDesc)));
    const size_t o_cnt = sg.reserve(((size_t) pl.n_units_total + pl.nc + 8) * 4 + 64);
    const size_t o_thr = sg.reserve((size_t) nq * 8);
    const size_t o_dud = sg.add(pl.deep_ud.data(), pl.deep_ud.size() * sizeof(UDesc));
    const size_t o_dcur = sg.reserve(pl.deep_q.empty() ? 0 : (size_t) nq * 8);
    CU(idx->d_stage.reserve(sg.host.size()));
    unsigned char* dbase = idx->d_stage.as<unsigned char>();
    const uint32_t* d_excl = reinterpret_cast<const uint32_t*>(dbase + o_excl);
    const uint32_t* d_fids = reinterpret_cast<const uint32_t*>(dbase + o_fids);
    for(uint32_t q = 0; q < nq; q++) {
        QDesc& qd = pl.qd[q];
        qd.excl = d_excl + b->q_excl_off[q];
        pl.q_excl_dev[q] = qd.excl;
        const int32_t fs = b->q_filter[q];
        qd.filter_bitmap = nullptr; qd.filter_empty = 0;
        if(fs >= 0) {
            const size_t n = (size_t) (b->filter_off[fs + 1] - b->filter_off[fs]);
            qd.filter_bitmap = bm + (size_t) fs * words;
            qd.filter_empty = n == 0;
            pl.q_filter_ids[q] = d_fids + b->filter_off[fs]; pl.q_filter_n[q] = n;
        } else if(fs <= -2) {
            const Filter& fl = idx->filters[(size_t) (-(fs + 2))];
            qd.filter_bitmap = fl.d_bitmap;
            qd.filter_empty = fl.n == 0;
            pl.q_filter_ids[q] = fl.d_ids; pl.q_filter_n[q] = fl.n;
        }
        pl.q_bitmap[q] = qd.filter_bitmap;
        qd.found_bitmap = nullptr;
    }
    for(size_t i = 0; i < pl.multi_q.size(); i++) pl.qd[pl.multi_q[i]].found_bitmap = fbm + i * fwords;
    for(size_t i = 0; i < pl.keep_q.size(); i++) {
        pl.qd[pl.keep_q[i]].found_bitmap = idx->d_keep_bm.as<uint32_t>() + i * fwords;
        idx->keep_bitmaps[pl.keep_q[i]] = pl.qd[pl.keep_q[i]].found_bitmap;
    }
    memcpy(sg.host.data() + o_qd, pl.qd.data(), pl.qd.size() * sizeof(QDesc));
    memcpy(sg.host.data() + o_cd, pl.cd.data(), pl.cd.size() * sizeof(CDesc));
    memcpy(sg.host.data() + o_ud, pl.ud.data(), pl.ud.size() * sizeof(UDesc));
    memcpy(sg.host.data() + o_mq, pl.multi_q.data(), pl.multi_q.size() * 4);
    memcpy(sg.host.data() + o_mk, pl.multi_keep_q.data(), pl.multi_keep_q.size() * 4);
    memset(sg.host.data() + o_cnt, 0, ((size_t) pl.n_units_total + pl.nc + 8) * 4 + 64);
    for(uint32_t q = 0; q < nq; q++) reinterpret_cast<long long*>(sg.host.data() + o_thr)[q] = INT64_MIN;
    if(!pl.deep_q.empty()) {                  // deep cursors start at their slices
        long long* cur = reinterpret_cast<long long*>(sg.host.data() + o_dcur);
        for(uint32_t q = 0; q < nq; q++) cur[q] = 0;
        for(size_t i = 0; i < pl.deep_q.size(); i++) cur[pl.deep_q[i]] = (long long) pl.deep_off[i];
    }
    CU(idx->h_stage.reserve(sg.host.size()));
    memcpy(idx->h_stage.p, sg.host.data(), sg.host.size());
    CU(cudaMemcpyAsync(dbase, idx->h_stage.p, sg.host.size(), cudaMemcpyHostToDevice, st));
    idx->stats.h2d_bytes += sg.host.size();
    pl.d_qd = reinterpret_cast<QDesc*>(dbase + o_qd);
    pl.d_cd = reinterpret_cast<CDesc*>(dbase + o_cd);
    pl.d_ud = reinterpret_cast<UDesc*>(dbase + o_ud);
    pl.d_multi_q = reinterpret_cast<uint32_t*>(dbase + o_mq);
    pl.d_multi_keep_q = reinterpret_cast<uint32_t*>(dbase + o_mk);
    pl.d_levels.clear();
    for(size_t o: o_lv) pl.d_levels.push_back(reinterpret_cast<MDesc*>(dbase + o));
    unsigned char* cnt = dbase + ((o_cnt + 63) & ~size_t(63));
    pl.d_stats = reinterpret_cast<unsigned long long*>(cnt);                 // 4 x u64
    pl.d_combo_matches = reinterpret_cast<uint32_t*>(cnt + 32);
    pl.d_unit_cnt = pl.d_combo_matches + pl.nc;
    pl.d_q_thr = reinterpret_cast<long long*>(dbase + o_thr);
    pl.d_deep_ud = reinterpret_cast<UDesc*>(dbase + o_dud);
    pl.d_deep_cur = reinterpret_cast<long long*>(dbase + o_dcur);
    // inline filter bitmaps
    for(size_t s = 0; s < n_inline; s++) {
        const size_t n = (size_t) (b->filter_off[s + 1] - b->filter_off[s]);
        if(!n) continue;
        bitmap_from_ids_kernel<<<(unsigned) ((n + 255) / 256), 256, 0, st>>>(d_fids + b->filter_off[s], n, bm + s * words, idx->n_docs);
        idx->stats.launches_total++;
    }
    CU(cudaGetLastError());
    return TSGPU_OK;
}

size_t kw_search_smem(uint32_t KP, uint32_t NL) { return (size_t) 2 * KP * 28 + (size_t) NL * kThreads * 4 + (size_t) kQCap * 4 + (size_t) NL * kQCap * 4; }
size_t kw_final_smem(const KwPlan& pl) { return (size_t) 2 * pl.KP * 30 + 16; }

struct KwDeviceOut { KVOut* kv; uint32_t* count; uint32_t* found; uint32_t* searched; uint32_t stride; };

// The deep buffer: the deep queries' emitted slices (structure of arrays, 30 bytes an entry, 64-bit index), then two
// DeepEntry arrays and the head flags for the largest slice, then CUB's scratch. Sized by the plan's upper bounds before
// anything runs; when it cannot be allocated the call fails with TSGPU_ERR_CAPACITY and the index stays usable.
constexpr size_t kDeepKeepBytes = size_t(256) << 20;

struct DeepBuf {
    int64_t *s0 = nullptr, *s1 = nullptr, *s2 = nullptr; uint32_t* key = nullptr; uint16_t* cmb = nullptr;
    DeepEntry *a = nullptr, *b = nullptr; uint8_t* head = nullptr; unsigned long long* n_sel = nullptr;
    void* temp = nullptr; size_t temp_bytes = 0;
};

tsgpu_status deep_reserve(tsgpu_index* idx, const KwPlan& pl, DeepBuf& db) {
    const size_t T = pl.deep_off.back(), M = pl.deep_max;
    size_t t1 = 0, t2 = 0, t3 = 0;
    DeepEntry* const none = nullptr;
    CU(cub::DeviceRadixSort::SortKeysDescending(nullptr, t1, none, none, M, DeepKvOrder{}));
    CU(cub::DeviceRadixSort::SortKeysDescending(nullptr, t2, none, none, M, DeepKeyOrder{}));
    CU(cub::DeviceSelect::Flagged(nullptr, t3, none, static_cast<const uint8_t*>(nullptr), none, static_cast<unsigned long long*>(nullptr), M));
    db.temp_bytes = std::max(t1, std::max(t2, t3));
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off = (off + bytes + 255) & ~size_t(255); return o; };
    const size_t o0 = take(T * 8), o1 = take(T * 8), o2 = take(T * 8), ok = take(T * 4), oc = take(T * 2);
    const size_t oa = take(M * sizeof(DeepEntry)), ob = take(M * sizeof(DeepEntry)), oh = take(M), on = take(8), ot = take(db.temp_bytes);
    idx->stats.deep_bytes = off;
    if(idx->d_deep.reserve(off) != cudaSuccess) {
        cudaGetLastError();                   // an allocation failure is not sticky: clear it so the next call starts clean
        return fail(TSGPU_ERR_CAPACITY, "deep Topster needs " + std::to_string(off) + " bytes of device memory; lower topk or split the batch");
    }
    unsigned char* p = idx->d_deep.as<unsigned char>();
    db.s0 = reinterpret_cast<int64_t*>(p + o0); db.s1 = reinterpret_cast<int64_t*>(p + o1); db.s2 = reinterpret_cast<int64_t*>(p + o2);
    db.key = reinterpret_cast<uint32_t*>(p + ok); db.cmb = reinterpret_cast<uint16_t*>(p + oc);
    db.a = reinterpret_cast<DeepEntry*>(p + oa); db.b = reinterpret_cast<DeepEntry*>(p + ob);
    db.head = p + oh; db.n_sel = reinterpret_cast<unsigned long long*>(p + on); db.temp = p + ot;
    return TSGPU_OK;
}

// After the unit kernels: de-duplicate, select and write every deep query's Topster (deep_topster.cuh). The entry counts
// come back to the host first, so the sorts are sized by what was emitted, not by the bound.
tsgpu_status run_deep_select(tsgpu_index* idx, const KwPlan& pl, DeepBuf& db, const KwDeviceOut& out) {
    cudaStream_t st = idx->stream;
    std::vector<long long> cur(pl.nq);
    std::vector<uint32_t> cm(pl.nc);
    CU(cudaMemcpyAsync(cur.data(), pl.d_deep_cur, (size_t) pl.nq * 8, cudaMemcpyDeviceToHost, st));
    if(pl.nc) CU(cudaMemcpyAsync(cm.data(), pl.d_combo_matches, (size_t) pl.nc * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const unsigned grid_cap = (unsigned) idx->n_sms * 8;
    auto grid = [&](size_t n) { return (unsigned) std::max<size_t>(1, std::min<size_t>((n + 255) / 256, grid_cap)); };
    float ms_dedup = 0, ms_select = 0;
    for(size_t i = 0; i < pl.deep_q.size(); i++) {
        const uint32_t q = pl.deep_q[i];
        const QDesc& qd = pl.qd[q];
        const size_t base = pl.deep_off[i];
        size_t n = (size_t) cur[q] - base;
        idx->stats.deep_entries += n;
        if(n == 0) continue;                  // kw_final_kernel wrote count 0
        uint32_t with_matches = 0;
        for(uint32_t c = qd.combo_begin; c < qd.combo_end; c++) with_matches += cm[c] != 0;
        const bool dedup = with_matches > 1;
        CU(cudaEventRecord(idx->deep_ev[1], st));
        deep_pack_kernel<<<grid(n), 256, 0, st>>>(db.s0 + base, db.s1 + base, db.s2 + base, db.key + base, db.cmb + base, n, dedup ? 1 : 0, db.a);
        idx->stats.launches_total++;
        CU(cudaGetLastError());
        if(dedup) {
            size_t tb = db.temp_bytes;
            CU(cub::DeviceRadixSort::SortKeysDescending(db.temp, tb, db.a, db.b, n, DeepKeyOrder{}, st));
            deep_heads_kernel<<<grid(n), 256, 0, st>>>(db.b, n, db.a, db.head);
            idx->stats.launches_total++;
            CU(cudaGetLastError());
            tb = db.temp_bytes;
            CU(cub::DeviceSelect::Flagged(db.temp, tb, db.a, static_cast<const uint8_t*>(db.head), db.b, db.n_sel, n, st));
            unsigned long long n_sel = 0;
            CU(cudaMemcpyAsync(&n_sel, db.n_sel, 8, cudaMemcpyDeviceToHost, st));
            CU(cudaStreamSynchronize(st));
            n = (size_t) n_sel;
            std::swap(db.a, db.b);            // the distinct entries are in a
        }
        CU(cudaEventRecord(idx->deep_ev[2], st));
        size_t tb = db.temp_bytes;
        CU(cub::DeviceRadixSort::SortKeysDescending(db.temp, tb, db.a, db.b, n, DeepKvOrder{}, st));
        const uint32_t n_out = (uint32_t) std::min<size_t>(n, std::min(qd.topk, out.stride));
        deep_write_kernel<<<grid(n_out), 256, 0, st>>>(db.b, n_out, pl.d_qd, q, pl.d_combo_matches, out.kv, out.stride, out.count);
        idx->stats.launches_total++;
        CU(cudaGetLastError());
        CU(cudaEventRecord(idx->deep_ev[3], st));
        CU(cudaEventSynchronize(idx->deep_ev[3]));
        float ms = 0;
        cudaEventElapsedTime(&ms, idx->deep_ev[1], idx->deep_ev[2]); ms_dedup += ms;
        cudaEventElapsedTime(&ms, idx->deep_ev[2], idx->deep_ev[3]); ms_select += ms;
    }
    idx->stats.ms_deep_dedup = ms_dedup; idx->stats.ms_deep_select = ms_select;
    return TSGPU_OK;
}

// intersect/score/select + per-query merge; leaves KVOut/count/found/searched in idx->d_kw_out
tsgpu_status run_keyword(tsgpu_index* idx, KwPlan& pl, uint32_t kv_stride, KwDeviceOut& out) {
    cudaStream_t st = idx->stream;
    const uint32_t nq = pl.nq;
    const size_t kv_bytes = (size_t) nq * kv_stride * sizeof(KVOut);
    CU(idx->d_kw_out.reserve(kv_bytes + (size_t) nq * 12 + 64));
    out.kv = idx->d_kw_out.as<KVOut>();
    out.count = reinterpret_cast<uint32_t*>(idx->d_kw_out.as<unsigned char>() + ((kv_bytes + 15) & ~size_t(15)));
    out.found = out.count + nq;
    out.searched = out.found + nq;
    out.stride = kv_stride;
    CU(idx->d_pool.reserve(pl.pool_slots * 30 + 64));
    int64_t* p0 = idx->d_pool.as<int64_t>();
    int64_t* p1 = p0 + pl.pool_slots;
    int64_t* p2 = p1 + pl.pool_slots;
    uint32_t* pk = reinterpret_cast<uint32_t*>(p2 + pl.pool_slots);
    uint16_t* pc = reinterpret_cast<uint16_t*>(pk + pl.pool_slots);
    const bool deep = !pl.deep_q.empty();
    DeepBuf db;
    if(deep) {
        tsgpu_status s = deep_reserve(idx, pl, db); if(s) return s;
        for(auto& e: idx->deep_ev) if(!e) CU(cudaEventCreate(&e));
    }
    const unsigned n_deep_units = (unsigned) pl.deep_ud.size();
    CU(cudaEventRecord(idx->ev[1], st));
    if((pl.n_units || n_deep_units) && pl.wildcard) {
        // per-query id arrays
        std::vector<const uint32_t*> qids(nq);
        for(uint32_t q = 0; q < nq; q++) qids[q] = pl.q_filter_ids[q];
        const size_t n_sc = pl.id_scores ? pl.n_inline_ids : 0;
        const size_t o_sp = ((size_t) nq * 12 + 63) & ~size_t(63), o_sc = o_sp + (size_t) nq * 8;
        const size_t tb = o_sc + n_sc * 8 + 64;
        CU(idx->d_small.reserve(tb));
        unsigned char* sb = idx->d_small.as<unsigned char>();
        CU(cudaMemcpyAsync(sb, qids.data(), (size_t) nq * 8, cudaMemcpyHostToDevice, st));            // on the kernel's stream: the default stream does not order with it
        CU(cudaMemcpyAsync(sb + (size_t) nq * 8, pl.q_nids.data(), (size_t) nq * 4, cudaMemcpyHostToDevice, st));
        idx->stats.h2d_bytes += (size_t) nq * 12;
        WcParams P{};
        P.qd = pl.d_qd; P.ud = pl.d_ud;
        P.q_ids = reinterpret_cast<const uint32_t* const*>(sb); P.q_nids = reinterpret_cast<const uint32_t*>(sb + (size_t) nq * 8);
        P.q_scores = nullptr;
        if(pl.id_scores) {                       // per-id match scores ride next to the ids they belong to
            CU(cudaMemcpyAsync(sb + o_sc, pl.id_scores, n_sc * 8, cudaMemcpyDefault, st));
            std::vector<const int64_t*> qsc(nq, nullptr);
            for(uint32_t q = 0; q < nq; q++) if(pl.q_inline_off[q] != ~0ull) qsc[q] = reinterpret_cast<const int64_t*>(sb + o_sc) + pl.q_inline_off[q];
            CU(cudaMemcpyAsync(sb + o_sp, qsc.data(), (size_t) nq * 8, cudaMemcpyHostToDevice, st));
            P.q_scores = reinterpret_cast<const int64_t* const*>(sb + o_sp);
            idx->stats.h2d_bytes += n_sc * 8 + (size_t) nq * 8;
        }
        P.pool_s0 = p0; P.pool_s1 = p1; P.pool_s2 = p2; P.pool_key = pk; P.pool_cmb = pc;
        P.unit_cnt = pl.d_unit_cnt; P.combo_matches = pl.d_combo_matches; P.q_thr = pl.d_q_thr; P.KP = pl.KP;
        const size_t smem = (size_t) 2 * pl.KP * 28;
        if(pl.n_units) {
            CU(cudaFuncSetAttribute(wc_unit_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) std::max<size_t>(smem, 48 * 1024)));
            wc_unit_kernel<false><<<pl.n_units, kThreads, smem, st>>>(P);
            idx->stats.launches_total++;
            CU(cudaGetLastError());
        }
        if(n_deep_units) {
            P.ud = pl.d_deep_ud; P.q_thr = pl.d_deep_cur; P.KP = 0;
            P.pool_s0 = db.s0; P.pool_s1 = db.s1; P.pool_s2 = db.s2; P.pool_key = db.key; P.pool_cmb = db.cmb;
            CU(cudaEventRecord(idx->deep_ev[0], st));
            wc_unit_kernel<true><<<n_deep_units, kThreads, 0, st>>>(P);
            idx->stats.launches_total++;
            CU(cudaGetLastError());
        }
    } else if(pl.n_units || n_deep_units) {
        KwParams P{};
        P.qd = pl.d_qd; P.cd = pl.d_cd; P.ud = pl.d_ud;
        P.pool_s0 = p0; P.pool_s1 = p1; P.pool_s2 = p2; P.pool_key = pk; P.pool_cmb = pc;
        P.unit_cnt = pl.d_unit_cnt; P.combo_matches = pl.d_combo_matches; P.stats = pl.d_stats;
        P.q_thr = pl.d_q_thr;
        P.F = pl.F; P.KP = pl.KP; P.NL = pl.NL;
        for(uint32_t f = 0; f < (uint32_t) kMaxFieldSlots; f++) P.field_ids[f] = pl.field_ids[f];
        if(pl.n_units) {
            const size_t smem = kw_search_smem(pl.KP, pl.NL);
            static const bool reg_score = !(getenv("TSGPU_REG_SCORE") && atoi(getenv("TSGPU_REG_SCORE")) == 0);   // default; =0 selects the general scorer (kw_search_kernel<false>) for A/B
            if(reg_score) CU(tsgpu_launch_kw_search_regscore(&idx->ixdev, &P, pl.n_units, smem, st));          // kw_regscore.cu
            else {
                CU(cudaFuncSetAttribute(kw_search_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) std::max<size_t>(smem, 48 * 1024)));
                kw_search_kernel<false><<<pl.n_units, kThreads, smem, st>>>(idx->ixdev, P);
            }
            idx->stats.launches_total++;
            CU(cudaGetLastError());
        }
        if(n_deep_units) {                    // the register-resident scorer without the top-K buffer (kw_deep.cu)
            P.ud = pl.d_deep_ud; P.q_thr = pl.d_deep_cur; P.KP = 0;
            P.pool_s0 = db.s0; P.pool_s1 = db.s1; P.pool_s2 = db.s2; P.pool_key = db.key; P.pool_cmb = db.cmb;
            CU(cudaEventRecord(idx->deep_ev[0], st));
            CU(tsgpu_launch_kw_search_deep(&idx->ixdev, &P, n_deep_units, kw_search_smem(0, pl.NL), st));
            idx->stats.launches_total++;
        }
    }
    CU(cudaEventRecord(idx->ev[6], st));
    {
        FinalParams P{};
        P.qd = pl.d_qd; P.ud = pl.d_ud; P.md = nullptr;
        P.pool_s0 = p0; P.pool_s1 = p1; P.pool_s2 = p2; P.pool_key = pk; P.pool_cmb = pc;
        P.unit_cnt = pl.d_unit_cnt; P.combo_matches = pl.d_combo_matches;
        P.out_kv = out.kv; P.out_count = out.count; P.out_found = out.found; P.out_searched = out.searched;
        P.kv_stride = kv_stride; P.KP = pl.KP;
        const size_t smem = kw_final_smem(pl);
        CU(cudaFuncSetAttribute(kw_final_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) std::max<size_t>(smem, 48 * 1024)));
        CU(cudaFuncSetAttribute(kw_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) std::max<size_t>(smem, 48 * 1024)));
        for(size_t lv = 0; lv < pl.levels.size(); lv++) {
            P.md = pl.d_levels[lv];
            kw_merge_kernel<<<(unsigned) pl.levels[lv].size(), kFinalThreads, smem, st>>>(P);
            idx->stats.launches_total++;
        }
        CU(cudaGetLastError());
        if(nq) {
            kw_final_kernel<<<nq, kFinalThreads, smem, st>>>(P);
            idx->stats.launches_total++;
        }
        CU(cudaGetLastError());
        if(!pl.multi_q.empty()) {
            const uint32_t n_vec = (uint32_t) (((((size_t) idx->n_docs + 31) / 32) + 3) / 4);
            found_popcount_kernel<<<dim3((unsigned) pl.multi_q.size(), 4), 256, 0, st>>>(pl.d_qd, pl.d_multi_q, n_vec, out.found, 1);
            idx->stats.launches_total++;
            CU(cudaGetLastError());
            idx->found_dirty = false;
        }
        if(!pl.multi_keep_q.empty()) {         // same count, bitmap left in place
            const uint32_t n_vec = (uint32_t) (((((size_t) idx->n_docs + 31) / 32) + 3) / 4);
            found_popcount_kernel<<<dim3((unsigned) pl.multi_keep_q.size(), 4), 256, 0, st>>>(pl.d_qd, pl.d_multi_keep_q, n_vec, out.found, 0);
            idx->stats.launches_total++;
            CU(cudaGetLastError());
        }
    }
    if(deep) {
        // kw_final_kernel gave the deep queries (no ordinary units) their found / query counts and count 0; the selection
        // below writes their records and count
        tsgpu_status s = run_deep_select(idx, pl, db, out); if(s) return s;
        if(n_deep_units) cudaEventElapsedTime(&idx->stats.ms_deep_emit, idx->deep_ev[0], idx->ev[6]);
        // run_deep_select has waited for its last kernel: a large deep buffer goes back to the device at once rather than
        // staying with the index (a q=* over 10 M documents needs 1.3 GB); small ones are kept for the next call
        if(idx->d_deep.cap > kDeepKeepBytes) idx->d_deep.release();
    }
    CU(cudaEventRecord(idx->ev[2], st));
    return TSGPU_OK;
}

// ------------------------------------------------------------------------------------------------- knn
struct KnnDeviceOut { float* dist; uint32_t* labels; uint32_t* n; uint32_t stride; };

template <int NCH>
void launch_hnsw(tsgpu_index* idx, const tsv::KnnParams& P, unsigned grid, size_t smem) {
    cudaFuncSetAttribute(tsv::hnsw_search_kernel<NCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) std::max<size_t>(smem, 48 * 1024));
    tsv::hnsw_search_kernel<NCH><<<grid, tsv::kKnnThreads, smem, idx->vs>>>(idx->hnsw, P);
}

template <int NCH>
void launch_walk(tsgpu_index* idx, const tsv::KnnParams& P, unsigned grid, size_t smem, int rs) {
    if(NCH == 6 && rs == 8) {            // ... and with an eight-row ring (few, long walks: everything a node's expansion needs in one round trip)
        cudaFuncSetAttribute(tsv::hnsw_walk_kernel<NCH == 6 ? 6 : 1, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) std::max<size_t>(smem, 48 * 1024));
        tsv::hnsw_walk_kernel<NCH == 6 ? 6 : 1, 8><<<grid, 32 * tsv::kWalkWarps, smem, idx->vs>>>(idx->hnsw, P);
        return;
    }
    if(NCH == 6 && rs == 2) {            // the 768-d build also exists with a two-row ring (more walks resident per SM)
        cudaFuncSetAttribute(tsv::hnsw_walk_kernel<NCH == 6 ? 6 : 1, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) std::max<size_t>(smem, 48 * 1024));
        tsv::hnsw_walk_kernel<NCH == 6 ? 6 : 1, 2><<<grid, 32 * tsv::kWalkWarps, smem, idx->vs>>>(idx->hnsw, P);
        return;
    }
    cudaFuncSetAttribute(tsv::hnsw_walk_kernel<NCH, tsv::kStageRows>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) std::max<size_t>(smem, 48 * 1024));
    tsv::hnsw_walk_kernel<NCH, tsv::kStageRows><<<grid, 32 * tsv::kWalkWarps, smem, idx->vs>>>(idx->hnsw, P);
}

// d_queries: [nq*dim] on device. q_bitmap/q_excl/q_nexcl/q_skip: host vectors (uploaded here). q_cost: optional per-query
// walk-length estimate (larger = longer; queries are handed out longest first so the batch does not end on a few long walks
// that started last). Results in d_knn_out.
tsgpu_status run_knn(tsgpu_index* idx, const float* d_queries, uint32_t nq, uint32_t k, uint32_t ef,
                     const std::vector<const uint32_t*>& q_bitmap, const std::vector<const uint32_t*>& q_excl,
                     const std::vector<uint32_t>& q_nexcl, const std::vector<uint8_t>& q_skip, const std::vector<float>& q_cost,
                     KnnDeviceOut& out) {
    cudaStream_t st = idx->vs;
    if(!idx->has_hnsw) return fail(TSGPU_ERR_INVALID, "no vector index loaded");
    if(k == 0) return fail(TSGPU_ERR_INVALID, "k must be > 0");
    const uint32_t efe = std::max(ef, k);
    if(efe > 4096) return fail(TSGPU_ERR_CAPACITY, "max(ef,k) must be <= 4096");
    const tsv::HnswDev& g = idx->hnsw;
    // persistent warps: 4 per CTA; residency is bounded by shared memory (result heap + candidate tier + visited tier 1)
    // register-resident queues (hnsw_walk_kernel) when they fit: max(ef,k) <= 128 and a link row per warp; TSGPU_KNN_HEAP=1
    // forces the general heap kernel (A/B runs)
    static const bool force_heap = getenv("TSGPU_KNN_HEAP") && atoi(getenv("TSGPU_KNN_HEAP")) == 1;
    const uint32_t dim = g.dim;
    const int nch = (dim % 128 == 0 && dim / 128 <= 8 && dim / 128 != 5 && dim / 128 != 7) ? (int) (dim / 128) : 0;
    const bool walk = !force_heap && efe <= 32 * tsv::kResPerLane && 2 * g.M <= 32 && nch > 0;
    const unsigned wpc = walk ? (unsigned) tsv::kWalkWarps : 4u;                       // walks (warps) per CTA
    // tuning knobs of the register-queue kernel (defaults are the measured best, see DESIGN.md): rows staged per walk, visited-
    // cache entries per walk, CTAs per SM
    static const int env_rs = getenv("TSGPU_WALK_ROWS") ? atoi(getenv("TSGPU_WALK_ROWS")) : 0;
    static const int env_cache = getenv("TSGPU_WALK_CACHE") ? atoi(getenv("TSGPU_WALK_CACHE")) : 0;
    static const int env_ctas = getenv("TSGPU_WALK_CTAS") ? atoi(getenv("TSGPU_WALK_CTAS")) : 0;
    const int rs = ((env_rs == 2 || env_rs == 8) && nch == 6) ? env_rs : tsv::kStageRows;
    const uint32_t vis_cache = env_cache >= 64 ? pow2_ceil((uint32_t) env_cache) : tsv::kVisCache;
    const size_t per_warp_smem = walk ? (size_t) rs * dim * 4 + (size_t) vis_cache * 4
                                      : ((size_t) efe + 1 + tsv::kCandSmem) * 8 + (size_t) tsv::kVisSmem * 4;
    const size_t q_bytes = nch ? 0 : (size_t) 4 * ((dim + 3) & ~3u) * 4;
    const size_t smem = wpc * per_warp_smem + q_bytes + (walk ? 128 : 0);
    if(smem > 200 * 1024) return fail(TSGPU_ERR_CAPACITY, "max(ef,k) / dim too large for the per-query shared-memory heaps");
    const unsigned smem_blocks = (unsigned) std::max<size_t>(1, (size_t) (227 * 1024) / (smem + 1024));
    const unsigned max_blocks = walk ? (unsigned) idx->n_sms * std::min(smem_blocks, (unsigned) (env_ctas > 0 ? env_ctas : (rs == 2 ? 2 : 1) * TSGPU_WALK_MIN_CTAS))
                                     : (unsigned) idx->n_sms * std::min(idx->knn_blocks_per_sm, smem_blocks);
    const unsigned grid = std::max(1u, std::min(max_blocks, (nq + wpc - 1) / wpc));
    const size_t slots = (size_t) grid * wpc;
    // per-warp scratch in HBM: tier 2 of the visited set (64 Ki keys: walks of up to 48 K visited nodes) and the overflow of
    // the candidate heap (with a selective filter hnswlib pushes every visited node until `ef` allowed results exist).
    // A walk that outgrows either is handed to the retry launch below, whose slots are sized for the whole graph.
    const uint32_t vis2_slots = 1u << 16, cand_cap = std::min<uint32_t>(1u << 16, std::max<uint32_t>(1024, 2 * (g.n_nodes + 1)));    // two pools (near / far) of half each
    if(slots > idx->knn_slots) {
        idx->d_knn_vis.release();
        CU(idx->d_knn_vis.reserve(slots * (size_t) vis2_slots * 4));
        CU(cudaMemsetAsync(idx->d_knn_vis.p, 0, idx->d_knn_vis.cap, st));
        idx->knn_slots = slots;
    }
    CU(idx->d_knn_cand.reserve(slots * (size_t) cand_cap * 8));
    // retry slots (one CTA): visited tier 2 with >= 2 n slots, candidate arena n + 1
    const uint32_t big_vis = pow2_ceil(std::max<uint32_t>(1u << 17, 2 * g.n_nodes + 64)), big_cand = 2 * (g.n_nodes + 1);        // every node is pushed at most once, and either pool may hold them all
    {
        const size_t need = (size_t) 16 * big_vis * 4;
        if(need > idx->d_knn_retry_vis.cap) {
            idx->d_knn_retry_vis.release();
            CU(idx->d_knn_retry_vis.reserve(need));
            CU(cudaMemsetAsync(idx->d_knn_retry_vis.p, 0, idx->d_knn_retry_vis.cap, st));
        }
        CU(idx->d_knn_retry_cand.reserve((size_t) 16 * big_cand * 8));
    }
    // hand-out order: longest expected walks first
    std::vector<uint32_t> order;
    if(!q_cost.empty()) {
        order.resize(nq);
        for(uint32_t q = 0; q < nq; q++) order[q] = q;
        std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b2) { return q_cost[a] > q_cost[b2]; });
    }
    // outputs + per-query pointer tables
    Stager sg;
    const size_t o_bm = sg.add(q_bitmap.empty() ? nullptr : q_bitmap.data(), (size_t) nq * 8);
    const size_t o_ex = sg.add(q_excl.empty() ? nullptr : q_excl.data(), (size_t) nq * 8);
    const size_t o_ne = sg.add(q_nexcl.empty() ? nullptr : q_nexcl.data(), (size_t) nq * 4);
    const size_t o_sk = sg.add(q_skip.empty() ? nullptr : q_skip.data(), (size_t) nq);
    const size_t o_or = sg.add(order.empty() ? nullptr : order.data(), (size_t) nq * 4);
    const size_t o_rl = sg.reserve((size_t) nq * 4 + 64);          // retry list
    const size_t o_wk = sg.reserve((size_t) nq * 8);               // per-walk work counters
    const size_t o_misc = sg.reserve(128);
    memset(sg.host.data() + o_misc, 0, 128);
    idx->knn_tables.swap(sg.host);                 // keep the pageable source alive until the call ends
    const size_t tbl_bytes = idx->knn_tables.size();
    const size_t out_bytes = (size_t) nq * k * 8 + (size_t) nq * 4;
    CU(idx->d_knn_out.reserve(tbl_bytes + out_bytes + 256));
    unsigned char* base = idx->d_knn_out.as<unsigned char>();
    // staging through a dedicated pinned region at the tail of h_stage is not safe while the kw stage is in flight,
    // so use a plain async copy from the pageable vector (small)
    CU(cudaMemcpyAsync(base, idx->knn_tables.data(), tbl_bytes, cudaMemcpyHostToDevice, st));
    idx->stats.h2d_bytes += tbl_bytes;
    unsigned char* ob = base + ((tbl_bytes + 255) & ~size_t(255));
    out.dist = reinterpret_cast<float*>(ob);
    out.labels = reinterpret_cast<uint32_t*>(ob + (size_t) nq * k * 4);
    out.n = reinterpret_cast<uint32_t*>(ob + (size_t) nq * k * 8);
    out.stride = k;
    // misc layout: [0] ticket, [4] retry ticket, [8..40) stats u64 x4, [40] retry_n, [44] retry_n of the retry launch (unused), [48] stats[5]: visited-table probes
    tsv::KnnParams P{};
    P.queries = d_queries; P.nq = nq; P.k = k; P.ef = ef;
    P.q_filter_bitmap = q_bitmap.empty() ? nullptr : reinterpret_cast<const uint32_t* const*>(base + o_bm);
    P.q_excl = q_excl.empty() ? nullptr : reinterpret_cast<const uint32_t* const*>(base + o_ex);
    P.q_n_excl = q_nexcl.empty() ? nullptr : reinterpret_cast<const uint32_t*>(base + o_ne);
    P.q_skip = q_skip.empty() ? nullptr : reinterpret_cast<const uint8_t*>(base + o_sk);
    P.q_order = order.empty() ? nullptr : reinterpret_cast<const uint32_t*>(base + o_or);
    P.n_order = nq; P.n_order_dev = nullptr;
    P.out_dist = out.dist; P.out_labels = out.labels; P.out_n = out.n;
    P.vis2 = idx->d_knn_vis.as<uint32_t>(); P.vis2_slots = vis2_slots;
    P.cand = idx->d_knn_cand.as<unsigned long long>(); P.cand_cap = cand_cap;
    P.counter = reinterpret_cast<uint32_t*>(base + o_misc);
    P.stats = reinterpret_cast<unsigned long long*>(base + o_misc + 8);
    P.retry_n = reinterpret_cast<uint32_t*>(base + o_misc + 40);
    P.retry_list = reinterpret_cast<uint32_t*>(base + o_rl);
    P.q_work = reinterpret_cast<uint32_t*>(base + o_wk);
    P.vis_cache = vis_cache;
    static const int env_pf = getenv("TSGPU_WALK_PREFETCH") ? atoi(getenv("TSGPU_WALK_PREFETCH")) : 5;
    P.walk_prefetch = (uint32_t) env_pf & 7u;
    idx->knn_work_dev = P.q_work; idx->knn_work_n = nq;
    // the retry launch: the same kernel over the queries the first one handed back, one CTA whose four slots can hold a
    // walk over the whole graph. It reads its ticket count from device memory, so it is issued unconditionally (no host
    // round trip between the two) and ends at once when nothing was handed back.
    tsv::KnnParams R = P;
    R.q_order = P.retry_list; R.n_order = 0; R.n_order_dev = P.retry_n; R.q_skip = nullptr;
    R.vis2 = idx->d_knn_retry_vis.as<uint32_t>(); R.vis2_slots = big_vis;
    R.cand = idx->d_knn_retry_cand.as<unsigned long long>(); R.cand_cap = big_cand;
    R.counter = reinterpret_cast<uint32_t*>(base + o_misc + 4);
    R.retry_n = reinterpret_cast<uint32_t*>(base + o_misc + 44);
    R.retry_list = reinterpret_cast<uint32_t*>(base + o_rl + (size_t) nq * 4);    // cannot be reached: nothing outgrows a full-size slot
    CU(cudaEventRecord(idx->ev[3], st));
    if(walk) switch(nch) {
        case 1: launch_walk<1>(idx, P, grid, smem, rs); launch_walk<1>(idx, R, 4, smem, rs); break;
        case 2: launch_walk<2>(idx, P, grid, smem, rs); launch_walk<2>(idx, R, 4, smem, rs); break;
        case 3: launch_walk<3>(idx, P, grid, smem, rs); launch_walk<3>(idx, R, 4, smem, rs); break;
        case 4: launch_walk<4>(idx, P, grid, smem, rs); launch_walk<4>(idx, R, 4, smem, rs); break;
        case 6: launch_walk<6>(idx, P, grid, smem, rs); launch_walk<6>(idx, R, 4, smem, rs); break;
        case 8: launch_walk<8>(idx, P, grid, smem, rs); launch_walk<8>(idx, R, 4, smem, rs); break;
        default: launch_walk<1>(idx, P, grid, smem, rs); launch_walk<1>(idx, R, 4, smem, rs); break;
    }
    else switch(nch) {
        case 1: launch_hnsw<1>(idx, P, grid, smem); launch_hnsw<1>(idx, R, 1, smem); break;
        case 2: launch_hnsw<2>(idx, P, grid, smem); launch_hnsw<2>(idx, R, 1, smem); break;
        case 3: launch_hnsw<3>(idx, P, grid, smem); launch_hnsw<3>(idx, R, 1, smem); break;
        case 4: launch_hnsw<4>(idx, P, grid, smem); launch_hnsw<4>(idx, R, 1, smem); break;
        case 6: launch_hnsw<6>(idx, P, grid, smem); launch_hnsw<6>(idx, R, 1, smem); break;
        case 8: launch_hnsw<8>(idx, P, grid, smem); launch_hnsw<8>(idx, R, 1, smem); break;
        default: launch_hnsw<0>(idx, P, grid, smem); launch_hnsw<0>(idx, R, 1, smem); break;
    }
    idx->stats.launches_total += 2;
    CU(cudaGetLastError());
    CU(cudaEventRecord(idx->ev[4], st));
    idx->knn_misc_dev = base + o_misc;        // counters are read by finish_knn() after the final sync
    return TSGPU_OK;
}

tsgpu_status finish_knn(tsgpu_index* idx) {
    if(!idx->knn_misc_dev) return TSGPU_OK;
    unsigned long long hst[6];
    CU(cudaMemcpy(hst, idx->knn_misc_dev + 8, 48, cudaMemcpyDeviceToHost));
    idx->stats.knn_table_probes += hst[5];
    idx->knn_misc_dev = nullptr;
    idx->stats.knn_dist += hst[0]; idx->stats.knn_expanded += hst[1]; idx->stats.knn_spec_hits += hst[2];
    idx->stats.knn_tier2_walks += hst[3];
    idx->stats.knn_retried += (uint32_t) hst[4];
    return TSGPU_OK;
}

// smallest group of flat-path queries sharing a candidate set that goes to the tensor-core scan (0 = never; TSGPU_FLAT_TC=0)
int flat_tc_min_group() {
    static const int v = [] {
        if(const char* e = getenv("TSGPU_FLAT_TC")) if(atoi(e) == 0) return 0;
        if(const char* e = getenv("TSGPU_FLAT_TC_MIN")) return std::max(1, atoi(e));
        return 8;
    }();
    return v;
}

bool flat_tc_forced() { static const bool v = [] { const char* e = getenv("TSGPU_FLAT_TC"); return e && atoi(e) == 1; }(); return v; }

template <int NCH>
void launch_flat(tsgpu_index* idx, const tsv::FlatParams& P, unsigned long long total, unsigned grid, size_t smem) {
    tsv::flat_distance_kernel<NCH><<<grid, 256, smem, idx->vs>>>(idx->hnsw, P, total);
}

tsgpu_status run_flat(tsgpu_index* idx, const tsv::FlatParams& P, unsigned long long total) {
    if(total == 0) return TSGPU_OK;
    const uint32_t dim = idx->hnsw.dim;
    const int nch = (dim % 128 == 0) ? (int) (dim / 128) : 0;
    const unsigned grid = (unsigned) std::min<unsigned long long>((total + 7) / 8, (unsigned long long) idx->n_sms * 8);
    const size_t q_bytes = (size_t) 8 * ((dim + 3) & ~3u) * 4;
    switch(nch) {
        case 1: launch_flat<1>(idx, P, total, grid, 0); break;
        case 2: launch_flat<2>(idx, P, total, grid, 0); break;
        case 3: launch_flat<3>(idx, P, total, grid, 0); break;
        case 4: launch_flat<4>(idx, P, total, grid, 0); break;
        case 6: launch_flat<6>(idx, P, total, grid, 0); break;
        case 8: launch_flat<8>(idx, P, total, grid, 0); break;
        default: launch_flat<0>(idx, P, total, grid, q_bytes); break;
    }
    idx->stats.launches_total++;
    CU(cudaGetLastError());
    return TSGPU_OK;
}

void begin_call(tsgpu_index* idx) {
    const uint64_t launches = idx->stats.launches_total;
    const uint64_t h2d = idx->stats.h2d_total + idx->stats.h2d_bytes, d2h = idx->stats.d2h_total + idx->stats.d2h_bytes, calls = idx->stats.calls_total + 1;
    idx->stats = tsgpu_stats{};
    idx->stats.launches_total = launches;
    idx->stats.h2d_total = h2d; idx->stats.d2h_total = d2h; idx->stats.calls_total = calls;      // totals up to (not including) this call
    cudaEventRecord(idx->ev[0], idx->stream);
}

tsgpu_status end_call(tsgpu_index* idx, bool kw, bool knn) {
    cudaStream_t st = idx->stream;
    CU(cudaEventRecord(idx->ev[5], st));
    CU(cudaStreamSynchronize(st));
    float ms = 0;
    cudaEventElapsedTime(&ms, idx->ev[0], idx->ev[5]); idx->stats.ms_total = ms;
    if(kw) {
        cudaEventElapsedTime(&ms, idx->ev[1], idx->ev[2]); idx->stats.ms_keyword = ms;
        if(cudaEventElapsedTime(&ms, idx->ev[1], idx->ev[6]) == cudaSuccess) idx->stats.ms_kw_search = ms;
        if(cudaEventElapsedTime(&ms, idx->ev[6], idx->ev[2]) == cudaSuccess) idx->stats.ms_kw_merge = ms;
        cudaGetLastError();
    }
    if(knn) { cudaEventElapsedTime(&ms, idx->ev[3], idx->ev[4]); idx->stats.ms_knn = ms; }
    idx->stats.ms_kernels = idx->stats.ms_keyword + idx->stats.ms_knn + idx->stats.ms_fuse;
    return TSGPU_OK;
}

tsgpu_status fetch_kw_stats(tsgpu_index* idx, const KwPlan& pl) {
    unsigned long long h[4];
    CU(cudaMemcpyAsync(h, pl.d_stats, 32, cudaMemcpyDeviceToHost, idx->stream));
    CU(cudaStreamSynchronize(idx->stream));
    idx->stats.kw_driver_ids = h[0]; idx->stats.kw_probe_ids = h[1]; idx->stats.kw_matches = h[2];
    return TSGPU_OK;
}

// vector stage shared by tsgpu_vector_search_batch / tsgpu_hybrid_search_batch: uploads the query vectors, splits
// queries into the flat (filtered set below flat_search_cutoff) and HNSW paths exactly as src/index.cpp:3664-3670 /
// 4056-4065 do, and runs both.
struct VecStage {
    KnnDeviceOut knn{};
    const float* flat_dist = nullptr; const uint32_t* flat_ids = nullptr; const unsigned long long* flat_off = nullptr;
    const uint8_t* d_is_flat = nullptr;
    const float* d_queries = nullptr;
    bool any_flat = false;
    uint32_t k = 0;
};

tsgpu_status run_vector_stage(tsgpu_index* idx, const tsgpu_kw_batch* b, KwPlan& pl, const float* qvecs,
                              const tsgpu_vec_params* vp, uint32_t k, VecStage& vs) {
    cudaStream_t st = idx->vs;
    const uint32_t nq = pl.nq, dim = idx->hnsw.dim;
    vs.k = k;
    // decide paths
    std::vector<uint8_t>& is_flat = idx->tmp_is_flat;
    std::vector<unsigned long long>& foff = idx->tmp_foff;
    is_flat.assign(nq, 0); foff.assign((size_t) nq + 1, 0);
    for(uint32_t q = 0; q < nq; q++) {
        const bool filter_given = b->q_filter[q] != -1;
        if(filter_given && pl.q_filter_n[q] < vp->flat_search_cutoff) is_flat[q] = 1;
        foff[q + 1] = foff[q] + (is_flat[q] ? pl.q_filter_n[q] : 0);
    }
    const unsigned long long total_flat = foff[nq];
    vs.any_flat = total_flat > 0 || std::any_of(is_flat.begin(), is_flat.end(), [](uint8_t x) { return x != 0; });
    // device scratch: queries | is_flat | flat_off | flat ids | flat dist
    const size_t q_bytes = (size_t) nq * dim * 4;
    const size_t o_q = 0;
    const size_t o_if = (q_bytes + 255) & ~size_t(255);
    const size_t o_fo = (o_if + nq + 255) & ~size_t(255);
    const size_t o_fi = (o_fo + (size_t) (nq + 1) * 8 + 255) & ~size_t(255);
    const size_t o_fd = (o_fi + total_flat * 4 + 255) & ~size_t(255);
    const size_t o_sk = (o_fd + total_flat * 4 + 255) & ~size_t(255);
    const size_t tot = o_sk + nq + 256;
    CU(idx->d_small.reserve(tot));
    unsigned char* base = idx->d_small.as<unsigned char>();
    CU(cudaMemcpyAsync(base + o_q, qvecs, q_bytes, cudaMemcpyDefault, st));
    CU(cudaMemcpyAsync(base + o_if, is_flat.data(), nq, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(base + o_fo, foff.data(), (size_t) (nq + 1) * 8, cudaMemcpyHostToDevice, st));
    idx->stats.h2d_bytes += q_bytes + nq + (size_t) (nq + 1) * 8;
    for(uint32_t q = 0; q < nq; q++) {
        if(is_flat[q] && pl.q_filter_n[q])
            CU(cudaMemcpyAsync(base + o_fi + foff[q] * 4, pl.q_filter_ids[q], pl.q_filter_n[q] * 4, cudaMemcpyDeviceToDevice, st));
    }
    vs.d_is_flat = base + o_if;
    vs.d_queries = reinterpret_cast<const float*>(base + o_q);
    vs.flat_off = reinterpret_cast<const unsigned long long*>(base + o_fo);
    vs.flat_ids = reinterpret_cast<const uint32_t*>(base + o_fi);
    vs.flat_dist = reinterpret_cast<const float*>(base + o_fd);
    if(total_flat) {
        // Flat queries that share a candidate set (the same filter's id array) are a GEMM [ids x dim] . [dim x queries]: those
        // groups go to the tensor-core scan (flat_tc.cu); the scalar kernel answers the rest.
        std::vector<uint8_t> tc_skip;
        std::vector<std::vector<uint32_t>> groups;
        if(flat_tc_min_group() > 0 && ((vp->flags & TSGPU_VEC_FLAT_TENSOR) || flat_tc_forced()) && tsgpu_flat_tc_supported_(dim)) {
            std::map<const uint32_t*, size_t> by_ids;
            for(uint32_t q = 0; q < nq; q++) {
                if(!is_flat[q] || pl.q_filter_n[q] < 128) continue;
                auto it = by_ids.find(pl.q_filter_ids[q]);
                if(it == by_ids.end()) { by_ids[pl.q_filter_ids[q]] = groups.size(); groups.emplace_back(1, q); }
                else groups[it->second].push_back(q);
            }
            groups.erase(std::remove_if(groups.begin(), groups.end(), [](const std::vector<uint32_t>& g) { return g.size() < (size_t) flat_tc_min_group(); }), groups.end());
        }
        size_t skipped = 0;
        if(!groups.empty()) {
            tc_skip.assign(nq, 0);
            // per group: [qsel u32 x ng | out_off u64 x ng] + the packed query tiles; one scratch buffer, laid out up front
            std::vector<size_t> o_sel(groups.size()), o_off(groups.size()), o_img(groups.size());
            size_t tot_tc = 0;
            for(size_t gi = 0; gi < groups.size(); gi++) {
                const size_t ng = groups[gi].size();
                o_sel[gi] = tot_tc; tot_tc = (tot_tc + ng * 4 + 255) & ~size_t(255);
                o_off[gi] = tot_tc; tot_tc = (tot_tc + ng * 8 + 1023) & ~size_t(1023);
                o_img[gi] = tot_tc; tot_tc += tsgpu_flat_tc_image_bytes_((uint32_t) ng, dim, nullptr, nullptr);
                tot_tc = (tot_tc + 1023) & ~size_t(1023);
            }
            CU(idx->d_flat_tc.reserve(tot_tc + 1024));
            unsigned char* tb = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(idx->d_flat_tc.p) + 1023) & ~uintptr_t(1023));
            std::vector<unsigned char>& hb = idx->flat_tc_host;
            hb.assign(tot_tc, 0);
            for(size_t gi = 0; gi < groups.size(); gi++) {
                const auto& g = groups[gi];
                for(size_t j = 0; j < g.size(); j++) {
                    reinterpret_cast<uint32_t*>(hb.data() + o_sel[gi])[j] = g[j];
                    reinterpret_cast<unsigned long long*>(hb.data() + o_off[gi])[j] = foff[g[j]];
                    tc_skip[g[j]] = 1; skipped += pl.q_filter_n[g[j]];
                }
            }
            // only the small index arrays travel (the image regions are written by the pack kernel)
            for(size_t gi = 0; gi < groups.size(); gi++)
                CU(cudaMemcpyAsync(tb + o_sel[gi], hb.data() + o_sel[gi], o_img[gi] - o_sel[gi], cudaMemcpyHostToDevice, st));
            for(size_t gi = 0; gi < groups.size(); gi++) {
                const auto& g = groups[gi];
                int launches = 0;
                CU(tsgpu_flat_tc_run_(idx->hnsw.vectors, idx->hnsw.n_nodes, dim, reinterpret_cast<const float*>(base + o_q),
                                      reinterpret_cast<const uint32_t*>(tb + o_sel[gi]), (uint32_t) g.size(), pl.q_filter_ids[g[0]],
                                      (uint32_t) pl.q_filter_n[g[0]], reinterpret_cast<const unsigned long long*>(tb + o_off[gi]),
                                      reinterpret_cast<float*>(base + o_fd), tb + o_img[gi], idx->n_sms, st, &launches));
                idx->stats.launches_total += launches;
                idx->stats.flat_tc_queries += (uint32_t) g.size();
            }
        }
        if(skipped < total_flat) {
            tsv::FlatParams FP{};
            FP.queries = reinterpret_cast<const float*>(base + o_q);
            FP.ids = vs.flat_ids; FP.q_off = vs.flat_off; FP.nq = nq;
            FP.out_dist = reinterpret_cast<float*>(base + o_fd);
            FP.stats = nullptr;
            if(!tc_skip.empty()) {
                CU(cudaMemcpyAsync(base + o_sk, tc_skip.data(), nq, cudaMemcpyHostToDevice, st));
                FP.q_skip = base + o_sk;
            }
            tsgpu_status s = run_flat(idx, FP, total_flat);
            if(s != TSGPU_OK) return s;
        }
    }
    // HNSW for the rest
    std::vector<uint32_t> nexcl(nq);
    for(uint32_t q = 0; q < nq; q++) nexcl[q] = pl.qd[q].n_excl;
    // a filter that matches nothing lets VectorFilterFunctor through only without exclusions; the reference returns
    // before searching in that case — mark such queries as skipped
    std::vector<uint8_t> skip(is_flat);
    for(uint32_t q = 0; q < nq; q++) if(pl.qd[q].filter_empty) skip[q] = 1;
    // expected walk length: a filter of selectivity s makes hnswlib visit ~1/s times as many nodes before `ef` allowed results exist
    std::vector<float> cost(nq, 1.0f);
    for(uint32_t q = 0; q < nq; q++)
        if(b->q_filter[q] != -1 && pl.q_filter_n[q]) cost[q] = std::min(1e6f, (float) idx->n_docs / (float) pl.q_filter_n[q]);
    return run_knn(idx, reinterpret_cast<const float*>(base + o_q), nq, k, vp->ef, pl.q_bitmap, pl.q_excl_dev, nexcl, skip, cost, vs.knn);
}

#include "deep_fuse_host.inc"

}  // namespace

// ===================================================================================================== C API
extern "C" {

const char* tsgpu_last_error(void) { return g_err.c_str(); }
tsgpu_status tsgpu_host_alloc(size_t bytes, void** out) {
    if(!out) return fail(TSGPU_ERR_INVALID, "null argument");
    *out = nullptr;
    CU(cudaHostAlloc(out, bytes ? bytes : 16, cudaHostAllocPortable));
    return TSGPU_OK;
}
tsgpu_status tsgpu_host_free(void* p) {
    if(p) CU(cudaFreeHost(p));
    return TSGPU_OK;
}
// for the other translation units of the library (art_kernels.cu)
extern "C" __attribute__((visibility("hidden"))) int tsgpu_index_device_(const tsgpu_index* idx) { return idx->device; }
extern "C" __attribute__((visibility("hidden"))) tsgpu_status tsgpu_fail_(tsgpu_status s, const char* msg) { return fail(s, msg); }

int tsgpu_device_count(void) {
    int n = 0;
    if(cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

tsgpu_status tsgpu_index_create(uint32_t n_docs, int device, tsgpu_index** out) {
    if(!out) return fail(TSGPU_ERR_INVALID, "null out");
    int n = 0;
    if(cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        cudaGetLastError();
        return fail(TSGPU_ERR_NO_DEVICE, "no CUDA device: libtsgpu has no CPU fallback");
    }
    if(device < 0 || device >= n) return fail(TSGPU_ERR_INVALID, "bad device ordinal");
    CU(cudaSetDevice(device));
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    tsgpu_index* idx = new tsgpu_index();
    idx->device = device; idx->n_docs = n_docs; idx->n_sms = prop.multiProcessorCount;
    idx->ixdev.n_docs = n_docs;
    if(cudaStreamCreateWithFlags(&idx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete idx; return fail(TSGPU_ERR_CUDA, "stream create failed"); }
    {   // TSGPU_KNN_PRIORITY=1 lets the graph walk's stream outrank the keyword stream (its persistent CTAs then become
        // resident as soon as keyword CTAs retire). Off by default: equal priorities with the keyword kernels launched first
        // were faster on the previous target; not re-measured on H100.
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        const bool prio = getenv("TSGPU_KNN_PRIORITY") && atoi(getenv("TSGPU_KNN_PRIORITY")) == 1;
        if(cudaStreamCreateWithPriority(&idx->stream2, cudaStreamNonBlocking, prio ? hi : lo) != cudaSuccess) { cudaGetLastError(); cudaStreamCreateWithFlags(&idx->stream2, cudaStreamNonBlocking); }
    }
    idx->vs = idx->stream;
    for(auto& e: idx->ev) cudaEventCreate(&e);
    cudaEventCreateWithFlags(&idx->evA, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&idx->evB, cudaEventDisableTiming);
    *out = idx;
    return TSGPU_OK;
}

void tsgpu_index_destroy(tsgpu_index* idx) {
    if(!idx) return;
    cudaSetDevice(idx->device);
    tsgpu_art_release_(idx);
    cudaStreamSynchronize(idx->stream);
    for(auto& f: idx->fields) for(void* p: f.d_alloc) if(p) cudaFree(p);
    for(auto* c: idx->sort_cols) cudaFree(c);
    for(void* p: idx->hnsw_alloc) cudaFree(p);
    if(idx->d_deleted) cudaFree(idx->d_deleted);
    for(auto& f: idx->filters) { if(f.d_bitmap) cudaFree(f.d_bitmap); if(f.d_ids) cudaFree(f.d_ids); }
    for(auto& fm: idx->facets) { if(fm.d_off) cudaFree(fm.d_off); if(fm.d_vals) cudaFree(fm.d_vals); }
    idx->d_keep_bm.release(); idx->d_facet.release(); idx->d_comm.release();
    if(idx->comm) { tsgpu_comm_destroy(idx); }
    DevBuf* bufs[] = {&idx->d_stage, &idx->d_pool, &idx->d_small, &idx->d_bitmaps, &idx->d_found_bm, &idx->d_out, &idx->d_knn_vis,
                      &idx->d_knn_retry_vis, &idx->d_knn_retry_cand, &idx->d_knn_cand, &idx->d_knn_out, &idx->d_isect, &idx->d_kw_out, &idx->d_deep, &idx->d_fuse};
    for(auto* b: bufs) b->release();
    idx->d_div.release(); idx->d_div_ws.release(); idx->h_div.release();
    idx->h_stage.release();
    for(auto& e: idx->ev) if(e) cudaEventDestroy(e);
    for(auto& e: idx->deep_ev) if(e) cudaEventDestroy(e);
    if(idx->evA) cudaEventDestroy(idx->evA);
    if(idx->evB) cudaEventDestroy(idx->evB);
    if(idx->stream2) cudaStreamDestroy(idx->stream2);
    cudaStreamDestroy(idx->stream);
    delete idx;
}

tsgpu_status tsgpu_index_load_field(tsgpu_index* idx, const tsgpu_field* f, uint32_t* out_field) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!f || !out_field) return fail(TSGPU_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(idx->mu);
    if(idx->fields.size() >= (size_t) kMaxIndexFields) return fail(TSGPU_ERR_CAPACITY, "too many fields");
    FieldMirror fm;
    const uint32_t L = f->n_lists;
    fm.h_list_off.resize((size_t) L + 1);
    CU(cudaMemcpy(fm.h_list_off.data(), f->list_off, ((size_t) L + 1) * 8, cudaMemcpyDefault));
    const uint64_t n_post = fm.h_list_off[L];
    std::vector<uint32_t> h_ids(n_post ? n_post : 1);
    if(n_post) CU(cudaMemcpy(h_ids.data(), f->ids, n_post * 4, cudaMemcpyDefault));
    for(uint32_t l = 0; l < L; l++) if(fm.h_list_off[l + 1] < fm.h_list_off[l]) return fail(TSGPU_ERR_INVALID, "list_off not monotone");
    for(uint32_t l = 0; l < L; l++) {
        const uint64_t a0 = fm.h_list_off[l], a1 = fm.h_list_off[l + 1];
        for(uint64_t i = a0; i < a1; i++) {
            if(h_ids[i] >= idx->n_docs) return fail(TSGPU_ERR_INVALID, "seq_id >= n_docs in a posting list");
            if(i > a0 && h_ids[i] <= h_ids[i - 1]) return fail(TSGPU_ERR_INVALID, "posting list ids must be strictly ascending");
        }
    }
    tspack::PackedField pk;
    tspack::pack_field(L, fm.h_list_off.data(), h_ids.data(), pk);
    fm.h_list_blk_off = pk.list_blk_off;
    uint64_t n_pos = 0;
    CU(cudaMemcpy(&n_pos, f->pos_off + n_post, 8, cudaMemcpyDefault));
    auto up = [&](int slot, const void* src, size_t bytes, bool from_user) -> cudaError_t {
        void* d = nullptr;
        cudaError_t e = cudaMalloc(&d, bytes ? bytes : 16);
        if(e != cudaSuccess) return e;
        fm.d_alloc[slot] = d;
        fm.d_bytes[slot] = bytes ? bytes : 16;
        if(bytes) e = cudaMemcpy(d, src, bytes, from_user ? cudaMemcpyDefault : cudaMemcpyHostToDevice);
        return e;
    };
    fm.dense_div = (uint32_t) std::max(1, getenv("TSGPU_DENSE_DIV") ? atoi(getenv("TSGPU_DENSE_DIV")) : 64);
    fm.dense_min_df = tspack::dense_min_df(idx->n_docs, fm.dense_div);
    CU(up(0, fm.h_list_off.data(), ((size_t) L + 1) * 8, false));
    CU(up(1, pk.list_blk_off.data(), pk.list_blk_off.size() * 4, false));
    CU(up(2, pk.blk_first.data(), pk.blk_first.size() * 4, false));
    CU(up(3, pk.blk_info.data(), pk.blk_info.size() * 8, false));
    CU(up(4, pk.packed.data(), pk.packed.size() * 4, false));
    CU(up(5, f->pos_off, (n_post + 1) * 8, true));
    CU(up(6, f->positions, n_pos * 4, true));
    // dense lists: bitmap + rank directory (see postings_device.cuh)
    tspack::pack_dense(L, fm.h_list_off.data(), h_ids.data(), idx->n_docs, fm.dense_min_df, pk);
    fm.h_list_dense = pk.list_dense;
    fm.h_list_first.clear(); fm.h_list_last.clear();
    list_id_range(L, fm.h_list_off.data(), h_ids.data(), 0, fm.h_list_first, fm.h_list_last);
    CU(up(7, pk.list_dense.data(), pk.list_dense.size() * 4, false));
    CU(up(8, pk.dense_bits.data(), pk.dense_bits.size() * 4, false));
    CU(up(9, pk.dense_rank.data(), pk.dense_rank.size() * 4, false));
    fm.dev.n_lists = L;
    fm.dev.is_array = f->is_array ? tsdev::kFieldIsArray : 0;
    if(!f->is_array) {      // validate once so the kernels may take the plain-field fast path
        std::vector<uint64_t> h_po(n_post + 1);
        std::vector<uint32_t> h_pos(n_pos ? n_pos : 1);
        CU(cudaMemcpy(h_po.data(), f->pos_off, (n_post + 1) * 8, cudaMemcpyDefault));
        if(n_pos) CU(cudaMemcpy(h_pos.data(), f->positions, n_pos * 4, cudaMemcpyDefault));
        if(tspack::plain_wellformed(h_po.data(), h_pos.data(), n_post)) {
            fm.dev.is_array |= tsdev::kFieldPlainOk;
            if(tspack::positions_fit_u16(h_pos.data(), n_pos)) fm.dev.is_array |= tsdev::kFieldPos16;
        }
    }
    fm.dev.list_off = (const uint64_t*) fm.d_alloc[0];
    fm.dev.list_blk_off = (const uint32_t*) fm.d_alloc[1];
    fm.dev.blk_first = (const uint32_t*) fm.d_alloc[2];
    fm.dev.blk_info = (const uint64_t*) fm.d_alloc[3];
    fm.dev.packed = (const uint32_t*) fm.d_alloc[4];
    fm.dev.pos_off = (const uint64_t*) fm.d_alloc[5];
    fm.dev.positions = (const uint32_t*) fm.d_alloc[6];
    fm.dev.list_dense = (const uint32_t*) fm.d_alloc[7];
    fm.dev.dense_bits = (const uint32_t*) fm.d_alloc[8];
    fm.dev.dense_rank = (const uint32_t*) fm.d_alloc[9];
    fm.dev.dense_words = pk.dense_words; fm.dev.dense_groups = pk.dense_groups;
    fm.n_post = n_post; fm.n_pos = n_pos; fm.n_words = pk.packed.size() - 1; fm.n_blocks = (uint32_t) pk.blk_first.size(); fm.n_dense = pk.n_dense;
    idx->ixdev.fields[idx->fields.size()] = fm.dev;
    *out_field = (uint32_t) idx->fields.size();
    idx->fields.push_back(std::move(fm));
    CU(cudaDeviceSynchronize());       // default-stream uploads (device-to-device ones are asynchronous) land before any search stream reads them
    return TSGPU_OK;
}

// SURVEY 8 f-4 (posting half). posting_t::upsert / erase (src/posting.cpp:247-333) change a token's list in place on the host; the
// device layout is read-optimised (CSR + packed blocks), so a changed list is WRITTEN AGAIN at the end of the field's arrays and the
// token is pointed at the new list id; the old list stays behind as garbage until the field is compacted (tsgpu_index_compact_field,
// mirror_host.inc). Every array grows by
// reallocation + device-to-device copy (O(field size) per call at HBM speed: batch the writes, as batch_memory_index does).
tsgpu_status tsgpu_index_append_lists(tsgpu_index* idx, uint32_t field, const tsgpu_field* f, uint32_t* out_first_list) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!f || !out_first_list) return fail(TSGPU_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(idx->mu);
    if(field >= idx->fields.size()) return fail(TSGPU_ERR_INVALID, "no such field");
    FieldMirror& fm = idx->fields[field];
    const bool was_array = (fm.dev.is_array & tsdev::kFieldIsArray) != 0;
    if((f->is_array != 0) != was_array) return fail(TSGPU_ERR_INVALID, "is_array differs from the loaded field");
    const uint32_t L0 = fm.dev.n_lists, Ln = f->n_lists;
    *out_first_list = L0;
    if(Ln == 0) return TSGPU_OK;
    if((uint64_t) L0 + Ln >= 0xFFFFFFFEull) return fail(TSGPU_ERR_CAPACITY, "too many lists");
    std::vector<uint64_t> lo((size_t) Ln + 1);
    CU(cudaMemcpy(lo.data(), f->list_off, ((size_t) Ln + 1) * 8, cudaMemcpyDefault));
    if(lo[0] != 0) return fail(TSGPU_ERR_INVALID, "list_off[0] must be 0");
    for(uint32_t l = 0; l < Ln; l++) if(lo[l + 1] < lo[l]) return fail(TSGPU_ERR_INVALID, "list_off not monotone");
    const uint64_t np = lo[Ln];
    std::vector<uint32_t> ids(np ? np : 1);
    if(np) CU(cudaMemcpy(ids.data(), f->ids, np * 4, cudaMemcpyDefault));
    for(uint32_t l = 0; l < Ln; l++)
        for(uint64_t i = lo[l]; i < lo[l + 1]; i++) {
            if(ids[i] >= idx->n_docs) return fail(TSGPU_ERR_INVALID, "seq_id >= n_docs in a posting list");
            if(i > lo[l] && ids[i] <= ids[i - 1]) return fail(TSGPU_ERR_INVALID, "posting list ids must be strictly ascending");
        }
    std::vector<uint64_t> po(np + 1);
    CU(cudaMemcpy(po.data(), f->pos_off, (np + 1) * 8, cudaMemcpyDefault));
    if(po[0] != 0) return fail(TSGPU_ERR_INVALID, "pos_off[0] must be 0");
    for(uint64_t i = 0; i < np; i++) if(po[i + 1] < po[i]) return fail(TSGPU_ERR_INVALID, "pos_off not monotone");
    const uint64_t npos = po[np];
    std::vector<uint32_t> pos(npos ? npos : 1);
    if(npos) CU(cudaMemcpy(pos.data(), f->positions, npos * 4, cudaMemcpyDefault));
    // the fast scoring paths hold only while every posting of the field qualifies
    uint32_t flags = fm.dev.is_array;
    if(!was_array && (flags & tsdev::kFieldPlainOk)) {
        if(!tspack::plain_wellformed(po.data(), pos.data(), np)) flags &= ~(tsdev::kFieldPlainOk | tsdev::kFieldPos16);
        else if((flags & tsdev::kFieldPos16) && !tspack::positions_fit_u16(pos.data(), npos)) flags &= ~tsdev::kFieldPos16;
    }
    tspack::PackedField pk;
    tspack::pack_field(Ln, lo.data(), ids.data(), pk);
    tspack::pack_dense(Ln, lo.data(), ids.data(), idx->n_docs, fm.dense_min_df, pk);
    const uint64_t nw_new = pk.packed.size() - 1;
    const uint32_t nb_new = (uint32_t) pk.blk_first.size();
    if((uint64_t) fm.n_blocks + nb_new >= 0xFFFFFFFFull) return fail(TSGPU_ERR_CAPACITY, "too many posting blocks");
    // rebase the new lists' offsets onto the end of the existing arrays
    for(auto& v: lo) v += fm.n_post;
    for(auto& v: po) v += fm.n_pos;
    for(auto& v: pk.list_blk_off) v += fm.n_blocks;
    for(auto& v: pk.blk_info) v = ((v & 0xFFFFFFFFFFull) + fm.n_words) | (v & ~0xFFFFFFFFFFull);
    for(auto& v: pk.list_dense) if(v != tsdev::kNone) v += fm.n_dense;
    if(fm.n_words + nw_new >= (1ull << 40)) return fail(TSGPU_ERR_CAPACITY, "packed postings exceed the 40-bit word offset");
    // grow: [old | new] into fresh allocations, swap on success
    void* fresh[10] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    size_t fresh_bytes[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    struct Guard { void** v; bool keep = false; ~Guard() { if(!keep) for(int i = 0; i < 10; i++) if(v[i]) cudaFree(v[i]); } } guard{fresh};
    auto grow = [&](int slot, size_t old_bytes, const void* add, size_t add_bytes, size_t tail_zero_bytes) -> cudaError_t {
        void* d = nullptr;
        cudaError_t e = cudaMalloc(&d, old_bytes + add_bytes + tail_zero_bytes + 16);
        if(e != cudaSuccess) return e;
        fresh[slot] = d;
        fresh_bytes[slot] = old_bytes + add_bytes + tail_zero_bytes + 16;
        if(old_bytes) { e = cudaMemcpy(d, fm.d_alloc[slot], old_bytes, cudaMemcpyDeviceToDevice); if(e != cudaSuccess) return e; }
        if(add_bytes) { e = cudaMemcpy((char*) d + old_bytes, add, add_bytes, cudaMemcpyHostToDevice); if(e != cudaSuccess) return e; }
        if(tail_zero_bytes) e = cudaMemset((char*) d + old_bytes + add_bytes, 0, tail_zero_bytes);
        return e;
    };
    const size_t dw = fm.dev.dense_words, dg = fm.dev.dense_groups;
    CU(grow(0, ((size_t) L0 + 1) * 8, lo.data() + 1, (size_t) Ln * 8, 0));
    CU(grow(1, ((size_t) L0 + 1) * 4, pk.list_blk_off.data() + 1, (size_t) Ln * 4, 0));
    CU(grow(2, (size_t) fm.n_blocks * 4, pk.blk_first.data(), (size_t) nb_new * 4, 0));
    CU(grow(3, (size_t) fm.n_blocks * 8, pk.blk_info.data(), (size_t) nb_new * 8, 0));
    CU(grow(4, (size_t) fm.n_words * 4, pk.packed.data(), (size_t) nw_new * 4, 4));              // + the padding word
    CU(grow(5, ((size_t) fm.n_post + 1) * 8, po.data() + 1, (size_t) np * 8, 0));
    CU(grow(6, (size_t) fm.n_pos * 4, pos.data(), (size_t) npos * 4, 0));
    CU(grow(7, (size_t) L0 * 4, pk.list_dense.data(), (size_t) Ln * 4, 0));
    CU(grow(8, (size_t) fm.n_dense * dw * 4, pk.dense_bits.data(), (size_t) pk.n_dense * dw * 4, 64));
    CU(grow(9, (size_t) fm.n_dense * dg * 4, pk.dense_rank.data(), (size_t) pk.n_dense * dg * 4, 4));
    CU(cudaDeviceSynchronize());              // no search of this index is in flight (idx->mu), other indexes' streams finish first
    for(int i = 0; i < 10; i++) { cudaFree(fm.d_alloc[i]); fm.d_alloc[i] = fresh[i]; fm.d_bytes[i] = fresh_bytes[i]; }
    guard.keep = true;
    fm.h_list_off.insert(fm.h_list_off.end(), lo.begin() + 1, lo.end());
    fm.h_list_blk_off.insert(fm.h_list_blk_off.end(), pk.list_blk_off.begin() + 1, pk.list_blk_off.end());
    fm.h_list_dense.resize(L0);               // (the loader keeps one spare entry for an empty field)
    fm.h_list_dense.insert(fm.h_list_dense.end(), pk.list_dense.begin(), pk.list_dense.begin() + Ln);
    list_id_range(Ln, lo.data(), ids.data(), fm.n_post, fm.h_list_first, fm.h_list_last);   // lo is rebased by n_post
    fm.n_post += np; fm.n_pos += npos; fm.n_words += nw_new; fm.n_blocks += nb_new; fm.n_dense += pk.n_dense;
    fm.dev.n_lists = L0 + Ln;
    fm.dev.is_array = flags;
    fm.dev.list_off = (const uint64_t*) fm.d_alloc[0];
    fm.dev.list_blk_off = (const uint32_t*) fm.d_alloc[1];
    fm.dev.blk_first = (const uint32_t*) fm.d_alloc[2];
    fm.dev.blk_info = (const uint64_t*) fm.d_alloc[3];
    fm.dev.packed = (const uint32_t*) fm.d_alloc[4];
    fm.dev.pos_off = (const uint64_t*) fm.d_alloc[5];
    fm.dev.positions = (const uint32_t*) fm.d_alloc[6];
    fm.dev.list_dense = (const uint32_t*) fm.d_alloc[7];
    fm.dev.dense_bits = (const uint32_t*) fm.d_alloc[8];
    fm.dev.dense_rank = (const uint32_t*) fm.d_alloc[9];
    idx->ixdev.fields[field] = fm.dev;
    return TSGPU_OK;
}

// sort_index[field] values of upserted / removed documents (src/index.cpp:1160-1180 on the write path): vals[i] -> column[ids[i]];
// INT64_MIN removes the value.
tsgpu_status tsgpu_index_set_sort_values(tsgpu_index* idx, uint32_t sort_col, const uint32_t* ids, const int64_t* vals, size_t n) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(n && (!ids || !vals)) return fail(TSGPU_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(idx->mu);
    if(sort_col >= idx->sort_cols.size()) return fail(TSGPU_ERR_INVALID, "no such sort column");
    std::vector<uint32_t> h_ids(n ? n : 1);
    std::vector<int64_t> h_vals(n ? n : 1);
    if(n) { CU(cudaMemcpy(h_ids.data(), ids, n * 4, cudaMemcpyDefault)); CU(cudaMemcpy(h_vals.data(), vals, n * 8, cudaMemcpyDefault)); }
    for(size_t i = 0; i < n; i++) if(h_ids[i] >= idx->n_docs) return fail(TSGPU_ERR_INVALID, "seq_id >= n_docs");
    CU(cudaDeviceSynchronize());
    // runs of consecutive ids travel as one copy (a batch of new documents is one run)
    for(size_t i = 0; i < n;) {
        size_t j = i + 1;
        while(j < n && h_ids[j] == h_ids[j - 1] + 1) j++;
        CU(cudaMemcpy(idx->sort_cols[sort_col] + h_ids[i], h_vals.data() + i, (j - i) * 8, cudaMemcpyHostToDevice));
        i = j;
    }
    CU(cudaDeviceSynchronize());
    return TSGPU_OK;
}

tsgpu_status tsgpu_index_load_sort_column(tsgpu_index* idx, const int64_t* vals, uint32_t* out_col) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!vals || !out_col) return fail(TSGPU_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(idx->mu);
    int64_t* d = nullptr;
    CU(cudaMalloc(&d, (size_t) std::max<uint32_t>(idx->n_docs, 1) * 8));
    CU(cudaMemcpy(d, vals, (size_t) idx->n_docs * 8, cudaMemcpyDefault));
    CU(cudaDeviceSynchronize());
    *out_col = (uint32_t) idx->sort_cols.size();
    idx->sort_cols.push_back(d);
    return TSGPU_OK;
}

tsgpu_status tsgpu_index_load_hnsw(tsgpu_index* idx, const tsgpu_hnsw* g) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!g) return fail(TSGPU_ERR_INVALID, "null graph");
    if(g->M == 0 || g->M > 32) return fail(TSGPU_ERR_CAPACITY, "M must be 1..32");
    std::lock_guard<std::mutex> lk(idx->mu);
    // Upload into allocations of their own, check what the kernels will follow blindly, and only then replace the graph the
    // index holds: a failed load (out of memory, a malformed export) leaves the previous graph in place.
    const size_t n = g->n_nodes;
    std::vector<void*> fresh;
    struct Guard { std::vector<void*>& v; bool keep = false; ~Guard() { if(!keep) for(void* p: v) cudaFree(p); } } guard{fresh};
    auto up = [&](const void* src, size_t bytes, const void** dst) -> cudaError_t {
        void* d = nullptr;
        cudaError_t e = cudaMalloc(&d, bytes ? bytes : 16);
        if(e != cudaSuccess) return e;
        fresh.push_back(d);
        *dst = d;
        return bytes ? cudaMemcpy(d, src, bytes, cudaMemcpyDefault) : cudaSuccess;
    };
    tsv::HnswDev h{};
    h.n_nodes = g->n_nodes; h.dim = g->dim; h.M = g->M; h.max_level = g->max_level; h.entry_point = g->entry_point; h.metric = g->metric;
    if(n && g->entry_point >= n) return fail(TSGPU_ERR_INVALID, "hnsw: entry point outside the graph");
    if(n && (!g->vectors || !g->levels || !g->links0 || !g->upper_off)) return fail(TSGPU_ERR_INVALID, "hnsw: null array");
    uint64_t n_up = 0;
    if(n) CU(cudaMemcpy(&n_up, g->upper_off + n, 8, cudaMemcpyDefault));
    if(n_up > (uint64_t) n * 64) return fail(TSGPU_ERR_INVALID, "hnsw: upper_off[n] is not a record count");
    if(n_up && !g->links_up) return fail(TSGPU_ERR_INVALID, "hnsw: null array");
    const void* p = nullptr;
    CU(up(g->vectors, n * g->dim * 4, &p)); h.vectors = (const float*) p;
    if(g->labels) { CU(up(g->labels, n * 4, &p)); h.labels = (const uint32_t*) p; } else h.labels = nullptr;
    CU(up(g->levels, n, &p)); h.levels = (const uint8_t*) p;
    CU(up(g->links0, n * (2 * (size_t) g->M + 1) * 4, &p)); h.links0 = (const uint32_t*) p;
    CU(up(g->upper_off, (n + 1) * 8, &p)); h.upper_off = (const unsigned long long*) p;
    CU(up(g->links_up, n_up * ((size_t) g->M + 1) * 4, &p)); h.links_up = (const uint32_t*) p;
    CU(cudaDeviceSynchronize());       // the uploads went through the default stream (device-to-device ones return at once); idx->stream does not order with it
    if(n) {
        uint32_t* d_bad = nullptr;
        CU(cudaMalloc(&d_bad, 4));
        fresh.push_back(d_bad);
        CU(cudaMemsetAsync(d_bad, 0, 4, idx->stream));
        tsv::hnsw_validate_kernel<<<(unsigned) std::min<size_t>((n + 255) / 256, (size_t) idx->n_sms * 16), 256, 0, idx->stream>>>(h, n_up, d_bad);
        CU(cudaGetLastError());
        uint32_t bad = 0;
        CU(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, idx->stream));
        CU(cudaStreamSynchronize(idx->stream));
        if(bad) {
            static const char* const what[] = {"", "hnsw: a level-0 link count exceeds 2M", "hnsw: a level-0 link points outside the graph", "hnsw: levels[] and upper_off[] disagree",
                                               "hnsw: an upper-level link count exceeds M", "hnsw: an upper-level link points outside the graph", "hnsw: a node's level exceeds max_level",
                                               "hnsw: the entry point is not on the top level"};
            return fail(TSGPU_ERR_INVALID, what[bad < 8 ? bad : 1]);
        }
        cudaFree(d_bad); fresh.pop_back();
    }
    if(h.labels) {   // identity labels are the common case: detect and drop the indirection
        std::vector<uint32_t> hl(n);
        CU(cudaMemcpy(hl.data(), h.labels, n * 4, cudaMemcpyDeviceToHost));
        bool ident = true;
        for(size_t i = 0; i < n && ident; i++) ident = hl[i] == i;
        if(ident) h.labels = nullptr;
    }
    if(idx->d_deleted) {                         // a newly loaded graph starts with nothing deleted
        CU(cudaMemsetAsync(idx->d_deleted, 0, idx->deleted_words * 4, idx->stream));
        CU(cudaStreamSynchronize(idx->stream));
    }
    guard.keep = true;
    for(void* q: idx->hnsw_alloc) cudaFree(q);
    idx->hnsw_alloc = std::move(fresh);
    idx->hnsw = h;
    idx->has_hnsw = true;
    return TSGPU_OK;
}

#include "hnsw_build_host.inc"
#include "facet_host.inc"
#include "comm_host.inc"
#include "mirror_host.inc"
#include "diversity_host.inc"

tsgpu_status tsgpu_filter_create(tsgpu_index* idx, const uint32_t* ids, size_t n, int32_t* out_handle) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!out_handle || (n && !ids)) return fail(TSGPU_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(idx->mu);
    Filter f;
    const size_t words = ((size_t) idx->n_docs + 31) / 32;
    // The clear, the upload and the kernel all go on the index's stream. (They used to be a cudaMemset and a cudaMemcpy on the legacy
    // default stream followed by the kernel on idx->stream, which is NON-BLOCKING: nothing ordered them — a pageable cudaMemcpy returns
    // once the data is staged, not once it has landed — and once in a while the clear ran after the kernel and wiped bits it had set:
    // a filter missing a few documents for the lifetime of the index, seen as 7 of 1024 bench queries differing from the CPU arm.)
    CU(cudaMalloc(&f.d_bitmap, std::max<size_t>(words, 4) * 4));
    CU(cudaMemsetAsync(f.d_bitmap, 0, std::max<size_t>(words, 4) * 4, idx->stream));
    CU(cudaMalloc(&f.d_ids, std::max<size_t>(n, 4) * 4));
    if(n) {
        CU(cudaMemcpyAsync(f.d_ids, ids, n * 4, cudaMemcpyDefault, idx->stream));
        bitmap_from_ids_kernel<<<(unsigned) ((n + 255) / 256), 256, 0, idx->stream>>>(f.d_ids, n, f.d_bitmap, idx->n_docs);
        CU(cudaGetLastError());
    }
    CU(cudaStreamSynchronize(idx->stream));
    f.n = n; f.live = true;
    idx->filters.push_back(f);
    *out_handle = -((int32_t) idx->filters.size() - 1) - 2;      // encoded for tsgpu_kw_batch::q_filter
    return TSGPU_OK;
}

// a bitmap already on the device -> a persistent filter (its ascending id list is extracted from the bits: the flat vector path
// and the wildcard search read ids)
static tsgpu_status filter_from_bitmap(tsgpu_index* idx, uint32_t* d_bitmap, int32_t* out_handle, size_t* out_n) {
    cudaStream_t st = idx->stream;
    const uint32_t n_words = (uint32_t) (((size_t) idx->n_docs + 31) / 32);
    const uint32_t n_tiles = (n_words + kThreads - 1) / kThreads;
    const size_t o_off = ((size_t) n_tiles * 4 + 255) & ~size_t(255);
    const size_t o_tot = o_off + (size_t) n_tiles * 8;
    CU(idx->d_isect.reserve(o_tot + 64));
    unsigned char* base = idx->d_isect.as<unsigned char>();
    setop_count_kernel<<<n_tiles, kThreads, 0, st>>>(d_bitmap, d_bitmap, n_words, 0, reinterpret_cast<uint32_t*>(base));
    scan_tiles_kernel<<<1, 1024, 0, st>>>(reinterpret_cast<uint32_t*>(base), n_tiles, reinterpret_cast<unsigned long long*>(base + o_off),
                                          reinterpret_cast<unsigned long long*>(base + o_tot));
    unsigned long long total = 0;
    CU(cudaMemcpyAsync(&total, base + o_tot, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    Filter f;
    f.d_bitmap = d_bitmap;
    CU(cudaMalloc(&f.d_ids, std::max<size_t>((size_t) total, 4) * 4));
    setop_extract_kernel<<<n_tiles, kThreads, 0, st>>>(d_bitmap, n_words, reinterpret_cast<unsigned long long*>(base + o_off), f.d_ids, (size_t) total);
    idx->stats.launches_total += 3;
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(st));
    f.n = (size_t) total; f.live = true;
    idx->filters.push_back(f);
    *out_handle = -((int32_t) idx->filters.size() - 1) - 2;
    if(out_n) *out_n = (size_t) total;
    return TSGPU_OK;
}

tsgpu_status tsgpu_filter_numeric(tsgpu_index* idx, uint32_t sort_col, int op, int64_t v1, int64_t v2, int32_t* out_handle, size_t* out_n) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!out_handle) return fail(TSGPU_ERR_INVALID, "null argument");
    if(op < 0 || op > 6) return fail(TSGPU_ERR_INVALID, "unknown comparator");
    std::lock_guard<std::mutex> lk(idx->mu);
    if(sort_col >= idx->sort_cols.size()) return fail(TSGPU_ERR_INVALID, "column out of range");
    begin_call(idx);
    const size_t words = ((size_t) idx->n_docs + 31) / 32;
    uint32_t* bm = nullptr;
    CU(cudaMalloc(&bm, std::max<size_t>((words + 3) & ~size_t(3), 4) * 4));
    CU(cudaMemsetAsync(bm, 0, std::max<size_t>((words + 3) & ~size_t(3), 4) * 4, idx->stream));
    CU(cudaEventRecord(idx->ev[1], idx->stream));
    if(words) filter_numeric_kernel<<<(unsigned) ((words + 255) / 256), 256, 0, idx->stream>>>(idx->sort_cols[sort_col], idx->n_docs, op, v1, v2, bm);
    idx->stats.launches_total++;
    CU(cudaGetLastError());
    s = filter_from_bitmap(idx, bm, out_handle, out_n);
    if(s) { cudaFree(bm); return s; }
    CU(cudaEventRecord(idx->ev[6], idx->stream)); CU(cudaEventRecord(idx->ev[2], idx->stream));
    return end_call(idx, true, false);
}

tsgpu_status tsgpu_filter_combine(tsgpu_index* idx, int op, int32_t a, int32_t b, int32_t* out_handle, size_t* out_n) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!out_handle) return fail(TSGPU_ERR_INVALID, "null argument");
    if(op < TSGPU_SET_AND || op > TSGPU_SET_EXCLUDE) return fail(TSGPU_ERR_INVALID, "unknown set operation");
    std::lock_guard<std::mutex> lk(idx->mu);
    auto get = [&](int32_t h) -> const Filter* {
        if(h > -2) return nullptr;
        const size_t i = (size_t) (-(h + 2));
        return (i < idx->filters.size() && idx->filters[i].live) ? &idx->filters[i] : nullptr;
    };
    const Filter* fa = get(a); const Filter* fb = get(b);
    if(!fa || !fb) return fail(TSGPU_ERR_INVALID, "unknown filter handle");
    begin_call(idx);
    const size_t words = ((size_t) idx->n_docs + 31) / 32;
    uint32_t* bm = nullptr;
    CU(cudaMalloc(&bm, std::max<size_t>((words + 3) & ~size_t(3), 4) * 4));
    CU(cudaMemsetAsync(bm, 0, std::max<size_t>((words + 3) & ~size_t(3), 4) * 4, idx->stream));
    CU(cudaEventRecord(idx->ev[1], idx->stream));
    if(words) filter_combine_kernel<<<(unsigned) ((words + 255) / 256), 256, 0, idx->stream>>>(fa->d_bitmap, fb->d_bitmap, (uint32_t) words, op, bm);
    idx->stats.launches_total++;
    CU(cudaGetLastError());
    s = filter_from_bitmap(idx, bm, out_handle, out_n);
    if(s) { cudaFree(bm); return s; }
    CU(cudaEventRecord(idx->ev[6], idx->stream)); CU(cudaEventRecord(idx->ev[2], idx->stream));
    return end_call(idx, true, false);
}

/* ids of a persistent filter (ascending), e.g. to hand a device-evaluated filter to host-side code */
tsgpu_status tsgpu_filter_ids(tsgpu_index* idx, int32_t handle, uint32_t* out_ids, size_t cap, size_t* out_n) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!out_n) return fail(TSGPU_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(idx->mu);
    if(handle > -2) return fail(TSGPU_ERR_INVALID, "bad filter handle");
    const size_t h = (size_t) (-(handle + 2));
    if(h >= idx->filters.size() || !idx->filters[h].live) return fail(TSGPU_ERR_INVALID, "bad filter handle");
    *out_n = idx->filters[h].n;
    if(idx->filters[h].n > cap) return fail(TSGPU_ERR_CAPACITY, "output buffer too small");
    if(idx->filters[h].n) CU(cudaMemcpy(out_ids, idx->filters[h].d_ids, idx->filters[h].n * 4, cudaMemcpyDefault));
    return TSGPU_OK;
}

tsgpu_status tsgpu_filter_destroy(tsgpu_index* idx, int32_t handle) {
    tsgpu_status s = check_device(idx); if(s) return s;
    std::lock_guard<std::mutex> lk(idx->mu);
    if(handle > -2) return fail(TSGPU_ERR_INVALID, "bad filter handle");
    const size_t h = (size_t) (-(handle + 2));
    if(h >= idx->filters.size() || !idx->filters[h].live) return fail(TSGPU_ERR_INVALID, "bad filter handle");
    cudaFree(idx->filters[h].d_bitmap); cudaFree(idx->filters[h].d_ids);
    idx->filters[h] = Filter{};
    return TSGPU_OK;
}

static tsgpu_status isect_common(tsgpu_index* idx, uint32_t field, const uint32_t* lists, uint32_t k, const uint32_t* ids,
                                 size_t n_ids, int mode, uint32_t* out_ids, size_t cap, size_t* out_n) {
    const bool phrase = mode != 0;          // every id-set mode (phrase / exact / prefix) shares the candidate-tile path
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!lists || !out_n || k == 0) return fail(TSGPU_ERR_INVALID, "bad argument");
    if(field >= idx->fields.size()) return fail(TSGPU_ERR_INVALID, "field out of range");
    if(k > TSGPU_MAX_TOKENS) return fail(TSGPU_ERR_CAPACITY, "k exceeds TSGPU_MAX_TOKENS");
    std::lock_guard<std::mutex> lk(idx->mu);
    begin_call(idx);
    cudaStream_t st = idx->stream;
    const FieldMirror& fm = idx->fields[field];
    IsectParams P{};
    P.field = field; P.k = k; P.phrase = mode;
    uint64_t best = ~0ull;
    for(uint32_t j = 0; j < k; j++) {
        if(lists[j] >= fm.dev.n_lists) return fail(TSGPU_ERR_INVALID, "list out of range");
        P.lists[j] = lists[j];
        const uint64_t df = fm.h_list_off[lists[j] + 1] - fm.h_list_off[lists[j]];
        if(df == 0) { *out_n = 0; return end_call(idx, false, false); }
        if(df < best) { best = df; P.driver = j; }
    }
    uint32_t n_tiles;
    if(phrase) {
        if(n_ids == 0) { *out_n = 0; return end_call(idx, false, false); }
        n_tiles = (uint32_t) ((n_ids + tsdev::kBlock - 1) / tsdev::kBlock);
    } else n_tiles = (uint32_t) ((best + tsdev::kBlock - 1) / tsdev::kBlock);
    // scratch: [ids?][tile_cnt][tile_off u64][total u64][tile_ids][out]
    const size_t o_ids = 0;
    const size_t o_cnt = (o_ids + (phrase ? n_ids * 4 : 0) + 255) & ~size_t(255);
    const size_t o_off = (o_cnt + (size_t) n_tiles * 4 + 255) & ~size_t(255);
    const size_t o_tot = o_off + (size_t) n_tiles * 8;
    const size_t o_tid = (o_tot + 8 + 255) & ~size_t(255);
    const size_t o_out = o_tid + (size_t) n_tiles * tsdev::kBlock * 4;
    CU(idx->d_isect.reserve(o_out + (size_t) n_tiles * tsdev::kBlock * 4 + 256));
    unsigned char* base = idx->d_isect.as<unsigned char>();
    if(phrase) { CU(cudaMemcpyAsync(base + o_ids, ids, n_ids * 4, cudaMemcpyDefault, st)); idx->stats.h2d_bytes += n_ids * 4; }
    P.ids = phrase ? reinterpret_cast<const uint32_t*>(base + o_ids) : nullptr;
    P.n_ids = n_ids; P.n_tiles = n_tiles;
    P.tile_cnt = reinterpret_cast<uint32_t*>(base + o_cnt);
    P.tile_ids = reinterpret_cast<uint32_t*>(base + o_tid);
    CU(cudaEventRecord(idx->ev[1], st));
    isect_tiles_kernel<<<n_tiles, kThreads, 0, st>>>(idx->ixdev, P);
    scan_tiles_kernel<<<1, 1024, 0, st>>>(P.tile_cnt, n_tiles, reinterpret_cast<unsigned long long*>(base + o_off),
                                          reinterpret_cast<unsigned long long*>(base + o_tot));
    gather_tiles_kernel<<<n_tiles, kThreads, 0, st>>>(P.tile_cnt, reinterpret_cast<unsigned long long*>(base + o_off), P.tile_ids,
                                                      reinterpret_cast<uint32_t*>(base + o_out), (size_t) n_tiles * tsdev::kBlock);
    idx->stats.launches_total += 3;
    CU(cudaGetLastError());
    CU(cudaEventRecord(idx->ev[2], st));
    unsigned long long total = 0;
    CU(cudaMemcpyAsync(&total, base + o_tot, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    *out_n = (size_t) total;
    if(total > cap) return fail(TSGPU_ERR_CAPACITY, "output buffer too small");
    if(total) { CU(cudaMemcpyAsync(out_ids, base + o_out, total * 4, cudaMemcpyDefault, st)); idx->stats.d2h_bytes += total * 4 + 8; }
    return end_call(idx, true, false);
}

tsgpu_status tsgpu_contains_atleast_one(tsgpu_index* idx, uint32_t field, uint32_t list, const uint32_t* ids, size_t n, int* out) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!out || (n && !ids)) return fail(TSGPU_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(idx->mu);
    if(field >= idx->fields.size()) return fail(TSGPU_ERR_INVALID, "field id out of range");
    if(list >= idx->fields[field].dev.n_lists) return fail(TSGPU_ERR_INVALID, "list out of range");
    begin_call(idx);
    *out = 0;
    if(n == 0) return end_call(idx, false, false);
    cudaStream_t st = idx->stream;
    CU(idx->d_isect.reserve(n * 4 + 512));
    unsigned char* base = idx->d_isect.as<unsigned char>();
    CU(cudaMemsetAsync(base, 0, 256, st));
    CU(cudaMemcpyAsync(base + 256, ids, n * 4, cudaMemcpyDefault, st));
    idx->stats.h2d_bytes += n * 4;
    const unsigned grid = (unsigned) std::min<size_t>((n + 255) / 256, (size_t) idx->n_sms * 8);
    CU(cudaEventRecord(idx->ev[1], st));
    contains_any_kernel<<<grid, 256, 0, st>>>(idx->ixdev, field, list, reinterpret_cast<const uint32_t*>(base + 256), n, reinterpret_cast<int*>(base));
    idx->stats.launches_total++;
    CU(cudaGetLastError());
    CU(cudaEventRecord(idx->ev[6], st));
    CU(cudaEventRecord(idx->ev[2], st));
    CU(cudaMemcpyAsync(out, base, 4, cudaMemcpyDeviceToHost, st));
    idx->stats.d2h_bytes += 4;
    return end_call(idx, true, false);
}

tsgpu_status tsgpu_intersect(tsgpu_index* idx, uint32_t field, const uint32_t* lists, uint32_t k, uint32_t* out_ids,
                             size_t cap, size_t* out_n) {
    return isect_common(idx, field, lists, k, nullptr, 0, 0, out_ids, cap, out_n);
}

tsgpu_status tsgpu_phrase_matches(tsgpu_index* idx, uint32_t field, const uint32_t* lists, uint32_t k, const uint32_t* ids,
                                  size_t n, uint32_t* out_ids, size_t* out_n) {
    return isect_common(idx, field, lists, k, ids, n, 1, out_ids, n, out_n);
}

tsgpu_status tsgpu_exact_matches(tsgpu_index* idx, uint32_t field, const uint32_t* lists, uint32_t k, const uint32_t* ids,
                                 size_t n, uint32_t* out_ids, size_t* out_n) {
    return isect_common(idx, field, lists, k, ids, n, 2, out_ids, n, out_n);
}

tsgpu_status tsgpu_prefix_matches(tsgpu_index* idx, uint32_t field, const uint32_t* lists, uint32_t k, const uint32_t* ids,
                                  size_t n, uint32_t* out_ids, size_t* out_n) {
    return isect_common(idx, field, lists, k, ids, n, 3, out_ids, n, out_n);
}

tsgpu_status tsgpu_ids_setop(tsgpu_index* idx, int op, const uint32_t* a, size_t na, const uint32_t* b, size_t nb,
                             uint32_t* out_ids, size_t cap, size_t* out_n) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!out_n || op < TSGPU_SET_AND || op > TSGPU_SET_EXCLUDE || (na && !a) || (nb && !b)) return fail(TSGPU_ERR_INVALID, "bad argument");
    std::lock_guard<std::mutex> lk(idx->mu);
    begin_call(idx);
    *out_n = 0;
    // the reference's degenerate cases (src/array_utils.cpp:6-8, 44-58, 118-133)
    if(op == TSGPU_SET_AND && (na == 0 || nb == 0)) return end_call(idx, false, false);
    if(op == TSGPU_SET_EXCLUDE && na == 0) return end_call(idx, false, false);
    if(na == 0 && nb == 0) return end_call(idx, false, false);
    cudaStream_t st = idx->stream;
    const uint32_t n_words = (uint32_t) (((size_t) idx->n_docs + 31) / 32);
    const uint32_t n_tiles = (n_words + kThreads - 1) / kThreads;
    auto al = [](size_t v) { return (v + 255) & ~size_t(255); };
    const size_t o_a = 0, o_b = al(na * 4), o_bma = al(o_b + nb * 4), o_bmb = al(o_bma + (size_t) n_words * 4);
    const size_t o_cnt = al(o_bmb + (size_t) n_words * 4), o_off = al(o_cnt + (size_t) n_tiles * 4), o_tot = o_off + (size_t) n_tiles * 8;
    const size_t o_bad = o_tot + 8, o_out = al(o_bad + 8);
    const size_t max_out = op == TSGPU_SET_AND ? std::min(na, nb) : op == TSGPU_SET_OR ? na + nb : na;
    CU(idx->d_isect.reserve(o_out + max_out * 4 + 256));
    unsigned char* base = idx->d_isect.as<unsigned char>();
    if(na) CU(cudaMemcpyAsync(base + o_a, a, na * 4, cudaMemcpyDefault, st));
    if(nb) CU(cudaMemcpyAsync(base + o_b, b, nb * 4, cudaMemcpyDefault, st));
    idx->stats.h2d_bytes += (na + nb) * 4;
    CU(cudaMemsetAsync(base + o_bma, 0, o_cnt - o_bma, st));
    CU(cudaMemsetAsync(base + o_tot, 0, 16, st));
    uint32_t* bma = reinterpret_cast<uint32_t*>(base + o_bma);
    uint32_t* bmb = reinterpret_cast<uint32_t*>(base + o_bmb);
    uint32_t* bad = reinterpret_cast<uint32_t*>(base + o_bad);
    CU(cudaEventRecord(idx->ev[1], st));
    if(na) bitmap_from_sorted_ids_kernel<<<(unsigned) ((na + 255) / 256), 256, 0, st>>>(reinterpret_cast<const uint32_t*>(base + o_a), na, bma, idx->n_docs, bad);
    if(nb) bitmap_from_sorted_ids_kernel<<<(unsigned) ((nb + 255) / 256), 256, 0, st>>>(reinterpret_cast<const uint32_t*>(base + o_b), nb, bmb, idx->n_docs, bad);
    setop_count_kernel<<<n_tiles, kThreads, 0, st>>>(bma, bmb, n_words, op, reinterpret_cast<uint32_t*>(base + o_cnt));
    scan_tiles_kernel<<<1, 1024, 0, st>>>(reinterpret_cast<uint32_t*>(base + o_cnt), n_tiles, reinterpret_cast<unsigned long long*>(base + o_off),
                                          reinterpret_cast<unsigned long long*>(base + o_tot));
    setop_extract_kernel<<<n_tiles, kThreads, 0, st>>>(bma, n_words, reinterpret_cast<unsigned long long*>(base + o_off),
                                                       reinterpret_cast<uint32_t*>(base + o_out), max_out);
    idx->stats.launches_total += 3 + (na ? 1 : 0) + (nb ? 1 : 0);
    CU(cudaGetLastError());
    CU(cudaEventRecord(idx->ev[2], st));
    unsigned long long tot_bad[2] = {0, 0};
    CU(cudaMemcpyAsync(tot_bad, base + o_tot, 16, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if((uint32_t) tot_bad[1]) return fail(TSGPU_ERR_INVALID, "ids must be strictly ascending and below n_docs");
    *out_n = (size_t) tot_bad[0];
    if(tot_bad[0] > cap) return fail(TSGPU_ERR_CAPACITY, "output buffer too small");
    if(tot_bad[0]) { CU(cudaMemcpyAsync(out_ids, base + o_out, tot_bad[0] * 4, cudaMemcpyDefault, st)); idx->stats.d2h_bytes += tot_bad[0] * 4 + 16; }
    return end_call(idx, true, false);
}

tsgpu_status tsgpu_keyword_search_batch(tsgpu_index* idx, const tsgpu_kw_batch* b, tsgpu_kv* out_kv, uint32_t kv_stride,
                                        uint32_t* out_count, uint32_t* out_found) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!b || !out_kv || !out_count || !out_found || kv_stride == 0) return fail(TSGPU_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(idx->mu);
    begin_call(idx);
    KwPlan pl;
    { const auto t0 = std::chrono::steady_clock::now();
      s = build_kw_plan(idx, b, true, pl);
      idx->stats.ms_host_plan = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count(); }
    if(s) return s;
    if(pl.nq == 0) return end_call(idx, false, false);
    s = upload_kw_plan(idx, b, pl); if(s) return s;
    KwDeviceOut o{};
    s = run_keyword(idx, pl, kv_stride, o); if(s) return s;
    cudaStream_t st = idx->stream;
    CU(cudaMemcpyAsync(out_kv, o.kv, (size_t) pl.nq * kv_stride * sizeof(KVOut), cudaMemcpyDefault, st));
    CU(cudaMemcpyAsync(out_count, o.count, (size_t) pl.nq * 4, cudaMemcpyDefault, st));
    CU(cudaMemcpyAsync(out_found, o.found, (size_t) pl.nq * 4, cudaMemcpyDefault, st));
    idx->stats.d2h_bytes += (size_t) pl.nq * kv_stride * sizeof(KVOut) + (size_t) pl.nq * 8;
    s = end_call(idx, true, false); if(s) return s;
    return fetch_kw_stats(idx, pl);
}

static tsgpu_status wildcard_common(tsgpu_index* idx, const tsgpu_kw_batch* b, const int64_t* id_scores, tsgpu_kv* out_kv, uint32_t kv_stride,
                                    uint32_t* out_count, uint32_t* out_found);

tsgpu_status tsgpu_wildcard_search_batch(tsgpu_index* idx, const tsgpu_kw_batch* b, tsgpu_kv* out_kv, uint32_t kv_stride,
                                         uint32_t* out_count, uint32_t* out_found) {
    return wildcard_common(idx, b, nullptr, out_kv, kv_stride, out_count, out_found);
}

tsgpu_status tsgpu_scored_ids_search_batch(tsgpu_index* idx, const tsgpu_kw_batch* b, const int64_t* id_scores, tsgpu_kv* out_kv, uint32_t kv_stride,
                                           uint32_t* out_count, uint32_t* out_found) {
    if(!id_scores) return fail(TSGPU_ERR_INVALID, "null id_scores");
    if(b) for(uint32_t q = 0; q < b->n_queries; q++) if(b->q_filter[q] < 0) return fail(TSGPU_ERR_INVALID, "every query needs its id set as an inline filter");
    return wildcard_common(idx, b, id_scores, out_kv, kv_stride, out_count, out_found);
}

static tsgpu_status wildcard_common(tsgpu_index* idx, const tsgpu_kw_batch* b, const int64_t* id_scores, tsgpu_kv* out_kv, uint32_t kv_stride,
                                    uint32_t* out_count, uint32_t* out_found) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!b || !out_kv || !out_count || !out_found || kv_stride == 0) return fail(TSGPU_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(idx->mu);
    begin_call(idx);
    KwPlan pl;
    pl.id_scores = id_scores;
    { const auto t0 = std::chrono::steady_clock::now();
      s = build_kw_plan(idx, b, false, pl, true);
      idx->stats.ms_host_plan = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count(); }
    if(s) return s;
    if(pl.nq == 0) return end_call(idx, false, false);
    s = upload_kw_plan(idx, b, pl); if(s) return s;
    KwDeviceOut o{};
    s = run_keyword(idx, pl, kv_stride, o); if(s) return s;
    cudaStream_t st = idx->stream;
    CU(cudaMemcpyAsync(out_kv, o.kv, (size_t) pl.nq * kv_stride * sizeof(KVOut), cudaMemcpyDefault, st));
    CU(cudaMemcpyAsync(out_count, o.count, (size_t) pl.nq * 4, cudaMemcpyDefault, st));
    CU(cudaMemcpyAsync(out_found, o.found, (size_t) pl.nq * 4, cudaMemcpyDefault, st));
    idx->stats.d2h_bytes += (size_t) pl.nq * kv_stride * sizeof(KVOut) + (size_t) pl.nq * 8;
    return end_call(idx, true, false);
}

tsgpu_status tsgpu_knn_batch(tsgpu_index* idx, const float* queries, uint32_t nq, uint32_t k, uint32_t ef,
                             const int32_t* q_filter, uint32_t n_filters, const uint64_t* filter_off,
                             const uint32_t* filter_ids, float* out_dist, uint32_t* out_labels, uint32_t* out_n) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!queries || !out_dist || !out_labels || !out_n) return fail(TSGPU_ERR_INVALID, "null argument");
    if(!idx->has_hnsw) return fail(TSGPU_ERR_INVALID, "no vector index loaded");
    std::lock_guard<std::mutex> lk(idx->mu);
    begin_call(idx);
    if(nq == 0) return end_call(idx, false, false);
    cudaStream_t st = idx->stream;
    const uint32_t dim = idx->hnsw.dim;
    const size_t words = ((size_t) idx->n_docs + 31) / 32;
    // queries + inline filter ids -> device
    const size_t q_bytes = (size_t) nq * dim * 4;
    const size_t n_fids = (q_filter && n_filters) ? (size_t) filter_off[n_filters] : 0;
    const size_t o_f = (q_bytes + 255) & ~size_t(255);
    CU(idx->d_small.reserve(o_f + n_fids * 4 + 256));
    unsigned char* base = idx->d_small.as<unsigned char>();
    CU(cudaMemcpyAsync(base, queries, q_bytes, cudaMemcpyDefault, st));
    idx->stats.h2d_bytes += q_bytes;
    std::vector<const uint32_t*> q_bitmap;
    std::vector<uint8_t> skip;
    if(q_filter) {
        q_bitmap.assign(nq, nullptr);
        skip.assign(nq, 0);
        if(n_fids) { CU(cudaMemcpyAsync(base + o_f, filter_ids, n_fids * 4, cudaMemcpyDefault, st)); idx->stats.h2d_bytes += n_fids * 4; }
        if(n_filters) {
            CU(idx->d_bitmaps.reserve((size_t) n_filters * words * 4));
            CU(cudaMemsetAsync(idx->d_bitmaps.p, 0, (size_t) n_filters * words * 4, st));
        }
        uint32_t* bm = idx->d_bitmaps.as<uint32_t>();
        for(uint32_t f = 0; f < n_filters; f++) {
            const size_t n = (size_t) (filter_off[f + 1] - filter_off[f]);
            if(n) bitmap_from_ids_kernel<<<(unsigned) ((n + 255) / 256), 256, 0, st>>>(reinterpret_cast<const uint32_t*>(base + o_f) + filter_off[f], n, bm + (size_t) f * words, idx->n_docs);
        }
        CU(cudaGetLastError());
        for(uint32_t q = 0; q < nq; q++) {
            const int32_t fs = q_filter[q];
            if(fs >= 0) {
                if((uint32_t) fs >= n_filters) return fail(TSGPU_ERR_INVALID, "filter slot out of range");
                q_bitmap[q] = bm + (size_t) fs * words;
            } else if(fs <= -2) {
                const size_t h = (size_t) (-(fs + 2));
                if(h >= idx->filters.size() || !idx->filters[h].live) return fail(TSGPU_ERR_INVALID, "unknown filter handle");
                q_bitmap[q] = idx->filters[h].d_bitmap;
            }
        }
    }
    KnnDeviceOut o{};
    idx->vs = idx->stream; idx->knn_blocks_per_sm = 7;
    std::vector<float> cost;
    if(q_filter) {
        cost.assign(nq, 1.0f);
        for(uint32_t q = 0; q < nq; q++) {
            const int32_t fs = q_filter[q];
            size_t n = 0;
            if(fs >= 0) n = (size_t) (filter_off[fs + 1] - filter_off[fs]);
            else if(fs <= -2) n = idx->filters[(size_t) (-(fs + 2))].n;
            if(fs != -1 && n) cost[q] = std::min(1e6f, (float) idx->n_docs / (float) n);
        }
    }
    s = run_knn(idx, reinterpret_cast<const float*>(base), nq, k, ef, q_bitmap, {}, {}, {}, cost, o); if(s) return s;
    CU(cudaMemcpyAsync(out_dist, o.dist, (size_t) nq * k * 4, cudaMemcpyDefault, st));
    CU(cudaMemcpyAsync(out_labels, o.labels, (size_t) nq * k * 4, cudaMemcpyDefault, st));
    CU(cudaMemcpyAsync(out_n, o.n, (size_t) nq * 4, cudaMemcpyDefault, st));
    idx->stats.d2h_bytes += (size_t) nq * k * 8 + (size_t) nq * 4;
    s = end_call(idx, false, true); if(s) return s;
    return finish_knn(idx);
}

tsgpu_status tsgpu_flat_distances(tsgpu_index* idx, const float* query, const uint32_t* ids, size_t n, float* out_dist) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!query || (n && (!ids || !out_dist))) return fail(TSGPU_ERR_INVALID, "null argument");
    if(!idx->has_hnsw) return fail(TSGPU_ERR_INVALID, "no vector index loaded");
    std::lock_guard<std::mutex> lk(idx->mu);
    begin_call(idx);
    if(n == 0) return end_call(idx, false, false);
    cudaStream_t st = idx->stream;
    const uint32_t dim = idx->hnsw.dim;
    const size_t o_off = ((size_t) dim * 4 + 255) & ~size_t(255);
    const size_t o_ids = o_off + 256;
    const size_t o_d = (o_ids + n * 4 + 255) & ~size_t(255);
    CU(idx->d_small.reserve(o_d + n * 4 + 256));
    unsigned char* base = idx->d_small.as<unsigned char>();
    unsigned long long off[2] = {0, (unsigned long long) n};
    CU(cudaMemcpyAsync(base, query, (size_t) dim * 4, cudaMemcpyDefault, st));
    CU(cudaMemcpyAsync(base + o_off, off, 16, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(base + o_ids, ids, n * 4, cudaMemcpyDefault, st));
    CU(cudaStreamSynchronize(st));
    idx->stats.h2d_bytes += (size_t) dim * 4 + n * 4;
    tsv::FlatParams FP{};
    FP.queries = reinterpret_cast<const float*>(base); FP.ids = reinterpret_cast<const uint32_t*>(base + o_ids);
    FP.q_off = reinterpret_cast<const unsigned long long*>(base + o_off); FP.nq = 1;
    FP.out_dist = reinterpret_cast<float*>(base + o_d);
    idx->vs = st;
    CU(cudaEventRecord(idx->ev[3], st));
    s = run_flat(idx, FP, n); if(s) return s;
    CU(cudaEventRecord(idx->ev[4], st));
    CU(cudaMemcpyAsync(out_dist, base + o_d, n * 4, cudaMemcpyDefault, st));
    idx->stats.d2h_bytes += n * 4;
    return end_call(idx, false, true);
}

tsgpu_status tsgpu_flat_distances_batch(tsgpu_index* idx, const float* queries, uint32_t nq, const uint32_t* ids, size_t n, float* out_dist) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(nq && n && (!queries || !ids || !out_dist)) return fail(TSGPU_ERR_INVALID, "null argument");
    if(!idx->has_hnsw) return fail(TSGPU_ERR_INVALID, "no vector index loaded");
    if(n > 0xFFFFFFFFull) return fail(TSGPU_ERR_INVALID, "candidate set too large");
    std::lock_guard<std::mutex> lk(idx->mu);
    begin_call(idx);
    if(n == 0 || nq == 0) return end_call(idx, false, false);
    cudaStream_t st = idx->stream;
    const uint32_t dim = idx->hnsw.dim;
    const bool tc = flat_tc_min_group() > 0 && tsgpu_flat_tc_supported_(dim);
    // scratch: queries | q_off (nq+1 u64) | ids | (scalar path: ids repeated per query)
    const size_t q_bytes = (size_t) nq * dim * 4;
    const size_t o_off = (q_bytes + 255) & ~size_t(255);
    const size_t o_ids = (o_off + (size_t) (nq + 1) * 8 + 255) & ~size_t(255);
    const size_t n_rep = tc ? n : n * nq;
    const size_t o_d = (o_ids + n_rep * 4 + 255) & ~size_t(255);
    CU(idx->d_small.reserve(o_d + (size_t) nq * n * 4 + 256));
    unsigned char* base = idx->d_small.as<unsigned char>();
    std::vector<unsigned long long>& off = idx->tmp_foff;
    off.resize((size_t) nq + 1);
    for(uint32_t q = 0; q <= nq; q++) off[q] = (unsigned long long) q * n;
    CU(cudaMemcpyAsync(base, queries, q_bytes, cudaMemcpyDefault, st));
    CU(cudaMemcpyAsync(base + o_off, off.data(), (size_t) (nq + 1) * 8, cudaMemcpyHostToDevice, st));
    for(size_t r = 0; r < (tc ? 1 : nq); r++) CU(cudaMemcpyAsync(base + o_ids + r * n * 4, ids, n * 4, cudaMemcpyDefault, st));
    idx->stats.h2d_bytes += q_bytes + n * 4;
    idx->vs = st;
    CU(cudaEventRecord(idx->ev[3], st));
    if(tc) {
        CU(idx->d_flat_tc.reserve(tsgpu_flat_tc_image_bytes_(nq, dim, nullptr, nullptr) + 2048));
        unsigned char* img = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(idx->d_flat_tc.p) + 1023) & ~uintptr_t(1023));
        int launches = 0;
        CU(tsgpu_flat_tc_run_(idx->hnsw.vectors, idx->hnsw.n_nodes, dim, reinterpret_cast<const float*>(base), nullptr, nq,
                              reinterpret_cast<const uint32_t*>(base + o_ids), (uint32_t) n, reinterpret_cast<const unsigned long long*>(base + o_off),
                              reinterpret_cast<float*>(base + o_d), img, idx->n_sms, st, &launches));
        idx->stats.launches_total += launches;
        idx->stats.flat_tc_queries += nq;
    } else {
        tsv::FlatParams FP{};
        FP.queries = reinterpret_cast<const float*>(base); FP.ids = reinterpret_cast<const uint32_t*>(base + o_ids);
        FP.q_off = reinterpret_cast<const unsigned long long*>(base + o_off); FP.nq = nq;
        FP.out_dist = reinterpret_cast<float*>(base + o_d);
        s = run_flat(idx, FP, (unsigned long long) nq * n); if(s) return s;
    }
    CU(cudaEventRecord(idx->ev[4], st));
    CU(cudaMemcpyAsync(out_dist, base + o_d, (size_t) nq * n * 4, cudaMemcpyDefault, st));
    idx->stats.d2h_bytes += (size_t) nq * n * 4;
    return end_call(idx, false, true);
}

// keyword results handed in by the caller instead of computed here (tsgpu_hybrid_fuse_batch)
struct GivenKw { const tsgpu_kv* kv; uint32_t stride; const uint32_t* count; const uint32_t* found; const uint32_t* searched; };

static tsgpu_status vec_or_hybrid(tsgpu_index* idx, const tsgpu_kw_batch* b, const float* qvecs, const tsgpu_vec_params* vp,
                                  tsgpu_kv* out_kv, uint32_t kv_stride, uint32_t* out_count, uint32_t* out_found, bool hybrid,
                                  const GivenKw* given = nullptr) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!b || !qvecs || !vp || !out_kv || !out_count || !out_found || kv_stride == 0) return fail(TSGPU_ERR_INVALID, "null argument");
    if(!idx->has_hnsw) return fail(TSGPU_ERR_INVALID, "no vector index loaded");
    const bool vdeep = (vp->flags & TSGPU_VEC_DEEP_TOPSTER) != 0;
    if(!vdeep)
        for(uint32_t q = 0; q < b->n_queries; q++)     // the ordinary fusion kernel holds its Topster in shared memory
            if(b->q_flags[q] & TSGPU_QFLAG_DEEP_TOPSTER) return fail(TSGPU_ERR_INVALID, "TSGPU_QFLAG_DEEP_TOPSTER is not supported by vector and hybrid searches");
    std::lock_guard<std::mutex> lk(idx->mu);
    begin_call(idx);
    KwPlan pl;
    { const auto t0 = std::chrono::steady_clock::now();
      s = build_kw_plan(idx, b, hybrid, pl);
      idx->stats.ms_host_plan = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count(); }
    if(s) return s;
    if(pl.nq == 0) return end_call(idx, false, false);
    // k as in src/index.cpp:3646 (wildcard) and :4061-4063 (hybrid)
    const uint32_t k = hybrid ? (vp->k == 0 ? std::max<uint32_t>(vp->fetch_size, 100) : vp->k)
                              : (vp->k == 0 ? std::max<uint32_t>(vp->k, vp->fetch_size) : vp->k);
    if(k == 0) return fail(TSGPU_ERR_INVALID, "k resolves to 0 (set k or fetch_size)");
    if(hybrid && k > 1024 && !vdeep) return fail(TSGPU_ERR_CAPACITY, "hybrid k must be <= 1024");
    // deep queries (TSGPU_VEC_DEEP_TOPSTER): planned and their device memory reserved before anything runs
    DeepFuse df;
    if(vdeep) { s = deep_fuse_plan(idx, b, pl, vp, k, hybrid, df); if(s) return s; }
    s = upload_kw_plan(idx, b, pl); if(s) return s;
    s = deep_fuse_upload(idx, pl, b, vp, k, df); if(s) return s;
    cudaStream_t st = idx->stream;
    const uint32_t nq = pl.nq;
    KwDeviceOut kwo{};
    const uint32_t kw_stride = std::max(std::max(kv_stride, pl.KMAX), df.kmax);     // a deep query's keyword Topster is whole
    // The vector stage and the keyword kernels are independent until the fusion: issue the vector stage on its own
    // stream (after the filter bitmaps built by upload_kw_plan) with a reduced residency so keyword CTAs co-run, and
    // let the long latency-bound tail of the graph walk hide under the keyword kernels.
    VecStage vs;
    if(hybrid) {
        CU(cudaEventRecord(idx->evA, st));
        CU(cudaStreamWaitEvent(idx->stream2, idx->evA, 0));
        const char* ov = getenv("TSGPU_KNN_OVERLAP_BLOCKS");      // 0 = no overlap (same stream, full residency)
        const int ovb = ov ? atoi(ov) : 5;
        if(ovb > 0) { idx->vs = idx->stream2; idx->knn_blocks_per_sm = (unsigned) std::min(ovb, 7); }
        else { idx->vs = st; idx->knn_blocks_per_sm = 7; }
    } else { idx->vs = st; idx->knn_blocks_per_sm = 7; }
    // Launch order decides who owns the SMs: the keyword kernels go first and fill every SM (8 CTAs each); the persistent
    // graph-walk CTAs then take the slots that free up (kw_search's tail, the small merge / final grids) and finish alone.
    // The other order lets the latency-bound walk hold half the register file while it uses a fifth of the memory system.
    static const bool kw_first = !(getenv("TSGPU_KW_FIRST") && atoi(getenv("TSGPU_KW_FIRST")) == 0);
    if(given) {
        // the keyword stage already ran (several rounds of it, on the host's schedule): its final Topster content comes in
        const size_t kvb = (size_t) nq * given->stride * sizeof(KVOut);
        CU(idx->d_kw_out.reserve(kvb + (size_t) nq * 12 + 64));
        kwo.kv = idx->d_kw_out.as<KVOut>();
        kwo.count = reinterpret_cast<uint32_t*>(idx->d_kw_out.as<unsigned char>() + ((kvb + 15) & ~size_t(15)));
        kwo.found = kwo.count + nq; kwo.searched = kwo.found + nq; kwo.stride = given->stride;
        CU(cudaMemcpyAsync(kwo.kv, given->kv, kvb, cudaMemcpyDefault, st));
        CU(cudaMemcpyAsync(kwo.count, given->count, (size_t) nq * 4, cudaMemcpyDefault, st));
        CU(cudaMemcpyAsync(kwo.found, given->found, (size_t) nq * 4, cudaMemcpyDefault, st));
        CU(cudaMemcpyAsync(kwo.searched, given->searched, (size_t) nq * 4, cudaMemcpyDefault, st));
        idx->stats.h2d_bytes += kvb + (size_t) nq * 12;
        CU(cudaEventRecord(idx->ev[1], st)); CU(cudaEventRecord(idx->ev[6], st)); CU(cudaEventRecord(idx->ev[2], st));
    }
    else if(hybrid && kw_first) { s = run_keyword(idx, pl, kw_stride, kwo); if(s) return s; }
    s = run_vector_stage(idx, b, pl, qvecs, vp, k, vs); if(s) return s;
    if(hybrid) {
        CU(cudaEventRecord(idx->evB, idx->stream2));
        if(!kw_first && !given) { s = run_keyword(idx, pl, kw_stride, kwo); if(s) return s; }
        CU(cudaStreamWaitEvent(st, idx->evB, 0));
    }
    // final assembly
    const size_t kv_bytes = (size_t) nq * kv_stride * sizeof(KVOut);
    CU(idx->d_out.reserve(kv_bytes + (size_t) nq * 8 + 64));
    KVOut* d_kv = idx->d_out.as<KVOut>();
    uint32_t* d_cnt = reinterpret_cast<uint32_t*>(idx->d_out.as<unsigned char>() + ((kv_bytes + 15) & ~size_t(15)));
    uint32_t* d_found = d_cnt + nq;
    tsf::VecParams dvp{k, vp->distance_threshold, vp->alpha, idx->hnsw.metric};
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0, st);
    if(!hybrid) {
        tsf::VecAssembleParams P{};
        P.qd = pl.d_qd;
        if(!df.q.empty()) {
            s = deep_fuse_counts(idx, pl, nullptr, vs.knn.n, df); if(s) return s;
            P.qd = df.d_qd_ord;
        }
        P.res_dist = vs.knn.dist; P.res_ids = vs.knn.labels; P.res_n = vs.knn.n; P.res_stride = vs.knn.stride;
        P.flat_dist = vs.flat_dist; P.flat_ids = vs.flat_ids;
        P.res_off = vs.flat_off; P.q_is_flat = vs.any_flat ? vs.d_is_flat : nullptr;
        P.vp = dvp;
        P.out_kv = d_kv; P.out_count = d_cnt; P.out_found = d_found; P.kv_stride = kv_stride;
        if(!df.q.empty()) P.res_n = df.d_res_n_ord;
        P.KP = std::max<uint32_t>(pl.KP, 256);          // 256 threads append per round
        const size_t smem = (size_t) 2 * P.KP * 32 + 16;
        CU(cudaFuncSetAttribute(tsf::vec_assemble_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) std::max<size_t>(smem, 48 * 1024)));
        tsf::vec_assemble_kernel<<<nq, kFinalThreads, smem, st>>>(P);
        idx->stats.launches_total++;
        CU(cudaGetLastError());
        if(!df.q.empty()) { s = run_vec_deep(idx, pl, vs, dvp, df, d_kv, kv_stride, d_cnt, d_found); if(s) return s; }
    } else {
        tsf::HybridParams P{};
        P.ix = idx->ixdev; P.qd = pl.d_qd; P.cd = pl.d_cd; P.F = pl.F;
        for(uint32_t f = 0; f < (uint32_t) kMaxFieldSlots; f++) P.field_ids[f] = pl.field_ids[f];
        P.kw_kv = kwo.kv; P.kw_count = kwo.count; P.kw_found = kwo.found; P.kw_searched = kwo.searched; P.kw_stride = kwo.stride;
        P.res_dist = vs.knn.dist; P.res_ids = vs.knn.labels; P.res_n = vs.knn.n; P.res_stride = vs.knn.stride;
        P.flat_dist = vs.flat_dist; P.flat_ids = vs.flat_ids;
        P.res_off = vs.flat_off; P.q_is_flat = vs.any_flat ? vs.d_is_flat : nullptr;
        P.vp = dvp;
        P.out_kv = d_kv; P.out_count = d_cnt; P.out_found = d_found; P.kv_stride = kv_stride;
        P.KMAX = pl.KMAX; P.VMAX = k;
        P.queries = vs.d_queries; P.vectors = idx->hnsw.vectors; P.dim = idx->hnsw.dim; P.n_nodes = idx->hnsw.n_nodes;
        const uint32_t KP2 = pow2_ceil(pl.KMAX), VP2 = pow2_ceil(k);
        const size_t smem = (size_t) pl.KMAX * sizeof(KVOut) + (size_t) (KP2 + 2) * 2 + (size_t) VP2 * (12 + 24 + 2) + 48;
        CU(cudaFuncSetAttribute(tsf::hybrid_fuse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) std::max<size_t>(smem, 48 * 1024)));
        const tsf::HybridParams whole = P;
        if(!df.q.empty()) {
            s = deep_fuse_counts(idx, pl, kwo.count, vs.knn.n, df); if(s) return s;
            P.qd = df.d_qd_ord; P.kw_count = df.d_kw_count_ord; P.res_n = df.d_res_n_ord;
        }
        tsf::hybrid_fuse_kernel<<<nq, kThreads, smem, st>>>(P);
        idx->stats.launches_total++;
        CU(cudaGetLastError());
        if(!df.q.empty()) { s = run_hybrid_deep(idx, whole, df); if(s) return s; }
    }
    cudaEventRecord(e1, st);
    CU(cudaMemcpyAsync(out_kv, d_kv, kv_bytes, cudaMemcpyDefault, st));
    CU(cudaMemcpyAsync(out_count, d_cnt, (size_t) nq * 4, cudaMemcpyDefault, st));
    CU(cudaMemcpyAsync(out_found, d_found, (size_t) nq * 4, cudaMemcpyDefault, st));
    idx->stats.d2h_bytes += kv_bytes + (size_t) nq * 8;
    s = end_call(idx, hybrid, true);
    if(!s) s = finish_knn(idx);
    deep_fuse_finish(idx, hybrid, df);
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    idx->stats.ms_fuse = ms; idx->stats.ms_kernels += ms;
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    if(s) return s;
    if(hybrid && !given) return fetch_kw_stats(idx, pl);
    return TSGPU_OK;
}

tsgpu_status tsgpu_vector_search_batch(tsgpu_index* idx, const tsgpu_kw_batch* b, const float* qvecs, const tsgpu_vec_params* vp,
                                       tsgpu_kv* out_kv, uint32_t kv_stride, uint32_t* out_count, uint32_t* out_found) {
    return vec_or_hybrid(idx, b, qvecs, vp, out_kv, kv_stride, out_count, out_found, false);
}

tsgpu_status tsgpu_hybrid_search_batch(tsgpu_index* idx, const tsgpu_kw_batch* b, const float* qvecs, const tsgpu_vec_params* vp,
                                       tsgpu_kv* out_kv, uint32_t kv_stride, uint32_t* out_count, uint32_t* out_found) {
    return vec_or_hybrid(idx, b, qvecs, vp, out_kv, kv_stride, out_count, out_found, true);
}

/* instrumentation: (expansions, distance evaluations) of every graph walk of the last call that ran the HNSW kernel */
tsgpu_status tsgpu_debug_knn_work(tsgpu_index* idx, uint32_t* out, uint32_t cap_queries, uint32_t* out_n) {
    tsgpu_status s = check_device(idx); if(s) return s;
    if(!out || !out_n) return fail(TSGPU_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(idx->mu);
    const uint32_t n = std::min(cap_queries, idx->knn_work_dev ? idx->knn_work_n : 0u);
    if(n) CU(cudaMemcpy(out, idx->knn_work_dev, (size_t) n * 8, cudaMemcpyDeviceToHost));
    *out_n = n;
    return TSGPU_OK;
}

tsgpu_status tsgpu_hybrid_fuse_batch(tsgpu_index* idx, const tsgpu_kw_batch* b, const tsgpu_kv* kw_kv, uint32_t kw_stride, const uint32_t* kw_count,
                                     const uint32_t* kw_found, const uint32_t* kw_searched, const float* qvecs, const tsgpu_vec_params* vp,
                                     tsgpu_kv* out_kv, uint32_t kv_stride, uint32_t* out_count, uint32_t* out_found) {
    if(!kw_kv || !kw_count || !kw_found || !kw_searched || kw_stride == 0) return fail(TSGPU_ERR_INVALID, "null argument");
    if(b) for(uint32_t q = 0; q < b->n_queries; q++) if(kw_count[q] > kw_stride || kw_count[q] > b->q_topk[q]) return fail(TSGPU_ERR_INVALID, "kw_count exceeds kw_stride / topk");
    const GivenKw g{kw_kv, kw_stride, kw_count, kw_found, kw_searched};
    return vec_or_hybrid(idx, b, qvecs, vp, out_kv, kv_stride, out_count, out_found, true, &g);
}

tsgpu_status tsgpu_get_stats(tsgpu_index* idx, tsgpu_stats* out) {
    if(!idx || !out) return fail(TSGPU_ERR_INVALID, "null argument");
    *out = idx->stats;
    return TSGPU_OK;
}

}  // extern "C"
