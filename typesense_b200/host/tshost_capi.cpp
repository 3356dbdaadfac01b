// C entry points over the C++ host layer (tsgpu_host.hpp) so that a non-C++ harness — bench.py, the Python tests — can drive
// the same code a server-side binding links: Index mirrors from flat arrays, persistent filters, and multi_search_batched
// (typo / prefix / drop-token control flow of Index::search per request, device rounds shared by the whole request list).
// Built twice: against libtsgpu.so (the product path bench.py's end-to-end leg times) and, for the CPU arm and the CPU test
// runs, against tests/cpp/tsgpu_oracle_double.cpp (the oracle behind the same C-ABI) — same host code either way.
#include <cstring>
#include <string>
#include <vector>

#include "tsgpu_host.hpp"

// This wrapper is also linked against the oracle-backed test double of the C-ABI (the CPU arm), which has no mirror maintenance
// calls: weak references let that build load, and its entry points report the missing call instead.
#pragma weak tsgpu_index_compact_field
#pragma weak tsgpu_index_reserve_docs

namespace {
thread_local std::string g_host_err;
struct HostCtx { tsgpu::Index* ix; };
tsgpu::Index& IX(void* h) { return *static_cast<HostCtx*>(h)->ix; }
}

extern "C" {

const char* tshost_last_error(void) { return g_host_err.c_str(); }

void* tshost_create(uint32_t n_docs, int device) {
    auto* ix = new tsgpu::Index(n_docs, device);
    if(!ix->ok()) { g_host_err = ix->error(); delete ix; return nullptr; }
    return new HostCtx{ix};
}
void tshost_destroy(void* h) { if(h) { delete static_cast<HostCtx*>(h)->ix; delete static_cast<HostCtx*>(h); } }
void* tshost_tsgpu_handle(void* h) { return IX(h).handle(); }

// tokens: n_tokens strings, tokens_blob[tok_off[i] .. tok_off[i+1])
int tshost_add_field_flat(void* h, const char* name, uint32_t n_tokens, const char* tokens_blob, const uint32_t* tok_off, const uint64_t* list_off,
                          const uint32_t* ids, const uint64_t* pos_off, const uint32_t* positions, int is_array) {
    std::vector<std::string> toks(n_tokens);
    for(uint32_t i = 0; i < n_tokens; i++) toks[i].assign(tokens_blob + tok_off[i], tokens_blob + tok_off[i + 1]);
    std::vector<uint64_t> lo(list_off, list_off + n_tokens + 1);
    std::vector<uint32_t> idv(ids, ids + lo.back());
    auto op = IX(h).add_field_flat(name, std::move(toks), std::move(lo), std::move(idv), pos_off, positions, is_array != 0);
    if(!op.ok()) { g_host_err = op.error(); return -1; }
    return (int) op.get();
}
int tshost_add_sort_column(void* h, const char* name, const int64_t* dense_values) {
    auto op = IX(h).add_sort_field_dense(name, dense_values);
    if(!op.ok()) { g_host_err = op.error(); return -1; }
    return (int) op.get();
}
// f-4 maintenance: the lists a field's tokens no longer name are freed (Index::compact_field); the seq_id capacity grows
// (Index::reserve_docs). 0 on success.
int tshost_compact_field(void* h, const char* name) {
    if(!tsgpu_index_compact_field) { g_host_err = "the linked tsgpu library has no tsgpu_index_compact_field"; return -1; }
    auto op = IX(h).compact_field(name);
    if(!op.ok()) { g_host_err = op.error(); return -1; }
    return 0;
}
int tshost_reserve_docs(void* h, uint32_t n_docs) {
    if(!tsgpu_index_reserve_docs) { g_host_err = "the linked tsgpu library has no tsgpu_index_reserve_docs"; return -1; }
    auto op = IX(h).reserve_docs(n_docs);
    if(!op.ok()) { g_host_err = op.error(); return -1; }
    return 0;
}
int32_t tshost_add_filter(void* h, const uint32_t* ids, size_t n) {
    auto op = IX(h).add_filter(std::vector<uint32_t>(ids, ids + n));
    if(!op.ok()) { g_host_err = op.error(); return 0; }
    return op.get();
}

typedef struct {
    uint32_t num_typos, prefix, max_candidates, typo_tokens_threshold, drop_tokens_threshold, topster_size, device_art_walk, n_threads;
    uint32_t vec_k, vec_ef, vec_flat_search_cutoff, vec_fetch_size;
    float vec_alpha, vec_distance_threshold;
    uint32_t vec_flags;          /* tsgpu_vec_params::flags of the vector requests (TSGPU_VEC_DEEP_TOPSTER: Topsters above 1024) */
} tshost_options;
typedef struct { uint64_t passes, kw_batches, kw_queries, walk_batches, walks, host_walk_fallbacks, fuse_queries; double ms_host_passes, ms_kw_calls, ms_walk_calls, ms_fuse_calls; } tshost_stats;

// nq requests over one searched field; request i's tokens are tokens[q_off[i] .. q_off[i+1]), token t = blob[tok_off[t] .. tok_off[t+1]).
// q_filter[i]: a handle from tshost_add_filter or -1. qvecs: nq * dim floats (hybrid) or NULL (keyword only).
// sort: _text_match desc, `sort_field` desc. Results: out_kv[i*stride ..], out_count[i], out_found[i].
int tshost_multi_search(void* h, const char* field, const char* sort_field, uint32_t nq, const char* blob, const uint32_t* tok_off, const uint32_t* q_off,
                        const int32_t* q_filter, const float* qvecs, uint32_t dim, const tshost_options* o, tsgpu_kv* out_kv, uint32_t stride,
                        uint32_t* out_count, uint32_t* out_found, tshost_stats* out_stats) {
    using Ix = tsgpu::Index;
    std::vector<Ix::batched_request> reqs(nq);
    for(uint32_t i = 0; i < nq; i++) {
        auto& r = reqs[i].r;
        for(uint32_t t = q_off[i]; t < q_off[i + 1]; t++) r.tokens.emplace_back(blob + tok_off[t], blob + tok_off[t + 1]);
        r.the_fields = {field};
        tsgpu::sort_by s0; s0.type = tsgpu::sort_by::text_match; s0.desc = true;
        tsgpu::sort_by s1; s1.type = tsgpu::sort_by::numeric; s1.name = sort_field; s1.desc = true;
        r.sort_fields = {s0, s1};
        r.drop_tokens_threshold = o->drop_tokens_threshold;
        r.topster_size = o->topster_size;
        r.opts.num_typos = o->num_typos; r.opts.prefix = o->prefix != 0; r.opts.max_candidates = o->max_candidates;
        r.opts.typo_tokens_threshold = o->typo_tokens_threshold; r.opts.device_art_walk = o->device_art_walk != 0;
        reqs[i].filter_handle = q_filter ? q_filter[i] : -1;
        reqs[i].hits = stride;
        if(qvecs) {
            reqs[i].query_vector = qvecs + (size_t) i * dim;
            reqs[i].vp = tsgpu_vec_params{o->vec_k, o->vec_ef, o->vec_flat_search_cutoff, o->vec_distance_threshold, o->vec_alpha, o->vec_fetch_size, o->vec_flags};
        }
    }
    Ix::batched_stats bs;
    auto resp = IX(h).multi_search_batched(reqs, o->n_threads, &bs);
    int rc = 0;
    for(uint32_t i = 0; i < nq; i++) {
        if(!resp[i].status.ok()) { g_host_err = resp[i].status.error(); rc = -1; out_count[i] = 0; out_found[i] = 0; continue; }
        const uint32_t n = (uint32_t) std::min<size_t>(resp[i].raw_result_kvs.size(), stride);
        std::memcpy(out_kv + (size_t) i * stride, resp[i].raw_result_kvs.data(), (size_t) n * sizeof(tsgpu_kv));
        out_count[i] = n; out_found[i] = (uint32_t) resp[i].found;
    }
    if(out_stats) *out_stats = tshost_stats{bs.passes, bs.kw_batches, bs.kw_queries, bs.walk_batches, bs.walks, bs.host_walk_fallbacks, bs.fuse_queries, bs.ms_host_passes, bs.ms_kw_calls, bs.ms_walk_calls, bs.ms_fuse_calls};
    return rc;
}

}  // extern "C"
