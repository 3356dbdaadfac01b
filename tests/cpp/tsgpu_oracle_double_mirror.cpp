// TEST INFRASTRUCTURE — the oracle-backed test double of the C-ABI (tsgpu_oracle_double.cpp, included whole) plus the mirror
// maintenance calls: tsgpu_index_compact_field, tsgpu_index_reserve_docs, tsgpu_index_field_info, tsgpu_debug_field_array. Built
// as one library (or linked into one program) so that the tests of those calls run their Python / C++ side on a machine without a
// GPU. The calls check their arguments as the library does; a field's arrays are what the library's own loader (postings_pack.h)
// builds from the lists the double holds. Never part of the product.
//
// Two facts the base double does not keep are recorded by wrapping its loaders: the dense threshold a field's lists were classified
// under (the library keeps the divisor per field and reclassifies only on compaction), and which index a facet belongs to.
#define tsgpu_index_load_field tsgpu_index_load_field_base_
#define tsgpu_index_load_facet tsgpu_index_load_facet_base_
#include "tsgpu_oracle_double.cpp"
#undef tsgpu_index_load_field
#undef tsgpu_index_load_facet

#pragma GCC diagnostic push
#pragma GCC diagnostic ignored "-Wunknown-pragmas"
#include "../../typesense_b200/csrc/postings_pack.h"
#pragma GCC diagnostic pop

namespace {
struct FieldExtra { uint32_t dense_div = 64; uint64_t min_df = 64; };
std::map<const FieldCopy*, FieldExtra> g_field_extra;           // keyed by the double's field copy
std::map<size_t, const tsgpu_index*> g_facet_owner;             // facet id -> index

FieldExtra extra_for(uint32_t n_docs) {
    FieldExtra e;
    e.dense_div = (uint32_t) std::max(1, getenv("TSGPU_DENSE_DIV") ? atoi(getenv("TSGPU_DENSE_DIV")) : 64);
    e.min_df = tspack::dense_min_df(n_docs, e.dense_div);
    return e;
}

void pack_copy(const FieldCopy& c, uint32_t n_docs, tspack::PackedField& pk, uint32_t& flags) {
    const uint32_t L = c.view.n_lists;
    const uint64_t n_post = c.list_off[L], n_pos = c.pos_off[n_post];
    tspack::pack_field(L, c.list_off.data(), c.ids.data(), pk);
    tspack::pack_dense(L, c.list_off.data(), c.ids.data(), n_docs, g_field_extra[&c].min_df, pk);
    flags = c.view.is_array ? tsdev::kFieldIsArray : 0;
    if(!c.view.is_array && tspack::plain_wellformed(c.pos_off.data(), c.positions.data(), n_post)) {
        flags |= tsdev::kFieldPlainOk;
        if(tspack::positions_fit_u16(c.positions.data(), n_pos)) flags |= tsdev::kFieldPos16;
    }
}

// bytes of the ten arrays as the library's loader allocates them, and their logical lengths
struct Arrays { const void* src[10]; size_t logical[10]; size_t alloc[10]; };
Arrays arrays_of(const FieldCopy& c, const tspack::PackedField& pk) {
    const uint32_t L = c.view.n_lists;
    const uint64_t n_post = c.list_off[L], n_pos = c.pos_off[n_post];
    Arrays a{{c.list_off.data(), pk.list_blk_off.data(), pk.blk_first.data(), pk.blk_info.data(), pk.packed.data(), c.pos_off.data(),
              c.positions.data(), pk.list_dense.data(), pk.dense_bits.data(), pk.dense_rank.data()},
             {((size_t) L + 1) * 8, ((size_t) L + 1) * 4, pk.blk_first.size() * 4, pk.blk_info.size() * 8, pk.packed.size() * 4,
              ((size_t) n_post + 1) * 8, (size_t) n_pos * 4, (size_t) L * 4, pk.dense_bits.size() * 4, pk.dense_rank.size() * 4},
             {}};
    for(int i = 0; i < 10; i++) a.alloc[i] = i == 7 ? pk.list_dense.size() * 4 : a.logical[i];
    for(auto& b: a.alloc) if(b == 0) b = 16;
    return a;
}
}

extern "C" {

tsgpu_status tsgpu_index_load_field(tsgpu_index* idx, const tsgpu_field* f, uint32_t* out_field) {
    const tsgpu_status s = tsgpu_index_load_field_base_(idx, f, out_field);
    if(s == TSGPU_OK) g_field_extra[D(idx)->fields.back()] = extra_for(D(idx)->n_docs);
    return s;
}
tsgpu_status tsgpu_index_load_facet(tsgpu_index* idx, const tsgpu_facet* f, uint32_t* out_facet) {
    const tsgpu_status s = tsgpu_index_load_facet_base_(idx, f, out_facet);
    if(s == TSGPU_OK) g_facet_owner[*out_facet] = idx;
    return s;
}

tsgpu_status tsgpu_index_compact_field(tsgpu_index* idx, uint32_t field, const uint32_t* live, uint32_t n_live) {
    Double* d = D(idx);
    if(field >= d->fields.size()) { g_err = "no such field"; return TSGPU_ERR_INVALID; }
    FieldCopy* c = d->fields[field];
    std::vector<char> seen(c->view.n_lists, 0);
    for(uint32_t i = 0; i < n_live; i++) {
        if(live[i] >= c->view.n_lists) { g_err = "live list id out of range"; return TSGPU_ERR_INVALID; }
        if(seen[live[i]]) { g_err = "live list named twice"; return TSGPU_ERR_INVALID; }
        seen[live[i]] = 1;
    }
    FieldCopy* n = new FieldCopy();
    n->list_off.assign(1, 0); n->pos_off.assign(1, 0);
    for(uint32_t i = 0; i < n_live; i++) {
        const uint32_t l = live[i];
        for(uint64_t p = c->list_off[l]; p < c->list_off[l + 1]; p++) {
            n->ids.push_back(c->ids[p]);
            n->positions.insert(n->positions.end(), c->positions.begin() + c->pos_off[p], c->positions.begin() + c->pos_off[p + 1]);
            n->pos_off.push_back(n->positions.size());
        }
        n->list_off.push_back(n->ids.size());
    }
    if(n->ids.empty()) n->ids.push_back(0);
    if(n->positions.empty()) n->positions.push_back(0);
    n->view.n_lists = n_live; n->view.is_array = c->view.is_array;
    n->view.list_off = n->list_off.data(); n->view.ids = n->ids.data(); n->view.pos_off = n->pos_off.data(); n->view.positions = n->positions.data();
    FieldExtra e = g_field_extra[c];
    e.min_df = tspack::dense_min_df(d->n_docs, e.dense_div);       // compaction classifies under the current capacity
    g_field_extra.erase(c);
    g_field_extra[n] = e;
    d->fields[field] = n;
    tso_index_set_field(d->oi, (int) field, &n->view);
    delete c;
    return TSGPU_OK;
}
// the oracle index is sized at creation: growth builds it again over the same (borrowed) arrays, columns extended
tsgpu_status tsgpu_index_reserve_docs(tsgpu_index* idx, uint32_t n_docs) {
    Double* d = D(idx);
    if(n_docs < d->n_docs) { g_err = "reserve_docs cannot shrink the capacity"; return TSGPU_ERR_INVALID; }
    if(n_docs == d->n_docs) return TSGPU_OK;
    d->n_docs = n_docs;
    for(auto* c: d->cols) c->resize(n_docs, INT64_MIN);
    tso_index_free(d->oi);
    d->oi = tso_index_new(n_docs);
    for(auto* f: d->fields) tso_index_add_field(d->oi, &f->view);
    for(auto* c: d->cols) tso_index_add_sort_column(d->oi, c->data());
    if(d->has_g) tso_index_set_hnsw(d->oi, &d->g);
    for(size_t i = 0; i < g_facets.size(); i++)
        if(g_facet_owner[i] == idx) g_facets[i]->off.resize((size_t) n_docs + 1, g_facets[i]->off.back());
    return TSGPU_OK;
}
tsgpu_status tsgpu_index_field_info(tsgpu_index* idx, uint32_t field, tsgpu_field_info* out) {
    Double* d = D(idx);
    if(field >= d->fields.size()) { g_err = "no such field"; return TSGPU_ERR_INVALID; }
    const FieldCopy& c = *d->fields[field];
    tspack::PackedField pk;
    uint32_t flags = 0;
    pack_copy(c, d->n_docs, pk, flags);
    const Arrays a = arrays_of(c, pk);
    const uint32_t L = c.view.n_lists;
    const uint64_t n_post = c.list_off[L];
    tsgpu_field_info r{};
    r.n_lists = L; r.flags = flags; r.n_postings = n_post; r.n_positions = c.pos_off[n_post]; r.n_blocks = pk.blk_first.size();
    r.n_words = pk.packed.size() - 1; r.n_dense = pk.n_dense; r.dense_words = pk.dense_words;
    for(size_t b: a.alloc) r.device_bytes += b;
    *out = r;
    return TSGPU_OK;
}
tsgpu_status tsgpu_debug_field_array(tsgpu_index* idx, uint32_t field, uint32_t slot, void* dst, size_t cap_bytes, size_t* out_bytes) {
    Double* d = D(idx);
    if(field >= d->fields.size() || slot >= 10 || !out_bytes) { g_err = "bad argument"; return TSGPU_ERR_INVALID; }
    const FieldCopy& c = *d->fields[field];
    tspack::PackedField pk;
    uint32_t flags = 0;
    pack_copy(c, d->n_docs, pk, flags);
    const Arrays a = arrays_of(c, pk);
    *out_bytes = a.logical[slot];
    if(a.logical[slot] > cap_bytes) { g_err = "output buffer too small"; return TSGPU_ERR_CAPACITY; }
    if(a.logical[slot]) memcpy(dst, a.src[slot], a.logical[slot]);
    return TSGPU_OK;
}

}  // extern "C"
