/* tsgpu — C-ABI of the H100-native query hot path for Typesense (libtsgpu.so).
 *
 * The reference has NO plugin/FFI seam for this path: it is reached by ordinary C++ member calls inlined into
 * src/index.cpp (SURVEY.md §8b). This header introduces the boundary at the narrowest existing seams; each entry
 * point names the reference call it replaces. INTEGRATION.md shows the binding a maintainer adds on the reference
 * side.
 *
 * Conventions (mirroring the reference's):
 *   - plain C, opaque handle, caller-allocated outputs (the reference's `uint32_t*&` / `KV*` out-param style);
 *   - every call returns tsgpu_status; nothing throws across the ABI; tsgpu_last_error() gives the message for the
 *     calling thread (the reference's Option<T>{code,error}, include/option.h);
 *   - tsgpu_index_load_* need exclusive access (host holds unique_lock(Index::mutex), src/index.cpp:7513);
 *     search calls are safe for concurrent readers (shared_lock, src/index.cpp:3488) — they serialise on an internal
 *     stream mutex;
 *   - seq_id == hnswlib label == row of every per-document array;
 *   - there is NO CPU fallback: without a CUDA device every call returns TSGPU_ERR_NO_DEVICE.
 */
#ifndef TSGPU_H
#define TSGPU_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int tsgpu_status;
enum {
    TSGPU_OK = 0,
    TSGPU_ERR_NO_DEVICE = 1,
    TSGPU_ERR_INVALID = 2,
    TSGPU_ERR_CUDA = 3,
    TSGPU_ERR_CAPACITY = 4
};

#define TSGPU_NO_LIST 0xFFFFFFFFu
#define TSGPU_MAX_FIELDS 8      /* searched fields per query (reference: FIELD_LIMIT_NUM 100; see DESIGN.md) */
#define TSGPU_MAX_TOKENS 16     /* token rows per combination (Match considers at most 10, include/match_score.h:11) */
#define TSGPU_MAX_TOPK 1024     /* Topster capacity per query of the shared-memory selection (DEFAULT_TOPSTER_SIZE 250); larger with
                                   TSGPU_QFLAG_DEEP_TOPSTER (keyword, wildcard and scored-ids searches) */

typedef struct tsgpu_index tsgpu_index;

/* One searchable string field, flattened. Replaces, for reading, the per-token posting_list_t chains
 * (include/posting_list.h:56-77,130): token t owns postings [list_off[t], list_off[t+1]). */
typedef struct {
    uint32_t n_lists;
    uint32_t is_array;            /* string[]: offsets carry the in-band array protocol of src/index.cpp:1384-1393 */
    const uint64_t* list_off;     /* [n_lists+1] */
    const uint32_t* ids;          /* ascending seq_ids per list */
    const uint64_t* pos_off;      /* [n_postings+1] */
    const uint32_t* positions;    /* raw reference offsets (src/index.cpp:1341-1348) */
} tsgpu_field;

/* Scalar fields of the reference's KV (include/topster.h:20-33), same meaning. */
typedef struct {
    uint64_t key;                 /* seq_id */
    uint64_t distinct_key;
    int64_t  scores[3];
    int64_t  text_match_score;
    float    vector_distance;
    int8_t   match_score_index;
    uint8_t  pad0;
    uint16_t query_index;
} tsgpu_kv;   /* 56 bytes */

enum { TSGPU_SORT_NONE = 0, TSGPU_SORT_TEXT_MATCH = 1, TSGPU_SORT_SEQ_ID = 2, TSGPU_SORT_NUMERIC = 3, TSGPU_SORT_VECTOR_DISTANCE = 4 };
enum { TSGPU_MATCH_MAX_SCORE = 0, TSGPU_MATCH_MAX_WEIGHT = 1, TSGPU_MATCH_SUM_SCORE = 2 };   /* text_match_type_t */
enum { TSGPU_FLAG_PRIORITIZE_EXACT_MATCH = 1, TSGPU_FLAG_PRIORITIZE_TOKEN_POSITION = 2, TSGPU_FLAG_PRIORITIZE_NUM_MATCHING_FIELDS = 4,
       /* hybrid calls: `rerank_hybrid_matches` — Index::compute_aux_scores (src/index.cpp:8793-8923) after the fusion: a result found only by
        * the vector query gets the text match score of the query's FIRST combination (its literal tokens; absent tokens are skipped), one found only
        * by keywords gets its vector distance, then every result is re-scored 1/keyword_rank * (1-alpha) + 1/semantic_rank * alpha */
       TSGPU_FLAG_RERANK_HYBRID_MATCHES = 0x40 };
enum { TSGPU_CFLAG_SYNONYM = 1, TSGPU_CFLAG_DEMOTE_SYNONYM = 2 };

/* A batch of keyword searches. Query q is ONE Index::search_all_candidates call (src/index.cpp:1794-1894): a list
 * of resolved token combinations, all scored into the same Topster. The host keeps the typo/drop-token control loop
 * (fuzzy_search_fields, src/index.cpp:4784) and calls this once per round, for all searches of a multi_search
 * (src/core_api.cpp:1080) at once. */
typedef struct {
    uint32_t n_queries;
    uint32_t n_combos;
    uint32_t n_fields;                 /* F searched fields; slot f -> index field field_ids[f] */
    uint32_t n_filters;                /* inline filters in this batch */
    const uint32_t* field_ids;         /* [F] */
    /* per query */
    const uint32_t* q_combo_off;       /* [nq+1] */
    const int32_t*  q_filter;          /* [nq]: -1 none; >=0 inline filter slot; <=-2 persistent handle -(v+2) */
    const uint32_t* q_excl_off;        /* [nq+1] -> excl_ids */
    const uint32_t* excl_ids;          /* sorted excluded_result_ids per query */
    const uint32_t* q_topk;            /* [nq] Topster capacity (src/index.cpp:3506-3512), <= TSGPU_MAX_TOPK, or any value >= 1 with
                                        * TSGPU_QFLAG_DEEP_TOPSTER; otherwise TSGPU_ERR_CAPACITY */
    const uint8_t*  q_sort_type;       /* [nq*3] TSGPU_SORT_* */
    const int32_t*  q_sort_col;        /* [nq*3] sort column for TSGPU_SORT_NUMERIC */
    const int8_t*   q_sort_order;      /* [nq*3] +1 desc, -1 asc (src/index.cpp:6853-6856) */
    const uint8_t*  q_sort_missing_first; /* [nq*3] or NULL */
    const uint8_t*  q_flags;           /* [nq] TSGPU_FLAG_* | TSGPU_QFLAG_* */
    const uint8_t*  q_match_type;      /* [nq] */
    const uint8_t*  q_num_query_tokens;/* [nq] query_tokens.size() */
    const uint8_t*  q_field_weight;    /* [nq*F] search_field_t::weight */
    /* per combination */
    const uint32_t* c_tok_off;         /* [nc+1] -> token rows */
    const uint32_t* c_total_cost;      /* [nc] next_suggestion2 cost (src/index.cpp:7204) */
    const uint8_t*  c_n_required;      /* [nc] first n rows are ANDed; the remaining rows are dropped_tokens */
    const uint8_t*  c_flags;           /* [nc] TSGPU_CFLAG_* or NULL */
    const int32_t*  c_syn_orig_num_tokens; /* [nc] or NULL (= -1) */
    const int32_t*  c_orig_num_tokens; /* [nc] or NULL (= -1) */
    /* per token row */
    const uint32_t* t_list;            /* [n_rows*F] posting list id in field slot f, TSGPU_NO_LIST if absent */
    /* inline filters: the materialised filter_result_iterator_t::to_filter_id_array() (sorted seq_ids) */
    const uint64_t* filter_off;        /* [n_filters+1] */
    const uint32_t* filter_ids;
} tsgpu_kw_batch;

/* hnswlib graph + vectors as exported from HierarchicalNSW<float> (include/index.h:356-368). */
typedef struct {
    uint32_t n_nodes;
    uint32_t dim;
    uint32_t M;                  /* maxM_; level 0 holds maxM0_ = 2M */
    uint32_t max_level;
    uint32_t entry_point;        /* enterpoint_node_ */
    uint32_t metric;             /* 0 ip, 1 cosine (vectors normalised at index time, src/index.cpp:1049-1052) */
    const float*    vectors;     /* [n*dim], row = internal id = label = seq_id */
    const uint32_t* labels;      /* [n] or NULL (identity) */
    const uint8_t*  levels;      /* [n] element_levels_ */
    const uint32_t* links0;      /* [n*(2M+1)] count, neighbours (get_linklist0) */
    const uint64_t* upper_off;   /* [n+1] record offsets; one (M+1)-u32 record per level 1..levels[i] */
    const uint32_t* links_up;
} tsgpu_hnsw;

typedef struct {
    uint32_t k;                  /* vector_query.k (0 = default, src/index.cpp:3646, 4061-4063) */
    uint32_t ef;                 /* vector_query.ef (default 10); effective max(ef, k) */
    uint32_t flat_search_cutoff;
    float    distance_threshold; /* FLT_MAX default */
    float    alpha;              /* 0.3 default */
    uint32_t fetch_size;
    uint32_t flags;              /* TSGPU_VEC_* (0 = the reference's fp32 loop everywhere: bit-equal distances) */
} tsgpu_vec_params;
/* Flat-path queries (filter below flat_search_cutoff) of one call that share a filter are scanned together on the tensor cores
 * (see tsgpu_flat_distances_batch): same ids, distances within ~1e-6 absolute of the fp32 loop instead of bit-equal — so two
 * candidates whose distances differ by less than that may swap ranks. Opt-in for that reason. */
#define TSGPU_VEC_FLAT_TENSOR 1u
/* Deep pagination for vector and hybrid searches: with this bit tsgpu_vector_search_batch, tsgpu_hybrid_search_batch and
 * tsgpu_hybrid_fuse_batch accept TSGPU_QFLAG_DEEP_TOPSTER with any q_topk >= 1, and the hybrid calls accept k up to the vector
 * stage's bound max(ef, k) <= 4096 (above it TSGPU_ERR_CAPACITY, as for every vector call). A query with the flag and q_topk >
 * TSGPU_MAX_TOPK is fused by the deep kernels (deep_fuse.cuh): the same answer as the reference at any Topster size, with a
 * per-call device buffer sized by the request (vector: 32 bytes per kNN / flat result; hybrid: 69 bytes per Topster slot and
 * 42 per vector result, both counts padded to a power of two, in shared memory when a query's workspace fits). When it cannot be allocated the call returns
 * TSGPU_ERR_CAPACITY (the message gives the bytes) and the index stays usable; a buffer above 256 MiB is freed when the call
 * returns. The other queries of the batch run the ordinary kernels, byte for byte as without the bit. Opt-in for the buffer's
 * sake, as TSGPU_QFLAG_DEEP_TOPSTER is; composes with TSGPU_VEC_FLAT_TENSOR. kv_stride, out_found, query_index and
 * TSGPU_QFLAG_KEEP_ALL_IDS keep their meaning. */
#define TSGPU_VEC_DEEP_TOPSTER 2u

const char* tsgpu_last_error(void);
int tsgpu_device_count(void);
/* Page-locked host memory for the buffers a caller passes to the search calls again and again (query vectors, KV records): copies to
 * and from it run at the link's full rate and without the page faults of a fresh allocation. Any host pointer is accepted by every
 * call; this is an optimisation, not a requirement. */
tsgpu_status tsgpu_host_alloc(size_t bytes, void** out);
tsgpu_status tsgpu_host_free(void* p);

/* ---- index mirror ------------------------------------------------------------------------------------------- */
tsgpu_status tsgpu_index_create(uint32_t n_docs, int device, tsgpu_index** out);
void         tsgpu_index_destroy(tsgpu_index* idx);
/* Mirror one field's posting lists (subscribes to Index::index_field_in_memory, src/index.cpp:700). Pointers may be
 * host or device memory. Returns the field id in *out_field. */
tsgpu_status tsgpu_index_load_field(tsgpu_index* idx, const tsgpu_field* f, uint32_t* out_field);
/* Mirror sort_index[field] (include/index.h:442-447): dense [n_docs], INT64_MIN where the doc has no value. */
tsgpu_status tsgpu_index_load_sort_column(tsgpu_index* idx, const int64_t* vals, uint32_t* out_col);
/* SURVEY 8 f-4 (posting half): the device side of posting_t::upsert / posting_t::erase (src/posting.cpp:247-333; callers
 * Index::index_field_in_memory src/index.cpp:1290-1400, Index::remove_field src/index.cpp:7295-7420). After a batch of writes the
 * binding hands over, in the form of tsgpu_index_load_field, the CURRENT full posting list of every token the batch touched (new
 * tokens included; an erased token = an empty list); they become lists *out_first_list .. *out_first_list + n_lists - 1 of `field`
 * and the caller points those tokens at the new ids. The lists they replace stay in HBM, unreferenced, until the field is
 * compacted (tsgpu_index_compact_field; the read-optimised layout has no holes to patch in place). seq_ids must stay below the
 * index's capacity (tsgpu_index_create, raised by tsgpu_index_reserve_docs). Searches on other threads wait on the index lock for
 * the duration of the call. */
tsgpu_status tsgpu_index_append_lists(tsgpu_index* idx, uint32_t field, const tsgpu_field* f, uint32_t* out_first_list);
/* sort_index values of upserted / removed documents: column[ids[i]] = vals[i] (INT64_MIN = no value). */
tsgpu_status tsgpu_index_set_sort_values(tsgpu_index* idx, uint32_t sort_col, const uint32_t* ids, const int64_t* vals, size_t n);
/* The garbage collection of the posting half of f-4: the field keeps only the lists live_lists[0 .. n_live-1] (the ones the
 * binding's tokens still name — the reference's art_tree leaves, Index::search_index, whose posting_list_t replaced the old
 * ones in place), and list live_lists[i] becomes list id i. Afterwards the field's arrays and flags are exactly what
 * tsgpu_index_load_field builds from those lists in that order at the index's current capacity; the plain-field fast paths a
 * replaced list had disabled come back. Nothing crosses PCIe but the list ids: the lists are gathered on the device, so the
 * peak is the old field plus the new one. A list id >= n_lists or a duplicate is TSGPU_ERR_INVALID and leaves the field
 * untouched. Needs the host's exclusive lock (as tsgpu_index_append_lists); list ids the caller held before are invalid after.
 * tsgpu_get_stats afterwards: ms_kernels = device time of the gather, ms_total = the whole call on the stream. */
tsgpu_status tsgpu_index_compact_field(tsgpu_index* idx, uint32_t field, const uint32_t* live_lists, uint32_t n_live);
/* Raise the seq_id capacity to n_docs (Collection::get_next_seq_id, src/collection.cpp:101-104, only counts up: a live
 * collection outgrows any capacity given at create time). Sort columns grow with INT64_MIN, persistent filters with zeros
 * (their handles stay valid and exclude the new documents), dense posting bitmaps take the new stride, facet rows of the new
 * documents are empty, the markDelete bitmap covers max(n_docs, graph nodes) and wildcard searches cover [0, n_docs). The
 * all_result_ids kept by the last search are dropped. The same value is a no-op, a smaller one TSGPU_ERR_INVALID. The HNSW
 * graph is not touched. Needs the host's exclusive lock. */
tsgpu_status tsgpu_index_reserve_docs(tsgpu_index* idx, uint32_t n_docs);
/* Shape of one mirrored field: what the host needs to decide when compaction pays (it knows how many lists are live). */
#define TSGPU_FIELD_IS_ARRAY 1u          /* string[] field */
#define TSGPU_FIELD_PLAIN_OK 2u          /* plain field, every posting's offsets well formed: the fast scoring path applies */
#define TSGPU_FIELD_POS16 4u             /* ... and every position fits 16 bits */
typedef struct {
    uint32_t n_lists;                    /* list ids in use, live or replaced */
    uint32_t flags;                      /* TSGPU_FIELD_* */
    uint64_t n_postings;
    uint64_t n_positions;
    uint64_t n_blocks;                   /* packed id blocks */
    uint64_t n_words;                    /* packed 32-bit words (without the padding word) */
    uint32_t n_dense;                    /* lists that also have a bitmap */
    uint32_t dense_words;                /* words per bitmap */
    uint64_t device_bytes;               /* HBM held by the field's arrays */
} tsgpu_field_info;
tsgpu_status tsgpu_index_field_info(tsgpu_index* idx, uint32_t field, tsgpu_field_info* out);
/* Mirror hnsw_index_t (vectors + graph). Pointers may be host or device memory. */
tsgpu_status tsgpu_index_load_hnsw(tsgpu_index* idx, const tsgpu_hnsw* g);
/* Build the vector index ON THE DEVICE: hnswlib's addPoint (the loop of Index::batch_memory_index, src/index.cpp:1003-1054,
 * which the reference runs on 4 host threads) as batched rounds — see csrc/hnsw_build.cuh. label == row index. Levels are
 * drawn exactly as hnswlib draws them (std::default_random_engine(seed)); with max_batch == 1 the graph equals the
 * single-threaded hnswlib build link for link; larger batches relax the insertion order the way hnswlib's own
 * multi-threaded build does, deterministically. M in 2..16. `vectors` may be host or device memory; with
 * keep_device_vectors != 0 a device buffer is used in place (the caller keeps it alive for the index's lifetime). */
tsgpu_status tsgpu_index_build_hnsw(tsgpu_index* idx, const float* vectors, uint32_t n, uint32_t dim, uint32_t M,
                                    uint32_t ef_construction, uint32_t seed, uint32_t metric, uint32_t max_batch,
                                    int keep_device_vectors);
/* SURVEY 8 f-4 (vector half): hnswlib's addPoint for `n_add` MORE vectors (labels n .. n + n_add - 1, n = current node count)
 * into the graph the index holds, built here or loaded (src/index.cpp:1052, the same call the reference makes for every new
 * document). The existing nodes keep their links except where a new node's reverse links change them, exactly as in a
 * sequential addPoint; levels continue the generator sequence of `seed`. Needs identity labels, M in 2..16. With
 * max_batch == 1, build(n1) + append(n2) equals build(n1 + n2) link for link. */
tsgpu_status tsgpu_index_append_hnsw(tsgpu_index* idx, const float* vectors, uint32_t n_add, uint32_t ef_construction, uint32_t seed, uint32_t max_batch);
/* hnswlib's markDelete / unmarkDelete (src/index.cpp:7423 on document removal): a deleted label is never returned by a search
 * but is still traversed. `labels`: host memory. Loading or rebuilding a graph clears all marks. (hnswlib's slot reuse for
 * replace_deleted inserts is not mirrored: appended vectors always get new labels.) */
tsgpu_status tsgpu_index_mark_deleted(tsgpu_index* idx, const uint32_t* labels, size_t n, int deleted);
/* Shape of the loaded / built graph; build_counters[5] (may be null) = distance evaluations of the construction searches,
 * expansions, heuristic distance evaluations, rows re-selected, rounds of the last tsgpu_index_build_hnsw. */
tsgpu_status tsgpu_index_hnsw_info(tsgpu_index* idx, uint32_t* n_nodes, uint32_t* dim, uint32_t* M, uint32_t* max_level,
                                   uint32_t* entry_point, uint64_t* n_upper_records, uint64_t* build_counters);
/* Copy the graph out (what a snapshot would persist; what the parity oracle walks). Destinations may be host or device
 * memory, any may be null: levels[n], links0[n*(2M+1)], upper_off[n+1], links_up[n_upper_records*(M+1)]. */
tsgpu_status tsgpu_index_export_hnsw(tsgpu_index* idx, uint8_t* levels, uint32_t* links0, uint64_t* upper_off, uint32_t* links_up);
/* Persistent filter (a mirrored filter leaf / cached filter result): sorted seq_ids -> device bitmap. */
tsgpu_status tsgpu_filter_create(tsgpu_index* idx, const uint32_t* ids, size_t n, int32_t* out_handle);
tsgpu_status tsgpu_filter_destroy(tsgpu_index* idx, int32_t handle);
/* filter_by evaluated ON THE DEVICE (SURVEY 8 f-2): the result never visits the host.
 * A numeric / bool leaf (filter_result_iterator_t over num_tree_t, src/filter_result_iterator.cpp:1507-1700, src/num_tree.cpp): one pass
 * over the mirrored column `sort_col` (tsgpu_index_load_sort_column; floats as float_to_int64_t, bools as 0 / 1). Docs without a value
 * match no comparator; TSGPU_CMP_NE is "every doc but the equal ones" (apply_not_equals). RANGE = [v1, v2] (`field:[v1..v2]`). */
enum { TSGPU_CMP_EQ = 0, TSGPU_CMP_NE = 1, TSGPU_CMP_LT = 2, TSGPU_CMP_LE = 3, TSGPU_CMP_GT = 4, TSGPU_CMP_GE = 5, TSGPU_CMP_RANGE = 6 };
tsgpu_status tsgpu_filter_numeric(tsgpu_index* idx, uint32_t sort_col, int op, int64_t v1, int64_t v2, int32_t* out_handle, size_t* out_n);
/* The tree's inner nodes on two persistent filters: op = TSGPU_SET_AND / TSGPU_SET_OR / TSGPU_SET_EXCLUDE (a AND NOT b); string leaves come from
 * tsgpu_exact_matches / tsgpu_prefix_matches / tsgpu_phrase_matches + tsgpu_filter_create. */
tsgpu_status tsgpu_filter_combine(tsgpu_index* idx, int op, int32_t a, int32_t b, int32_t* out_handle, size_t* out_n);
tsgpu_status tsgpu_filter_ids(tsgpu_index* idx, int32_t handle, uint32_t* out_ids, size_t cap, size_t* out_n);

/* ---- search -------------------------------------------------------------------------------------------------- */
/* posting_list_t::intersect / posting_t::intersect (src/posting_list.cpp:708, src/posting.cpp:388): k-way AND of
 * whole posting lists of one field. out_ids capacity `cap`; *out_n = result count (ascending). */
tsgpu_status tsgpu_intersect(tsgpu_index* idx, uint32_t field, const uint32_t* lists, uint32_t k,
                             uint32_t* out_ids, size_t cap, size_t* out_n);

/* posting_t::contains_atleast_one / posting_list_t::contains_atleast_one (src/posting.cpp:365, src/posting_list.cpp:1090-1112;
 * call sites src/index.cpp:6519, src/art.cpp:992): *out = 1 when any of the ascending `ids` is in the list. */
tsgpu_status tsgpu_contains_atleast_one(tsgpu_index* idx, uint32_t field, uint32_t list, const uint32_t* ids, size_t n, int* out);

/* posting_t::get_phrase_matches (src/posting_list.cpp:1791; call site src/index.cpp:5960): of the ascending `ids`,
 * keep those where the k lists' tokens occur as a consecutive sequence. */
tsgpu_status tsgpu_phrase_matches(tsgpu_index* idx, uint32_t field, const uint32_t* lists, uint32_t k,
                                  const uint32_t* ids, size_t n, uint32_t* out_ids, size_t* out_n);

/* posting_t::get_exact_matches / posting_list_t::get_exact_matches (src/posting.cpp:485, src/posting_list.cpp:1281-1452;
 * call sites src/index.cpp:3232, src/filter_result_iterator.cpp:3050 — the `:=` string filter): of the ascending
 * `ids`, keep those whose field value (or one of its array elements) is exactly the k tokens in order.
 * As at the reference's call sites, `ids` must come from the intersection of the same lists; an id absent from one
 * of the lists is dropped (the reference would read the next posting's offsets instead). */
tsgpu_status tsgpu_exact_matches(tsgpu_index* idx, uint32_t field, const uint32_t* lists, uint32_t k,
                                 const uint32_t* ids, size_t n, uint32_t* out_ids, size_t* out_n);

/* posting_list_t::get_prefix_matches (src/posting_list.cpp:1129-1279; call site src/filter_result_iterator.cpp:3002):
 * same, but the value only has to START with the k tokens. */
tsgpu_status tsgpu_prefix_matches(tsgpu_index* idx, uint32_t field, const uint32_t* lists, uint32_t k,
                                  const uint32_t* ids, size_t n, uint32_t* out_ids, size_t* out_n);

/* ArrayUtils::and_scalar / or_scalar / exclude_scalar (include/array_utils.h:13-19, src/array_utils.cpp:4-170; the
 * all_result_ids maintenance at src/index.cpp:5081-5090 and the filter combinators): set operation on two STRICTLY
 * ascending id arrays with ids < n_docs (what the index always holds; anything else is TSGPU_ERR_INVALID).
 * EXCLUDE = a minus b. Result ascending in out_ids (capacity `cap`), count in *out_n. */
enum { TSGPU_SET_AND = 0, TSGPU_SET_OR = 1, TSGPU_SET_EXCLUDE = 2 };
tsgpu_status tsgpu_ids_setop(tsgpu_index* idx, int op, const uint32_t* a, size_t na, const uint32_t* b, size_t nb,
                             uint32_t* out_ids, size_t cap, size_t* out_n);

/* ---- SURVEY 8 f-1: typo / prefix candidate tokens (timed by tools/bench_art_gpu.py and the bench's end-to-end leg) ----
 * A field's token index (art_tree, include/art.h:124-127; one per string field, Index::search_index) as flat arrays:
 * inner nodes with the first 8 bytes of their compressed path (MAX_PREFIX_LEN), child links ascending by key byte, leaf
 * keys. typesense_b200/host/art_mirror.hpp builds them from an export of the live tree. */
typedef struct tsgpu_art {
    uint32_t n_nodes, n_children, n_leaves;
    int32_t  root;                      /* >= 0: inner node; < 0: leaf ~root (a one-token index); ignored when n_leaves == 0 */
    const uint32_t* node_first_child;   /* [n_nodes] -> child_byte / child_ref */
    const uint16_t* node_n_children;    /* [n_nodes] */
    const uint8_t*  node_partial_len;   /* [n_nodes] art_node::partial_len */
    const uint8_t*  node_partial;       /* [n_nodes * 8] art_node::partial */
    const uint8_t*  child_byte;         /* [n_children] */
    const int32_t*  child_ref;          /* [n_children] >= 0 inner node, < 0 leaf ~ref */
    const uint64_t* leaf_key_off;       /* [n_leaves + 1] -> leaf_keys (keys without the terminating NUL) */
    const uint8_t*  leaf_keys;
    const uint32_t* node_rank;          /* [n_nodes], [n_leaves]: position in the pre-order of the tree with children from the largest */
    const uint32_t* leaf_rank;          /* byte down (the order art_fuzzy_recurse visits); NULL: computed at load */
} tsgpu_art;

/* Replaces / extends the mirror of `field` (an id returned by tsgpu_index_load_field). Needs the host's exclusive lock. */
tsgpu_status tsgpu_index_load_art(tsgpu_index* idx, uint32_t field, const tsgpu_art* art);

/* The tree walk of art_fuzzy_search_i (src/art.cpp:1825-1894: art_fuzzy_recurse :1596-1738 with fuzzy_search_state
 * :1487-1594), batched: search i looks for keys within [min_cost[i], max_cost[i]] edits of terms[term_off[i]..term_off[i+1])
 * (prefix[i] != 0: keys having such a prefix) — Index::fuzzy_search_fields issues one such search per (token, cost, field),
 * src/index.cpp:4949/5004. out_hits[i*cap ..] receives the matching subtrees / leaves (node >= 0, leaf ~ref) in the order
 * the reference's recursion meets them, out_counts[i] their number. out_flags[i] != 0 means the search must be walked on
 * the host instead (1: deeper than the device stack, 2: term longer than 31 bytes, 4: more than cap hits). The second half
 * — art_topk_iter, validate_and_add_leaf, the final sort (a few dozen leaves per search) — is host code:
 * art_mirror_t::finish. */
tsgpu_status tsgpu_art_walk_batch(tsgpu_index* idx, uint32_t field, uint32_t n, const uint32_t* term_off, const uint8_t* terms,
                                  const uint8_t* min_cost, const uint8_t* max_cost, const uint8_t* prefix,
                                  int32_t* out_hits, uint32_t cap, uint32_t* out_counts, uint8_t* out_flags);

/* search_all_candidates -> search_across_fields -> or_iterator_t::intersect + compute_aggregated_score +
 * compute_sort_scores + Topster::add (src/index.cpp:1794, 5385-5596), batched over queries.
 * out_kv[q*kv_stride ..] = the query's Topster in Topster::sort() order, out_count[q] entries;
 * out_found[q] = |all_result_ids| contributed by this call. */
tsgpu_status tsgpu_keyword_search_batch(tsgpu_index* idx, const tsgpu_kw_batch* b, tsgpu_kv* out_kv,
                                        uint32_t kv_stride, uint32_t* out_count, uint32_t* out_found);

/* Index::search_wildcard (src/index.cpp:6616-6800), `q=*`: every id of the query's filter (all seq_ids < n_docs when it
 * has none) minus the exclusion list is given sort scores (text-match clause = 100) and goes through the Topster.
 * The combinations of `b` are ignored. Same outputs as tsgpu_keyword_search_batch; query_index is 0. */
tsgpu_status tsgpu_wildcard_search_batch(tsgpu_index* idx, const tsgpu_kw_batch* b, tsgpu_kv* out_kv, uint32_t kv_stride,
                                         uint32_t* out_count, uint32_t* out_found);

/* VectorIndex::searchKnn: vecdex->searchKnnCloserFirst(q, k, ef, &VectorFilterFunctor) (src/index.cpp:3384-3386),
 * batched. queries [nq*dim] (already normalised for cosine). q_filter as in tsgpu_kw_batch (inline slots refer to
 * filter_off/filter_ids). Outputs [nq*k] closest first; out_n[q] valid entries. */
tsgpu_status tsgpu_knn_batch(tsgpu_index* idx, const float* queries, uint32_t nq, uint32_t k, uint32_t ef,
                             const int32_t* q_filter, uint32_t n_filters, const uint64_t* filter_off,
                             const uint32_t* filter_ids, float* out_dist, uint32_t* out_labels, uint32_t* out_n);

/* process_results_bruteforce (src/index.cpp:3345-3374): distance of the query to every id, in id order. */
tsgpu_status tsgpu_flat_distances(tsgpu_index* idx, const float* query, const uint32_t* ids, size_t n, float* out_dist);
/* The same for nq queries that share ONE candidate set (the requests of a multi_search that carry the same filter_by, each below
 * flat_search_cutoff): out_dist[q*n + i] = distance(query q, ids[i]). The loop of src/index.cpp:3345-3374 over (query, id) pairs is
 * the contraction [n x dim] . [dim x nq]: it runs on the tensor cores (wgmma .tf32, 3-term split of the fp32 operands,
 * fp32 accumulation in registers; csrc/flat_tc.cu) when dim is a multiple of 32, else pair by pair like tsgpu_flat_distances. Distances
 * agree with the fp32 loop to ~1e-6 absolute (gate: 1e-4 relative), not bit for bit. queries / ids / out_dist: host or device memory.
 * tsgpu_vector_search_batch / tsgpu_hybrid_search_batch route their flat-path queries through the same kernel when >= 8 of them
 * share a filter. */
tsgpu_status tsgpu_flat_distances_batch(tsgpu_index* idx, const float* queries, uint32_t nq, const uint32_t* ids, size_t n, float* out_dist);

/* Wildcard + vector query (src/index.cpp:3645-3732). Filters / exclusions / sort clauses / topk come from `b`
 * (its combinations are ignored). */
tsgpu_status tsgpu_vector_search_batch(tsgpu_index* idx, const tsgpu_kw_batch* b, const float* qvecs,
                                       const tsgpu_vec_params* vp, tsgpu_kv* out_kv, uint32_t kv_stride,
                                       uint32_t* out_count, uint32_t* out_found);

/* The scoring half of Index::do_phrase_search for a phrase-ONLY query (src/index.cpp:6019-6082): query q's result ids are its
 * inline filter (the phrase matches, already ANDed with filter_by and minus exclusions), id_scores[i] — aligned with the
 * batch's filter_ids — the match score of each (the reference's `100000 + field weight` for the first 10000 matches of a field,
 * 0 beyond); every id goes through compute_sort_scores into the Topster. found = number of ids. */
tsgpu_status tsgpu_scored_ids_search_batch(tsgpu_index* idx, const tsgpu_kw_batch* b, const int64_t* id_scores, tsgpu_kv* out_kv,
                                           uint32_t kv_stride, uint32_t* out_count, uint32_t* out_found);

/* Keyword + vector query with reciprocal-rank fusion (src/index.cpp:4036-4221). */
tsgpu_status tsgpu_hybrid_search_batch(tsgpu_index* idx, const tsgpu_kw_batch* b, const float* qvecs,
                                       const tsgpu_vec_params* vp, tsgpu_kv* out_kv, uint32_t kv_stride,
                                       uint32_t* out_count, uint32_t* out_found);

/* The tail of a keyword + vector query whose keyword stage has already run (Index::search reaches the vector query only
 * after fuzzy_search_fields and the drop-token rounds, src/index.cpp:4036): kw_kv[q*kw_stride ..] holds query q's final
 * keyword Topster in Topster::sort() order (kw_count[q] <= q_topk[q] entries), kw_found[q] its all_result_ids_len and
 * kw_searched[q] its searched_queries.size(); the batch's combinations are every combination the rounds executed (they are
 * only probed to tell vector results that are keyword matches from new ids). Runs the vector stage and the rank fusion as
 * tsgpu_hybrid_search_batch does. */
tsgpu_status tsgpu_hybrid_fuse_batch(tsgpu_index* idx, const tsgpu_kw_batch* b, const tsgpu_kv* kw_kv, uint32_t kw_stride,
                                     const uint32_t* kw_count, const uint32_t* kw_found, const uint32_t* kw_searched,
                                     const float* qvecs, const tsgpu_vec_params* vp, tsgpu_kv* out_kv, uint32_t kv_stride,
                                     uint32_t* out_count, uint32_t* out_found);

/* ---- multi-GPU (SURVEY 8e) --------------------------------------------------------------------------------------- */
/* A multi_search batch shards over queries: one process per GPU, a full replica each, rank r answers its contiguous slice,
 * and the ONLY exchange is the gather of the slices' result records on the rank that answers the request
 * (src/core_api.cpp:1080-1131 spread over ranks). The exchange runs inside the library: NCCL over NVLink, bound at run time
 * (dlopen of libnccl.so.2; override with TSGPU_NCCL_LIB), device to device on the index's stream. */
tsgpu_status tsgpu_comm_unique_id(void* out128);                      /* ncclGetUniqueId: create on one rank, hand to the others */
tsgpu_status tsgpu_comm_init(tsgpu_index* idx, int rank, int world, const void* id128);
tsgpu_status tsgpu_comm_destroy(tsgpu_index* idx);
/* every rank sends `bytes` from src (host or device); on `root`, dst (host or device) receives world * bytes in rank order */
tsgpu_status tsgpu_comm_gather(tsgpu_index* idx, const void* src, size_t bytes, void* dst, int root);
tsgpu_status tsgpu_comm_last_ms(tsgpu_index* idx, float* out_ms);     /* device time of the last gather on this rank */

/* ---- facets (SURVEY 8 f-3) ---------------------------------------------------------------------------------------- */
/* tsgpu_kw_batch::q_flags bit: keep the query's all_result_ids (the id_buff / vec_search_ids union of src/index.cpp:5081-5090,
 * 4215-4219) on the device after a keyword / hybrid search, as one bit per doc — the `out_all_ids` of SURVEY 8(b). */
#define TSGPU_QFLAG_KEEP_ALL_IDS 0x80u
/* tsgpu_kw_batch::q_flags bit: the query may have q_topk > TSGPU_MAX_TOPK (deep pagination: page 40 at 250 per page needs a
 * Topster of 10,000). Such a query's every match goes to a device buffer, which is then de-duplicated per seq_id and sorted;
 * the memory this takes grows with the query's match count (at most the sum over its combinations of the driver list's
 * postings; a wildcard or scored-ids query: its id count), not with q_topk. When that buffer cannot be allocated the call
 * returns TSGPU_ERR_CAPACITY (the message gives the bytes) and the index stays usable. A buffer above 256 MiB is freed when the
 * call returns; a smaller one stays with the index for the next call. With q_topk <= TSGPU_MAX_TOPK the
 * flag changes nothing. Outputs keep their meaning: kv_stride truncates a query's records, out_found and query_index are
 * as without the flag. Honoured by tsgpu_keyword_search_batch, tsgpu_wildcard_search_batch and
 * tsgpu_scored_ids_search_batch; the vector and hybrid calls (tsgpu_vector_search_batch, tsgpu_hybrid_search_batch,
 * tsgpu_hybrid_fuse_batch) reject it with TSGPU_ERR_INVALID, since their fusion keeps the Topster in shared memory, unless
 * tsgpu_vec_params::flags has TSGPU_VEC_DEEP_TOPSTER. */
#define TSGPU_QFLAG_DEEP_TOPSTER 0x20u
/* Mirror of one facet field: facet_index_t's seq_id -> facet ids (src/facet_index.cpp:27-90; ids are the dense counter the
 * reference assigns per distinct value; a binding densifies numeric facets the same way). Host or device pointers. */
typedef struct {
    uint32_t n_values;           /* ids are 0 .. n_values-1 */
    const uint64_t* doc_off;     /* [n_docs+1] */
    const uint32_t* value_ids;   /* per doc in stored order: array_pos = index inside the doc's slice */
} tsgpu_facet;
typedef struct { uint32_t value_id, count, doc_id, array_pos; } tsgpu_facet_count;
tsgpu_status tsgpu_index_load_facet(tsgpu_index* idx, const tsgpu_facet* f, uint32_t* out_facet);
/* Index::do_facets, hash-index branch (src/index.cpp:1674-1780) over ascending `result_ids` (host or device), then the
 * (count, id)-descending order of Collection::search (include/collection.h:552): writes the top_n (<= 1024) entries,
 * *out_n = entries written, *out_distinct = values with a count. sample_mod > 1: `estimate_facets`, every sample_mod-th id.
 * doc_id / array_pos: of the largest result id holding the value (one sequential do_facets pass). */
tsgpu_status tsgpu_facet_counts(tsgpu_index* idx, uint32_t facet, const uint32_t* result_ids, size_t n, uint32_t sample_mod,
                                uint32_t top_n, tsgpu_facet_count* out, uint32_t* out_n, uint32_t* out_distinct);
/* The same over the all_result_ids the LAST keyword / hybrid search kept (TSGPU_QFLAG_KEEP_ALL_IDS), every query of that
 * batch at once: out[q*top_n ..], out_n[q], out_distinct[q] (0 for queries that did not keep their ids). */
tsgpu_status tsgpu_facet_counts_last(tsgpu_index* idx, uint32_t facet, uint32_t top_n, tsgpu_facet_count* out, uint32_t* out_n,
                                     uint32_t* out_distinct);
/* all_result_ids of query q of the last search (ascending; needs TSGPU_QFLAG_KEEP_ALL_IDS). */
tsgpu_status tsgpu_all_result_ids_last(tsgpu_index* idx, uint32_t q, uint32_t* out_ids, size_t cap, size_t* out_n);

/* ---- diversity re-ranking ------------------------------------------------------------------------------------------ */
/* One term of a curation rule's `diversity.similarity_metric` (include/diversity.h similarity_metric_t), resolved to the mirror. */
enum { TSGPU_DIV_EQUALITY = 0, TSGPU_DIV_JACCARD = 1 };
#define TSGPU_MAX_DIV_METRICS 16
typedef struct {
    uint32_t facet;      /* id from tsgpu_index_load_facet, or TSGPU_NO_LIST: use sort_col */
    int32_t  sort_col;   /* sort column (tsgpu_index_load_sort_column) when facet == TSGPU_NO_LIST */
    uint32_t method;     /* TSGPU_DIV_* */
    float    weight;     /* 1 by default */
} tsgpu_div_metric;
/* Index::populate_result_kvs, diversity branch (src/index.cpp:9016-9064; similarity_t::calculate, src/diversity.cpp), batched:
 * query q's records kv[q*kv_stride .. + count[q]] (a Topster after sort(), unique keys) are written to out_kv[q*kv_stride ..] in
 * MMR order; the records themselves are unchanged. kv / out_kv: host or device memory (out_kv may be kv); lambda / count: host
 * memory. lambda[q] in [0, 1]. Position 0 stays first; each next pick is the unpicked record with the greatest
 * lambda * vector_distance - (1 - lambda) * (max similarity to the picked ones), the lowest position on a tie. Similarity sums the
 * metrics in list order: a facet metric compares the two documents' facet values as sets (jaccard: |∩| / |∪| * weight; equality:
 * weight when the sets are equal), a sort metric adds weight when both documents have a value and the values are equal (equality
 * only); a document without values (an empty facet row, INT64_MIN, a seq_id >= the capacity) adds nothing. Arithmetic in the
 * reference's float / double types, so the order is the reference's bit for bit. An unknown facet id or sort column, a method
 * outside the enum, n_metrics == 0, count[q] > kv_stride or a lambda that is NaN or outside [0, 1] is TSGPU_ERR_INVALID;
 * n_metrics > TSGPU_MAX_DIV_METRICS or a device scratch that cannot be allocated is TSGPU_ERR_CAPACITY (the message gives the
 * bytes); the index stays usable. tsgpu_get_stats afterwards: ms_kernels = device time of the kernels, ms_total = the whole
 * call on the stream. */
tsgpu_status tsgpu_diversify_batch(tsgpu_index* idx, const tsgpu_div_metric* metrics, uint32_t n_metrics, uint32_t nq,
                                   const float* lambda, const tsgpu_kv* kv, uint32_t kv_stride, const uint32_t* count,
                                   tsgpu_kv* out_kv);

/* ---- instrumentation ------------------------------------------------------------------------------------------ */
/* Device-time breakdown of the last search call on this index (CUDA events on the library's stream), kernel launch
 * count since index creation, and algorithmic work counters of the last call. */
typedef struct {
    float    ms_total;           /* whole call on the device stream, including H2D / D2H copies */
    float    ms_kernels;         /* between first kernel launch and last kernel completion */
    float    ms_keyword;         /* intersect+score+select kernels */
    float    ms_knn;             /* HNSW / flat kernels */
    float    ms_fuse;            /* RRF / final top-k kernels */
    uint64_t launches_total;     /* kernels launched by this library since index creation */
    uint64_t kw_driver_ids;      /* candidate ids scanned: driver-list ids, or the documents a bitmap tile covers (all-dense combinations) */
    uint64_t kw_probe_ids;       /* posting ids covered by probed blocks */
    uint64_t kw_matches;         /* docs scored */
    uint64_t knn_dist;           /* distance evaluations */
    uint64_t knn_expanded;       /* expanded nodes */
    uint64_t h2d_bytes;
    uint64_t d2h_bytes;
    float    ms_kw_search;       // kw_search_kernel alone
    float    ms_kw_merge;        // kw_merge_kernel levels + kw_final_kernel + found_popcount_kernel
    float    ms_host_plan;       /* host wall time of batch planning (build_kw_plan) inside the call; the GPU idles meanwhile */
    uint64_t knn_spec_hits;      /* expansions whose node was the one the walk had prefetched for (speculation hit) */
    uint64_t knn_tier2_walks;    /* graph walks whose visited set outgrew shared memory (continued in the HBM tier) */
    uint64_t knn_retried;        /* graph walks that outgrew their slot's scratch and were re-run alone with a full-size slot */
    uint64_t h2d_total;          /* host->device / device->host bytes since index creation (every call; h2d_bytes / d2h_bytes: last call) */
    uint64_t d2h_total;
    uint64_t calls_total;        /* C-ABI search calls since index creation */
    uint64_t knn_table_probes;   /* neighbour tests of the graph walks that missed the shared-memory visited cache (went to the HBM table) */
    uint64_t flat_tc_queries;    /* flat-path queries answered by the tensor-core scan (groups sharing a candidate set) in the last call */
    uint64_t deep_entries;       /* entries the deep queries (TSGPU_QFLAG_DEEP_TOPSTER) of the last call emitted */
    uint64_t deep_bytes;         /* device bytes the deep buffer of the last call needed */
    float    ms_deep_emit;       /* unit kernels of the deep queries (also inside ms_kw_search) */
    float    ms_deep_dedup;      /* de-duplication of the deep queries' entries per seq_id */
    float    ms_deep_select;     /* sort of the distinct entries and the record write */
    float    pad_deep;
    uint64_t deep_fuse_bytes;    /* device bytes of the deep vector / hybrid workspace of the last call (TSGPU_VEC_DEEP_TOPSTER) */
    float    ms_deep_fuse_prep;  /* deep hybrid fusion, slowest deep query of each phase: keyword Topster, text ranks, vector list, */
    float    ms_deep_fuse_replay;/*   per-result work | the serial replay of the loop | rerank_hybrid_matches | final sort and */
    float    ms_deep_fuse_rerank;/*   write. Deep vector assembly: ms_deep_fuse_sort = the sorts and record writes */
    float    ms_deep_fuse_sort;
} tsgpu_stats;
tsgpu_status tsgpu_get_stats(tsgpu_index* idx, tsgpu_stats* out);
/* Instrumentation: per graph walk of the last HNSW launch, out[2q] = expanded nodes, out[2q+1] = distance evaluations. */
tsgpu_status tsgpu_debug_knn_work(tsgpu_index* idx, uint32_t* out, uint32_t cap_queries, uint32_t* out_n);
/* Instrumentation: one of a field's ten device arrays over its logical length (bytes in *out_bytes; TSGPU_ERR_CAPACITY when
 * cap_bytes is smaller). slot: 0 list_off, 1 list_blk_off, 2 blk_first, 3 blk_info, 4 packed (with its padding word), 5 pos_off,
 * 6 positions, 7 list_dense, 8 dense_bits (with its 16 padding words), 9 dense_rank (with its padding entry); see
 * csrc/postings_device.cuh. dst: host memory. */
tsgpu_status tsgpu_debug_field_array(tsgpu_index* idx, uint32_t field, uint32_t slot, void* dst, size_t cap_bytes, size_t* out_bytes);

#ifdef __cplusplus
}
#endif
#endif
