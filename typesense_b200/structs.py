"""ctypes mirrors of include/tsgpu.h (and, layout-identical, oracle/ts_oracle.h) plus numpy-backed builders.

Harness-side only: the product is libtsgpu.so (CUDA + C-ABI); this module just fills its plain-C structs from numpy
arrays so tests and bench.py can hand the SAME buffers to the CUDA library and to the CPU oracle.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

NO_LIST = 0xFFFFFFFF
MAX_FIELDS = 8
MAX_TOKENS = 16

SORT_NONE, SORT_TEXT_MATCH, SORT_SEQ_ID, SORT_NUMERIC, SORT_VECTOR_DISTANCE = 0, 1, 2, 3, 4
MATCH_MAX_SCORE, MATCH_MAX_WEIGHT, MATCH_SUM_SCORE = 0, 1, 2
FLAG_PRIORITIZE_EXACT_MATCH, FLAG_PRIORITIZE_TOKEN_POSITION, FLAG_PRIORITIZE_NUM_MATCHING_FIELDS = 1, 2, 4
FLAG_RERANK_HYBRID_MATCHES, FLAG_KEEP_ALL_IDS = 0x40, 0x80
FLAG_DEEP_TOPSTER = 0x20                  # q_topk may exceed MAX_TOPK (keyword, wildcard and scored-ids searches)
MAX_TOPK = 1024
CFLAG_SYNONYM, CFLAG_DEMOTE_SYNONYM = 1, 2

u8p, u16p, u32p, u64p = (C.POINTER(C.c_uint8), C.POINTER(C.c_uint16), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64))
i8p, i32p, i64p, f32p = (C.POINTER(C.c_int8), C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_float))

KV_DTYPE = np.dtype([
    ("key", "<u8"), ("distinct_key", "<u8"), ("scores", "<i8", (3,)), ("text_match_score", "<i8"),
    ("vector_distance", "<f4"), ("match_score_index", "i1"), ("pad0", "u1"), ("query_index", "<u2"),
])
assert KV_DTYPE.itemsize == 56


class FieldStruct(C.Structure):
    _fields_ = [("n_lists", C.c_uint32), ("is_array", C.c_uint32), ("list_off", u64p), ("ids", u32p),
                ("pos_off", u64p), ("positions", u32p)]


class KwBatchStruct(C.Structure):
    _fields_ = [
        ("n_queries", C.c_uint32), ("n_combos", C.c_uint32), ("n_fields", C.c_uint32), ("n_filters", C.c_uint32),
        ("field_ids", u32p),
        ("q_combo_off", u32p), ("q_filter", i32p), ("q_excl_off", u32p), ("excl_ids", u32p), ("q_topk", u32p),
        ("q_sort_type", u8p), ("q_sort_col", i32p), ("q_sort_order", i8p), ("q_sort_missing_first", u8p),
        ("q_flags", u8p), ("q_match_type", u8p), ("q_num_query_tokens", u8p), ("q_field_weight", u8p),
        ("c_tok_off", u32p), ("c_total_cost", u32p), ("c_n_required", u8p), ("c_flags", u8p),
        ("c_syn_orig_num_tokens", i32p), ("c_orig_num_tokens", i32p),
        ("t_list", u32p),
        ("filter_off", u64p), ("filter_ids", u32p),
    ]


class HnswStruct(C.Structure):
    _fields_ = [("n_nodes", C.c_uint32), ("dim", C.c_uint32), ("M", C.c_uint32), ("max_level", C.c_uint32),
                ("entry_point", C.c_uint32), ("metric", C.c_uint32), ("vectors", f32p), ("labels", u32p),
                ("levels", u8p), ("links0", u32p), ("upper_off", u64p), ("links_up", u32p)]


class VecParamsStruct(C.Structure):
    _fields_ = [("k", C.c_uint32), ("ef", C.c_uint32), ("flat_search_cutoff", C.c_uint32),
                ("distance_threshold", C.c_float), ("alpha", C.c_float), ("fetch_size", C.c_uint32), ("flags", C.c_uint32)]


class ArtStruct(C.Structure):
    """tsgpu_art (include/tsgpu.h)"""
    _fields_ = [("n_nodes", C.c_uint32), ("n_children", C.c_uint32), ("n_leaves", C.c_uint32), ("root", C.c_int32),
                ("node_first_child", C.c_void_p), ("node_n_children", C.c_void_p), ("node_partial_len", C.c_void_p), ("node_partial", C.c_void_p),
                ("child_byte", C.c_void_p), ("child_ref", C.c_void_p), ("leaf_key_off", C.c_void_p), ("leaf_keys", C.c_void_p),
                ("node_rank", C.c_void_p), ("leaf_rank", C.c_void_p)]


class StatsStruct(C.Structure):
    _fields_ = [("ms_total", C.c_float), ("ms_kernels", C.c_float), ("ms_keyword", C.c_float), ("ms_knn", C.c_float),
                ("ms_fuse", C.c_float), ("launches_total", C.c_uint64), ("kw_driver_ids", C.c_uint64),
                ("kw_probe_ids", C.c_uint64), ("kw_matches", C.c_uint64), ("knn_dist", C.c_uint64),
                ("knn_expanded", C.c_uint64), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64),
                ("ms_kw_search", C.c_float), ("ms_kw_merge", C.c_float), ("ms_host_plan", C.c_float), ("knn_spec_hits", C.c_uint64),
                ("knn_tier2_walks", C.c_uint64), ("knn_retried", C.c_uint64), ("h2d_total", C.c_uint64), ("d2h_total", C.c_uint64),
                ("calls_total", C.c_uint64), ("knn_table_probes", C.c_uint64), ("flat_tc_queries", C.c_uint64),
                ("deep_entries", C.c_uint64), ("deep_bytes", C.c_uint64), ("ms_deep_emit", C.c_float), ("ms_deep_dedup", C.c_float),
                ("ms_deep_select", C.c_float), ("pad_deep", C.c_float), ("deep_fuse_bytes", C.c_uint64), ("ms_deep_fuse_prep", C.c_float),
                ("ms_deep_fuse_replay", C.c_float), ("ms_deep_fuse_rerank", C.c_float), ("ms_deep_fuse_sort", C.c_float)]


def _ptr(a: Optional[np.ndarray], typ):
    if a is None:
        return C.cast(None, typ)
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(typ)


@dataclass
class FlatField:
    """One string field in the flattened posting form shared by the oracle and tsgpu_index_load_field."""
    list_off: np.ndarray      # u64 [L+1]
    ids: np.ndarray           # u32
    pos_off: np.ndarray       # u64 [P+1]
    positions: np.ndarray     # u32
    is_array: bool = False

    @property
    def n_lists(self) -> int:
        return len(self.list_off) - 1

    def df(self, l: int) -> int:
        return int(self.list_off[l + 1] - self.list_off[l])

    def struct(self) -> FieldStruct:
        s = FieldStruct()
        s.n_lists = self.n_lists
        s.is_array = 1 if self.is_array else 0
        s.list_off = _ptr(self.list_off, u64p)
        s.ids = _ptr(self.ids, u32p)
        s.pos_off = _ptr(self.pos_off, u64p)
        s.positions = _ptr(self.positions, u32p)
        return s

    @staticmethod
    def from_postings(lists: Sequence[Sequence], is_array: bool = False) -> "FlatField":
        """lists[t] = [(seq_id, [raw offsets...]), ...] ascending seq_id."""
        list_off = [0]
        ids: List[int] = []
        pos_off = [0]
        positions: List[int] = []
        for pl in lists:
            for sid, offs in pl:
                ids.append(sid)
                positions.extend(offs)
                pos_off.append(len(positions))
            list_off.append(len(ids))
        return FlatField(np.asarray(list_off, np.uint64), np.asarray(ids, np.uint32),
                         np.asarray(pos_off, np.uint64), np.asarray(positions, np.uint32), is_array)


@dataclass
class Combo:
    rows: List[List[int]]                 # rows[r][f] = list id or NO_LIST; required rows first, then dropped
    n_required: int
    total_cost: int = 0
    flags: int = 0
    syn_orig_num_tokens: int = -1
    orig_num_tokens: int = -1


@dataclass
class Query:
    combos: List[Combo]
    topk: int = 250
    filter: int = -1                       # inline filter slot (>=0), persistent handle (<=-2 encoded) or -1
    excl: Sequence[int] = ()
    sort: Sequence[tuple] = ((SORT_TEXT_MATCH, -1, 1, 0), (SORT_NONE, -1, 1, 0), (SORT_NONE, -1, 1, 0))
    flags: int = FLAG_PRIORITIZE_EXACT_MATCH
    match_type: int = MATCH_MAX_SCORE
    num_query_tokens: Optional[int] = None
    field_weight: Optional[Sequence[int]] = None


class KwBatch:
    """Flattens Query objects into the SoA arrays of tsgpu_kw_batch and keeps them alive."""

    def __init__(self, queries: Sequence[Query], field_ids: Sequence[int], filters: Sequence[np.ndarray] = ()):
        F = len(field_ids)
        nq = len(queries)
        self.n_queries, self.n_fields = nq, F
        self.queries = list(queries)
        self.field_ids = np.asarray(field_ids, np.uint32)
        q_combo_off = [0]
        q_excl_off = [0]
        excl: List[int] = []
        c_tok_off = [0]
        c_cost, c_nreq, c_flags, c_syn, c_orig = [], [], [], [], []
        t_list: List[int] = []
        self.q_filter = np.zeros(nq, np.int32)
        self.q_topk = np.zeros(nq, np.uint32)
        self.q_sort_type = np.zeros(nq * 3, np.uint8)
        self.q_sort_col = np.zeros(nq * 3, np.int32)
        self.q_sort_order = np.ones(nq * 3, np.int8)
        self.q_sort_missing_first = np.zeros(nq * 3, np.uint8)
        self.q_flags = np.zeros(nq, np.uint8)
        self.q_match_type = np.zeros(nq, np.uint8)
        self.q_num_query_tokens = np.zeros(nq, np.uint8)
        self.q_field_weight = np.zeros(nq * F, np.uint8)
        for qi, q in enumerate(queries):
            for c in q.combos:
                for row in c.rows:
                    assert len(row) == F
                    t_list.extend(row)
                c_tok_off.append(c_tok_off[-1] + len(c.rows))
                c_cost.append(c.total_cost); c_nreq.append(c.n_required); c_flags.append(c.flags)
                c_syn.append(c.syn_orig_num_tokens); c_orig.append(c.orig_num_tokens)
            q_combo_off.append(q_combo_off[-1] + len(q.combos))
            excl.extend(sorted(q.excl))
            q_excl_off.append(len(excl))
            self.q_filter[qi] = q.filter
            self.q_topk[qi] = q.topk
            for i, (ty, col, order, mf) in enumerate(q.sort):
                self.q_sort_type[qi * 3 + i] = ty
                self.q_sort_col[qi * 3 + i] = col
                self.q_sort_order[qi * 3 + i] = order
                self.q_sort_missing_first[qi * 3 + i] = mf
            self.q_flags[qi] = q.flags
            self.q_match_type[qi] = q.match_type
            nqt = q.num_query_tokens
            if nqt is None:
                nqt = q.combos[0].n_required if q.combos else 0
            self.q_num_query_tokens[qi] = nqt
            fw = q.field_weight if q.field_weight is not None else [max(0, 15 - f) for f in range(F)]
            self.q_field_weight[qi * F:(qi + 1) * F] = fw
        self.n_combos = len(c_cost)
        self.q_combo_off = np.asarray(q_combo_off, np.uint32)
        self.q_excl_off = np.asarray(q_excl_off, np.uint32)
        self.excl_ids = np.asarray(excl if excl else [0], np.uint32)
        self.c_tok_off = np.asarray(c_tok_off, np.uint32)
        self.c_total_cost = np.asarray(c_cost if c_cost else [0], np.uint32)
        self.c_n_required = np.asarray(c_nreq if c_nreq else [0], np.uint8)
        self.c_flags = np.asarray(c_flags if c_flags else [0], np.uint8)
        self.c_syn = np.asarray(c_syn if c_syn else [-1], np.int32)
        self.c_orig = np.asarray(c_orig if c_orig else [-1], np.int32)
        self.t_list = np.asarray(t_list if t_list else [NO_LIST], np.uint32)
        self.set_filters(filters)

    def set_filters(self, filters: Sequence[np.ndarray]):
        self.n_filters = len(filters)
        off = [0]
        for f in filters:
            off.append(off[-1] + len(f))
        self.filter_off = np.asarray(off, np.uint64)
        self.filter_ids = (np.concatenate([np.asarray(f, np.uint32) for f in filters]) if filters and off[-1] > 0
                           else np.zeros(1, np.uint32))

    def with_filter_handles(self, handles: Sequence[int]) -> "KwBatch":
        """Shallow copy whose inline filter slots are replaced by persistent filter handles (tsgpu_filter_create)."""
        import copy
        b = copy.copy(self)
        h = np.asarray(list(handles) + [0], np.int32)
        b.q_filter = np.where(self.q_filter >= 0, h[np.clip(self.q_filter, 0, len(h) - 1)], self.q_filter).astype(np.int32)
        b.set_filters([])
        return b

    def head(self, n: int) -> "KwBatch":
        """First n queries (shares the per-combination / per-row arrays)."""
        import copy
        b = copy.copy(self)
        b.n_queries = n
        b.n_combos = int(self.q_combo_off[n])
        return b

    def struct(self) -> KwBatchStruct:
        s = KwBatchStruct()
        s.n_queries, s.n_combos, s.n_fields, s.n_filters = self.n_queries, self.n_combos, self.n_fields, self.n_filters
        s.field_ids = _ptr(self.field_ids, u32p)
        s.q_combo_off = _ptr(self.q_combo_off, u32p)
        s.q_filter = _ptr(self.q_filter, i32p)
        s.q_excl_off = _ptr(self.q_excl_off, u32p)
        s.excl_ids = _ptr(self.excl_ids, u32p)
        s.q_topk = _ptr(self.q_topk, u32p)
        s.q_sort_type = _ptr(self.q_sort_type, u8p)
        s.q_sort_col = _ptr(self.q_sort_col, i32p)
        s.q_sort_order = _ptr(self.q_sort_order, i8p)
        s.q_sort_missing_first = _ptr(self.q_sort_missing_first, u8p)
        s.q_flags = _ptr(self.q_flags, u8p)
        s.q_match_type = _ptr(self.q_match_type, u8p)
        s.q_num_query_tokens = _ptr(self.q_num_query_tokens, u8p)
        s.q_field_weight = _ptr(self.q_field_weight, u8p)
        s.c_tok_off = _ptr(self.c_tok_off, u32p)
        s.c_total_cost = _ptr(self.c_total_cost, u32p)
        s.c_n_required = _ptr(self.c_n_required, u8p)
        s.c_flags = _ptr(self.c_flags, u8p)
        s.c_syn_orig_num_tokens = _ptr(self.c_syn, i32p)
        s.c_orig_num_tokens = _ptr(self.c_orig, i32p)
        s.t_list = _ptr(self.t_list, u32p)
        s.filter_off = _ptr(self.filter_off, u64p)
        s.filter_ids = _ptr(self.filter_ids, u32p)
        return s


@dataclass
class HnswGraph:
    vectors: np.ndarray          # f32 [n, dim]
    levels: np.ndarray           # u8 [n]
    links0: np.ndarray           # u32 [n*(2M+1)]
    upper_off: np.ndarray        # u64 [n+1]
    links_up: np.ndarray         # u32
    M: int
    max_level: int
    entry_point: int
    metric: int = 0
    labels: Optional[np.ndarray] = None

    def struct(self) -> HnswStruct:
        s = HnswStruct()
        n, dim = self.vectors.shape
        s.n_nodes, s.dim, s.M, s.max_level = n, dim, self.M, self.max_level
        s.entry_point, s.metric = self.entry_point, self.metric
        s.vectors = _ptr(self.vectors, f32p)
        if self.labels is None:
            self.labels = np.arange(n, dtype=np.uint32)
        s.labels = _ptr(self.labels, u32p)
        s.levels = _ptr(self.levels, u8p)
        s.links0 = _ptr(self.links0, u32p)
        s.upper_off = _ptr(self.upper_off, u64p)
        s.links_up = _ptr(self.links_up, u32p)
        return s


VEC_FLAT_TENSOR = 1
VEC_DEEP_TOPSTER = 2          # q_topk > MAX_TOPK (with FLAG_DEEP_TOPSTER) and hybrid k up to 4096 in the vector / hybrid calls


def vec_params(k=0, ef=10, flat_search_cutoff=0, distance_threshold=3.4028234663852886e38, alpha=0.3, fetch_size=10, flags=0):
    s = VecParamsStruct()
    s.flags = flags
    s.k, s.ef, s.flat_search_cutoff = k, ef, flat_search_cutoff
    s.distance_threshold, s.alpha, s.fetch_size = distance_threshold, alpha, fetch_size
    return s
