"""ctypes binding of libtsgpu.so (include/tsgpu.h) — harness side.

Importing this module never falls back to a CPU implementation: if the shared library is missing it raises, and on a
machine without a CUDA device every call returns TSGPU_ERR_NO_DEVICE.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence

import numpy as np

from .structs import (ArtStruct, FieldStruct, FlatField, HnswGraph, HnswStruct, KV_DTYPE, KwBatch, KwBatchStruct, StatsStruct,
                      VecParamsStruct, f32p, i32p, u32p, u64p)

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("TSGPU_LIB_PATH") or os.path.join(HERE, "libtsgpu.so")   # override: A/B builds only

EXPORTS = [
    "tsgpu_last_error", "tsgpu_device_count", "tsgpu_host_alloc", "tsgpu_host_free", "tsgpu_index_create", "tsgpu_index_destroy", "tsgpu_index_load_field",
    "tsgpu_index_load_sort_column", "tsgpu_index_append_lists", "tsgpu_index_set_sort_values", "tsgpu_index_load_hnsw", "tsgpu_index_build_hnsw", "tsgpu_index_append_hnsw", "tsgpu_index_mark_deleted", "tsgpu_index_hnsw_info", "tsgpu_index_export_hnsw", "tsgpu_filter_create", "tsgpu_filter_destroy", "tsgpu_filter_numeric", "tsgpu_filter_combine", "tsgpu_filter_ids", "tsgpu_scored_ids_search_batch",
    "tsgpu_intersect", "tsgpu_contains_atleast_one", "tsgpu_phrase_matches", "tsgpu_exact_matches", "tsgpu_prefix_matches", "tsgpu_ids_setop", "tsgpu_keyword_search_batch", "tsgpu_wildcard_search_batch", "tsgpu_knn_batch", "tsgpu_flat_distances", "tsgpu_flat_distances_batch",
    "tsgpu_vector_search_batch", "tsgpu_hybrid_search_batch", "tsgpu_get_stats", "tsgpu_debug_knn_work", "tsgpu_comm_unique_id", "tsgpu_comm_init", "tsgpu_comm_destroy", "tsgpu_comm_gather", "tsgpu_comm_last_ms", "tsgpu_hybrid_fuse_batch", "tsgpu_index_load_facet", "tsgpu_facet_counts", "tsgpu_facet_counts_last", "tsgpu_all_result_ids_last", "tsgpu_index_load_art", "tsgpu_art_walk_batch",
    "tsgpu_index_compact_field", "tsgpu_index_reserve_docs", "tsgpu_index_field_info", "tsgpu_debug_field_array", "tsgpu_diversify_batch",
]


class FieldInfoStruct(C.Structure):
    """tsgpu_field_info"""
    _fields_ = [("n_lists", C.c_uint32), ("flags", C.c_uint32), ("n_postings", C.c_uint64), ("n_positions", C.c_uint64), ("n_blocks", C.c_uint64),
                ("n_words", C.c_uint64), ("n_dense", C.c_uint32), ("dense_words", C.c_uint32), ("device_bytes", C.c_uint64)]


class DivMetricStruct(C.Structure):
    """tsgpu_div_metric: facet id (NO_LIST: use sort_col), sort column, TSGPU_DIV_* method, weight"""
    _fields_ = [("facet", C.c_uint32), ("sort_col", C.c_int32), ("method", C.c_uint32), ("weight", C.c_float)]


NO_LIST = 0xFFFFFFFF
DIV_EQUALITY, DIV_JACCARD = 0, 1
MAX_DIV_METRICS = 16
FIELD_IS_ARRAY, FIELD_PLAIN_OK, FIELD_POS16 = 1, 2, 4
# tsgpu_debug_field_array slots: name and element type
FIELD_ARRAYS = [("list_off", np.uint64), ("list_blk_off", np.uint32), ("blk_first", np.uint32), ("blk_info", np.uint64), ("packed", np.uint32),
                ("pos_off", np.uint64), ("positions", np.uint32), ("list_dense", np.uint32), ("dense_bits", np.uint32), ("dense_rank", np.uint32)]
FACET_DTYPE = np.dtype([("value_id", np.uint32), ("count", np.uint32), ("doc_id", np.uint32), ("array_pos", np.uint32)])
QFLAG_KEEP_ALL_IDS = 0x80
QFLAG_DEEP_TOPSTER = 0x20       # q_topk may exceed MAX_TOPK (tsgpu_keyword / wildcard / scored_ids_search_batch)
MAX_TOPK = 1024
VEC_DEEP_TOPSTER = 2            # tsgpu_vec_params::flags: the vector / hybrid calls accept QFLAG_DEEP_TOPSTER (deep fusion)


class TsgpuError(RuntimeError):
    pass


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise TsgpuError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                             "(there is no CPU fallback)")
        _lib = declare(C.CDLL(LIB_PATH))
    return _lib


def declare(L):
    """Argument types of every tsgpu_* entry point on a loaded library (libtsgpu.so itself, or one that re-exports it: the C++
    host layer's wrapper, the test double)."""
    if True:
        vp = C.c_void_p
        L.tsgpu_last_error.restype = C.c_char_p
        L.tsgpu_index_create.argtypes = [C.c_uint32, C.c_int, C.POINTER(vp)]
        L.tsgpu_index_destroy.argtypes = [vp]
        L.tsgpu_index_load_field.argtypes = [vp, C.POINTER(FieldStruct), u32p]
        L.tsgpu_index_load_sort_column.argtypes = [vp, C.c_void_p, u32p]
        L.tsgpu_index_append_lists.argtypes = [vp, C.c_uint32, C.POINTER(FieldStruct), u32p]
        L.tsgpu_index_set_sort_values.argtypes = [vp, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t]
        # the mirror maintenance calls: libtsgpu.so always has them; a library that re-exports an older C-ABI (the base test
        # double, the host layer linked against it) may not, and then only calling them fails
        for name, args in (("tsgpu_index_compact_field", [vp, C.c_uint32, C.c_void_p, C.c_uint32]), ("tsgpu_index_reserve_docs", [vp, C.c_uint32]),
                           ("tsgpu_index_field_info", [vp, C.c_uint32, C.POINTER(FieldInfoStruct)]),
                           ("tsgpu_debug_field_array", [vp, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)])):
            if hasattr(L, name):
                getattr(L, name).argtypes = args
        if hasattr(L, "tsgpu_diversify_batch"):      # absent from the base test double
            L.tsgpu_diversify_batch.argtypes = [vp, C.POINTER(DivMetricStruct), C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                                C.c_void_p, C.c_void_p]
        L.tsgpu_index_load_hnsw.argtypes = [vp, C.POINTER(HnswStruct)]
        L.tsgpu_index_build_hnsw.argtypes = [vp, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int]
        L.tsgpu_index_append_hnsw.argtypes = [vp, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
        L.tsgpu_index_mark_deleted.argtypes = [vp, C.c_void_p, C.c_size_t, C.c_int]
        L.tsgpu_index_hnsw_info.argtypes = [vp, u32p, u32p, u32p, u32p, u32p, u64p, u64p]
        L.tsgpu_index_export_hnsw.argtypes = [vp, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.tsgpu_filter_create.argtypes = [vp, C.c_void_p, C.c_size_t, i32p]
        L.tsgpu_filter_destroy.argtypes = [vp, C.c_int32]
        L.tsgpu_filter_numeric.argtypes = [vp, C.c_uint32, C.c_int, C.c_int64, C.c_int64, i32p, C.POINTER(C.c_size_t)]
        L.tsgpu_filter_combine.argtypes = [vp, C.c_int, C.c_int32, C.c_int32, i32p, C.POINTER(C.c_size_t)]
        L.tsgpu_filter_ids.argtypes = [vp, C.c_int32, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.tsgpu_scored_ids_search_batch.argtypes = [vp, C.POINTER(KwBatchStruct), C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        L.tsgpu_intersect.argtypes = [vp, C.c_uint32, u32p, C.c_uint32, u32p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.tsgpu_contains_atleast_one.argtypes = [vp, C.c_uint32, C.c_uint32, u32p, C.c_size_t, C.POINTER(C.c_int)]
        L.tsgpu_ids_setop.argtypes = [vp, C.c_int, u32p, C.c_size_t, u32p, C.c_size_t, u32p, C.c_size_t, C.POINTER(C.c_size_t)]
        for n in ("tsgpu_phrase_matches", "tsgpu_exact_matches", "tsgpu_prefix_matches"):
            getattr(L, n).argtypes = [vp, C.c_uint32, u32p, C.c_uint32, u32p, C.c_size_t, u32p, C.POINTER(C.c_size_t)]
        L.tsgpu_keyword_search_batch.argtypes = [vp, C.POINTER(KwBatchStruct), C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        L.tsgpu_wildcard_search_batch.argtypes = [vp, C.POINTER(KwBatchStruct), C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        L.tsgpu_knn_batch.argtypes = [vp, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, i32p, C.c_uint32, u64p, u32p,
                                      C.c_void_p, C.c_void_p, C.c_void_p]
        L.tsgpu_flat_distances.argtypes = [vp, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        L.tsgpu_flat_distances_batch.argtypes = [vp, C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p]
        for n in ("tsgpu_vector_search_batch", "tsgpu_hybrid_search_batch"):
            getattr(L, n).argtypes = [vp, C.POINTER(KwBatchStruct), C.c_void_p, C.POINTER(VecParamsStruct), C.c_void_p,
                                      C.c_uint32, C.c_void_p, C.c_void_p]
        L.tsgpu_get_stats.argtypes = [vp, C.POINTER(StatsStruct)]
        L.tsgpu_comm_unique_id.argtypes = [C.c_void_p]
        L.tsgpu_comm_init.argtypes = [vp, C.c_int, C.c_int, C.c_void_p]
        L.tsgpu_comm_destroy.argtypes = [vp]
        L.tsgpu_comm_gather.argtypes = [vp, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int]
        L.tsgpu_comm_last_ms.argtypes = [vp, C.POINTER(C.c_float)]
        L.tsgpu_index_load_facet.argtypes = [vp, C.c_void_p, u32p]
        L.tsgpu_facet_counts.argtypes = [vp, C.c_uint32, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_void_p, u32p, u32p]
        L.tsgpu_facet_counts_last.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.tsgpu_all_result_ids_last.argtypes = [vp, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.tsgpu_debug_knn_work.argtypes = [vp, C.c_void_p, C.c_uint32, u32p]
        L.tsgpu_index_load_art.argtypes = [vp, C.c_uint32, C.POINTER(ArtStruct)]
        L.tsgpu_art_walk_batch.argtypes = [vp, C.c_uint32, C.c_uint32, u32p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                           u32p, C.c_void_p]
    return L


def _ck(rc: int):
    if rc != 0:
        raise TsgpuError(f"tsgpu status {rc}: {lib().tsgpu_last_error().decode()}")


def _addr(x):
    """numpy array / torch tensor (cpu, pinned or cuda) / int -> raw address."""
    if x is None:
        return None
    if isinstance(x, np.ndarray):
        assert x.flags["C_CONTIGUOUS"]
        return x.ctypes.data
    if hasattr(x, "data_ptr"):
        assert x.is_contiguous()
        return x.data_ptr()
    return int(x)


class GpuIndex:
    """Device mirror of one Typesense Index (postings, sort columns, HNSW graph + vectors) behind the C-ABI."""

    def __init__(self, n_docs: int, device: int = 0):
        self.L = lib()
        self.h = C.c_void_p()
        _ck(self.L.tsgpu_index_create(n_docs, device, C.byref(self.h)))
        self.n_docs = n_docs
        self._keep = []

    @classmethod
    def from_handle(cls, handle, n_docs: int, library=None) -> "GpuIndex":
        """A view over an index somebody else owns (the C++ host layer's): same calls, never destroyed from here."""
        g = cls.__new__(cls)
        g.L = library if library is not None else lib()
        g.h = C.c_void_p(handle)
        g.n_docs = n_docs
        g._keep = []
        g._borrowed = True
        return g

    def close(self):
        if self.h and not getattr(self, "_borrowed", False):
            self.L.tsgpu_index_destroy(self.h)
        self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- mirror loading
    def load_field(self, f: FlatField) -> int:
        s = f.struct()
        out = C.c_uint32(0)
        _ck(self.L.tsgpu_index_load_field(self.h, C.byref(s), C.byref(out)))
        return out.value

    def append_lists(self, field: int, f: FlatField) -> int:
        """tsgpu_index_append_lists (f-4): the current full lists of the tokens a batch of writes touched; returns the first new list id."""
        s = f.struct()
        out = C.c_uint32(0)
        _ck(self.L.tsgpu_index_append_lists(self.h, field, C.byref(s), C.byref(out)))
        return out.value

    def set_sort_values(self, col: int, ids, vals):
        ids = np.ascontiguousarray(ids, np.uint32)
        vals = np.ascontiguousarray(vals, np.int64)
        _ck(self.L.tsgpu_index_set_sort_values(self.h, col, ids.ctypes.data, vals.ctypes.data, len(ids)))

    def compact_field(self, field: int, live_lists) -> None:
        """tsgpu_index_compact_field: keep only `live_lists` (list live_lists[i] becomes list i) and free the rest."""
        a = np.ascontiguousarray(live_lists, np.uint32)
        _ck(self.L.tsgpu_index_compact_field(self.h, field, a.ctypes.data if len(a) else None, len(a)))

    def reserve_docs(self, n_docs: int) -> None:
        """tsgpu_index_reserve_docs: raise the seq_id capacity."""
        _ck(self.L.tsgpu_index_reserve_docs(self.h, n_docs))
        self.n_docs = n_docs

    def diversify(self, metrics, lambdas, kv, count, out=None, stride=None):
        """tsgpu_diversify_batch: each query's records kv[q, :count[q]] in MMR order. metrics: (facet id or None, sort column, method,
        weight) tuples; lambdas: one per query. kv / out: numpy [nq, stride] KV_DTYPE arrays, or CUDA tensors holding such
        records (then `stride` gives the records per row). Returns `out` (a new array when kv is a numpy array and out is None)."""
        m = (DivMetricStruct * max(1, len(metrics)))()
        for i, (facet, col, method, weight) in enumerate(metrics):
            m[i].facet = NO_LIST if facet is None else facet
            m[i].sort_col, m[i].method, m[i].weight = col, method, weight
        cnt = np.ascontiguousarray(count, np.uint32)
        lam = np.ascontiguousarray(lambdas, np.float32)
        if isinstance(kv, np.ndarray):
            stride = kv.shape[1]
            if out is None:
                out = np.zeros_like(kv)
        _ck(self.L.tsgpu_diversify_batch(self.h, m, len(metrics), len(cnt), lam.ctypes.data, _addr(kv), stride, cnt.ctypes.data, _addr(out)))
        return out

    def field_info(self, field: int) -> dict:
        s = FieldInfoStruct()
        _ck(self.L.tsgpu_index_field_info(self.h, field, C.byref(s)))
        return {n: getattr(s, n) for n, _ in FieldInfoStruct._fields_}

    def field_array(self, field: int, slot: int) -> np.ndarray:
        """tsgpu_debug_field_array: one of the field's ten device arrays (FIELD_ARRAYS) over its logical length."""
        n = C.c_size_t(0)
        rc = self.L.tsgpu_debug_field_array(self.h, field, slot, None, 0, C.byref(n))
        if rc not in (0, 4):
            _ck(rc)
        out = np.zeros(max(n.value, 8), np.uint8)
        _ck(self.L.tsgpu_debug_field_array(self.h, field, slot, out.ctypes.data, len(out), C.byref(n)))
        return out[:n.value].view(FIELD_ARRAYS[slot][1]).copy()

    def load_field_raw(self, n_lists: int, is_array: bool, list_off, ids, pos_off, positions) -> int:
        """Pointers may be torch CUDA tensors (device-resident synthetic data)."""
        s = FieldStruct()
        s.n_lists, s.is_array = n_lists, int(is_array)
        s.list_off = C.cast(_addr(list_off), u64p)
        s.ids = C.cast(_addr(ids), u32p)
        s.pos_off = C.cast(_addr(pos_off), u64p)
        s.positions = C.cast(_addr(positions), u32p)
        out = C.c_uint32(0)
        _ck(self.L.tsgpu_index_load_field(self.h, C.byref(s), C.byref(out)))
        return out.value

    def load_sort_column(self, vals) -> int:
        if isinstance(vals, np.ndarray):
            vals = np.ascontiguousarray(vals, np.int64)
        out = C.c_uint32(0)
        _ck(self.L.tsgpu_index_load_sort_column(self.h, _addr(vals), C.byref(out)))
        return out.value

    def load_hnsw(self, g: HnswGraph):
        s = g.struct()
        _ck(self.L.tsgpu_index_load_hnsw(self.h, C.byref(s)))

    def load_hnsw_raw(self, n, dim, M, max_level, entry_point, metric, vectors, levels, links0, upper_off, links_up):
        s = HnswStruct()
        s.n_nodes, s.dim, s.M, s.max_level, s.entry_point, s.metric = n, dim, M, max_level, entry_point, metric
        s.vectors = C.cast(_addr(vectors), f32p)
        s.labels = C.cast(None, u32p)
        s.levels = C.cast(_addr(levels), C.POINTER(C.c_uint8))
        s.links0 = C.cast(_addr(links0), u32p)
        s.upper_off = C.cast(_addr(upper_off), u64p)
        s.links_up = C.cast(_addr(links_up), u32p)
        _ck(self.L.tsgpu_index_load_hnsw(self.h, C.byref(s)))

    def build_hnsw(self, vectors, M=16, ef_construction=200, seed=100, metric=0, max_batch=4096, keep_device_vectors=False) -> dict:
        """tsgpu_index_build_hnsw: hnswlib's addPoint as batched rounds on the device. `vectors`: numpy [n, dim] f32 or a CUDA
        tensor. Returns the graph's shape and the build counters."""
        if isinstance(vectors, np.ndarray):
            vectors = np.ascontiguousarray(vectors, np.float32)
        n, dim = int(vectors.shape[0]), int(vectors.shape[1])
        _ck(self.L.tsgpu_index_build_hnsw(self.h, _addr(vectors), n, dim, M, ef_construction, seed, metric, max_batch, 1 if keep_device_vectors else 0))
        if keep_device_vectors:
            self._keep_vectors = vectors
        return self.hnsw_info()

    def append_hnsw(self, vectors, ef_construction=200, seed=100, max_batch=4096) -> dict:
        """tsgpu_index_append_hnsw: addPoint for more vectors into the graph the index holds (labels continue)."""
        if isinstance(vectors, np.ndarray):
            vectors = np.ascontiguousarray(vectors, np.float32)
        _ck(self.L.tsgpu_index_append_hnsw(self.h, _addr(vectors), int(vectors.shape[0]), ef_construction, seed, max_batch))
        return self.hnsw_info()

    def mark_deleted(self, labels, deleted=True):
        """tsgpu_index_mark_deleted: hnswlib's markDelete / unmarkDelete."""
        l = np.ascontiguousarray(labels, np.uint32)
        _ck(self.L.tsgpu_index_mark_deleted(self.h, l.ctypes.data, len(l), 1 if deleted else 0))

    def hnsw_info(self) -> dict:
        v = [C.c_uint32(0) for _ in range(5)]
        nup = C.c_uint64(0)
        bc = (C.c_uint64 * 5)()
        _ck(self.L.tsgpu_index_hnsw_info(self.h, *[C.byref(x) for x in v], C.byref(nup), bc))
        return {"n": v[0].value, "dim": v[1].value, "M": v[2].value, "max_level": v[3].value, "entry_point": v[4].value, "n_upper": nup.value,
                "build": {"search_dist": bc[0], "expanded": bc[1], "heuristic_dist": bc[2], "rows_reselected": bc[3], "rounds": bc[4]}}

    def export_hnsw(self, vectors: np.ndarray, metric: int = 0) -> HnswGraph:
        """The device graph as host arrays (the form the oracle walks)."""
        i = self.hnsw_info()
        n, M = i["n"], i["M"]
        levels = np.zeros(max(n, 1), np.uint8)[:n]
        links0 = np.zeros(n * (2 * M + 1), np.uint32)
        upper_off = np.zeros(n + 1, np.uint64)
        links_up = np.zeros(max(i["n_upper"] * (M + 1), 1), np.uint32)
        _ck(self.L.tsgpu_index_export_hnsw(self.h, levels.ctypes.data if n else None, links0.ctypes.data if n else None, upper_off.ctypes.data,
                                           links_up.ctypes.data))
        return HnswGraph(np.ascontiguousarray(vectors, np.float32), levels, links0, upper_off, links_up[:i["n_upper"] * (M + 1)] if i["n_upper"] else links_up,
                         M, i["max_level"], i["entry_point"], metric)

    def filter_create(self, ids) -> int:
        if isinstance(ids, np.ndarray):
            ids = np.ascontiguousarray(ids, np.uint32)
        n = int(ids.shape[0]) if hasattr(ids, "shape") else len(ids)
        out = C.c_int32(0)
        _ck(self.L.tsgpu_filter_create(self.h, _addr(ids) if n else None, n, C.byref(out)))
        return out.value

    # ---- filter_by on the device (SURVEY 8 f-2)
    CMP = {"=": 0, "!=": 1, "<": 2, "<=": 3, ">": 4, ">=": 5, "range": 6}

    def filter_numeric(self, col: int, op: str, v1: int, v2: int = 0):
        """A numeric / bool leaf evaluated over the mirrored column: (handle, number of docs)."""
        h, n = C.c_int32(0), C.c_size_t(0)
        _ck(self.L.tsgpu_filter_numeric(self.h, col, self.CMP[op], int(v1), int(v2), C.byref(h), C.byref(n)))
        return h.value, n.value

    def filter_combine(self, op: int, a: int, b: int):
        h, n = C.c_int32(0), C.c_size_t(0)
        _ck(self.L.tsgpu_filter_combine(self.h, op, a, b, C.byref(h), C.byref(n)))
        return h.value, n.value

    def filter_ids(self, handle: int, cap: int) -> np.ndarray:
        out = np.zeros(max(cap, 1), np.uint32)
        n = C.c_size_t(0)
        _ck(self.L.tsgpu_filter_ids(self.h, handle, out.ctypes.data, cap, C.byref(n)))
        return out[:n.value]

    # ---- search
    def contains_atleast_one(self, field: int, lst: int, ids) -> bool:
        a = np.ascontiguousarray(ids, np.uint32)
        out = C.c_int(0)
        _ck(self.L.tsgpu_contains_atleast_one(self.h, field, lst, a.ctypes.data_as(u32p), len(a), C.byref(out)))
        return bool(out.value)

    def intersect(self, field: int, lists: Sequence[int], cap: int) -> np.ndarray:
        ls = np.asarray(lists, np.uint32)
        out = np.zeros(max(cap, 1), np.uint32)
        n = C.c_size_t(0)
        _ck(self.L.tsgpu_intersect(self.h, field, ls.ctypes.data_as(u32p), len(ls), out.ctypes.data_as(u32p), cap, C.byref(n)))
        return out[:n.value].copy()

    def phrase_matches(self, field: int, lists: Sequence[int], ids: np.ndarray) -> np.ndarray:
        ls = np.asarray(lists, np.uint32)
        ids = np.ascontiguousarray(ids, np.uint32)
        out = np.zeros(max(len(ids), 1), np.uint32)
        n = C.c_size_t(0)
        _ck(self.L.tsgpu_phrase_matches(self.h, field, ls.ctypes.data_as(u32p), len(ls), ids.ctypes.data_as(u32p), len(ids),
                                        out.ctypes.data_as(u32p), C.byref(n)))
        return out[:n.value].copy()

    def _idset(self, fn, field, lists, ids):
        ls = np.asarray(lists, np.uint32)
        ids = np.ascontiguousarray(ids, np.uint32)
        out = np.zeros(max(len(ids), 1), np.uint32)
        n = C.c_size_t(0)
        _ck(fn(self.h, field, ls.ctypes.data_as(u32p), len(ls), ids.ctypes.data_as(u32p), len(ids), out.ctypes.data_as(u32p), C.byref(n)))
        return out[:n.value].copy()

    def exact_matches(self, field: int, lists: Sequence[int], ids: np.ndarray) -> np.ndarray:
        return self._idset(self.L.tsgpu_exact_matches, field, lists, ids)

    def prefix_matches(self, field: int, lists: Sequence[int], ids: np.ndarray) -> np.ndarray:
        return self._idset(self.L.tsgpu_prefix_matches, field, lists, ids)

    def load_art(self, field: int, root: int, node_first_child, node_n_children, node_partial_len, node_partial, child_byte, child_ref,
                 leaf_key_off, leaf_keys):
        """tsgpu_index_load_art: the flat ART mirror of a field (arrays as art_mirror_t::flatten() gives them)."""
        arrs = [np.ascontiguousarray(node_first_child, np.uint32), np.ascontiguousarray(node_n_children, np.uint16),
                np.ascontiguousarray(node_partial_len, np.uint8), np.ascontiguousarray(node_partial, np.uint8),
                np.ascontiguousarray(child_byte, np.uint8), np.ascontiguousarray(child_ref, np.int32),
                np.ascontiguousarray(leaf_key_off, np.uint64), np.ascontiguousarray(leaf_keys, np.uint8)]
        a = ArtStruct(len(arrs[0]), len(arrs[4]), len(arrs[6]) - 1, root, *[x.ctypes.data if len(x) else None for x in arrs], None, None)
        _ck(self.L.tsgpu_index_load_art(self.h, field, C.byref(a)))

    def art_walk(self, field: int, terms: Sequence[bytes], min_cost: Sequence[int], max_cost: Sequence[int], prefix: Sequence[int], cap: int = 256):
        """tsgpu_art_walk_batch -> (hits per search as lists of refs, flags)"""
        n = len(terms)
        off = np.zeros(n + 1, np.uint32)
        off[1:] = np.cumsum([len(t) for t in terms])
        blob = np.frombuffer(b"".join(terms) + b"\0", np.uint8).copy()
        mn, mx, pf = (np.ascontiguousarray(x, np.uint8) for x in (min_cost, max_cost, prefix))
        hits = np.zeros((max(n, 1), cap), np.int32)
        cnt = np.zeros(max(n, 1), np.uint32)
        flags = np.zeros(max(n, 1), np.uint8)
        _ck(self.L.tsgpu_art_walk_batch(self.h, field, n, off.ctypes.data_as(u32p), blob.ctypes.data, mn.ctypes.data, mx.ctypes.data, pf.ctypes.data,
                                        hits.ctypes.data, cap, cnt.ctypes.data_as(u32p), flags.ctypes.data))
        return [hits[i, :min(int(cnt[i]), cap)].tolist() for i in range(n)], flags[:n].copy()

    def ids_setop(self, op: int, a: np.ndarray, b: np.ndarray) -> np.ndarray:
        """op: 0 and, 1 or, 2 exclude (a minus b)"""
        a = np.ascontiguousarray(a, np.uint32)
        b = np.ascontiguousarray(b, np.uint32)
        cap = max(1, len(a) + len(b))
        out = np.zeros(cap, np.uint32)
        n = C.c_size_t(0)
        _ck(self.L.tsgpu_ids_setop(self.h, op, a.ctypes.data_as(u32p), len(a), b.ctypes.data_as(u32p), len(b),
                                   out.ctypes.data_as(u32p), cap, C.byref(n)))
        return out[:n.value].copy()

    def _outs(self, nq, stride, out):
        if out is None:
            kv = np.zeros((nq, stride), KV_DTYPE)
            cnt = np.zeros(nq, np.uint32)
            found = np.zeros(nq, np.uint32)
            return kv, cnt, found
        return out

    def keyword_search(self, b: KwBatch, stride: int = 256, out=None, bstruct=None):
        kv, cnt, found = self._outs(b.n_queries, stride, out)
        s = bstruct if bstruct is not None else b.struct()
        _ck(self.L.tsgpu_keyword_search_batch(self.h, C.byref(s), _addr(kv), stride, _addr(cnt), _addr(found)))
        return kv, cnt, found

    def wildcard_search(self, b: KwBatch, stride: int = 256, out=None, bstruct=None):
        kv, cnt, found = self._outs(b.n_queries, stride, out)
        s = bstruct if bstruct is not None else b.struct()
        _ck(self.L.tsgpu_wildcard_search_batch(self.h, C.byref(s), _addr(kv), stride, _addr(cnt), _addr(found)))
        return kv, cnt, found

    def vector_search(self, b: KwBatch, qvecs, vp: VecParamsStruct, stride: int = 256, out=None, bstruct=None):
        kv, cnt, found = self._outs(b.n_queries, stride, out)
        if isinstance(qvecs, np.ndarray):
            qvecs = np.ascontiguousarray(qvecs, np.float32)
        s = bstruct if bstruct is not None else b.struct()
        _ck(self.L.tsgpu_vector_search_batch(self.h, C.byref(s), _addr(qvecs), C.byref(vp), _addr(kv), stride, _addr(cnt), _addr(found)))
        return kv, cnt, found

    def hybrid_search(self, b: KwBatch, qvecs, vp: VecParamsStruct, stride: int = 256, out=None, bstruct=None):
        kv, cnt, found = self._outs(b.n_queries, stride, out)
        if isinstance(qvecs, np.ndarray):
            qvecs = np.ascontiguousarray(qvecs, np.float32)
        s = bstruct if bstruct is not None else b.struct()
        _ck(self.L.tsgpu_hybrid_search_batch(self.h, C.byref(s), _addr(qvecs), C.byref(vp), _addr(kv), stride, _addr(cnt), _addr(found)))
        return kv, cnt, found

    def knn(self, queries, k: int, ef: int, q_filter=None, filters=(), out=None):
        if isinstance(queries, np.ndarray):
            queries = np.ascontiguousarray(queries, np.float32)
        nq = int(queries.shape[0])
        if out is None:
            d = np.zeros((nq, k), np.float32)
            l = np.zeros((nq, k), np.uint32)
            n = np.zeros(nq, np.uint32)
        else:
            d, l, n = out
        off = [0]
        for f in filters:
            off.append(off[-1] + len(f))
        foff = np.asarray(off, np.uint64)
        fids = np.concatenate([np.asarray(f, np.uint32) for f in filters]) if filters and off[-1] else np.zeros(1, np.uint32)
        qf = None if q_filter is None else np.ascontiguousarray(q_filter, np.int32)
        _ck(self.L.tsgpu_knn_batch(self.h, _addr(queries), nq, k, ef,
                                   qf.ctypes.data_as(i32p) if qf is not None else C.cast(None, i32p), len(filters),
                                   foff.ctypes.data_as(u64p), fids.ctypes.data_as(u32p), _addr(d), _addr(l), _addr(n)))
        return d, l, n

    def flat_distances(self, query: np.ndarray, ids: np.ndarray) -> np.ndarray:
        q = np.ascontiguousarray(query, np.float32)
        ids = np.ascontiguousarray(ids, np.uint32)
        out = np.zeros(max(len(ids), 1), np.float32)
        _ck(self.L.tsgpu_flat_distances(self.h, q.ctypes.data, ids.ctypes.data, len(ids), out.ctypes.data))
        return out[:len(ids)]

    def flat_distances_batch(self, queries: np.ndarray, ids: np.ndarray) -> np.ndarray:
        """tsgpu_flat_distances_batch: [nq, n] distances of nq queries to one shared candidate set (tensor-core scan)."""
        q = np.ascontiguousarray(queries, np.float32)
        ids = np.ascontiguousarray(ids, np.uint32)
        out = np.zeros((q.shape[0], max(len(ids), 1)), np.float32)
        if len(ids):
            out = np.zeros((q.shape[0], len(ids)), np.float32)
            _ck(self.L.tsgpu_flat_distances_batch(self.h, q.ctypes.data, q.shape[0], ids.ctypes.data, len(ids), out.ctypes.data))
        return out[:, :len(ids)]

    # ---- multi-GPU (SURVEY 8e): the library's own NCCL exchange
    def comm_unique_id(self) -> np.ndarray:
        out = np.zeros(128, np.uint8)
        _ck(self.L.tsgpu_comm_unique_id(out.ctypes.data))
        return out

    def comm_init(self, rank: int, world: int, ident: np.ndarray):
        a = np.ascontiguousarray(ident, np.uint8)
        _ck(self.L.tsgpu_comm_init(self.h, rank, world, a.ctypes.data))

    def comm_destroy(self):
        _ck(self.L.tsgpu_comm_destroy(self.h))

    def comm_gather(self, src, nbytes: int, dst, root: int = 0):
        """src / dst: numpy arrays or torch tensors (host, pinned or device); dst is only read on `root`."""
        _ck(self.L.tsgpu_comm_gather(self.h, _addr(src), nbytes, _addr(dst) if dst is not None else None, root))

    def comm_last_ms(self) -> float:
        v = C.c_float(0)
        _ck(self.L.tsgpu_comm_last_ms(self.h, C.byref(v)))
        return v.value

    # ---- facets (SURVEY 8 f-3)
    def load_facet(self, n_values: int, doc_off, value_ids) -> int:
        class _F(C.Structure):
            _fields_ = [("n_values", C.c_uint32), ("doc_off", C.c_void_p), ("value_ids", C.c_void_p)]
        self._facet_keep = getattr(self, "_facet_keep", []) + [(doc_off, value_ids)]
        f = _F(n_values, _addr(doc_off), _addr(value_ids))
        out = C.c_uint32(0)
        _ck(self.L.tsgpu_index_load_facet(self.h, C.byref(f), C.byref(out)))
        return out.value

    def facet_counts(self, facet: int, ids, top_n: int, sample_mod: int = 0):
        a = np.ascontiguousarray(ids, np.uint32)
        out = np.zeros(top_n, FACET_DTYPE)
        n, dis = C.c_uint32(0), C.c_uint32(0)
        _ck(self.L.tsgpu_facet_counts(self.h, facet, a.ctypes.data if len(a) else None, len(a), sample_mod, top_n, out.ctypes.data, C.byref(n), C.byref(dis)))
        return out[:n.value], dis.value

    def facet_counts_last(self, facet: int, nq: int, top_n: int):
        out = np.zeros((nq, top_n), FACET_DTYPE)
        n, dis = np.zeros(nq, np.uint32), np.zeros(nq, np.uint32)
        _ck(self.L.tsgpu_facet_counts_last(self.h, facet, top_n, out.ctypes.data, n.ctypes.data, dis.ctypes.data))
        return out, n, dis

    def all_result_ids_last(self, q: int, cap: int) -> np.ndarray:
        out = np.zeros(max(cap, 1), np.uint32)
        n = C.c_size_t(0)
        _ck(self.L.tsgpu_all_result_ids_last(self.h, q, out.ctypes.data, cap, C.byref(n)))
        return out[:n.value]

    def knn_work(self, nq: int) -> np.ndarray:
        """[(expanded nodes, distance evaluations)] of every graph walk of the last call (instrumentation)."""
        out = np.zeros((nq, 2), np.uint32)
        n = C.c_uint32(0)
        _ck(self.L.tsgpu_debug_knn_work(self.h, out.ctypes.data, nq, C.byref(n)))
        return out[:n.value]

    def stats(self) -> dict:
        s = StatsStruct()
        _ck(self.L.tsgpu_get_stats(self.h, C.byref(s)))
        return {n: getattr(s, n) for n, _ in StatsStruct._fields_}
