"""ctypes binding of the C++ host layer's C wrapper (typesense_b200/host/tshost_capi.cpp) — harness side.

libtshost.so is the host layer (tsgpu_host.hpp: tokens -> candidate walks -> typo / prefix / drop-token control flow -> device
rounds shared by a whole multi_search) linked against libtsgpu.so: the code path a server-side binding takes. The same source
linked against the oracle-backed test double of the C-ABI (tests/cpp) is the CPU arm of bench.py and of the CPU test runs;
this module loads whichever library it is pointed at."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Optional, Sequence

import numpy as np

from . import capi
from .structs import KV_DTYPE

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_GPU = os.path.join(HERE, "libtshost.so")
# tsgpu_kw_batch::q_flags bit the host layer sets when a keyword, wildcard or phrase-only search's topster_size exceeds
# capi.MAX_TOPK (deep pagination); vector and hybrid searches stay at MAX_TOPK unless Options.vec_flags has VEC_DEEP_TOPSTER
QFLAG_DEEP_TOPSTER = capi.QFLAG_DEEP_TOPSTER
VEC_DEEP_TOPSTER = capi.VEC_DEEP_TOPSTER


def build_gpu_lib(force: bool = False) -> str:
    """g++ the wrapper against the in-tree libtsgpu.so (host code only: no nvcc needed)."""
    src = os.path.join(HERE, "host", "tshost_capi.cpp")
    deps = [src, os.path.join(HERE, "host", "tsgpu_host.hpp"), os.path.join(HERE, "host", "art_mirror.hpp"), os.path.join(ROOT, "include", "tsgpu.h")]
    if force or not os.path.exists(LIB_GPU) or any(os.path.getmtime(d) > os.path.getmtime(LIB_GPU) for d in deps):
        tmp = LIB_GPU + ".tmp"
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", src, "-o", tmp, "-L", HERE, "-l:libtsgpu.so", "-Wl,-rpath,$ORIGIN", "-pthread"])
        os.replace(tmp, LIB_GPU)
    return LIB_GPU


class Options(C.Structure):
    """tshost_options: Collection::search defaults of the typo / prefix machinery + the vector query's parameters."""
    _fields_ = [("num_typos", C.c_uint32), ("prefix", C.c_uint32), ("max_candidates", C.c_uint32), ("typo_tokens_threshold", C.c_uint32),
                ("drop_tokens_threshold", C.c_uint32), ("topster_size", C.c_uint32), ("device_art_walk", C.c_uint32), ("n_threads", C.c_uint32),
                ("vec_k", C.c_uint32), ("vec_ef", C.c_uint32), ("vec_flat_search_cutoff", C.c_uint32), ("vec_fetch_size", C.c_uint32),
                ("vec_alpha", C.c_float), ("vec_distance_threshold", C.c_float), ("vec_flags", C.c_uint32)]

    def __init__(self, **kw):
        super().__init__(num_typos=2, prefix=1, max_candidates=4, typo_tokens_threshold=1, drop_tokens_threshold=1, topster_size=250, device_art_walk=1,
                         n_threads=0, vec_k=0, vec_ef=10, vec_flat_search_cutoff=0, vec_fetch_size=10, vec_alpha=0.3, vec_distance_threshold=3.4028234663852886e38,
                         vec_flags=0)
        for k, v in kw.items():
            setattr(self, k, v)


class Stats(C.Structure):
    _fields_ = ([(n, C.c_uint64) for n in ("passes", "kw_batches", "kw_queries", "walk_batches", "walks", "host_walk_fallbacks", "fuse_queries")] +
                [(n, C.c_double) for n in ("ms_host_passes", "ms_kw_calls", "ms_walk_calls", "ms_fuse_calls")])


def pack_strings(strings: Sequence[bytes]):
    off = np.zeros(len(strings) + 1, np.uint32)
    off[1:] = np.cumsum([len(s) for s in strings])
    return b"".join(strings), off


class HostIndex:
    def __init__(self, n_docs: int, device: int = 0, lib_path: Optional[str] = None):
        path = lib_path or build_gpu_lib()
        self.L = capi.declare(C.CDLL(path))          # re-exports the tsgpu_* entry points it links
        L = self.L
        L.tshost_last_error.restype = C.c_char_p
        L.tshost_create.restype = C.c_void_p
        L.tshost_create.argtypes = [C.c_uint32, C.c_int]
        L.tshost_destroy.argtypes = [C.c_void_p]
        L.tshost_tsgpu_handle.restype = C.c_void_p
        L.tshost_tsgpu_handle.argtypes = [C.c_void_p]
        L.tshost_add_field_flat.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.tshost_add_sort_column.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p]
        L.tshost_compact_field.argtypes = [C.c_void_p, C.c_char_p]
        L.tshost_reserve_docs.argtypes = [C.c_void_p, C.c_uint32]
        L.tshost_add_filter.restype = C.c_int32
        L.tshost_add_filter.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.tshost_multi_search.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_uint32, C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                          C.POINTER(Options), C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(Stats)]
        self.n_docs = n_docs
        self.h = L.tshost_create(n_docs, device)
        if not self.h:
            raise capi.TsgpuError(L.tshost_last_error().decode())

    def close(self):
        if self.h:
            self.L.tshost_destroy(self.h)
            self.h = None

    def _err(self):
        return capi.TsgpuError(self.L.tshost_last_error().decode())

    def device_index(self) -> capi.GpuIndex:
        """The host layer's tsgpu_index, for the calls the wrapper does not re-export (vector index build / load, stats)."""
        return capi.GpuIndex.from_handle(self.L.tshost_tsgpu_handle(self.h), self.n_docs, self.L)

    def add_field_flat(self, name: str, tokens: Sequence[bytes], flat) -> int:
        blob, off = pack_strings(tokens)
        assert len(tokens) + 1 == len(flat.list_off)
        lo = np.ascontiguousarray(flat.list_off, np.uint64); ids = np.ascontiguousarray(flat.ids, np.uint32)
        po = np.ascontiguousarray(flat.pos_off, np.uint64); pos = np.ascontiguousarray(flat.positions, np.uint32)
        rc = self.L.tshost_add_field_flat(self.h, name.encode(), len(tokens), blob, off.ctypes.data, lo.ctypes.data, ids.ctypes.data, po.ctypes.data, pos.ctypes.data,
                                          int(flat.is_array))
        if rc < 0:
            raise self._err()
        return rc

    def add_sort_column(self, name: str, values: np.ndarray) -> int:
        v = np.ascontiguousarray(values, np.int64)
        rc = self.L.tshost_add_sort_column(self.h, name.encode(), v.ctypes.data)
        if rc < 0:
            raise self._err()
        return rc

    def compact_field(self, name: str) -> None:
        """Index::compact_field: free the posting lists the field's tokens no longer name (needs the host's exclusive lock)."""
        if self.L.tshost_compact_field(self.h, name.encode()) != 0:
            raise self._err()

    def reserve_docs(self, n_docs: int) -> None:
        """Index::reserve_docs: raise the seq_id capacity."""
        if self.L.tshost_reserve_docs(self.h, n_docs) != 0:
            raise self._err()
        self.n_docs = n_docs

    def add_filter(self, ids: np.ndarray) -> int:
        a = np.ascontiguousarray(ids, np.uint32)
        hnd = self.L.tshost_add_filter(self.h, a.ctypes.data, len(a))
        if hnd > -2:
            raise self._err()
        return hnd

    def multi_search(self, field: str, sort_field: str, queries: Sequence[Sequence[bytes]], stride: int, q_filter=None, qvecs: Optional[np.ndarray] = None,
                     options: Optional[Options] = None, packed=None, out=None):
        """queries: per request its tokens (bytes). Returns (kv [nq, stride] KV_DTYPE, count, found, stats dict). `packed` = a
        (blob, tok_off, q_off) triple from pack_queries() to keep the packing outside a timed region."""
        nq = len(queries) if packed is None else len(packed[2]) - 1
        blob, tok_off, q_off = packed if packed is not None else pack_queries(queries)
        o = options or Options()
        if out is not None:
            kv, cnt, found = out                                   # caller-owned result buffers (kept outside a timed region)
        else:
            kv = np.zeros((nq, stride), KV_DTYPE)
            cnt = np.zeros(nq, np.uint32); found = np.zeros(nq, np.uint32)
        st = Stats()
        qf = None if q_filter is None else np.ascontiguousarray(q_filter, np.int32)
        dim = 0
        if qvecs is not None:
            qvecs = np.ascontiguousarray(qvecs, np.float32)
            dim = qvecs.shape[1]
        rc = self.L.tshost_multi_search(self.h, field.encode(), sort_field.encode(), nq, blob, tok_off.ctypes.data, q_off.ctypes.data,
                                        None if qf is None else qf.ctypes.data, None if qvecs is None else qvecs.ctypes.data, dim, C.byref(o),
                                        kv.ctypes.data, stride, cnt.ctypes.data, found.ctypes.data, C.byref(st))
        if rc != 0:
            raise self._err()
        return kv, cnt, found, {n: getattr(st, n) for n, _ in Stats._fields_}


def pack_queries(queries: Sequence[Sequence[bytes]]):
    toks = [t for q in queries for t in q]
    blob, tok_off = pack_strings(toks)
    q_off = np.zeros(len(queries) + 1, np.uint32)
    q_off[1:] = np.cumsum([len(q) for q in queries])
    return blob, tok_off, q_off
