"""TEST INFRASTRUCTURE: the oracle of the diversity re-ranking and the test double that answers tsgpu_diversify_batch with it
(tests/cpp/tso_diversify.cpp, tests/cpp/tsgpu_oracle_double_diversity.cpp: the mirror double plus that call), built into a
per-process temporary directory. The tests of the call use the double where the library they would load does not implement it
(the base double of the dry run); on a GPU they use libtsgpu.so, and the oracle from this library."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import oracle_lib as ol
from typesense_b200 import capi
from typesense_b200.structs import KV_DTYPE

ROOT = ol.ROOT
SRC = os.path.join(ROOT, "tests", "cpp", "tsgpu_oracle_double_diversity.cpp")
CXXFLAGS = ["-std=c++17", "-O1", "-Wall", "-Wno-unused", "-ffp-contract=off"]
_TMP = []


def _dir() -> str:
    if not _TMP:
        _TMP.append(tempfile.mkdtemp(prefix="tsgpu_double_diversity_"))
    return _TMP[0]


def link_args():
    """g++ arguments that add the extended double (and the oracle behind it) to a program or library"""
    ol.build_oracle()
    return [SRC, "-L", os.path.join(ROOT, "oracle"), "-l:liboracle.so", f"-Wl,-rpath,{os.path.join(ROOT, 'oracle')}", "-pthread"]


def _build(name, extra_src):
    so = os.path.join(_dir(), name)
    if not os.path.exists(so):
        subprocess.check_call(["g++", *CXXFLAGS, "-fPIC", "-shared", *extra_src, *link_args(), "-o", so + ".tmp"])
        os.replace(so + ".tmp", so)
    return so


def build_lib() -> str:
    return _build("libtsgpu_double_diversity.so", [])


def build_host_lib() -> str:
    """the host layer's C wrapper over the extended double"""
    return _build("libtshost_double_diversity.so", [os.path.join(ROOT, "typesense_b200", "host", "tshost_capi.cpp")])


def lib_has_diversify() -> bool:
    return hasattr(capi.lib(), "tsgpu_diversify_batch")


def load_lib():
    return capi.declare(C.CDLL(build_lib()))


class MetricStruct(C.Structure):
    """tso_div_metric"""
    _fields_ = [("doc_off", C.c_void_p), ("value_ids", C.c_void_p), ("sort_col", C.c_void_p), ("method", C.c_uint32), ("weight", C.c_float)]


_oracle = []


def _oracle_lib():
    if not _oracle:
        L = C.CDLL(build_lib())
        L.tso_diversify.restype = None
        L.tso_diversify.argtypes = [C.c_uint32, C.POINTER(MetricStruct), C.c_uint32, C.c_float, C.c_void_p, C.c_uint32, C.c_void_p]
        L.div_k2_order.restype = None
        L.div_k2_order.argtypes = [C.c_uint32, C.POINTER(MetricStruct), C.c_uint32, C.c_float, C.c_void_p, C.c_uint32, C.c_void_p]
        L.tso_div_similarity.restype = C.c_double
        L.tso_div_similarity.argtypes = [C.c_uint32, C.POINTER(MetricStruct), C.c_uint32, C.c_uint32, C.c_uint32]
        _oracle.append(L)
    return _oracle[0]


def _metric_structs(metrics):
    """metrics: ("facet", doc_off u64 [n_docs + 1], value_ids u32, method, weight) or ("sort", column i64 [n_docs], method, weight)"""
    keep = []
    m = (MetricStruct * max(1, len(metrics)))()
    for i, spec in enumerate(metrics):
        if spec[0] == "facet":
            off = np.ascontiguousarray(spec[1], np.uint64)
            vals = np.ascontiguousarray(spec[2] if len(spec[2]) else np.zeros(1, np.uint32), np.uint32)
            keep += [off, vals]
            m[i].doc_off, m[i].value_ids, m[i].sort_col = off.ctypes.data, vals.ctypes.data, None
            m[i].method, m[i].weight = spec[3], spec[4]
        else:
            col = np.ascontiguousarray(spec[1], np.int64)
            keep.append(col)
            m[i].doc_off, m[i].value_ids, m[i].sort_col = None, None, col.ctypes.data
            m[i].method, m[i].weight = spec[2], spec[3]
    return m, keep


def oracle_diversify(n_docs: int, metrics, lam: float, kv: np.ndarray) -> np.ndarray:
    """tso_diversify: the reference's loop over one sorted Topster (a 1-D KV_DTYPE array); returns the records in MMR order"""
    L = _oracle_lib()
    m, keep = _metric_structs(metrics)
    src = np.ascontiguousarray(kv, KV_DTYPE)
    out = np.zeros(max(1, len(src)), KV_DTYPE)
    L.tso_diversify(n_docs, m, len(metrics), lam, src.ctypes.data, len(src), out.ctypes.data)
    return out[:len(src)]


def k2_diversify(n_docs: int, metrics, lam: float, kv: np.ndarray) -> np.ndarray:
    """div_k2_reference.cpp: the same order by the K^2 formulation (serial), for Topsters too long for the transcription's loop"""
    L = _oracle_lib()
    m, keep = _metric_structs(metrics)
    src = np.ascontiguousarray(kv, KV_DTYPE)
    order = np.zeros(max(1, len(src)), np.uint32)
    L.div_k2_order(n_docs, m, len(metrics), lam, src.ctypes.data, len(src), order.ctypes.data)
    return src[order[:len(src)]]


def oracle_similarity(n_docs: int, metrics, i: int, j: int) -> float:
    L = _oracle_lib()
    m, keep = _metric_structs(metrics)
    return L.tso_div_similarity(n_docs, m, len(metrics), i, j)
