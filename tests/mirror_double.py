"""TEST INFRASTRUCTURE: the oracle-backed test double of the C-ABI extended with the mirror maintenance calls
(tests/cpp/tsgpu_oracle_double_mirror.cpp), built into a per-process temporary directory. The tests of those calls use it where the
library they would load does not implement them (the base double of the dry run); on a GPU they use libtsgpu.so."""
import ctypes as C
import os
import subprocess
import tempfile

import oracle_lib as ol
from typesense_b200 import capi

ROOT = ol.ROOT
SRC = os.path.join(ROOT, "tests", "cpp", "tsgpu_oracle_double_mirror.cpp")
_TMP = []


def _dir() -> str:
    if not _TMP:
        _TMP.append(tempfile.mkdtemp(prefix="tsgpu_double_mirror_"))
    return _TMP[0]


def link_args():
    """g++ arguments that add the extended double (and the oracle behind it) to a program or library"""
    ol.build_oracle()
    return [SRC, "-L", os.path.join(ROOT, "oracle"), "-l:liboracle.so", f"-Wl,-rpath,{os.path.join(ROOT, 'oracle')}", "-pthread"]


def _build(name, extra_src):
    so = os.path.join(_dir(), name)
    if not os.path.exists(so):
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wno-unused", "-fPIC", "-shared", *extra_src, *link_args(), "-o", so + ".tmp"])
        os.replace(so + ".tmp", so)
    return so


def build_lib() -> str:
    return _build("libtsgpu_double_mirror.so", [])


def build_host_lib() -> str:
    """the host layer's C wrapper over the extended double"""
    return _build("libtshost_double_mirror.so", [os.path.join(ROOT, "typesense_b200", "host", "tshost_capi.cpp")])


def lib_has_maintenance() -> bool:
    return hasattr(capi.lib(), "tsgpu_index_compact_field")


def load_lib():
    return capi.declare(C.CDLL(build_lib()))
