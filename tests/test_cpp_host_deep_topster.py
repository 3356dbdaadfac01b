"""Runs tests/cpp/host_deep_topster.cpp: through Index::multi_search_batched, keyword-only q=* and phrase-only requests take deep
Topsters at topster_size 5000, and the same requests with a query vector stay at 1024 (their keyword stage feeds
tsgpu_hybrid_fuse_batch). On the CPU it links the oracle-backed test double of the C-ABI; the gpu-marked run links libtsgpu.so."""
import os
import subprocess
import tempfile

import pytest

import oracle_lib as ol
from typesense_b200 import capi

ROOT = ol.ROOT
SRC = os.path.join(ROOT, "tests", "cpp", "host_deep_topster.cpp")
ORACLE = ["-L", os.path.join(ROOT, "oracle"), "-l:liboracle.so", f"-Wl,-rpath,{os.path.join(ROOT, 'oracle')}", "-pthread"]


def _run(exe):
    r = subprocess.run([exe], capture_output=True, text=True, cwd=ROOT, timeout=600)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


def test_host_deep_topster_on_oracle_double():
    ol.build_oracle()
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "host_deep_topster_oracle_double")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wno-unused", SRC, os.path.join(ROOT, "tests", "cpp", "tsgpu_oracle_double.cpp"),
                               "-o", exe, *ORACLE])
        _run(exe)


@pytest.mark.gpu
def test_host_deep_topster():
    if os.environ.get("TSGPU_TEST_DOUBLE") == "1":
        pytest.skip("links the real libtsgpu.so; the CPU run of this program is test_host_deep_topster_on_oracle_double")
    ol.build_oracle()
    lib = os.path.abspath(capi.LIB_PATH)
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "host_deep_topster")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wno-unused", SRC, "-o", exe, "-L", os.path.dirname(lib),
                               f"-l:{os.path.basename(lib)}", f"-Wl,-rpath,{os.path.dirname(lib)}", *ORACLE])
        _run(exe)
