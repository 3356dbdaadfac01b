"""Runs tests/cpp/host_diversity.cpp: the C++ host layer's diversity re-ranking (search_options::diversity) through Index::search,
the lock-step multi_search and multi_search_batched, against the oracle's transcription of the reference loop. On the CPU it links the
oracle-backed test double extended with tsgpu_diversify_batch (tests/diversity_double.py); the gpu-marked run links the library the
Python binding loads (libtsgpu.so)."""
import os
import subprocess
import tempfile

import pytest

import diversity_double as dd
import oracle_lib as ol
from typesense_b200 import capi

ROOT = ol.ROOT
SRC = os.path.join(ROOT, "tests", "cpp", "host_diversity.cpp")
ORACLE = ["-L", os.path.join(ROOT, "oracle"), "-l:liboracle.so", f"-Wl,-rpath,{os.path.join(ROOT, 'oracle')}"]


def _run(exe):
    r = subprocess.run([exe], capture_output=True, text=True, cwd=ROOT, timeout=600)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "all checks passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]


def test_host_diversity_on_oracle_double():
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "host_diversity_oracle_double")
        subprocess.check_call(["g++", *dd.CXXFLAGS, SRC, *dd.link_args(), "-o", exe])
        _run(exe)


@pytest.mark.gpu
def test_host_diversity():
    lib = os.path.abspath(capi.LIB_PATH)
    ol.build_oracle()
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "host_diversity")
        if dd.lib_has_diversify():
            link = ["-DWITH_ORACLE_DIVERSIFY", "-L", os.path.dirname(lib), f"-l:{os.path.basename(lib)}", f"-Wl,-rpath,{os.path.dirname(lib)}",
                    *ORACLE, "-pthread"]
        else:                                                     # the harness loads the base test double: the extended one
            link = dd.link_args()
        subprocess.check_call(["g++", *dd.CXXFLAGS, SRC, *link, "-o", exe])
        _run(exe)
