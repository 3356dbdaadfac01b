"""Runs tests/cpp/host_deep_fusion.cpp: hybrid requests of Index::multi_search_batched at topster_size 5000 with
TSGPU_VEC_DEEP_TOPSTER return their whole fused Topster (more than 1024 records), without the bit they return the topster_size
1024 answer, and a deep request with diversity metrics is re-ranked over its whole fused list. On the CPU it links the
oracle-backed test double of the C-ABI; the gpu-marked run links libtsgpu.so and must write the same records as the CPU arm."""
import os
import subprocess
import tempfile

import pytest

import oracle_lib as ol
from typesense_b200 import capi

ROOT = ol.ROOT
SRC = os.path.join(ROOT, "tests", "cpp", "host_deep_fusion.cpp")
ORACLE = ["-L", os.path.join(ROOT, "oracle"), "-l:liboracle.so", f"-Wl,-rpath,{os.path.join(ROOT, 'oracle')}", "-pthread"]


def _run(exe, dump):
    r = subprocess.run([exe, dump], capture_output=True, text=True, cwd=ROOT, timeout=900)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    with open(dump, "rb") as f:
        return f.read()


def _cpu_arm(d):
    ol.build_oracle()
    exe = os.path.join(d, "host_deep_fusion_oracle_double")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wno-unused", SRC, os.path.join(ROOT, "tests", "cpp", "tsgpu_oracle_double.cpp"),
                           "-o", exe, *ORACLE])
    return _run(exe, os.path.join(d, "cpu.bin"))


def test_host_deep_fusion_on_oracle_double():
    with tempfile.TemporaryDirectory() as d:
        assert len(_cpu_arm(d)) > 0


@pytest.mark.gpu
def test_host_deep_fusion():
    if os.environ.get("TSGPU_TEST_DOUBLE") == "1":
        pytest.skip("links the real libtsgpu.so; the CPU run of this program is test_host_deep_fusion_on_oracle_double")
    lib = os.path.abspath(capi.LIB_PATH)
    with tempfile.TemporaryDirectory() as d:
        cpu = _cpu_arm(d)
        exe = os.path.join(d, "host_deep_fusion")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wno-unused", SRC, "-o", exe, "-L", os.path.dirname(lib),
                               f"-l:{os.path.basename(lib)}", f"-Wl,-rpath,{os.path.dirname(lib)}", *ORACLE])
        gpu = _run(exe, os.path.join(d, "gpu.bin"))
        # the GPU run also writes the diversity requests (the test double has no tsgpu_diversify_batch): compare the common prefix
        assert len(gpu) > len(cpu) and gpu[:len(cpu)] == cpu
