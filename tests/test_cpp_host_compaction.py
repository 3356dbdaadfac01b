"""Runs tests/cpp/host_compaction.cpp: the C++ host layer through Index::update_field -> compact_field -> reserve_docs -> search,
against an Index loaded from the final documents. On the CPU it links the oracle-backed test double of the C-ABI extended with the
maintenance calls (tests/mirror_double.py); the gpu-marked runs link the library the Python binding loads (libtsgpu.so). The C entry
points of the host layer's wrapper (tshost_compact_field / tshost_reserve_docs) are driven through hostapi."""
import os
import subprocess
import tempfile

import pytest

import mirror_double as md
import oracle_lib as ol
from typesense_b200 import capi, hostapi, synth

ROOT = ol.ROOT
SRC = os.path.join(ROOT, "tests", "cpp", "host_compaction.cpp")


def _run(exe):
    for env in ({}, {"TSGPU_HOST_DEVICE_ART": "1"}):              # host walks, then candidate walks through tsgpu_art_walk_batch
        r = subprocess.run([exe], capture_output=True, text=True, cwd=ROOT, env=dict(os.environ, **env), timeout=600)
        print(r.stdout, r.stderr)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


def test_host_compaction_on_oracle_double():
    ol.build_oracle()
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "host_compaction_oracle_double")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wno-unused", SRC, *md.link_args(), "-o", exe])
        _run(exe)


@pytest.mark.gpu
def test_host_compaction():
    lib = os.path.abspath(capi.LIB_PATH)
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "host_compaction")
        if md.lib_has_maintenance():
            link = ["-L", os.path.dirname(lib), f"-l:{os.path.basename(lib)}", f"-Wl,-rpath,{os.path.dirname(lib)}", "-pthread"]
        else:                                                     # the harness loads the base test double: the extended one
            link = md.link_args()
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wno-unused", SRC, *link, "-o", exe])
        _run(exe)


def _host_search(h, tokens, n):
    kv, cnt, found, _ = h.multi_search("title", "points", [[t] for t in tokens], 16, options=hostapi.Options(num_typos=0, prefix=0))
    return [kv["key"][i, :cnt[i]].tolist() for i in range(len(tokens))], found.tolist()


@pytest.mark.gpu
def test_host_wrappers_compact_and_grow():
    """tshost_compact_field / tshost_reserve_docs through hostapi: a compacted field answers as before, a grown index keeps
    answering, and an unknown field or a shrink is an error"""
    n = 2000
    fd = synth.make_string_field(n, 120, 3, 8, seed=5)
    toks = [synth.vocab_word(r) for r in range(fd.flat.n_lists)]
    h = hostapi.HostIndex(n, lib_path=None if md.lib_has_maintenance() else md.build_host_lib())
    h.add_field_flat("title", toks, fd.flat)
    h.add_sort_column("points", synth.make_points(n, 3))
    q = toks[:40]
    before = _host_search(h, q, n)
    assert sum(before[1]) > 0
    h.compact_field("title")
    assert _host_search(h, q, n) == before
    h.reserve_docs(3 * n)
    assert _host_search(h, q, n) == before
    with pytest.raises(capi.TsgpuError):
        h.compact_field("no_such_field")
    with pytest.raises(capi.TsgpuError):
        h.reserve_docs(n)
    h.close()
