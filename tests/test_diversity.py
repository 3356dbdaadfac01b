"""Diversity re-ranking (tsgpu_diversify_batch): the MMR order of Index::populate_result_kvs (src/index.cpp:9016-9064) over facet and
sort-field similarity (similarity_t::calculate, src/diversity.cpp).

CPU: the oracle's transcription (tso_diversify) equals a Python transcription of the two reference functions, typed as the
reference types them; the reference's DiversityOverride expectations hold on it; the device's pair functions compiled by g++ agree
with it pair for pair; the K^2 formulation agrees with it. GPU: the device's records are byte-identical to the oracle's."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import diversity_double as dd
import oracle_lib as ol
from typesense_b200 import capi
from typesense_b200.structs import KV_DTYPE

ON_DOUBLE = os.environ.get("TSGPU_TEST_DOUBLE") == "1"
I64_MIN = np.iinfo(np.int64).min
EQ, JAC = capi.DIV_EQUALITY, capi.DIV_JACCARD


# ---------------------------------------------------------------------------------------------------------------- inputs
def _facet(rng, n_docs, n_values, max_row, p_empty=0.2, single=False):
    off, vals = [0], []
    for _ in range(n_docs):
        if rng.random() >= p_empty:
            k = 1 if single else int(rng.integers(1, max_row + 1))
            vals += [int(v) for v in rng.integers(0, n_values, k)]            # repeats: a set compares them once
        off.append(len(vals))
    return np.asarray(off, np.uint64), np.asarray(vals, np.uint32)


def _column(rng, n_docs, n_values, p_missing=0.25):
    c = rng.integers(0, n_values, n_docs).astype(np.int64)
    c[rng.random(n_docs) < p_missing] = I64_MIN
    return c


def _topster(rng, n_docs, K, vd_mode):
    kv = np.zeros(K, KV_DTYPE)
    kv["key"] = rng.choice(n_docs, K, replace=False)
    kv["scores"][:, 0] = rng.integers(0, 1000, K)
    kv["distinct_key"] = kv["key"]
    if vd_mode == "keyword":
        kv["vector_distance"] = -1.0                                            # what keyword and q=* records carry
    else:
        kv["vector_distance"] = rng.integers(0, 5, K).astype(np.float32) * np.float32(0.125)    # many exact ties
    return kv


# ---------------------------------------------------------------------------------------------------------------- Python transcription
def py_populate_result_kvs(n_docs, metrics, lam, kv):
    """Index::populate_result_kvs (diversity branch) and similarity_t::calculate as the reference types them: float products, double
    sums and quotients. Returns positions in MMR order."""
    lam = np.float32(lam)
    keys = [int(k) for k in kv["key"]]
    cache = {}

    def facet_set(off, vals, s):
        if s >= n_docs or off[s + 1] == off[s]:
            return None                                                        # facet_it lands past the document
        return set(int(v) for v in vals[int(off[s]):int(off[s + 1])])

    def calculate(i, j):
        if j < i:
            i, j = j, i
        if (i, j) in cache:
            return cache[(i, j)]
        sim = 0.0
        for m in metrics:
            if m[0] == "facet":
                _, off, vals, method, w = m
                a = facet_set(off, vals, i)
                if a is None:
                    continue
                b = facet_set(off, vals, j)
                if b is None:
                    continue
                if method == JAC:
                    if not a and not b:
                        continue
                    sim += (len(a & b) / len(a | b)) * float(np.float32(w))
                elif method == EQ:
                    if len(a) != len(b):
                        continue
                    sim += float(np.float32(w) * np.float32(len(a - b) == 0))
            else:
                _, col, method, w = m
                if i >= n_docs or col[i] == I64_MIN or j >= n_docs or col[j] == I64_MIN:
                    continue
                if method == EQ and col[i] == col[j]:
                    sim += float(np.float32(w))
        cache[(i, j)] = sim
        return sim

    lowest = -sys.float_info.max
    result, processed = [0], {keys[0]}
    while len(result) < len(keys):
        mmr, best = lowest, None
        for i in range(1, len(keys)):
            if keys[i] in processed:
                continue
            left = lam * np.float32(kv["vector_distance"][i])                 # float * float
            max_similarity = lowest
            for j in result:
                max_similarity = max(max_similarity, calculate(keys[i], keys[j]))
            right = float(np.float32(1) - lam) * max_similarity
            mr = float(left) - right
            if mr > mmr:
                best, mmr = i, mr
        processed.add(keys[best])
        result.append(best)
    return result


def _metric_sets(rng, n_docs):
    fa = _facet(rng, n_docs, 9, 5)
    fs = _facet(rng, n_docs, 4, 1, single=True)
    col = _column(rng, n_docs, 5)
    return [
        [("facet", *fa, JAC, 1.0)],
        [("facet", *fa, JAC, 0.6), ("sort", col, EQ, 0.1)],
        [("sort", col, EQ, 1.0), ("facet", *fs, EQ, 0.6), ("facet", *fa, EQ, 0.1)],
        [("sort", col, JAC, 1.0), ("facet", *fs, JAC, 0.1), ("facet", *fa, JAC, 0.6)],      # jaccard on a sort field adds 0
    ]


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_oracle_equals_python_transcription():
    rng = np.random.default_rng(3)
    n_docs = 120
    checked = 0
    for metrics in _metric_sets(rng, n_docs):
        for lam in (0.0, 0.3, 0.5, 1.0):
            for vd_mode in ("keyword", "vector"):
                for K in (1, 2, 9, 40):
                    kv = _topster(rng, n_docs + 10, K, vd_mode)                 # some ids beyond the data: no values
                    want = kv[py_populate_result_kvs(n_docs, metrics, lam, kv)]
                    got = dd.oracle_diversify(n_docs, metrics, lam, kv)
                    assert got.tobytes() == want.tobytes(), (metrics[0][0], lam, vd_mode, K)
                    checked += 1
    assert checked == 4 * 4 * 2 * 4


def _override():
    tags = [["gold", "silver"], ["FINE PLATINUM"], ["bronze", "gold"], ["silver"], ["silver", "gold", "bronze"], ["silver", "FINE PLATINUM"]]
    ids = {}
    off, vals = [0], []
    for t in tags:
        vals += [ids.setdefault(v, len(ids)) for v in t]
        off.append(len(vals))
    kv = np.zeros(6, KV_DTYPE)
    kv["key"] = [5, 4, 3, 2, 1, 0]                                              # q=*: seq_id descending
    kv["vector_distance"] = -1.0
    return np.asarray(off, np.uint64), np.asarray(vals, np.uint32), kv


def test_diversity_override_on_oracle():
    """TEST_F(CollectionCurationTest, DiversityOverride), test/collection_curation_test.cpp:5591-5691"""
    off, vals, kv = _override()
    m = [("facet", off, vals, JAC, 1.0)]
    assert dd.oracle_diversify(6, m, 0.5, kv)["key"].tolist() == [5, 2, 0, 3, 1, 4]
    assert dd.oracle_diversify(6, m, 1.0, kv)["key"].tolist() == [5, 4, 3, 2, 1, 0]
    assert [kv["key"][i] for i in py_populate_result_kvs(6, m, 0.5, kv)] == [5, 2, 0, 3, 1, 4]


def test_device_functions_agree_with_oracle_pair_for_pair(tmp_path):
    """diversity.cuh's __host__ __device__ similarity and mmr, compiled by g++, against tso_div_similarity"""
    lib = dd.build_lib()
    exe = str(tmp_path / "diversity_pairs")
    subprocess.check_call(["g++", *dd.CXXFLAGS, os.path.join(ol.ROOT, "tests", "cpp", "diversity_pairs.cpp"), lib,
                           f"-Wl,-rpath,{os.path.dirname(lib)}", "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "mismatches 0" in r.stdout, r.stdout + r.stderr


def test_k2_formulation_equals_oracle():
    """the reference used for the device's longest lists (div_k2_reference.cpp) orders like the transcription"""
    rng = np.random.default_rng(8)
    n_docs = 400
    for metrics in _metric_sets(rng, n_docs):
        for lam in (0.0, 0.3, 0.5, 1.0):
            for vd_mode in ("keyword", "vector"):
                kv = _topster(rng, n_docs + 20, 120, vd_mode)
                assert dd.k2_diversify(n_docs, metrics, lam, kv).tobytes() == dd.oracle_diversify(n_docs, metrics, lam, kv).tobytes()


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def lib_with_diversify():
    """libtsgpu.so has the call; where the harness loaded the base test double instead, the double extended with it answers"""
    if dd.lib_has_diversify():
        yield
        return
    saved = capi._lib
    capi._lib = dd.load_lib()
    yield
    capi._lib = saved


def _mirror(rng, n0, n_docs):
    """an index created for n0 documents and grown to n_docs: documents n0.. have empty facet rows and no sort values"""
    gi = capi.GpuIndex(n0, 0)
    fa = _facet(rng, n0, 60, 6)
    fs = _facet(rng, n0, 5, 1, single=True)
    fb = _facet(rng, n0, 3000, 120, p_empty=0.5)                               # long rows: workspaces that leave shared memory
    col = _column(rng, n0, 4)
    ids = [gi.load_facet(int(f[1].max()) + 1 if len(f[1]) else 1, f[0], f[1]) for f in (fa, fs, fb)]
    c = gi.load_sort_column(col)
    gi.reserve_docs(n_docs)
    grow = lambda f: (np.concatenate([f[0], np.full(n_docs - n0, f[0][-1], np.uint64)]), f[1])
    fa, fs, fb = grow(fa), grow(fs), grow(fb)
    col = np.concatenate([col, np.full(n_docs - n0, I64_MIN, np.int64)])
    metric_lists = [
        ([(ids[0], 0, JAC, 1.0)], [("facet", *fa, JAC, 1.0)]),
        ([(ids[0], 0, JAC, 0.6), (None, c, EQ, 0.1)], [("facet", *fa, JAC, 0.6), ("sort", col, EQ, 0.1)]),
        ([(None, c, EQ, 1.0), (ids[1], 0, EQ, 0.6), (ids[0], 0, EQ, 0.1), (None, c, JAC, 0.3)],
         [("sort", col, EQ, 1.0), ("facet", *fs, EQ, 0.6), ("facet", *fa, EQ, 0.1), ("sort", col, JAC, 0.3)]),
        ([(ids[2], 0, JAC, 0.6), (ids[1], 0, JAC, 0.1)], [("facet", *fb, JAC, 0.6), ("facet", *fs, JAC, 0.1)]),
    ]
    return gi, metric_lists


def _expected(n_docs, metrics, lam, kv):
    return (dd.oracle_diversify if len(kv) <= 250 else dd.k2_diversify)(n_docs, metrics, lam, kv)


@pytest.mark.gpu
def test_device_records_equal_oracle(lib_with_diversify):
    rng = np.random.default_rng(17)
    n0, n_docs = 6000, 8000
    gi, metric_lists = _mirror(rng, n0, n_docs)
    sizes = [0, 1, 2, 7, 250] if ON_DOUBLE else [0, 1, 2, 7, 250, 1024, 3000]     # the double answers with the cubic loop
    lams = [0.0, 0.3, 0.5, 1.0]
    for mi, (dev_m, ora_m) in enumerate(metric_lists):
        stride = max(sizes)
        nq = len(sizes) * 2
        kv = np.zeros((nq, stride), KV_DTYPE)
        kv["key"] = 0xDEAD                                                      # beyond count: never read, never written
        cnt = np.zeros(nq, np.uint32)
        lam = np.zeros(nq, np.float32)
        for q in range(nq):
            K = sizes[q % len(sizes)]
            kv[q, :K] = _topster(rng, n_docs, K, "keyword" if q < len(sizes) else "vector")
            cnt[q], lam[q] = K, lams[(q + mi) % 4]
        out = np.full(nq * stride * KV_DTYPE.itemsize, 0xAB, np.uint8).view(KV_DTYPE).reshape(nq, stride)
        gi.diversify(dev_m, lam, kv, cnt, out=out)
        for q in range(nq):
            K = int(cnt[q])
            assert out[q, :K].tobytes() == _expected(n_docs, ora_m, float(lam[q]), kv[q, :K]).tobytes(), (mi, q, K)
            assert (out[q, K:].view(np.uint8) == 0xAB).all()                    # only count[q] records are written
        # in place, from device memory to device memory
        try:
            import torch
            dev = torch.cuda.is_available() and not ON_DOUBLE
        except Exception:
            dev = False
        if dev:
            t = torch.from_numpy(kv.view(np.uint8).copy()).cuda()
            gi.diversify(dev_m, lam, t, cnt, out=t, stride=stride)
            back = t.cpu().numpy().view(KV_DTYPE).reshape(nq, stride)
            for q in range(nq):
                assert back[q, :cnt[q]].tobytes() == out[q, :cnt[q]].tobytes(), (mi, q)
        else:
            again = kv.copy()
            gi.diversify(dev_m, lam, again, cnt, out=again)
            for q in range(nq):
                assert again[q, :cnt[q]].tobytes() == out[q, :cnt[q]].tobytes(), (mi, q)
    s = gi.stats()
    if not ON_DOUBLE:
        assert s["ms_kernels"] > 0 and s["ms_total"] >= s["ms_kernels"]


@pytest.mark.gpu
def test_diversity_override_on_device(lib_with_diversify):
    off, vals, kv = _override()
    gi = capi.GpuIndex(6, 0)
    f = gi.load_facet(4, off, vals)
    rows = np.stack([kv, kv])
    out = gi.diversify([(f, 0, JAC, 1.0)], [0.5, 1.0], rows, [6, 6])
    assert out[0]["key"].tolist() == [5, 2, 0, 3, 1, 4]
    assert out[1]["key"].tolist() == [5, 4, 3, 2, 1, 0]


@pytest.mark.gpu
def test_rejections_leave_the_index_usable(lib_with_diversify):
    off, vals, kv = _override()
    gi = capi.GpuIndex(6, 0)
    f = gi.load_facet(4, off, vals)
    c = gi.load_sort_column(np.arange(6, dtype=np.int64))
    L = capi.lib()
    rows = np.stack([kv, kv])
    out = np.zeros_like(rows)

    def call(metrics, lam=(0.5, 0.5), cnt=(6, 6), stride=6, n=None):
        m = (capi.DivMetricStruct * max(1, len(metrics)))()
        for i, (facet, col, method, w) in enumerate(metrics):
            m[i].facet, m[i].sort_col, m[i].method, m[i].weight = capi.NO_LIST if facet is None else facet, col, method, w
        la = np.asarray(lam, np.float32)
        ca = np.asarray(cnt, np.uint32)
        return L.tsgpu_diversify_batch(gi.h, m, len(metrics) if n is None else n, len(ca), la.ctypes.data, rows.ctypes.data, stride,
                                       ca.ctypes.data, out.ctypes.data)

    ok = [(f, 0, JAC, 1.0)]
    assert call([(f + 1, 0, JAC, 1.0)]) == 2                                    # unknown facet id
    assert call([(None, c + 1, EQ, 1.0)]) == 2                                  # unknown sort column
    assert call([(None, -1, EQ, 1.0)]) == 2
    assert call([(f, 0, 2, 1.0)]) == 2                                          # method outside the enum
    assert call(ok, n=0) == 2                                                   # no metric
    assert call(ok, cnt=(6, 7)) == 2                                            # count > kv_stride
    assert call(ok, lam=(0.5, math.nan)) == 2
    assert call(ok, lam=(1.5, 0.5)) == 2
    assert call(ok, lam=(0.5, -0.25)) == 2
    assert call(ok * (capi.MAX_DIV_METRICS + 1)) == 4                           # TSGPU_ERR_CAPACITY
    assert call(ok * capi.MAX_DIV_METRICS) == 0
    assert call(ok) == 0
    assert out[0]["key"].tolist() == [5, 2, 0, 3, 1, 4]
