"""Deep pagination for vector and hybrid searches (TSGPU_VEC_DEEP_TOPSTER): Topsters larger than TSGPU_MAX_TOPK in the deep
vector assembly and the deep hybrid fusion (csrc/deep_fuse.cuh). Every answer is compared with the oracle, which runs the
reference's Topster at any capacity: ids, all three scores, text_match_score, vector_distance, query_index, counts and found
bit-equal."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle_lib as ol
from typesense_b200 import capi, structs as S, synth
from test_gpu_parity import assert_kv_equal

DEEP = capi.QFLAG_DEEP_TOPSTER
VDEEP = capi.VEC_DEEP_TOPSTER
RERANK = 0x40
ON_DOUBLE = os.environ.get("TSGPU_TEST_DOUBLE") == "1"
device_only = pytest.mark.skipif(ON_DOUBLE, reason="asserts what only the device library does")

TEXT = ((S.SORT_TEXT_MATCH, -1, 1, 0), (S.SORT_NUMERIC, 0, 1, 0), (S.SORT_NONE, -1, 1, 0))
VSORTS = [((S.SORT_VECTOR_DISTANCE, -1, -1, 0), (S.SORT_NUMERIC, 0, 1, 0), (S.SORT_NONE, -1, 1, 0)),
          ((S.SORT_NUMERIC, 0, -1, 1), (S.SORT_VECTOR_DISTANCE, -1, -1, 0), (S.SORT_SEQ_ID, -1, 1, 0)),
          ((S.SORT_NUMERIC, 0, 1, 0), (S.SORT_SEQ_ID, -1, -1, 0), (S.SORT_NONE, -1, 1, 0))]


@pytest.fixture(scope="module")
def vc():
    n, dim = 6000, 128
    vec = synth.make_vectors(n, dim, 5).numpy()
    g = ol.hnsw_build(vec, 16, 100, 100)
    fd = synth.make_string_field(n, 200, 3, 8, seed=31)
    pts = synth.make_points(n, 8, hi=100, missing_frac=0.05)
    gi = capi.GpuIndex(n, 0)
    gi.load_field(fd.flat)
    gi.load_sort_column(pts)
    gi.load_hnsw(g)
    oi = ol.OracleIndex(n, [fd.flat], [pts], g)
    yield n, dim, vec, fd, pts, gi, oi
    gi.close()


def deep(q: S.Query, k: int) -> S.Query:
    q.topk = k
    q.flags |= DEEP
    return q


def vec_batch(rng, n_docs, nq, K, filters):
    qs = []
    for i in range(nq):
        q = deep(S.Query([], sort=VSORTS[i % 3]), K)
        if filters and i % 3 == 1:
            q.filter = int(rng.integers(0, len(filters)))
        if i % 4 == 0:
            q.excl = np.unique(rng.integers(0, n_docs, 40)).tolist()
        qs.append(q)
    return S.KwBatch(qs, [0], filters)


def hybrid_batch(rng, fd, nq, K, filters, rerank_half=True):
    """keyword sides from one rare token (fewer matches than K) to several frequent combinations (more than K); text-match
    scores tie a lot (few positions per field), so shared text ranks matter"""
    toks = synth.sample_queries(fd, nq, 2, int(rng.integers(0, 1 << 30)))
    qs = []
    for i, row in enumerate(toks):
        if i % 3 == 0:
            combos = [S.Combo([[int(row[0])], [int(row[1])]], 2)]
        elif i % 3 == 1:
            combos = [S.Combo([[0]], 1), S.Combo([[1]], 1, total_cost=1), S.Combo([[int(row[0])]], 1, total_cost=2)]
        else:
            combos = [S.Combo([[int(row[0])], [2]], 1), S.Combo([[3]], 1, total_cost=1)]
        q = deep(S.Query(combos, sort=TEXT, num_query_tokens=2), K)
        if filters and i % 4 == 1:
            q.filter = int(rng.integers(0, len(filters)))
        if i % 5 == 0:
            q.excl = np.unique(rng.integers(0, 6000, 30)).tolist()
        if rerank_half and i % 2:
            q.flags |= RERANK
        qs.append(q)
    return S.KwBatch(qs, [0], filters)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1025, 2500, 4096])
def test_vector_search(vc, K):
    n, dim, vec, fd, pts, gi, oi = vc
    rng = np.random.default_rng(K)
    # (an empty filter is left to the hybrid tests: for q=* the oracle searches where the reference and the device return early)
    filters = [np.unique(rng.integers(0, n, 3500)).astype(np.uint32), np.arange(0, n, 2, dtype=np.uint32)]
    b = vec_batch(rng, n, 12, K, filters)
    qv = synth.make_vectors(12, dim, 43 + K).numpy()
    for vp in [S.vec_params(k=0, fetch_size=K, flags=VDEEP), S.vec_params(k=min(K, 3000), ef=64, fetch_size=10, flags=VDEEP),
               S.vec_params(k=0, fetch_size=K, distance_threshold=0.95, flags=VDEEP)]:
        kv, cnt, found = gi.vector_search(b, qv, vp, K)
        okv, ocnt, ofound = oi.vector_search(b, qv, vp, K)
        assert_kv_equal(kv, cnt, found, okv, ocnt, ofound)
        assert int(cnt.max()) > 1024
    # persistent filters answer as the same ids inline
    handles = [gi.filter_create(f) for f in filters]
    vp = S.vec_params(k=0, fetch_size=K, flags=VDEEP)
    kv, cnt, found = gi.vector_search(b.with_filter_handles(handles), qv, vp, K)
    assert_kv_equal(kv, cnt, found, *oi.vector_search(b, qv, vp, K))


@pytest.mark.gpu
@pytest.mark.parametrize("tensor", [False, True])
def test_vector_search_flat_path(vc, tensor):
    # filters below flat_search_cutoff take the brute-force path; with TSGPU_VEC_FLAT_TENSOR queries sharing a filter go to the
    # tensor-core scan, whose distances are within ~1e-6 of the fp32 loop
    n, dim, vec, fd, pts, gi, oi = vc
    rng = np.random.default_rng(7)
    filters = [np.unique(rng.integers(0, n, 2200)).astype(np.uint32), np.arange(1, n, 3, dtype=np.uint32)]
    qs = [deep(S.Query([], sort=VSORTS[i % 3], filter=i % 2, excl=list(range(0, 300, 7)) if i % 5 == 0 else ()), [1025, 1800, 4096][i % 3])
          for i in range(18)]
    b = S.KwBatch(qs, [0], filters)
    qv = synth.make_vectors(len(qs), dim, 91).numpy()
    vp = S.vec_params(k=0, fetch_size=4096, flat_search_cutoff=5000, flags=VDEEP | (S.VEC_FLAT_TENSOR if tensor else 0))
    kv, cnt, found = gi.vector_search(b, qv, vp, 4096)
    okv, ocnt, ofound = oi.vector_search(b, qv, vp, 4096)
    if not tensor:
        assert_kv_equal(kv, cnt, found, okv, ocnt, ofound)
    else:
        assert cnt.tolist() == ocnt.tolist() and found.tolist() == ofound.tolist()
        for q in range(len(qs)):
            c = int(cnt[q])
            assert len(set(kv["key"][q, :c].tolist()) ^ set(okv["key"][q, :c].tolist())) <= 4, q
            assert np.allclose(np.sort(kv["vector_distance"][q, :c]), np.sort(okv["vector_distance"][q, :c]), rtol=0, atol=1e-5)
    assert int(cnt.max()) > 1024


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1025, 3000, 4096])
def test_hybrid_search(vc, K):
    n, dim, vec, fd, pts, gi, oi = vc
    rng = np.random.default_rng(300 + K)
    filters = [np.unique(rng.integers(0, n, 4000)).astype(np.uint32), np.zeros(0, np.uint32)]
    b = hybrid_batch(rng, fd, 10, K, filters)
    qv = synth.make_vectors(10, dim, 17 + K).numpy()
    grew = 0
    for k in (100, 1500, 4096):
        for alpha in (0.3, 0.8):
            vp = S.vec_params(k=k, ef=10, alpha=alpha, flags=VDEEP)
            kv, cnt, found = gi.hybrid_search(b, qv, vp, K)
            okv, ocnt, ofound = oi.hybrid_search(b, qv, vp, K)
            assert_kv_equal(kv, cnt, found, okv, ocnt, ofound)
            grew = max(grew, int(cnt.max()))
    assert grew > 1024


@pytest.mark.gpu
def test_hybrid_search_flat_path(vc):
    # filters below flat_search_cutoff: the vector list is the brute-force distances in the filter's id order, ranked by position
    n, dim, vec, fd, pts, gi, oi = vc
    rng = np.random.default_rng(77)
    filters = [np.unique(rng.integers(0, n, 2600)).astype(np.uint32), np.arange(2, n, 4, dtype=np.uint32)]
    b = hybrid_batch(rng, fd, 9, 3000, filters)
    for i in range(b.n_queries):
        b.q_filter[i] = i % 2
    qv = synth.make_vectors(b.n_queries, dim, 78).numpy()
    for alpha in (0.3, 0.8):
        vp = S.vec_params(k=1500, ef=10, alpha=alpha, flat_search_cutoff=3000, flags=VDEEP)
        kv, cnt, found = gi.hybrid_search(b, qv, vp, 3000)
        assert_kv_equal(kv, cnt, found, *oi.hybrid_search(b, qv, vp, 3000))
        assert int(cnt.max()) > 1024


@pytest.mark.gpu
def test_hybrid_eviction_of_a_keyword_entry_that_comes_back(vc):
    # A full keyword Topster (1025 entries of three frequent tokens) and alpha 0.8. The query vector is that of the best keyword
    # entry X, which is data[0] of the sorted array. A near neighbour of X with a smaller seq_id that the keyword Topster does not
    # hold has a vector rank of 1-3, so its KV is not smaller than data[0] and Topster::add evicts X. When X's own result comes
    # (ascending seq_id), topster->map no longer finds X and it enters as a new vector-only KV: text_match_score 0 although X is
    # in the keyword Topster. The oracle's answer must show that, and the device must agree with it.
    n, dim, vec, fd, pts, gi, oi = vc
    K = 1025
    qs = [deep(S.Query([S.Combo([[t]], 1), S.Combo([[t + 1]], 1, total_cost=1), S.Combo([[t + 2]], 1, total_cost=2)], sort=TEXT), K)
          for t in range(12)]
    b = S.KwBatch(qs, [0])
    kw, kw_cnt, _ = oi.keyword_search(b, K)
    qv = np.stack([vec[int(kw["key"][q, 0])] for q in range(len(qs))])
    vp = S.vec_params(k=4096, ef=10, alpha=0.8, flags=VDEEP)
    okv, ocnt, ofound = oi.hybrid_search(b, qv, vp, K)
    came_back = 0
    for q in range(len(qs)):
        if int(kw_cnt[q]) < K:                                               # the keyword Topster is not full
            continue
        x = int(kw["key"][q, 0])
        c = int(ocnt[q])
        row = [i for i in range(c) if int(okv["key"][q, i]) == x]
        came_back += bool(row) and int(okv["text_match_score"][q, row[0]]) == 0
    assert came_back > 0
    kv, cnt, found = gi.hybrid_search(b, qv, vp, K)
    assert_kv_equal(kv, cnt, found, okv, ocnt, ofound)


@pytest.mark.gpu
def test_hybrid_keep_all_ids(vc):
    # all_result_ids of a deep hybrid query (src/index.cpp:4215-4219): the ids of every keyword combination plus the vector search's
    # ids. The expected set is built from the posting lists and the oracle's kNN answer; the ordinary path must keep the same set
    n, dim, vec, fd, pts, gi, oi = vc
    combos = [S.Combo([[0]], 1), S.Combo([[4]], 1, total_cost=1)]
    qv = synth.make_vectors(1, dim, 55).numpy()
    lo = fd.flat.list_off.astype(np.int64)
    od, olab, on, _ = oi.knn(qv, 2000, 10)
    expect = np.union1d(np.union1d(fd.flat.ids[lo[0]:lo[1]], fd.flat.ids[lo[4]:lo[5]]), olab[0, :on[0]]).tolist()
    res = []
    for K, flags in ((1000, capi.QFLAG_KEEP_ALL_IDS), (3000, capi.QFLAG_KEEP_ALL_IDS | DEEP)):
        b = S.KwBatch([S.Query(list(combos), sort=TEXT, topk=K, flags=S.FLAG_PRIORITIZE_EXACT_MATCH | flags)], [0])
        vp = S.vec_params(k=2000, ef=10, alpha=0.5, flags=VDEEP)
        kv, cnt, found = gi.hybrid_search(b, qv, vp, K)
        assert_kv_equal(kv, cnt, found, *oi.hybrid_search(b, qv, vp, K))
        assert int(found[0]) == len(expect)
        if not ON_DOUBLE:         # the test double keeps no all_result_ids: they live in device memory (tsgpu_all_result_ids_last)
            res.append(gi.all_result_ids_last(0, n).tolist())
            assert res[-1] == expect
    assert int(cnt[0]) > 1024


def _fuse(ix, b, kw, stride, qv, vp):
    kw_kv, kw_cnt, kw_found = kw
    nq = b.n_queries
    searched = np.ones(nq, np.uint32)
    out = np.zeros((nq, stride), S.KV_DTYPE)
    cnt, found = np.zeros(nq, np.uint32), np.zeros(nq, np.uint32)
    s = b.struct()
    q = np.ascontiguousarray(qv, np.float32)
    args = (C.byref(s), C.c_void_p(kw_kv.ctypes.data), C.c_uint32(kw_kv.shape[1]), C.c_void_p(kw_cnt.ctypes.data), C.c_void_p(kw_found.ctypes.data),
            C.c_void_p(searched.ctypes.data), C.c_void_p(q.ctypes.data), C.byref(vp), C.c_void_p(out.ctypes.data), C.c_uint32(stride),
            C.c_void_p(cnt.ctypes.data), C.c_void_p(found.ctypes.data))
    if isinstance(ix, ol.OracleIndex):
        assert ix.L.tso_hybrid_fuse_batch(ix.h, *args, 1) == 0
    else:
        capi._ck(ix.L.tsgpu_hybrid_fuse_batch(ix.h, *args))
    return out, cnt, found


@pytest.mark.gpu
def test_hybrid_fuse_batch_with_deep_keyword_topsters(vc):
    n, dim, vec, fd, pts, gi, oi = vc
    rng = np.random.default_rng(21)
    b = hybrid_batch(rng, fd, 9, 2600, [np.unique(rng.integers(0, n, 3000)).astype(np.uint32)])
    kw = oi.keyword_search(b, 2600)                                         # the oracle's deep keyword Topsters
    assert int(kw[1].max()) > 1024
    qv = synth.make_vectors(b.n_queries, dim, 22).numpy()
    for vp in (S.vec_params(k=2000, ef=10, alpha=0.3, flags=VDEEP), S.vec_params(k=300, ef=10, alpha=0.8, flags=VDEEP)):
        got = _fuse(gi, b, kw, 2600, qv, vp)
        want = _fuse(oi, b, kw, 2600, qv, vp)
        assert_kv_equal(*got, *want)


@pytest.mark.gpu
def test_mixed_batches(vc):
    n, dim, vec, fd, pts, gi, oi = vc
    rng = np.random.default_rng(5)
    plain = hybrid_batch(rng, fd, 8, 200, [], rerank_half=True).queries
    for q in plain:
        q.flags &= ~DEEP
    deeps = hybrid_batch(rng, fd, 3, 3000, []).queries
    mixed = S.KwBatch(plain[:4] + deeps + plain[4:], [0])
    qv_plain = synth.make_vectors(8, dim, 8).numpy()
    qv = np.concatenate([qv_plain[:4], synth.make_vectors(3, dim, 9).numpy(), qv_plain[4:]])
    vp = S.vec_params(k=600, ef=10, alpha=0.3, flags=VDEEP)
    kv, cnt, found = gi.hybrid_search(mixed, qv, vp, 3000)
    assert_kv_equal(kv, cnt, found, *oi.hybrid_search(mixed, qv, vp, 3000))
    keep = [0, 1, 2, 3, 7, 8, 9, 10]
    for vp0 in (vp, S.vec_params(k=600, ef=10, alpha=0.3)):            # without the deep queries; without the bit
        kv0, cnt0, found0 = gi.hybrid_search(S.KwBatch(plain, [0]), qv_plain, vp0, 3000)
        assert cnt[keep].tolist() == cnt0.tolist() and found[keep].tolist() == found0.tolist()
        for i, q in enumerate(keep):
            assert kv[q, :cnt[q]].tobytes() == kv0[i, :cnt0[i]].tobytes(), q
    # vector search: the same
    vb = S.KwBatch([S.Query([], sort=VSORTS[0], topk=100), deep(S.Query([], sort=VSORTS[1]), 2000), S.Query([], sort=VSORTS[2], topk=10)], [0])
    vq = synth.make_vectors(3, dim, 10).numpy()
    vp = S.vec_params(k=0, fetch_size=2000, flags=VDEEP)
    kv, cnt, found = gi.vector_search(vb, vq, vp, 2000)
    assert_kv_equal(kv, cnt, found, *oi.vector_search(vb, vq, vp, 2000))
    kv0, cnt0, found0 = gi.vector_search(S.KwBatch([vb.queries[0], vb.queries[2]], [0]), vq[[0, 2]], vp, 2000)
    assert cnt[[0, 2]].tolist() == cnt0.tolist()
    for i, q in enumerate((0, 2)):
        assert kv[q, :cnt[q]].tobytes() == kv0[i, :cnt0[i]].tobytes()
    # a kv_stride below K truncates
    kvt, cntt, foundt = gi.vector_search(vb, vq, vp, 1500)
    assert cntt.tolist() == np.minimum(cnt, 1500).tolist() and foundt.tolist() == found.tolist()
    assert kvt[1, :1500].tobytes() == kv[1, :1500].tobytes()


@pytest.mark.gpu
@device_only
def test_device_rejections(vc):
    n, dim, vec, fd, pts, gi, oi = vc
    qv = synth.make_vectors(1, dim, 3).numpy()
    b = S.KwBatch([deep(S.Query([S.Combo([[0]], 1)], sort=TEXT), 2000)], [0])
    plain = S.KwBatch([S.Query([S.Combo([[0]], 1)], sort=TEXT, topk=100)], [0])

    def still_answers():
        vp = S.vec_params(k=1500, ef=10, flags=VDEEP)
        assert_kv_equal(*gi.hybrid_search(b, qv, vp, 2000), *oi.hybrid_search(b, qv, vp, 2000))

    with pytest.raises(capi.TsgpuError, match="DEEP_TOPSTER"):              # without the bit: today's errors
        gi.vector_search(b, qv, S.vec_params(k=10), 16)
    still_answers()
    with pytest.raises(capi.TsgpuError, match="DEEP_TOPSTER"):
        gi.hybrid_search(b, qv, S.vec_params(k=10), 16)
    still_answers()
    with pytest.raises(capi.TsgpuError, match="hybrid k"):
        gi.hybrid_search(plain, qv, S.vec_params(k=2000), 16)
    still_answers()
    for fn in (gi.vector_search, gi.hybrid_search):                         # with it: the vector stage's bound
        with pytest.raises(capi.TsgpuError, match="max\\(ef,k\\)"):
            fn(b, qv, S.vec_params(k=5000, flags=VDEEP), 16)
        still_answers()
        with pytest.raises(capi.TsgpuError, match="max\\(ef,k\\)"):
            fn(b, qv, S.vec_params(k=100, ef=4097, flags=VDEEP), 16)
        still_answers()
    st = gi.stats()
    assert st["deep_fuse_bytes"] > 0
