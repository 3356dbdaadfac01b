"""Deep Topsters (TSGPU_QFLAG_DEEP_TOPSTER): keyword, wildcard and scored-ids queries whose Topster is larger than
TSGPU_MAX_TOPK, as deep pagination needs them (page 5 at 250 per page is a Topster of 1,250). Every answer is compared with the
oracle, which runs the reference's Topster at any capacity: ids, scores, found, query_index and counts bit-equal."""
import ctypes as C
import os

import numpy as np
import pytest

import hostlib
import oracle_lib as ol
from typesense_b200 import capi, hostapi, structs as S, synth
from test_gpu_parity import assert_kv_equal
from test_oracle_ref import random_batch, small_collection  # noqa: F401

DEEP = capi.QFLAG_DEEP_TOPSTER
ON_DOUBLE = os.environ.get("TSGPU_TEST_DOUBLE") == "1"
device_only = pytest.mark.skipif(ON_DOUBLE, reason="asserts what only the device library does")


def deep(q: S.Query, k: int) -> S.Query:
    q.topk = k
    q.flags |= DEEP
    return q


def scored_ids(ix, b: S.KwBatch, scores: np.ndarray, stride: int):
    """tsgpu_scored_ids_search_batch on the device index, tso_scored_ids_search_batch on the oracle"""
    kv = np.zeros((b.n_queries, stride), S.KV_DTYPE)
    cnt = np.zeros(b.n_queries, np.uint32)
    found = np.zeros(b.n_queries, np.uint32)
    s = b.struct()
    sc = np.ascontiguousarray(scores, np.int64)
    if isinstance(ix, ol.OracleIndex):
        assert ix.L.tso_scored_ids_search_batch(ix.h, C.byref(s), C.c_void_p(sc.ctypes.data), C.c_void_p(kv.ctypes.data), stride,
                                                cnt.ctypes.data_as(S.u32p), found.ctypes.data_as(S.u32p), 1) == 0
    else:
        capi._ck(ix.L.tsgpu_scored_ids_search_batch(ix.h, C.byref(s), sc.ctypes.data, kv.ctypes.data, stride, cnt.ctypes.data, found.ctypes.data))
    return kv, cnt, found


@pytest.fixture(scope="module")
def coll(small_collection):
    n_docs, fds, pts = small_collection
    flats = [fd.flat for fd in fds]
    gi = capi.GpuIndex(n_docs, 0)
    for f in flats:
        gi.load_field(f)
    gi.load_sort_column(pts)
    oi = ol.OracleIndex(n_docs, flats, [pts])
    yield n_docs, fds, flats, pts, gi, oi
    gi.close()


TIED = ((S.SORT_NUMERIC, 0, -1, 0), (S.SORT_NONE, -1, 1, 0), (S.SORT_NONE, -1, 1, 0))        # 50 distinct values over 4000 docs
TEXT = ((S.SORT_TEXT_MATCH, -1, 1, 0), (S.SORT_NUMERIC, 0, 1, 1), (S.SORT_SEQ_ID, -1, -1, 0))


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1025, 4096, 1_000_000])
def test_keyword_single_combination(coll, k):
    n_docs, fds, flats, pts, gi, oi = coll
    qs = []
    for t in range(6):
        for sort in (TIED, TEXT):
            qs.append(deep(S.Query([S.Combo([[t, S.NO_LIST, S.NO_LIST]], 1)], sort=sort), k))
    qs.append(deep(S.Query([S.Combo([[0, 0, 0], [1, 1, 1]], 2)], sort=TIED, num_query_tokens=2), k))
    b = S.KwBatch(qs, [0, 1, 2])
    stride = min(k, n_docs)
    kv, cnt, found = gi.keyword_search(b, stride)
    okv, ocnt, ofound = oi.keyword_search(b, stride)
    assert_kv_equal(kv, cnt, found, okv, ocnt, ofound)
    assert int(cnt.max()) > 1024


@pytest.mark.gpu
def test_overlapping_combinations_keep_the_best_entry_and_the_later_tie(coll):
    # a document matching several combinations enters once: with the greater KV (text-match sort, the cost-0 combination scores
    # higher), or, when the KV is equal (no text-match clause), from the later combination, which decides its query_index
    n_docs, fds, flats, pts, gi, oi = coll
    combos = [S.Combo([[0, S.NO_LIST, S.NO_LIST]], 1), S.Combo([[0, S.NO_LIST, S.NO_LIST], [1, S.NO_LIST, S.NO_LIST]], 1, total_cost=1),
              S.Combo([[2, S.NO_LIST, S.NO_LIST]], 1, total_cost=2), S.Combo([[S.NO_LIST, 0, S.NO_LIST]], 1, total_cost=2)]
    qs = [deep(S.Query(list(combos), sort=TEXT), 3000), deep(S.Query(list(combos), sort=TIED), 3000),
          deep(S.Query(list(combos[::-1]), sort=((S.SORT_SEQ_ID, -1, 1, 0), (S.SORT_NONE, -1, 1, 0), (S.SORT_NONE, -1, 1, 0))), 1500)]
    b = S.KwBatch(qs, [0, 1, 2])
    kv, cnt, found = gi.keyword_search(b, 3000)
    okv, ocnt, ofound = oi.keyword_search(b, 3000)
    assert_kv_equal(kv, cnt, found, okv, ocnt, ofound)
    assert len(set(okv["query_index"][1, :ocnt[1]].tolist())) > 1


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(3))
def test_filters_exclusions_and_field_shapes(coll, seed):
    # inline / persistent / empty filters, exclusions, dropped tokens, an array field, three fields, three sort clauses with
    # missing_first (random_batch), all with deep Topsters
    n_docs, fds, flats, pts, gi, oi = coll
    rng = np.random.default_rng(4100 + seed)
    filters = [np.unique(rng.integers(0, n_docs, 2600)).astype(np.uint32), np.arange(0, n_docs, 3, dtype=np.uint32), np.zeros(0, np.uint32)]
    b = random_batch(rng, fds, 24, filters)
    for q in b.queries:
        deep(q, int(rng.choice([1025, 1500, 5000])))
    b = S.KwBatch(b.queries, [0, 1, 2], filters)
    kv, cnt, found = gi.keyword_search(b, 5000)
    okv, ocnt, ofound = oi.keyword_search(b, 5000)
    assert_kv_equal(kv, cnt, found, okv, ocnt, ofound)
    handles = [gi.filter_create(f) for f in filters]
    bh = b.with_filter_handles(handles)
    kv, cnt, found = gi.keyword_search(bh, 5000)
    assert_kv_equal(kv, cnt, found, okv, ocnt, ofound)
    assert int(cnt.max()) > 1024


@pytest.fixture(scope="module")
def big():
    n_docs = 120_000
    fd = synth.make_string_field(n_docs, 2000, 3, 8, seed=31)
    pts = synth.make_points(n_docs, 17, hi=40, missing_frac=0.02)
    gi = capi.GpuIndex(n_docs, 0)
    gi.load_field(fd.flat)
    gi.load_sort_column(pts)
    oi = ol.OracleIndex(n_docs, [fd.flat], [pts])
    yield n_docs, fd, pts, gi, oi
    gi.close()


@pytest.mark.gpu
def test_wildcard(big):
    # unfiltered over 120 k docs (many units feed one query), filtered, and sorted by a column with 40 distinct values
    n_docs, fd, pts, gi, oi = big
    rng = np.random.default_rng(8)
    filters = [np.unique(rng.integers(0, n_docs, 30000)).astype(np.uint32)]
    sorts = [((S.SORT_NUMERIC, 0, 1, 0), (S.SORT_NONE, -1, 1, 0), (S.SORT_NONE, -1, 1, 0)),
             ((S.SORT_NUMERIC, 0, -1, 1), (S.SORT_SEQ_ID, -1, 1, 0), (S.SORT_NONE, -1, 1, 0)),
             ((S.SORT_TEXT_MATCH, -1, 1, 0), (S.SORT_NUMERIC, 0, 1, 0), (S.SORT_NONE, -1, 1, 0))]
    qs = [deep(S.Query([], sort=sorts[0]), 10_000), deep(S.Query([], sort=sorts[1], excl=list(range(0, 5000, 3))), 2048),
          deep(S.Query([], sort=sorts[2], filter=0), 25_000), deep(S.Query([], sort=sorts[0], filter=0), 1025)]
    b = S.KwBatch(qs, [0], filters)
    kv, cnt, found = gi.wildcard_search(b, 25_000)
    okv, ocnt, ofound = oi.wildcard_search(b, 25_000)
    assert_kv_equal(kv, cnt, found, okv, ocnt, ofound, check_query_index=False)
    assert cnt.tolist()[:3] == [10_000, 2048, 25_000]


@pytest.mark.gpu
def test_scored_ids(big):
    # phrase-only queries (Index::do_phrase_search): the ids that matched the phrase with their match scores
    n_docs, fd, pts, gi, oi = big
    rng = np.random.default_rng(9)
    filters = [np.unique(rng.integers(0, n_docs, 6000)).astype(np.uint32), np.unique(rng.integers(0, n_docs, 40000)).astype(np.uint32)]
    scores = rng.integers(0, 4, sum(len(f) for f in filters)).astype(np.int64) * 1000
    sort = ((S.SORT_TEXT_MATCH, -1, 1, 0), (S.SORT_NUMERIC, 0, 1, 0), (S.SORT_NONE, -1, 1, 0))
    qs = [deep(S.Query([], sort=sort, filter=0), 5000), deep(S.Query([], sort=sort, filter=1, excl=list(range(0, 3000, 2))), 30_000),
          S.Query([], sort=sort, filter=1, topk=250)]
    b = S.KwBatch(qs, [0], filters)
    got = scored_ids(gi, b, scores, 30_000)
    want = scored_ids(oi, b, scores, 30_000)
    assert_kv_equal(*got, *want, check_query_index=False)


@pytest.mark.gpu
def test_mixed_batches_prefix_and_repeat(coll):
    n_docs, fds, flats, pts, gi, oi = coll
    rng = np.random.default_rng(77)
    plain = random_batch(rng, fds, 16, ()).queries
    deeps = [deep(S.Query([S.Combo([[t, t if fds[1].flat.df(t) else S.NO_LIST, S.NO_LIST]], 1)], sort=TIED), 3000) for t in range(3)]
    mixed = S.KwBatch(plain[:8] + deeps + plain[8:], [0, 1, 2])
    kv, cnt, found = gi.keyword_search(mixed, 3000)
    okv, ocnt, ofound = oi.keyword_search(mixed, 3000)
    assert_kv_equal(kv, cnt, found, okv, ocnt, ofound)
    # the ordinary queries' records are byte-identical to the same batch without the deep ones
    kv0, cnt0, found0 = gi.keyword_search(S.KwBatch(plain, [0, 1, 2]), 3000)
    keep = list(range(8)) + list(range(11, 19))
    assert cnt[keep].tolist() == cnt0.tolist() and found[keep].tolist() == found0.tolist()
    for i, q in enumerate(keep):
        assert kv[q, :cnt[q]].tobytes() == kv0[i, :cnt0[i]].tobytes(), q
    # a kv_stride below K truncates
    kvt, cntt, foundt = gi.keyword_search(mixed, 1500)
    assert cntt.tolist() == np.minimum(cnt, 1500).tolist() and foundt.tolist() == found.tolist()
    for q in range(mixed.n_queries):
        assert kvt[q, :cntt[q]].tobytes() == kv[q, :cntt[q]].tobytes()
    # K = 1025 with the flag is the K = 1024 result plus one entry; repeated calls give identical records
    one = S.Query([S.Combo([[0, S.NO_LIST, S.NO_LIST]], 1), S.Combo([[1, S.NO_LIST, S.NO_LIST]], 1, total_cost=1)], sort=TIED)
    k1024, c1024, f1024 = gi.keyword_search(S.KwBatch([S.Query(one.combos, sort=TIED, topk=1024)], [0, 1, 2]), 1025)
    k1025, c1025, f1025 = gi.keyword_search(S.KwBatch([deep(S.Query(one.combos, sort=TIED), 1025)], [0, 1, 2]), 1025)
    assert c1024[0] == 1024 and c1025[0] == 1025 and f1024[0] == f1025[0]
    assert k1025[0, :1024].tobytes() == k1024[0, :1024].tobytes()
    again = gi.keyword_search(S.KwBatch([deep(S.Query(one.combos, sort=TIED), 1025)], [0, 1, 2]), 1025)
    assert again[0].tobytes() == k1025.tobytes()


@pytest.mark.gpu
def test_keep_all_ids_with_a_deep_query(coll):
    n_docs, fds, flats, pts, gi, oi = coll
    off = np.arange(n_docs + 1, dtype=np.uint64)
    vals = (np.arange(n_docs) % 37).astype(np.uint32)
    f = gi.load_facet(37, off, vals)
    combos = [S.Combo([[0, S.NO_LIST, S.NO_LIST]], 1), S.Combo([[3, 3, S.NO_LIST]], 1, total_cost=1)]
    res = []
    for k, flags in ((250, capi.QFLAG_KEEP_ALL_IDS), (4000, capi.QFLAG_KEEP_ALL_IDS | DEEP)):
        q = S.Query(list(combos), sort=TEXT, topk=k, flags=S.FLAG_PRIORITIZE_EXACT_MATCH | flags)
        b = S.KwBatch([q], [0, 1, 2])
        kv, cnt, found = gi.keyword_search(b, k)
        assert_kv_equal(kv, cnt, found, *oi.keyword_search(b, k))
        if ON_DOUBLE:         # the test double keeps no all_result_ids: they live in device memory (tsgpu_all_result_ids_last)
            res.append(int(found[0]))
            continue
        res.append((int(found[0]), gi.all_result_ids_last(0, n_docs).tolist(), gi.facet_counts_last(f, 1, 37)[0].tobytes()))
    assert res[0] == res[1] and int(cnt[0]) > 1024


@pytest.mark.gpu
@device_only
def test_device_rejections_and_limits(coll):
    n_docs, fds, flats, pts, gi, oi = coll
    with pytest.raises(capi.TsgpuError):                                   # without the flag the cap stays
        gi.keyword_search(S.KwBatch([S.Query([S.Combo([[0, 0, 0]], 1)], topk=2000)], [0, 1, 2]), 4)
    with pytest.raises(capi.TsgpuError):
        gi.wildcard_search(S.KwBatch([S.Query([], topk=2000)], [0]), 4)
    vec = synth.make_vectors(500, 16, 3).numpy()
    gv = capi.GpuIndex(500, 0)
    gv.load_hnsw(ol.hnsw_build(vec, 8, 40, 100))
    for k in (200, 2000):
        b = S.KwBatch([deep(S.Query([S.Combo([[0]], 1)]), k)], [0])
        with pytest.raises(capi.TsgpuError, match="DEEP_TOPSTER"):
            gv.vector_search(b, vec[:1], S.vec_params(k=10), 16)
        with pytest.raises(capi.TsgpuError, match="DEEP_TOPSTER"):
            gv.hybrid_search(b, vec[:1], S.vec_params(k=10), 16)
        kw = np.zeros((1, 16), S.KV_DTYPE)
        one, qv = np.ones(1, np.uint32), np.ascontiguousarray(vec[:1], np.float32)
        out, oc, of = np.zeros((1, 16), S.KV_DTYPE), np.zeros(1, np.uint32), np.zeros(1, np.uint32)
        s, vp = b.struct(), S.vec_params(k=10)
        with pytest.raises(capi.TsgpuError, match="DEEP_TOPSTER"):
            capi._ck(gv.L.tsgpu_hybrid_fuse_batch(gv.h, C.byref(s), C.c_void_p(kw.ctypes.data), C.c_uint32(16), C.c_void_p(one.ctypes.data),
                                                  C.c_void_p(one.ctypes.data), C.c_void_p(one.ctypes.data), C.c_void_p(qv.ctypes.data), C.byref(vp),
                                                  C.c_void_p(out.ctypes.data), C.c_uint32(16), C.c_void_p(oc.ctypes.data), C.c_void_p(of.ctypes.data)))
    gv.close()
    # the index still answers after the rejections
    kv, cnt, found = gi.keyword_search(S.KwBatch([deep(S.Query([S.Combo([[0, 0, 0]], 1)]), 2000)], [0, 1, 2]), 2000)
    okv, ocnt, ofound = oi.keyword_search(S.KwBatch([deep(S.Query([S.Combo([[0, 0, 0]], 1)]), 2000)], [0, 1, 2]), 2000)
    assert_kv_equal(kv, cnt, found, okv, ocnt, ofound)
    st = gi.stats()
    assert st["deep_entries"] >= ofound[0] and st["deep_bytes"] > 0


@pytest.mark.gpu
@device_only
def test_one_million_docs_sample():
    n_docs = 1_000_000
    fd = synth.make_string_field(n_docs, 100_000, 4, 12, seed=7, device="cuda")
    pts = synth.make_points(n_docs, 13, hi=200)
    gi = capi.GpuIndex(n_docs, 0)
    gi.load_field(fd.flat)
    gi.load_sort_column(pts)
    oi = ol.OracleIndex(n_docs, [fd.flat], [pts])
    toks = synth.sample_queries(fd, 6, 2, 5)
    qs = [deep(S.Query([S.Combo([[0]], 1)], sort=TIED), 100_000), deep(S.Query([S.Combo([[3]], 1), S.Combo([[3], [4]], 2, total_cost=1)], sort=TEXT), 20_000)]
    qs += [deep(S.Query([S.Combo([[int(t)] for t in r], 1)], sort=TEXT, num_query_tokens=2), 5000) for r in toks]
    b = S.KwBatch(qs, [0])
    kv, cnt, found = gi.keyword_search(b, 100_000)
    okv, ocnt, ofound = oi.keyword_search(b, 100_000, threads=8)
    assert_kv_equal(kv, cnt, found, okv, ocnt, ofound)
    w = S.KwBatch([deep(S.Query([], sort=TIED), 50_000)], [0])
    kv, cnt, found = gi.wildcard_search(w, 50_000)
    okv, ocnt, ofound = oi.wildcard_search(w, 50_000)
    assert_kv_equal(kv, cnt, found, okv, ocnt, ofound, check_query_index=False)
    gi.close()


# ---- host layer: topster_size above TSGPU_MAX_TOPK takes the deep path; vector and hybrid requests keep the cap
def host_collection():
    n_docs, vocab = 6000, 300
    fd = synth.make_string_field(n_docs, vocab, 4, 10, seed=11)
    pts = synth.make_points(n_docs, 5, hi=30)
    words = synth.vocab_words(vocab)
    rng = np.random.default_rng(3)
    taken = set(words)
    qs = []
    for row in synth.sample_queries(fd, 24, 2, 21):
        q = [words[int(t)] for t in row]
        if rng.random() < 0.4:
            q[1] = synth.misspell(q[1], rng, taken)
        qs.append(q)
    qs += [[words[0]], [words[1], words[2]]]
    return n_docs, fd, pts, words, qs


def host_search(lib_path, topster_size, stride, with_vectors=False):
    n_docs, fd, pts, words, qs = host_collection()
    hi = hostapi.HostIndex(n_docs, 0, lib_path)
    hi.add_field_flat("title", words, fd.flat)
    hi.add_sort_column("points", pts)
    qv = None
    if with_vectors:
        vec = synth.make_vectors(n_docs, 16, 4).numpy()
        hi.device_index().load_hnsw(ol.hnsw_build(vec, 8, 40, 100))
        qv = synth.make_vectors(len(qs), 16, 5).numpy()
    opt = hostapi.Options(topster_size=topster_size, n_threads=2, vec_fetch_size=100)
    kv, cnt, found, _ = hi.multi_search("title", "points", qs, stride, None, qv, opt)
    hi.close()
    return kv, cnt, found


def test_host_layer_deep_topster_on_the_oracle_double():
    lib = hostlib.build_host_cpu()
    kv, cnt, found = host_search(lib, 5000, 5000)
    assert int(cnt.max()) > 1024                                           # the host layer no longer clamps to 1024
    assert cnt.tolist() == np.minimum(found, 5000).tolist()
    kv250, cnt250, _ = host_search(lib, 250, 250)
    for q in range(len(cnt)):
        assert kv[q, :cnt250[q]].tobytes() == kv250[q, :cnt250[q]].tobytes()
    # a hybrid request keeps the 1024 cap: topster_size 5000 returns what topster_size 1024 returns
    h5000 = host_search(lib, 5000, 5000, with_vectors=True)
    h1024 = host_search(lib, 1024, 5000, with_vectors=True)
    for q in range(len(h5000[1])):
        assert h5000[0][q, :h5000[1][q]].tobytes() == h1024[0][q, :h1024[1][q]].tobytes(), q
    assert h5000[1].tolist() == h1024[1].tolist() and h5000[2].tolist() == h1024[2].tolist() and int(h5000[1].max()) <= 1024


@pytest.mark.gpu
@pytest.mark.skipif(ON_DOUBLE, reason="links the real libtsgpu.so; its CPU-arm half is test_host_layer_deep_topster_on_the_oracle_double")
def test_host_layer_deep_topster_on_the_gpu():
    cpu = host_search(hostlib.build_host_cpu(), 5000, 5000)
    gpu = host_search(hostapi.build_gpu_lib(), 5000, 5000)
    assert gpu[1].tolist() == cpu[1].tolist() and gpu[2].tolist() == cpu[2].tolist()
    for q in range(len(gpu[1])):
        n = int(gpu[1][q])
        assert gpu[0][q, :n].tobytes() == cpu[0][q, :n].tobytes(), q
    assert int(gpu[1].max()) > 1024
    # a hybrid request keeps the 1024 cap: topster_size 5000 returns what topster_size 1024 returns
    h5000 = host_search(hostapi.build_gpu_lib(), 5000, 5000, with_vectors=True)
    h1024 = host_search(hostapi.build_gpu_lib(), 1024, 5000, with_vectors=True)
    for q in range(len(h5000[1])):
        assert h5000[0][q, :h5000[1][q]].tobytes() == h1024[0][q, :h1024[1][q]].tobytes(), q
    assert h5000[1].tolist() == h1024[1].tolist() and h5000[2].tolist() == h1024[2].tolist()
