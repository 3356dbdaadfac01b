"""Keyword scoring on long documents, long arrays and long queries (tests/longdocs.py builds the collection):
  - the oracle against the reference's own compiled scoring (oracle/_ref; stored digests in tests/golden/ref_long_documents.json
    where it is not built), on combinations and on the phrase / exact / prefix filters, CPU only;
  - libtsgpu against the oracle bit for bit (-m gpu): every field class (plain with 16-bit positions: the register scorer;
    plain with positions past 65535: score_field_plain; arrays: score_field), 1-16 token rows, exactly 32 lists, K up to
    1024 and deep K, with the bitmap path of the all-dense combinations on and off;
  - a metamorphic test of the scorer switch: one extra long document that no query touches moves a field from the
    register scorer to score_field_plain, and no record may change;
  - TEST_F(CollectionTest, SearchLargeTextField) (test/collection_test.cpp:2119-2176) replayed on the oracle and the device.
Positions past 65535 wrap in Match's uint16 offsets (src/posting_list.cpp:906); the collection places query tokens at
65,535, 65,536 (offset MAX_DISPLACEMENT), 65,537 (offset 0), 131,073-131,075, across the wrap and as a last token."""
import contextlib
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import longdocs as LD
import oracle_lib as ol
import refflow
from test_gpu_parity import assert_kv_equal
from test_oracle_ref import _ref_combo
from typesense_b200 import capi, structs as S

ON_DOUBLE = os.environ.get("TSGPU_TEST_DOUBLE") == "1"
GOLD = os.path.join(os.path.dirname(__file__), "golden")
NL = S.NO_LIST
P16, PLONG, ARR = 0, 1, 2
FIELDS8 = [P16, PLONG, ARR, P16, PLONG, ARR, P16, PLONG]      # loaded as eight fields (8 x 4 rows = 32 lists)
SORTS = [((S.SORT_TEXT_MATCH, -1, 1, 0), (S.SORT_NUMERIC, 0, 1, 0), (S.SORT_SEQ_ID, -1, 1, 0)),
         ((S.SORT_TEXT_MATCH, -1, 1, 0), (S.SORT_NUMERIC, 0, -1, 1), (S.SORT_SEQ_ID, -1, -1, 0)),
         ((S.SORT_NUMERIC, 0, -1, 1), (S.SORT_TEXT_MATCH, -1, 1, 0), (S.SORT_NONE, -1, 1, 0))]


@pytest.fixture(scope="module")
def lc():
    return LD.LongCollection()


def filters_of(lc):
    rng = np.random.default_rng(4)
    return [np.unique(np.append(rng.integers(0, lc.n_docs, lc.n_docs // 2), [lc.LONG_WRAP, lc.LONG_LAST, lc.ARRAY_WIDE])).astype(np.uint32),
            np.arange(0, lc.n_docs, 3, dtype=np.uint32),
            np.asarray([lc.LONG_WRAP, lc.LONG_LAST, lc.LONG_GAPS, lc.ARRAY_WIDE], np.uint32)]


def make_batch(lc, rng, flats, fids, n_queries, max_rows, topk, flags=0, filters=()):
    """flats[i]: the field of fids[i]. Queries from contiguous spans of the collection's documents: duplicate tokens, typo-cost combinations that share hits,
    dropped rows, flags 0-7, match types, field weights, numeric sorts with many ties, exclusions and filters."""
    F = len(fids)
    qs = []
    for qi in range(n_queries):
        nt = max_rows if qi == 0 else int(rng.integers(1, max_rows + 1))
        toks = lc.span(rng, nt, 1.0 if qi == 0 else 0.35) or [0]         # the first query spans a long document: max_rows rows
        nt = len(toks)
        if nt > 1 and rng.random() < 0.25:
            toks[int(rng.integers(1, nt))] = toks[0]                          # a duplicate query token
        combos = []
        for c in range(int(rng.integers(1, 4))):
            ct = list(toks)
            if c:
                ct[int(rng.integers(0, nt))] = int(rng.integers(0, 40))      # a typo candidate: a frequent token
            rows = []
            for t in ct:
                row = [t if fl.df(t) > 0 else NL for fl in flats]
                if all(x == NL for x in row):
                    row = [0 if fl.df(0) > 0 else NL for fl in flats]
                rows.append(row)
            n_req = nt - int(rng.integers(1, min(3, nt - 1) + 1)) if nt > 2 and rng.random() < 0.3 else nt
            combos.append(S.Combo(rows, n_req, total_cost=c * int(rng.integers(1, 3))))
        q = S.Query(combos, topk=topk, flags=int(rng.integers(0, 8)) | flags, match_type=int(rng.integers(0, 3)),
                    num_query_tokens=nt, field_weight=[int(x) for x in rng.integers(1, 16, F)], sort=SORTS[int(rng.integers(0, 3))])
        if filters and rng.random() < 0.35:
            q.filter = int(rng.integers(0, len(filters)))
        if rng.random() < 0.2:
            q.excl = np.unique(rng.integers(0, lc.n_docs, 300)).tolist()
        qs.append(q)
    return S.KwBatch(qs, list(range(F)), filters)


# ------------------------------------------------------------------ the collection's encoding (CPU)
def test_collection_covers_the_wrap(lc):
    f16, flong, farr = lc.flats
    assert int(f16.positions.max()) < 65536 and not f16.is_array
    assert int(flong.positions.max()) >= 131075 and not flong.is_array
    assert farr.is_array

    def offsets(f, tok, doc):
        a, b = int(f.list_off[tok]), int(f.list_off[tok + 1])
        i = a + int(np.searchsorted(f.ids[a:b], doc))
        assert int(f.ids[i]) == doc
        return f.positions[int(f.pos_off[i]):int(f.pos_off[i + 1])].tolist()
    for m, p in LD.WRAP_PLACEMENTS:
        assert p in offsets(flong, LD.MARK + m, lc.LONG_WRAP)
    assert offsets(flong, LD.MARK + 9, lc.LONG_LAST)[-2:] == [65540, 0]           # the last token, past 65535
    assert 65536 in offsets(flong, LD.MARK + 1, lc.LONG_GAPS)
    wide = offsets(farr, LD.MARK + 9, lc.ARRAY_WIDE)
    assert [wide[i] for i in range(2, len(wide), 3)][-3:] == [65536, 65537, 69999]  # element indices past 65535
    assert (np.diff(flong.list_off.astype(np.int64)) >= 64).sum() > 50             # dense lists


# ------------------------------------------------------------------ oracle vs the reference's compiled scoring (CPU)
@pytest.fixture(scope="module")
def answers():
    a = ol.RefAnswers("long_documents")
    yield a
    a.save()


@pytest.mark.parametrize("seed", range(3))
def test_ref_keyword_combo_long(lc, answers, seed):
    """or_iterator_t::intersect + score_results2 of the reference against OracleIndex.keyword_combo, both filter paths."""
    rng = np.random.default_rng(200 + seed)
    filters = filters_of(lc)
    ix = ol.OracleIndex(lc.n_docs, lc.flats, [lc.pts])
    b = make_batch(lc, rng, lc.flats, [P16, PLONG, ARR], 12, 10, 250, filters=filters)
    total = 0
    for q in range(b.n_queries):
        for c in range(int(b.q_combo_off[q]), int(b.q_combo_off[q + 1])):
            ids, sc, nkm = ix.keyword_combo(b, q, c)
            for use_fit in (0, 1):
                block = int(rng.choice([4, 256]))
                answers.check(f"combo/{seed}/{q}/{c}/{use_fit}", [ids.tolist(), sc.tolist()],
                              lambda: [x.tolist() for x in _ref_combo(lc.flats, b, q, c, block=block, use_fit=use_fit, filters=filters)[:2]])
            total += len(ids)
    assert total > 30


def marker_batch(lc):
    """Queries on the placed tokens: pairs across the wrap, the 0 / MAX_DISPLACEMENT offsets, the last token past 65535,
    the array elements past index 65535, against each field class."""
    M = LD.MARK
    rows = [[9, 2], [9, 0], [9, 1], [2, 3], [3, 4, 10], [5, 6, 7, 8, 11], [0, 1, 2], [9], [1], [2, 9, 0, 1, 3, 4, 10, 5, 6, 7]]
    qs = []
    for i, r in enumerate(rows):
        toks = [M + m for m in r]
        qs.append(S.Query([S.Combo([[t] * 3 for t in toks], len(toks)), S.Combo([[t] * 3 for t in toks[:1]] + [[0, 0, 0]], 1, total_cost=1)],
                          topk=50, flags=i % 8, match_type=i % 3, num_query_tokens=len(toks), sort=SORTS[i % 3]))
    flats = lc.flats
    for q in qs:
        for c in q.combos:
            c.rows = [[t if flats[f].df(t) > 0 else NL for f, t in enumerate(row)] for row in c.rows]
    return S.KwBatch(qs, [P16, PLONG, ARR])


def test_ref_keyword_combo_markers(lc, answers):
    ix = ol.OracleIndex(lc.n_docs, lc.flats, [lc.pts])
    b = marker_batch(lc)
    hits = 0
    for q in range(b.n_queries):
        for c in range(int(b.q_combo_off[q]), int(b.q_combo_off[q + 1])):
            ids, sc, _ = ix.keyword_combo(b, q, c)
            for use_fit in (0, 1):
                answers.check(f"markers/{q}/{c}/{use_fit}", [ids.tolist(), sc.tolist()],
                              lambda: [x.tolist() for x in _ref_combo(lc.flats, b, q, c, block=16, use_fit=use_fit)[:2]])
            hits += int(np.isin(ids, [lc.LONG_WRAP, lc.LONG_LAST, lc.LONG_GAPS, lc.ARRAY_WIDE]).sum())
    assert hits >= 10


def idset_cases(lc, rng, fid, n_cases):
    """(lists, candidate ids): 1-4 tokens from a document's start (exact / prefix hits), a window (phrase hits) or shuffled;
    candidates are the lists' intersection, as at the reference's call sites"""
    f = lc.flats[fid]
    out = []
    while len(out) < n_cases:
        k = int(rng.integers(1, 5))
        mode = int(rng.integers(0, 3))
        if fid == ARR:
            d = int(rng.integers(0, lc.n_regular))
            elems = [e for e in lc.elems[d] if len(e.tok)]
            e = elems[int(rng.integers(0, len(elems)))].tok if rng.random() < 0.9 else lc.elems[lc.ARRAY_WIDE][65536].tok
            k = min(k, len(e))
            s = 0 if mode == 0 else int(rng.integers(0, len(e) - k + 1))
            lists = e[s:s + k]
        else:
            lists = np.asarray(lc.span(rng, k, 0.5) if mode else lc.docs[int(rng.integers(0, lc.n_regular))].tok[:k])
        lists = np.ascontiguousarray(lists[rng.permutation(len(lists))] if mode == 2 else lists, np.uint32)
        cand = None
        for l in lists:
            ids = f.ids[int(f.list_off[l]):int(f.list_off[l + 1])]
            cand = ids if cand is None else np.intersect1d(cand, ids)
        if len(lists) and cand is not None and len(cand):
            out.append((lists, np.ascontiguousarray(cand, np.uint32)))
    return out


IDSET_FNS = (("phrase", "tso_phrase_matches", "ref_plist_phrase_matches", "phrase_matches"),
             ("exact", "tso_exact_matches", "ref_plist_exact_matches", "exact_matches"),
             ("prefix", "tso_prefix_matches", "ref_plist_prefix_matches", "prefix_matches"))


def test_ref_phrase_exact_prefix_long(lc, answers):
    """get_phrase_matches / get_exact_matches / get_prefix_matches (src/posting_list.cpp) on the long plain field and the
    array field: the oracle's restatement against the reference's compiled code."""
    R, L = (ol.ref() if answers.live else None), ol.oracle()
    ix = ol.OracleIndex(lc.n_docs, lc.flats, [])
    rng = np.random.default_rng(31)
    hits = {n: 0 for n, *_ in IDSET_FNS}
    got, want = [], []
    for fid in (PLONG, ARR):
        for lists, ids in idset_cases(lc, rng, fid, 60):
            k = len(lists)
            if R is not None:
                pls = ol.ref_plists_of(lc.flats[fid], lists.tolist(), 256)
                hs = (C.c_void_p * k)(*[p.h for p in pls])
            for name, ofn, rfn, _ in IDSET_FNS:
                out = np.zeros(len(ids), np.uint32)
                n = getattr(L, ofn)(ix.h, fid, ol.p32(lists), k, ol.p32(ids), len(ids), ol.p32(out))
                got.append(out[:n].tolist())
                hits[name] += n
                if R is not None:
                    rout = np.zeros(len(ids), np.uint32)
                    rn = getattr(R, rfn)(hs, k, int(fid == ARR), ol.p32(ids), len(ids), ol.p32(rout))
                    want.append(rout[:rn].tolist())
    answers.check("phrase_exact_prefix", got, lambda: want)
    assert min(hits.values()) > 10, hits


# ------------------------------------------------------------------ SearchLargeTextField (oracle on the CPU, device with -m gpu)
LARGE_TEXT_SORT = ((S.SORT_TEXT_MATCH, -1, 1, 0), (S.SORT_NUMERIC, 0, 1, 0), (S.SORT_NONE, -1, 1, 0))   # _text_match, age DESC


def large_text_collection():
    docs = [json.loads(l) for l in open(os.path.join(GOLD, "large_text_field.jsonl")) if l.strip()]
    return refflow.Collection([dict(d, points=d["age"]) for d in docs], fields=("text",))


def large_text_scenarios(backend, coll):
    # test/collection_test.cpp:2144-2175 (num_typos 0, drop_tokens_threshold 1); the highlight is not replayed
    got, _ = refflow.search(backend, coll, "eguilazer", LARGE_TEXT_SORT)
    assert len(got) == 1
    got, _ = refflow.search(backend, coll, "tristique", LARGE_TEXT_SORT)
    assert len(got) == 2
    # twelve tokens: longer than the Match window (WINDOW_SIZE 10)
    got, _ = refflow.search(backend, coll, "Phasellus non tristique elit Praesent non arcu id lectus accumsan venenatis at", LARGE_TEXT_SORT)
    assert got == [1]
    got, _ = refflow.search(backend, coll, "molestie maecenas accumsan", LARGE_TEXT_SORT)
    assert len(got) == 1


def test_search_large_text_field_oracle():
    coll = large_text_collection()
    assert len(refflow.tokenize(coll.docs[1]["text"])) > 250
    oi = ol.OracleIndex(coll.n_docs, coll.flats, [coll.points])
    large_text_scenarios(lambda b, k: oi.keyword_search(b, k), coll)


# ------------------------------------------------------------------ device vs oracle (-m gpu)
@contextlib.contextmanager
def dense_cost(v):
    """TSGPU_DENSE_COST is read on every call: 0 keeps every combination on the driver tiles, a large value sends every
    all-dense combination to the bitmap path"""
    old = os.environ.get("TSGPU_DENSE_COST")
    os.environ["TSGPU_DENSE_COST"] = v
    try:
        yield
    finally:
        if old is None:
            del os.environ["TSGPU_DENSE_COST"]
        else:
            os.environ["TSGPU_DENSE_COST"] = old


DENSE_OFF, DENSE_ALWAYS = "0", "1e9"


@pytest.fixture(scope="module")
def dev(lc):
    flats = [lc.flats[f] for f in FIELDS8]
    filters = filters_of(lc)
    gi = capi.GpuIndex(lc.n_docs, 0)
    for f in flats:
        gi.load_field(f)
    gi.load_sort_column(lc.pts)
    oi = ol.OracleIndex(lc.n_docs, flats, [lc.pts])
    yield gi, oi, filters
    gi.close()


def run_both_paths(dev, b, stride):
    """the batch on the device with the bitmap path off and always on, each compared with the oracle; returns the stats"""
    gi, oi, _ = dev
    okv, ocnt, ofound = oi.keyword_search(b, stride)
    out = []
    for cost in (DENSE_OFF, DENSE_ALWAYS):
        with dense_cost(cost):
            kv, cnt, found = gi.keyword_search(b, stride)
            out.append(gi.stats())
        assert_kv_equal(kv, cnt, found, okv, ocnt, ofound)
    return out, ocnt


@pytest.mark.gpu
def test_field_classes(dev):
    if ON_DOUBLE:
        return                         # the test double does not mirror fields
    gi = dev[0]
    want = {P16: capi.FIELD_PLAIN_OK | capi.FIELD_POS16, PLONG: capi.FIELD_PLAIN_OK, ARR: capi.FIELD_IS_ARRAY}
    for fid, cls in enumerate(FIELDS8):
        assert gi.field_info(fid)["flags"] & 7 == want[cls], (fid, cls)


SHAPES = {"p16": ([P16], 16), "plong": ([PLONG], 16), "array": ([ARR], 16), "mixed": ([P16, PLONG, ARR], 10),
          "rows16x2": ([PLONG, ARR], 16), "rows4x8": (list(range(8)), 4)}


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 10, 250, 1024])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_keyword_long_documents(lc, dev, shape, k):
    fids, max_rows = SHAPES[shape]
    seed = list(SHAPES).index(shape) * 10 + [1, 10, 250, 1024].index(k)
    rng = np.random.default_rng(300 + seed)
    flats = [lc.flats[FIELDS8[f]] for f in fids]
    b = make_batch(lc, rng, flats, fids, 10, max_rows, k, filters=dev[2])
    b.field_ids = np.asarray(fids, np.uint32)
    stats, cnt = run_both_paths(dev, b, k)
    assert int(cnt.sum()) > 0
    if max_rows * len(fids) == 32:
        assert len(b.queries[0].combos[0].rows) * len(fids) == 32            # exactly kMaxLists lists
    if not ON_DOUBLE:
        assert all(s["kw_matches"] > 0 for s in stats)


@pytest.mark.gpu
def test_keyword_markers(lc, dev):
    b = marker_batch(lc)
    _, cnt = run_both_paths(dev, b, 50)
    assert int(cnt.sum()) > 20


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1500, 5000])
def test_keyword_deep_topster(lc, dev, k):
    rng = np.random.default_rng(k)
    b = make_batch(lc, rng, lc.flats, [P16, PLONG, ARR], 6, 6, k, flags=capi.QFLAG_DEEP_TOPSTER, filters=dev[2])
    # one query whose typo combinations reach past 1024 hits
    wide = S.Query([S.Combo([[t, t, t]], 1, total_cost=c) for c, t in enumerate((0, 1, 2, 3))], topk=k, flags=1 | capi.QFLAG_DEEP_TOPSTER,
                   num_query_tokens=1, sort=SORTS[1])
    b = S.KwBatch(b.queries + [wide], [P16, PLONG, ARR], dev[2])
    stats, cnt = run_both_paths(dev, b, k)
    assert int(cnt.max()) > 1024
    if not ON_DOUBLE:
        assert all(s["deep_entries"] > 0 for s in stats)


def bitmap_docs(n_docs, flats, rows):
    """documents the bitmap tiles of one combination cover (kw_kernels.cuh: 32 ids per word, the word range aligned down to
    32 words)"""
    lo, hi = 0, n_docs - 1
    for r in rows:
        ls = [(f, l) for f, l in zip(flats, r) if l != NL]
        lo = max(lo, min(int(f.ids[f.list_off[l]]) for f, l in ls))
        hi = min(hi, max(int(f.ids[f.list_off[l + 1] - 1]) for f, l in ls))
    w0 = (lo >> 5) & ~31
    return 32 * ((hi >> 5) + 1 - w0) if lo <= hi else 0


@pytest.mark.gpu
@pytest.mark.parametrize("fid", [P16, PLONG, ARR])
def test_bitmap_and_driver_paths_score_long_documents(lc, dev, fid):
    """all-dense rows whose lists hold the long documents: the bitmap path (cost large) and the driver tiles (cost 0) both
    score them, and the work counters show which ran"""
    gi, oi, _ = dev
    f = lc.flats[fid]
    rows = [[0], [1], [3]]
    assert all(f.df(r[0]) >= max(64, lc.n_docs // 64) for r in rows)
    q = S.Query([S.Combo(rows, 3)], topk=250, num_query_tokens=3, flags=3, sort=SORTS[0])
    b = S.KwBatch([q], [fid])
    stats, cnt = run_both_paths(dev, b, 250)
    assert int(cnt[0]) > 50
    if not ON_DOUBLE:
        off, on = stats
        assert off["kw_driver_ids"] == min(f.df(r[0]) for r in rows)                 # the driver's postings
        assert on["kw_driver_ids"] == bitmap_docs(lc.n_docs, [f], rows) and on["kw_probe_ids"] == 0
        assert off["kw_matches"] > 0 and on["kw_matches"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("fid", [PLONG, ARR])
def test_phrase_exact_prefix_device(lc, dev, fid):
    gi, oi, _ = dev
    L = ol.oracle()
    rng = np.random.default_rng(41 + fid)
    hits = 0
    for lists, ids in idset_cases(lc, rng, fid, 40):
        for name, ofn, _, dfn in IDSET_FNS:
            out = np.zeros(len(ids), np.uint32)
            n = getattr(L, ofn)(oi.h, fid, ol.p32(lists), len(lists), ol.p32(ids), len(ids), ol.p32(out))
            assert getattr(gi, dfn)(fid, lists, ids).tolist() == out[:n].tolist(), (name, lists.tolist())
            hits += n
    assert hits > 20


@pytest.mark.gpu
def test_scorer_switch_keeps_records(lc):
    """Field A holds the regular documents (16-bit positions: the register scorer); field B the same documents plus one
    110,000-token document of tokens no query uses (score_field_plain). Every query answers the same on both, and as the
    oracle does."""
    n_docs = lc.n_docs + 1
    rng = np.random.default_rng(55)
    extra = LD.Doc(rng.integers(LD.UNQUERIED, LD.N_TOKENS, 110000))
    fa = LD.plain_field(lc.docs[:lc.n_regular])
    fb = LD.plain_field(lc.docs[:lc.n_regular] + [LD.Doc([]) for _ in range(n_docs - 1 - lc.n_regular)] + [extra])
    gi = capi.GpuIndex(n_docs, 0)
    try:
        gi.load_field(fa)
        gi.load_field(fb)
        gi.load_sort_column(np.append(lc.pts, 2))
        if not ON_DOUBLE:
            assert gi.field_info(0)["flags"] & capi.FIELD_POS16 and not gi.field_info(1)["flags"] & capi.FIELD_POS16
            assert gi.field_info(1)["flags"] & capi.FIELD_PLAIN_OK
        oi = ol.OracleIndex(n_docs, [fa, fb], [np.append(lc.pts, 2)])
        for max_rows in (4, 16):
            b = make_batch(lc, rng, [fa], [0], 24, max_rows, 250)
            kva, cnta, fnda = gi.keyword_search(b, 250)
            b.field_ids = np.asarray([1], np.uint32)
            kvb, cntb, fndb = gi.keyword_search(b, 250)
            assert_kv_equal(kva, cnta, fnda, kvb, cntb, fndb)
            assert_kv_equal(kvb, cntb, fndb, *oi.keyword_search(b, 250))
            assert int(cnta.sum()) > 100
    finally:
        gi.close()


@pytest.mark.gpu
def test_search_large_text_field_device():
    coll = large_text_collection()
    gi = capi.GpuIndex(coll.n_docs, 0)
    try:
        for f in coll.flats:
            gi.load_field(f)
        gi.load_sort_column(coll.points)
        large_text_scenarios(lambda b, k: gi.keyword_search(b, k), coll)
    finally:
        gi.close()


@pytest.mark.gpu
def test_long_documents_with_general_scoring_kernel():
    """TSGPU_REG_SCORE is read once per process: the gpu tests above again in a child process with the general scorer
    (kw_search_kernel<false>) instead of the register-resident one"""
    env = dict(os.environ, TSGPU_REG_SCORE="0")
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__),
           "-k", "not general_scoring_kernel" if not ON_DOUBLE else "large_text_field_device"]   # the double has one scorer
    r = subprocess.run(cmd, cwd=ol.ROOT, env=env, capture_output=True, text=True, timeout=600)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0 and " passed" in r.stdout, tail
