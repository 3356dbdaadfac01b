"""The keyword kernel's bitmap path (CDesc mode 1): combinations whose required lists all have dense bitmaps are intersected word
by word over the lists' common id range instead of probing every driver id. The collection is small enough that every frequent
token is dense (df >= max(64, n_docs / 64)); tokens 0-2 never occur below doc 6000, so their word range does not start at doc 0.
Every answer is compared with the oracle bit for bit (ids, scores, found, query_index), and the work counters show which path ran:
a bitmap tile counts the documents it covers as driver ids, a driver tile the driver's postings."""
import os

import numpy as np
import pytest
import torch

import oracle_lib as ol
from typesense_b200 import capi, structs as S, synth
from test_gpu_parity import assert_kv_equal

ON_DOUBLE = os.environ.get("TSGPU_TEST_DOUBLE") == "1"
N_DOCS = 20000
LATE = 6000                      # tokens 0..2 start here
RARE = 8                         # a sparse token
TEXT = ((S.SORT_TEXT_MATCH, -1, 1, 0), (S.SORT_NUMERIC, 0, 1, 1), (S.SORT_SEQ_ID, -1, -1, 0))
NL = S.NO_LIST


def make_field(seed: int):
    rng = np.random.default_rng(seed)
    lens = rng.integers(4, 9, N_DOCS)
    doc = np.repeat(np.arange(N_DOCS), lens)
    p = np.full(9, (1 - 0.002) / 8)
    p[RARE] = 0.002
    tok = rng.choice(9, size=len(doc), p=p)
    early = (doc < LATE) & (tok < 3)
    tok[early] += 5
    off = np.concatenate([[0], np.cumsum(lens)])
    pos = np.arange(len(doc)) - off[doc] + 1
    last = off[1:] - 1
    tok_all = torch.from_numpy(np.concatenate([tok, tok[last]]))
    doc_all = torch.from_numpy(np.concatenate([doc, np.arange(N_DOCS)]))
    pos_all = torch.from_numpy(np.concatenate([pos, np.full(N_DOCS, 0xFFFF)]))
    return S.FlatField(*synth._flatten(tok_all, doc_all, pos_all, 9), False)


@pytest.fixture(scope="module")
def coll():
    flats = [make_field(1), make_field(2)]
    pts = synth.make_points(N_DOCS, 5, hi=40, missing_frac=0.05)
    rng = np.random.default_rng(3)
    filters = [np.unique(rng.integers(0, N_DOCS, 7000)).astype(np.uint32), np.zeros(0, np.uint32)]
    gi = capi.GpuIndex(N_DOCS, 0)
    for f in flats:
        gi.load_field(f)
    gi.load_sort_column(pts)
    handles = [gi.filter_create(f) for f in filters]
    oi = ol.OracleIndex(N_DOCS, flats, [pts])
    yield flats, filters, handles, gi, oi
    gi.close()


def df(flat, l):
    return int(flat.list_off[l + 1] - flat.list_off[l])


def is_dense(flat, l):
    return df(flat, l) >= max(64, N_DOCS // 64)


def bitmap_docs(flats, rows, fields):
    """documents the bitmap tiles of one combination cover: 32 x the words from the common id range's first (aligned down to
    32 words) to its last"""
    lo, hi = 0, N_DOCS - 1
    for r in rows:
        ls = [(flats[fi], l) for fi, l in zip(fields, r) if l != NL]
        lo = max(lo, min(int(f.ids[f.list_off[l]]) for f, l in ls))
        hi = min(hi, max(int(f.ids[f.list_off[l + 1] - 1]) for f, l in ls))
    w0 = (lo >> 5) & ~31
    return 32 * ((hi >> 5) + 1 - w0) if lo <= hi else 0


def run(coll, qs, fields, k=100, persistent=True):
    flats, filters, handles, gi, oi = coll
    b = S.KwBatch(qs, fields, filters)
    kv, cnt, found = gi.keyword_search(b.with_filter_handles(handles) if persistent else b, k)
    st = gi.stats()
    okv, ocnt, ofound = oi.keyword_search(b, k)
    assert_kv_equal(kv, cnt, found, okv, ocnt, ofound)
    return st, cnt, found


def q(rows, n_req=None, **kw):
    n_req = len(rows) if n_req is None else n_req
    return S.Query([S.Combo([list(r) for r in rows], n_req)], sort=TEXT, num_query_tokens=len(rows), **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [[0, 3], [0, 1, 4], [2, 5, 6, 7], [3, 4, 5]])
@pytest.mark.parametrize("filt", [-1, 0, 1])
def test_all_dense_rows(coll, rows, filt):
    flats = coll[0]
    assert all(is_dense(flats[0], t) for t in rows)
    st, cnt, found = run(coll, [q([[t] for t in rows], filter=filt)], [0])
    assert (int(found[0]) == 0) == (filt == 1)
    if not ON_DOUBLE:
        assert st["kw_driver_ids"] == bitmap_docs(flats, [[t] for t in rows], [0])
        assert st["kw_probe_ids"] == 0


@pytest.mark.gpu
def test_word_range_starts_past_doc_zero(coll):
    flats = coll[0]
    assert min(int(flats[0].ids[flats[0].list_off[t]]) for t in (0, 1, 2)) >= LATE
    st, cnt, found = run(coll, [q([[0], [1], [2]])], [0])
    if not ON_DOUBLE:
        assert 0 < st["kw_driver_ids"] <= N_DOCS - LATE + 1024


@pytest.mark.gpu
def test_two_fields_every_list_dense(coll):
    flats = coll[0]
    rows = [[0, 1], [3, 3], [5, NL]]
    st, cnt, found = run(coll, [q(rows, filter=0), q(rows)], [0, 1])
    if not ON_DOUBLE:
        assert st["kw_driver_ids"] == 2 * bitmap_docs(flats, rows, [0, 1])


@pytest.mark.gpu
def test_sparse_required_list_stays_on_driver_tiles(coll):
    flats = coll[0]
    assert not is_dense(flats[0], RARE)
    st, cnt, found = run(coll, [q([[RARE], [3]])], [0])
    if not ON_DOUBLE:
        assert st["kw_driver_ids"] == df(flats[0], RARE)


@pytest.mark.gpu
def test_dropped_rows_sparse_and_dense(coll):
    # required rows dense; the dropped rows (a sparse and a dense token) only contribute to the score
    flats = coll[0]
    st, cnt, found = run(coll, [q([[3], [4], [RARE], [6]], n_req=2), q([[3], [RARE]], n_req=1, filter=0)], [0])
    if not ON_DOUBLE:
        assert st["kw_driver_ids"] == bitmap_docs(flats, [[3], [4]], [0]) + bitmap_docs(flats, [[3]], [0])


@pytest.mark.gpu
def test_exclusions_and_inline_filter(coll):
    rng = np.random.default_rng(7)
    excl = sorted(set(rng.integers(0, N_DOCS, 3000).tolist()))
    run(coll, [q([[3], [4]], excl=excl), q([[0], [5]], excl=excl, filter=0)], [0], persistent=False)


@pytest.mark.gpu
def test_several_combinations_deduplicate(coll):
    combos = [S.Combo([[3], [4]], 2), S.Combo([[3], [5]], 2, total_cost=1), S.Combo([[3], [4], [RARE]], 3, total_cost=2),
              S.Combo([[6]], 1, total_cost=2)]
    qs = [S.Query(list(combos), sort=TEXT, num_query_tokens=2), S.Query(list(combos), sort=TEXT, num_query_tokens=2, filter=0)]
    run(coll, qs, [0], k=250)


@pytest.mark.gpu
def test_keep_all_ids(coll):
    flats, filters, handles, gi, oi = coll
    combos = [S.Combo([[3], [4]], 2), S.Combo([[0], [5]], 2, total_cost=1)]
    qs = [S.Query(list(combos), sort=TEXT, num_query_tokens=2, flags=capi.QFLAG_KEEP_ALL_IDS, filter=0)]
    st, cnt, found = run(coll, qs, [0])
    if ON_DOUBLE:             # the test double keeps no all_result_ids: they live in device memory (tsgpu_all_result_ids_last)
        return
    ids = gi.all_result_ids_last(0, N_DOCS)
    want = set()
    for c in combos:
        docs = set(range(N_DOCS))
        for r in c.rows:
            f = flats[0]
            docs &= set(f.ids[f.list_off[r[0]]:f.list_off[r[0] + 1]].tolist())
        want |= docs
    want &= set(filters[0].tolist())
    assert sorted(ids.tolist()) == sorted(want) and int(found[0]) == len(want)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1025, 5000])
def test_deep_topster(coll, k):
    combos = [S.Combo([[3], [4]], 2), S.Combo([[3], [5]], 2, total_cost=1)]
    qs = [S.Query(list(combos), sort=TEXT, topk=k, num_query_tokens=2, flags=capi.QFLAG_DEEP_TOPSTER),
          S.Query([S.Combo([[0], [6]], 2)], sort=TEXT, topk=k, num_query_tokens=2, flags=capi.QFLAG_DEEP_TOPSTER, filter=0)]
    st, cnt, found = run(coll, qs, [0], k=k)
    assert int(cnt.max()) > 1024
