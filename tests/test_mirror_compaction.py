"""Mirror maintenance (f-4): tsgpu_index_compact_field frees the lists tsgpu_index_append_lists left behind, tsgpu_index_reserve_docs
raises the seq_id capacity. A patched-then-compacted field must be byte for byte what a fresh load of its live lists builds, and
answer like the oracle and a fresh mirror of the final state; a grown index must answer like one created at the new capacity."""
import os

import numpy as np
import pytest

import mirror_double as md
import oracle_lib as ol
from typesense_b200 import capi, structs as S, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, scope="module")
def _library_with_maintenance_calls():
    """libtsgpu.so has the calls; where the harness loaded the base test double instead, the double extended with them answers"""
    if md.lib_has_maintenance():
        yield
        return
    saved = capi._lib
    capi._lib = md.load_lib()
    yield
    capi._lib = saved

I64_MIN = np.iinfo(np.int64).min
SORT = ((S.SORT_TEXT_MATCH, -1, 1, 0), (S.SORT_NUMERIC, 0, 1, 0), (S.SORT_SEQ_ID, -1, -1, 0))
SORT2 = ((S.SORT_NUMERIC, 0, -1, 1), (S.SORT_TEXT_MATCH, -1, 1, 0), (S.SORT_NONE, -1, 1, 0))


def _lists_of(flat: S.FlatField):
    out = []
    for l in range(flat.n_lists):
        a, b = int(flat.list_off[l]), int(flat.list_off[l + 1])
        out.append([(int(flat.ids[i]), flat.positions[int(flat.pos_off[i]):int(flat.pos_off[i + 1])].tolist()) for i in range(a, b)])
    return out


def _flat(lists, is_array):
    return S.FlatField.from_postings(lists, is_array)


def _scenario(is_array, n_docs=6000, vocab=400, seed=21):
    """An early state and the final state of one field, and the write batches between them: inserted documents, documents with new
    offsets under their old seq_ids, removed documents, tokens that disappear and tokens that appear."""
    fd = (synth.make_array_field(n_docs, vocab, 1, 3, 2, 5, seed=seed) if is_array else synth.make_string_field(n_docs, vocab, 3, 9, seed=seed))
    final = _lists_of(fd.flat)
    rng = np.random.default_rng(seed)
    cut = 2 * n_docs // 3                                # the early state holds documents below `cut`
    changed = set(rng.choice(cut, n_docs // 20, replace=False).tolist())
    removed = set(rng.choice(np.arange(cut, cut + n_docs // 12), n_docs // 30, replace=False).tolist())
    nonempty = [t for t in range(vocab) if final[t]]
    erased = set(nonempty[150:160])                      # tokens whose every document goes away
    appearing = set(nonempty[40:45])                     # tokens no document of the early state holds

    def early(t, pl):
        if t in appearing:
            return []
        out = []
        for sid, offs in pl:
            if sid < cut or sid in removed:
                o = list(offs)
                if sid in changed and not is_array and len(o) and o[0] > 1:
                    o[0] -= 1
                out.append((sid, o))
        return out
    lists0 = [early(t, pl) for t, pl in enumerate(final)]
    final = [[] if t in erased else [p for p in pl if p[0] not in removed] for t, pl in enumerate(final)]
    touched = [t for t in range(vocab) if lists0[t] != final[t]]
    pts = synth.make_points(n_docs, 5)
    pts[list(removed)] = I64_MIN
    return dict(n_docs=n_docs, lists0=lists0, final=final, touched=touched, pts=pts, is_array=is_array)


def _patch(gi, f, sc, n_batches=3):
    """append the touched lists in n_batches; returns token -> current list id"""
    remap = np.arange(len(sc["final"]), dtype=np.int64)
    parts = np.array_split(np.asarray(sc["touched"]), n_batches)
    for part in parts:
        first = gi.append_lists(f, _flat([sc["final"][t] for t in part], sc["is_array"]))
        for k, t in enumerate(part):
            remap[int(t)] = first + k
    return remap


def _live_order(sc, remap):
    """live tokens (a non-empty final list) in ascending current list id: the order compaction keeps them in"""
    live_toks = [t for t in range(len(sc["final"])) if sc["final"][t]]
    return sorted(live_toks, key=lambda t: int(remap[t]))


def _snapshot(gi, f):
    return [gi.field_array(f, s) for s in range(10)], gi.field_info(f)


def _assert_same_field(a, b):
    (arrs_a, info_a), (arrs_b, info_b) = a, b
    for s in range(10):
        assert arrs_a[s].dtype == arrs_b[s].dtype and arrs_a[s].tolist() == arrs_b[s].tolist(), f"array {capi.FIELD_ARRAYS[s][0]} differs"
    assert info_a == info_b


def _queries(sc, tok_map, r, n=60, filt=-1, excl=()):
    live = [t for t in range(len(sc["final"])) if sc["final"][t]]
    qs_o, qs_m = [], []
    for i in range(n):
        nt = int(r.integers(1, 4))
        toks = [int(t) for t in r.choice(live, nt, replace=False)]
        if i % 3 == 0:                                   # tokens of one document: guaranteed hits
            d = int(r.integers(0, sc["n_docs"]))
            cand = [t for t in live[:150] if any(p[0] == d for p in sc["final"][t])]
            if len(cand) >= nt:
                toks = cand[:nt]
        sort = SORT if i % 2 == 0 else SORT2
        topk = int(r.choice([10, 100]))
        qs_o.append(S.Query([S.Combo([[t] for t in toks], nt)], topk=topk, sort=sort, num_query_tokens=nt, filter=filt if i % 4 == 1 else -1,
                            excl=excl if i % 5 == 2 else ()))
        qs_m.append(S.Query([S.Combo([[int(tok_map[t])] for t in toks], nt)], topk=topk, sort=sort, num_query_tokens=nt,
                            filter=filt if i % 4 == 1 else -1, excl=excl if i % 5 == 2 else ()))
    return qs_o, qs_m


def _assert_same_answers(a, b):
    kv, cnt, found = a
    okv, ocnt, ofound = b
    assert cnt.tolist() == ocnt.tolist() and found.tolist() == ofound.tolist()
    for q in range(len(cnt)):
        n = int(cnt[q])
        for k in ("key", "scores", "text_match_score", "query_index"):
            assert kv[k][q, :n].tolist() == okv[k][q, :n].tolist(), f"query {q}: {k}"


def _check_answers(sc, oi, gi, tok_map, gf=None, fresh_map=None, seed=0):
    r = np.random.default_rng(100 + seed)
    flt = np.sort(r.choice(sc["n_docs"], sc["n_docs"] // 3, replace=False)).astype(np.uint32)
    excl = tuple(int(x) for x in r.choice(sc["n_docs"], 40, replace=False))
    qs_o, qs_m = _queries(sc, tok_map, np.random.default_rng(7 + seed), filt=0, excl=excl)
    want = oi.keyword_search(S.KwBatch(qs_o, [0], [flt]), 128)
    assert int(want[1].sum()) > 100
    _assert_same_answers(gi.keyword_search(S.KwBatch(qs_m, [0], [flt]), 128), want)
    if gf is not None:
        _, qs_f = _queries(sc, fresh_map, np.random.default_rng(7 + seed), filt=0, excl=excl)
        _assert_same_answers(gf.keyword_search(S.KwBatch(qs_f, [0], [flt]), 128), want)


def _check_primitives(sc, gi, tok_map, gf, fresh_map):
    """intersect / phrase / exact / prefix / contains_atleast_one through the ids each index uses now"""
    live = [t for t in range(len(sc["final"])) if sc["final"][t]]
    r = np.random.default_rng(5)
    for _ in range(12):
        d = int(r.integers(0, sc["n_docs"]))
        toks = [t for t in live if any(p[0] == d for p in sc["final"][t])][:2] or [live[0]]
        a, b = [int(tok_map[t]) for t in toks], [int(fresh_map[t]) for t in toks]
        ia, ib = gi.intersect(0, a, sc["n_docs"]), gf.intersect(0, b, sc["n_docs"])
        assert ia.tolist() == ib.tolist()
        if len(ia):
            assert gi.phrase_matches(0, a, ia).tolist() == gf.phrase_matches(0, b, ib).tolist()
            assert gi.exact_matches(0, a, ia).tolist() == gf.exact_matches(0, b, ib).tolist()
            assert gi.prefix_matches(0, a, ia).tolist() == gf.prefix_matches(0, b, ib).tolist()
        probe = r.choice(sc["n_docs"], 20, replace=False)
        probe.sort()
        assert gi.contains_atleast_one(0, a[0], probe) == gf.contains_atleast_one(0, b[0], probe)


@pytest.mark.parametrize("is_array", [False, True])
def test_compacted_field_is_a_fresh_load_of_its_live_lists(is_array):
    sc = _scenario(is_array)
    n_docs, L = sc["n_docs"], len(sc["final"])
    gi = capi.GpuIndex(n_docs, 0)
    f = gi.load_field(_flat(sc["lists0"], is_array))
    gi.load_sort_column(sc["pts"])
    # compacting a field that was never patched keeps it as it is
    before = _snapshot(gi, f)
    gi.compact_field(f, np.arange(L))
    _assert_same_field(_snapshot(gi, f), before)
    remap = _patch(gi, f, sc)
    oi = ol.OracleIndex(n_docs, [_flat(sc["final"], is_array)], [sc["pts"]])
    order = _live_order(sc, remap)
    new_id = {t: i for i, t in enumerate(order)}
    gf = capi.GpuIndex(n_docs, 0)
    gf.load_field(_flat([sc["final"][t] for t in order], is_array))
    gf.load_sort_column(sc["pts"])
    _check_answers(sc, oi, gi, remap, gf, new_id, seed=1)                     # patched, not compacted yet
    assert gi.field_info(f)["n_lists"] > L
    gi.compact_field(f, [int(remap[t]) for t in order])
    _assert_same_field(_snapshot(gi, f), _snapshot(gf, 0))
    _check_answers(sc, oi, gi, new_id, gf, new_id, seed=2)
    _check_primitives(sc, gi, new_id, gf, new_id)
    gi.close(); gf.close()


def test_compaction_brings_the_plain_field_fast_path_back():
    sc = _scenario(False, n_docs=3000, vocab=200, seed=4)
    n_docs = sc["n_docs"]
    gi = capi.GpuIndex(n_docs, 0)
    f = gi.load_field(_flat(sc["final"], False))
    gi.load_sort_column(sc["pts"])
    flags0 = gi.field_info(f)["flags"]
    assert flags0 & capi.FIELD_PLAIN_OK and flags0 & capi.FIELD_POS16
    bad = [(sid, [p + 70000 if p else 0 for p in offs]) for sid, offs in sc["final"][0]]     # a document with offsets past 65535
    first = gi.append_lists(f, _flat([bad], False))
    assert not gi.field_info(f)["flags"] & capi.FIELD_POS16
    first = gi.append_lists(f, _flat([sc["final"][0]], False))          # the document is written again: the bad list is garbage
    remap = np.arange(len(sc["final"]), dtype=np.int64)
    remap[0] = first
    assert not gi.field_info(f)["flags"] & capi.FIELD_POS16             # appending only ever clears the flags
    order = _live_order(sc, remap)
    gi.compact_field(f, [int(remap[t]) for t in order])
    assert gi.field_info(f)["flags"] == flags0
    new_id = {t: i for i, t in enumerate(order)}
    gf = capi.GpuIndex(n_docs, 0)
    gf.load_field(_flat([sc["final"][t] for t in order], False))
    gf.load_sort_column(sc["pts"])
    _assert_same_field(_snapshot(gi, f), _snapshot(gf, 0))
    oi = ol.OracleIndex(n_docs, [_flat(sc["final"], False)], [sc["pts"]])
    _check_answers(sc, oi, gi, new_id, gf, new_id, seed=3)
    gi.close(); gf.close()


def test_repeated_writes_with_compaction_keep_the_field_bounded():
    sc = _scenario(False, n_docs=3000, vocab=200, seed=9)
    n_docs = sc["n_docs"]
    gi = capi.GpuIndex(n_docs, 0)
    f = gi.load_field(_flat(sc["final"], False))
    fresh = gi.field_info(f)
    batch = _flat([sc["final"][t] for t in sc["touched"]], False)
    remap = np.arange(len(sc["final"]), dtype=np.int64)
    grown = 0
    for cycle in range(20):
        first = gi.append_lists(f, batch)
        for k, t in enumerate(sc["touched"]):
            remap[t] = first + k
        grown = max(grown, gi.field_info(f)["device_bytes"])
        order = sorted(range(len(sc["final"])), key=lambda t: int(remap[t]))      # every token stays (empty lists included)
        gi.compact_field(f, [int(remap[t]) for t in order])
        remap = np.empty(len(order), np.int64)
        remap[order] = np.arange(len(order))
        info = gi.field_info(f)
        assert info["device_bytes"] == fresh["device_bytes"] and info["n_postings"] == fresh["n_postings"], f"cycle {cycle}"
    assert grown > fresh["device_bytes"]
    gi.close()


def test_compaction_and_growth_reject_bad_input():
    n_docs = 1000
    fd = synth.make_string_field(n_docs, 50, 3, 6, seed=2)
    gi = capi.GpuIndex(n_docs, 0)
    f = gi.load_field(fd.flat)
    before = _snapshot(gi, f)
    L = fd.flat.n_lists
    for live in ([0, 1, 1, 2], [0, L], list(range(L)) + [L + 5]):
        with pytest.raises(capi.TsgpuError, match="status 2"):
            gi.compact_field(f, live)
    with pytest.raises(capi.TsgpuError, match="status 2"):
        gi.reserve_docs(n_docs - 1)
    gi.reserve_docs(n_docs)                                              # the same capacity: nothing to do
    _assert_same_field(_snapshot(gi, f), before)
    assert gi.intersect(f, [0], n_docs).tolist() == fd.flat.ids[int(fd.flat.list_off[0]):int(fd.flat.list_off[1])].tolist()
    gi.close()


def _facet(n_docs, n_values, seed):
    r = np.random.default_rng(seed)
    cnt = r.integers(0, 3, n_docs)
    off = np.zeros(n_docs + 1, np.uint64)
    off[1:] = np.cumsum(cnt)
    return off, r.integers(0, n_values, int(off[-1])).astype(np.uint32)


def test_growth_follows_a_collection_past_its_capacity():
    """A mirror created for N documents, grown past a dense-bitmap stride boundary, then fed documents >= N: it answers like the
    oracle and a mirror created at the new capacity; filters made before the growth still exclude the new documents."""
    N, N2 = 3000, 5000
    fd = synth.make_string_field(N2, 300, 3, 9, seed=31)
    final = _lists_of(fd.flat)
    lists0 = [[p for p in pl if p[0] < N] for pl in final]
    touched = [t for t in range(len(final)) if lists0[t] != final[t]]
    pts = synth.make_points(N2, 8)
    gi = capi.GpuIndex(N, 0)
    f = gi.load_field(_flat(lists0, False))
    col = gi.load_sort_column(pts[:N])
    info0 = gi.field_info(f)
    assert info0["n_dense"] > 0
    r = np.random.default_rng(3)
    old_ids = np.sort(r.choice(N, 900, replace=False)).astype(np.uint32)
    h_old = gi.filter_create(old_ids)
    h_num_old, n_num_old = gi.filter_numeric(col, ">", 500000)
    foff, fvals = _facet(N, 12, 4)
    fc = gi.load_facet(12, foff, fvals)
    kw_keep = S.KwBatch([S.Query([S.Combo([[0]], 1)], topk=10, flags=S.FLAG_PRIORITIZE_EXACT_MATCH | capi.QFLAG_KEEP_ALL_IDS)], [0])
    gi.keyword_search(kw_keep, 16)
    gi.reserve_docs(N2)
    info1 = gi.field_info(f)
    assert info1["dense_words"] > info0["dense_words"] and info1["n_dense"] == info0["n_dense"]
    with pytest.raises(capi.TsgpuError):                                 # the kept all_result_ids were sized for N documents
        gi.facet_counts_last(fc, 1, 10)
    first = gi.append_lists(f, _flat([final[t] for t in touched], False))
    remap = np.arange(len(final), dtype=np.int64)
    for k, t in enumerate(touched):
        remap[t] = first + k
    gi.set_sort_values(col, np.arange(N, N2, dtype=np.uint32), pts[N:])
    oi = ol.OracleIndex(N2, [_flat(final, False)], [pts])
    gf = capi.GpuIndex(N2, 0)
    gf.load_field(_flat(final, False)); gf.load_sort_column(pts)
    sc = dict(n_docs=N2, final=final)
    ident = np.arange(len(final))
    _check_answers(sc, oi, gi, remap, gf, ident, seed=4)
    # filters: the old handles still hold only old documents; a new one with new documents works
    new_ids = np.sort(np.concatenate([old_ids[:300], np.arange(N, N2, 3, dtype=np.uint32)])).astype(np.uint32)
    h_new = gi.filter_create(new_ids)
    assert gi.filter_ids(h_old, N2).tolist() == old_ids.tolist()
    assert gi.filter_ids(h_num_old, N2).tolist() == np.nonzero(pts[:N] > 500000)[0].tolist()
    h_num, n_num = gi.filter_numeric(col, ">", 500000)                   # sees the grown column
    assert gi.filter_ids(h_num, N2).tolist() == np.nonzero(pts > 500000)[0].tolist() and n_num > n_num_old
    qs_o, qs_m = _queries(sc, remap, np.random.default_rng(11), n=40)
    for h, ids in ((h_old, old_ids), (h_new, new_ids), (h_num_old, np.nonzero(pts[:N] > 500000)[0]), (h_num, np.nonzero(pts > 500000)[0])):
        want = oi.keyword_search(S.KwBatch([S.Query(q.combos, q.topk, 0, q.excl, q.sort, q.flags, q.match_type, q.num_query_tokens) for q in qs_o], [0],
                                           [ids.astype(np.uint32)]), 128)
        got = gi.keyword_search(S.KwBatch([S.Query(q.combos, q.topk, h, q.excl, q.sort, q.flags, q.match_type, q.num_query_tokens) for q in qs_m], [0]), 128)
        _assert_same_answers(got, want)
    # wildcard: every document up to the new capacity
    wq = [S.Query([], topk=50, sort=((S.SORT_NUMERIC, 0, 1, 0), (S.SORT_SEQ_ID, -1, 1, 0), (S.SORT_NONE, -1, 1, 0))),
          S.Query([], topk=50, sort=((S.SORT_SEQ_ID, -1, 1, 0), (S.SORT_NONE, -1, 1, 0), (S.SORT_NONE, -1, 1, 0)))]
    want = oi.wildcard_search(S.KwBatch(wq, [0]), 64)
    got = gi.wildcard_search(S.KwBatch(wq, [0]), 64)
    _assert_same_answers(got, want)
    assert int(got[2][0]) == N2 and max(got[0]["key"][1, :50].tolist()) == N2 - 1
    # facets: new documents have no values, so they add nothing
    res = np.sort(np.concatenate([old_ids, np.arange(N, N2, 7, dtype=np.uint32)])).astype(np.uint32)
    a, da = gi.facet_counts(fc, res, 12)
    b, db = gi.facet_counts(fc, old_ids, 12)
    assert a.tolist() == b.tolist() and da == db
    # compacting after the growth: dense lists below the new threshold drop their bitmaps; still a fresh load
    order = _live_order(dict(final=final), remap)
    gi.compact_field(f, [int(remap[t]) for t in order])
    gc = capi.GpuIndex(N2, 0)
    gc.load_field(_flat([final[t] for t in order], False))
    _assert_same_field(_snapshot(gi, f), _snapshot(gc, 0))
    new_id = {t: i for i, t in enumerate(order)}
    _check_answers(sc, oi, gi, new_id, gf, ident, seed=5)
    gi.close(); gf.close(); gc.close()


@pytest.mark.skipif(os.environ.get("TSGPU_TEST_DOUBLE") == "1", reason="builds its graph on the device (the test double has no device build)")
def test_growth_lets_filtered_knn_reach_appended_labels():
    N, N2, dim = 2000, 3000, 32
    vec = synth.make_vectors(N2, dim, 17).numpy()
    gi = capi.GpuIndex(N, 0)
    gi.build_hnsw(vec[:N], M=8, ef_construction=64, seed=5, max_batch=1)
    gi.reserve_docs(N2)
    gi.append_hnsw(vec[N:], ef_construction=64, seed=5, max_batch=1)
    graph = gi.export_hnsw(vec)
    oi = ol.OracleIndex(N2, [], [], graph)
    r = np.random.default_rng(1)
    flt = np.sort(np.concatenate([r.choice(N, 300, replace=False), r.choice(np.arange(N, N2), 300, replace=False)])).astype(np.uint32)
    qv = synth.make_vectors(16, dim, 23).numpy()
    d, l, n = gi.knn(qv, 10, 64, q_filter=np.zeros(16, np.int32), filters=[flt])
    od, olab, on, _ = oi.knn(qv, 10, 64, q_filter=np.zeros(16, np.int32), filters=[flt])
    assert n.tolist() == on.tolist() and l.tolist() == olab.tolist()
    assert (l[n > 0] >= N).any()
    gi.close()
