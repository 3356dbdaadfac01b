#!/usr/bin/env python
"""Cost of deep Topsters (TSGPU_QFLAG_DEEP_TOPSTER: deep pagination, a Topster larger than TSGPU_MAX_TOPK = 1024) at bench.py's
field shape: 10 M documents, 1 M-token Zipf vocabulary, 4..12 tokens per document, one sort column. Queries, one per device call:

  kw_<rank>     a one-token keyword query on the token of that frequency rank (rare to head), sorted by text match, then the column
  kw2_<rank>    the same token plus a second combination (the token AND the next rank's token, cost 1) whose documents all match
                the first one too: every one of them is emitted twice and de-duplicated
  wildcard      q=* sorted by the column (every document is a match)

each at K in {250, 1024, 1025, 10 000, 100 000}: K <= 1024 is the ordinary shared-memory selection, K > 1024 the deep path. Per
query and K it reports the device time of the call (tsgpu_get_stats ms_total: CUDA events around the whole call on the library's
stream, copies included; median of --reps calls after one warm-up call), the host wall time, and for the deep path the entries
emitted, the deep buffer's bytes and the time in emit (the deep unit kernel), de-duplicate (packing the entries for the sorts
included, so a one-combination query shows that alone) and select (sort + record write). A
sample of the queries at K = 1025 and 10 000 is compared with the CPU oracle over the same arrays. Prints one JSON line with
the GPU's name and power limit, read in the same run. Needs a CUDA device."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from typesense_b200 import capi, structs as S, synth      # noqa: E402


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:                                  # noqa: BLE001
        return {"gpu": None, "power_limit": None, "error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--ks", default="250,1024,1025,10000,100000")
    ap.add_argument("--ranks", default="0,10,100,1000,10000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_deep_topster needs a CUDA device")
    ident = gpu_identity()
    ks = [int(x) for x in args.ks.split(",")]
    fd = synth.make_string_field(args.docs, args.vocab, 4, 12, seed=7, device="cuda")
    pts = synth.make_points(args.docs, seed=13)
    gi = capi.GpuIndex(args.docs, 0)
    gi.load_field(fd.flat)
    gi.load_sort_column(pts)
    sort = ((S.SORT_TEXT_MATCH, -1, 1, 0), (S.SORT_NUMERIC, 0, 1, 0), (S.SORT_NONE, -1, 1, 0))
    wsort = ((S.SORT_NUMERIC, 0, -1, 0), (S.SORT_SEQ_ID, -1, 1, 0), (S.SORT_NONE, -1, 1, 0))

    def make(name, k):
        flags = S.FLAG_PRIORITIZE_EXACT_MATCH | (capi.QFLAG_DEEP_TOPSTER if k > capi.MAX_TOPK else 0)
        if name == "wildcard":
            return S.KwBatch([S.Query([], topk=k, sort=wsort, flags=flags)], [0]), True
        kind, rank = name.split("_")
        t = int(rank)
        combos = [S.Combo([[t]], 1)]
        if kind == "kw2":
            combos.append(S.Combo([[t], [t + 1]], 2, total_cost=1))
        return S.KwBatch([S.Query(combos, topk=k, sort=sort, flags=flags, num_query_tokens=1)], [0]), False

    names = [f"kw_{r}" for r in args.ranks.split(",")] + [f"kw2_{r}" for r in args.ranks.split(",")] + ["wildcard"]
    rows = []
    for name in names:
        for k in ks:
            b, wc = make(name, k)
            call = gi.wildcard_search if wc else gi.keyword_search
            call(b, k)                                      # warm-up
            dev, wall, st = [], [], None
            for _ in range(args.reps):
                t0 = time.perf_counter()
                kv, cnt, found = call(b, k)
                wall.append((time.perf_counter() - t0) * 1e3)
                st = gi.stats()
                dev.append(st["ms_total"])
            row = {"query": name, "k": k, "found": int(found[0]), "count": int(cnt[0]), "deep": k > capi.MAX_TOPK,
                   "device_ms": round(statistics.median(dev), 3), "wall_ms": round(statistics.median(wall), 3)}
            if k > capi.MAX_TOPK:
                row.update(entries=int(st["deep_entries"]), deep_bytes=int(st["deep_bytes"]), emit_ms=round(st["ms_deep_emit"], 3),
                           dedup_ms=round(st["ms_deep_dedup"], 3), select_ms=round(st["ms_deep_select"], 3))
            rows.append(row)
            print(json.dumps(row), flush=True)
    parity = None
    if not args.no_parity:
        import oracle_lib as ol
        oi = ol.OracleIndex(args.docs, [fd.flat], [pts])
        checked, bad = 0, []
        for name in [n for n in names if n.endswith(("_100", "_1000", "_10000"))] + ["wildcard"]:
            for k in (1025, 10_000):
                b, wc = make(name, k)
                kv, cnt, found = (gi.wildcard_search if wc else gi.keyword_search)(b, k)
                okv, ocnt, ofound = (oi.wildcard_search if wc else oi.keyword_search)(b, k, threads=16)
                n = int(cnt[0])
                same = (cnt.tolist() == ocnt.tolist() and found.tolist() == ofound.tolist()
                        and all(np.array_equal(kv[f][0, :n], okv[f][0, :n]) for f in ("key", "scores", "text_match_score", "query_index")))
                checked += 1
                if not same:
                    bad.append(f"{name}@{k}")
        parity = {"checked": checked, "mismatches": bad}
    gi.close()
    print(json.dumps({"tool": "bench_deep_topster", **ident, "docs": args.docs, "vocab": args.vocab, "reps": args.reps,
                      "rows": rows, "parity": parity}))


if __name__ == "__main__":
    main()
