#!/usr/bin/env python
"""Where the keyword kernel's time goes at bench.py's shape, split by the planner's density test. Builds the bench's collection
(bench.build_workload: 10 M documents, 1 M-token Zipf vocabulary, 4..12 tokens, persistent `cat` filters) and its batch 0
(bench.make_batches, rank 0) in the resolved form the `value` step times: one 3-token combination per query, Topster 250, stride
100, half the queries filtered. The batch is split into its ALL-DENSE queries (every required list has a dense bitmap: the
library's own list_dense array, i.e. df >= n_docs / TSGPU_DENSE_DIV) and the rest; each subset and the whole batch go through
keyword_search. For every (subset, TSGPU_DENSE_COST) it reports kw_search_kernel's device time (ms_kw_search), the whole call
(ms_total), kw_driver_ids, kw_probe_ids and kw_matches: median of --reps calls after one warm-up call. TSGPU_DENSE_COST is read
by every planning call, so one process sweeps it; 0 keeps every combination on the driver-probe tiles.

A/B against another build: TSGPU_LIB_PATH=<other libtsgpu.so> and --costs default. Prints one JSON line per measurement and
a final one with the GPU's name and power limit, read in the same run. Needs a CUDA device."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


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
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--costs", default="0,0.5,1,2,4,8", help="TSGPU_DENSE_COST values to sweep, or 'default' (leave it unset)")
    ap.add_argument("--label", default="")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_dense_kw needs a CUDA device")
    import bench
    from typesense_b200 import capi, structs as S
    ident = gpu_identity()
    wargs = types.SimpleNamespace(docs=args.docs, vocab=args.vocab, dim=768, batch=args.batch, workload="keyword10m")
    w = bench.build_workload(wargs, "cuda", 0, False)
    b0 = bench.make_batches(wargs, w, 1, 0)[0][0]
    gi = capi.GpuIndex(args.docs, 0)
    fid = gi.load_field(w.fd.flat)
    gi.load_sort_column(w.points)
    handles = [gi.filter_create(f) for f in w.filters]
    list_dense = gi.field_array(fid, 7)                    # dense slot of each list, or 0xFFFFFFFF
    dense_q = [i for i, q in enumerate(b0.queries)
               if all(list_dense[r[0]] != 0xFFFFFFFF for r in q.combos[0].rows[:q.combos[0].n_required])]
    rest_q = sorted(set(range(len(b0.queries))) - set(dense_q))
    subsets = {"all": b0.with_filter_handles(handles),
               "dense": S.KwBatch([b0.queries[i] for i in dense_q], [0], w.filters).with_filter_handles(handles),
               "rest": S.KwBatch([b0.queries[i] for i in rest_q], [0], w.filters).with_filter_handles(handles)}
    costs = [None] if args.costs == "default" else [float(x) for x in args.costs.split(",")]
    rows = []
    for cost in costs:
        if cost is None:
            os.environ.pop("TSGPU_DENSE_COST", None)
        else:
            os.environ["TSGPU_DENSE_COST"] = repr(cost)
        for name, b in subsets.items():
            bs = b.struct()
            gi.keyword_search(b, 100, bstruct=bs)          # warm-up
            st = []
            for _ in range(args.reps):
                gi.keyword_search(b, 100, bstruct=bs)
                st.append(gi.stats())
            row = {"label": args.label, "dense_cost": cost, "subset": name, "queries": b.n_queries,
                   "ms_kw_search": round(statistics.median(s["ms_kw_search"] for s in st), 3),
                   "ms_kw_search_min": round(min(s["ms_kw_search"] for s in st), 3),
                   "ms_total": round(statistics.median(s["ms_total"] for s in st), 3)}
            row.update({k: int(st[-1][k]) for k in ("kw_driver_ids", "kw_probe_ids", "kw_matches")})
            rows.append(row)
            print(json.dumps(row), flush=True)
    gi.close()
    print(json.dumps({"tool": "bench_dense_kw", **ident, "label": args.label, "docs": args.docs, "vocab": args.vocab,
                      "batch": args.batch, "dense_queries": len(dense_q), "reps": args.reps, "rows": rows}))


if __name__ == "__main__":
    main()
