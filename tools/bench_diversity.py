#!/usr/bin/env python
"""Cost of the diversity re-ranking (tsgpu_diversify_batch, the MMR order of Index::populate_result_kvs) for (nq, K) in
{(1, 250), (64, 250), (4096, 250), (64, 1024), (1, 5000)}: nq queries of K records each, two metrics — jaccard on an array facet
(1..7 values, about 4, of 1,000 per document) and equality on a sort column (20 values). Records are keyword-like (vector distance -1)
over 1 M documents, passed in host memory.

Per shape: the device time of the call (tsgpu_get_stats: ms_kernels = the counting pass + the re-ranking kernel, ms_total = the
whole call on the library's stream, copies included; median of --reps calls after one warm-up call) and the host wall time. Next to
it, the CPU time of tso_diversify — the oracle's transcription of the reference loop (K^3 / 6 pair lookups through a map), which is
not the reference's own code — on a sample of the same lists (--oracle-queries of them, single-threaded, K <= --oracle-max-k);
the re-ranked records of those lists are compared with the oracle's. Prints the GPU's name and power limit, read in the same run,
and one JSON line. Needs a CUDA device."""
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
from typesense_b200 import capi                           # noqa: E402
from typesense_b200.structs import KV_DTYPE              # noqa: E402


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:                                  # noqa: BLE001
        return {"gpu": None, "power_limit": None, "error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--shapes", default="1x250,64x250,4096x250,64x1024,1x5000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-queries", type=int, default=2)
    ap.add_argument("--oracle-max-k", type=int, default=250)
    args = ap.parse_args()
    ident = gpu_identity()
    print(f"GPU: {ident.get('gpu')}, power limit {ident.get('power_limit')}", flush=True)
    rng = np.random.default_rng(1)
    n = args.docs
    lens = rng.integers(1, 8, n)
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    vals = rng.integers(0, 1000, int(off[-1])).astype(np.uint32)
    col = rng.integers(0, 20, n).astype(np.int64)
    gi = capi.GpuIndex(n, 0)
    f = gi.load_facet(1000, off, vals)
    c = gi.load_sort_column(col)
    dev_metrics = [(f, 0, capi.DIV_JACCARD, 1.0), (None, c, capi.DIV_EQUALITY, 1.0)]
    ora_metrics = [("facet", off, vals, capi.DIV_JACCARD, 1.0), ("sort", col, capi.DIV_EQUALITY, 1.0)]
    import diversity_double as dd
    dd.build_lib()                                               # the oracle's library is compiled before anything is timed
    rows = []
    for shape in args.shapes.split(","):
        nq, K = (int(x) for x in shape.split("x"))
        kv = np.zeros((nq, K), KV_DTYPE)
        for q in range(nq):
            kv["key"][q] = rng.choice(n, K, replace=False)
        kv["vector_distance"] = -1.0
        kv["scores"][:, :, 0] = np.arange(K, 0, -1)
        cnt = np.full(nq, K, np.uint32)
        lam = np.full(nq, 0.5, np.float32)
        out = np.zeros_like(kv)
        gi.diversify(dev_metrics, lam, kv, cnt, out=out)            # warm-up
        dev_ms, tot_ms, wall_ms = [], [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            gi.diversify(dev_metrics, lam, kv, cnt, out=out)
            wall_ms.append((time.perf_counter() - t0) * 1e3)
            s = gi.stats()
            dev_ms.append(s["ms_kernels"])
            tot_ms.append(s["ms_total"])
        row = {"nq": nq, "K": K, "device_kernels_ms": round(statistics.median(dev_ms), 4), "device_call_ms": round(statistics.median(tot_ms), 4),
               "host_wall_ms": round(statistics.median(wall_ms), 3)}
        if K <= args.oracle_max_k and args.oracle_queries > 0:
            m = min(nq, args.oracle_queries)
            t0 = time.perf_counter()
            same = True
            for q in range(m):
                same &= dd.oracle_diversify(n, ora_metrics, 0.5, kv[q]).tobytes() == out[q].tobytes()
            row["oracle_transcription_cpu_ms_per_query"] = round((time.perf_counter() - t0) * 1e3 / m, 2)
            row["oracle_equal"] = bool(same)
        else:
            row["oracle_transcription_cpu_ms_per_query"] = None
        rows.append(row)
        print(f"nq {nq:5d} K {K:5d}: device kernels {row['device_kernels_ms']:9.3f} ms, call {row['device_call_ms']:9.3f} ms, host wall "
              f"{row['host_wall_ms']:9.3f} ms | oracle transcription of the reference loop (CPU, 1 thread): "
              f"{row['oracle_transcription_cpu_ms_per_query']} ms per query, equal {row.get('oracle_equal')}", flush=True)
    print(json.dumps({"bench": "diversity", **ident, "docs": n, "rows": rows}))


if __name__ == "__main__":
    main()
