#!/usr/bin/env python
"""Cost of deep vector and hybrid searches (TSGPU_VEC_DEEP_TOPSTER: a Topster larger than TSGPU_MAX_TOPK = 1024).

Data: --docs documents (default 1 M) with a Zipf title field (4..12 tokens, 100 k vocabulary), one sort column and --dim-d
vectors (default 768), the graph built on the device by tsgpu_index_build_hnsw. Runs, each with batches of 1 and 64 queries:

  vector_K   q=* + vector query, k = K, sorted by vector distance
  hybrid_K   one frequent token (more keyword matches than K) + vector query, k = K, alpha 0.3, sorted by text match

at K = 1024 (the ordinary kernels) and K in {1025, 2500, 4096} (the deep path). Per run: the median over --reps calls (after a
warm-up call) of the whole call on the device (tsgpu_get_stats ms_total), the vector stage (ms_knn), the fusion / assembly
(ms_fuse) and, on the deep hybrid path, its phases (prep, serial replay, rerank, final sort: the slowest deep query of each),
the workspace bytes, and the oracle's CPU time for the same queries (one thread, --oracle-queries of them). Prints one JSON
line with the GPU's name and power limit, read in the same run. Needs a CUDA device."""
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    name, power = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-queries", type=int, default=1)
    a = ap.parse_args()
    import torch
    import oracle_lib as ol
    assert torch.cuda.is_available(), "needs a CUDA device"
    ident = gpu_identity()
    n, dim = a.docs, a.dim
    t0 = time.time()
    fd = synth.make_string_field(n, 100_000, 4, 12, seed=7, device="cuda")
    pts = synth.make_points(n, 13, hi=1000)
    vec = synth.make_vectors(n, dim, 5, device="cuda")
    gi = capi.GpuIndex(n, 0)
    gi.load_field(fd.flat)
    gi.load_sort_column(pts)
    gi.build_hnsw(vec, 16, 100, 100, keep_device_vectors=True)
    t_setup = time.time() - t0
    vec_np = vec.cpu().numpy()
    graph = gi.export_hnsw(vec_np)
    oi = ol.OracleIndex(n, [fd.flat], [pts], graph) if a.oracle_queries > 0 else None
    rng = np.random.default_rng(3)
    qv_all = synth.make_vectors(64, dim, 99).numpy()
    VSORT = ((S.SORT_VECTOR_DISTANCE, -1, -1, 0), (S.SORT_NUMERIC, 0, 1, 0), (S.SORT_NONE, -1, 1, 0))
    TSORT = ((S.SORT_TEXT_MATCH, -1, 1, 0), (S.SORT_NUMERIC, 0, 1, 0), (S.SORT_NONE, -1, 1, 0))
    rows = []
    for kind in ("vector", "hybrid"):
        for K in (1024, 1025, 2500, 4096):
            for nq in (1, 64):
                flags = capi.QFLAG_DEEP_TOPSTER if K > 1024 else 0
                if kind == "vector":
                    qs = [S.Query([], sort=VSORT, topk=K, flags=S.FLAG_PRIORITIZE_EXACT_MATCH | flags) for _ in range(nq)]
                else:
                    qs = [S.Query([S.Combo([[int(rng.integers(0, 20))]], 1)], sort=TSORT, topk=K, flags=S.FLAG_PRIORITIZE_EXACT_MATCH | flags)
                          for _ in range(nq)]
                b = S.KwBatch(qs, [0])
                vp = S.vec_params(k=K, ef=10, alpha=0.3, fetch_size=K, flags=capi.VEC_DEEP_TOPSTER)
                call = gi.vector_search if kind == "vector" else gi.hybrid_search
                qv = qv_all[:nq]
                call(b, qv, vp, K)
                st = []
                wall = []
                for _ in range(a.reps):
                    t1 = time.perf_counter()
                    out = call(b, qv, vp, K)
                    wall.append((time.perf_counter() - t1) * 1e3)
                    st.append(gi.stats())
                med = lambda key: round(statistics.median(s[key] for s in st), 3)   # noqa: E731
                row = {"run": f"{kind}_{K}", "batch": nq, "records_max": int(out[1].max()), "ms_call": med("ms_total"),
                       "ms_vector_stage": med("ms_knn"), "ms_fuse": med("ms_fuse"), "ms_keyword": med("ms_keyword"),
                       "ms_host_wall": round(statistics.median(wall), 3)}
                if K > 1024:
                    row.update({"ms_deep_prep": med("ms_deep_fuse_prep"), "ms_deep_replay": med("ms_deep_fuse_replay"),
                                "ms_deep_rerank": med("ms_deep_fuse_rerank"), "ms_deep_sort": med("ms_deep_fuse_sort"),
                                "deep_fuse_bytes": int(st[-1]["deep_fuse_bytes"])})
                if oi is not None and nq == 1 and a.oracle_queries > 0:
                    t1 = time.perf_counter()
                    (oi.vector_search if kind == "vector" else oi.hybrid_search)(b, qv, vp, K)
                    row["oracle_cpu_ms"] = round((time.perf_counter() - t1) * 1e3, 1)
                rows.append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
    gi.close()
    print(json.dumps({**ident, "docs": n, "dim": dim, "setup_s": round(t_setup, 1), "runs": rows}))


if __name__ == "__main__":
    main()
