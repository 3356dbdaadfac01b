#!/usr/bin/env python
"""Cost of keeping the device mirror of one string field in step with a live collection, at bench.py's field shape (10 M documents,
1 M-token Zipf vocabulary, 4..12 tokens per document). Each figure is a host clock around one C-ABI call, which ends synchronised:

  append_ms    tsgpu_index_append_lists of one write batch: the current full lists of every token that `--batch-docs` random documents
               hold (what the binding hands over after such a batch; the Zipf head makes a few of them millions of postings long)
  compact_ms   tsgpu_index_compact_field after `--k` such batches (their garbage included), keeping the live lists
  reserve_ms   tsgpu_index_reserve_docs from --docs to --grow-to (one sort column on the index)
  reload_ms    the alternative without compaction: tsgpu_index_load_field of the same live lists into a fresh index, from host memory

plus the field's device bytes fresh, after the k batches and after compaction, and the gather's HBM rate: the bytes it reads and
writes (the new field's posting arrays, twice) over the device time between its first and last kernel, as a fraction of the
H100 SXM data sheet's 3.35 TB/s. Prints one JSON line with the GPU's name and power limit. Needs a CUDA device."""
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
from typesense_b200 import capi, structs as S, synth      # noqa: E402

HBM_PEAK = 3.35e12


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:                                  # noqa: BLE001
        return {"gpu": None, "power_limit": None, "error": str(e)}


def sub_field(flat: S.FlatField, toks: np.ndarray) -> S.FlatField:
    """the lists of `toks` (in that order) as one flat field"""
    lo = flat.list_off.astype(np.int64)
    a, b = lo[toks], lo[toks + 1]
    df = b - a
    list_off = np.zeros(len(toks) + 1, np.uint64)
    list_off[1:] = np.cumsum(df)
    post = np.concatenate([np.arange(x, y) for x, y in zip(a, b)]) if len(toks) else np.zeros(0, np.int64)
    po = flat.pos_off.astype(np.int64)
    pa, pb = po[post], po[post + 1]
    pos_off = np.zeros(len(post) + 1, np.uint64)
    pos_off[1:] = np.cumsum(pb - pa)
    # the raw offsets of consecutive postings of a list are contiguous: one slice per list
    positions = np.concatenate([flat.positions[po[x]:po[y]] for x, y in zip(a, b)]) if len(toks) else np.zeros(0, np.uint32)
    return S.FlatField(list_off, flat.ids[post].astype(np.uint32), pos_off, positions.astype(np.uint32), flat.is_array)


def gather_bytes(info: dict) -> int:
    """bytes of the arrays the gather writes (and reads as much of): blocks, packed words, offsets, dense rows"""
    return 2 * (info["n_blocks"] * 12 + info["n_words"] * 4 + info["n_postings"] * 8 + info["n_positions"] * 4
                + info["n_dense"] * info["dense_words"] * 4 * 5 // 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--batch-docs", type=int, default=1000)
    ap.add_argument("--k", type=int, default=4, help="write batches between two compactions")
    ap.add_argument("--cycles", type=int, default=3, help="timed (k appends + compaction) cycles after one warm-up cycle")
    ap.add_argument("--grow-to", type=int, default=12_000_000)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_mirror_maintenance: no CUDA device (this measures the device mirror; there is no CPU path)")
    fd = synth.make_string_field(args.docs, args.vocab, 4, 12, seed=7, device="cuda")
    flat = fd.flat
    rng = np.random.default_rng(3)
    gi = capi.GpuIndex(args.docs, 0)
    f = gi.load_field(flat)
    gi.load_sort_column(synth.make_points(args.docs, seed=13))
    fresh_info = gi.field_info(f)
    L = flat.n_lists
    cur = np.arange(L, dtype=np.int64)                      # token -> list id in the mirror now

    def batch():
        docs = rng.choice(args.docs, args.batch_docs, replace=False)
        toks = np.unique(np.concatenate([fd.doc_tok[fd.doc_off[d]:fd.doc_off[d + 1]] for d in docs])).astype(np.int64)
        return toks, sub_field(flat, toks)

    batches = [batch() for _ in range(args.k)]
    appends, compacts, gather_ms, peak_bytes, rates = [], [], [], [], []
    for cycle in range(args.cycles + 1):
        for toks, bf in batches:
            t0 = time.perf_counter()
            first = gi.append_lists(f, bf)
            t1 = time.perf_counter()
            cur[toks] = first + np.arange(len(toks))
            if cycle:
                appends.append(1e3 * (t1 - t0))
        peak = gi.field_info(f)["device_bytes"]
        live = np.sort(cur)                                  # every token keeps its list
        t0 = time.perf_counter()
        gi.compact_field(f, live)
        t1 = time.perf_counter()
        order = np.argsort(cur, kind="stable")
        cur[order] = np.arange(L)
        info = gi.field_info(f)
        st = gi.stats()
        if cycle:
            compacts.append(1e3 * (t1 - t0))
            gather_ms.append(st["ms_kernels"])
            peak_bytes.append(peak)
            rates.append(gather_bytes(info) / (st["ms_kernels"] * 1e-3) / HBM_PEAK)
    after_info = gi.field_info(f)
    live_flat = sub_field(flat, np.argsort(cur, kind="stable"))
    reloads = []
    for _ in range(2):
        gr = capi.GpuIndex(args.docs, 0)
        t0 = time.perf_counter()
        gr.load_field(live_flat)
        reloads.append(1e3 * (time.perf_counter() - t0))
        gr.close()
    t0 = time.perf_counter()
    gi.reserve_docs(args.grow_to)
    reserve_ms = 1e3 * (time.perf_counter() - t0)
    gi.close()
    out = {"tool": "bench_mirror_maintenance", **gpu_identity(), "docs": args.docs, "vocab": args.vocab, "batch_docs": args.batch_docs,
           "k": args.k, "cycles": args.cycles, "batch_lists": [len(t) for t, _ in batches], "batch_postings": [int(b.list_off[-1]) for _, b in batches],
           "append_ms_median": statistics.median(appends), "compact_ms_median": statistics.median(compacts),
           "gather_kernel_ms_median": statistics.median(gather_ms), "gather_hbm_fraction_median": statistics.median(rates),
           "reload_ms_min": min(reloads), "reserve_ms": reserve_ms, "grow_to": args.grow_to,
           "field_bytes_fresh": fresh_info["device_bytes"], "field_bytes_before_compaction_max": max(peak_bytes),
           "field_bytes_after_compaction": after_info["device_bytes"], "n_dense": after_info["n_dense"]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
