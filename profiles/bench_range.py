"""Range search (nk_search_range) at the headline shape, against nk_search k=10 on the same queries.  Prints one JSON line
per threshold level and appends them to --out (default: nothing written).

    python profiles/bench_range.py --steps 10 --warmup 2 --out profiles/range_h100.jsonl

Corpus: the counter-based generator of bench.py (seed 42), N=10M d=1024 fp32 cosine, generated on the device; queries:
seed 1337, Q=64.  Thresholds per query, one level at a time: the score of its 10th and 1000th neighbour (nk_search k=1000),
and of its ~100 000th (the 10 000th best of a 1M-row sample, rows regenerated on the device and scored with torch in
fp32).  Timing: host wall clock around each synchronous call (both calls end in a device synchronise), range search and
nk_search alternating, medians reported; scan ms = CUDA events around the scan kernels (nk_index_scan_time_ms), per call.
The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CORPUS_SEED, QUERY_SEED = 42, 1337


def gpu_record():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout.strip()
        name, plim, sm, smax = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock_after_timing": sm, "sm_clock_max": smax}
    except Exception as e:  # the record says so instead of guessing
        return {"error": f"nvidia-smi: {e}"}


def median(v):
    v = sorted(v)
    return v[len(v) // 2] if len(v) % 2 else 0.5 * (v[len(v) // 2 - 1] + v[len(v) // 2])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--q", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import numpy as np
    import torch
    from nornicdb_b200.knn import KnnIndex, fill_uniform_device
    import oracle

    n, d, Q = args.rows, args.dim, args.q
    ix = KnnIndex(d, metric="cosine")
    ix.fill_uniform(n, CORPUS_SEED)
    q = oracle.fill_uniform(Q, d, QUERY_SEED)
    _, s1000 = ix.search(q, 1000)
    # ~100 000th neighbour: the 10 000th best of rows [0, n/10), scored in fp32 on the device
    sample = n // 10
    x = torch.empty((sample, d), dtype=torch.float32, device="cuda")
    fill_uniform_device(0, x.data_ptr(), sample, d, CORPUS_SEED, 0, 0)
    torch.cuda.synchronize()
    qt = torch.from_numpy(q).cuda()
    qt = qt / qt.norm(dim=1, keepdim=True)
    xn = x.norm(dim=1)
    s_big = torch.cat([(qt @ x[i:i + 1_000_000].T) / xn[i:i + 1_000_000][None, :] for i in range(0, sample, 1_000_000)], dim=1)
    t_big = torch.topk(s_big, 10_000, dim=1).values[:, -1].cpu().numpy().astype(np.float32)
    del x, s_big, xn
    torch.cuda.empty_cache()
    levels = {"10th": s1000[:, 9].copy(), "1000th": s1000[:, 999].copy(), "~100000th": t_big}
    records = []
    for name, thr in levels.items():
        for _ in range(args.warmup):
            ix.search_range(q, thr)
            ix.search(q, 10)
        t_range, t_knn, scan_range, scan_knn = [], [], [], []
        ix.enable_timing(True)
        ix.scan_time_ms()
        for _ in range(args.steps):
            t0 = time.perf_counter()
            res = ix.search_range(q, thr)
            t_range.append((time.perf_counter() - t0) * 1e3)
            scan_range.append(ix.scan_time_ms()[0])
            path_range = ix.last_path()
            t0 = time.perf_counter()
            ix.search(q, 10)
            t_knn.append((time.perf_counter() - t0) * 1e3)
            scan_knn.append(ix.scan_time_ms()[0])
            path_knn = ix.last_path()
        ix.enable_timing(False)
        counts = np.array([len(i) for i, _ in res])
        # the threshold came from a returned score: at least that many rows qualify (10th / 1000th levels)
        need = {"10th": 10, "1000th": 1000}.get(name, 0)
        assert (counts >= need).all(), (name, counts.min())
        rec = {"bench": "range_search", "rows": n, "dim": d, "Q": Q, "metric": "cosine", "dtype": "f32", "threshold_at": name,
               "range_ms_per_batch_median": round(median(t_range), 3), "range_scan_ms_median": round(median(scan_range), 3),
               "knn_k10_ms_per_batch_median": round(median(t_knn), 3), "knn_k10_scan_ms_median": round(median(scan_knn), 3),
               "results_per_query_min": int(counts.min()), "results_per_query_median": float(np.median(counts)),
               "results_per_query_max": int(counts.max()), "results_total": int(counts.sum()),
               "path_range": path_range, "path_knn": path_knn, "steps": args.steps, "warmup": args.warmup,
               "timing": "median wall clock per synchronous call, range and k=10 alternating; scan ms: CUDA events around the scan kernels"}
        records.append(rec)
    gpu = gpu_record()
    for rec in records:
        rec["gpu"] = gpu
        line = json.dumps(rec)
        print(line)
        if args.out:
            with open(args.out, "a") as f:
                f.write(line + "\n")
    ix.release()


if __name__ == "__main__":
    main()
