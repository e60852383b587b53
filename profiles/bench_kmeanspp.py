"""k-means++ seeding over every row on the device (nk_index_kmeanspp) against the host path ClusterIndex uses by default.
Prints one JSON line per run and appends them to --out (default: nothing written).

    python profiles/bench_kmeanspp.py --out profiles/kmeanspp_h100.jsonl

Corpora: N=1M d=1024 fp32 generated on the device: uniform (bench.py's generator, seed 42) and fill_clustered (seed 42,
1000 centres, sigma 0.1).  Runs: K = 707 (optimalK(1M)) and K = 1000, with the triangle-inequality skip on and off
(NK_KMPP_PRUNE).  Per run: whole-call time (host clock around the synchronous call), rows read, kernel time per seed (CUDA
events around each seed's kernels, nk_index_scan_time_ms, in a second call with timing on), the rest of the call per
seed (host pick and copies: whole call / K - kernel time per seed), and the GB/s of rows actually read over the kernel
time.  The host path (ClusterIndex._init_rows + _init_kmeanspp over a 200 000-row sample) is timed once, over its first
10 seeds, and reported per seed; it is not extrapolated.  The card's name and power limit are read in the same run."""
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

CORPUS_SEED = 42


def gpu_record():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout.strip()
        name, plim, sm, smax = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock_after_timing": sm, "sm_clock_max": smax}
    except Exception as e:  # the record says so instead of guessing
        return {"error": f"nvidia-smi: {e}"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--ks", default="707,1000")
    ap.add_argument("--host-steps", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import numpy as np
    from nornicdb_b200.cluster_index import ClusterIndex
    from nornicdb_b200.knn import KnnIndex

    n, d = args.rows, args.dim
    lines = []
    for corpus in ("uniform", "clustered"):
        ix = KnnIndex(d, metric="euclidean")
        if corpus == "uniform":
            ix.fill_uniform(n, CORPUS_SEED)
        else:
            ix.fill_clustered(n, CORPUS_SEED, 1000, 0.1)
        ix.kmeanspp(4, 0, [0.5, 0.5, 0.5])  # warm-up: module load, scratch allocation
        for K in [int(k) for k in args.ks.split(",")]:
            rng = np.random.default_rng(K)
            first, u = int(rng.integers(n)), rng.random(K - 1)
            outs = {}
            for prune in ("1", "0"):
                os.environ["NK_KMPP_PRUNE"] = prune
                t0 = time.perf_counter()
                r = ix.kmeanspp(K, first, u)
                wall = time.perf_counter() - t0
                ix.enable_timing(True)
                ix.kmeanspp(K, first, u)
                ix.enable_timing(False)
                kms, _ = ix.scan_time_ms()
                outs[prune] = r
                bytes_read = r.rows_read * d * 4
                rec = {"bench": "kmeanspp", "corpus": corpus, "rows": n, "dim": d, "K": K, "prune": int(prune),
                       "call_s": round(wall, 4), "rows_read": r.rows_read, "rows_read_per_seed": round(r.rows_read / K),
                       "kernel_ms_per_seed": round(kms / K, 4), "rest_ms_per_seed": round(wall * 1e3 / K - kms / K, 4),
                       "rest_share_of_seed": round(1.0 - kms / (wall * 1e3), 4),
                       "gbps_rows_read": round(bytes_read / (kms * 1e-3) / 1e9, 1),
                       "potential": float(r.potential[-1])}
                lines.append(rec)
                print(json.dumps(rec), flush=True)
            same = bool((outs["1"].seeds == outs["0"].seeds).all() and (outs["1"].potential == outs["0"].potential).all())
            print(json.dumps({"bench": "kmeanspp_prune_identical", "corpus": corpus, "K": K, "identical": same}), flush=True)
            assert same
        if corpus == "uniform":
            # the host path ClusterIndex takes by default: a 200 000-row sample read back one row per call, then numpy
            ci = ClusterIndex.__new__(ClusterIndex)
            ci._ix, ci.dimensions, ci.rng, ci.init_sample = ix, d, np.random.default_rng(1), 200_000
            t0 = time.perf_counter()
            rows = ci._init_rows(n)
            t_rows = time.perf_counter() - t0
            t0 = time.perf_counter()
            ci._init_kmeanspp(args.host_steps, rows)
            t_steps = time.perf_counter() - t0
            rec = {"bench": "kmeanspp_host_sample", "rows": n, "dim": d, "sample": 200_000, "read_sample_s": round(t_rows, 3),
                   "seeds_timed": args.host_steps, "s_per_seed": round(t_steps / args.host_steps, 4)}
            lines.append(rec)
            print(json.dumps(rec), flush=True)
        ix.release()
    os.environ.pop("NK_KMPP_PRUNE", None)
    rec = {"bench": "kmeanspp_card", **gpu_record()}
    lines.append(rec)
    print(json.dumps(rec), flush=True)
    if args.out:
        with open(args.out, "a") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
