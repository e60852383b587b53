"""Search by stored row (nk_search_rows): the k-NN graph of an index, against the same blocks of queries sent through
nk_search (host queries, k+1, the query's own row dropped on the host).  Prints one JSON line per workload and appends them
to --out (default: nothing written).

    python profiles/bench_knn_graph.py --out profiles/knn_graph_h100.jsonl

Workloads (fp32, cosine, d=1024, k=10; corpora from the device generators with seed 42, as in bench.py):
  graph_1m            the full graph of N=1M uniform rows: 1M queries, 977 blocks of 1024
  rows_10m_q16384     N=10M uniform rows, the first 16 384 rows as queries
  graph_1m_clustered  the full graph of N=1M clustered rows (1000 centres, sigma 0.1): near-ties and near-duplicates, with
                      the filter's retry counters over the timed calls
Timing: host wall clock around each synchronous call (both end in a device synchronise); nk_search_rows and the nk_search
blocks alternate, --steps times each after one warm-up pass over a few blocks; medians and every sample are reported.  scan ms
= CUDA events around the scan kernels (nk_index_scan_time_ms), summed over the call.  The nk_search arm reads the query rows
back to the host once, untimed, and its per-block host work (slicing, dropping self) is inside its timed region.  Results of
the two arms are compared bit for bit.  The whole-call pair rate is 2*N*Q*d / wall time (every (query, row) pair scored once
at d multiply-adds); it is put beside NVIDIA's data-sheet dense BF16 figure for the H100 SXM, which it is not a kernel's share
of.  The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.bench_range import gpu_record, median  # noqa: E402

CORPUS_SEED = 42
BLOCK = 1024
DATASHEET_DENSE_BF16_TFLOPS = 989.0  # H100 SXM, dense, 700 W card


def drop_self(idx, sc, ids, k):
    """The self rule of nk_search_rows on [Q x k'] lists: remove the query's own row, else the last slot; keep min(k, k')."""
    import numpy as np
    Q, kk = idx.shape
    hit = idx == ids[:, None].astype(np.uint32)
    drop = np.where(hit.any(1), hit.argmax(1), kk - 1)
    keep = np.ones((Q, kk), bool)
    keep[np.arange(Q), drop] = False
    ke, m = min(k, kk), min(k, kk - 1)
    out_i, out_s = np.full((Q, ke), 0xFFFFFFFF, np.uint32), np.zeros((Q, ke), np.float32)
    out_i[:, :m], out_s[:, :m] = idx[keep].reshape(Q, kk - 1)[:, :m], sc[keep].reshape(Q, kk - 1)[:, :m]
    return out_i, out_s


def run_workload(ix, name, ids, k, steps, corpus, n, d):
    import numpy as np
    Q = len(ids)
    x = ix.read_rows(0, int(ids.max()) + 1)  # the query rows as stored, for the nk_search arm
    ref_i = np.empty((Q, k), np.uint32)
    ref_s = np.empty((Q, k), np.float32)

    def by_search():
        for b in range(0, Q, BLOCK):
            i, s = ix.search(x[ids[b:b + BLOCK]], k + 1)
            ref_i[b:b + BLOCK], ref_s[b:b + BLOCK] = drop_self(i, s, ids[b:b + BLOCK], k)

    # warm-up: every block shape both arms use (a full block, and the last one)
    tail = ids[(Q - 1) // BLOCK * BLOCK:]
    for w in (ids[:BLOCK], tail):
        ix.search_rows(w, k)
        ix.search(x[w], k + 1)
    c0 = ix.debug_counters()
    ix.enable_timing(True)
    ix.scan_time_ms()
    t_rows, t_search, scan_rows, scan_search = [], [], [], []
    for _ in range(steps):
        t0 = time.perf_counter()
        gi, gs = ix.search_rows(ids, k)
        t_rows.append(time.perf_counter() - t0)
        scan_rows.append(ix.scan_time_ms()[0])
        path_rows = ix.last_path()
        t0 = time.perf_counter()
        by_search()
        t_search.append(time.perf_counter() - t0)
        scan_search.append(ix.scan_time_ms()[0])
        path_search = ix.last_path()
    ix.enable_timing(False)
    c1 = ix.debug_counters()
    identical = bool(np.array_equal(gi, ref_i) and np.array_equal(gs.view(np.uint32), ref_s.view(np.uint32)))
    assert identical, f"{name}: nk_search_rows differs from nk_search(k+1) with self dropped"
    assert not (gi == ids[:, None]).any()
    t = median(t_rows)
    pair_rate = 2.0 * n * Q * d / t / 1e12
    return {
        "bench": "knn_graph", "workload": name, "corpus": corpus, "rows": n, "dim": d, "Q": Q, "k": k, "metric": "cosine",
        "dtype": "f32", "blocks": (Q + BLOCK - 1) // BLOCK,
        "search_rows_s_median": round(t, 4), "search_rows_s": [round(v, 4) for v in t_rows],
        "search_rows_scan_ms_median": round(median(scan_rows), 2),
        "search_rows_queries_per_s": round(Q / t, 1),
        "nk_search_blocks_s_median": round(median(t_search), 4), "nk_search_blocks_s": [round(v, 4) for v in t_search],
        "nk_search_blocks_scan_ms_median": round(median(scan_search), 2),
        "search_rows_minus_nk_search_s": round(t - median(t_search), 4),
        "whole_call_pair_rate_tflops": round(pair_rate, 1),
        "whole_call_pair_rate_over_datasheet_dense_bf16": round(pair_rate / DATASHEET_DENSE_BF16_TFLOPS, 3),
        "datasheet_dense_bf16_tflops": DATASHEET_DENSE_BF16_TFLOPS,
        "retry_counters_over_timed_and_warmup_calls": {"bf16_stage_retries": c1["bf16_stage_retries"] - c0["bf16_stage_retries"],
                                                       "exact_stage_runs": c1["exact_stage_runs"] - c0["exact_stage_runs"]},
        "bit_identical_to_nk_search_k_plus_1": identical, "path_search_rows": path_rows, "path_nk_search": path_search,
        "steps": steps,
        "timing": "median wall clock per synchronous call, nk_search_rows and the nk_search blocks alternating; scan ms: CUDA "
                  "events around the scan kernels, summed over the call; pair rate = 2*N*Q*d / search_rows wall time",
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default="")
    ap.add_argument("--only", default="", help="comma-separated workload names (default: all three)")
    ap.add_argument("--scale", type=float, default=1.0, help="multiply every N (a small value rehearses the script)")
    args = ap.parse_args()
    import numpy as np
    from nornicdb_b200.knn import KnnIndex

    d, k = 1024, 10
    n1, n10 = int(1_000_000 * args.scale), int(10_000_000 * args.scale)
    work = [("graph_1m", "uniform", n1, n1), ("rows_10m_q16384", "uniform", n10, min(16_384, n10)),
            ("graph_1m_clustered", "clustered 1000 centres sigma 0.1", n1, n1)]
    only = set(filter(None, args.only.split(",")))
    records = []
    for name, corpus, n, Q in work:
        if only and name not in only:
            continue
        ix = KnnIndex(d, metric="cosine")
        if corpus == "uniform":
            ix.fill_uniform(n, CORPUS_SEED)
        else:
            ix.fill_clustered(n, CORPUS_SEED, n_centres=1000, sigma=0.1)
        rec = run_workload(ix, name, np.arange(Q, dtype=np.int64), k, args.steps, corpus, n, d)
        ix.release()
        print(json.dumps(rec), flush=True)
        records.append(rec)
    gpu = gpu_record()
    for rec in records:
        rec["gpu"] = gpu
        line = json.dumps(rec)
        print(line)
        if args.out:
            with open(args.out, "a") as f:
                f.write(line + "\n")


if __name__ == "__main__":
    main()
