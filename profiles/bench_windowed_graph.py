"""Windowed k-NN graph (a time-local graph: each row's list holds only rows within +-1 day of its own timestamp): the full
windowed build (nk_search_rows_windowed over every row), and nk_knn_graph_update_windowed / nk_knn_graph_remap_windowed
against a windowed rebuild.  Prints one JSON line per workload and appends them to --out (default: nothing written).

    python profiles/bench_windowed_graph.py --out profiles/windowed_graph_h100.jsonl

Base: N=1M uniform fp32 rows from the device generator (seed 42, as in bench.py), d=1024, cosine, k=10, the AUTO path (the
graph calls run the graph path it resolves to).  Value keys: uniform timestamps in seconds over one year; row r's window is
its own key +-1 day (knn.band_windows).  Workloads: append 1024 rows stamped within the last day (the realistic insert),
append 1024 rows at random times, rewrite 100 rows, re-value 100 rows (each moved by a week: its band moves with it,
reported as rewritten), remove 100 random rows with nk_index_remove_swap (the remap, the row map kept by GraphRowMap, the keys
and windows following the swaps).  The changes are drawn once and replayed every repetition.  Each repetition restores the
base index and its keys, makes the change, runs the update on the base graph, then the windowed rebuild, and asserts that
both are bit-identical.  Timing: host wall clock around each synchronous call; scan ms = CUDA events around the scan kernels
(nk_index_scan_time_ms), summed over the call.  Medians of --steps repetitions, every sample reported.  The card's name and
power limit are read in the same run."""
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
K = 10
DAY = 86_400
T0 = 1_700_000_000
YEAR = 365 * DAY


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--out", default="")
    ap.add_argument("--scale", type=float, default=1.0, help="multiply N and the change sizes (a small value rehearses the script)")
    ap.add_argument("--workloads", default="", help="comma-separated names to run (default: all)")
    args = ap.parse_args()
    import numpy as np
    from nornicdb_b200.knn import GraphRowMap, KnnIndex, band_windows
    n, d = max(int(1_000_000 * args.scale), 4096), 1024
    rng = np.random.default_rng(12)
    keys0 = (T0 + rng.integers(0, YEAR, n)).astype(np.uint64)

    ix = KnnIndex(d, metric="cosine")
    ix.set_path("auto")

    def restore():
        ix.fill_uniform(n, CORPUS_SEED)
        ix.set_row_values(keys0)

    lines = []

    def emit(rec):
        rec.update({"rows_before": n, "dim": d, "k": K, "metric": "cosine", "dtype": "f32", "path": "auto",
                    "keys": "uniform timestamps (s) over 365 days", "window": "own key +- 1 day", "steps": args.steps,
                    "gpu": gpu_record()})
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    restore()
    w0 = band_windows(keys0, DAY)
    ix.enable_timing(True)
    ix.scan_time_ms()
    t_b, s_b = [], []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        base_i, base_s = ix.search_rows(np.arange(n), K, windows=w0)
        t_b.append(time.perf_counter() - t0)
        s_b.append(ix.scan_time_ms()[0])
    ix.enable_timing(False)
    emit({"bench": "windowed_graph", "workload": "build", "call": "nk_search_rows_windowed (every row)",
          "windowed_build_s_median": round(median(t_b), 3), "windowed_build_s": [round(v, 3) for v in t_b],
          "windowed_build_scan_ms_median": round(median(s_b), 1),
          "short_lists": int((base_i[:, K - 1] == 0xFFFFFFFF).sum()),
          "timing": "median wall clock per synchronous call; scan ms: CUDA events around the scan kernels, summed over the call"})

    n_app = max(int(1024 * args.scale), 2)
    last = int(keys0.max())
    workloads = [("append_1024_last_day", n_app, "last_day", 0, 0, 0), ("append_1024_random_time", n_app, "random", 0, 0, 0),
                 ("rewrite_100", 0, "", 100, 0, 0), ("revalue_100_by_a_week", 0, "", 0, 100, 0), ("remove_100", 0, "", 0, 0, 100)]
    if args.workloads:
        wanted = args.workloads.split(",")
        workloads = [wl for wl in workloads if wl[0] in wanted]
    for name, n_new, when, n_rewrite, n_revalue, n_remove in workloads:
        new = rng.uniform(-1, 1, (n_new, d)).astype(np.float32)
        if when == "last_day":
            new_keys = (last - DAY + rng.integers(0, DAY, n_new)).astype(np.uint64)
        else:
            new_keys = (T0 + rng.integers(0, YEAR, n_new)).astype(np.uint64)
        rewrite = rng.choice(n, n_rewrite, replace=False)
        vecs = rng.uniform(-1, 1, (n_rewrite, d)).astype(np.float32)
        revalue = rng.choice(n, n_revalue, replace=False)
        removes = [int(rng.integers(n - i)) for i in range(n_remove)]
        t_up, t_rb, scan_up, scan_rb, changed_lists = [], [], [], [], []
        c0 = ix.debug_counters()
        for _ in range(args.steps):
            restore()
            keys = keys0.copy()
            m = GraphRowMap(n)
            changed = []
            if n_new:
                ix.append(new)
                ix.set_row_values(new_keys, first_row=n)
                keys = np.concatenate([keys, new_keys])
                m.append(n_new)
            for r, v in zip(rewrite, vecs):
                ix.update_row(int(r), v)
                m.update_row(int(r))
                changed.append(int(r))
            for r in revalue:
                keys[r] += np.uint64(7 * DAY)
                ix.set_row_values(keys[r:r + 1], first_row=int(r))
                m.update_row(int(r))
                changed.append(int(r))
            for r in removes:
                ix.remove_swap(r)
                m.remove_swap(r)
                keys[r] = keys[len(keys) - 1]
                keys = keys[:-1]
            w = band_windows(keys, DAY)
            ix.enable_timing(True)
            ix.scan_time_ms()
            t0 = time.perf_counter()
            if n_remove:
                ui, us, nch = ix.remap_knn_graph(base_i, base_s, n, m, windows=w)
            else:
                ui, us, nch = ix.update_knn_graph(base_i, base_s, n, changed, windows=w)
            t_up.append(time.perf_counter() - t0)
            scan_up.append(ix.scan_time_ms()[0])
            t0 = time.perf_counter()
            ri, rs = ix.search_rows(np.arange(len(ix)), K, windows=w)
            t_rb.append(time.perf_counter() - t0)
            scan_rb.append(ix.scan_time_ms()[0])
            ix.enable_timing(False)
            identical = bool(np.array_equal(ui, ri) and np.array_equal(us.view(np.uint32), rs.view(np.uint32)))
            assert identical, f"{name}: the updated windowed graph differs from the windowed rebuild"
            changed_lists.append(nch)
        c1 = ix.debug_counters()
        emit({"bench": "windowed_graph", "workload": name,
              "call": "nk_knn_graph_remap_windowed" if n_remove else "nk_knn_graph_update_windowed",
              "appended": n_new, "appended_at": when or None, "rewritten": n_rewrite, "revalued": n_revalue, "removed": n_remove,
              "update_s_median": round(median(t_up), 4), "update_s": [round(v, 4) for v in t_up],
              "update_scan_ms_median": round(median(scan_up), 2),
              "rebuild_s_median": round(median(t_rb), 4), "rebuild_s": [round(v, 4) for v in t_rb],
              "rebuild_scan_ms_median": round(median(scan_rb), 2),
              "rebuild_over_update": round(median(t_rb) / median(t_up), 1),
              "old_lists_changed": changed_lists[-1],
              "retry_counters": {c: c1[c] - c0[c] for c in ("bf16_stage_retries", "exact_stage_runs")},
              "bit_identical_to_rebuild": True,
              "timing": "median wall clock per synchronous call, update and windowed rebuild alternating on a restored base "
                        "index; scan ms: CUDA events around the scan kernels, summed over the call"})
    ix.release()
    if args.out:
        with open(args.out, "a") as fo:
            for rec in lines:
                fo.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
