"""k-NN graph update (nk_knn_graph_update, or nk_knn_graph_remap once rows are removed) against a full rebuild (nk_search_rows
over every row).  Prints one JSON line per workload and appends them to --out (default: nothing written).

    python profiles/bench_graph_update.py --out profiles/knn_graph_update_h100.jsonl

Base: N=1M uniform fp32 rows from the device generator (seed 42, as in bench.py), d=1024, cosine, k=10, the 16-bit (shadow)
path forced; its graph is built once.  Workloads: append 1, 1024 or 10 240 uniform rows (host), or rewrite 100 rows
(nk_knn_graph_update); remove 1 or 100 random rows with nk_index_remove_swap, or 100 removals + 100 appends + 100 rewrites
in random order (nk_knn_graph_remap, the row map kept by GraphRowMap).  The changes of a workload are drawn once and replayed
every repetition.  Each repetition restores the base index first (the generator refills it), makes the change, runs the
update or remap on the base graph, then the rebuild, and asserts that both are bit-identical.  Timing: host
wall clock around each synchronous call; scan ms = CUDA events around the scan kernels (nk_index_scan_time_ms), summed over
the call.  Medians of --steps repetitions, every sample reported.  The card's name and power limit are read in the same run."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default="")
    ap.add_argument("--scale", type=float, default=1.0, help="multiply N and the change sizes (a small value rehearses the script)")
    ap.add_argument("--workloads", default="", help="comma-separated names to run (default: all)")
    args = ap.parse_args()
    import numpy as np
    from nornicdb_b200.knn import GraphRowMap, KnnIndex
    n, d = max(int(1_000_000 * args.scale), 4096), 1024
    # (name, appended, rewritten, removed); the workloads that remove rows interleave their changes and run the remap
    workloads = [("append_1", 1, 0, 0), ("append_1024", max(int(1024 * args.scale), 2), 0, 0),
                 ("append_10240", max(int(10240 * args.scale), 4), 0, 0), ("rewrite_100", 0, 100, 0),
                 ("remove_1", 0, 0, 1), ("remove_100", 0, 0, 100), ("mixed_300", 100, 100, 100)]
    if args.workloads:
        wanted = args.workloads.split(",")
        workloads = [w for w in workloads if w[0] in wanted]
    rng = np.random.default_rng(7)
    ix = KnnIndex(d, metric="cosine")
    ix.set_path("shadow")

    def restore():
        ix.fill_uniform(n, CORPUS_SEED)

    restore()
    base_i, base_s = ix.search_rows(np.arange(n), K)
    lines = []
    for name, n_new, n_rewrite, n_remove in workloads:
        new = rng.uniform(-1, 1, (n_new, d)).astype(np.float32)
        rewrite = rng.choice(n, n_rewrite, replace=False) if n_rewrite else np.empty(0, np.int64)
        vecs = rng.uniform(-1, 1, (n_rewrite, d)).astype(np.float32)
        ops = []  # removal workloads: (op, row, vector) in random order, rows drawn against the row count at that point
        if n_remove:
            kinds = ["remove"] * n_remove + ["append"] * n_new + ["rewrite"] * n_rewrite
            rng.shuffle(kinds)
            rows_now, a, w = n, 0, 0
            for op in kinds:
                if op == "append":
                    ops.append((op, None, new[a:a + 1])); a += 1; rows_now += 1
                elif op == "rewrite":
                    ops.append((op, int(rng.integers(rows_now)), vecs[w])); w += 1
                else:
                    ops.append((op, int(rng.integers(rows_now)), None)); rows_now -= 1
        t_up, t_rb, scan_up, scan_rb, changed_lists = [], [], [], [], []
        c0 = ix.debug_counters()
        for _ in range(args.steps):
            restore()
            m = GraphRowMap(n)
            if n_remove:
                for op, r, v in ops:
                    if op == "append":
                        ix.append(v); m.append(1)
                    elif op == "rewrite":
                        ix.update_row(r, v); m.update_row(r)
                    else:
                        ix.remove_swap(r); m.remove_swap(r)
            else:
                if n_new:
                    ix.append(new)
                for r, v in zip(rewrite, vecs):
                    ix.update_row(int(r), v)
            ix.enable_timing(True)
            ix.scan_time_ms()
            t0 = time.perf_counter()
            if n_remove:
                ui, us, nch = ix.remap_knn_graph(base_i, base_s, n, m)
            else:
                ui, us, nch = ix.update_knn_graph(base_i, base_s, n, rewrite)
            t_up.append(time.perf_counter() - t0)
            scan_up.append(ix.scan_time_ms()[0])
            t0 = time.perf_counter()
            ri, rs = ix.search_rows(np.arange(len(ix)), K)
            t_rb.append(time.perf_counter() - t0)
            scan_rb.append(ix.scan_time_ms()[0])
            ix.enable_timing(False)
            identical = bool(np.array_equal(ui, ri) and np.array_equal(us.view(np.uint32), rs.view(np.uint32)))
            assert identical, f"{name}: the updated graph differs from the rebuild"
            changed_lists.append(nch)
        c1 = ix.debug_counters()
        rec = {
            "bench": "knn_graph_update", "workload": name, "call": "nk_knn_graph_remap" if n_remove else "nk_knn_graph_update",
            "rows_before": n, "appended": n_new, "rewritten": n_rewrite, "removed": n_remove, "dim": d,
            "k": K, "metric": "cosine", "dtype": "f32", "path": "shadow",
            "update_s_median": round(median(t_up), 4), "update_s": [round(v, 4) for v in t_up],
            "update_scan_ms_median": round(median(scan_up), 2),
            "rebuild_s_median": round(median(t_rb), 4), "rebuild_s": [round(v, 4) for v in t_rb],
            "rebuild_scan_ms_median": round(median(scan_rb), 2),
            "rebuild_over_update": round(median(t_rb) / median(t_up), 1),
            "old_lists_changed": changed_lists[-1],
            "retry_counters": {c: c1[c] - c0[c] for c in ("bf16_stage_retries", "exact_stage_runs")},
            "bit_identical_to_rebuild": True, "steps": args.steps,
            "timing": "median wall clock per synchronous call, update and rebuild alternating on a restored base index; scan ms: "
                      "CUDA events around the scan kernels, summed over the call",
            "gpu": gpu_record(),
        }
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    ix.release()
    if args.out:
        with open(args.out, "a") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
