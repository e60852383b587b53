"""Filtered k-NN graph ("same collection" lists of one shared index): the full filtered build (nk_search_rows_filtered over
every row) against the unfiltered build, and nk_knn_graph_update_filtered / nk_knn_graph_remap_filtered against a filtered
rebuild.  Prints one JSON line per workload and appends them to --out (default: nothing written).

    python profiles/bench_filtered_graph.py --out profiles/filtered_graph_h100.jsonl

Base: N=1M uniform fp32 rows from the device generator (seed 42, as in bench.py), d=1024, cosine, k=10, the 16-bit (shadow)
path forced.  16 collections of Zipf sizes (s = 1.1): row r's tag is its collection bit and its filter admits that bit only.
Workloads: append 1024 uniform rows (random collections), rewrite 100 rows, retag 100 rows (each moves to another
collection: new tag and new filter, reported as rewritten), remove 100 random rows with nk_index_remove_swap (the remap,
the row map kept by GraphRowMap, the filters following the swaps).  The changes are drawn once and replayed every
repetition.  Each repetition restores the base index and its tags, makes the change, runs the update on the base graph, then
the filtered rebuild, and asserts that both are bit-identical.  Timing: host wall clock around each synchronous call; scan ms
= CUDA events around the scan kernels (nk_index_scan_time_ms), summed over the call.  Medians of --steps repetitions, every
sample reported.  The card's name and power limit are read in the same run."""
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
N_COLL = 16


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--out", default="")
    ap.add_argument("--scale", type=float, default=1.0, help="multiply N and the change sizes (a small value rehearses the script)")
    ap.add_argument("--workloads", default="", help="comma-separated names to run (default: all)")
    args = ap.parse_args()
    import numpy as np
    from nornicdb_b200.knn import GraphRowMap, KnnIndex
    n, d = max(int(1_000_000 * args.scale), 4096), 1024
    rng = np.random.default_rng(11)
    w = 1.0 / np.arange(1, N_COLL + 1) ** 1.1
    coll0 = rng.choice(N_COLL, n, p=w / w.sum())
    sizes = np.bincount(coll0, minlength=N_COLL).tolist()

    def tags_of(c):
        return (np.uint64(1) << np.asarray(c).astype(np.uint64)).astype(np.uint64)

    def filters_of(c):
        f = np.zeros((len(c), 3), np.uint64)
        f[:, 2] = tags_of(c)
        return f

    ix = KnnIndex(d, metric="cosine")
    ix.set_path("shadow")

    def restore():
        ix.fill_uniform(n, CORPUS_SEED)
        ix.set_row_tags(tags_of(coll0))

    lines = []

    def emit(rec):
        rec.update({"rows_before": n, "dim": d, "k": K, "metric": "cosine", "dtype": "f32", "path": "shadow",
                    "collections": N_COLL, "collection_sizes": sizes, "steps": args.steps, "gpu": gpu_record()})
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    restore()
    f0 = filters_of(coll0)
    ix.enable_timing(True)
    ix.scan_time_ms()
    t_f, t_u, s_f, s_u = [], [], [], []
    for _ in range(args.steps):  # the full builds, filtered and unfiltered, alternating
        t0 = time.perf_counter()
        base_i, base_s = ix.search_rows(np.arange(n), K, filters=f0)
        t_f.append(time.perf_counter() - t0)
        s_f.append(ix.scan_time_ms()[0])
        t0 = time.perf_counter()
        ix.search_rows(np.arange(n), K)
        t_u.append(time.perf_counter() - t0)
        s_u.append(ix.scan_time_ms()[0])
    ix.enable_timing(False)
    emit({"bench": "filtered_graph", "workload": "build", "call": "nk_search_rows_filtered vs nk_search_rows (every row)",
          "filtered_build_s_median": round(median(t_f), 3), "filtered_build_s": [round(v, 3) for v in t_f],
          "filtered_build_scan_ms_median": round(median(s_f), 1),
          "unfiltered_build_s_median": round(median(t_u), 3), "unfiltered_build_s": [round(v, 3) for v in t_u],
          "unfiltered_build_scan_ms_median": round(median(s_u), 1),
          "filtered_over_unfiltered": round(median(t_f) / median(t_u), 3),
          "short_lists": int((base_i[:, K - 1] == 0xFFFFFFFF).sum()),
          "timing": "median wall clock per synchronous call, filtered and unfiltered alternating; scan ms: CUDA events around "
                    "the scan kernels, summed over the call"})

    workloads = [("append_1024", max(int(1024 * args.scale), 2), 0, 0, 0), ("rewrite_100", 0, 100, 0, 0),
                 ("retag_100", 0, 0, 100, 0), ("remove_100", 0, 0, 0, 100)]
    if args.workloads:
        wanted = args.workloads.split(",")
        workloads = [wl for wl in workloads if wl[0] in wanted]
    for name, n_new, n_rewrite, n_retag, n_remove in workloads:
        new = rng.uniform(-1, 1, (n_new, d)).astype(np.float32)
        new_coll = rng.choice(N_COLL, n_new, p=w / w.sum())
        rewrite = rng.choice(n, n_rewrite, replace=False)
        vecs = rng.uniform(-1, 1, (n_rewrite, d)).astype(np.float32)
        retag = rng.choice(n, n_retag, replace=False)
        retag_to = (coll0[retag] + rng.integers(1, N_COLL, n_retag)) % N_COLL
        removes = [int(rng.integers(n - i)) for i in range(n_remove)]
        t_up, t_rb, scan_up, scan_rb, changed_lists = [], [], [], [], []
        c0 = ix.debug_counters()
        for _ in range(args.steps):
            restore()
            coll = coll0.copy()
            m = GraphRowMap(n)
            changed = []
            if n_new:
                ix.append(new)
                ix.set_row_tags(tags_of(new_coll), first_row=n)
                coll = np.concatenate([coll, new_coll])
                m.append(n_new)
            for r, v in zip(rewrite, vecs):
                ix.update_row(int(r), v)
                m.update_row(int(r))
                changed.append(int(r))
            for r, c in zip(retag, retag_to):
                ix.set_row_tags(tags_of([c]), first_row=int(r))
                coll[r] = c
                m.update_row(int(r))
                changed.append(int(r))
            for r in removes:
                ix.remove_swap(r)
                m.remove_swap(r)
                coll[r] = coll[len(coll) - 1]
                coll = coll[:-1]
            f = filters_of(coll)
            ix.enable_timing(True)
            ix.scan_time_ms()
            t0 = time.perf_counter()
            if n_remove:
                ui, us, nch = ix.remap_knn_graph(base_i, base_s, n, m, filters=f)
            else:
                ui, us, nch = ix.update_knn_graph(base_i, base_s, n, changed, filters=f)
            t_up.append(time.perf_counter() - t0)
            scan_up.append(ix.scan_time_ms()[0])
            t0 = time.perf_counter()
            ri, rs = ix.search_rows(np.arange(len(ix)), K, filters=f)
            t_rb.append(time.perf_counter() - t0)
            scan_rb.append(ix.scan_time_ms()[0])
            ix.enable_timing(False)
            identical = bool(np.array_equal(ui, ri) and np.array_equal(us.view(np.uint32), rs.view(np.uint32)))
            assert identical, f"{name}: the updated filtered graph differs from the filtered rebuild"
            changed_lists.append(nch)
        c1 = ix.debug_counters()
        emit({"bench": "filtered_graph", "workload": name,
              "call": "nk_knn_graph_remap_filtered" if n_remove else "nk_knn_graph_update_filtered",
              "appended": n_new, "rewritten": n_rewrite, "retagged": n_retag, "removed": n_remove,
              "update_s_median": round(median(t_up), 4), "update_s": [round(v, 4) for v in t_up],
              "update_scan_ms_median": round(median(scan_up), 2),
              "rebuild_s_median": round(median(t_rb), 4), "rebuild_s": [round(v, 4) for v in t_rb],
              "rebuild_scan_ms_median": round(median(scan_rb), 2),
              "rebuild_over_update": round(median(t_rb) / median(t_up), 1),
              "old_lists_changed": changed_lists[-1],
              "retry_counters": {c: c1[c] - c0[c] for c in ("bf16_stage_retries", "exact_stage_runs")},
              "bit_identical_to_rebuild": True,
              "timing": "median wall clock per synchronous call, update and filtered rebuild alternating on a restored base "
                        "index; scan ms: CUDA events around the scan kernels, summed over the call"})
    ix.release()
    if args.out:
        with open(args.out, "a") as fo:
            for rec in lines:
                fo.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
