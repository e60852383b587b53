"""Self-join kept current: nk_pairs_remap after a change against a whole-index rebuild (nk_search_pairs over every row), and the
incident scan it runs (nk_search_pairs_rows of the new and moved rows) on its own.  Prints one JSON line per workload and
appends them to --out (default: nothing written).

    python profiles/bench_pairs_update.py --out profiles/pairs_update_h100.jsonl

Base: N=1M clustered fp32 rows from the device generator (fill_clustered: 1000 centres, sigma 0.1, seed 42), d=1024, cosine,
the AUTO path (the incident scans run the graph path it resolves to; the rebuild runs with that path forced, so both use one
arithmetic).  Threshold: the median score of the 20th nearest other row of the first 1024 rows, about 10 pairs per row.
Windowed: the same with uniform timestamps (s) over one year and a +-1 day band (max_gap).  Workloads: append 1024 rows,
rewrite 100 rows (both near-copies of stored rows, noise sigma 0.002), remove 100 random rows with nk_index_remove_swap, retag 100 rows (under a tag filter, reported as new
contents).  Each repetition restores the base index and its join, makes the change, runs the remap, the incident scan of the
same rows and the rebuild, and asserts that remap and rebuild are bit-identical.  Timing: host wall clock around each
synchronous call; scan ms = CUDA events around the scan kernels (nk_index_scan_time_ms); host merge = remap - incident scan
call.  Medians of --steps repetitions.  The card's name and power limit are read in the same run."""
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
DAY = 86_400
T0 = 1_700_000_000
YEAR = 365 * DAY


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--out", default="")
    ap.add_argument("--scale", type=float, default=1.0, help="multiply N and the change sizes (a small value rehearses the script)")
    args = ap.parse_args()
    import numpy as np
    from nornicdb_b200.knn import GraphRowMap, KnnIndex
    n, d = max(int(1_000_000 * args.scale), 4096), 1024
    rng = np.random.default_rng(13)
    keys0 = (T0 + rng.integers(0, YEAR, n)).astype(np.uint64)
    tags0 = rng.integers(0, 4, n).astype(np.uint64)

    ix = KnnIndex(d, metric="cosine")

    def restore():
        ix.fill_clustered(n, CORPUS_SEED, 1000, 0.1)
        ix.set_row_values(keys0)
        ix.set_row_tags(tags0)

    restore()
    ix.set_path("auto")
    _, s20 = ix.search_rows(np.arange(1024), 20)
    t = float(np.median(s20[:, 19]))
    ix.search_pairs_rows([0], t)
    graph_path = ix.last_path()  # the path the incident call resolved AUTO to
    lines = []

    def emit(rec):
        rec.update({"rows_before": n, "dim": d, "metric": "cosine", "dtype": "f32", "corpus": "fill_clustered(1000, 0.1)",
                    "threshold": t, "path": graph_path, "steps": args.steps, "gpu": gpu_record()})
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    n_app = max(int(1024 * args.scale), 2)
    n_chg = max(int(100 * args.scale), 2)
    # appended and rewritten rows: near-copies of stored rows, so they form pairs
    src_rows = ix.read_rows(int(rng.integers(0, n - n_app - n_chg)), n_app + n_chg)
    new = (src_rows[:n_app] + rng.normal(0, 0.002, (n_app, d))).astype(np.float32)
    new_keys = (T0 + rng.integers(0, YEAR, n_app)).astype(np.uint64)
    rewrite = rng.choice(n, n_chg, replace=False)
    vecs = (src_rows[n_app:] + rng.normal(0, 0.002, (n_chg, d))).astype(np.float32)
    retag = rng.choice(n, n_chg, replace=False)
    removes = [int(rng.integers(n - i)) for i in range(n_chg)]
    flt = (0, 2, 0)  # rows tagged 2 or 3 are refused: a retag can add and remove pairs
    for windowed in (False, True):
        kw = {"filter": flt}
        if windowed:
            kw["max_gap"] = DAY
        restore()
        ix.set_path(graph_path)
        ix.enable_timing(True)
        ix.scan_time_ms()
        t0 = time.perf_counter()
        base = ix.search_pairs(t, **kw)
        t_build = time.perf_counter() - t0
        s_build = ix.scan_time_ms()[0]
        ix.enable_timing(False)
        emit({"bench": "pairs_update", "workload": "build", "windowed": windowed, "kw": str(kw),
              "pairs": int(base[0][-1]), "pairs_per_row": round(int(base[0][-1]) / n, 2),
              "build_s": round(t_build, 3), "build_scan_ms": round(s_build, 1)})
        for name in ("append_1024", "rewrite_100", "remove_100", "retag_100"):
            t_rm, t_inc, s_inc, t_rb, s_rb, info = [], [], [], [], [], {}
            c0 = ix.debug_counters()
            for _ in range(args.steps):
                restore()
                tags = tags0.copy()
                m = GraphRowMap(n)
                if name == "append_1024":
                    ix.append(new)
                    ix.set_row_values(new_keys, first_row=n)
                    m.append(n_app)
                elif name == "rewrite_100":
                    for r, v in zip(rewrite, vecs):
                        ix.update_row(int(r), v)
                        m.update_row(int(r))
                elif name == "remove_100":
                    for r in removes:
                        ix.remove_swap(r)
                        m.remove_swap(r)
                else:
                    tags[retag] = (tags[retag] + 2) % 4
                    ix.set_row_tags(tags)
                    for r in retag:
                        m.update_row(int(r))
                src = m.src_of_row
                changed = np.flatnonzero(src != np.arange(len(src)))
                ix.set_path("auto")
                t0 = time.perf_counter()
                off, idx, sc, dropped, found = ix.remap_pairs(base, n, m, t, **kw)
                t_rm.append(time.perf_counter() - t0)
                ix.enable_timing(True)
                ix.scan_time_ms()
                t0 = time.perf_counter()
                inc = ix.search_pairs_rows(changed, t, **kw)
                t_inc.append(time.perf_counter() - t0)
                s_inc.append(ix.scan_time_ms()[0])
                ix.set_path(graph_path)
                t0 = time.perf_counter()
                fresh = ix.search_pairs(t, **kw)
                t_rb.append(time.perf_counter() - t0)
                s_rb.append(ix.scan_time_ms()[0])
                ix.enable_timing(False)
                same = (np.array_equal(off, fresh[0]) and np.array_equal(idx, fresh[1])
                        and np.array_equal(sc.view(np.uint32), fresh[2].view(np.uint32)))
                assert same, f"{name}: the remapped join differs from the rebuild"
                assert found == int(inc[0][-1])
                info = {"changed_rows": int(changed.size), "pairs_dropped": dropped, "pairs_found": found}
            c1 = ix.debug_counters()
            emit({"bench": "pairs_update", "workload": name, "windowed": windowed, "kw": str(kw), **info,
                  "remap_s_median": round(median(t_rm), 4), "remap_s": [round(v, 4) for v in t_rm],
                  "incident_s_median": round(median(t_inc), 4), "incident_scan_ms_median": round(median(s_inc), 2),
                  "host_merge_s_median": round(median(t_rm) - median(t_inc), 4),
                  "rebuild_s_median": round(median(t_rb), 3), "rebuild_scan_ms_median": round(median(s_rb), 1),
                  "rebuild_over_remap": round(median(t_rb) / median(t_rm), 1),
                  "retry_counters": {c: c1[c] - c0[c] for c in ("bf16_stage_retries", "exact_stage_runs")},
                  "bit_identical_to_rebuild": True,
                  "timing": "median wall clock per synchronous call on a restored base index; the remap's host merge is its "
                            "time minus the incident call's; scan ms: CUDA events around the scan kernels"})
    ix.release()
    if args.out:
        with open(args.out, "a") as fo:
            for rec in lines:
                fo.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
