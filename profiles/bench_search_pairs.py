"""Similarity self-join (nk_search_pairs) of a whole index, against the baseline it replaces: the rows read back and sent
through nk_search_range as host queries in blocks of 1024, with the lower-triangle entries (row <= query row) dropped on the
host.  Prints one JSON line per workload and appends them to --out (default: nothing written).

    python profiles/bench_search_pairs.py --out profiles/search_pairs_h100.jsonl

Workloads (fp32, cosine, d=1024; corpora from the device generators with seed 42, as in bench.py):
  pairs_1m_p1 / _p10 / _p100  N=1M uniform rows, whole index, thresholds giving ~1, ~10 and ~100 pairs per row: the median,
                              over the first 1024 rows, of the score of their 2nd, 20th and 200th nearest other row
                              (nk_search_rows, the k-NN graph's scores)
  pairs_1m_clustered_p10      N=1M clustered rows (1000 centres, sigma 0.1), the 20th-neighbour threshold: near-ties
Timing: host wall clock around each synchronous call; the two arms alternate, --steps times each after one warm-up call
each, medians and every sample reported.  scan ms = CUDA events around the scan kernels (nk_index_scan_time_ms), summed
over the call.  The baseline reads the rows back once, untimed; its per-block host work (dropping the lower triangle) is
inside its timed region.  The two arms' results are compared bit for bit.  Retry counters: the filter's 16-bit stage retries
and exact-stage runs (nk_index_debug_counters) over the timed and warm-up calls.  The card's name and power limit are read
in the same run."""
from __future__ import annotations

import argparse
import ctypes as C
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


class RangeBaseline:
    """nk_search_range over the stored rows in blocks of BLOCK, lower triangle dropped on the host -> CSR like search_pairs."""

    def __init__(self, ix, n):
        import numpy as np
        self.ix, self.n = ix, n
        self.x = ix.read_rows(0, n)
        self.cap = 0
        self.idx = np.empty(1, np.uint32)
        self.sc = np.empty(1, np.float32)

    def __call__(self, t):
        import numpy as np
        ix, lib = self.ix, self.ix.lib
        thr = np.full(BLOCK, t, np.float32)
        off = np.zeros(BLOCK + 1, np.uint64)
        total = C.c_uint64(0)
        counts, idx, sc = [], [], []
        for b in range(0, self.n, BLOCK):
            nb = min(BLOCK, self.n - b)
            q = self.x[b:b + nb]
            while True:
                if lib.nk_search_range(ix.ptr, q.ctypes.data_as(C.c_void_p), thr.ctypes.data_as(C.c_void_p), None, nb, self.cap,
                                       off.ctypes.data_as(C.c_void_p), self.idx.ctypes.data_as(C.c_void_p),
                                       self.sc.ctypes.data_as(C.c_void_p), C.byref(total)) < 0:
                    raise RuntimeError(f"nk_search_range: {lib.nk_last_error()}")
                if total.value <= self.cap:
                    break
                self.cap = int(total.value)
                self.idx = np.empty(self.cap, np.uint32)
                self.sc = np.empty(self.cap, np.float32)
            m = int(total.value)
            per = np.diff(off[:nb + 1].astype(np.int64))
            row = np.repeat(np.arange(b, b + nb, dtype=np.int64), per)
            keep = self.idx[:m].astype(np.int64) > row
            idx.append(self.idx[:m][keep])
            sc.append(self.sc[:m][keep])
            counts.append(np.bincount(row[keep] - b, minlength=nb))
        offsets = np.zeros(self.n + 1, np.uint64)
        offsets[1:] = np.cumsum(np.concatenate(counts))
        return offsets, np.concatenate(idx), np.concatenate(sc)


def run_workload(ix, name, corpus, n, d, per_row, steps):
    import numpy as np
    _, s = ix.search_rows(np.arange(BLOCK), 2 * per_row)  # the k-NN graph's scores of the first block
    t = np.float32(np.median(s[:, 2 * per_row - 1]))
    base = RangeBaseline(ix, n)
    c0 = ix.debug_counters()
    ix.search_pairs(t)  # warm-up (and the wrapper's buffer sized)
    base(t)
    ix.enable_timing(True)
    ix.scan_time_ms()
    t_pairs, t_base, scan_pairs, scan_base = [], [], [], []
    for _ in range(steps):
        t0 = time.perf_counter()
        res = ix.search_pairs(t)
        t_pairs.append(time.perf_counter() - t0)
        scan_pairs.append(ix.scan_time_ms()[0])
        path_pairs = ix.last_path()
        t0 = time.perf_counter()
        ref = base(t)
        t_base.append(time.perf_counter() - t0)
        scan_base.append(ix.scan_time_ms()[0])
        path_base = ix.last_path()
    ix.enable_timing(False)
    c1 = ix.debug_counters()
    identical = bool(np.array_equal(res[0], ref[0]) and np.array_equal(res[1], ref[1])
                     and np.array_equal(res[2].view(np.uint32), ref[2].view(np.uint32)))
    assert identical, f"{name}: nk_search_pairs differs from nk_search_range with the lower triangle dropped"
    tp, tb = median(t_pairs), median(t_base)
    total = int(res[0][-1])
    return {
        "bench": "search_pairs", "workload": name, "corpus": corpus, "rows": n, "dim": d, "metric": "cosine", "dtype": "f32",
        "threshold": float(t), "threshold_from": f"median score of the {2 * per_row}th other row, first {BLOCK} rows",
        "pairs": total, "pairs_per_row": round(total / n, 2),
        "search_pairs_s_median": round(tp, 4), "search_pairs_s": [round(v, 4) for v in t_pairs],
        "search_pairs_scan_ms_median": round(median(scan_pairs), 2),
        "range_blocks_s_median": round(tb, 4), "range_blocks_s": [round(v, 4) for v in t_base],
        "range_blocks_scan_ms_median": round(median(scan_base), 2),
        "wall_speedup": round(tb / tp, 3), "scan_speedup": round(median(scan_base) / max(median(scan_pairs), 1e-9), 3),
        "search_pairs_pairs_per_s": round(total / tp, 1),
        "retry_counters_over_timed_and_warmup_calls": {"bf16_stage_retries": c1["bf16_stage_retries"] - c0["bf16_stage_retries"],
                                                       "exact_stage_runs": c1["exact_stage_runs"] - c0["exact_stage_runs"]},
        "bit_identical_to_range_blocks": identical, "path_search_pairs": path_pairs, "path_range_blocks": path_base,
        "steps": steps,
        "timing": "median wall clock per synchronous call, the two arms alternating; scan ms: CUDA events around the scan "
                  "kernels, summed over the call; the baseline's row read-back is untimed",
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default="")
    ap.add_argument("--only", default="", help="comma-separated workload names (default: all four)")
    ap.add_argument("--scale", type=float, default=1.0, help="multiply N (a small value rehearses the script)")
    args = ap.parse_args()
    from nornicdb_b200.knn import KnnIndex

    d, n = 1024, int(1_000_000 * args.scale)
    work = [("pairs_1m_p1", "uniform", 1), ("pairs_1m_p10", "uniform", 10), ("pairs_1m_p100", "uniform", 100),
            ("pairs_1m_clustered_p10", "clustered 1000 centres sigma 0.1", 10)]
    only = set(filter(None, args.only.split(",")))
    records = []
    ix, built = None, None
    for name, corpus, per_row in work:
        if only and name not in only:
            continue
        if built != corpus:
            if ix is not None:
                ix.release()
            ix = KnnIndex(d, metric="cosine")
            if corpus == "uniform":
                ix.fill_uniform(n, CORPUS_SEED)
            else:
                ix.fill_clustered(n, CORPUS_SEED, n_centres=1000, sigma=0.1)
            built = corpus
        rec = run_workload(ix, name, corpus, n, d, per_row, args.steps)
        print(json.dumps(rec), flush=True)
        records.append(rec)
    if ix is not None:
        ix.release()
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
