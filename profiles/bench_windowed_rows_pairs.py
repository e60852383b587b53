"""Value windows for search by stored row and for the self-join, at the headline row shape: a windowed search_rows batch against
the same batch unwindowed, and a band self-join against the unwindowed join at one threshold.  Prints one JSON line per entry
and, with --out, writes them to a JSONL file.

    python profiles/bench_windowed_rows_pairs.py --out profiles/windowed_rows_pairs_h100.jsonl

Corpus: the counter-based generator of bench.py (seed 42), N=1M d=1024 fp32 cosine, generated on the device, on the 16-bit
shadow path.  Row values: row order as timestamps spread evenly over one year (int64 seconds, knn.value_keys), so the window
of row r is its own +-1 day (knn.band_windows), about 0.55 % of the rows.  search_rows: Q query rows spread evenly over the
index, k = 10.  Pairs: a stripe of STRIPE left rows from the middle of the index, band = 1 day; the threshold is chosen so the
unwindowed stripe joins a few pairs per row.  Timing: host wall clock around each synchronous call, medians over --steps after
--warmup, all unwindowed calls first, then the windowed ones.  Each entry records the retry counters (16-bit stage retries,
exact-stage runs) over its timed calls.  Parity (untimed, every run): the windowed search_rows equals search_windowed of the
rows read back with the self rule; the band join equals the unwindowed join with out-of-band pairs dropped, bit for bit."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CORPUS_SEED = 42
DAY = 86_400
YEAR = 365 * DAY


def gpu_record():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout.strip()
        name, plim, sm, smax = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock_after_timing": sm, "sm_clock_max": smax}
    except Exception as e:  # the record says so instead of guessing
        return {"error": f"nvidia-smi: {e}"}


def timed(ix, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    c0 = ix.debug_counters()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        out = fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    c1 = ix.debug_counters()
    retries = {key: c1[key] - c0[key] for key in ("bf16_stage_retries", "exact_stage_runs")}
    return out, statistics.median(ts), retries


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--q", type=int, default=4096)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--stripe", type=int, default=4096)
    ap.add_argument("--threshold", type=float, default=0.115)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None, help="write the JSON lines to this file")
    args = ap.parse_args()
    import numpy as np
    from nornicdb_b200.knn import KnnIndex, band_windows, value_keys

    n, d, Q, k = args.rows, args.dim, args.q, args.k
    ix = KnnIndex(d, metric="cosine", dtype="f32")
    ix.fill_uniform(n, CORPUS_SEED)
    ix.set_path("shadow")
    keys = value_keys((np.arange(n, dtype=np.int64) * YEAR) // n)
    ix.set_row_values(keys)
    ids = np.linspace(0, n - 1, Q).astype(np.int64)
    w = band_windows(keys[ids], DAY)
    config = {"N": n, "dim": d, "corpus_dtype": "f32", "metric": "cosine", "path": "shadow", "steps": args.steps,
              "warmup": args.warmup}
    lines = []

    def emit(entry):
        entry["config"] = config
        entry["gpu"] = gpu_record()
        print(json.dumps(entry), flush=True)
        lines.append(entry)

    plain = lambda: ix.search_rows(ids, k)
    windowed = lambda: ix.search_rows(ids, k, windows=w)
    (pi, _), t_plain, r_plain = timed(ix, plain, args.steps, args.warmup)
    (wi, ws), t_win, r_win = timed(ix, windowed, args.steps, args.warmup)
    x = np.stack([ix.read_rows(int(r), 1)[0] for r in ids])  # parity: search_windowed of the stored rows, k + 1, self rule
    for b in range(0, Q, 1024):
        bid = ids[b:b + 1024]
        ri, rs = ix.search_windowed(x[b:b + 1024], k + 1, w[b:b + 1024])
        for q, self_row in enumerate(bid):
            li, ls = list(ri[q]), list(rs[q])
            drop = li.index(self_row) if self_row in li else len(li) - 1
            del li[drop], ls[drop]
            assert li == list(wi[b + q]) and np.array_equal(np.float32(ls).view(np.uint32), ws[b + q].view(np.uint32)), (b + q,)
    emit({"entry": "search_rows", "what": f"search_rows of {Q} rows, k={k}", "ms": round(t_plain, 3), "retries": r_plain})
    emit({"entry": "search_rows_windowed", "what": "the same rows, each windowed to its own +-1 day (band_windows)",
          "ms": round(t_win, 3), "ratio_vs_unwindowed": round(t_win / t_plain, 3), "retries": r_win, "bit_equal_to_contract": True})

    first = n // 2
    pairs = lambda: ix.search_pairs(args.threshold, first, args.stripe)
    band = lambda: ix.search_pairs(args.threshold, first, args.stripe, max_gap=DAY)
    base, t_pairs, r_pairs = timed(ix, pairs, args.steps, args.warmup)
    got, t_band, r_band = timed(ix, band, args.steps, args.warmup)
    off, idx, sc = base
    left = first + np.repeat(np.arange(args.stripe), np.diff(off.astype(np.int64)))
    ki, kj = keys[left], keys[idx.astype(np.int64)]
    keep = np.where(ki > kj, ki - kj, kj - ki) <= np.uint64(DAY)
    kept = np.concatenate([[0], np.cumsum(keep)]).astype(np.uint64)
    assert np.array_equal(got[0], kept[off.astype(np.int64)]) and np.array_equal(got[1], idx[keep])
    assert np.array_equal(got[2].view(np.uint32), sc[keep].view(np.uint32))
    emit({"entry": "pairs", "what": f"search_pairs, stripe of {args.stripe} rows at row {first}, threshold {args.threshold}",
          "ms": round(t_pairs, 3), "pairs": int(idx.size), "retries": r_pairs})
    emit({"entry": "pairs_band", "what": "the same stripe with max_gap = 1 day", "ms": round(t_band, 3), "pairs": int(got[1].size),
          "ratio_vs_unwindowed": round(t_band / t_pairs, 3), "retries": r_band, "bit_equal_to_contract": True})
    ix.release()
    if args.out:
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
