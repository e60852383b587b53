"""Per-query value windows at the headline shape: one windowed batch against the same batch unfiltered, against tag filters
of about the same selectivity, and against the per-query masked searches it replaces.  Prints one JSON line per entry and,
with --out, appends them to a JSONL file.

    python profiles/bench_value_windows.py --q 64 --steps 20 --warmup 3 --out profiles/value_windows_h100.jsonl

Corpus: the counter-based generator of bench.py (seed 42), N=10M d=1024 fp32, generated on the device.  Row values:
timestamps spread uniformly over one year (int64 nanoseconds, knn.value_keys).  Windows: query q asks for the last
WINDOW_FRACTIONS[q % 4] of the year, i.e. about 100 %, 10 %, 1 % and 0.1 % of the rows.  Tag filters: query q gets an all_of of
TAG_BITS[q % 4] random bits of knn.synthetic_tags (about 100 %, 12.5 %, 0.8 %, 0.1 %).  Timing: one CUDA event pair per
search on an explicit stream, the unfiltered, windowed and tag-filtered batches alternating on the same queries, medians
reported; scan_ms = the event-timed scan kernels only.  Each entry records the index's retry counters (16-bit stage retries
and exact-stage runs) over its timed searches.  Parity (untimed): every returned row inside its query's window, every
returned score recomputed in fp64 from the rows read back."""
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

CORPUS_SEED, QUERY_SEED, VALUE_SEED, TAG_SEED, FILTER_SEED = 42, 1337, 91, 77, 78
WINDOW_FRACTIONS = (1.0, 0.1, 0.01, 0.001)
TAG_BITS = (0, 3, 7, 10)
YEAR_NS = 365 * 86400 * 10 ** 9


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
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--q", type=int, default=64)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--metric", default="cosine", choices=["cosine", "dot", "euclidean"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-masked", action="store_true", help="skip the per-query masked searches (Q <= 64 only anyway)")
    ap.add_argument("--out", default=None, help="append the JSON lines to this file")
    args = ap.parse_args()
    import numpy as np
    import torch
    from nornicdb_b200.knn import KnnIndex, admits, fill_uniform_device, synthetic_tags, value_keys, window_admits

    n, d, Q, k, metric = args.rows, args.dim, args.q, args.k, args.metric
    st = torch.cuda.Stream()
    torch.cuda.set_stream(st)
    stream = st.cuda_stream
    ix = KnnIndex(d, metric=metric)
    ix.fill_uniform(n, CORPUS_SEED)
    t_end = np.int64(1_767_225_600 * 10 ** 9)  # 2026-01-01T00:00:00 in ns
    ts = t_end - np.random.default_rng(VALUE_SEED).integers(0, YEAR_NS, n, dtype=np.int64)
    keys = value_keys(ts)
    ix.set_row_values(keys)
    tags = synthetic_tags(n, TAG_SEED)
    ix.set_row_tags(tags)
    windows = np.zeros((Q, 2), dtype=np.uint64)
    for q in range(Q):
        lo = t_end - np.int64(WINDOW_FRACTIONS[q % 4] * YEAR_NS)
        windows[q] = (int(value_keys(np.int64(lo))), int(value_keys(t_end)))
    rng = np.random.default_rng(FILTER_SEED)
    filters = np.zeros((Q, 3), dtype=np.uint64)
    for q in range(Q):
        for b in rng.choice(64, size=TAG_BITS[q % 4], replace=False):
            filters[q, 0] |= np.uint64(1) << np.uint64(int(b))
    w_dev = torch.from_numpy(windows.view(np.int64)).cuda()
    f_dev = torch.from_numpy(filters.view(np.int64)).cuda()
    n_all = args.warmup + args.steps
    q_all = torch.empty((n_all, Q, d), dtype=torch.float32, device="cuda")
    fill_uniform_device(0, q_all.data_ptr(), n_all * Q, d, QUERY_SEED, 0, stream)
    out = {name: (torch.empty((Q, k), dtype=torch.int32, device="cuda"), torch.empty((Q, k), dtype=torch.float32, device="cuda"))
           for name in ("unfiltered", "windows", "tags")}

    def run(name, i):
        oi, os_ = out[name]
        if name == "unfiltered":
            ix.search_device(q_all[i].data_ptr(), Q, k, oi.data_ptr(), os_.data_ptr(), stream)
        elif name == "windows":
            ix.search_windowed_device(q_all[i].data_ptr(), 0, w_dev.data_ptr(), Q, k, oi.data_ptr(), os_.data_ptr(), stream)
        else:
            ix.search_filtered_device(q_all[i].data_ptr(), f_dev.data_ptr(), Q, k, oi.data_ptr(), os_.data_ptr(), stream)

    def timed(name, i):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        run(name, i)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    names = ("unfiltered", "windows", "tags")
    for i in range(args.warmup):
        for name in names:
            run(name, i)
    ix.status(stream)
    ix.enable_timing(True)
    ix.scan_time_ms()
    t = {name: [] for name in names}
    scan = {name: [] for name in names}
    retries = {name: [0, 0] for name in names}
    for s in range(args.steps):
        for name in names:
            c0 = ix.debug_counters()
            t[name].append(timed(name, args.warmup + s))
            scan[name].append(ix.scan_time_ms()[0])
            ix.status(stream)
            c1 = ix.debug_counters()
            retries[name][0] += c1["bf16_stage_retries"] - c0["bf16_stage_retries"]
            retries[name][1] += c1["exact_stage_runs"] - c0["exact_stage_runs"]
    ix.enable_timing(False)
    gpu = gpu_record()
    path = ix.last_path()
    qs = q_all[n_all - 1].cpu().numpy()

    # ---- parity of the last windowed step
    gi = out["windows"][0].cpu().numpy().view(np.uint32).copy()
    gs = out["windows"][1].cpu().numpy()
    outside = bad_score = 0
    for q in range(Q):
        live = gi[q] != 0xFFFFFFFF
        outside += int((~window_admits(keys[gi[q][live].astype(np.int64)], *[int(v) for v in windows[q]])).sum())
        x = np.stack([ix.read_rows(int(r), 1)[0] for r in gi[q][live]]).astype(np.float64)
        qq = qs[q].astype(np.float64)
        ex = x @ qq
        if metric == "cosine":
            ex = ex / np.maximum(np.linalg.norm(x, axis=1) * np.linalg.norm(qq), 1e-300)
        elif metric == "euclidean":
            ex = np.sqrt(((x - qq) ** 2).sum(1))
        bad_score += int((np.abs(gs[q][live] - ex) > 1e-4 * np.abs(ex) + 1e-6).sum())

    sample = slice(0, 2_000_000)
    win_sel = {str(WINDOW_FRACTIONS[j]): float(window_admits(keys[sample], *[int(v) for v in windows[j]]).mean()) for j in range(min(4, Q))}
    tag_sel = {str(TAG_BITS[j]): float(admits(tags[sample], int(filters[j, 0]), 0, 0).mean()) for j in range(min(4, Q))}
    config = {"N": n, "dim": d, "corpus_dtype": "f32", "Q": Q, "k": k, "metric": metric, "path": path,
              "value_bytes": n * 8, "corpus_bytes": n * d * 4, "steps": args.steps, "warmup": args.warmup}
    timing = ("median of one CUDA event pair per search (explicit stream, synchronised on both sides); unfiltered, windowed and "
              "tag-filtered batches alternate on the same queries; scan_ms = event-timed scan kernels only")

    def entry(name, what, extra):
        ms = float(np.median(t[name]))
        return {"entry": name, "what": what, "config": config, "gpu": gpu, "ms": ms, "value": Q / (ms / 1e3), "unit": "queries/s",
                "scan_ms": float(np.median(scan[name])), "spread_ms": [min(t[name]), max(t[name])],
                "retries": {"bf16_stage_retries": retries[name][0], "exact_stage_runs": retries[name][1]}, "timing": timing, **extra}

    um = float(np.median(t["unfiltered"]))
    lines = [entry("unfiltered", "nk_search_device, no filter", {}),
             entry("windows", "nk_search_windowed_device: query q keeps the last %s of the year's timestamps (cycling)"
                   % (list(WINDOW_FRACTIONS),), {"selectivity": win_sel, "ratio_over_unfiltered": float(np.median(t["windows"])) / um,
                                                  "parity": {"rows_outside_window": outside, "scores_off_fp64": bad_score}}),
             entry("tags", "nk_search_filtered_device: query q an all_of of %s random tag bits (cycling)" % (list(TAG_BITS),),
                   {"selectivity": tag_sel, "ratio_over_unfiltered": float(np.median(t["tags"])) / um})]
    if Q <= 64 and not args.no_masked:
        # what the batch replaces: one masked search per query, the row mask built and set on the host in between
        t0 = time.perf_counter()
        mask_s = 0.0
        for q in range(Q):
            m0 = time.perf_counter()
            ix.set_row_mask(window_admits(keys, *[int(v) for v in windows[q]]))
            mask_s += time.perf_counter() - m0
            ix.search(qs[q:q + 1], k)
        total = (time.perf_counter() - t0) * 1e3
        ix.set_row_mask(None)
        lines.append({"entry": "masked_searches", "what": "Q x (host mask build + nk_index_set_row_mask + nk_search of 1 query)",
                      "config": config, "gpu": gpu, "ms": total, "mask_ms": mask_s * 1e3, "search_ms": total - mask_s * 1e3,
                      "speedup_of_one_windowed_batch": total / float(np.median(t["windows"])), "timing": "wall clock"})
    ix.release()
    for line in lines:
        print(json.dumps(line))
    if args.out:
        with open(args.out, "a") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
