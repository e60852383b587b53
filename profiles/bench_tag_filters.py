"""Per-query tag filters at the headline shape: one filtered batch against the same batch unfiltered, and against the
per-filter masked searches it replaces.  Prints one JSON line; writes nothing.

    python profiles/bench_tag_filters.py --q 64 --steps 20 --warmup 3
    python profiles/bench_tag_filters.py --q 1024 --steps 10 --warmup 3

Corpus: the counter-based generator of bench.py (seed 42), N=10M d=1024 fp32, generated on the device.  Tags: every row 64
bits, each set with probability 1/2 (splitmix64 of (seed, row), knn.synthetic_tags).  Filters: query q gets an all_of of
FILTER_BITS[q % 5] random bits, i.e. about 100 %, 50 %, 12.5 %, 0.8 % and 0.1 % of the rows.  Timing: one CUDA event pair
per search on an explicit stream, filtered and unfiltered alternating on the same queries, medians reported.  Parity (untimed):
every returned row admissible, every returned score recomputed in fp64 from the rows read back, planted near-copies that a
query admits come back first and planted ones it rejects never come back."""
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

CORPUS_SEED, QUERY_SEED, TAG_SEED, FILTER_SEED = 42, 1337, 77, 78
FILTER_BITS = (0, 1, 3, 7, 10)


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
    ap.add_argument("--no-masked", action="store_true", help="skip the per-filter masked searches (Q <= 64 only anyway)")
    args = ap.parse_args()
    import numpy as np
    import torch
    from nornicdb_b200.knn import KnnIndex, admits, fill_uniform_device, synthetic_tags

    n, d, Q, k, metric = args.rows, args.dim, args.q, args.k, args.metric
    st = torch.cuda.Stream()
    torch.cuda.set_stream(st)
    stream = st.cuda_stream  # non-zero: the events below sit on the stream the kernels run on
    ix = KnnIndex(d, metric=metric)
    ix.fill_uniform(n, CORPUS_SEED)
    tags = synthetic_tags(n, TAG_SEED)
    ix.set_row_tags(tags)
    rng = np.random.default_rng(FILTER_SEED)
    filters = np.zeros((Q, 3), dtype=np.uint64)
    for q in range(Q):
        for b in rng.choice(64, size=FILTER_BITS[q % len(FILTER_BITS)], replace=False):
            filters[q, 0] |= np.uint64(1) << np.uint64(int(b))
    f_dev = torch.from_numpy(filters.view(np.int64)).cuda()
    n_all = args.warmup + args.steps
    q_all = torch.empty((n_all, Q, d), dtype=torch.float32, device="cuda")
    fill_uniform_device(0, q_all.data_ptr(), n_all * Q, d, QUERY_SEED, 0, stream)
    oi = torch.empty((Q, k), dtype=torch.int32, device="cuda")
    os_ = torch.empty((Q, k), dtype=torch.float32, device="cuda")
    ui = torch.empty((Q, k), dtype=torch.int32, device="cuda")
    us = torch.empty((Q, k), dtype=torch.float32, device="cuda")

    def filt(i):
        ix.search_filtered_device(q_all[i].data_ptr(), f_dev.data_ptr(), Q, k, oi.data_ptr(), os_.data_ptr(), stream)

    def plain(i):
        ix.search_device(q_all[i].data_ptr(), Q, k, ui.data_ptr(), us.data_ptr(), stream)

    def timed(fn, i):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn(i)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for i in range(args.warmup):
        filt(i)
        plain(i)
    ix.enable_timing(True)
    ix.scan_time_ms()
    t = {"filtered": [], "unfiltered": []}
    scan = {"filtered": [], "unfiltered": []}
    for s in range(args.steps):
        for name, fn in (("filtered", filt), ("unfiltered", plain)):
            t[name].append(timed(fn, args.warmup + s))
            scan[name].append(ix.scan_time_ms()[0])
    ix.enable_timing(False)
    gpu = gpu_record()
    path = ix.last_path()
    ix.status(stream)
    gi = oi.cpu().numpy().view(np.uint32).copy()
    gs = os_.cpu().numpy()
    qs = q_all[n_all - 1].cpu().numpy()

    # ---- parity of the last filtered step
    bad_adm = bad_score = 0
    for q in range(Q):
        live = gi[q] != 0xFFFFFFFF
        bad_adm += int((~admits(tags[gi[q][live].astype(np.int64)], *[int(v) for v in filters[q]])).sum())
        x = np.stack([ix.read_rows(int(r), 1)[0] for r in gi[q][live]]).astype(np.float64)
        qq = qs[q].astype(np.float64)
        ex = x @ qq
        if metric == "cosine":
            ex = ex / np.maximum(np.linalg.norm(x, axis=1) * np.linalg.norm(qq), 1e-300)
        elif metric == "euclidean":
            ex = np.sqrt(((x - qq) ** 2).sum(1))
        bad_score += int((np.abs(gs[q][live] - ex) > 1e-4 * np.abs(ex) + 1e-6).sum())
    # planted near-copies (rows and tags restored afterwards)
    plant_q = [q for q in range(Q) if filters[q, 0]][:8]
    prow = rng.choice(n, size=2 * len(plant_q), replace=False)
    saved = [(int(r), ix.read_rows(int(r), 1)[0].copy(), tags[int(r)]) for r in prow]
    for j, q in enumerate(plant_q):
        g, b = int(prow[2 * j]), int(prow[2 * j + 1])
        ix.update_row(g, (qs[q] * 1.5).astype(np.float32))
        ix.update_row(b, (qs[q] * 1.7).astype(np.float32))
        ix.set_row_tags(np.array([tags[g] | filters[q, 0]], dtype=np.uint64), first_row=g)   # admitted
        ix.set_row_tags(np.array([tags[b] & ~filters[q, 0]], dtype=np.uint64), first_row=b)  # rejected
    qd = torch.from_numpy(qs).cuda()
    ix.search_filtered_device(qd.data_ptr(), f_dev.data_ptr(), Q, k, oi.data_ptr(), os_.data_ptr(), stream)
    ix.status(stream)
    pi = oi.cpu().numpy().view(np.uint32)
    planted_ok = sum(int(int(pi[q][0]) == int(prow[2 * j]) and int(prow[2 * j + 1]) not in pi[q].tolist())
                     for j, q in enumerate(plant_q))
    for r, row, tg in saved:
        ix.update_row(r, row)
        ix.set_row_tags(np.array([tg], dtype=np.uint64), first_row=r)

    sel = {}
    for m in FILTER_BITS:
        qm = [q for q in range(Q) if FILTER_BITS[q % len(FILTER_BITS)] == m][:4]
        if qm:
            sel[str(m)] = float(np.mean([admits(tags[:2_000_000], int(filters[q, 0]), 0, 0).mean() for q in qm]))
    fm, um = float(np.median(t["filtered"])), float(np.median(t["unfiltered"]))
    line = {"config": {"N": n, "dim": d, "corpus_dtype": "f32", "Q": Q, "k": k, "metric": metric, "path": path,
                       "filters": "query q: all_of of %s random bits (cycling)" % (list(FILTER_BITS),),
                       "selectivity_by_bits": sel, "tag_bytes": n * 8, "corpus_bytes": n * d * 4},
            "gpu": gpu,
            "filtered": {"ms": fm, "value": Q / (fm / 1e3), "unit": "queries/s", "scan_ms": float(np.median(scan["filtered"])),
                         "spread_ms": [min(t["filtered"]), max(t["filtered"])]},
            "unfiltered": {"ms": um, "value": Q / (um / 1e3), "unit": "queries/s", "scan_ms": float(np.median(scan["unfiltered"])),
                           "spread_ms": [min(t["unfiltered"]), max(t["unfiltered"])]},
            "ratio_filtered_over_unfiltered": fm / um, "steps": args.steps, "warmup": args.warmup,
            "timing": "median of one CUDA event pair per search (explicit stream, synchronised on both sides); filtered and "
                      "unfiltered alternate on the same queries; scan_ms = event-timed scan kernels only",
            "parity": {"inadmissible_rows_returned": bad_adm, "scores_off_fp64": bad_score, "planted_ok": planted_ok,
                       "planted": len(plant_q)}}
    if Q <= 64 and not args.no_masked:
        # what the batch replaces: one masked search per query, the row mask built and set on the host in between
        t0 = time.perf_counter()
        mask_s = 0.0
        for q in range(Q):
            m0 = time.perf_counter()
            ix.set_row_mask(admits(tags, *[int(v) for v in filters[q]]))
            mask_s += time.perf_counter() - m0
            ix.search(qs[q:q + 1], k)
        total = (time.perf_counter() - t0) * 1e3
        ix.set_row_mask(None)
        line["vs_separate_masked_searches"] = {"ms": total, "mask_ms": mask_s * 1e3, "search_ms": total - mask_s * 1e3,
                                               "speedup_of_one_filtered_batch": total / fm,
                                               "timing": "wall clock: Q x (host mask build + nk_index_set_row_mask + nk_search of 1 query)"}
    ix.release()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
