"""Do two builds of the index host layer compute the same thing the same way?  Calls every search entry point whose host
staging is shared (plain, _filtered, _windowed and _device searches, search_rows*, search_range*, search_pairs*,
search_pairs_rows*, k-NN graph update / remap* and nk_pairs_remap) once per configuration: seeded clustered rows, cosine and
euclidean, a 1-shard and a 3-shard index on device 0, AUTO and TENSOR_FILTER, with and without a row mask.  Prints one JSON
line per call: a sha256 of its outputs, its NkStats deltas and last_path.  Run it once per source tree, with PYTHONPATH set
to that tree (each built in place); every line must be identical.  Needs a GPU.

    PYTHONPATH=/tmp/parent python profiles/host_parity.py > parent.jsonl
    PYTHONPATH=. python profiles/host_parity.py > this.jsonl
    cmp parent.jsonl this.jsonl
"""
from __future__ import annotations

import hashlib
import json

import numpy as np
import torch

from nornicdb_b200.knn import GraphRowMap, KnnIndex, synthetic_tags

N, D, Q, K = 3000, 128, 16, 8
COUNTERS = ("kernel_launches", "bytes_h2d", "bytes_d2h", "bytes_scanned", "searches", "queries")


def digest(out) -> str:
    h = hashlib.sha256()
    for a in out if isinstance(out, tuple) else (out,):
        if isinstance(a, list):  # search_range: one (idx, score) pair per query
            for i, s in a:
                h.update(np.ascontiguousarray(i).tobytes()); h.update(np.ascontiguousarray(s).tobytes()); h.update(b"|")
        else:
            h.update(np.ascontiguousarray(np.asarray(a)).tobytes())
        h.update(b"/")
    return h.hexdigest()[:16]


def filter_of(tags):  # a row's own filter, from its tag: any of two of the tag's bits
    return np.stack([np.zeros_like(tags), np.zeros_like(tags), tags & np.uint64(0x0000_0000_0101_0000)], axis=1)


def window_of(values):  # a row's own window: its value +- 150
    v = values.astype(np.int64)
    return np.stack([np.maximum(v - 150, 1), v + 150], axis=1).astype(np.uint64)


def run(cfg: dict) -> None:
    rng = np.random.default_rng(11)
    ix = KnnIndex(D, metric=cfg["metric"], devices=cfg["devices"])
    ix.fill_clustered(N, 7, n_centres=32, sigma=0.1, unit_norm=True)
    ix.set_path(cfg["path"])
    tags = synthetic_tags(N, 3)
    values = rng.integers(1, 1000, N).astype(np.uint64)
    ix.set_row_tags(tags)
    ix.set_row_values(values)
    keep = rng.random(N) > 0.2

    def mask():
        if cfg["masked"]:
            ix.set_row_mask(np.resize(keep, len(ix)))

    def call(name, fn):
        s0 = ix.stats()
        out = fn()
        s1 = ix.stats()
        print(json.dumps({**cfg, "call": name, "sha": digest(out), "last_path": ix.last_path(),
                          **{c: s1[c] - s0[c] for c in COUNTERS}}), flush=True)
        return out

    mask()
    q = rng.standard_normal((Q, D)).astype(np.float32)
    qf = np.zeros((Q, 3), np.uint64); qf[:, 2] = np.uint64(1) << (np.arange(Q, dtype=np.uint64) % np.uint64(16))
    qw = np.stack([np.arange(Q) * 50 + 1, np.arange(Q) * 50 + 400], axis=1).astype(np.uint64)
    call("search", lambda: ix.search(q, K))
    call("search_filtered", lambda: ix.search_filtered(q, K, qf))
    call("search_windowed", lambda: ix.search_windowed(q, K, qw))
    call("search_windowed+f", lambda: ix.search_windowed(q, K, qw, filters=qf))
    if len(cfg["devices"]) == 1:
        dq, df, dw = (torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).cuda() for a in (q, qf, qw))
        oi = torch.empty((Q, K), dtype=torch.int32, device="cuda")
        os_ = torch.empty((Q, K), dtype=torch.float32, device="cuda")
        okeys = torch.empty((Q, K), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()

        def dev(fn):
            fn()
            torch.cuda.synchronize()
            ix.status()
            return oi.cpu().numpy(), os_.cpu().numpy()

        call("search_device", lambda: dev(lambda: ix.search_device(dq.data_ptr(), Q, K, oi.data_ptr(), os_.data_ptr())))
        call("search_filtered_device", lambda: dev(lambda: ix.search_filtered_device(dq.data_ptr(), df.data_ptr(), Q, K, oi.data_ptr(),
                                                                                     os_.data_ptr())))
        call("search_windowed_device", lambda: dev(lambda: ix.search_windowed_device(dq.data_ptr(), 0, dw.data_ptr(), Q, K, oi.data_ptr(),
                                                                                     os_.data_ptr())))
        call("search_windowed_device+f", lambda: dev(lambda: ix.search_windowed_device(dq.data_ptr(), df.data_ptr(), dw.data_ptr(), Q, K,
                                                                                       oi.data_ptr(), os_.data_ptr())))
        call("search_keys_device", lambda: (ix.search_keys_device(dq.data_ptr(), Q, K, okeys.data_ptr()), torch.cuda.synchronize(),
                                            okeys.cpu().numpy())[2])

    rows = np.arange(0, N, 7)
    call("search_rows", lambda: ix.search_rows(rows, K))
    call("search_rows_filtered", lambda: ix.search_rows(rows, K, filters=filter_of(tags[rows])))
    call("search_rows_windowed", lambda: ix.search_rows(rows, K, windows=window_of(values[rows])))
    _, sc5 = ix.search(q, 5)
    thr = float(np.median(sc5[:, -1]))  # each query's 5th neighbour: a few rows per query
    call("search_range", lambda: ix.search_range(q, thr))
    call("search_range_filtered", lambda: ix.search_range(q, thr, filters=qf))
    call("search_range_windowed", lambda: ix.search_range(q, thr, windows=qw))
    call("search_range_windowed+f", lambda: ix.search_range(q, thr, filters=qf, windows=qw))
    _, rs = ix.search_rows(np.arange(0, N, 97), 3)
    pthr = float(np.median(rs[:, -1]))  # a row's 3rd neighbour: a few pairs per row
    one_f = (0, 0, 0x0000_0000_0303_0000)
    call("search_pairs", lambda: ix.search_pairs(pthr))
    call("search_pairs_filtered", lambda: ix.search_pairs(pthr, first_row=500, n_rows=1500, filter=one_f))
    call("search_pairs_windowed", lambda: ix.search_pairs(pthr, window=(100, 900), max_gap=200))
    listed = np.arange(3, N, 11)
    call("search_pairs_rows", lambda: ix.search_pairs_rows(listed, pthr))
    call("search_pairs_rows_windowed", lambda: ix.search_pairs_rows(listed, pthr, filter=one_f, window=(1, 800), max_gap=300))

    # k-NN graphs (plain, filtered, windowed) and the self-join, brought up to date across append / update_row / remove_swap
    every = np.arange(N)
    kinds = {"": {}, "_filtered": {"filters": filter_of(tags)}, "_windowed": {"windows": window_of(values), "filters": filter_of(tags)}}
    graphs = {}
    for kind, a in kinds.items():
        gi, gs = call("graph_build" + kind, lambda: ix.search_rows(every, K, **a))
        graphs[kind] = (gi, gs, 0)
    pairs = call("pairs_build", lambda: ix.search_pairs(pthr, window=(1, 900), max_gap=250))
    add = rng.standard_normal((40, D)).astype(np.float32)
    add /= np.linalg.norm(add, axis=1, keepdims=True)
    ix.append(add)
    tags = np.concatenate([tags, synthetic_tags(40, 5)])
    values = np.concatenate([values, rng.integers(1, 1000, 40).astype(np.uint64)])
    ix.set_row_tags(tags[N:], first_row=N)
    ix.set_row_values(values[N:], first_row=N)
    ix.update_row(17, add[0])
    mask()
    for kind, a in kinds.items():
        b = {n: (filter_of(tags) if n == "filters" else window_of(values)) for n in a}
        gi, gs, _ = graphs[kind]
        graphs[kind] = call("knn_graph_update" + kind, lambda: ix.update_knn_graph(gi, gs, N, changed=[17], k=K, **b))
    m = GraphRowMap(len(ix))
    pm = GraphRowMap(N)
    pm.append(40)
    pm.update_row(17)
    for r in (5, 1200, 2999):
        ix.remove_swap(r)
        m.remove_swap(r)
        pm.remove_swap(r)
        tags[r], values[r] = tags[len(ix)], values[len(ix)]
    tags, values = tags[:len(ix)], values[:len(ix)]
    mask()
    for kind, a in kinds.items():
        b = {n: (filter_of(tags) if n == "filters" else window_of(values)) for n in a}
        gi, gs, _ = graphs[kind]
        call("knn_graph_remap" + kind, lambda: ix.remap_knn_graph(gi, gs, N + 40, m, k=K, **b))
    call("pairs_remap", lambda: ix.remap_pairs(pairs, N, pm, pthr, window=(1, 900), max_gap=250))
    ix.release()


def main() -> None:
    for metric in ("cosine", "euclidean"):
        for devices in ((0,), (0, 0, 0)):
            for path in ("auto", "filter"):
                for masked in (False, True):
                    run({"metric": metric, "devices": devices, "path": path, "masked": masked})


if __name__ == "__main__":
    main()
