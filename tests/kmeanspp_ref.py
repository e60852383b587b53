"""Host restatements of k-means++ seeding for the tests (test infrastructure only).

* kmeanspp_chunked: the rule nk_index_kmeanspp computes (include/nornic_knn.h, DESIGN §7 item 3): D² in squaredEuclidean's
  arithmetic, weights summed in chunks of 256 rows from each shard's first row, chunk sums in row order.
* kmeanspp_seq: initCentroidsKMeansPlusPlus (kmeans.go:364-426) literally: one sequential total, one sequential
  cumulative sum.
* sq_euclid64_rows: squaredEuclidean (kmeans.go:430-454, oracle.sq_euclid64) from every row to one point, bit for bit.

np.cumsum and np.add.accumulate add sequentially, in index order: they are the sequential fp64 sums of the contract."""
from __future__ import annotations

import numpy as np

CHUNK = 256
EPS = 2.0 ** -18  # the skip rule's margin


def sq_euclid64_rows(rows: np.ndarray, c: np.ndarray) -> np.ndarray:
    """fp32 differences, fp64 squares (exact: 24-bit operands), element j into s[j % 4] in ascending j, the tail past the
    last whole group of four into s0, then ((s0 + s1) + s2) + s3."""
    x = np.asarray(rows, dtype=np.float32)
    dim = x.shape[1]
    s = np.zeros((4, x.shape[0]), dtype=np.float64)
    full = dim // 4 * 4
    with np.errstate(invalid="ignore", over="ignore"):
        d = (x - np.asarray(c, dtype=np.float32)).astype(np.float64)
        sq = d * d
        for j in range(0, full, 4):
            s[0] += sq[:, j]; s[1] += sq[:, j + 1]; s[2] += sq[:, j + 2]; s[3] += sq[:, j + 3]
        for j in range(full, dim):
            s[0] += sq[:, j]
        return ((s[0] + s[1]) + s[2]) + s[3]


def _update(rows, d2, near, c, seed_row):
    dist = sq_euclid64_rows(rows, seed_row)
    if c == 0:
        d2[:] = dist  # kmeans.go:379-384: assigned, a NaN stays NaN
        near[:] = 0
    else:
        with np.errstate(invalid="ignore"):
            lower = dist < d2  # kmeans.go:418
        d2[lower] = dist[lower]
        near[lower] = c


def _chunk_sums(w: np.ndarray, shard_sizes) -> np.ndarray:
    out = []
    off = 0
    for sz in shard_sizes:
        part = w[off:off + sz]
        pad = np.zeros(-len(part) % CHUNK)
        with np.errstate(invalid="ignore", over="ignore"):
            out.append(np.add.accumulate(np.concatenate([part, pad]).reshape(-1, CHUNK), axis=1)[:, -1])
        off += sz
    return np.concatenate(out)


def _chunk_starts(shard_sizes):
    starts, counts, off = [], [], 0
    for sz in shard_sizes:
        for r in range(0, sz, CHUNK):
            starts.append(off + r)
            counts.append(min(CHUNK, sz - r))
        off += sz
    return starts, counts


def kmeanspp_chunked(rows, K, first_row, u, shard_sizes=None):
    """-> (seeds [K], potential [K], min_d2 [n]) of the device rule with the given shard sizes (default: one shard)."""
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    n = rows.shape[0]
    shard_sizes = [n] if shard_sizes is None else [s for s in shard_sizes if s]
    assert sum(shard_sizes) == n
    starts, counts = _chunk_starts(shard_sizes)
    d2 = np.zeros(n)
    near = np.zeros(n, dtype=np.int64)
    seeds, pot = [], []
    seed = int(first_row)
    for c in range(K):
        seeds.append(seed)
        _update(rows, d2, near, c, rows[seed])
        with np.errstate(invalid="ignore", over="ignore"):
            P = np.cumsum(_chunk_sums(d2, shard_sizes))
        T = float(P[-1])
        pot.append(T)
        if c + 1 == K:
            break
        target = float(u[c]) * T
        hit = np.nonzero(P >= target)[0]
        if hit.size == 0:
            seed = n - 1
            continue
        j = int(hit[0])
        before = float(P[j - 1]) if j else 0.0
        with np.errstate(invalid="ignore", over="ignore"):
            L = np.cumsum(d2[starts[j]:starts[j] + counts[j]])
            ok = np.nonzero(before + L >= target)[0]
        seed = starts[j] + int(ok[0])
    return np.array(seeds, dtype=np.uint32), np.array(pot), d2


def kmeanspp_seq(rows, K, first_row, u):
    """kmeans.go:364-426 literally (with the draws given): -> (seeds [K], potential [K], min_d2 [n])."""
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    n = rows.shape[0]
    d2 = np.zeros(n)
    near = np.zeros(n, dtype=np.int64)
    seeds, pot = [], []
    seed = int(first_row)
    for c in range(K):
        seeds.append(seed)
        _update(rows, d2, near, c, rows[seed])
        with np.errstate(invalid="ignore", over="ignore"):
            cum = np.cumsum(d2)
        total = float(cum[-1])
        pot.append(total)
        if c + 1 == K:
            break
        target = float(u[c]) * total
        hit = np.nonzero(cum >= target)[0]
        seed = int(hit[0]) if hit.size else n - 1
    return np.array(seeds, dtype=np.uint32), np.array(pot), d2


def skips(delta, m, dim):
    """The pass's row skip: the new seed lies at computed δ² = delta from the row's nearest seed, the row at computed D² = m."""
    with np.errstate(invalid="ignore", over="ignore"):
        return (dim <= 32768) & (delta < np.inf) & (delta >= 4.0 * m * (1.0 + EPS))
