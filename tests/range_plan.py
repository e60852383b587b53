"""The sizes where the range pipeline's plan changes, computed from the rules the library applies, so that a test names each
edge by its rule rather than by a number.  Shared by tests/test_range_plan_cpu.py (the rules, the planted corpora and the
merge placement, no GPU) and tests/test_gpu_range_plan.py (every path on both sides of every edge).

Every range call (nk_search_range, the self-join, the incident pairs, the graph update's reverse scan) runs, per shard:
  * the scan: on the tensor paths one query prep and then the launches of plan_launches (scan_tensor.cu): 64 query columns
    while at most 64 queries remain, else 128; 4 query groups per launch while more than 384 remain (grid % 4 == 0 and
    grid >= 8), 2 while more than 128 remain (grid even and >= 4), grid = min(SMs, tiles of ROWS rows).  On CUDA cores
    one launch per query group of 8 / 4 / 2 / 1 (4 / 1 on scalar loads), halved while the group's queries pass 96 KB.
  * list capacity (range.cu): LIST0, or what an earlier call left in the workspace; one re-run at the exact size if the
    longest fill is over it.  The pass count shows in NkStats::bytes_scanned (scan_bytes, index_api.cu).
  * re-scoring (RS_ENTRIES list entries per CTA), compaction (CP_THREADS per CTA) and the sort of RUN-key runs, each
    looped over blocks of MAX_GRID_Y queries; then merge passes w = RUN, 2 RUN, .. while w < the longest list.
And the planted corpora the GPU tests run on: each query gets an exact, chosen number of survivors, with a gap on both sides of
its threshold many times wider than any filter's error bound."""
from __future__ import annotations

import os
import re
from dataclasses import dataclass

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "nornicdb_b200", "csrc")

NUM_SMS_H100 = 132          # cudaDeviceProp::multiProcessorCount of an H100 SXM
SIMT_BUDGET = 96 * 1024     # the CUDA-core range scan's query bytes per CTA (scan_simt_range)


def _constant(src: str, name: str) -> int:
    text = open(os.path.join(CSRC, src)).read()
    m = re.findall(rf"constexpr\s+\w+\s+{name}\s*=\s*(\d+)\s*;", text)
    assert len(m) == 1, f"{name} in {src}: {m}"
    return int(m[0])


LIST0 = _constant("range.cu", "LIST0")
RS_ENTRIES = _constant("range.cu", "RS_ENTRIES")
CP_THREADS = _constant("range.cu", "CP_THREADS")
RUN = _constant("range.cu", "RUN")
MAX_GRID_Y = _constant("range.cu", "MAX_GRID_Y")
ROWS = _constant("scan_tensor_shared.cuh", "ROWS")
QT_BIG = _constant("scan_tensor_shared.cuh", "QT_BIG")
SEARCH_ROWS_BLOCK = _constant("index_api.cu", "SEARCH_ROWS_BLOCK")
SCAN_TILE_ROWS = _constant("index_api.cu", "SCAN_TILE_ROWS")

TENSOR_PATHS = ("filter", "shadow")


# ---- the plan ---------------------------------------------------------------------------------------------------------
def grid(n: int, num_sms: int = NUM_SMS_H100) -> int:
    """CTAs of a tensor-core scan over n rows (make_filter_plan)"""
    return min(num_sms, -(-n // ROWS))


def tensor_launches(Q: int, grid: int, max_groups: int = 4) -> list:
    """(qt, q0, nq, groups) of every tensor-core scan launch over Q queries (plan_launches)"""
    out, q0 = [], 0
    while q0 < Q:
        left = Q - q0
        qt, groups, nq = 64, 1, left
        if left > 64:
            if left > 3 * 128 and max_groups >= 4 and grid % 4 == 0 and grid >= 8:
                groups = 4
            elif left > 128 and max_groups >= 2 and grid % 2 == 0 and grid >= 4:
                groups = 2
            qt = 128
            nq = min(left, 128 * groups)
        out.append((qt, q0, nq, groups))
        q0 += nq
    return out


def simt_range_groups(Q: int, vec: bool, d: int = 64) -> list:
    """query-group sizes of the CUDA-core range scan's launches, in order (scan_simt_range)"""
    out, left = [], Q
    while left:
        qt = 8 if left >= 5 else 4 if left >= 3 else 2 if left == 2 else 1
        if not vec:
            qt = 4 if left >= 3 else 1
        while qt > 1 and qt * d * 4 > SIMT_BUDGET:
            qt = qt // 2 if vec else 1
        out.append(qt)
        left -= min(left, qt)
    return out


def simt_vec(d: int, dtype: str = "f32") -> bool:
    """vector loads: whole 16-byte row chunks (the rows themselves are 16-byte aligned)"""
    return d % (4 if dtype == "f32" else 8) == 0


def merge_passes(longest: int) -> int:
    """merge passes after the run sort: w = RUN, 2 RUN, .. while w < the longest list (range_sorted_keys)"""
    p, w = 0, RUN
    while w < longest:
        p, w = p + 1, w * 2
    return p


def query_blocks(Q: int) -> int:
    return -(-Q // MAX_GRID_Y)


def scan_launches(path: str, Q: int, n: int, d: int = 64, dtype: str = "f32", max_groups: int = 4) -> int:
    """launches of one range scan pass: the prep and the plan_launches split, or the CUDA-core groups"""
    if path == "simt":
        return len(simt_range_groups(Q, simt_vec(d, dtype), d))
    return 1 + len(tensor_launches(Q, grid(n), max_groups))


def range_launches(path: str, Q: int, n: int, survivors, retried: bool, d: int = 64, dtype: str = "f32",
                   fills=None) -> int:
    """what one shard's share of an nk_search_range call adds to NkStats::kernel_launches: the scan passes, re-scoring per
    query block if any list is non-empty, compaction and sort per query block if any query survives, the merge passes.
    survivors: per query; fills: the list fills (default: the survivors, as on a planted corpus)"""
    survivors = np.asarray(survivors)
    fills = survivors if fills is None else np.asarray(fills)
    out = scan_launches(path, Q, n, d, dtype) * (2 if retried else 1)
    if fills.max(initial=0) > 0:
        out += query_blocks(Q)
    if survivors.sum() > 0:
        out += 2 * query_blocks(Q) + merge_passes(int(survivors.max()))
    return out


def row_bytes(path: str, d: int, dtype: str = "f32", image: str = "bf16") -> int:
    """bytes per row one scan pass streams: the rows, or on `shadow` the image (BF16 padded to 64 columns, int8 to 128,
    16-bit rows in place)"""
    if path != "shadow":
        return d * (4 if dtype == "f32" else 2)
    if dtype != "f32":
        return d * 2
    return -(-d // 128) * 128 if image == "int8" else -(-d // 64) * 64 * 2


def scan_bytes(path: str, n: int, rbytes: int, Q: int, passes: int) -> int:
    """NkStats::bytes_scanned of `passes` range scans of n rows (scan_bytes): once per 8 queries on CUDA cores, per 128 in
    the filters"""
    width = 8 if path == "simt" else 128
    return n * rbytes * -(-Q // width) * passes


def edges() -> dict:
    """edge name -> the sizes on both sides of it"""
    return {
        "list capacity (fill)": [LIST0 - 1, LIST0, LIST0 + 1],
        "re-scoring CTA (fill)": [RS_ENTRIES - 1, RS_ENTRIES, RS_ENTRIES + 1],
        "compaction CTA (fill)": [CP_THREADS - 1, CP_THREADS, CP_THREADS + 1],
        "sort run (survivors)": [RUN - 1, RUN, RUN + 1],
        "second merge pass (survivors)": [2 * RUN - 1, 2 * RUN, 2 * RUN + 1],
        "third merge pass (survivors)": [4 * RUN, 4 * RUN + 1],
        "query blocks (Q)": [MAX_GRID_Y, MAX_GRID_Y + 1],
        "tensor columns (Q)": [64, 65],
        "2 query groups (Q)": [128, 129],
        "4 query groups (Q)": [384, 385],
        "one 4-group launch (Q)": [512, 513],
        "4-group launch and a tail (Q)": [640, 641],
        "tensor grid (tiles)": [NUM_SMS_H100, 8, 7, 6, 4, 3, 1],
        "CUDA-core groups (Q)": [1, 2, 3, 4, 5, 8, 9, 13],
    }


# ---- the merge kernel, restated -----------------------------------------------------------------------------------------
def merge_pass(src: np.ndarray, off: np.ndarray, w: int) -> np.ndarray:
    """range_merge_kernel's placement: each key goes to min(start, pstart) + its index in its own run + its rank in the
    partner run (an equal key counts as before it only when it sits in the earlier run); a run without a partner stays"""
    off = np.asarray(off, dtype=np.int64)
    Q = len(off) - 1
    g = np.arange(int(off[Q]))
    seg = np.searchsorted(off[:Q], g, side="right") - 1  # the last segment starting at or before g (empty ones included)
    base, n = off[seg], off[seg + 1] - off[seg]
    j = g - base
    run = j // w
    start = run * w
    at = g.copy()  # no partner run: already in place
    for s in np.unique(seg):
        for r in np.unique(run[seg == s]):
            sel = (seg == s) & (run == r)
            ps = (r ^ 1) * w
            if ps >= n[sel][0]:
                continue
            b0 = int(off[s])
            asc = src[b0 + ps: b0 + min(int(n[sel][0]), ps + w)][::-1]  # the partner run, ascending
            # descending runs: the partner keys placed before this one (strictly greater; or equal, from the earlier run)
            a = len(asc) - np.searchsorted(asc, src[g[sel]], side="right" if r % 2 == 0 else "left")
            at[sel] = base[sel] + np.minimum(start[sel], ps) + (j[sel] - start[sel]) + a
    placed = np.bincount(at, minlength=len(src))
    assert (placed == 1).all(), "the merge placement is not a permutation"
    dst = np.zeros_like(src)
    dst[at] = src[g]
    return dst


def sort_runs(keys: np.ndarray, off: np.ndarray) -> np.ndarray:
    """range_sort_runs_kernel: runs of RUN keys of every segment sorted descending"""
    out = keys.copy()
    for q in range(len(off) - 1):
        for r0 in range(int(off[q]), int(off[q + 1]), RUN):
            r1 = min(r0 + RUN, int(off[q + 1]))
            out[r0:r1] = np.sort(out[r0:r1])[::-1]
    return out


def make_keys(score: np.ndarray, row: np.ndarray) -> np.ndarray:
    """make_key (common.cuh): order-preserving score bits above the inverted row, so keys sort (score desc, row asc)"""
    b = np.asarray(score, np.float32).view(np.uint32).astype(np.uint64)
    ordb = np.where(b & np.uint64(0x80000000), ~b & np.uint64(0xFFFFFFFF), b | np.uint64(0x80000000))
    return (ordb << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - np.asarray(row, np.uint64))


# ---- planted corpora ----------------------------------------------------------------------------------------------------
EPS = 0.05       # a planted row is its query plus EPS times a unit vector: cosine >= 1 / sqrt(1 + EPS^2) ~ 0.9988
MIN_GAP = 0.05   # the gap (in key units of |q| |x| or |q|^2 + |x|^2) a planted corpus must keep on both sides of every threshold


@dataclass
class Planted:
    rows: np.ndarray      # [n x d] fp32
    queries: np.ndarray   # [Q x d] fp32
    thr: np.ndarray       # [Q] API thresholds (euclidean: distances), fp32
    owner: np.ndarray     # [n] the query whose planted row this is, -1 for background rows
    counts: np.ndarray    # [Q] planted rows per query
    gap: float            # the narrowest half-gap around a threshold, relative to the pair's scale

    def expected(self, q: int, admitted=None) -> np.ndarray:
        """rows query q must return (sorted), restricted to `admitted` (bool per row) if given"""
        m = self.owner == q
        if admitted is not None:
            m &= admitted
        return np.flatnonzero(m)


def _unit(rng, n, d):
    g = rng.standard_normal((n, d))
    return g / np.linalg.norm(g, axis=1, keepdims=True)


def keys64(rows, queries, metric):
    """fp64 keys [Q x n] (cosine / dot: score; euclidean: -distance^2) and their scale (|q||x|; |q|^2 + |x|^2)"""
    x = np.asarray(rows, np.float64)
    q = np.asarray(queries, np.float64)
    s = q @ x.T
    xn, qn = np.linalg.norm(x, axis=1)[None, :], np.linalg.norm(q, axis=1)[:, None]
    if metric == "cosine":
        return s / (qn * xn), np.ones_like(s)
    if metric == "dot":
        return s, qn * xn
    return -(qn ** 2 + xn ** 2 - 2.0 * s), qn ** 2 + xn ** 2


def bounds_np(rows, queries, owner, metric, chunk=1024):
    """per query: the highest background key, the lowest planted key (nan if none), and the scale at each"""
    Q = len(queries)
    bg, pl, sb, sp = (np.full(Q, np.nan) for _ in range(4))
    for c in range(0, Q, chunk):
        k, s = keys64(rows, queries[c:c + chunk], metric)
        mine = owner[None, :] == np.arange(c, c + len(k))[:, None]
        kb = np.where(mine, -np.inf, k)
        kp = np.where(mine, k, np.inf)
        ib, ip = kb.argmax(1), kp.argmin(1)
        r = np.arange(len(k))
        bg[c:c + len(k)], sb[c:c + len(k)] = kb[r, ib], s[r, ib]
        has = mine.any(1)
        pl[c:c + len(k)] = np.where(has, kp[r, ip], np.nan)
        sp[c:c + len(k)] = np.where(has, s[r, ip], np.nan)
    return bg, pl, sb, sp


def planted(counts, d: int, metric: str, n: int, seed: int, dup_min: int = RUN, bounds=bounds_np) -> Planted:
    """A corpus of n rows where query q has exactly counts[q] rows above its threshold: near-copies of the query (cosine
    >= 0.998) at random positions, the rest unit directions of norm 0.5 .. 1 (|cosine| mostly < 0.6).  A query with at least
    dup_min planted rows has half of them exact copies of one row, so they share one score across run and merge
    boundaries.  Each threshold lies halfway between the query's lowest planted key and its highest background key (fp64,
    `bounds` computes them); a query with no planted row gets its threshold 0.3 |q|^2 above its best background row."""
    counts = np.asarray(counts, dtype=np.int64)
    Q, planted_rows = len(counts), int(counts.sum())
    assert planted_rows <= n
    rng = np.random.default_rng(seed)
    q = _unit(rng, Q, d)
    x = _unit(rng, n, d) * rng.uniform(0.5, 1.0, size=(n, 1))
    owner = np.full(n, -1, dtype=np.int64)
    at = rng.permutation(n)[:planted_rows]
    pos = 0
    for qi in np.flatnonzero(counts):
        c = int(counts[qi])
        v = q[qi][None, :] + EPS * _unit(rng, c, d)
        if c >= dup_min:
            v[: c // 2] = v[0]
        x[at[pos:pos + c]] = v
        owner[at[pos:pos + c]] = qi
        pos += c
    rows, queries = x.astype(np.float32), q.astype(np.float32)
    bg, pl, sb, sp = bounds(rows, queries, owner, metric)
    pl = np.where(np.isnan(pl), bg + 0.6, pl)
    sp = np.where(np.isnan(sp), sb, sp)
    tk = (bg + pl) / 2
    thr = (np.sqrt(-tk) if metric == "euclidean" else tk).astype(np.float32)
    tk32 = -(thr.astype(np.float64) ** 2) if metric == "euclidean" else thr.astype(np.float64)
    gap = float(min(((pl - tk32) / sp).min(), ((tk32 - bg) / sb).min()))
    return Planted(rows, queries, thr, owner, counts, gap)
