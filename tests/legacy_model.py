"""The legacy boundary's arithmetic (include/nornic_knn.h part 1, the drop-in for pkg/gpu/cuda/cuda_bridge.go:231-375) as
closed-form code, and the score arrays and launch edges where a device restatement of it goes wrong.  Shared by
tests/test_legacy_model_cpu.py (the model against the C restatement of the reference, no GPU) and
tests/test_gpu_legacy_edges.py (every legacy call against the model).

  * cuda_topk (cuda_bridge.go:327-375): k slots start as (0, -1e30f); a forward scan inserts score s only if s > the last
    slot, ahead of every slot it is strictly greater than.  So NaN, -inf and anything <= -1e30f never enter, equal scores
    keep the lower index first, -0.0 and +0.0 are equal, each score keeps its own bits and unused slots stay (0, -1e30f).
  * cuda_compute_norms: cublasSnrm2 per row, free of intermediate overflow and underflow; modelled as the fp64 norm
    rounded once to fp32.
  * cuda_normalize_vectors (cuda_bridge.go:249-284): rows whose norm is > 1e-10f are scaled by fl32(1.0f / norm) with
    cublasSscal; the others are left as they are.
  * The launch constants the device top-k and the row kernels are planned with, read from the sources, so the tested edges
    move when a constant does."""
from __future__ import annotations

import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "nornicdb_b200", "csrc")

FLOOR = np.float32(-1e30)        # the reference's empty-slot score
NORM_FLOOR = np.float32(1e-10)   # cuda_bridge.go:267: rows with norm <= this are left untouched
F32_MAX = np.finfo(np.float32).max
U = 2.0 ** -24                   # unit roundoff of fp32


def _read(path: str) -> str:
    with open(path) as f:
        return f.read()


def _constant(src: str, name: str) -> int:
    m = re.findall(rf"constexpr\s+\w+\s+{name}\s*=\s*(\d+)\s*;", _read(os.path.join(CSRC, src)))
    assert len(m) == 1, f"{name} in {src}: {m}"
    return int(m[0])


def _define(name: str) -> int:
    m = re.findall(rf"#define\s+{name}\s+(\d+)u?\b", _read(os.path.join(ROOT, "include", "nornic_knn.h")))
    assert len(m) == 1, f"{name}: {m}"
    return int(m[0])


def _warp_grid_constants() -> tuple:
    """(CTAs per SM, warps = rows per CTA) of warp_grid in rowops.cu: one sweep of the grid covers SMs * both rows"""
    text = _read(os.path.join(CSRC, "rowops.cu"))
    per_sm = re.findall(r"static inline unsigned warp_grid\(uint64_t n, int per_sm = (\d+)\)", text)
    rows = re.findall(r"uint64_t blocks = \(n \+ (\d+)\) / (\d+);", text)
    assert len(per_sm) == 1 and len(rows) == 1 and int(rows[0][0]) + 1 == int(rows[0][1]), (per_sm, rows)
    return int(per_sm[0]), int(rows[0][1])


TOPK_IV = _constant("merge.cu", "TOPK_IV")            # scores per CTA interval of topk_scores_kernel
TOPK_THREADS = _constant("merge.cu", "TOPK_THREADS")
NK_MAX_K = _define("NK_MAX_K")                        # one device pass; larger k runs ceil(k / NK_MAX_K) passes
NK_MAX_K_TOTAL = _define("NK_MAX_K_TOTAL")
ROWS_PER_SM, ROWS_PER_CTA = _warp_grid_constants()


def warp_sweep(num_sms: int) -> int:
    """rows one sweep of a row kernel's grid covers (one warp per row): past it, warps take a second row"""
    return num_sms * ROWS_PER_SM * ROWS_PER_CTA


# ---- launch arithmetic of topk_scores -----------------------------------------------------------------------------------
def topk_launch(n, num_sms: int, bits: int):
    """(intervals, grid, rows the intervals cover) of topk_scores over n scores, with its index arithmetic in `bits`-bit
    unsigned integers: 32 is what the launch did before, 64 what it does.  n may be a numpy array."""
    t = np.uint32 if bits == 32 else np.uint64
    n = np.asarray(n, dtype=np.uint64).astype(t)
    with np.errstate(over="ignore"):
        num_iv = (n + t(TOPK_IV - 1)) // t(TOPK_IV)
        grid = np.minimum(t(2 * num_sms), num_iv)
        # interval iv covers [iv * TOPK_IV, min((iv + 1) * TOPK_IV, n)); the intervals are 0 .. num_iv - 1
        last = np.where(num_iv > 0, num_iv - t(1), t(0))
        last_lo, last_hi = last * t(TOPK_IV), np.minimum((last + t(1)) * t(TOPK_IV), n)
        last_rows = np.where((num_iv > 0) & (last_hi > last_lo), last_hi - last_lo, t(0))
        covered = np.where(num_iv > 0, last * t(TOPK_IV) + last_rows, t(0))
    return num_iv.astype(np.uint64), grid.astype(np.uint64), covered.astype(np.uint64)


# ---- cuda_topk ----------------------------------------------------------------------------------------------------------
def admissible(scores) -> np.ndarray:
    """the scores the reference's scan can insert: not NaN and > -1e30f"""
    s = np.asarray(scores, dtype=np.float32)
    with np.errstate(invalid="ignore"):
        return ~np.isnan(s) & (s > FLOOR)


def topk_model(scores, k: int):
    """cuda_topk in closed form -> (idx uint32 [k'], score float32 [k']), k' = min(k, n) (0 when k or n is 0)"""
    s = np.ascontiguousarray(np.asarray(scores, dtype=np.float32).reshape(-1))
    n = s.size
    k = min(int(k), n)
    if k <= 0:
        return np.zeros(0, np.uint32), np.zeros(0, np.float32)
    ok = np.flatnonzero(admissible(s))
    # stable by value, descending: -s in fp64 maps -0.0 and +0.0 to equal keys, so they keep index order
    top = ok[np.argsort(-s[ok].astype(np.float64), kind="stable")][:k]
    idx = np.zeros(k, np.uint32)
    out = np.full(k, FLOOR, np.float32)
    idx[:top.size] = top
    out[:top.size] = s[top]
    return idx, out


# ---- cuda_compute_norms / cuda_normalize_vectors ------------------------------------------------------------------------
def nrm2_model(x) -> np.ndarray:
    """per-row fp64 2-norm rounded once to fp32 (no intermediate overflow or underflow); inf with an inf element, NaN with
    a NaN element"""
    x = np.asarray(x, dtype=np.float32)
    x = x.reshape(-1, x.shape[-1]).astype(np.float64)
    # every fp32 square and every sum of up to 2^32 of them is a normal fp64 number: no scaling needed
    with np.errstate(over="ignore"):
        return np.sqrt(np.sum(x * x, axis=1)).astype(np.float32)


def normalize_model(x, norm32) -> np.ndarray:
    """x * fl32(1.0f / norm32) per row where norm32 > 1e-10f (cublasSscal with the reference's scale), else x"""
    x = np.asarray(x, dtype=np.float32)
    x = x.reshape(-1, x.shape[-1])
    norm32 = np.asarray(norm32, dtype=np.float32).reshape(-1)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore", under="ignore"):
        keep = ~(norm32 > NORM_FLOOR)
        inv = np.float32(1.0) / np.where(keep, np.float32(1.0), norm32)
        return np.where(keep[:, None], x, x * inv[:, None]).astype(np.float32)


def gamma(d: int) -> float:
    """gamma_d = d u / (1 - d u): the relative error bound of a d-term fp32 sum of products"""
    return d * U / (1.0 - d * U)


# ---- score arrays -------------------------------------------------------------------------------------------------------
def _next(x, toward):
    return np.nextafter(np.float32(x), np.float32(toward), dtype=np.float32)


TINY = np.finfo(np.float32).smallest_subnormal
SUB_MAX = _next(np.finfo(np.float32).tiny, 0)     # the largest subnormal
# scores at the reference's edges: the ones below never enter its top-k
INADMISSIBLE = np.array([np.nan, -np.inf, -F32_MAX, FLOOR, _next(FLOOR, -np.inf)], np.float32)
# ... and the ones above do, whatever their neighbours
EDGE_ADMISSIBLE = np.array([np.inf, F32_MAX, -0.0, 0.0, TINY, -TINY, SUB_MAX, -SUB_MAX, _next(FLOOR, 0)], np.float32)

MIXES = ("plain", "nan1", "nan50", "nan100", "inf", "fltmax", "floor", "subnormal", "zeros", "runs", "all")


def special_scores(n: int, mix: str, seed: int) -> np.ndarray:
    """n fp32 scores of one kind the reference's scan treats specially.  Ordinary scores come from a grid of 1/8 steps in
    [-4, 4), so ties are common at every size.
      plain / nan1 / nan50 / nan100: NaN at 0%, 1%, 50%, 100%;  inf: +-inf;  fltmax: +-FLT_MAX;  floor: -1e30f and both its
      fp32 neighbours;  subnormal: +-subnormals among zeros and a few grid values;  zeros: +-0.0 interleaved at random,
      with few scores above them;  runs: runs of up to thousands of equal scores;  all: every ingredient at once."""
    rng = np.random.default_rng([seed, n, MIXES.index(mix)])
    s = (rng.integers(-32, 32, n) / 8.0).astype(np.float32)

    def sprinkle(values, frac):
        at = rng.random(n) < frac
        s[at] = rng.choice(np.asarray(values, np.float32), int(at.sum()))

    if mix in ("nan1", "nan50", "nan100"):
        sprinkle([np.nan], {"nan1": 0.01, "nan50": 0.5, "nan100": 1.01}[mix])
    elif mix == "inf":
        sprinkle([np.inf, -np.inf], 0.05)
    elif mix == "fltmax":
        sprinkle([F32_MAX, -F32_MAX], 0.05)
    elif mix == "floor":
        s[:] = -4.0 - s * s  # all below 0 so the floor values reach the top k of short arrays
        sprinkle(INADMISSIBLE[3:].tolist() + [_next(FLOOR, 0)], 0.3)
    elif mix == "subnormal":
        s[:] = 0.0
        sprinkle([TINY, -TINY, SUB_MAX, -SUB_MAX, 2 * TINY, -3 * TINY], 0.5)
        sprinkle([0.125, -0.125], 0.01)
    elif mix == "zeros":
        s[:] = np.where(rng.random(n) < 0.5, np.float32(-0.0), np.float32(0.0))
        sprinkle([1.0, -1.0, 0.5], 0.02)
    elif mix == "runs":
        pos = 0
        while pos < n:
            run = int(rng.integers(1, 4000))
            s[pos:pos + run] = rng.integers(-8, 8) / 4.0
            pos += run
    elif mix == "all":
        sprinkle(np.concatenate([INADMISSIBLE, EDGE_ADMISSIBLE]), 0.4)
        if n > 64:
            a = int(rng.integers(0, n - 32))
            s[a:a + 32] = s[a]  # one run
    else:
        assert mix == "plain", mix
    return s


def short_admissible(n: int, count: int, seed: int) -> np.ndarray:
    """n scores of which exactly `count` are admissible (ties, +-0.0, subnormals, the floor's upper neighbour among them);
    every other one is NaN, -inf, -FLT_MAX, -1e30f or its lower neighbour"""
    rng = np.random.default_rng([seed, n, count])
    s = rng.choice(INADMISSIBLE, n)
    at = rng.permutation(n)[:count]
    pool = np.concatenate([EDGE_ADMISSIBLE, (np.arange(-16, 16) / 4.0).astype(np.float32)])
    s[at] = rng.choice(pool, count)
    assert admissible(s).sum() == count
    return s


def straddle(n: int, edges, run: int, seed: int, zeros: bool = False) -> np.ndarray:
    """n scores with a run of `run` equal scores across every rank in `edges` (rank r = the r-th best, from 1): the run at
    edge e holds ranks e - run // 2 + 1 .. e - run // 2 + run.  Ranks between runs are distinct.  zeros: the run at the
    last edge is -0.0 and +0.0 alternately, at random rows, so only index order can split it.  Every score below the runs is lower
    than all of them."""
    rng = np.random.default_rng([seed, n, run, len(edges)])
    edges = sorted(edges)
    R = edges[-1] - run // 2 + run  # ranks that carry a chosen score
    assert R <= n and edges[0] - run // 2 >= 0
    value = np.arange(R, 0, -1, dtype=np.float64)  # rank i (0-based) -> R - i: distinct, exact in fp32
    for e in edges:
        lo = e - run // 2
        value[lo:lo + run] = value[lo]
    if zeros:
        value -= value[edges[-1] - run // 2]  # the last run lands on 0
    s = np.empty(n, np.float32)
    pos = rng.permutation(n)
    s[pos[:R]] = value
    if zeros:
        lo = edges[-1] - run // 2
        z = pos[lo:lo + run]
        s[z] = np.where(np.arange(run) % 2 == 0, np.float32(-0.0), np.float32(0.0))  # z is in random order
    s[pos[R:]] = value.min() - 1.0 - rng.integers(0, 1000, n - R)
    return s
