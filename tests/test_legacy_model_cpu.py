"""The legacy boundary's model (tests/legacy_model.py) against the C restatement of the reference (oracle/knn_oracle.c), and
the launch arithmetic of the device top-k at the top of the 32-bit row range.  No GPU."""
import numpy as np
import pytest

import legacy_model as lm


def test_constants_parse():
    assert lm.TOPK_IV > 0 and lm.TOPK_IV % lm.TOPK_THREADS == 0
    assert lm.NK_MAX_K == 1024 and lm.NK_MAX_K_TOTAL % lm.NK_MAX_K == 0
    assert (lm.ROWS_PER_SM, lm.ROWS_PER_CTA) == (16, 8)
    assert lm.warp_sweep(132) == 132 * 16 * 8


def _same(model, oracle):
    (mi, ms), (oi, os_) = model, oracle
    assert mi.dtype == np.uint32 and ms.dtype == np.float32
    assert mi.tolist() == oi.tolist()
    assert ms.view(np.uint32).tolist() == os_.view(np.uint32).tolist()


def test_topk_model_small_n_every_k(oracle_mod):
    """every k from 1 to n and past it, on every mix, at n up to 40"""
    cases = 0
    for mix in lm.MIXES:
        for n in (1, 2, 3, 5, 8, 13, 40):
            for seed in range(4):
                s = lm.special_scores(n, mix, seed)
                for k in range(1, n + 3):
                    _same(lm.topk_model(s, k), oracle_mod.topk_insertion(s, k))
                    cases += 1
    assert cases > 3000


def test_topk_model_edges(oracle_mod):
    """the examples of each rule, then short admissible counts, runs and +-0.0 straddling rank k"""
    nan, inf = np.float32(np.nan), np.float32(np.inf)
    idx, sc = lm.topk_model([nan, 1, -inf], 3)
    assert idx.tolist() == [1, 0, 0] and sc.view(np.uint32).tolist() == np.float32([1, -1e30, -1e30]).view(np.uint32).tolist()
    assert lm.topk_model(np.float32([-0.0, 0.0]), 1)[0].tolist() == [0]
    assert lm.topk_model(np.float32([0.0, -0.0]), 2)[1].view(np.uint32).tolist() == [0, 0x80000000]
    assert lm.topk_model(np.float32([-1e30, -3e38, 5]), 3)[0].tolist() == [2, 0, 0]
    assert lm.topk_model([], 3)[0].size == 0 and lm.topk_model([1.0], 0)[0].size == 0
    for k in (1, 2, 7, 64):
        for count in (k - 1, k, k + 1):
            s = lm.short_admissible(300, count, k)
            _same(lm.topk_model(s, k), oracle_mod.topk_insertion(s, k))
    for k, run in ((10, 4), (64, 9), (100, 31)):
        for zeros in (False, True):
            s = lm.straddle(500, [k // 2, k], run, 5, zeros=zeros)
            for kk in (k - 1, k, k + 1):
                _same(lm.topk_model(s, kk), oracle_mod.topk_insertion(s, kk))
            # the run really straddles rank k: its scores sit on both sides of it
            idx, sc = lm.topk_model(s, k + run)
            assert sc[k - 1] == sc[k] and (not zeros or np.signbit(sc[k - run // 2:k + run - run // 2]).any())


@pytest.mark.parametrize("mix", lm.MIXES)
def test_topk_model_medium(oracle_mod, mix):
    for n, k in ((1000, 10), (3000, 129), (5000, 5000), (5000, 6000)):
        s = lm.special_scores(n, mix, 11)
        _same(lm.topk_model(s, k), oracle_mod.topk_insertion(s, k))


def test_topk_launch_wraps_in_32_bits():
    """the 32-bit interval count wraps to 0 for n > 2^32 - 1024: a launch with grid 0; 64-bit arithmetic covers every row"""
    top = 2 ** 32
    n = np.arange(top - 1023, top, dtype=np.uint64)
    iv32, grid32, cov32 = lm.topk_launch(n, 132, 32)
    assert (iv32 == 0).all() and (grid32 == 0).all() and (cov32 == 0).all()
    iv64, grid64, cov64 = lm.topk_launch(n, 132, 64)
    assert (iv64 == 2 ** 32 // lm.TOPK_IV).all() and (grid64 == 264).all() and (cov64 == n).all()
    # below the edge the two agree
    n = np.array([1, lm.TOPK_IV - 1, lm.TOPK_IV, lm.TOPK_IV + 1, 300001, top - 1025, top - 1024], np.uint64)
    for a, b in zip(lm.topk_launch(n, 132, 32), lm.topk_launch(n, 132, 64)):
        assert (a == b).all()
    assert (lm.topk_launch(n, 132, 64)[2] == n).all()


def test_nrm2_model():
    rng = np.random.default_rng(3)
    for d in (1, 3, 4, 33, 129, 4097):
        x = rng.standard_normal((20, d)).astype(np.float32)
        want = np.linalg.norm(x.astype(np.float64), axis=1)
        got = lm.nrm2_model(x)
        assert (np.abs(got - want) <= np.abs(want) * lm.U).all()
        for scale in (1e-30, 1e-20, 1e19, 1e25, float(lm.F32_MAX) / np.sqrt(d)):
            xs = (x.astype(np.float64) * scale / np.abs(x).max(axis=1, keepdims=True)).astype(np.float32)
            m = lm.nrm2_model(xs)
            with np.errstate(over="ignore", under="ignore"):
                sumsq32 = np.sum(xs * xs, axis=1, dtype=np.float32)
            assert np.isfinite(m).all() and (m > 0).all(), (d, scale)
            w = np.linalg.norm(xs.astype(np.float64) / scale, axis=1) * scale
            assert (np.abs(m.astype(np.float64) - w) <= w * lm.U * 1.0001).all(), (d, scale)
            if scale >= 1e25 or (scale >= 1e19 and d >= 33):
                assert np.isinf(sumsq32).any()  # where a plain fp32 sum of squares overflows
    x = np.ones((3, 5), np.float32)
    x[0, 2], x[1, 1], x[2] = np.inf, np.nan, 0
    assert np.isinf(lm.nrm2_model(x)[0]) and np.isnan(lm.nrm2_model(x)[1]) and lm.nrm2_model(x)[2] == 0


def test_normalize_model():
    x = np.float32([[3, 4], [1e-11, 0], [np.nan, 1], [np.inf, 1]])
    n = lm.nrm2_model(x)
    y = lm.normalize_model(x, n)
    assert y[0].tolist() == [np.float32(3) * (np.float32(1) / np.float32(5)), np.float32(4) * (np.float32(1) / np.float32(5))]
    assert y[1].tolist() == x[1].tolist()           # norm <= 1e-10: untouched
    assert np.isnan(y[2, 0]) and y[2, 1] == 1        # NaN norm: untouched
    assert np.isnan(y[3, 0]) and y[3, 1] == 0        # inf norm: scaled by 1/inf = 0
    # the 1e-10 threshold in one dimension: sqrtf(x*x) == |x|, so the edge is exact
    for v in (lm.NORM_FLOOR, -lm.NORM_FLOOR):
        assert lm.normalize_model([[v]], lm.nrm2_model([[v]]))[0, 0] == v
        up = np.nextafter(v, np.float32(2 * v), dtype=np.float32)
        assert abs(lm.normalize_model([[up]], lm.nrm2_model([[up]]))[0, 0]) == 1.0


def test_special_scores_ingredients():
    n = 20000
    frac = {m: np.isnan(lm.special_scores(n, m, 1)).mean() for m in ("plain", "nan1", "nan50", "nan100")}
    assert frac["plain"] == 0 and 0.005 < frac["nan1"] < 0.02 and 0.45 < frac["nan50"] < 0.55 and frac["nan100"] == 1
    s = lm.special_scores(n, "floor", 1)
    assert {lm.FLOOR, lm._next(lm.FLOOR, 0), lm._next(lm.FLOOR, -np.inf)} <= set(s.tolist())
    z = lm.special_scores(n, "zeros", 1)
    assert np.signbit(z[z == 0]).mean() > 0.3 and (~np.signbit(z[z == 0])).mean() > 0.3
    sub = lm.special_scores(n, "subnormal", 1)
    assert ((np.abs(sub) > 0) & (np.abs(sub) < np.finfo(np.float32).tiny)).sum() > n // 4
    r = lm.special_scores(n, "runs", 1)
    assert (np.diff(np.flatnonzero(np.diff(r) != 0)) > 1000).any()
    a = lm.special_scores(n, "all", 1)
    for v in np.concatenate([lm.INADMISSIBLE, lm.EDGE_ADMISSIBLE]):
        assert (np.isnan(a).any() if np.isnan(v) else (a.view(np.uint32) == np.float32(v).view(np.uint32)).any()), v
