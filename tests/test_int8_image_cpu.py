"""The int8 image of fp32 shards (scan_tensor_shadow.cu build_image_s8_kernel, filter_prep_kernel) restated in numpy, and
the filter's error bound checked on it.  Per row x ~ xb = s_x xq with s_x = max|x_i| / 127 and xq = round(x / s_x) in
[-127, 127]; the queries the same way.  The estimate is the EXACT integer dot product times the two fp32 scales, so the
BF16 identity x.q - xb.qb = dx.qb + x.dq carries over unchanged:
    |s_hat - s| <= |dx||qb| + |x||dq| + acc_c |x||q|,   acc_c = d 2^-22 + 4e-6
with |dx| = |x - s_x xq| measured in fp32 and inflated by 1.0001, exactly the factors of the BF16 shadow."""
import numpy as np
import pytest

F32 = np.float32


def quantize(x):
    """(s, xq, |x - s xq|^2 in fp32) as the device computes them: s = max|x| / 127 (NaN for a non-finite row),
    xq = clamp(rint(x * (127 / max)), -127, 127) (0 where the product is NaN), residue e = fma(-s, xq, x)."""
    x = np.asarray(x, dtype=F32)
    with np.errstate(invalid="ignore", over="ignore"):
        bad = not np.isfinite(x).all()
        mx = F32(np.abs(x).max()) if x.size else F32(0)
        s = F32(np.nan) if bad else F32(mx / F32(127))
        sinv = F32(0) if bad or not mx > 0 else F32(F32(127) / mx)
        t = (x * sinv).astype(F32)
        xq = np.where(np.isnan(t), 0, np.clip(np.rint(t), -127, 127)).astype(np.int8)
        e = (x.astype(np.float64) - np.float64(s) * xq.astype(np.float64)).astype(F32)  # fma: one rounding of the exact value
        d2 = F32(0)
        for v in e:  # fp32 accumulation (the device's order differs; both are within the 1.0001 inflation)
            d2 = F32(d2 + F32(v * v))
    return s, xq, d2


def estimate(sx, xq, sq, qq):
    """float(exact int32 dot) * s_q * s_x: the three fp32 roundings of the device's estimate."""
    acc = int(xq.astype(np.int64) @ qq.astype(np.int64))
    assert abs(acc) < 2 ** 31
    return float(F32(F32(F32(acc) * sq) * sx))


CASES = ["uniform", "same_sign", "tiny", "huge", "sparse", "outlier"]


def make(case, d, rng):
    x = rng.uniform(-1, 1, d).astype(F32)
    q = rng.uniform(-1, 1, d).astype(F32)
    if case == "same_sign":
        x, q = np.abs(x), np.abs(q)
    elif case == "tiny":
        x, q = x * F32(1e-6), q * F32(3e-6)
    elif case == "huge":
        x, q = x * F32(1e6), q * F32(2e5)
    elif case == "sparse":
        x[rng.random(d) < 0.9] = 0
        q[rng.random(d) < 0.5] = 0
    elif case == "outlier":  # one element per vector dominates the scale: the other elements keep few levels
        x[rng.integers(d)] = F32(40.0)
        q[rng.integers(d)] = F32(-25.0)
    return x.astype(F32), q.astype(F32)


def n64(v):
    return float(np.sqrt((np.asarray(v, np.float64) ** 2).sum()))


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("d", [32, 100, 1024])
def test_int8_image_bound_is_rigorous(case, d):
    rng = np.random.default_rng(d * 13 + CASES.index(case))
    acc_c = d * 2.0 ** -22 + 4e-6
    for _ in range(40):
        x, q = make(case, d, rng)
        sx, xq, dx2 = quantize(x)
        sq, qq, dq2 = quantize(q)
        s = float(x.astype(np.float64) @ q.astype(np.float64))
        s_hat = estimate(sx, xq, sq, qq)
        qb = (sq * qq.astype(F32)).astype(F32)
        ra, rb = float(np.sqrt(dx2)) * 1.0001, n64(x)
        qa, qbnd = n64(qb) * 1.0001, (float(np.sqrt(dq2)) + acc_c * n64(q)) * 1.0001
        bound = ra * qa + rb * qbnd
        assert abs(s_hat - s) <= bound, (case, d, s, s_hat, bound)
        if case == "uniform" and d == 1024:  # useful: a small fraction of |x||q| (about 2.5x the BF16 shadow's)
            assert bound < 2.0 ** -6 * n64(x) * n64(q)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("d", [32, 100, 1024])
def test_fp32_residue_is_within_its_inflation(case, d):
    rng = np.random.default_rng(d * 17 + CASES.index(case))
    for _ in range(20):
        x, _ = make(case, d, rng)
        sx, xq, dx2 = quantize(x)
        exact = n64(x.astype(np.float64) - np.float64(sx) * xq.astype(np.float64))
        assert exact <= float(np.sqrt(dx2)) * 1.0001, (case, d, exact, float(np.sqrt(dx2)))
        assert (np.abs(xq.astype(np.int32)) <= 127).all()
        assert np.abs(xq.astype(np.int32)).max() == 127 or not np.any(x)


def test_accumulator_cannot_overflow_at_the_largest_dimension():
    assert 127 * 127 * 32768 < 2 ** 31


def test_zero_and_non_finite_rows():
    s, xq, d2 = quantize(np.zeros(64, F32))
    assert s == 0 and not xq.any() and d2 == 0
    for bad in (np.nan, np.inf, -np.inf):
        x = np.linspace(-1, 1, 64).astype(F32)
        x[5] = bad
        s, xq, d2 = quantize(x)
        assert np.isnan(s) and not xq.any() and np.isnan(d2)
        # every estimate of such a row is NaN: the keep rule keeps it with bound +inf, the exact re-scoring judges
        assert np.isnan(F32(F32(3.0) * s))
