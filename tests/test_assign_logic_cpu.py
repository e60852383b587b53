"""CPU restatement of the k-means assignment's near-tie logic (assign_tensor.cu, DESIGN §7 item 3): the epilogue's
candidate selection against brute force, the BF16 traps tests/test_gpu_assign.py plants (proved here to invert the BF16
estimate of a score difference), and the fix-up's squaredEuclidean arithmetic against the oracle, bit for bit."""
import numpy as np
import pytest

NONE, ALL = 0xFFFFFFFF, 0xFFFFFFFE
QT = 64
F32_INF = np.float32(np.inf)


# ---- BF16 emulation ---------------------------------------------------------------------------------------------------
def to_bf16_bits(a):
    """Round-to-nearest-even to bf16 (cvt.rn.bf16.f32 / ptx::f32_to_bf16_bits) for finite inputs: the 16 high bits."""
    u = np.asarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF).astype(np.uint16)


def bf16(a):
    return (to_bf16_bits(a).astype(np.uint32) << 16).view(np.float32)


# ---- the epilogue's selection (assign_scan_kernel) ---------------------------------------------------------------------
def thread_columns(q, K):
    """Centroids thread q (lane & 3) of a row scores, in the order it scores them: ci = 64 qbk + 2 q + 8 (jj / 2) + jj % 2."""
    return [ci for qbk in range((K + QT - 1) // QT) for jj in range(QT // 4)
            if (ci := qbk * QT + 2 * q + 8 * (jj >> 1) + (jj & 1)) < K]


def thread_top4(up, cols):
    """Strict insertion of the upper bounds over ascending centroids: equal bounds keep the lower index ahead."""
    u, ids = [-F32_INF] * 4, [NONE] * 4
    for ci in cols:
        if up[ci] > u[3]:
            u[3], ids[3] = up[ci], ci
            for e in (3, 2, 1):
                if u[e] > u[e - 1]:
                    u[e], u[e - 1], ids[e], ids[e - 1] = u[e - 1], u[e], ids[e - 1], ids[e]
    return u, ids


def merge(own, other):
    """One shuffle step: insert the partner's four entries, ordered by (bound desc, centroid asc)."""
    u, ids = list(own[0]), list(own[1])
    for pu, pid in zip(*other):
        if pu > u[3] or (pu == u[3] and pid < ids[3]):
            u[3], ids[3] = pu, pid
            for e in (3, 2, 1):
                if u[e] > u[e - 1] or (u[e] == u[e - 1] and ids[e] < ids[e - 1]):
                    u[e], u[e - 1], ids[e], ids[e - 1] = u[e - 1], u[e], ids[e - 1], ids[e]
    return u, ids


def row_lists(up):
    """The merged list every lane of the row holds after the xor-1 and xor-2 shuffles."""
    K = len(up)
    lists = [thread_top4(up, thread_columns(q, K)) for q in range(4)]
    step1 = [merge(lists[q], lists[q ^ 1]) for q in range(4)]
    step2 = [merge(step1[q], step1[q ^ 2]) for q in range(4)]
    return step2


def decide(u, ids, maxlo, xx):
    """('decided', i0) | ('cand', [i0, i1, i2 or NONE]) | ('all', None), as the epilogue writes the near-tie list."""
    i0, i1, i2 = ids[:3]
    if i0 != NONE and not (u[1] >= maxlo) and xx > 0 and xx < np.inf:
        return "decided", i0
    if i0 == NONE or u[3] >= maxlo or not (xx > 0) or not (xx < np.inf):
        return "all", None
    return "cand", [i0, i1, i2 if u[2] >= maxlo else NONE]


def f32max_lo(lo):
    m = -F32_INF
    for v in lo:  # fmaxf: a NaN operand is ignored
        if v == v and v > m:
            m = v
    return m


def _columns(rng, K, kind):
    """(est, bnd, exact score) per centroid, with exact real-valued scores inside [est - bnd, est + bnd]."""
    est = (rng.integers(-6, 7, K) / 8).astype(np.float32)
    bnd = rng.choice(np.array([0, 1 / 64, 1 / 8, 1 / 4], dtype=np.float32), K)
    true = est.astype(np.float64) + rng.integers(-1, 2, K) * bnd.astype(np.float64) / 2
    if kind == "nan":
        bad = rng.choice(K, max(1, K // 5), replace=False)
        est[bad] = np.nan
        true[bad] = np.nan
    if kind == "neginf":
        bad = rng.choice(K, max(1, K // 5), replace=False)
        est[bad] = -np.inf
        true[bad] = -np.inf
    if kind == "lanes" and K > 2:  # the same top score in two lanes (and in two centroid blocks where K allows)
        est[:] = np.float32(-1.0); bnd[:] = 0; true[:] = -1.0
        pair = [2, 0] if K <= 65 else [65, 1]
        est[pair] = np.float32(0.5); true[pair] = 0.5
    return est, bnd, true


@pytest.mark.parametrize("K", [1, 2, 3, 4, 5, 63, 64, 65, 129, 200])
@pytest.mark.parametrize("kind", ["plain", "nan", "neginf", "lanes"])
def test_epilogue_selection_matches_brute_force_and_keeps_the_winner(K, kind):
    rng = np.random.default_rng(K * 7 + len(kind))
    for trial in range(40):
        est, bnd, true = _columns(rng, K, kind)
        up = (est + bnd).astype(np.float32)
        lo = (est - bnd).astype(np.float32)
        lists = row_lists(list(up))
        assert all(l == lists[0] for l in lists)  # every lane of the row ends with the same list
        u, ids = lists[0]
        # brute force: the four best upper bounds by (bound desc, centroid asc); NaN and -inf never enter
        order = sorted((-float(up[c]), c) for c in range(K) if up[c] > -np.inf)[:4]
        want = [c for _, c in order] + [NONE] * (4 - len(order))
        assert ids == want, (trial, ids, want)
        ml = f32max_lo(lo)
        xx = [1.0, 1.0, 1.0, 0.0, np.inf, np.nan][trial % 6]
        kind_, val = decide(u, ids, ml, xx)
        if not (xx > 0 and xx < np.inf):
            assert kind_ == "all"  # a zero or non-finite row is never decided by the bound
        valid = [c for c in range(K) if true[c] == true[c] and true[c] > -np.inf]
        if not valid:
            assert kind_ == "all"
            continue
        best = max(true[c] for c in valid)
        winner = min(c for c in valid if true[c] == best)  # lowest index among equal scores
        if kind_ == "decided":
            assert val == winner
            assert sum(true[c] == best for c in valid) == 1  # a decided row never has an exact tie
        elif kind_ == "cand":
            assert winner in val
        if kind == "lanes" and K > 2 and kind_ != "all":
            assert kind_ == "cand" and ids[:2] == sorted(ids[:2])  # the tie is listed, lower index first


def test_five_equal_upper_bounds_list_every_centroid():
    up = [np.float32(1.0)] * 5 + [np.float32(-1.0)] * 60
    lists = row_lists(up)
    u, ids = lists[0]
    assert ids == [0, 1, 2, 3]
    assert decide(u, ids, np.float32(1.0), 1.0) == ("all", None)


# ---- BF16 traps (tests/test_gpu_assign.py) -----------------------------------------------------------------------------
TRAP_GAPS = [1e-9, 1e-7, 1e-5, 1e-4]  # exact score gap / (mul |x| |c|); the BF16 residues reach a few 1e-4 of that scale
def cosine_bf16_centroid(c):
    """filter_prep_kernel under cosine: bf16(fp32(c * (1 / sqrtf(|c|^2)))); |c|^2 is exact here (c on the 1/16 grid)."""
    t = np.float32(np.sum(c.astype(np.float64) ** 2))
    inv = np.float32(1) / np.sqrt(t)
    return bf16((c * inv).astype(np.float32))


def trap_pair(rng, d, metric, shift=0.0):
    """Two centroids on the 1/16 grid (bf16-exact, fp32 |c|^2 exact in any order) with the same multiset of elements:
    c_b permutes a quarter (cosine: half; at least 16) of c_a's coordinates, so |c_a| = |c_b| and the score difference is mul x.(c_b - c_a) / |c|.
    Under cosine the elements are +-1: every normalised element is the same bf16 value, so the BF16 estimate of the
    difference is a positive multiple of bf16(x).(c_b - c_a)."""
    while True:
        if metric == "cosine":
            ca = rng.choice(np.array([-1.0, 1.0], np.float32), d)
        else:
            ca = (rng.integers(-15, 16, d) / 16).astype(np.float32)
        S = rng.choice(d, max(16, d // (2 if metric == "cosine" else 4)), replace=False)
        cb = ca.copy()
        cb[S] = ca[rng.permutation(S)]
        if np.count_nonzero(cb - ca) >= 6:
            # a constant shift keeps the multiset equal (and sum (c_b - c_a) = 0), so |c_a| = |c_b| still
            return (ca + np.float32(shift)).astype(np.float32), (cb + np.float32(shift)).astype(np.float32)


def score_diffs(x, ca, cb, metric):
    """(exact, BF16 estimate) of score(c_b) - score(c_a), in fp64 with exact accumulation, and the score scale
    mul |x| |c| (the estimate is what the wgmma products sum to; |c|^2 cancels under euclidean)."""
    x64 = x.astype(np.float64)
    xb = bf16(x).astype(np.float64)
    nc = float(np.sqrt(np.sum(ca.astype(np.float64) ** 2)))
    if metric == "euclidean":
        delta = (cb - ca).astype(np.float64)
        exact, est = 2 * x64 @ delta, 2 * xb @ delta
        scale = 2 * float(np.linalg.norm(x64)) * nc
    else:
        exact = x64 @ (cb - ca).astype(np.float64) / nc
        est = xb @ (cosine_bf16_centroid(cb) - cosine_bf16_centroid(ca)).astype(np.float64)
        scale = float(np.linalg.norm(x64))
    return exact, est, scale


def trap_row(rng, ca, cb, metric, rel_gap):
    """A row x next to c_a and c_b whose exact score prefers c_b by about rel_gap * scale while the BF16 estimate
    prefers c_a.  Where c_a and c_b differ, x holds one bf16 value b (sum (c_b - c_a) = 0, so b contributes nothing) plus
    a rounding residue r_j that points along c_b - c_a, so the estimate undercounts x.(c_b - c_a) by
    sum |r_j (c_b - c_a)_j|; one coordinate then tunes the exact difference to the wanted gap."""
    d = ca.size
    delta = (cb - ca).astype(np.float64)
    nz = np.nonzero(delta)[0]
    j1 = int(nz[np.argmin(np.abs(delta[nz]))])  # the tuning coordinate moves by sum |r_j delta_j| / |delta_j1|
    for _ in range(50):
        y = ca.astype(np.float64) + rng.normal(0, 0.05, d)
        y[delta != 0] = float(bf16(np.float32(np.mean(ca) + 0.75)))
        b = bf16(y.astype(np.float32)).astype(np.float64)
        e = np.floor(np.log2(np.maximum(np.abs(b), 2.0 ** -100)))
        s = np.where(delta != 0, np.sign(delta), rng.choice([-1.0, 1.0], d))
        x = (b + s * rng.uniform(0.3, 0.45, d) * 2.0 ** (e - 8)).astype(np.float32)  # |r| < half the bf16 spacing
        assert (bf16(x) == b.astype(np.float32)).all()
        nc = float(np.sqrt(np.sum(ca.astype(np.float64) ** 2)))
        mul = 2.0 if metric == "euclidean" else 1.0 / nc
        scale = score_diffs(x, ca, cb, metric)[2]
        rest = float(np.delete(x.astype(np.float64), j1) @ np.delete(delta, j1))
        x[j1] = np.float32((rel_gap * scale / mul - rest) / delta[j1])
        for _ in range(64):  # nudge by ulps until the exact difference is positive
            exact, est, _ = score_diffs(x, ca, cb, metric)
            if exact > 0:
                break
            x[j1] = np.nextafter(x[j1], np.float32(np.sign(delta[j1]) * np.inf))
        exact, est, scale = score_diffs(x, ca, cb, metric)
        # an inversion the fp32 MMA accumulation cannot undo at d <= 4096 would need |est| > d 2^-24 scale; the claim
        # proved here is the BF16 rounding's, with exact accumulation
        if exact > 0 and est < 0:
            return x, exact / scale
    raise AssertionError("no trap found")


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("d", [32, 36, 96, 1024, 4096])
def test_traps_invert_the_bf16_estimate(metric, d):
    rng = np.random.default_rng(d + (metric == "cosine"))
    for rel in TRAP_GAPS:
        ca, cb = trap_pair(rng, d, metric)
        x, got = trap_row(rng, ca, cb, metric, rel)
        exact, est, scale = score_diffs(x, ca, cb, metric)
        assert exact > 0 > est  # c_b is nearer, the BF16 estimate says c_a
        # the gap is what was asked for up to the tuning coordinate's fp32 step
        assert got <= max(rel * 1.1, 1e-7)
        # and it is below the residue term of the scan's bound (|x - bf16(x)| |c| per centroid): never decided
        dx = float(np.linalg.norm(x.astype(np.float64) - bf16(x).astype(np.float64)))
        nc = float(np.linalg.norm(ca.astype(np.float64)))
        mul = 2.0 if metric == "euclidean" else 1.0 / nc
        assert exact < 2 * mul * dx * nc


# ---- the fix-up's arithmetic (assign_fixup_kernel) ---------------------------------------------------------------------
def sq_euclid64_np(x, c):
    """squaredEuclidean as assign_fixup_kernel computes it: fp32 differences, fp64 squares in four interleaved sums,
    the tail into s0, then ((s0 + s1) + s2) + s3."""
    dlt = (np.asarray(x, np.float32) - np.asarray(c, np.float32)).astype(np.float64)
    n = dlt.size
    s = [0.0, 0.0, 0.0, 0.0]
    m = n - n % 4
    for j in range(0, m, 4):
        for t in range(4):
            s[t] = s[t] + dlt[j + t] * dlt[j + t]
    for j in range(m, n):
        s[0] = s[0] + dlt[j] * dlt[j]
    return ((s[0] + s[1]) + s[2]) + s[3]


@pytest.mark.parametrize("d", [1, 3, 4, 5, 32, 36, 97, 1024])
def test_fixup_arithmetic_is_the_oracles_bit_for_bit(oracle_mod, d):
    rng = np.random.default_rng(d)
    for scale in [1e-20, 1.0, 1e3, 1e19]:
        x = (rng.standard_normal(d) * scale).astype(np.float32)
        c = (x + rng.standard_normal(d).astype(np.float32) * np.float32(scale * 1e-3)).astype(np.float32)
        got, want = sq_euclid64_np(x, c), oracle_mod.sq_euclid64(x, c)
        assert got == want or (got != got and want != want), (scale, got, want)
    # a finite row whose fp32 |x|^2 overflows: the fp64 sums stay finite and keep the order
    x = np.full(d, 1e20, np.float32)
    assert np.isinf(np.float32(np.sum(x.astype(np.float32) ** 2))) or d == 0
    near, far = np.full(d, 9e19, np.float32), np.full(d, 5e19, np.float32)
    assert sq_euclid64_np(x, near) == oracle_mod.sq_euclid64(x, near) < oracle_mod.sq_euclid64(x, far)
