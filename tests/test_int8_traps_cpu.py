"""Rank-inversion traps for the int8 filter scan (scan_tensor_shadow.cu, Opnd::S8), built and proven decisive on the host.

The int8 image is the one filter image whose estimate is exactly predictable off the device: the s32 accumulation is exact
and the estimate is fl(fl(float(acc) s_q) mul).  So rows can be planted whose estimate is wrong by almost exactly the
error bound, in a chosen direction:

  * a trap row of query q is x = s (127 e_0 + (u + sigma a) g), g = sign(q) (g_0 = 0), u a non-negative integer code, s a
    power of two and 0.40 <= a < 0.5: x quantizes to exactly s (127 e_0 + u g), its residue s a g points along q, and
    the estimate misses the true score by |dx||q|, about 0.99 of the bound (the rest is the fp32 accumulation allowance);
  * TARGETS (sigma = +1) are the true top k of their query but sit one bound low; DECOYS (sigma = -1) score just below
    the targets but sit one bound high.  The true gaps run from 2e-5 of the score scale to half the bound;
  * background and crowd rows are exact int8 codes (zero residue), so the per-CTA bound maxima B_max are the traps'.

test_gpu_int8_traps.py runs the device on these fixtures; here the replica shows that each fixture decides: ranking by
the estimate loses every target, a prune or finish margin of one bound instead of two loses one per query, and a range
threshold lies between each target's estimate and its upper bound."""
import math

import numpy as np
import pytest

from test_int8_image_cpu import quantize

F32 = np.float32
EUC_EPS = 4e-6
EUC_KEEP = float(F32(1.0) - F32(EUC_EPS))
TILE = 256
S_TRAP, S_BG = 2.0 ** -4, 2.0 ** -5  # row scales (powers of two: the int8 image of a trap row is exact)
GAPS = [0.5, 0.25, 0.1, 0.03, 0.01, 3e-3, 1e-3, 3e-4, 1e-4, 0.0]  # target - best decoy, in bounds (0: the 2e-5 floor)
GAP_FLOOR = 2e-5  # of the score scale: far above fp32 re-scoring noise


# ---------------------------------------------------------------------------------------------------- host replica
def acc_c(d):
    return float(F32(F32(d) * F32(2.384185791015625e-7) + F32(4e-6)))


def quantize_rows(x):
    """quantize() of every row of x at once: (s, xq)"""
    x = np.asarray(x, F32)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        bad = ~np.isfinite(x).all(1)
        mx = np.abs(x).max(1).astype(F32)
        s = np.where(bad, F32(np.nan), mx / F32(127)).astype(F32)
        sinv = np.where(bad | ~(mx > 0), F32(0), F32(127) / mx).astype(F32)
        t = (x * sinv[:, None]).astype(F32)
        xq = np.where(np.isnan(t), 0, np.clip(np.rint(t), -127, 127)).astype(np.int8)
    return s, xq


def _fma_sq(a, acc):
    """fmaf(a, a, acc) in fp32: one rounding of the exact value (a^2 is exact in the 64-bit long double)"""
    a = np.asarray(a, np.longdouble)
    return (a * a + np.asarray(acc, np.longdouble)).astype(F32)


def _butterfly(v):
    """the warp's xor-shuffle sum (offsets 16 .. 1) over the last axis (32 lanes): lane 0's value"""
    v = np.asarray(v, F32)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., lanes ^ o]).astype(F32)
    return v[..., 0]


def _row_sum_sq(vals):
    """sum of squares of each row as build_image_s8_kernel accumulates it: lane l takes elements 128 t + 4 l .. + 3 in
    order (fmaf), then the butterfly"""
    n, w = vals.shape
    v = np.zeros((n, (w + 127) // 128 * 128), F32)
    v[:, :w] = vals
    v = v.reshape(n, -1, 32, 4)
    acc = np.zeros((n, 32), F32)
    for t in range(v.shape[1]):
        for e in range(4):
            acc = _fma_sq(v[:, t, :, e], acc)
    return _butterfly(acc)


def _prep_sum_sq(vals):
    """sum of squares of each query as filter_prep_kernel accumulates it: thread i of 1024 takes elements i, i + 1024, ..
    (fmaf), each warp's butterfly, then the 32 warp sums in order"""
    n, w = vals.shape
    v = np.zeros((n, (w + 1023) // 1024 * 1024), F32)
    v[:, :w] = vals
    v = v.reshape(n, -1, 1024)
    acc = np.zeros((n, 1024), F32)
    for t in range(v.shape[1]):
        acc = _fma_sq(v[:, t], acc)
    red = _butterfly(acc.reshape(n, 32, 32))
    tot = np.zeros(n, F32)
    for i in range(32):
        tot = (tot + red[:, i]).astype(F32)
    return tot


def row_image(rows):
    """Per row (s_x, xq, |x|^2, |x - s_x xq|^2) of build_image_s8_kernel, the sums in the device's order."""
    rows = np.asarray(rows, F32)
    xs, xq = quantize_rows(rows)
    e = (rows.astype(np.float64) - xs.astype(np.float64)[:, None] * xq.astype(np.float64)).astype(F32)  # fmaf(-s, q, x)
    return xs, xq, _row_sum_sq(rows), _row_sum_sq(e)


def query_prep(q, metric):
    """filter_prep_kernel for an int8 image: (s_q, qq, qa, qb, qn) per query, cosine queries normalised first; the sums
    in the device's order."""
    q = np.asarray(q, F32)
    d = q.shape[1]
    t = _prep_sum_sq(q)
    nrm = np.sqrt(t).astype(F32)
    if metric == "cosine":
        with np.errstate(divide="ignore"):
            inv = np.where(t > 0, F32(1) / nrm, F32(0)).astype(F32)
        qn = np.where(t > 0, F32(1), F32(0)).astype(F32)
    else:
        inv = np.ones_like(t)
        qn = nrm
    v = (q * inv[:, None]).astype(F32)
    sq, qq = quantize_rows(v)
    vb = (sq[:, None] * qq.astype(F32)).astype(F32)
    e = (v.astype(np.float64) - sq.astype(np.float64)[:, None] * qq.astype(np.float64)).astype(F32)
    hh, dd = _prep_sum_sq(vb), _prep_sum_sq(e)
    qa = (np.sqrt(hh) * F32(1.0001)).astype(F32)
    qb = (fma32(F32(acc_c(d)), qn, np.sqrt(dd)) * F32(1.0001)).astype(F32)  # (the compiler contracts a * b + c)
    return dict(sq=sq, qq=qq, qa=qa, qb=qb, qn=qn)


def row_factors(img, metric):
    """(mul, ra, rb) of Bf16Est for each row of an int8 image (scan_tensor_shadow.cu)."""
    xs, _, x2, d2 = img
    xn = np.sqrt(x2).astype(F32)
    dxn = (np.sqrt(d2) * F32(1.0001)).astype(F32)
    if metric == "cosine":
        with np.errstate(divide="ignore"):
            mul = np.where(x2 > 0, F32(1) / xn, F32(0)).astype(F32)
        ra = (dxn * mul * F32(1.000001)).astype(F32)
        rb = np.ones_like(xn)
    elif metric == "euclidean":
        mul, ra, rb = np.full_like(xn, 2), (F32(2) * dxn).astype(F32), (F32(2) * xn).astype(F32)
    else:
        mul, ra, rb = np.ones_like(xn), dxn, xn
    return (mul * xs).astype(F32), ra, rb


def fma32(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


def scan_values(img, qp, metric):
    """[rows x Q] (est, bound, upper) of the int8 scan: est and bound as the DUMP instantiation writes them, upper as the
    keep rule compares it (Bf16Est::upper, EUC_KEEP included)."""
    _, xq, x2, _ = img
    mul, ra, rb = row_factors(img, metric)
    acc = xq.astype(np.float64) @ qp["qq"].astype(np.float64).T  # exact: |acc| < 2^31 < 2^53
    v = (acc.astype(F32) * qp["sq"][None, :]).astype(F32)
    bnd = fma32(ra[:, None], qp["qa"][None, :], (rb[:, None] * qp["qb"][None, :]).astype(F32))
    est = (v * mul[:, None]).astype(F32)
    upper = fma32(v, mul[:, None], bnd)
    if metric == "euclidean":
        qx = fma32(qp["qn"][None, :], qp["qn"][None, :], x2[:, None])
        est = (est - qx).astype(F32)
        bnd = (bnd + F32(EUC_EPS) * qx).astype(F32)
        upper = (upper - F32(EUC_KEEP) * qx).astype(F32)
    return est, bnd, upper


def margin2(metric, max_ra, max_rb, maxxx, qa, qb, qn):
    """bf16_margin2: twice the largest bound of the rows seen (cosine: max_rb = 1)."""
    m = F32(2) * fma32(max_ra, qa, F32(max_rb) * qb)
    if metric == "euclidean":
        m = m + F32(2) * F32(EUC_EPS) * (F32(maxxx) + qn * qn)
    return np.asarray(m, F32)


def exact_keys(rows, q, metric):
    """fp64 key-space score [rows x Q] (cosine / dot: the score; euclidean: -distance^2)."""
    x = np.asarray(rows, np.float64)
    qq = np.asarray(q, np.float64)
    dots = x @ qq.T
    if metric == "dot":
        return dots
    xn = (x * x).sum(1)[:, None]
    qn = (qq * qq).sum(1)[None, :]
    if metric == "cosine":
        den = np.sqrt(xn * qn)
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.where(den > 0, dots / den, 0.0)
    return 2.0 * dots - xn - qn


def api_score(key, metric):
    """key-space score -> what the API returns (euclidean: the distance)"""
    return np.sqrt(np.maximum(-key, 0.0)) if metric == "euclidean" else key


def ri_of(pos):
    """accumulator fragment row of a tile row: rows rbase + 64 (ri >> 1) + 8 (ri & 1), rbase = 128 m + 16 wq + lane / 4"""
    r = pos % TILE
    return ((r >> 3) & 1) | (((r >> 6) & 1) << 1)


# ---------------------------------------------------------------------------------------------------- fixtures
def _sign_queries(rng, Q, d):
    """Q sign-vector queries (exact in int8): coordinate 0 is 0, a spine of (d-1)/2 coordinates is +1 in every query,
    the rest random; scales 2 and 4 alternate (distinct int8 scales in neighbouring columns)."""
    g = np.zeros((Q, d), np.int64)
    h = (d - 1) // 2
    g[:, 1:1 + h] = 1
    g[:, 1 + h:] = rng.choice([-1, 1], size=(Q, d - 1 - h))
    c = np.where(np.arange(Q) % 2 == 0, 2.0, 4.0)
    return g, c


def _keys_closed(metric, A, B2, a, D, c):
    """Key of a trap row s (127 e_0 + (u + a) g) for its own query c g, from A = sum(u), B2 = sum(u^2) (fp64)."""
    s = S_TRAP
    sw = A + a * D
    sw2 = B2 + 2 * a * A + a * a * D
    if metric == "dot":
        return s * c * sw
    if metric == "cosine":
        return sw / (math.sqrt(D) * np.sqrt(127.0 ** 2 + sw2))
    return 2 * s * c * sw - s * s * (127.0 ** 2 + sw2) - c * c * D


def _trap_row(code, a, g):
    x = np.zeros(g.shape[0], F32)
    x[0] = F32(127 * S_TRAP)
    x[1:] = (F32(S_TRAP) * (code[1:].astype(F32) + F32(a)).astype(F32) * g[1:].astype(F32)).astype(F32)
    return x


def _targets_for(metric, U, g, c, want_keys, rng):
    """Codes u = U + 1_T and shifts a (in [0.40, 0.495]) whose keys hit want_keys (one target each)."""
    D = U.size - 1
    order = np.argsort(U[1:], kind="stable") + 1  # the extra units go to the smallest codes first
    u = U[order].astype(np.float64)
    A = float(U[1:].sum()) + np.arange(D + 1)
    B2 = float((U[1:].astype(np.float64) ** 2).sum()) + np.concatenate([[0.0], np.cumsum(2 * u + 1)])
    reach = _keys_closed(metric, A, B2, 0.495, D, c)
    rows = []
    for wk in want_keys:
        ok = np.nonzero(reach >= wk)[0]
        assert ok.size, "target key out of reach"
        m = int(ok[0])
        A_m, B_m = A[m], B2[m]
        lo, hi = 0.40, 0.495
        assert _keys_closed(metric, A_m, B_m, lo, D, c) <= wk, "target key out of reach"
        for _ in range(60):
            mid = 0.5 * (lo + hi)
            if _keys_closed(metric, A_m, B_m, mid, D, c) < wk:
                lo = mid
            else:
                hi = mid
        code = U.copy()
        code[order[:m]] += 1
        rows.append(_trap_row(code, hi, g))
    return rows


class Fixture:
    """rows, queries, k, metric, and per query the target and decoy row ids; .role: 0 background, 1 target, 2 decoy,
    3 crowd, 4 a stored query (.owner: the query of a trap row)."""


def make_fixture(metric, d, Q, k, n, seed, place="spread", crowd_tile=None, n_decoys=None):
    """place: "spread": trap rows at stride 257 over the shard (every row position mod 256, the first and the last
    partial tile); "sampled": the decoys on the prep's sampled rows i n / S, the targets at fragment rows ri != 0 whose
    thread's row ri = 0 is a background row; "crowd": every trap row in tile crowd_tile at ri != 0, the tile's other rows
    a crowd above the sampled threshold and below the traps; "split": targets in one tile, decoys in another.
    n_decoys: decoys per query (default k)."""
    rng = np.random.default_rng(seed)
    nd = k if n_decoys is None else n_decoys
    g, c = _sign_queries(rng, Q, d)
    q = (g * c[:, None]).astype(F32)
    D = d - 1
    # background: exact codes, negative on the spine, far below every trap for every metric
    h = D // 2
    bg = np.zeros((n, d), np.int64)
    bg[:, 0] = 127
    bg[:, 1:1 + h] = -60 + rng.integers(-4, 5, (n, h))
    bg[:, 1 + h:] = rng.integers(-30, 31, (n, D - h))
    rows = (bg.astype(F32) * F32(S_BG)).astype(F32)
    role = np.zeros(n, np.int8)
    owner = np.full(n, -1, np.int64)

    # trap positions
    n_traps = Q * (k + nd)
    if place == "spread":
        assert math.gcd(257, n) == 1 and n_traps <= n
        tpos = [(t * 257) % n for t in range(Q * k)]
        dpos = [((Q * k + t) * 257) % n for t in range(Q * nd)]
    elif place == "sampled":
        S = min(max(1 << (8 * k - 1).bit_length(), 128), 2048)
        samp = [i * n // S for i in range(S)]
        assert Q * nd <= S
        dpos = samp[:Q * nd]
        taken = set(samp)
        tpos = []
        for p in range(TILE, n):
            # ri != 0 whose ri = 0 partner row (same thread) holds a background row
            if len(tpos) == Q * k:
                break
            ri = ri_of(p)
            mate = p - 8 * (ri & 1) - 64 * (ri >> 1)
            if ri and p not in taken and mate not in taken and ri_of(mate) == 0 and p % 3 == 0:
                tpos.append(p)
                taken.add(p)
        assert len(tpos) == Q * k
    elif place == "crowd":
        base = crowd_tile * TILE
        slots = [base + r for r in range(TILE) if ri_of(r) != 0]
        assert n_traps <= len(slots)
        tpos, dpos = slots[:Q * k], slots[Q * k:n_traps]
        crowd = [base + r for r in range(TILE) if base + r not in set(tpos) | set(dpos)]
        cc = np.zeros((len(crowd), d), np.int64)
        cc[:, 0] = 127
        cc[:, 1:1 + h] = 4
        rows[crowd] = (cc.astype(F32) * F32(S_TRAP)).astype(F32)
        role[crowd] = 3
    elif place == "split":
        tpos = [3 * TILE + i * 3 for i in range(Q * k)]
        dpos = [(n // TILE - 2) * TILE + i * 3 for i in range(Q * nd)]
        assert max(Q * k, Q * nd) * 3 <= TILE
    else:
        raise ValueError(place)
    assert len(set(tpos) | set(dpos)) == n_traps

    targets, decoys = [], []
    n1 = round(0.9 * D)
    for j in range(Q):
        U = np.zeros(d, np.int64)
        U[1:] = np.clip(8 + np.rint(rng.normal(0, 3, D)), 1, 40).astype(np.int64)
        # decoys: u = U + 1 on n1 random coordinates, shifted -a_d: true key just below the targets, estimate one bound high.
        # One code per query, a_d spread over [0.44, 0.46]: the decoys' true keys are distinct and ordered by a_d, so a
        # filter that lets some decoys into the top k leaves no near-tie at the k-th
        code = U.copy()
        code[1 + rng.permutation(D)[:n1]] += 1
        drows = []
        for r in range(nd):
            a_d = 0.45 + 0.02 * ((r + 0.5) / nd - 0.5)
            x = np.zeros(d, F32)
            x[0] = F32(127 * S_TRAP)
            x[1:] = (F32(S_TRAP) * (code[1:].astype(F32) - F32(a_d)).astype(F32) * g[j, 1:].astype(F32)).astype(F32)
            drows.append(x)
        dk = exact_keys(np.array(drows), q[j:j + 1], metric)[:, 0]
        top = dk.max()
        # the bound at the traps in key units: |dx||q| with |dx| = 0.45 s sqrt(D) (cosine: over |x|; euclidean: twice)
        if metric == "cosine":
            bscale = 0.45 * math.sqrt(D / (127.0 ** 2 + float((U[1:] ** 2).sum())))
        else:
            bscale = 0.45 * S_TRAP * D * c[j] * (2.0 if metric == "euclidean" else 1.0)
        scale = 1.0 if metric == "cosine" else abs(top)
        want = [top + max(GAPS[t % len(GAPS)] * bscale, GAP_FLOOR * scale) for t in range(k)]
        trows = _targets_for(metric, U, g[j], c[j], want, rng)
        ids_t = tpos[j * k:(j + 1) * k]
        ids_d = dpos[j * nd:(j + 1) * nd]
        rows[ids_t] = np.array(trows)
        rows[ids_d] = np.array(drows)
        role[ids_t], role[ids_d] = 1, 2
        owner[ids_t] = owner[ids_d] = j
        targets.append(np.array(ids_t))
        decoys.append(np.array(ids_d))
    f = Fixture()
    f.metric, f.d, f.Q, f.k, f.n, f.place = metric, d, Q, k, n, place
    f.rows, f.q, f.role, f.owner = rows, q, role, owner
    f.targets, f.decoys = targets, decoys
    return f


def replica(f):
    """(exact keys, est, bound, upper) [rows x Q] of the int8 scan on fixture f (cached)."""
    if not hasattr(f, "_rep"):
        img = row_image(f.rows)
        qp = query_prep(f.q, f.metric)
        est, bnd, upper = scan_values(img, qp, f.metric)
        _, ra, rb = row_factors(img, f.metric)
        f._rep = (exact_keys(f.rows, f.q, f.metric), est, bnd, upper, qp, img, ra, rb)
    return f._rep


def range_thresholds(f):
    """Key-space threshold per query halfway between its best decoy and its worst target (true scores)."""
    ex = replica(f)[0]
    return np.array([0.5 * (ex[f.decoys[j], j].max() + ex[f.targets[j], j].min()) for j in range(f.Q)])


def api_thresholds(f):
    """range_thresholds as search_range takes them (euclidean: a distance), and their key-space value after fp32."""
    t = range_thresholds(f)
    if f.metric == "euclidean":
        dist = np.sqrt(-t).astype(F32)
        return dist, -(dist.astype(np.float64) ** 2)
    t32 = t.astype(F32)
    return t32, t32.astype(np.float64)


def check_decisive(f, rng_check=False, exclude=(), admit=None):
    """The fixture's traps decide: asserts what the module docstring promises, with the replica's numbers.  exclude: rows
    the search leaves out (search_rows: the query's own row).  admit: [rows x Q] per-query tag filter (a search then
    ranks the admitted rows only; its true top k are the admitted targets and the best admitted decoys)."""
    ex, est, bnd, upper, qp, img, ra, rb = replica(f)
    keep = np.setdiff1d(np.arange(f.n), exclude)
    ex, est, bnd, upper = ex[keep], est[keep], bnd[keep], upper[keep]
    ra, rb, x2 = ra[keep], rb[keep], img[2][keep]
    adm = np.ones((keep.size, f.Q), bool) if admit is None else np.asarray(admit)[keep]
    pos = np.full(f.n, -1)
    pos[keep] = np.arange(keep.size)
    targets, decoys, role = [pos[t] for t in f.targets], [pos[dc] for dc in f.decoys], f.role[keep]
    n = keep.size
    k = f.k
    # B_max: the largest bound of any row a CTA sees (filters do not change it) is a trap's: every other row is exact
    assert np.isin(role[ra == ra.max()], (1, 2)).all()
    for j in range(f.Q):
        t, dc = targets[j][adm[targets[j], j]], decoys[j][adm[decoys[j], j]]
        assert t.size and dc.size >= k, ("the filter leaves too few traps to decide", j)
        rows_j = np.nonzero(adm[:, j])[0]
        others = np.setdiff1d(rows_j, np.concatenate([t, dc]))
        # the true top k are the admitted targets (and, under a filter, the best admitted decoys), with gaps far above
        # fp32 re-scoring noise, at the targets and at the k-th
        scale = 1.0 if f.metric == "cosine" else float(np.abs(ex[t, j]).max())
        assert ex[t, j].min() - ex[dc, j].max() >= 0.9 * GAP_FLOOR * scale, ("gap", j)
        srt = np.sort(ex[rows_j, j])[::-1]
        assert srt[k - 1] - srt[k] >= 0.9 * GAP_FLOOR * scale, ("near-tie at the k-th", j)
        assert ex[others, j].max() < ex[dc, j].min(), ("background above a decoy", j)
        # every target's estimate is below the k-th largest estimate: ranking by the estimate loses it
        kth_est = np.sort(est[rows_j, j])[::-1][k - 1]
        assert (est[t, j] < kth_est).all(), ("a target's estimate reaches the k-th estimate", j)
        # the estimate misses the true score by most of the bound, in the chosen direction
        assert ((ex[t, j] - est[t, j]) > 0.9 * bnd[t, j]).all() and ((est[dc, j] - ex[dc, j]) > 0.9 * bnd[dc, j]).all(), j
        # a margin of one bound loses a target: upper < U_k - B_max
        uk = np.sort(upper[rows_j, j])[::-1][k - 1]
        max_rb = 1.0 if f.metric == "cosine" else rb.max()
        m2 = float(margin2(f.metric, ra.max(), max_rb, x2.max(), qp["qa"][j], qp["qb"][j], qp["qn"][j]))
        assert (upper[t, j] < uk - 0.5 * m2).any(), ("no target lost by a one-bound margin", j)
        # ... and the true two-bound margin keeps every target
        assert (upper[t, j] >= uk - m2).all(), j
        # every row outside the query's traps lies below the margin: the traps alone decide
        assert upper[others, j].max() < uk - m2, ("a background row inside the margin", j)
    if rng_check:
        _, thr_key = api_thresholds(f)
        for j in range(f.Q):
            t, dc = targets[j], decoys[j]
            assert (est[t, j] < thr_key[j]).all() and (thr_key[j] <= upper[t, j]).all() and (ex[t, j] >= thr_key[j]).all(), j
            assert (est[dc, j] >= thr_key[j]).all() and (thr_key[j] > ex[dc, j]).all(), j
            others = np.setdiff1d(np.arange(n), np.concatenate([t, dc]))
            assert upper[others, j].max() < thr_key[j], j


# The fixtures of test_gpu_int8_traps.py.  kNN: (metric, d, Q, k); Q = 300 runs QT = 128 in several query groups without
# a sampled threshold (the flood tiles' prunes decide)
KNN = [(m, d, Q, k) for m in ("cosine", "dot", "euclidean")
       for d, Q, k in ((36, 1, 1), (100, 64, 10), (1024, 128, 16), (100, 300, 10))] + [("cosine", 100, 64, 100)]


def knn_fixture(metric, d, Q, k):
    return make_fixture(metric, d, Q, k, n=max(20_100, 3 * Q * k + 300) | 1, seed=d * 1000 + Q * 7 + k)


def sampled_fixture(metric):
    return make_fixture(metric, 100, 4, 10, n=8001, seed=11, place="sampled")


def crowd_fixture(metric):
    return make_fixture(metric, 100, 3, 10, n=8001, seed=12, place="crowd", crowd_tile=5)


def split_fixture(metric):
    return make_fixture(metric, 100, 8, 10, n=20_001, seed=13, place="split")


def range_fixture(metric, d=100):
    return make_fixture(metric, d, 16, 10, n=12_001, seed=14 + d)


def filtered_fixture(metric):
    """range_fixture's layout with two decoys per target: a filter that refuses a third of a query's traps still leaves
    more than k admitted decoys above its targets' upper bounds"""
    return make_fixture(metric, 100, 16, 10, n=12_001, seed=16, n_decoys=20)


def tagged(f):
    """row tags 1 << (row % 3); even queries refuse tag 1 (a third of their targets and decoys: decoys enter the filtered
    top k), odd queries admit every row -> per-query filters [Q x 3] (all_of, none_of, any_of)"""
    f.tags = (np.uint64(1) << (np.arange(f.n) % 3).astype(np.uint64)).astype(np.uint64)
    filt = np.zeros((f.Q, 3), np.uint64)
    filt[::2, 1] = 1
    return filt


def admits(tags, filters):
    """[rows x Q]: row tag admitted by each query's filter (all_of, none_of, any_of)"""
    t = np.asarray(tags, np.uint64)[:, None]
    a, n, y = (np.asarray(filters, np.uint64)[:, i][None, :] for i in range(3))
    return ((t & a) == a) & ((t & n) == 0) & ((y == 0) | ((t & y) != 0))


def graph_fixture(metric, filtered):
    """k-NN graph update (k = 1): old rows = background, a trap row t, its neighbour p and (filtered) a blocker b; the
    appended row A is t's query exactly (a sign vector, exact in int8).  K(t, A) exceeds t's threshold K(t, p) by half a
    bound, so A belongs in t's list, while the int8 estimate of (t, A) sits one bound low: below the threshold, its upper
    bound above it.  Filtered graphs: b, nearer to t than A, carries tag 2 while every row's filter asks for tag 1, so
    only the row-side filter makes t's threshold K(t, p)."""
    rng = np.random.default_rng(31 + ("cosine", "dot", "euclidean").index(metric) + 7 * filtered)
    d, n_old, T_, P_, B_ = 100, 1500, 700, 1200, 300
    D = d - 1
    g, c = _sign_queries(rng, 1, d)
    A = (g[0] * c[0]).astype(F32)
    h = D // 2
    bg = np.zeros((n_old, d), np.int64)
    bg[:, 0] = 127
    bg[:, 1:1 + h] = -60 + rng.integers(-4, 5, (n_old, h))
    bg[:, 1 + h:] = rng.integers(-30, 31, (n_old, D - h))
    rows = (bg.astype(F32) * F32(S_BG)).astype(F32)
    U = np.zeros(d, np.int64)
    U[1:] = np.clip(8 + np.rint(rng.normal(0, 3, D)), 1, 40).astype(np.int64)
    t = _trap_row(U, 0.45, g[0])
    rows[T_] = t
    bnd = scan_values(row_image(t[None]), query_prep(A[None], metric), metric)[1][0, 0]
    K = exact_keys(t[None], A[None], metric)[0, 0]
    want = K - 0.5 * float(bnd)
    t64, a64 = t.astype(np.float64), A.astype(np.float64)

    def ortho(*vs):  # a random unit vector orthogonal to vs
        basis = np.linalg.qr(np.stack(vs, 1))[0]
        z = rng.standard_normal(d)
        z -= basis @ (basis.T @ z)
        return z / np.linalg.norm(z)
    z = ortho(t64, a64)
    na = np.linalg.norm(a64)
    if metric == "cosine":
        p = a64 + na * math.sqrt((K / want) ** 2 - 1.0) * z
    elif metric == "dot":
        p = (want / K) * a64 + 0.3 * na * z
    else:
        p = a64 + math.sqrt(K - want) * z
    rows[P_] = p.astype(F32)
    tags = np.ones(n_old + 1, np.uint64)
    if filtered:
        zb = ortho(t64, a64, z)
        rows[B_] = ((1.5 if metric == "dot" else 1.0) * t64 + 0.1 * np.linalg.norm(t64) * zb).astype(F32)
        tags[B_] = 2
    f = Fixture()
    f.metric, f.d, f.k, f.n_old, f.t, f.p, f.b = metric, d, 1, n_old, T_, P_, (B_ if filtered else None)
    f.rows = np.concatenate([rows, A[None]])
    f.n = n_old + 1
    f.tags = tags
    f.filters = np.tile(np.array([[1, 0, 0]], np.uint64), (f.n, 1)) if filtered else None
    return f


def graph_want(f):
    """fp64 k-NN graph of every current row of a graph fixture: (idx, key) [n x k], own row left out, each row's list
    bounded by its own filter"""
    ex = exact_keys(f.rows, f.rows, f.metric)
    np.fill_diagonal(ex, -np.inf)
    if f.filters is not None:
        ex[~admits(f.tags, f.filters).T] = -np.inf  # [row r, candidate j]: j's tag admitted by r's filter
    idx = np.empty((f.n, f.k), np.int64)
    for r in range(f.n):
        idx[r] = np.lexsort((np.arange(f.n), -ex[r]))[:f.k]
    return idx, np.take_along_axis(ex, idx, 1)


def check_graph_decisive(f):
    """A belongs in t's list (K(t, A) above t's threshold, by a gap far above noise), yet the int8 estimate of the pair
    is below the threshold and only its upper bound reaches it; without the row filter (filtered fixtures) A would not
    enter t's list"""
    A = f.n_old
    ex = exact_keys(f.rows, f.rows, f.metric)
    old = np.setdiff1d(np.arange(f.n_old), [f.t] + ([f.b] if f.b is not None else []))
    assert ex[f.t, f.p] == ex[f.t, old[old != f.t]].max()  # t's admitted neighbour among the old rows is p
    thr = ex[f.t, f.p]
    est, bnd, upper = scan_values(row_image(f.rows[:f.n_old]), query_prep(f.rows[A:], f.metric), f.metric)
    assert est[f.t, 0] < thr <= ex[f.t, A] <= upper[f.t, 0], (est[f.t, 0], thr, ex[f.t, A], upper[f.t, 0])
    assert thr - est[f.t, 0] > 0.3 * bnd[f.t, 0] and upper[f.t, 0] - thr > 0.3 * bnd[f.t, 0]
    scale = 1.0 if f.metric == "cosine" else abs(ex[f.t, A])
    assert ex[f.t, A] - thr > 100 * GAP_FLOOR * scale
    if f.b is not None:
        assert ex[f.t, f.b] > ex[f.t, A]  # unfiltered, b would hold t's list
    wi, _ = graph_want(f)
    assert wi[f.t, 0] == A


def anchor_fixture(metric):
    """one query stored as row 0 (an exact int8 code): the query of search_rows and the left row of search_pairs"""
    f = make_fixture(metric, 100, 1, 10, n=8001, seed=15, place="split")
    f.rows[0] = f.q[0]
    f.role[0] = 4
    return f


# ---------------------------------------------------------------------------------------------------- tests
def test_replica_estimate_matches_the_scalar_restatement():
    rng = np.random.default_rng(0)
    rows = rng.standard_normal((50, 100)).astype(F32)
    q = (rng.standard_normal((6, 100)) * np.array([[1], [3], [0.1], [7], [1e-3], [50]])).astype(F32)
    est = scan_values(row_image(rows), query_prep(q, "dot"), "dot")[0]
    from test_int8_image_cpu import estimate
    for i in range(50):
        sx, xq, _ = quantize(rows[i])
        for j in range(6):
            sq, qq, _ = quantize(q[j])
            assert est[i, j] == F32(estimate(sx, xq, sq, qq))


def test_trap_rows_quantize_exactly():
    f = make_fixture("dot", 36, 2, 3, n=1001, seed=1)
    img = row_image(f.rows)
    t = np.concatenate(f.targets + f.decoys)
    assert (img[0][t] == F32(S_TRAP)).all() and (img[1][t, 0] == 127).all()
    assert (img[3][f.role == 0] == 0).all()  # background rows: zero residue


@pytest.mark.parametrize("metric,d,Q,k", KNN)
def test_knn_fixture_is_decisive(metric, d, Q, k):
    f = knn_fixture(metric, d, Q, k)
    check_decisive(f)
    pos = np.concatenate(f.targets)
    if Q * k >= TILE:  # every row position of a tile (warpgroup, warp, lane / 4, fragment row) holds a target
        assert np.unique(pos % TILE).size == TILE
    assert (pos < TILE).any()
    if Q * k * 257 > f.n:
        assert (np.concatenate(f.targets + f.decoys) >= f.n // TILE * TILE).any()  # the last, partial tile


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_threshold_fixtures_are_decisive(metric):
    for f in (sampled_fixture(metric), crowd_fixture(metric), split_fixture(metric)):
        check_decisive(f)
    # crowd: the traps' tile holds no trap at fragment row 0, and for every query more than 192 of its rows reach the
    # sampled threshold (the k-th best of the background rows the prep samples): the tile's prune decides
    f = crowd_fixture(metric)
    ex, est, bnd, upper = replica(f)[:4]
    assert (np.array([ri_of(p) for p in np.concatenate(f.targets + f.decoys)]) != 0).all()
    samp = sample_rows(f)
    assert (f.role[samp] != 0).sum() < f.k  # the sampled threshold is a background row's
    tile = slice(5 * TILE, 6 * TILE)
    for j in range(f.Q):
        tau = np.sort(ex[samp, j])[::-1][f.k - 1]
        assert (upper[tile, j] >= tau).sum() > 192, j
    # sampled: the decoys are the sample's best rows, so the prep's threshold sits at the decoys' true scores: every
    # target's upper bound reaches it, its estimate alone does not; the target's thread has a background row at ri = 0
    f = sampled_fixture(metric)
    ex, est, bnd, upper = replica(f)[:4]
    samp = sample_rows(f)
    for j in range(f.Q):
        tau = np.sort(ex[samp, j])[::-1][f.k - 1]
        assert tau <= ex[f.decoys[j], j].max()
        t = f.targets[j]
        assert (upper[t, j] >= tau).all() and (est[t, j] < tau).all() and (est[t, j] + bnd[t, j] * 0.5 < tau).any(), j
    for p in np.concatenate(f.targets):
        ri = ri_of(p)
        assert ri != 0 and f.role[p - 8 * (ri & 1) - 64 * (ri >> 1)] == 0
    # split: targets and decoys in different tiles (different CTAs): the finish kernel's global margin decides
    f = split_fixture(metric)
    assert len({p // TILE for p in np.concatenate(f.targets)} & {p // TILE for p in np.concatenate(f.decoys)}) == 0


def sample_rows(f):
    """The rows filter_prep_kernel scores for the initial threshold (Q <= 128, n >= 4096): i n / S, S = next_pow2(8 k)
    in [128, 2048]."""
    S = min(max(1 << (8 * f.k - 1).bit_length(), 128), 2048)
    return np.array([i * f.n // S for i in range(S)])


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_range_fixture_is_decisive(metric):
    check_decisive(range_fixture(metric), rng_check=True)
    check_decisive(anchor_fixture(metric), rng_check=True, exclude=[0])


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_filtered_fixture_is_decisive(metric):
    f = filtered_fixture(metric)
    filt = tagged(f)
    admit = admits(f.tags, filt)
    assert any(not admit[f.targets[j], j].all() for j in range(f.Q))  # the filter refuses targets: decoys enter the top k
    check_decisive(f, admit=admit)


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_graph_fixture_is_decisive(metric, filtered):
    check_graph_decisive(graph_fixture(metric, filtered))


def test_default_selection_fixture_is_decisive():
    check_decisive(make_fixture("cosine", 1000, 64, 10, n=20_000, seed=21))
