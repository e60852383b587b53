"""The k-means++ seeding contract of nk_index_kmeanspp restated on the host (no GPU): the chunked pick against kmeans.go's
sequential one, and the triangle-inequality row skip (DESIGN §7 item 3)."""
import numpy as np
import pytest

from kmeanspp_ref import CHUNK, EPS, kmeanspp_chunked, kmeanspp_seq, skips, sq_euclid64_rows


def _dyadic(n, d, seed, centres=6):
    rng = np.random.default_rng(seed)
    mu = rng.uniform(-1, 1, (centres, d))
    x = mu[rng.integers(0, centres, n)] + rng.standard_normal((n, d)) * 0.2
    return (np.round(x * 64) / 64).astype(np.float32)  # multiples of 1/64: every fp64 sum below is exact


@pytest.mark.parametrize("d", [1, 3, 7, 36])
def test_sq_euclid64_rows_is_the_oracles(oracle_mod, d):
    rng = np.random.default_rng(d)
    rows = rng.standard_normal((50, d)).astype(np.float32) * np.float32(3)
    c = rng.standard_normal(d).astype(np.float32)
    got = sq_euclid64_rows(rows, c)
    want = np.array([oracle_mod.sq_euclid64(r, c) for r in rows])
    assert (got.view(np.uint64) == want.view(np.uint64)).all()


@pytest.mark.parametrize("shards", [None, [600, 413], [1, 1012], [256, 256, 501]])
def test_dyadic_rows_chunked_pick_is_the_sequential_one_and_the_mirrors(shards):
    from nornicdb_b200.cluster_index import ClusterIndex
    n, d, K = 1013, 12, 40
    rows = _dyadic(n, d, 3)
    rows[100:110] = rows[5]  # duplicates: zero weights once row 5 is a seed
    first, u = 17, np.random.default_rng(1).random(K - 1)
    u[3] = 0.0
    s1, p1, m1 = kmeanspp_chunked(rows, K, first, u, shards)
    s2, p2, m2 = kmeanspp_seq(rows, K, first, u)
    assert (s1 == s2).all() and (p1 == p2).all() and (m1 == m2).all()
    # ClusterIndex._init_kmeanspp (numpy sums, host) draws the same stream: rng.integers(n), then rng.random() per seed
    ci = ClusterIndex.__new__(ClusterIndex)
    ci.dimensions, ci.rng = d, np.random.default_rng(9)
    cen = ci._init_kmeanspp(K, rows)
    rng = np.random.default_rng(9)
    f = int(rng.integers(n))
    s3, _, _ = kmeanspp_chunked(rows, K, f, rng.random(K - 1), shards)
    assert (cen.view(np.uint32) == rows[s3].view(np.uint32)).all()


def test_one_vector_draw_is_the_scalar_draws():
    a, b = np.random.default_rng(4), np.random.default_rng(4)
    assert int(a.integers(1000)) == int(b.integers(1000))
    assert (a.random(50) == np.array([b.random() for _ in range(50)])).all()


def test_fixtures_follow_go():
    rng = np.random.default_rng(2)
    n, d = 700, 5
    rows = _dyadic(n, d, 7)
    # K = n drives the total to 0: every later pick is row 0 (target 0, cumWeight 0 >= 0)
    s, p, _ = kmeanspp_chunked(rows, n, 3, rng.random(n - 1))
    assert p[-1] == 0.0
    z = int(np.argmax(p == 0.0))
    assert (s[z + 1:] == 0).all()
    # a NaN row: every pick after seed 0 is the last row (the total and the target are NaN)
    bad = rows.copy()
    bad[50, 2] = np.nan
    s, p, m = kmeanspp_chunked(bad, 6, 0, rng.random(5))
    assert (s[1:] == n - 1).all() and np.isnan(p).all() and np.isnan(m[50])
    # an infinite element: infinite weight, the first infinite row is picked (u > 0)
    inf = rows.copy()
    inf[300, 0] = np.inf
    s, _, _ = kmeanspp_chunked(inf, 2, 0, [0.5])
    assert s[1] == 300
    s2, _, _ = kmeanspp_seq(inf, 2, 0, [0.5])
    assert s2[1] == 300


def test_random_rows_differ_only_within_the_rounding_of_the_sums():
    rng = np.random.default_rng(11)
    n, d, K = 3000, 9, 60
    rows = rng.standard_normal((n, d)).astype(np.float32)
    differ = 0
    for trial in range(8):
        u = rng.random(K - 1)
        first = int(rng.integers(n))
        sc, _, _ = kmeanspp_chunked(rows, K, first, u, [1234, n - 1234])
        ss, _, _ = kmeanspp_seq(rows, K, first, u)
        if (sc == ss).all():
            continue
        differ += 1
        c = int(np.argmax(sc != ss))  # the first different pick; both runs agree up to it
        _, _, m = kmeanspp_seq(rows, c, first, u)
        cum = np.cumsum(m)
        T = cum[-1]
        target = u[c - 1] * T
        # the target lies within n 2^-52 T of the sequential prefix boundary one of the picks sits at
        lo = min(int(sc[c]), int(ss[c]))
        bound = n * 2.0 ** -52 * T
        assert abs(cum[lo] - target) <= bound or (lo and abs(cum[lo - 1] - target) <= bound), (trial, c)
    assert differ <= 8


def test_skip_rule_never_skips_a_row_the_strict_update_would_lower():
    rng = np.random.default_rng(5)
    d = 24
    seeds = rng.uniform(-1, 1, (40, d)).astype(np.float32)
    rows = (seeds[rng.integers(0, 40, 20000)] + rng.standard_normal((20000, d)) * 0.05).astype(np.float32)
    skipped = 0
    for a in range(8):
        m = sq_euclid64_rows(rows, seeds[a])
        for c in range(8, 40):
            delta = sq_euclid64_rows(seeds[c:c + 1], seeds[a])[0]
            s = skips(delta, m, d)
            skipped += int(s.sum())
            new = sq_euclid64_rows(rows[s], seeds[c])
            assert (new >= m[s]).all()
    assert skipped > 100_000


def test_planted_midpoints_need_the_margin():
    """Rows at the rounded midpoint of a seed a and the new seed c: in exact arithmetic delta = 4 m.  Where the rounding puts
    the computed delta at or above 4 m while the computed new distance is below m, a skip with no margin would keep a value
    kmeans.go lowers.  The rule's margin of 2^-18 does not skip any of them, nor any planted row."""
    rng = np.random.default_rng(8)
    d, trials = 33, 20000
    a = rng.uniform(-1, 1, (trials, d)).astype(np.float32)
    c = rng.uniform(-1, 1, (trials, d)).astype(np.float32)
    t = np.float32(0.5) + rng.uniform(-1e-6, 1e-6, (trials, 1)).astype(np.float32)  # just inside and just outside delta = 4 m
    x = (a + t * (c - a)).astype(np.float32)
    m = np.array([sq_euclid64_rows(x[i:i + 1], a[i])[0] for i in range(trials)])
    new = np.array([sq_euclid64_rows(x[i:i + 1], c[i])[0] for i in range(trials)])
    delta = np.array([sq_euclid64_rows(c[i:i + 1], a[i])[0] for i in range(trials)])
    wrong_without_margin = (delta >= 4.0 * m) & (new < m)
    assert wrong_without_margin.sum() > 0
    s = skips(delta, m, d)
    assert not (s & (new < m)).any()
    assert not s[wrong_without_margin].any()


def test_chunks_start_at_each_shard():
    from kmeanspp_ref import _chunk_starts
    starts, counts = _chunk_starts([300, 513])
    assert starts == [0, 256, 300, 556, 812] and counts == [256, 44, 256, 256, 1]
    assert CHUNK == 256 and EPS == 2.0 ** -18
