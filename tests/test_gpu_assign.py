"""GPU tests of nk_index_assign_nearest's exact contract (DESIGN §7 item 3) on both paths (the tensor-core scan over the
BF16 shadow, and the k = min(2, K) search used without a usable shadow): planted BF16 traps, many-way ties, non-finite and
extreme rows and centroids, and the near-tie list (nk_debug_assign_ties) the error bound leaves to the exact fix-up."""
import numpy as np
import pytest

from test_assign_logic_cpu import ALL, NONE, TRAP_GAPS, trap_pair, trap_row

pytestmark = pytest.mark.gpu


def cosine64(rows, cen):
    """fp64 cosine of the fp32 inputs: 0 for a zero row or centroid, NaN for non-finite inputs.  Identical centroids get
    identical scores (computed once per distinct centroid)."""
    uniq, inv = np.unique(cen.astype(np.float32).view(np.uint32), axis=0, return_inverse=True)
    u = uniq.view(np.float32).astype(np.float64)
    x = rows.astype(np.float64)
    with np.errstate(all="ignore"):
        xx = (x * x).sum(1)[:, None]
        cc = (u * u).sum(1)[None, :]
        s = np.where((xx == 0) | (cc == 0), 0.0, (x @ u.T) / (np.sqrt(xx) * np.sqrt(cc)))
    return s[:, inv.reshape(-1)]


def want_assign(oracle_mod, rows, cen, metric):
    if metric == "euclidean":
        want = np.zeros(len(rows), np.int32)
        oracle_mod.kmeans_assign(rows, cen, want)
        return want
    s = cosine64(rows, cen)
    s = np.where(np.isnan(s), -np.inf, s)
    return np.argmax(s, axis=1).astype(np.int32)  # first maximum: the lowest index among equal scores


def scores64(rows, cen, metric, i):
    """Row i's fp64 scores (higher is better): -squaredEuclidean as kmeans.go computes it, or the fp64 cosine."""
    if metric == "cosine":
        return cosine64(rows[i:i + 1], cen)[0]
    d = (rows[i][None, :] - cen).astype(np.float64)  # fp32 differences
    return -(d * d).sum(1)


def run(knn_lib, oracle_mod, rows, cen, metric, tensor, monkeypatch, check_ties=True):
    """assign_nearest against the contract: exact assignment, exact `changed`, an idempotent second call; returns the
    near-tie rows.  Every row the bound decided has the fp64 winner with a positive fp64 gap."""
    from nornicdb_b200.knn import KnnIndex
    monkeypatch.setenv("NK_ASSIGN_TENSOR", "1" if tensor else "0")
    n, d = rows.shape
    ix = KnnIndex(d, metric="cosine")
    try:
        ix.upload(rows)
        prev = np.random.default_rng(1).integers(0, cen.shape[0], n).astype(np.int32)
        got = prev.copy()
        changed = ix.assign_nearest(cen, got, metric=metric)
        again = got.copy()
        assert ix.assign_nearest(cen, again, metric=metric) == 0 and (again == got).all()
        tie_rows, tie_cand = ix.assign_ties(cen, metric=metric)
    finally:
        ix.release()
    want = want_assign(oracle_mod, rows, cen, metric)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, (bad[:10], got[bad[:10]], want[bad[:10]])
    assert changed == int((prev != want).sum())
    assert len(set(tie_rows.tolist())) == tie_rows.size and (tie_rows < n).all()
    K = cen.shape[0]
    ok_cand = (tie_cand == ALL) | (tie_cand == NONE) | (tie_cand < K)
    assert ok_cand.all()
    if check_ties:
        listed = np.zeros(n, bool)
        listed[tie_rows] = True
        for i in np.nonzero(~listed)[0]:
            s = scores64(rows, cen, metric, i)
            top = np.sort(s[~np.isnan(s)])[::-1]
            assert got[i] == want[i] and (top.size == 1 or top[0] > top[1]), (i, top[:3])
        # a listed row's candidates hold its winner
        for r, c in zip(tie_rows, tie_cand):
            assert c[0] == ALL or want[r] in c[:3], (r, c, want[r])
    return set(tie_rows.tolist())


SHAPES = [(32, 2), (32, 5), (36, 3), (36, 64), (96, 4), (96, 63), (96, 600), (1024, 65), (1024, 129), (4096, 2), (4096, 129)]


def trap_data(metric, d, K, seed):
    """K centroids (trap pairs at random places, the last one unpaired when K is odd) and n rows, n not a multiple of
    256: trap rows at every gap of TRAP_GAPS, each nearer to its pair's c_b while the BF16 estimate says c_a."""
    rng = np.random.default_rng(seed)
    n = 301 if d <= 1024 else 45
    cen = np.zeros((K, d), np.float32)
    place = rng.permutation(K)
    pairs = []
    for p in range(K // 2):
        ca, cb = trap_pair(rng, d, metric)
        a, b = place[2 * p], place[2 * p + 1]
        cen[a], cen[b] = ca, cb
        pairs.append((a, b))
    if K % 2:
        cen[place[-1]] = trap_pair(rng, d, metric)[0]
    rows = np.zeros((n, d), np.float32)
    trap = []
    for i in range(n):
        a, b = pairs[i % len(pairs)]
        rows[i], _ = trap_row(rng, cen[a], cen[b], metric, TRAP_GAPS[i % len(TRAP_GAPS)])
        trap.append((i, a, b))
    return rows, cen, trap


@pytest.mark.parametrize("tensor", [True, False], ids=["tensor", "search"])
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("d,K", SHAPES)
def test_assign_traps_are_near_ties_and_exact(knn_lib, oracle_mod, monkeypatch, metric, d, K, tensor):
    rows, cen, trap = trap_data(metric, d, K, seed=d * 1000 + K)
    listed = run(knn_lib, oracle_mod, rows, cen, metric, tensor, monkeypatch)
    want = want_assign(oracle_mod, rows, cen, metric)
    planted = 0
    for i, a, b in trap:
        s = scores64(rows, cen, metric, i)
        if set(np.argsort(-s, kind="stable")[:2].tolist()) != {a, b}:
            continue  # at small d another centroid can come nearer than the pair: not a trap, exactness still holds
        planted += 1
        # the planted winner, where the gap is above kmeans.go's own fp32 rounding (~2^-22 d^2 under euclidean)
        if TRAP_GAPS[i % len(TRAP_GAPS)] >= 1e-5:
            assert want[i] == b, (i, a, b, want[i])
        else:
            assert want[i] in (a, b), (i, a, b, want[i])
        if tensor:  # the BF16 estimate is inverted: the bound cannot have decided these rows
            assert i in listed, (i, a, b)
    assert planted >= len(trap) // 2


@pytest.mark.parametrize("tensor", [True, False], ids=["tensor", "search"])
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("d", [32, 36, 96])
def test_assign_many_way_ties(knn_lib, oracle_mod, monkeypatch, metric, d, tensor):
    rng = np.random.default_rng(d)
    n, K = 517, 129
    cen = rng.uniform(-1, 1, (K, d)).astype(np.float32)
    # six identical centroids spread over lanes and blocks, and duplicate pairs in different lanes / blocks
    six = [3, 5, 17, 64, 66, 128]
    cen[six] = cen[40]
    cen[1] = cen[2]
    cen[9] = cen[73]
    # near-identical: one fp32 ulp away in one element
    cen[100] = cen[101]
    cen[100, 0] = np.nextafter(cen[101, 0], np.float32(np.inf))
    rows = (cen[rng.integers(0, K, n)] + rng.standard_normal((n, d)).astype(np.float32) * 0.01).astype(np.float32)
    rows[:50] = cen[40] + rng.standard_normal((50, d)).astype(np.float32) * 0.01
    listed = run(knn_lib, oracle_mod, rows, cen, metric, tensor, monkeypatch)
    want = want_assign(oracle_mod, rows, cen, metric)
    assert (want[:50] == 3).all()  # the lowest of the seven identical centroids wins
    assert not (np.isin(want, six[1:] + [40, 2, 73])).any()
    assert set(range(50)) <= listed
    # every centroid identical: every row is a tie, and centroid 0 wins
    same = np.repeat(cen[:1], K, axis=0)
    listed = run(knn_lib, oracle_mod, rows, same, metric, tensor, monkeypatch)
    assert listed == set(range(n))


@pytest.mark.parametrize("tensor", [True, False], ids=["tensor", "search"])
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("K", [1, 2, 5, 65])
def test_assign_non_finite_and_extreme_rows(knn_lib, oracle_mod, monkeypatch, metric, K, tensor):
    rng = np.random.default_rng(K)
    n, d = 389, 64
    cen = rng.uniform(-1, 1, (K, d)).astype(np.float32)
    rows = (cen[rng.integers(0, K, n)] + rng.standard_normal((n, d)).astype(np.float32) * 0.2).astype(np.float32)
    rows[0] = 0.0
    rows[1, 3] = np.nan
    rows[2, 5] = np.inf
    rows[3, :] = -np.inf
    rows[10:30] = (cen[rng.integers(0, K, 20)] * np.float32(3e19)).astype(np.float32)  # |x|^2 overflows fp32
    rows[40:60] = (rows[40:60] * np.float32(1e-22)).astype(np.float32)  # tiny rows
    run(knn_lib, oracle_mod, rows, cen, metric, tensor, monkeypatch, check_ties=False)
    # finite rows and centroids whose fp32 |x|^2 and |c|^2 overflow (elements 1e19 to 1e20): kmeans.go's fp64 sums
    # still order the centroids, an fp32 fix-up would see inf everywhere and answer centroid 0
    big_cen = (cen * np.float32(5e19)).astype(np.float32)
    big = (big_cen[rng.integers(0, K, n)] + rng.uniform(-2e19, 2e19, (n, d))).astype(np.float32)
    assert np.isinf((big[:5] ** 2).sum(1, dtype=np.float32)).all()
    run(knn_lib, oracle_mod, big, big_cen, metric, tensor, monkeypatch, check_ties=False)
    if K >= 2:
        want = want_assign(oracle_mod, big, big_cen, metric)
        assert (want != 0).sum() > n // 4
    if K >= 5:
        cen2 = cen.copy()
        cen2[1] = 0.0          # zero centroid: cosine 0 for every row
        cen2[2, 7] = np.nan    # non-finite centroids never win
        cen2[3, 0] = np.inf
        rows2 = rows.copy()
        rows2[100:120] = -cen2[4]  # every finite centroid but the zero one may score below 0 under cosine
        run(knn_lib, oracle_mod, rows2, cen2, metric, tensor, monkeypatch, check_ties=False)


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_assign_near_tie_share_on_mixture_data(knn_lib, oracle_mod, monkeypatch, metric):
    """The bound decides almost every row of a Gaussian mixture (see GUARD)."""
    from nornicdb_b200.knn import KnnIndex
    rng = np.random.default_rng(5)
    n, d, K = 100_000 + 37, 256, 200
    mu = rng.uniform(-1, 1, (K, d)).astype(np.float32)
    rows = (mu[rng.integers(0, K, n)] + rng.standard_normal((n, d)).astype(np.float32) * 0.15).astype(np.float32)
    cen = (mu + 0.01).astype(np.float32)
    monkeypatch.setenv("NK_ASSIGN_TENSOR", "1")
    ix = KnnIndex(d, metric="cosine")
    ix.upload(rows)
    tie_rows, _ = ix.assign_ties(cen, metric=metric)
    got = np.zeros(n, np.int32)
    ix.assign_nearest(cen, got, metric=metric)
    ix.release()
    share = tie_rows.size / n
    print(f"near-tie share {metric}: {share:.3e}")
    assert (got == want_assign(oracle_mod, rows, cen, metric)).all()
    assert share <= GUARD[metric], share


# Near-tie share of the mixture above, measured on one H100 80GB HBM3 at a 700 W power limit: 0 of 100 037 rows under
# both metrics (and 0 of 1M rows at d = 1024, K = 1000).  The guard allows 10 rows.
GUARD = {"euclidean": 1e-4, "cosine": 1e-4}


def test_assign_multi_shard_offsets(knn_lib, oracle_mod):
    from nornicdb_b200 import cuda
    from nornicdb_b200.knn import KnnIndex
    if cuda.DeviceCount() < 2:
        pytest.skip("needs two GPUs")
    rng = np.random.default_rng(3)
    n, d, K = 20_011, 64, 37
    cen = rng.uniform(-1, 1, (K, d)).astype(np.float32)
    rows = (cen[rng.integers(0, K, n)] + rng.standard_normal((n, d)).astype(np.float32) * 0.3).astype(np.float32)
    for metric in ["euclidean", "cosine"]:
        ix = KnnIndex(d, metric="cosine", devices=(0, 1))
        ix.upload(rows)
        got = np.full(n, 5, np.int32)
        changed = ix.assign_nearest(cen, got, metric=metric)
        ix.release()
        want = want_assign(oracle_mod, rows, cen, metric)
        assert (got == want).all() and changed == int((want != 5).sum())
