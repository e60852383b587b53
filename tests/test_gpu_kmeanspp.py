"""k-means++ seeding on the device (nk_index_kmeanspp, DESIGN §7 item 3): seeds, potentials and D² bit for bit against the
host restatement with the index's shard sizes, the triangle-inequality skip against the full passes, the ClusterIndex
mirror, the refusals and two devices."""
import ctypes as C

import numpy as np
import pytest

from kmeanspp_ref import kmeanspp_chunked

pytestmark = pytest.mark.gpu


def _rows(n, d, seed, centres=8):
    rng = np.random.default_rng(seed)
    mu = rng.uniform(-1, 1, (centres, d))
    return (mu[rng.integers(0, centres, n)] + rng.standard_normal((n, d)) * 0.1).astype(np.float32)


def _same(a, b):
    """Bit for bit, NaN for NaN (the device and the host write NaNs with different sign bits)."""
    nan = np.isnan(a)
    return bool((nan == np.isnan(b)).all() and (a[~nan].view(np.uint64) == b[~nan].view(np.uint64)).all())


def _check(ix, rows, K, first, u, shards=None, prune="1", monkeypatch=None):
    if monkeypatch is not None:
        monkeypatch.setenv("NK_KMPP_PRUNE", prune)
    got = ix.kmeanspp(K, first, u, min_d2=True)
    ws, wp, wm = kmeanspp_chunked(rows, K, first, u, shards)
    assert (got.seeds == ws).all(), np.nonzero(got.seeds != ws)[0][:5]
    assert _same(got.potential, wp) and _same(got.min_d2, wm)
    assert (got.centroids.view(np.uint32) == rows[ws].view(np.uint32)).all()
    return got


@pytest.mark.parametrize("d", [1, 3, 36, 100, 1024])
@pytest.mark.parametrize("n", [200, 256, 1000])
def test_exact_against_the_restatement(knn_lib, monkeypatch, d, n):
    from nornicdb_b200.cluster_index import optimalK
    from nornicdb_b200.knn import KnnIndex
    rows = _rows(n, d, d * 7 + n)
    ix = KnnIndex(d, metric="euclidean")
    ix.upload(rows)
    rng = np.random.default_rng(n + d)
    for K in sorted({1, 2, optimalK(n), n}):
        first = int(rng.integers(n))
        _check(ix, rows, K, first, rng.random(K - 1), monkeypatch=monkeypatch)
    ix.release()


def test_fixtures(knn_lib, monkeypatch):
    from nornicdb_b200.knn import KnnIndex
    n, d = 1000, 36
    rows = _rows(n, d, 3)
    rows[400:420] = rows[7]  # duplicates: zero weights
    rng = np.random.default_rng(5)
    ix = KnnIndex(d, metric="euclidean")
    ix.upload(rows)
    u = rng.random(29)
    u[0] = 0.0  # target 0
    _check(ix, rows, 30, 7, u, monkeypatch=monkeypatch)
    # K = n: the total reaches 0, after which row 0 is picked again and again, as in Go
    got = _check(ix, rows, n, 11, rng.random(n - 1), monkeypatch=monkeypatch)
    assert got.potential[-1] == 0.0 and got.seeds[-1] == 0
    ix.release()
    # a NaN row: every pick after seed 0 is the last row
    bad = rows.copy()
    bad[123, 5] = np.nan
    ix = KnnIndex(d, metric="euclidean")
    ix.upload(bad)
    got = _check(ix, bad, 12, 0, rng.random(11), monkeypatch=monkeypatch)
    assert (got.seeds[1:] == n - 1).all() and np.isnan(got.min_d2[123])
    ix.release()
    # an infinite element: the first infinite row is drawn
    inf = rows.copy()
    inf[777, 0] = np.inf
    ix = KnnIndex(d, metric="euclidean")
    ix.upload(inf)
    got = _check(ix, inf, 5, 0, np.array([0.5, 0.25, 0.9, 0.1]), monkeypatch=monkeypatch)
    assert got.seeds[1] == 777
    ix.release()


@pytest.mark.parametrize("d", [64, 37])
def test_pruning_changes_nothing_but_the_rows_read(knn_lib, monkeypatch, d):
    from nornicdb_b200.knn import KnnIndex
    n, K = 60_000, 120
    rng = np.random.default_rng(d)
    u = rng.random(K - 1)
    ix = KnnIndex(d, metric="euclidean")
    ix.fill_clustered(n, 42, 100, 0.1)
    out = {}
    for p in ("0", "1"):
        monkeypatch.setenv("NK_KMPP_PRUNE", p)
        out[p] = ix.kmeanspp(K, 5, u, min_d2=True)
    a, b = out["0"], out["1"]
    assert (a.seeds == b.seeds).all() and (a.potential == b.potential).all()
    assert (a.min_d2.view(np.uint64) == b.min_d2.view(np.uint64)).all()
    assert a.rows_read == n * K and b.rows_read < a.rows_read
    rows = ix.read_rows(0, n)
    ws, wp, wm = kmeanspp_chunked(rows, K, 5, u)
    assert (b.seeds == ws).all() and (b.min_d2.view(np.uint64) == wm.view(np.uint64)).all()
    ix.release()
    # uniform rows: the skip finds little, the outputs are the same
    ix = KnnIndex(d, metric="euclidean")
    ix.fill_uniform(20_000, 42)
    for p in ("0", "1"):
        monkeypatch.setenv("NK_KMPP_PRUNE", p)
        out[p] = ix.kmeanspp(40, 3, u[:39], min_d2=True)
    a, b = out["0"], out["1"]
    assert (a.seeds == b.seeds).all() and (a.min_d2.view(np.uint64) == b.min_d2.view(np.uint64)).all()
    assert b.rows_read <= a.rows_read
    ix.release()


def test_cluster_index_without_a_sample_seeds_on_the_device(knn_lib, oracle_mod):
    from nornicdb_b200.cluster_index import ClusterIndex, KMeansConfig
    from test_gpu_cluster import _mixture, _want_assign
    n, d, K = 6_000, 48, 12
    rows, _ = _mixture(n, d, K, 21, sigma=0.08)
    rows = (np.round(rows * 64) / 64).astype(np.float32)  # dyadic: every fp64 sum exact, host and device pick alike
    ci = ClusterIndex(d, KMeansConfig(NumClusters=K, AutoK=False, MaxIterations=25), rng=np.random.default_rng(7), init_sample=None)
    ci.AddBatch([f"n{i}" for i in range(n)], rows)
    host = ClusterIndex.__new__(ClusterIndex)
    host.dimensions, host.rng = d, np.random.default_rng(7)
    init = host._init_kmeanspp(K, rows)
    ci.Cluster()
    cen = init.copy()
    want = np.zeros(n, dtype=np.int32)
    iters = 0
    for _ in range(25):
        nxt = _want_assign(oracle_mod, rows, cen, False)
        changed = int((nxt != want).sum())
        want = nxt
        cen, _ = oracle_mod.kmeans_update(rows, want, cen)
        iters += 1
        if changed == 0:
            break
    assert ci.iterations == iters
    assert (ci.assignments == want).all()
    assert (ci.centroids.view(np.uint32) == cen.view(np.uint32)).all()
    ci.Release()


def test_refusals(knn_lib):
    from nornicdb_b200 import _lib
    from nornicdb_b200.knn import KnnIndex
    lib = knn_lib
    n, d = 300, 8
    ix = KnnIndex(d, metric="euclidean")
    ix.upload(_rows(n, d, 1))
    seeds = np.zeros(n + 1, dtype=np.uint32)
    u = np.full(n, 0.5)

    def call(K, first=0, uu=u, p=ix.ptr, out=seeds):
        uptr = uu.ctypes.data_as(C.c_void_p) if uu is not None else None
        optr = out.ctypes.data_as(C.c_void_p) if out is not None else None
        return lib.nk_index_kmeanspp(p, K, first, uptr, optr, None, None, None, None)

    assert call(3) == 0 and call(1, uu=None) == 0
    for args in [dict(K=3, p=None), dict(K=3, out=None), dict(K=2, uu=None), dict(K=0), dict(K=n + 1), dict(K=3, first=n)]:
        assert call(**args) == -1, args
        assert _lib.last_error()
    for bad in (np.nan, 1.0, -0.25, np.inf):
        v = u.copy()
        v[1] = bad
        assert call(3, uu=v) == -1 and "u[1]" in _lib.last_error()
    ix.release()
    h = KnnIndex(d, metric="euclidean", dtype="f16")
    h.upload(_rows(n, d, 1))
    assert lib.nk_index_kmeanspp(h.ptr, 2, 0, u.ctypes.data_as(C.c_void_p), seeds.ctypes.data_as(C.c_void_p), None, None, None, None) == -1
    assert "fp32" in _lib.last_error()
    h.release()


def test_two_devices(knn_lib):
    """Shard g of G holds rows [g N / G, (g + 1) N / G): the chunks restart at row N / 2."""
    from nornicdb_b200 import cuda
    from nornicdb_b200.knn import KnnIndex
    if cuda.DeviceCount() < 2:
        pytest.skip("needs two GPUs")
    n, d, K = 5_001, 36, 70
    rows = _rows(n, d, 9)
    ix = KnnIndex(d, metric="euclidean", devices=(0, 1))
    ix.upload(rows)
    u = np.random.default_rng(3).random(K - 1)
    got = ix.kmeanspp(K, 4, u, min_d2=True)
    ws, wp, wm = kmeanspp_chunked(rows, K, 4, u, [n // 2, n - n // 2])
    assert (got.seeds == ws).all() and (got.potential == wp).all()
    assert (got.min_d2.view(np.uint64) == wm.view(np.uint64)).all()
    ix.release()
