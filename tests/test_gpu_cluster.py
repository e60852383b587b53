"""GPU parity tests of the k-means routing row (SURVEY.md §8(f)4): device assignment / update steps and the
gpu.ClusterIndex mirror against the oracle's restatement of pkg/gpu/kmeans.go."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _mixture(n, d, centres, seed, sigma=0.15):
    rng = np.random.default_rng(seed)
    mu = rng.uniform(-1, 1, (centres, d)).astype(np.float32)
    lab = rng.integers(0, centres, n)
    return (mu[lab] + rng.standard_normal((n, d)).astype(np.float32) * sigma).astype(np.float32), mu


def _want_assign(oracle_mod, rows, cen, by_cosine):
    """The contract of nk_index_assign_nearest (DESIGN §7 item 3): kmeans.go's assignment under euclidean; under cosine the
    argmax of the fp64 cosine of the fp32 inputs, lowest index among equal scores, 0 for zero vectors, NaN never."""
    if not by_cosine:
        want = np.zeros(len(rows), dtype=np.int32)
        oracle_mod.kmeans_assign(rows, cen, want)
        return want
    uniq, inv = np.unique(cen.view(np.uint32), axis=0, return_inverse=True)  # identical centroids, identical scores
    u = uniq.view(np.float32).astype(np.float64)
    x = rows.astype(np.float64)
    with np.errstate(all="ignore"):
        xx, cc = (x * x).sum(1)[:, None], (u * u).sum(1)[None, :]
        s = np.where((xx == 0) | (cc == 0), 0.0, (x @ u.T) / (np.sqrt(xx) * np.sqrt(cc)))[:, inv.reshape(-1)]
    return np.argmax(np.where(np.isnan(s), -np.inf, s), axis=1).astype(np.int32)


@pytest.mark.parametrize("tensor", ["1", "0"])
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("shape", [(20_000, 64, 37), (5_000, 128, 200), (3_000, 30, 5), (2_500, 256, 1), (12_000, 96, 600)])
def test_assign_nearest_matches_oracle(knn_lib, oracle_mod, metric, shape, tensor, monkeypatch):
    """tensor=1: one pass of the tensor-core scan with an argmax epilogue over the BF16 shadow (+ exact fp32 fix-up of
    near-ties); tensor=0 (or no shadow / dim % 4 != 0): the fused kNN scan with the roles swapped."""
    from nornicdb_b200.knn import KnnIndex
    monkeypatch.setenv("NK_ASSIGN_TENSOR", tensor)
    n, d, K = shape
    rows, mu = _mixture(n, d, max(K, 2), 5)
    cen = (mu[:K] + 0.01).astype(np.float32)
    rows[11] = 0.0            # zero row: cosine 0 to every centroid -> centroid 0
    if K > 3:
        cen[3] = cen[1]       # duplicate centroid: exact tie, the lower index must win
    ix = KnnIndex(d, metric="cosine")
    ix.upload(rows)
    got = np.zeros(n, dtype=np.int32)
    changed = ix.assign_nearest(cen, got, metric=metric)
    again = got.copy()
    assert ix.assign_nearest(cen, again, metric=metric) == 0 and (again == got).all()  # idempotent: nothing changes
    ix.release()
    want = _want_assign(oracle_mod, rows, cen, metric == "cosine")
    assert (got == want).all(), np.nonzero(got != want)[0][:10]
    assert changed == int((want != 0).sum())


def test_cluster_means_matches_oracle_and_keeps_empty_clusters(knn_lib, oracle_mod):
    from nornicdb_b200.knn import KnnIndex
    n, d, K = 30_000, 96, 50
    rows, mu = _mixture(n, d, K, 9)
    rng = np.random.default_rng(2)
    assign = rng.integers(0, K - 2, n).astype(np.int32)  # clusters K-2 and K-1 stay empty
    assign[17] = -1                                       # out-of-range assignments are ignored
    prev = rng.uniform(-1, 1, (K, d)).astype(np.float32)
    ix = KnnIndex(d, metric="cosine")
    ix.upload(rows)
    got, counts = ix.cluster_means(assign, prev)
    ix.release()
    want, wcounts = oracle_mod.kmeans_update(rows, assign, prev)
    assert (counts == wcounts).all() and counts[-1] == 0 and counts[-2] == 0
    assert (got[-2:] == prev[-2:]).all()                  # empty clusters keep their previous position (kmeans.go:608-617)
    # fp64 sums in another order differ from the oracle's far below fp32 rounding: at most one ulp of the fp32 mean
    ulps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    assert (np.sign(got) == np.sign(want)).all() and ulps.max() <= 1, ulps.max()


@pytest.mark.parametrize("assign", ["euclidean", "cosine"])
def test_cluster_index_lloyd_iterations_follow_the_oracle(knn_lib, oracle_mod, assign):
    from nornicdb_b200.cluster_index import ClusterIndex, KMeansConfig
    n, d, K = 6_000, 48, 12
    rows, mu = _mixture(n, d, K, 21, sigma=0.08)
    # dyadic data (multiples of 1/64): every fp64 sum of the update step is exact, so cluster_means is bit-reproducible
    # and the whole Lloyd loop must follow the oracle exactly
    rows = (np.round(rows * 64) / 64).astype(np.float32)
    ci = ClusterIndex(d, KMeansConfig(NumClusters=K, AutoK=False, MaxIterations=25), assign=assign, rng=np.random.default_rng(7))
    ci.AddBatch([f"n{i}" for i in range(n)], rows)
    init = ci._init_kmeanspp(K, rows)
    ci.Cluster(initial_centroids=init)
    assert ci.IsClustered() and ci.NumClusters() == K
    # the same Lloyd loop on the oracle from the same initial centroids
    cen = init.copy()
    want = np.zeros(n, dtype=np.int32)
    iters = 0
    for _ in range(25):
        nxt = _want_assign(oracle_mod, rows, cen, assign == "cosine")
        changed = int((nxt != want).sum())
        want = nxt
        cen, _ = oracle_mod.kmeans_update(rows, want, cen)
        iters += 1
        if changed == 0:
            break
    assert ci.iterations == iters
    assert (ci.assignments == want).all()
    assert (ci.centroids.view(np.uint32) == cen.view(np.uint32)).all()
    st = ci.ClusterStats()
    assert st.Clustered and st.NumClusters == K and st.EmbeddingCount == n and st.MinClusterSize >= 1
    members = ci.GetClusterMembers(list(range(K)))
    assert sorted(members) == list(range(n))
    # routing: every well-separated mixture component maps to the cluster holding its points
    c0 = ci.FindNearestCentroid(rows[0])
    assert c0 == ci.assignments[0] or assign == "cosine"
    near = ci.FindNearestClusters(rows[0], 3)
    assert len(near) == 3 and near[0] == ci.FindNearestCentroid(rows[0])
    # cluster-restricted search = brute force restricted to the members of those clusters
    res = ci.SearchWithClusters(rows[5], 10, 2)
    cand = ci.GetClusterMembers(ci.FindNearestClusters(rows[5], 2))
    sub = rows[cand].astype(np.float64)
    q = rows[5].astype(np.float64)
    cos = sub @ q / np.sqrt((sub * sub).sum(1) * (q @ q))
    order = np.argsort(-cos, kind="stable")[:10]
    assert [r.ID for r in res] == [f"n{cand[i]}" for i in order]
    assert np.allclose([r.Score for r in res], cos[order], rtol=1e-4, atol=1e-6)
    ci.Release()


def test_cluster_index_reference_kats(knn_lib):
    from nornicdb_b200.cluster_index import ClusterIndex, ErrInvalidDimensions
    kats = json.load(open(os.path.join(HERE, "golden", "reference_kats.json")))
    seen = 0
    for t in kats:
        if t["op"] != "kmeans.search_candidates":
            continue
        seen += 1
        ci = ClusterIndex(t["dims"])
        for i in range(t["n"]):  # kmeans_test.go:747-752
            emb = np.zeros(t["dims"], dtype=np.float32)
            emb[i % t["dims"]] = float(i)
            ci.Add("node-" + chr(ord("A") + i), emb)
        if "want_error" in t:
            with pytest.raises(ErrInvalidDimensions):
                ci.SearchCandidates(t["query"], t["candidates"], t["topk"])
        else:
            res = ci.SearchCandidates(t["query"], t["candidates"], t["topk"])
            assert len(res or []) == t["want_len"], t
        ci.Release()
    assert seen == 4


def test_cluster_index_auto_k_errors_and_updates(knn_lib, oracle_mod):
    from nornicdb_b200.cluster_index import ClusterIndex, KMeansConfig
    d = 32
    ci = ClusterIndex(d, rng=np.random.default_rng(3))
    ci.Cluster()  # empty index: nothing happens (kmeans.go:239-241)
    assert not ci.IsClustered() and ci.FindNearestCentroid(np.zeros(d)) == -1 and ci.FindNearestClusters(np.zeros(d), 2) is None
    rows, _ = _mixture(5, d, 2, 1)
    ci.AddBatch([f"a{i}" for i in range(5)], rows)
    ci.config = KMeansConfig(NumClusters=10, AutoK=False)
    ci.Cluster()  # k > n -> k = n (kmeans_test.go: "adjusted to n")
    assert ci.NumClusters() == 5
    rows2, _ = _mixture(400, d, 4, 2)
    ci.AddBatch([f"b{i}" for i in range(400)], rows2)
    ci.config = KMeansConfig()  # AutoK: optimalK(405) = 14
    ci.Cluster()
    assert ci.NumClusters() == 14 and len(ci.assignments) == 405
    before = ci.updatesSinceCluster
    ci.OnNodeUpdate("b7", rows2[300])  # moved next to another point: reassigned to that point's cluster
    assert ci.assignments[ci.idToIndex["b7"]] == ci.FindNearestCentroid(rows2[300])
    ci.OnNodeUpdate("fresh", rows2[10])
    assert len(ci.assignments) == 406 and ci.updatesSinceCluster == before + 2
    ci.UpdateCentroidsBatch()
    assert not ci.pendingUpdates
    ci.Release()
