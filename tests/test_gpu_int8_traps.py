"""The int8 filter scan on rank-inversion traps (test_int8_traps_cpu.py): rows whose estimate is wrong by almost exactly
its error bound, so only a correct keep rule, prune margin and finish margin return the exact answer.

Each search runs on the int8 image alone (NK_SHADOW=int8, path "shadow") and is compared with the fp64 answer: identical
indices, scores within tests/parity.py's tolerance.  Each also proves that the filter alone decided: no retry stage, no
exact stage (either would return exact results whatever the keep rule does), no fatal flag, and for kNN and range
searches exactly the int8 image's bytes scanned.  The dump check compares the device's estimates with the host replica
bit for bit."""
import numpy as np
import pytest

from parity import ABS_FLOOR, REL_TOL
import test_int8_traps_cpu as T

pytestmark = pytest.mark.gpu


def _index(monkeypatch, f, image="int8"):
    from nornicdb_b200.knn import KnnIndex
    if image is None:
        monkeypatch.delenv("NK_SHADOW", raising=False)
    else:
        monkeypatch.setenv("NK_SHADOW", image)  # read at creation
    ix = KnnIndex(f.d, metric=f.metric)
    ix.upload(f.rows)
    ix.set_path("shadow")
    return ix


def _filter_decided(ix, f, Q, fn, bytes_check=True):
    """fn() on ix, asserting that the int8 filter decided it alone"""
    c0, b0 = ix.debug_counters(), ix.stats()["bytes_scanned"]
    out = fn()
    c1, b1 = ix.debug_counters(), ix.stats()["bytes_scanned"]
    assert ix.last_path() == "shadow"
    assert (c1["bf16_stage_retries"], c1["exact_stage_runs"]) == (c0["bf16_stage_retries"], c0["exact_stage_runs"]), (c0, c1)
    assert ix.debug_flags()[0] == 0
    if bytes_check:  # the int8 image: dimpad = ceil(d / 128) * 128 bytes per row, one pass per 128 queries
        assert b1 - b0 == f.n * ((f.d + 127) // 128 * 128) * ((Q + 127) // 128), (b1 - b0, f.n, f.d, Q)
    return out


def _want_knn(f, k, admit=None):
    ex = T.replica(f)[0]
    idx = np.empty((f.Q, k), np.int64)
    for j in range(f.Q):
        rows = np.arange(f.n) if admit is None else np.nonzero(admit[:, j])[0]
        order = np.lexsort((rows, -ex[rows, j]))[:k]
        idx[j] = rows[order]
    return idx, T.api_score(np.take_along_axis(ex.T, idx, 1), f.metric)


def _same(got, want, what):
    gi, gs = got
    wi, ws = want
    assert gi.shape == wi.shape, (what, gi.shape, wi.shape)
    bad = np.nonzero((gi != wi).any(1))[0]
    assert bad.size == 0, (what, "queries with other rows than the fp64 answer", bad[:5], gi[bad[:1]], wi[bad[:1]])
    err = np.abs(gs.astype(np.float64) - ws)
    assert (err <= REL_TOL * np.abs(ws) + ABS_FLOOR).all(), (what, float(err.max()))


@pytest.mark.parametrize("metric,d,Q,k", T.KNN)
def test_knn_traps(knn_lib, monkeypatch, metric, d, Q, k):
    f = T.knn_fixture(metric, d, Q, k)
    ix = _index(monkeypatch, f)
    try:
        got = _filter_decided(ix, f, Q, lambda: ix.search(f.q, k))
    finally:
        ix.release()
    _same(got, _want_knn(f, k), (metric, d, Q, k))


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
@pytest.mark.parametrize("where", ["sampled", "crowd", "split"])
def test_threshold_traps(knn_lib, monkeypatch, metric, where):
    """(a) decoys on the prep's sampled rows: the sampled initial threshold decides; (b) a crowd above it in the traps'
    tile forces the tile's prune; (c) targets and decoys in different CTAs: the finish kernel's margin decides."""
    f = {"sampled": T.sampled_fixture, "crowd": T.crowd_fixture, "split": T.split_fixture}[where](metric)
    ix = _index(monkeypatch, f)
    try:
        got = _filter_decided(ix, f, f.Q, lambda: ix.search(f.q, f.k))
    finally:
        ix.release()
    _same(got, _want_knn(f, f.k), (metric, where))


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_filtered_traps(knn_lib, monkeypatch, metric):
    """even queries refuse a third of their targets and decoys: admitted decoys enter the top k, and the bound still
    decides for the admitted targets (test_int8_traps_cpu.py proves it with the filter applied)"""
    f = T.filtered_fixture(metric)
    filt = T.tagged(f)
    admit = T.admits(f.tags, filt)
    ix = _index(monkeypatch, f)
    try:
        ix.set_row_tags(f.tags)
        got = _filter_decided(ix, f, f.Q, lambda: ix.search_filtered(f.q, f.k, filt))
    finally:
        ix.release()
    _same(got, _want_knn(f, f.k, admit), (metric, "filtered"))


@pytest.mark.parametrize("tags", [False, True])
@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_range_traps(knn_lib, monkeypatch, metric, tags):
    f = T.range_fixture(metric)
    thr, thr_key = T.api_thresholds(f)
    filt = T.tagged(f) if tags else None
    admit = T.admits(f.tags, filt) if tags else np.ones((f.n, f.Q), bool)
    ex = T.replica(f)[0]
    ix = _index(monkeypatch, f)
    try:
        if tags:
            ix.set_row_tags(f.tags)
        ix.search_range(f.q, thr, filt)  # sizes the result buffer: the checked call below scans once
        got = _filter_decided(ix, f, f.Q, lambda: ix.search_range(f.q, thr, filt))
    finally:
        ix.release()
    for j, (gi, gs) in enumerate(got):
        want = np.nonzero((ex[:, j] >= thr_key[j]) & admit[:, j])[0]
        assert np.isin(f.targets[j][admit[f.targets[j], j]], want).all()
        order = np.argsort(gi)
        assert np.array_equal(gi[order], want), (metric, tags, j, np.setdiff1d(want, gi)[:5], np.setdiff1d(gi, want)[:5])
        ws = T.api_score(ex[want, j], metric)
        assert (np.abs(gs[order] - ws) <= REL_TOL * np.abs(ws) + ABS_FLOOR).all(), (metric, j)


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_rows_and_pairs_traps(knn_lib, monkeypatch, metric):
    """search_rows and search_pairs with a stored anchor row (exactly its query, so exact in int8) as the query / left row"""
    f = T.anchor_fixture(metric)
    ex = T.replica(f)[0]
    ix = _index(monkeypatch, f)
    try:
        gi, gs = _filter_decided(ix, f, 1, lambda: ix.search_rows(np.array([0]), f.k), bytes_check=False)
        thr, thr_key = T.api_thresholds(f)
        off, pi, ps = _filter_decided(ix, f, 1, lambda: ix.search_pairs(float(thr[0]), 0, 1), bytes_check=False)
    finally:
        ix.release()
    rows = np.arange(1, f.n)
    order = np.lexsort((rows, -ex[rows, 0]))[:f.k]
    want = rows[order]
    assert np.array_equal(gi[0].astype(np.int64), want), (metric, gi[0], want)
    ws = T.api_score(ex[want, 0], metric)
    assert (np.abs(gs[0] - ws) <= REL_TOL * np.abs(ws) + ABS_FLOOR).all()
    want_p = rows[ex[rows, 0] >= thr_key[0]]
    assert np.isin(f.targets[0], want_p).all()
    order = np.argsort(pi)
    assert np.array_equal(pi[order].astype(np.int64), want_p), (metric, np.setdiff1d(want_p, pi)[:5], np.setdiff1d(pi, want_p)[:5])
    ws = T.api_score(ex[want_p, 0], metric)
    assert (np.abs(ps[order] - ws) <= REL_TOL * np.abs(ws) + ABS_FLOOR).all(), metric


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_graph_update_traps(knn_lib, monkeypatch, metric, filtered):
    """update_knn_graph after appending a stored query A: A belongs in trap row t's list, while the int8 estimate of
    (t, A) is half a bound below t's threshold (the reverse scan's per-row threshold decides); filtered graphs: only
    t's own filter keeps a nearer row out of its list (the row-side filter decides too)"""
    from parity import check_parity
    f = T.graph_fixture(metric, filtered)
    n_old = f.n_old
    F = f.filters
    from nornicdb_b200.knn import KnnIndex
    monkeypatch.setenv("NK_SHADOW", "int8")
    ix = KnnIndex(f.d, metric=metric)
    try:
        ix.upload(f.rows[:n_old])
        ix.set_path("shadow")
        if F is not None:
            ix.set_row_tags(f.tags[:n_old])
        gi, gs = ix.search_rows(np.arange(n_old), f.k, None if F is None else F[:n_old])
        ix.append(f.rows[n_old:])
        if F is not None:
            ix.set_row_tags(f.tags[n_old:], first_row=n_old)
        ui, us, changed = _filter_decided(ix, f, 1, lambda: ix.update_knn_graph(gi, gs, n_old, k=f.k, filters=F), bytes_check=False)
    finally:
        ix.release()
    assert gi[f.t, 0] == f.p and ui[f.t, 0] == n_old and changed >= 1, (gi[f.t], ui[f.t], changed)
    wi, wk = T.graph_want(f)
    check_parity(f.rows, f.rows, f.k, metric, ui, us, wi, T.api_score(wk, metric))


def test_default_selection_serves_the_traps_from_the_int8_image(knn_lib, monkeypatch):
    """NK_SHADOW unset: both images exist, and a k = 10 search of an 80 MB shard picks the int8 image"""
    f = T.make_fixture("cosine", 1000, 64, 10, n=20_000, seed=21)
    T.check_decisive(f)
    ix = _index(monkeypatch, f, image=None)
    try:
        got = _filter_decided(ix, f, 64, lambda: ix.search(f.q, 10))
    finally:
        ix.release()
    _same(got, _want_knn(f, 10), "default")


@pytest.mark.parametrize("d", [36, 100, 1024])
def test_dump_estimates_are_the_replica_bit_for_bit(knn_lib, monkeypatch, d):
    """DUMP instantiation, dot: the int8 estimate equals fl(fl(float(acc) s_q) s_x) for every (row, query) pair: the s8
    operand layout, the padding to a multiple of 128 and the column -> s_q mapping (queries of 64 different scales); the
    bound within a few ulps of the replica's, which sums in the device's order."""
    from nornicdb_b200.knn import KnnIndex
    rng = np.random.default_rng(d)
    n = 3000
    rows = (rng.standard_normal((n, d)) * rng.uniform(0.01, 100, (n, 1))).astype(np.float32)
    q = (rng.standard_normal((64, d)) * np.exp2(rng.integers(-6, 7, (64, 1))) * rng.uniform(1, 2, (64, 1))).astype(np.float32)
    monkeypatch.setenv("NK_SHADOW", "int8")
    ix = KnnIndex(d, metric="dot")
    ix.upload(rows)
    try:
        est, bnd = ix.filter_dump(q, "shadow")
    finally:
        ix.release()
    w_est, w_bnd, _ = T.scan_values(T.row_image(rows), T.query_prep(q, "dot"), "dot")
    bad = np.argwhere(est.view(np.uint32) != w_est.view(np.uint32))
    assert bad.size == 0, (d, bad[:4].tolist(), est[tuple(bad[0])], w_est[tuple(bad[0])])
    rel = np.abs(bnd.astype(np.float64) - w_bnd) / w_bnd
    assert rel.max() < 1e-6, (d, float(rel.max()))  # ~8 ulps
