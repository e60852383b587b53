"""The int8 image of fp32 shards alone (NK_SHADOW=int8) against the BF16 shadow alone (NK_SHADOW=bf16) on
the same rows: both filters re-score their survivors exactly in fp32, so every search path built on the image — kNN, tag
filters, range, search by row, the self-join, graph update / remap, k-means assignment — returns the same indices and the
same score bits.  Also: the image follows append / update / remove like a freshly built one, non-finite rows and queries,
d not a multiple of 128, and no retry stage on uniform and clustered corpora."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _index(monkeypatch, image, rows, metric="cosine", path="shadow"):
    from nornicdb_b200.knn import KnnIndex
    monkeypatch.setenv("NK_SHADOW", image)  # read at creation
    ix = KnnIndex(rows.shape[1], metric=metric)
    ix.upload(rows)
    ix.set_path(path)
    return ix


def _same(a, b, what):
    ai, asc = a
    bi, bsc = b
    assert ai.shape == bi.shape, (what, ai.shape, bi.shape)
    bad = np.nonzero((ai != bi) | (asc.view(np.uint32) != bsc.view(np.uint32)))
    assert bad[0].size == 0, (what, bad[0][:5], ai[bad][:5], bi[bad][:5])


def _both(monkeypatch, rows, metric, fn, path="shadow"):
    out = {}
    for image in ("int8", "bf16"):
        ix = _index(monkeypatch, image, rows, metric, path)
        try:
            out[image] = fn(ix)
        finally:
            ix.release()
    return out["int8"], out["bf16"]


def _rows(rng, n, d):
    return rng.standard_normal((n, d)).astype(np.float32)


def test_int8_image_halves_the_scanned_bytes(knn_lib, monkeypatch):
    rng = np.random.default_rng(1)
    n, d = 20_000, 1000
    rows = _rows(rng, n, d)
    q = _rows(rng, 64, d)
    seen = {}
    for image in ("int8", "bf16"):
        ix = _index(monkeypatch, image, rows)
        b0 = ix.stats()["bytes_scanned"]
        ix.search(q, 10)
        assert ix.last_path() == "shadow"
        seen[image] = ix.stats()["bytes_scanned"] - b0
        ix.release()
    assert seen["int8"] == n * 1024 and seen["bf16"] == n * 1024 * 2, seen


def test_default_keeps_both_images_and_picks_per_search(knn_lib, monkeypatch):
    """NK_SHADOW unset: the int8 image serves k <= 16 on a shard of >= 64 MB, the BF16 shadow larger k, range searches and
    small shards; after a search on the int8 image overflowed its margins the shard keeps to the BF16 shadow (the clustered
    corpus of bench.py is what overflows it; DESIGN §3.3)."""
    from nornicdb_b200.knn import KnnIndex
    monkeypatch.delenv("NK_SHADOW", raising=False)
    rng = np.random.default_rng(2)
    n, d = 20_000, 1000  # 80 MB of fp32 rows
    rows = _rows(rng, n, d)
    q = _rows(rng, 64, d)
    ix = KnnIndex(d, metric="cosine")
    ix.upload(rows)
    ix.set_path("shadow")

    def scanned(fn):
        b0 = ix.stats()["bytes_scanned"]
        out = fn()
        assert ix.last_path() == "shadow"
        return ix.stats()["bytes_scanned"] - b0, out

    b8, r8 = scanned(lambda: ix.search(q, 10))
    b16, r16 = scanned(lambda: ix.search(q, 17))
    assert (b8, b16) == (n * 1024, n * 1024 * 2)
    assert (r8[0] == r16[0][:, :10]).all() and (r8[1].view(np.uint32) == r16[1][:, :10].view(np.uint32)).all()
    assert scanned(lambda: ix.search_range(q[:4], 0.2))[0] == n * 1024 * 2
    ix.release()
    # 3000 copies of one row: thousands of exact ties inside a query's margin.  Whichever image serves the second search,
    # the results are the same bits, and it is the BF16 shadow exactly when the first search overflowed
    tie = rows.copy()
    tie[:3000] = rows[0]
    ix = KnnIndex(d, metric="cosine")
    ix.upload(tie)
    ix.set_path("shadow")
    qt = np.concatenate([tie[:1] * np.float32(2.0), q[1:]]).astype(np.float32)
    c0 = ix.debug_counters()
    b1, r1 = scanned(lambda: ix.search(qt, 10))
    c1 = ix.debug_counters()
    overflowed = c1["bf16_stage_retries"] + c1["exact_stage_runs"] > c0["bf16_stage_retries"] + c0["exact_stage_runs"]
    assert b1 == n * 1024
    b2, r2 = scanned(lambda: ix.search(qt, 10))
    assert b2 == n * 1024 * (2 if overflowed else 1), (c0, c1, b2)
    assert (r1[0] == r2[0]).all() and (r1[1].view(np.uint32) == r2[1].view(np.uint32)).all()
    ix.release()
    small = KnnIndex(64, metric="cosine")
    small.upload(_rows(rng, 20_000, 64))
    small.set_path("shadow")
    b0 = small.stats()["bytes_scanned"]
    small.search(q[:, :64].copy(), 10)
    assert small.stats()["bytes_scanned"] - b0 == 20_000 * 64 * 2  # small shard: the BF16 shadow
    small.release()


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
@pytest.mark.parametrize("d", [36, 100, 1000, 1024])
def test_knn_matches_the_bf16_shadow(knn_lib, monkeypatch, metric, d):
    rng = np.random.default_rng(d)
    n = 30_000
    rows = _rows(rng, n, d)
    q = np.concatenate([rows[rng.integers(0, n, 512)] + _rows(rng, 512, d) * 0.3, _rows(rng, 512, d)]).astype(np.float32)
    cases = [(1, 10), (64, 10), (64, 100), (300, 10), (1024, 10)] + ([(64, 192), (300, 100)] if d in (100, 1024) else [])

    def run(ix):
        res = {}
        for Q, k in cases:
            res[Q, k] = ix.search(q[:Q], k)
            assert ix.last_path() == "shadow" and ix.debug_flags()[0] == 0
        return res

    a, b = _both(monkeypatch, rows, metric, run)
    for key in a:
        _same(a[key], b[key], (metric, d, key))


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_filters_range_rows_pairs_match_the_bf16_shadow(knn_lib, monkeypatch, metric):
    from nornicdb_b200.knn import synthetic_tags
    rng = np.random.default_rng(7)
    n, d = 20_000, 128
    rows = _rows(rng, n, d)
    rows[5000:5200] = rows[:200] + _rows(rng, 200, d) * 0.05  # near-duplicates: the self-join has pairs to find
    q = _rows(rng, 80, d)
    tags = synthetic_tags(n, 3)
    filt = np.array([[1 << (i % 5), 1 << 7, 0] for i in range(len(q))], np.uint64)
    thr = 0.3 if metric == "cosine" else 14.0
    pthr = 0.97 if metric == "cosine" else 4.0

    def run(ix):
        ix.set_row_tags(tags)
        out = {"filtered": ix.search_filtered(q, 20, filt)}
        for i, (gi, gs) in enumerate(ix.search_range(q[:16], thr)):
            out[f"range{i}"] = (gi, gs)
        out["rows"] = ix.search_rows(np.arange(0, n, 97), 15)
        off, pi, ps = ix.search_pairs(pthr)
        out["pairs"] = (np.concatenate([off.astype(np.uint32), pi]), np.concatenate([np.zeros(off.size, np.float32), ps]))
        return out

    a, b = _both(monkeypatch, rows, metric, run)
    assert a["pairs"][0].size > n + 100  # the join found pairs
    for key in a:
        _same(a[key], b[key], (metric, key))


def test_graph_update_and_remap_match_the_bf16_shadow(knn_lib, monkeypatch):
    from nornicdb_b200.knn import GraphRowMap
    rng = np.random.default_rng(11)
    n, d, k = 6000, 64, 10
    rows = _rows(rng, n, d)
    extra = _rows(rng, 300, d)

    def run(ix):
        gi, gs = ix.search_rows(np.arange(n), k)
        ix.append(extra)
        ix.update_row(17, extra[5])
        ui, us, _ = ix.update_knn_graph(gi, gs, n, np.array([17], np.uint32), k=k)
        m = GraphRowMap(len(ix))
        g2i, g2s = ix.search_rows(np.arange(len(ix)), k)
        for r in (3, 40, 500):
            ix.remove_swap(r)
            m.remove_swap(r)
        ri, rs, _ = ix.remap_knn_graph(g2i, g2s, m.n_old, m, k=k)
        return {"update": (ui, us), "remap": (ri, rs)}

    a, b = _both(monkeypatch, rows, "cosine", run)
    for key in a:
        _same(a[key], b[key], key)


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_assignment_matches_the_bf16_shadow(knn_lib, monkeypatch, metric):
    rng = np.random.default_rng(5)
    n, d, K = 50_000, 256, 100
    mu = rng.uniform(-1, 1, (K, d)).astype(np.float32)
    rows = (mu[rng.integers(0, K, n)] + rng.standard_normal((n, d)).astype(np.float32) * 0.15).astype(np.float32)
    cen = (mu + 0.01).astype(np.float32)
    monkeypatch.setenv("NK_ASSIGN_TENSOR", "1")

    def run(ix):
        got = np.zeros(n, np.int32)
        ix.assign_nearest(cen, got, metric=metric)
        ties, _ = ix.assign_ties(cen, metric=metric)
        return got, ties.size

    (ga, ta), (gb, tb) = _both(monkeypatch, rows, "cosine", run)
    assert (ga == gb).all()
    assert ta <= 10, ta  # the int8 bound still decides almost every row of a mixture


def test_maintained_image_equals_a_fresh_one(knn_lib, monkeypatch):
    rng = np.random.default_rng(3)
    n, d = 8000, 100
    rows = _rows(rng, n, d)
    extra = _rows(rng, 500, d)
    q = _rows(rng, 64, d)
    ix = _index(monkeypatch, "int8", rows)
    ix.append(extra)
    want = np.concatenate([rows, extra])
    for r, src in ((10, 0), (7000, 1), (8100, 2)):
        ix.update_row(r, extra[src] * 3.0)
        want[r] = extra[src] * 3.0
    for r in (5, 8498, 100):  # (8498: the last row once one is gone)
        ix.remove_swap(r)
        want[r] = want[-1]
        want = want[:-1]
    got = ix.search(q, 25)
    ix.release()
    fresh = _index(monkeypatch, "int8", want)
    _same(got, fresh.search(q, 25), "maintained vs fresh")
    fresh.release()


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_non_finite_rows_and_queries(knn_lib, monkeypatch, metric):
    rng = np.random.default_rng(9)
    n, d = 5000, 64
    rows = _rows(rng, n, d)
    rows[10, 3] = np.nan
    rows[20, 5] = np.inf
    rows[30, :] = -np.inf
    rows[40] = 0.0
    q = _rows(rng, 40, d)
    q[3, 1] = np.nan
    q[4, 2] = np.inf
    q[5] = 0.0
    a, b = _both(monkeypatch, rows, metric, lambda ix: ix.search(q, 12))
    _same(a, b, metric)


@pytest.mark.parametrize("corpus", ["uniform", "clustered"])
def test_no_retries_at_one_million_rows(knn_lib, monkeypatch, corpus):
    from nornicdb_b200.knn import KnnIndex
    monkeypatch.setenv("NK_SHADOW", "int8")
    ix = KnnIndex(1024, metric="cosine")
    if corpus == "uniform":
        ix.fill_uniform(1_000_000, 42)
    else:
        ix.fill_clustered(1_000_000, 42)
    q = np.ascontiguousarray(ix.read_rows(12345, 64) + np.float32(0.01))
    c0 = ix.debug_counters()
    ix.search(q, 10)
    assert ix.last_path() == "shadow"
    c1 = ix.debug_counters()
    ix.release()
    assert c1["bf16_stage_retries"] == c0["bf16_stage_retries"] and c1["exact_stage_runs"] == c0["exact_stage_runs"], (c0, c1)
