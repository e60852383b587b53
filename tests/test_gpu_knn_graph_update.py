"""nk_knn_graph_update (KnnIndex.update_knn_graph): a k-NN graph from search_rows, brought up to date after appends and
rewritten rows, equals search_rows over every row now, bit for bit, pad slots included, on the path the graph was built on."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PAD = 0xFFFFFFFF
K = 10


def make_index(rows, metric, dtype="f32", path="shadow", devices=(0,)):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex(rows.shape[1], metric=metric, dtype=dtype, devices=devices)
    ix.upload(rows)
    ix.set_path(path)
    return ix


def check_update(ix, gi, gs, n_old, changed=None, k=K):
    """update_knn_graph(G_old) == search_rows(all rows), bits of the scores included; n_lists_changed exact"""
    ui, us, nch = ix.update_knn_graph(gi, gs, n_old, changed, k=k)
    ri, rs = ix.search_rows(np.arange(len(ix)), k)
    assert ui.shape == ri.shape, (ui.shape, ri.shape)
    bad = np.nonzero((ui != ri).any(axis=1) | (us.view(np.uint32) != rs.view(np.uint32)).any(axis=1))[0]
    assert bad.size == 0, (bad[:5], ui[bad[:2]], ri[bad[:2]], us[bad[:2]], rs[bad[:2]])
    w = ri.shape[1]
    oi = np.full((n_old, w), PAD, np.uint32)
    osc = np.zeros((n_old, w), np.float32)
    oi[:, :gi.shape[1]] = gi[:, :w]
    osc[:, :gs.shape[1]] = gs[:, :w]
    differ = int(((ri[:n_old] != oi).any(axis=1) | (rs[:n_old].view(np.uint32) != osc.view(np.uint32)).any(axis=1)).sum())
    assert nch == differ, (nch, differ)
    return ui, us


def near_ties(rng, base, n, scale=1e-6):
    """copies of old rows and copies nudged by a few ulps: new rows that tie with, or nearly tie with, old neighbours"""
    pick = rng.integers(0, base.shape[0], n)
    out = base[pick].astype(np.float32).copy()
    out[n // 2:] += (rng.standard_normal(out[n // 2:].shape) * scale).astype(np.float32)
    return out


CASES = [(path, metric, dtype, shape) for shape in ((3000, 64), (2000, 1024)) for metric in ("cosine", "dot", "euclidean")
         for path, dtype in (("shadow", "f32"), ("shadow", "f16"), ("shadow", "bf16"), ("filter", "f32"))]


@pytest.mark.parametrize("path,metric,dtype,shape", CASES)
def test_update_equals_rebuild(path, metric, dtype, shape):
    rng = np.random.default_rng(CASES.index((path, metric, dtype, shape)))
    n, d = shape
    n_old = n - 300
    rows = rng.uniform(-1, 1, (n, d)).astype(np.float32)
    rows[n_old:n_old + 60] = near_ties(rng, rows[:n_old], 60)  # duplicates and near ties among the appended rows
    rows[5] = rows[7]  # an old duplicate pair
    ix = make_index(rows[:n_old], metric, dtype, path)
    gi, gs = ix.search_rows(np.arange(n_old), K)
    # a new row identical to row 0's k-th neighbour: it ties and must lose on row id
    rows[n_old + 60] = rows[gi[0, K - 1]]
    ix.append(rows[n_old:])
    changed = [3, 3, 100, int(gi[1, 0])]  # repeats allowed; row 1's best neighbour rewritten
    for c in sorted(set(changed)):
        ix.update_row(c, rng.uniform(-1, 1, d).astype(np.float32))
    check_update(ix, gi, gs, n_old, changed)
    ix.release()


@pytest.mark.parametrize("n_new", [1, 5, 1500])
def test_appends_only(n_new):
    rng = np.random.default_rng(n_new)
    n_old, d = 2500, 64
    rows = rng.uniform(-1, 1, (n_old + n_new, d)).astype(np.float32)
    ix = make_index(rows[:n_old], "cosine")
    gi, gs = ix.search_rows(np.arange(n_old), K)
    ix.append(rows[n_old:])
    check_update(ix, gi, gs, n_old)
    ix.release()


def test_two_shards_reverse_scan_spans_both():
    rng = np.random.default_rng(11)
    n_old, d = 4000, 128
    rows = rng.uniform(-1, 1, (n_old + 700, d)).astype(np.float32)
    for metric in ("cosine", "euclidean"):
        ix = make_index(rows[:n_old], metric, devices=(0, 0))
        gi, gs = ix.search_rows(np.arange(n_old), K)
        ix.append(rows[n_old:])
        ix.update_row(10, rows[3000])  # a rewritten row in the first shard copies one in the second
        check_update(ix, gi, gs, n_old, [10])
        ix.release()


def test_mask_reset_after_append_and_short_lists_under_a_floor():
    rng = np.random.default_rng(5)
    n_old, d = 3000, 64
    rows = rng.uniform(-1, 1, (n_old + 400, d)).astype(np.float32)
    keep = rng.random(n_old + 400) > 0.3
    ix = make_index(rows[:n_old], "cosine")
    ix.set_min_score(0.35)  # most lists end short of k
    ix.set_row_mask(keep[:n_old])
    gi, gs = ix.search_rows(np.arange(n_old), K)
    assert (gi == PAD).any(), "the floor leaves some lists short"
    ix.append(rows[n_old:])
    ix.set_row_mask(keep)  # append clears the mask; masked-out new rows must enter no list
    ix.update_row(1, rows[2])
    check_update(ix, gi, gs, n_old, [1])
    ix.release()


def test_hub_enters_more_than_1024_lists():
    from nornicdb_b200.knn import KnnIndex
    n_old, d = 6000, 64
    ix = KnnIndex(d, metric="cosine")
    ix.fill_clustered(n_old, 3, n_centres=1, sigma=0.05, unit_norm=True)
    ix.set_path("shadow")
    rows = ix.read_rows(0, n_old)
    gi, gs = ix.search_rows(np.arange(n_old), K)
    hub = rows.mean(axis=0, keepdims=True).astype(np.float32)  # the centre of the data: everyone's nearest
    ix.append(hub)
    ui, _ = check_update(ix, gi, gs, n_old)
    assert (ui[:n_old] == n_old).any(axis=1).sum() > 1024
    ix.release()


def test_nan_rows_old_and_new():
    """A search block that holds a NaN row as a query overflows the filter and falls through to a later stage, and on the
    exact stage the arithmetic differs, so the rebuild's lists of that block's other rows depend on the block: the rows of
    blocks without a NaN query are held to bit equality.  A NaN row's own list holds the first k other rows by id; its scores
    are those of the stage that served it (cosine: 0 from the filter's finish, -inf from the exact stage)."""
    rng = np.random.default_rng(9)
    n_old, d, n_new = 3000, 64, 50
    rows = rng.uniform(-1, 1, (n_old + n_new, d)).astype(np.float32)
    rows[17, 3] = np.nan
    rows[n_old + 4, 0] = np.nan
    nan_rows = [17, 40, n_old + 4]
    for metric in ("cosine", "euclidean"):
        ix = make_index(rows[:n_old], metric)
        gi, gs = ix.search_rows(np.arange(n_old), K)
        ix.append(rows[n_old:])
        bad = rows[40].copy()
        bad[5] = np.nan
        ix.update_row(40, bad)
        ui, us, _ = ix.update_knn_graph(gi, gs, n_old, [40])
        ri, rs = ix.search_rows(np.arange(n_old + n_new), K)
        clean = np.arange(1024, 2048)  # the one search block without a NaN query, old or new
        assert (ui[clean] == ri[clean]).all() and (us[clean].view(np.uint32) == rs[clean].view(np.uint32)).all(), metric
        assert (ui[nan_rows] == ri[nan_rows]).all(), metric
        assert not np.isin(nan_rows, ui[clean]).any(), metric  # a NaN row enters no finite list
        ix.release()


def test_large_clustered_update_without_retries():
    from nornicdb_b200.knn import KnnIndex
    n, d, n_new = 200_000, 1024, 4096
    ix = KnnIndex(d, metric="cosine")
    ix.fill_clustered(n + n_new, 21, n_centres=1000, sigma=0.1, unit_norm=True)
    new = ix.read_rows(n, n_new)
    tail = ix.read_rows(n - 8, 8)
    ix.release()
    ix = KnnIndex(d, metric="cosine")
    ix.fill_clustered(n, 21, n_centres=1000, sigma=0.1, unit_norm=True)  # counter-based generator: the same rows [0, n)
    assert (ix.read_rows(n - 8, 8) == tail).all()
    ix.set_path("shadow")
    gi, gs = ix.search_rows(np.arange(n), K)
    ix.append(new)
    rng = np.random.default_rng(3)
    changed = rng.choice(n, 64, replace=False)
    for c in changed:
        ix.update_row(int(c), new[int(c) % n_new] * np.float32(0.5))
    before = ix.debug_counters()
    ui, us, nch = ix.update_knn_graph(gi, gs, n, changed)
    after = ix.debug_counters()
    for c in ("bf16_stage_retries", "exact_stage_runs"):
        assert after[c] == before[c], (before, after)  # no retry or exact stage
    ri, rs = ix.search_rows(np.arange(n + n_new), K)
    assert (ui == ri).all() and (us.view(np.uint32) == rs.view(np.uint32)).all()
    assert nch == int(((ri[:n] != gi).any(axis=1) | (rs[:n].view(np.uint32) != gs.view(np.uint32)).any(axis=1)).sum())
    ix.release()


def test_refusals_leave_the_arrays_untouched():
    from nornicdb_b200 import _lib
    rng = np.random.default_rng(2)
    n_old, d = 500, 64
    rows = rng.uniform(-1, 1, (n_old + 20, d)).astype(np.float32)
    ix = make_index(rows[:n_old], "cosine")
    gi, gs = ix.search_rows(np.arange(n_old), K)
    ix.append(rows[n_old:])
    lib = _lib.load()
    n = len(ix)

    def call(k=K, n_old_=n_old, changed=(), gi_=None, gs_=None, null=False):
        a = np.full((n, k), PAD, np.uint32)
        s = np.zeros((n, k), np.float32)
        w = min(k, K)
        a[:n_old, :w] = gi[:, :w] if gi_ is None else gi_[:, :w]
        s[:n_old, :w] = gs[:, :w] if gs_ is None else gs_[:, :w]
        a0, s0 = a.copy(), s.copy()
        ch = np.asarray(changed, np.uint32)
        rc = lib.nk_knn_graph_update(ix.ptr, k, n_old_, ch.ctypes.data_as(C.c_void_p) if ch.size else None, int(ch.size),
                                     None if null else a.ctypes.data_as(C.c_void_p), s.ctypes.data_as(C.c_void_p), None)
        return rc, (a == a0).all() and (s.view(np.uint32) == s0.view(np.uint32)).all()

    for path in ("simt", "tensor"):
        ix.set_path(path)
        assert call() == (-1, True)
    ix.set_path("shadow")
    assert call(k=192) == (-1, True)
    assert call(k=0) == (-1, True)
    assert call(n_old_=n + 1) == (-1, True)
    assert call(changed=[n_old]) == (-1, True)
    g2 = gi.copy()
    g2[3, 2] = n_old  # an appended row cannot be in the old graph
    assert call(gi_=g2) == (-1, True)
    assert call(null=True)[0] == -1
    ix.set_path("filter")
    rc, same = call()
    assert rc == K and not same  # the same call on a graph path is served
    ix.release()
    # a shape the filter paths do not serve: dim 30 has no 16-bit image and no TF32 filter alignment
    ix = make_index(rng.uniform(-1, 1, (300, 30)).astype(np.float32), "cosine", path="auto")
    g, s = ix.search_rows(np.arange(300), K)
    a, sc = g.copy(), s.copy()
    from nornicdb_b200.knn import KnnError
    with pytest.raises(KnnError):
        ix.update_knn_graph(a, sc, 300)
    assert (a == g).all()
    ix.release()
