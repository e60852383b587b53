"""nk_knn_graph_remap (KnnIndex.remap_knn_graph + GraphRowMap): a k-NN graph from search_rows, brought up to date after rows
were removed (swap with the last row), appended and rewritten, equals search_rows over every row now, bit for bit, pad slots
included, on the path the graph was built on."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PAD = 0xFFFFFFFF
NEW = 0xFFFFFFFF
K = 10


def make_index(rows, metric, dtype="f32", path="shadow", devices=(0,)):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex(rows.shape[1], metric=metric, dtype=dtype, devices=devices)
    ix.upload(rows)
    ix.set_path(path)
    return ix


class Tracked:
    """An index and the GraphRowMap of its graph, changed together"""

    def __init__(self, ix, n_old):
        from nornicdb_b200.knn import GraphRowMap
        self.ix, self.map = ix, GraphRowMap(n_old)

    def remove(self, r):
        self.ix.remove_swap(int(r))
        self.map.remove_swap(int(r))

    def append(self, rows):
        self.ix.append(rows)
        self.map.append(len(rows))

    def rewrite(self, r, v):
        self.ix.update_row(int(r), v)
        self.map.update_row(int(r))


def check_remap(t, gi, gs, k=K):
    """remap_knn_graph(G_old) == search_rows(all rows), bits of the scores included; n_lists_changed exact"""
    ix, m = t.ix, t.map
    ui, us, nch = ix.remap_knn_graph(gi, gs, m.n_old, m, k=k)
    ri, rs = ix.search_rows(np.arange(len(ix)), k)
    assert ui.shape == ri.shape, (ui.shape, ri.shape)
    bad = np.nonzero((ui != ri).any(axis=1) | (us.view(np.uint32) != rs.view(np.uint32)).any(axis=1))[0]
    assert bad.size == 0, (bad[:5], ui[bad[:2]], ri[bad[:2]], us[bad[:2]], rs[bad[:2]])
    w = ri.shape[1]
    src = m.src_of_row
    kept = np.nonzero(src == np.arange(len(src)))[0]
    oi = np.full((len(kept), w), PAD, np.uint32)
    osc = np.zeros((len(kept), w), np.float32)
    oi[:, :min(w, gi.shape[1])] = gi[kept, :w]
    osc[:, :min(w, gs.shape[1])] = gs[kept, :w]
    differ = int(((ri[kept] != oi).any(axis=1) | (rs[kept].view(np.uint32) != osc.view(np.uint32)).any(axis=1)).sum())
    assert nch == differ, (nch, differ)
    return ui, us


def near_ties(rng, base, n, scale=1e-6):
    """copies of old rows and copies nudged by a few ulps"""
    pick = rng.integers(0, base.shape[0], n)
    out = base[pick].astype(np.float32).copy()
    out[n // 2:] += (rng.standard_normal(out[n // 2:].shape) * scale).astype(np.float32)
    return out


CASES = [(path, metric, dtype, shape) for shape in ((3000, 64), (2000, 1024)) for metric in ("cosine", "dot", "euclidean")
         for path, dtype in (("shadow", "f32"), ("shadow", "f16"), ("shadow", "bf16"), ("filter", "f32"))]


@pytest.mark.parametrize("path,metric,dtype,shape", CASES)
def test_remap_equals_rebuild(path, metric, dtype, shape):
    rng = np.random.default_rng(CASES.index((path, metric, dtype, shape)))
    n, d = shape
    n_old = n - 300
    rows = rng.uniform(-1, 1, (n, d)).astype(np.float32)
    rows[n_old:n_old + 60] = near_ties(rng, rows[:n_old - 1], 60)  # duplicates and near ties among the appended rows
    rows[5] = rows[7]  # an old duplicate pair
    # the tie trap: the last old row B is a copy of A, row 0's k-th neighbour, and loses the tie to it on row id
    pre = make_index(rows[:n_old - 1], metric, dtype, path)
    a = int(pre.search_rows([0], K)[0][0, K - 1])
    pre.release()
    rows[n_old - 1] = rows[a]
    t = Tracked(make_index(rows[:n_old], metric, dtype, path), n_old)
    gi, gs = t.ix.search_rows(np.arange(n_old), K)
    assert gi[0, K - 1] == a
    x = next(j for j in range(1, a) if j not in gi[0])
    t.remove(x)  # B moves to id x < a and takes A's slot in row 0's list, though that list holds no moved or removed row
    ui, _ = check_remap(t, gi, gs)
    assert ui[0, K - 1] == x
    # then appends with near ties, removals of an appended row, the last row, row 0 and a hub, and rewrites, interleaved
    hub = int(np.bincount(gi.ravel(), minlength=n_old)[1:].argmax()) + 1
    t.append(rows[n_old:n_old + 150])
    t.remove(len(t.ix) - 1)
    t.rewrite(3, rng.uniform(-1, 1, d).astype(np.float32))
    t.remove(n_old + 20)  # an appended row
    t.remove(hub)
    t.append(rows[n_old + 150:])
    t.remove(0)
    t.rewrite(int(gi[1, 0]), rng.uniform(-1, 1, d).astype(np.float32))  # at its id, or where the last row moved
    t.remove(1234 % len(t.ix))
    check_remap(t, gi, gs)
    t.ix.release()


def test_euclidean_pairs_one_ulp_apart():
    """Two rows at squared distances 1 and 1 + 2^-23 from a third decode to the same distance, 1: their order is the key's.
    Moving the farther one below the nearer one's id must not reorder them."""
    rng = np.random.default_rng(12)
    n, d = 3000, 64
    rows = rng.uniform(-1, 1, (n, d)).astype(np.float32)
    qs = [100, 300, 700]
    for i, q in enumerate(qs):
        rows[q, :2] = 0.0
        near = rows[q].copy()
        near[0] = 1.0  # d^2 = 1
        far = rows[q].copy()
        far[0], far[1] = 1.0, np.float32(3 * 2.0 ** -13)  # d^2 = fl(1 + 9 * 2^-26) = 1 + 2^-23
        rows[500 + i] = near
        rows[n - 1 - i] = far  # the last rows: each removal below moves one of them below its twin
    assert np.sqrt(np.float32(1.0) + np.float32(2.0 ** -23)) == np.float32(1.0)
    for path in ("shadow", "filter"):
        t = Tracked(make_index(rows, "euclidean", path=path), n)
        gi, gs = t.ix.search_rows(np.arange(n), K)
        for i, q in enumerate(qs):
            assert gi[q, :2].tolist() == [500 + i, n - 1 - i] and gs[q, 0] == gs[q, 1] == 1.0
        for r in (10, 11, 12):
            t.remove(r)
        ui, _ = check_remap(t, gi, gs)
        for i, q in enumerate(qs):
            assert ui[q, :2].tolist() == [500 + i, 10 + i], ui[q]  # the far row at a lower id, still second
        t.ix.release()


def test_two_shards_removals_move_rows_across_the_boundary():
    rng = np.random.default_rng(11)
    n_old, d = 4000, 128
    rows = rng.uniform(-1, 1, (n_old + 300, d)).astype(np.float32)
    for metric in ("cosine", "euclidean"):
        t = Tracked(make_index(rows[:n_old], metric, devices=(0, 0)), n_old)
        gi, gs = t.ix.search_rows(np.arange(n_old), K)
        for r in (5, 1000, 1999, 2500):  # the last row of the second shard moves into the first
            t.remove(r)
        t.append(rows[n_old:])
        t.rewrite(10, rows[3000])
        t.remove(7)
        check_remap(t, gi, gs)
        t.ix.release()


def test_mask_set_again_after_removals_and_short_lists_under_a_floor():
    rng = np.random.default_rng(5)
    n_old, d = 3000, 64
    rows = rng.uniform(-1, 1, (n_old + 200, d)).astype(np.float32)
    keep = rng.random(n_old + 200) > 0.3
    t = Tracked(make_index(rows[:n_old], "cosine"), n_old)
    t.ix.set_min_score(0.35)  # most lists end short of k
    t.ix.set_row_mask(keep[:n_old])
    gi, gs = t.ix.search_rows(np.arange(n_old), K)
    assert (gi == PAD).any(), "the floor leaves some lists short"
    cur = list(keep[:n_old])  # each row's mask bit travels with its contents
    for r in (17, 400, 2997, 1500):  # 2997: the last row by then
        t.remove(r)
        cur[r] = cur[-1]
        cur.pop()
    t.append(rows[n_old:])
    cur += list(keep[n_old:])
    t.rewrite(1, rows[2])
    t.ix.set_row_mask(np.array(cur))  # remove_swap and append clear the mask
    check_remap(t, gi, gs)
    t.ix.release()


@pytest.mark.parametrize("how", ["shrink", "remove_then_grow"])
def test_no_more_than_k_admissible_rows(how):
    rng = np.random.default_rng(6)
    d, n_old = 64, 300
    rows = rng.uniform(-1, 1, (n_old + 6, d)).astype(np.float32)
    if how == "shrink":
        keep = np.zeros(n_old, bool)
        keep[rng.choice(n_old - 1, K + 4, replace=False)] = True  # the last row is not admissible
        t = Tracked(make_index(rows[:n_old], "cosine"), n_old)
        t.ix.set_row_mask(keep)
        gi, gs = t.ix.search_rows(np.arange(n_old), K)
        assert (gi[:, K - 1] != PAD).any()  # some old lists are full
        cur = list(keep)
        for r in np.nonzero(keep)[0][:5]:
            t.remove(r)  # K - 1 admissible rows remain
            cur[r] = cur[-1]
            cur.pop()
        t.ix.set_row_mask(np.array(cur))
    else:
        keep = np.zeros(n_old, bool)
        keep[[2, 9, 30, 41, 55, 77, 120]] = True  # 7 <= K admissible: every old list is short
        t = Tracked(make_index(rows[:n_old], "cosine"), n_old)
        t.ix.set_row_mask(keep)
        gi, gs = t.ix.search_rows(np.arange(n_old), K)
        cur = list(keep)
        for r in (20, 9):  # an inadmissible row, then an admissible one
            t.remove(r)
            cur[r] = cur[-1]
            cur.pop()
        t.append(rows[n_old:])
        t.ix.set_row_mask(np.array(cur + [True] * 6))  # 12 admissible now
    check_remap(t, gi, gs)
    t.ix.release()


def test_nan_rows_old_and_new():
    """The caveat of nk_knn_graph_update: rows of rebuild blocks without a NaN query are held to bit equality, and a NaN row's
    own list holds the right rows."""
    rng = np.random.default_rng(9)
    n_old, d, n_new = 3000, 64, 50
    rows = rng.uniform(-1, 1, (n_old + n_new, d)).astype(np.float32)
    rows[17, 3] = np.nan
    rows[40, 5] = np.nan
    rows[n_old + 4, 0] = np.nan
    for metric in ("cosine", "euclidean"):
        t = Tracked(make_index(rows[:n_old], metric), n_old)
        gi, gs = t.ix.search_rows(np.arange(n_old), K)
        t.append(rows[n_old:])
        t.remove(17)   # a NaN row removed; a clean row takes its id
        t.remove(300)  # a clean row removed
        nan_rows = [40, n_old + 4]
        ui, us, _ = t.ix.remap_knn_graph(gi, gs, n_old, t.map)
        ri, rs = t.ix.search_rows(np.arange(len(t.ix)), K)
        clean = np.arange(1024, 2048)  # the one search block without a NaN query
        assert (ui[clean] == ri[clean]).all() and (us[clean].view(np.uint32) == rs[clean].view(np.uint32)).all(), metric
        assert (ui[nan_rows] == ri[nan_rows]).all(), metric
        assert not np.isin(nan_rows, ui[clean]).any(), metric
        t.ix.release()


def test_large_clustered_mixed_changes_without_retries():
    from nornicdb_b200.knn import KnnIndex
    n, d, n_new = 200_000, 1024, 1000
    ix = KnnIndex(d, metric="cosine")
    ix.fill_clustered(n + n_new + 100, 21, n_centres=1000, sigma=0.1, unit_norm=True)
    new = ix.read_rows(n, n_new + 100)
    ix.release()
    ix = KnnIndex(d, metric="cosine")
    ix.fill_clustered(n, 21, n_centres=1000, sigma=0.1, unit_norm=True)  # counter-based generator: the same rows [0, n)
    ix.set_path("shadow")
    gi, gs = ix.search_rows(np.arange(n), K)
    t = Tracked(ix, n)
    rng = np.random.default_rng(3)
    ops = np.array(["remove"] * 1000 + ["append"] * 1000 + ["rewrite"] * 100)
    rng.shuffle(ops)
    a = w = 0
    for op in ops:
        if op == "remove":
            t.remove(int(rng.integers(len(ix))))
        elif op == "append":
            t.append(new[a:a + 1])
            a += 1
        else:
            t.rewrite(int(rng.integers(len(ix))), new[n_new + w])
            w += 1
    before = ix.debug_counters()
    ui, us, nch = ix.remap_knn_graph(gi, gs, n, t.map)
    after = ix.debug_counters()
    for c in ("bf16_stage_retries", "exact_stage_runs"):
        assert after[c] == before[c], (before, after)  # no retry or exact stage
    ri, rs = ix.search_rows(np.arange(len(ix)), K)
    assert (ui == ri).all() and (us.view(np.uint32) == rs.view(np.uint32)).all()
    src = t.map.src_of_row
    kept = np.nonzero(src == np.arange(len(src)))[0]
    assert nch == int(((ri[kept] != gi[kept]).any(axis=1) | (rs[kept].view(np.uint32) != gs[kept].view(np.uint32)).any(axis=1)).sum())
    ix.release()


def test_update_and_remap_agree_without_removals():
    rng = np.random.default_rng(4)
    n_old, d = 2500, 64
    rows = rng.uniform(-1, 1, (n_old + 200, d)).astype(np.float32)
    ix = make_index(rows[:n_old], "euclidean")
    gi, gs = ix.search_rows(np.arange(n_old), K)
    t = Tracked(ix, n_old)
    t.append(rows[n_old:])
    changed = [3, 3, 100, int(gi[1, 0])]
    for c in sorted(set(changed)):
        t.rewrite(c, rng.uniform(-1, 1, d).astype(np.float32))
    a = ix.update_knn_graph(gi, gs, n_old, changed)
    b = check_remap(t, gi, gs)
    assert (a[0] == b[0]).all() and (a[1].view(np.uint32) == b[1].view(np.uint32)).all()
    ix.release()


def test_refusals_leave_the_output_untouched():
    from nornicdb_b200 import _lib
    rng = np.random.default_rng(2)
    n_old, d = 500, 64
    rows = rng.uniform(-1, 1, (n_old, d)).astype(np.float32)
    ix = make_index(rows, "cosine")
    gi, gs = ix.search_rows(np.arange(n_old), K)
    ix.remove_swap(10)
    ix.remove_swap(20)
    lib = _lib.load()
    n = len(ix)
    ok_src = np.arange(n, dtype=np.uint32)
    ok_src[10], ok_src[20] = n_old - 1, n_old - 2

    def call(k=K, src=ok_src, gi_=gi, null_src=False, overlap=False):
        oi = np.full((n, k), 7, np.uint32)
        os_ = np.full((n, k), 3.0, np.float32)
        ii = np.full((n_old, k), PAD, np.uint32)
        si = np.zeros((n_old, k), np.float32)
        w = min(k, K)
        ii[:, :w] = gi_[:, :w]
        si[:, :w] = gs[:, :w]
        o0, s0 = oi.copy(), os_.copy()
        s = np.ascontiguousarray(np.asarray(src, np.uint32))
        out_i = ii[:n] if overlap else oi  # a view of the input graph
        rc = lib.nk_knn_graph_remap(ix.ptr, k, n_old, None if null_src else s.ctypes.data_as(C.c_void_p), ii.ctypes.data_as(C.c_void_p),
                                    si.ctypes.data_as(C.c_void_p), out_i.ctypes.data_as(C.c_void_p), os_.ctypes.data_as(C.c_void_p),
                                    None)
        return rc, (oi == o0).all() and (os_.view(np.uint32) == s0.view(np.uint32)).all()

    for path in ("simt", "tensor"):
        ix.set_path(path)
        assert call() == (-1, True)
    ix.set_path("shadow")
    assert call(k=192) == (-1, True)
    assert call(k=0) == (-1, True)
    bad = ok_src.copy()
    bad[3] = n_old  # not an old row
    assert call(src=bad) == (-1, True)
    bad = ok_src.copy()
    bad[3] = ok_src[10]  # named twice
    assert call(src=bad) == (-1, True)
    assert call(null_src=True) == (-1, True)
    assert call(overlap=True)[0] == -1
    g2 = gi.copy()
    g2[3, 2] = n_old  # not a row of the old graph
    assert call(gi_=g2) == (-1, True)
    rc, same = call()
    assert rc == K and not same  # the same call with valid arguments is served
    ix.release()
