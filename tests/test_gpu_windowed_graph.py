"""Windowed k-NN graphs kept exact across updates (nk_knn_graph_update_windowed, nk_knn_graph_remap_windowed): a time-local
graph (each row's list bounded by its own +-band around its value key, and optionally its tag filter) kept across append,
rewrite, remove_swap, re-valued rows and window changes equals search_rows(every row, k, filters=, windows=), bit for bit, on
the int8 image, the BF16 shadow, bf16 rows in place and the TF32 filter.  New rows outside a list's window never enter it,
however close they are; windows=None is the filtered call."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PAD = 0xFFFFFFFF
K = 10
DAY = 86_400
T0 = 1_700_000_000  # value keys: timestamps in seconds
GAP = DAY


def make_index(monkeypatch, rows, metric, dtype="f32", path="shadow", image=None, devices=(0,)):
    from nornicdb_b200.knn import KnnIndex
    if image is not None:
        monkeypatch.setenv("NK_SHADOW", image)  # read at creation
    ix = KnnIndex(rows.shape[1], metric=metric, dtype=dtype, devices=devices)
    ix.upload_from_f32(rows)
    ix.set_path(path)
    return ix


def assert_same(a, b, what=""):
    (ai, as_), (bi, bs) = a, b
    assert ai.shape == bi.shape, (what, ai.shape, bi.shape)
    bad = np.nonzero((ai != bi).any(axis=1) | (as_.view(np.uint32) != bs.view(np.uint32)).any(axis=1))[0]
    assert bad.size == 0, (what, bad[:5], ai[bad[:2]], bi[bad[:2]], as_[bad[:2]], bs[bad[:2]])


def stamps(rng, n, days=60):
    """uniform timestamps over `days` days; about 1 % of rows without a value (key 0: their window admits nothing)"""
    k = (T0 + rng.integers(0, days * DAY, n)).astype(np.uint64)
    k[rng.random(n) < 0.01] = 0
    return k


def bands(keys):
    from nornicdb_b200.knn import band_windows
    return band_windows(keys, GAP)


def collections_of(rng, n):
    coll = rng.integers(0, 4, n)
    tags = np.uint64(1) << coll.astype(np.uint64)
    f = np.zeros((n, 3), np.uint64)
    f[:, 2] = tags
    f[rng.random(n) < 0.2] = 0  # unfiltered lists
    return tags, f


class Tracked:
    """an index, its GraphRowMap, and each current row's value key, window, tag and filter (filters None: an unfiltered
    windowed graph), changed together"""

    def __init__(self, ix, keys, tags=None, filters=None):
        from nornicdb_b200.knn import GraphRowMap
        self.ix, self.map = ix, GraphRowMap(len(ix))
        self.keys, self.w = keys.copy(), bands(keys)
        self.tags = None if tags is None else tags.copy()
        self.f = None if filters is None else filters.copy()
        ix.set_row_values(self.keys)
        if tags is not None:
            ix.set_row_tags(self.tags)
        self.changed = []  # update_knn_graph's changed rows, when nothing was removed

    def graph(self, k=K):
        return self.ix.search_rows(np.arange(len(self.ix)), k, filters=self.f, windows=self.w)

    def append(self, rows, keys, rng=None):
        n0 = len(self.ix)
        self.ix.append(rows)
        self.ix.set_row_values(keys, first_row=n0)
        self.map.append(len(rows))
        self.keys = np.concatenate([self.keys, keys])
        self.w = np.concatenate([self.w, bands(keys)])
        if self.f is not None:
            tags, f = collections_of(rng, len(rows))
            self.ix.set_row_tags(tags, first_row=n0)
            self.tags = np.concatenate([self.tags, tags])
            self.f = np.concatenate([self.f, f])

    def rewrite(self, r, v):
        self.ix.update_row(int(r), v)
        self.map.update_row(int(r))
        self.changed.append(int(r))

    def revalue(self, r, key):
        """a new value key; the band window moves with it: reported as new contents"""
        self.ix.set_row_values(np.array([key], np.uint64), first_row=int(r))
        self.keys[r] = key
        self.w[r] = bands(np.array([key], np.uint64))[0]
        self.map.update_row(int(r))
        self.changed.append(int(r))

    def rewindow(self, r, lo, hi):
        self.w[r] = (lo, hi)
        self.map.update_row(int(r))
        self.changed.append(int(r))

    def remove(self, r):
        r = int(r)
        last = len(self.ix) - 1
        self.ix.remove_swap(r)
        self.map.remove_swap(r)
        arrays = [self.keys, self.w] + ([] if self.f is None else [self.tags, self.f])
        for a in arrays:
            a[r] = a[last]
        self.keys, self.w = self.keys[:last], self.w[:last]
        if self.f is not None:
            self.tags, self.f = self.tags[:last], self.f[:last]


def lists_changed(gi, gs, ri, rs, kept):
    w = ri.shape[1]
    oi = np.full((len(kept), w), PAD, np.uint32)
    osc = np.zeros((len(kept), w), np.float32)
    oi[:, :min(w, gi.shape[1])] = gi[kept, :w]
    osc[:, :min(w, gs.shape[1])] = gs[kept, :w]
    return int(((ri[kept] != oi).any(axis=1) | (rs[kept].view(np.uint32) != osc.view(np.uint32)).any(axis=1)).sum())


def check_remap(t, gi, gs, k=K):
    m = t.map
    ui, us, nch = t.ix.remap_knn_graph(gi, gs, m.n_old, m, k=k, filters=t.f, windows=t.w)
    want = t.graph(k)
    assert_same((ui, us), want, "remap")
    src = m.src_of_row
    assert nch == lists_changed(gi, gs, *want, np.nonzero(src == np.arange(len(src)))[0])
    return want


def check_update(t, gi, gs, n_old, k=K):
    ui, us, nch = t.ix.update_knn_graph(gi, gs, n_old, changed=t.changed, k=k, filters=t.f, windows=t.w)
    want = t.graph(k)
    assert_same((ui, us), want, "update")
    assert nch == lists_changed(gi, gs, *want, np.arange(n_old))
    return want


def base(monkeypatch, rng, n, d, metric, dtype, path, image, filtered, k=K):
    rows = rng.uniform(-1, 1, (n, d)).astype(np.float32)
    keys = stamps(rng, n)
    keys[-4:] = T0 + 500 * DAY + np.arange(4)  # four rows alone in their day: short lists
    ix = make_index(monkeypatch, rows, metric, dtype, path, image)
    tags, f = collections_of(rng, n) if filtered else (None, None)
    t = Tracked(ix, keys, tags, f)
    gi, gs = t.graph(k)
    return t, rows, gi, gs


# (image, path, dtype): the int8 image and the BF16 shadow of fp32 rows, bf16 rows scanned in place, the TF32 filter
PATHS = [("int8", "shadow", "f32"), ("bf16", "shadow", "f32"), (None, "shadow", "bf16"), (None, "filter", "f32")]
CASES = [(p, metric, filtered) for p in range(len(PATHS)) for metric in ("cosine", "dot", "euclidean") for filtered in (False, True)]


def mixed_changes(t, rng, rows, d):
    n = len(t.ix)
    lone = n - 1
    add = rng.uniform(-1, 1, (60, d)).astype(np.float32)
    add[:3] = rows[lone] + (1e-3 * rng.standard_normal((3, d))).astype(np.float32)
    akeys = stamps(rng, 60)
    akeys[:2] = T0 + 500 * DAY + 10          # into the lone day: its short lists take them
    akeys[2] = T0 + 400 * DAY                 # a near copy far from the lone day: it enters no lone list
    akeys[3:30] = T0 + 59 * DAY + rng.integers(0, DAY, 27).astype(np.uint64)  # the realistic insert: the last day
    t.append(add, akeys, rng)
    t.rewrite(3, rng.uniform(-1, 1, d).astype(np.float32))
    t.remove(7)
    t.revalue(11, int(t.keys[11]) + 7 * DAY if t.keys[11] else T0)
    t.revalue(12, 0)                         # the row loses its value: it leaves every list, its own list empties
    t.rewindow(13, int(t.w[13][0]), int(t.w[13][1]) + 5 * DAY)
    t.remove(len(t.ix) - 1)
    t.remove(int(rng.integers(100, 1000)))
    t.append(rng.uniform(-1, 1, (3, d)).astype(np.float32), stamps(rng, 3), rng)


@pytest.mark.parametrize("p,metric,filtered", CASES)
def test_windowed_remap_equals_windowed_rebuild(knn_lib, monkeypatch, p, metric, filtered):
    image, path, dtype = PATHS[p]
    rng = np.random.default_rng(200 + CASES.index((p, metric, filtered)))
    n, d = 3000, 64
    t, rows, gi, gs = base(monkeypatch, rng, n, d, metric, dtype, path, image, filtered)
    if not filtered:
        assert ((gi[-4:] != PAD).sum(axis=1) == 3).all()  # the lone day's lists are short
    assert (gi[t.keys == 0] == PAD).all()  # rows without a value: empty lists
    mixed_changes(t, rng, rows, d)
    want = check_remap(t, gi, gs)
    if not filtered:
        lone = [r for r in range(len(t.ix)) if t.keys[r] >= T0 + 500 * DAY]
        assert len(lone) >= 5 and all((want[0][r] != PAD).sum() == len(lone) - 1 for r in lone)
    t.ix.release()


@pytest.mark.parametrize("p", range(len(PATHS)))
def test_windowed_update_equals_windowed_rebuild(knn_lib, monkeypatch, p):
    image, path, dtype = PATHS[p]
    rng = np.random.default_rng(300 + p)
    n, d = 2500, 128
    t, rows, gi, gs = base(monkeypatch, rng, n, d, "cosine", dtype, path, image, p % 2 == 1)
    add = np.concatenate([rows[5:25] + 1e-3, rng.uniform(-1, 1, (30, d)).astype(np.float32)])
    t.append(add, stamps(rng, 50), rng)
    for r in (3, 40, 41):
        t.rewrite(r, rng.uniform(-1, 1, d).astype(np.float32))
    t.revalue(100, int(t.keys[100]) + 7 * DAY if t.keys[100] else T0)
    t.revalue(101, T0 + 500 * DAY + 100)     # into the lone day
    t.rewindow(102, 1, (1 << 64) - 1)        # every row with a value
    check_update(t, gi, gs, n)
    t.ix.release()


@pytest.mark.parametrize("p", range(len(PATHS)))
def test_row_side_window_keeps_out_of_window_rows_out(knn_lib, monkeypatch, p):
    """Near copies of old rows, keyed three days after their originals: they beat the k-th entry of their originals' lists,
    yet lie outside those lists' windows and must not enter.  Re-valued into the windows and reported, they do enter."""
    image, path, dtype = PATHS[p]
    rng = np.random.default_rng(55 + p)
    n, d = 2000, 64
    rows = rng.uniform(-1, 1, (n, d)).astype(np.float32)
    keys = (T0 + np.arange(n) * 600).astype(np.uint64)  # one row every 10 minutes: ~290 rows per band
    ix = make_index(monkeypatch, rows, "cosine", dtype, path, image)
    t = Tracked(ix, keys)
    gi, gs = t.graph()
    src = np.arange(0, 400, 4)
    t.append(rows[src] + 1e-4, keys[src] + np.uint64(3 * DAY))
    want = check_update(t, gi, gs, n)
    new_ids = np.arange(n, n + len(src))
    assert not (want[0][src] == new_ids[:, None]).any()  # no copy in its original's list
    # re-valued into their originals' windows and reported as changed: each copy tops its original's list
    gi2, gs2 = want
    t.changed = []
    for i, r in enumerate(src):
        t.revalue(n + i, int(keys[r]) + 60)
    want2 = check_update(t, gi2, gs2, len(t.ix))
    assert (want2[0][src] == new_ids[:, None]).any(axis=1).all()
    ix.release()


def test_windows_none_is_the_filtered_call(knn_lib, monkeypatch):
    """nk_knn_graph_update_windowed / _remap_windowed with windows NULL: the _filtered calls' output, bit for bit"""
    rng = np.random.default_rng(71)
    n, d, k = 2000, 64, K
    rows = rng.uniform(-1, 1, (n, d)).astype(np.float32)
    ix = make_index(monkeypatch, rows, "dot", "f32", "shadow")
    tags, f = collections_of(rng, n)
    ix.set_row_tags(tags)
    gi, gs = ix.search_rows(np.arange(n), k, filters=f)
    ix.append(rng.uniform(-1, 1, (30, d)).astype(np.float32))
    ix.update_row(4, rng.uniform(-1, 1, d).astype(np.float32))
    nt, nf = collections_of(rng, 30)
    ix.set_row_tags(nt, first_row=n)
    f = np.ascontiguousarray(np.concatenate([f, nf]))
    N = len(ix)
    ch = np.array([4], np.uint32)
    vp = C.c_void_p
    outs = []
    for name in ("nk_knn_graph_update_filtered", "nk_knn_graph_update_windowed"):
        g_i = np.full((N, k), PAD, np.uint32)
        g_s = np.zeros((N, k), np.float32)
        g_i[:n], g_s[:n] = gi, gs
        nch = C.c_uint64(0)
        extra = (None,) if name.endswith("windowed") else ()
        rc = getattr(ix.lib, name)(ix.ptr, k, n, ch.ctypes.data_as(vp), 1, f.ctypes.data_as(vp), *extra, g_i.ctypes.data_as(vp),
                                   g_s.ctypes.data_as(vp), C.byref(nch))
        assert rc == k, ix.lib.nk_last_error()
        outs.append((g_i, g_s, nch.value))
    assert_same(outs[0][:2], outs[1][:2])
    assert outs[0][2] == outs[1][2]
    assert_same(outs[0][:2], ix.search_rows(np.arange(N), k, filters=f))
    src = np.arange(N, dtype=np.uint32)
    src[4] = PAD
    remaps = []
    for name in ("nk_knn_graph_remap_filtered", "nk_knn_graph_remap_windowed"):
        g_i = np.full((N, k), PAD, np.uint32)
        g_s = np.zeros((N, k), np.float32)
        oi, osc = np.ascontiguousarray(outs[0][0]), np.ascontiguousarray(outs[0][1])
        nch = C.c_uint64(0)
        extra = (None,) if name.endswith("windowed") else ()
        rc = getattr(ix.lib, name)(ix.ptr, k, N, src.ctypes.data_as(vp), f.ctypes.data_as(vp), *extra, oi.ctypes.data_as(vp),
                                   osc.ctypes.data_as(vp), g_i.ctypes.data_as(vp), g_s.ctypes.data_as(vp), C.byref(nch))
        assert rc == k, ix.lib.nk_last_error()
        remaps.append((g_i, g_s, nch.value))
    assert_same(remaps[0][:2], remaps[1][:2])
    assert remaps[0][2] == remaps[1][2]
    ix.release()


def test_windowed_graph_mask_and_floor(knn_lib, monkeypatch):
    rng = np.random.default_rng(81)
    n, d = 3000, 64
    rows = rng.uniform(-1, 1, (n, d)).astype(np.float32)
    ix = make_index(monkeypatch, rows, "cosine", "f32", "shadow")
    keep = rng.random(n) > 0.3
    ix.set_row_mask(keep)
    ix.set_min_score(0.1)
    t = Tracked(ix, stamps(rng, n))
    gi, gs = t.graph()
    for r in (3, 100, 2500):
        t.remove(r)
        keep[r] = keep[len(keep) - 1]
        keep = keep[:-1]
    t.append(rng.uniform(-1, 1, (40, d)).astype(np.float32), stamps(rng, 40))
    keep = np.concatenate([keep, rng.random(40) > 0.5])
    ix.set_row_mask(keep)  # append clears the mask: set it again
    t.revalue(50, T0 + 3 * DAY)
    want = check_remap(t, gi, gs)
    for r in range(0, len(ix), 37):
        li = want[0][r][want[0][r] != PAD].astype(np.int64)
        assert keep[li].all() and (want[1][r][:len(li)] >= 0.1).all()
        lo, hi = int(t.w[r][0]), int(t.w[r][1])
        assert all(lo <= int(t.keys[j]) <= hi for j in li)
    ix.release()


@pytest.mark.parametrize("k", (1, 10, 191))
def test_windowed_graph_k(knn_lib, monkeypatch, k):
    rng = np.random.default_rng(90 + k)
    n, d = 2000, 64
    t, rows, gi, gs = base(monkeypatch, rng, n, d, "euclidean", "f32", "shadow", None, False, k=k)
    mixed_changes(t, rng, rows, d)
    check_remap(t, gi, gs, k=k)
    t.ix.release()


def test_windowed_graph_two_devices(knn_lib, monkeypatch):
    from nornicdb_b200 import cuda
    if cuda.DeviceCount() < 2:
        pytest.skip("one device")
    rng = np.random.default_rng(95)
    n, d = 6000, 64
    rows = rng.uniform(-1, 1, (n, d)).astype(np.float32)
    ix = make_index(monkeypatch, rows, "dot", "f32", "shadow", devices=(0, 1))
    tags, f = collections_of(rng, n)
    t = Tracked(ix, stamps(rng, n), tags, f)
    gi, gs = t.graph()
    mixed_changes(t, rng, rows, d)
    check_remap(t, gi, gs)
    ix.release()


def test_windowed_graph_refusals_write_nothing(knn_lib, monkeypatch):
    from nornicdb_b200.knn import KnnError
    rng = np.random.default_rng(9)
    n, d = 500, 64
    t, rows, gi, gs = base(monkeypatch, rng, n, d, "cosine", "f32", "shadow", None, False)
    with pytest.raises(KnnError):
        t.ix.remap_knn_graph(gi, gs, n, t.map, windows=t.w[:-1])  # one window short
    with pytest.raises(KnnError):
        t.ix.update_knn_graph(gi, gs, n, windows=t.w[:-1])
    vp = C.c_void_p
    w = np.ascontiguousarray(t.w)
    for path, k in (("simt", K), ("shadow", 192)):
        t.ix.set_path(path)
        g_i = np.full((n, k), 7, np.uint32)
        g_s = np.full((n, k), 2.0, np.float32)
        rc = t.ix.lib.nk_knn_graph_update_windowed(t.ix.ptr, k, n, None, 0, None, w.ctypes.data_as(vp), g_i.ctypes.data_as(vp),
                                                   g_s.ctypes.data_as(vp), None)
        assert rc == -1 and (g_i == 7).all() and (g_s == 2.0).all(), (path, k)
        with pytest.raises(KnnError):
            t.ix.update_knn_graph(gi, gs, n, k=k, windows=t.w)
    t.ix.release()
