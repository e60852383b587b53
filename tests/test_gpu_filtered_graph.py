"""Tag filters for search by stored row and for k-NN graphs (nk_search_rows_filtered, nk_knn_graph_update_filtered,
nk_knn_graph_remap_filtered): search_rows(filters=...) equals nk_search_filtered over the stored rows with k + 1 and the self
rule, bit for bit; a filtered graph kept across append, rewrite, remove_swap and retag equals a filtered rebuild, bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PAD = 0xFFFFFFFF
BLOCK = 1024
K = 10
NONE = (0xFFFFFFFFFFFFFFFF, 0xFFFFFFFFFFFFFFFF, 0)  # admits no row


def make_index(rows, metric, dtype="f32", path="auto", devices=(0,)):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex(rows.shape[1], metric=metric, dtype=dtype, devices=devices)
    ix.upload_from_f32(rows)
    ix.set_path(path)
    return ix


def stored_f32(ix):
    from nornicdb_b200.knn import from_bf16_bits
    a = ix.read_rows(0, len(ix))
    return from_bf16_bits(a) if ix.dtype == 2 else a.astype(np.float32)


def admissible(ix_mask):
    return len(ix_mask) if ix_mask is None else int(np.count_nonzero(ix_mask))


def by_search_filtered(ix, ids, filters, k, n_adm):
    """the contract: nk_search_filtered(stored rows, filters, k' = min(k + 1, rows passing the mask)) per block of 1024,
    the query's own row dropped (or the last slot where it is not in the list), padded back to min(k, n_adm) columns"""
    x = stored_f32(ix)
    kk = min(k + 1, n_adm)
    ke = min(k, n_adm)
    oi, osc = [], []
    for b in range(0, len(ids), BLOCK):
        bid = ids[b:b + BLOCK]
        ri, rs = ix.search_filtered(x[bid], kk, filters[b:b + BLOCK])
        for q, self_row in enumerate(bid):
            li, ls = list(ri[q]), list(rs[q])
            drop = li.index(self_row) if self_row in li else len(li) - 1
            del li[drop], ls[drop]
            li, ls = li[:ke], ls[:ke]
            li += [PAD] * (ke - len(li))
            ls += [0.0] * (ke - len(ls))
            oi.append(np.array(li, np.uint32))
            osc.append(np.array(ls, np.float32))
    return np.stack(oi), np.stack(osc)


def assert_same(a, b, what=""):
    (ai, as_), (bi, bs) = a, b
    assert ai.shape == bi.shape, (what, ai.shape, bi.shape)
    bad = np.nonzero((ai != bi).any(axis=1) | (as_.view(np.uint32) != bs.view(np.uint32)).any(axis=1))[0]
    assert bad.size == 0, (what, bad[:5], ai[bad[:2]], bi[bad[:2]], as_[bad[:2]], bs[bad[:2]])


def collections(rng, n, n_coll=16, s=1.3):
    """collection id per row, Zipf-sized; collection 14 has 6 rows, collection 15 none"""
    w = 1.0 / np.arange(1, n_coll - 1) ** s
    coll = rng.choice(n_coll - 2, n - 6, p=w / w.sum())
    coll = np.concatenate([coll, np.full(6, n_coll - 2)])
    rng.shuffle(coll)
    return coll


def tags_of(coll, rng):
    """bit c: collection c; bits 16..19: labels, at random"""
    labels = rng.integers(0, 16, coll.size).astype(np.uint64) << np.uint64(16)
    return (np.uint64(1) << coll.astype(np.uint64)) | labels


def filters_of(coll, rng):
    """mostly "same collection" (any_of), some with a none_of label, some any_of two collections, a few empty collection 15,
    a few admitting nothing, a few unfiltered"""
    n = coll.size
    f = np.zeros((n, 3), np.uint64)
    f[:, 2] = np.uint64(1) << coll.astype(np.uint64)
    kind = rng.integers(0, 20, n)
    f[kind == 1, 1] = np.uint64(1 << 17)                                     # same collection, without label 17
    f[kind == 2, 2] |= np.uint64(1) << ((coll[kind == 2] + 1) % 14).astype(np.uint64)  # two collections
    f[kind == 3] = (0, 0, 1 << 15)                                           # the empty collection
    f[kind == 4] = NONE
    f[kind == 5] = (0, 0, 0)
    f[kind == 6] = (1 << 18, 0, 0)                                           # all_of a label, any collection
    return f


# ---- search by row with filters ---------------------------------------------------------------------------------------

def paths_for(dtype, metric):
    return ("auto", "simt", "shadow") + (("filter",) if dtype == "f32" else ())


CASES = [(dtype, metric, path) for dtype in ("f32", "f16", "bf16") for metric in ("cosine", "dot", "euclidean")
         for path in paths_for(dtype, metric)]


@pytest.mark.parametrize("dtype,metric,path", CASES)
def test_search_rows_filtered_equals_search_filtered(knn_lib, dtype, metric, path):
    from nornicdb_b200.knn import KnnError, admits
    rng = np.random.default_rng(CASES.index((dtype, metric, path)))
    n, d = 3000, 64
    rows = rng.standard_normal((n, d)).astype(np.float32)
    rows[100:104] = rows[50]  # duplicates
    coll = collections(rng, n)
    tags = tags_of(coll, rng)
    ix = make_index(rows, metric, dtype, path)
    ix.set_row_tags(tags)
    ids = np.concatenate([rng.choice(n, 1200, replace=False), [50, 100, 101]])  # two blocks
    f = filters_of(coll[ids], rng)
    f[0] = NONE                                         # admits nothing
    f[1] = (0, 0, 1 << int((coll[ids[1]] + 1) % 14))    # refuses the query's own row
    for k in (1, K, 191, 192, 1023, 1024):
        try:
            want = by_search_filtered(ix, ids, f, k, n)
        except KnnError:
            with pytest.raises(KnnError):
                ix.search_rows(ids, k, filters=f)
            continue
        got = ix.search_rows(ids, k, filters=f)
        assert_same(got, want, f"k={k}")
        assert np.all(got[0][0] == PAD)
        assert ids[1] not in got[0][1]
        for q in range(0, len(ids), 97):  # every listed row is admitted by the query's filter
            li = got[0][q][got[0][q] != PAD].astype(np.int64)
            assert admits(tags[li], *[int(x) for x in f[q]]).all()
    # filters=None is search_rows
    assert_same(ix.search_rows(ids, K, filters=None), ix.search_rows(ids, K))
    ix.release()


def test_search_rows_filtered_mask_floor_and_self(knn_lib):
    from nornicdb_b200.knn import admits
    rng = np.random.default_rng(31)
    n, d = 2000, 128
    rows = rng.standard_normal((n, d)).astype(np.float32)
    coll = collections(rng, n)
    tags = tags_of(coll, rng)
    ix = make_index(rows, "cosine", "f32", "shadow")
    ix.set_row_tags(tags)
    keep = rng.random(n) > 0.3
    ix.set_row_mask(keep)
    ix.set_min_score(0.05)
    ids = np.arange(0, n, 3)
    f = filters_of(coll[ids], rng)
    got = ix.search_rows(ids, K, filters=f)
    assert_same(got, by_search_filtered(ix, ids, f, K, int(keep.sum())))
    for q in range(len(ids)):
        li = got[0][q][got[0][q] != PAD].astype(np.int64)
        assert keep[li].all() and (li != ids[q]).all()
        assert admits(tags[li], *[int(x) for x in f[q]]).all()
        assert (got[1][q][:len(li)] >= 0.05).all()
    # a masked-out query row still gets its list
    masked = np.nonzero(~keep)[0][:50]
    fm = filters_of(coll[masked], rng)
    assert_same(ix.search_rows(masked, K, filters=fm), by_search_filtered(ix, masked, fm, K, int(keep.sum())))
    ix.release()


def test_search_rows_filtered_two_devices(knn_lib):
    from nornicdb_b200 import cuda
    if cuda.DeviceCount() < 2:
        pytest.skip("one device")
    rng = np.random.default_rng(32)
    n, d = 6000, 64
    rows = rng.standard_normal((n, d)).astype(np.float32)
    coll = collections(rng, n)
    ix = make_index(rows, "dot", "f32", "auto", devices=(0, 1))
    ix.set_row_tags(tags_of(coll, rng))
    ids = rng.choice(n, 1500, replace=False)
    f = filters_of(coll[ids], rng)
    assert_same(ix.search_rows(ids, K, filters=f), by_search_filtered(ix, ids, f, K, n))
    ix.release()


# ---- filtered graphs ----------------------------------------------------------------------------------------------------

class Tracked:
    """an index, its GraphRowMap, and each current row's collection, tag and filter, changed together"""

    def __init__(self, ix, coll, tags, filters):
        from nornicdb_b200.knn import GraphRowMap
        self.ix, self.map = ix, GraphRowMap(len(ix))
        self.coll, self.tags, self.f = coll.copy(), tags.copy(), filters.copy()
        self.changed = []  # update_knn_graph's changed rows, when nothing was removed

    def append(self, rows, coll, tags, filters):
        n0 = len(self.ix)
        self.ix.append(rows)
        self.ix.set_row_tags(tags, first_row=n0)
        self.map.append(len(rows))
        self.coll = np.concatenate([self.coll, coll])
        self.tags = np.concatenate([self.tags, tags])
        self.f = np.concatenate([self.f, filters])

    def rewrite(self, r, v):
        self.ix.update_row(int(r), v)
        self.map.update_row(int(r))
        self.changed.append(int(r))

    def retag(self, r, coll, tag, filt):
        """a row moves to another collection: new tag and new filter, reported as new contents"""
        self.ix.set_row_tags(np.array([tag], np.uint64), first_row=int(r))
        self.coll[r], self.tags[r], self.f[r] = coll, tag, filt
        self.map.update_row(int(r))
        self.changed.append(int(r))

    def remove(self, r):
        r = int(r)
        last = len(self.ix) - 1
        self.ix.remove_swap(r)
        self.map.remove_swap(r)
        for a in (self.coll, self.tags, self.f):
            a[r] = a[last]
        self.coll, self.tags, self.f = self.coll[:last], self.tags[:last], self.f[:last]


def lists_changed(gi, gs, ri, rs, kept):
    w = ri.shape[1]
    oi = np.full((len(kept), w), PAD, np.uint32)
    osc = np.zeros((len(kept), w), np.float32)
    oi[:, :min(w, gi.shape[1])] = gi[kept, :w]
    osc[:, :min(w, gs.shape[1])] = gs[kept, :w]
    return int(((ri[kept] != oi).any(axis=1) | (rs[kept].view(np.uint32) != osc.view(np.uint32)).any(axis=1)).sum())


def check_remap(t, gi, gs, k=K):
    ix, m = t.ix, t.map
    ui, us, nch = ix.remap_knn_graph(gi, gs, m.n_old, m, k=k, filters=t.f)
    want = ix.search_rows(np.arange(len(ix)), k, filters=t.f)
    assert_same((ui, us), want, "remap")
    src = m.src_of_row
    assert nch == lists_changed(gi, gs, *want, np.nonzero(src == np.arange(len(src)))[0])
    return want


def check_update(t, gi, gs, n_old, k=K):
    ix = t.ix
    ui, us, nch = ix.update_knn_graph(gi, gs, n_old, changed=t.changed, k=k, filters=t.f)
    want = ix.search_rows(np.arange(len(ix)), k, filters=t.f)
    assert_same((ui, us), want, "update")
    assert nch == lists_changed(gi, gs, *want, np.arange(n_old))
    return want


def base_graph(rng, n, d, metric, dtype, path):
    rows = rng.uniform(-1, 1, (n, d)).astype(np.float32)
    coll = collections(rng, n)
    tags = tags_of(coll, rng)
    f = filters_of(coll, rng)
    f[coll == 14] = (0, 0, 1 << 14)  # the small collection's lists hold its other 5 rows: short
    ix = make_index(rows, metric, dtype, path)
    ix.set_row_tags(tags)
    t = Tracked(ix, coll, tags, f)
    gi, gs = ix.search_rows(np.arange(n), K, filters=f)
    return t, gi, gs


GRAPH_CASES = [(path, metric, dtype) for path, dtype in (("shadow", "f32"), ("shadow", "bf16"), ("filter", "f32"))
               for metric in ("cosine", "dot", "euclidean")]


@pytest.mark.parametrize("path,metric,dtype", GRAPH_CASES)
def test_filtered_remap_equals_filtered_rebuild(knn_lib, path, metric, dtype):
    rng = np.random.default_rng(100 + GRAPH_CASES.index((path, metric, dtype)))
    n, d = 3000, 64
    t, gi, gs = base_graph(rng, n, d, metric, dtype, path)
    small = np.nonzero(t.coll == 14)[0]
    assert len(small) <= K and ((gi[small] != PAD).sum(axis=1) == len(small) - 1).all()  # short lists
    # mixed: appends (two into the small collection, near copies of one of its rows), rewrites, removals, retags and a
    # filter change
    add = rng.uniform(-1, 1, (40, d)).astype(np.float32)
    add[:5] = stored_f32(t.ix)[small[0]] + (1e-3 * rng.standard_normal((5, d))).astype(np.float32)
    ac = rng.choice(14, 40)
    ac[:2] = 14
    t.append(add, ac, tags_of(ac, rng), filters_of(ac, rng))
    t.rewrite(3, rng.uniform(-1, 1, d).astype(np.float32))
    t.remove(7)
    t.remove(len(t.ix) - 1)
    t.retag(11, 2, np.uint64(1 << 2), np.array([0, 0, 1 << 2], np.uint64))
    r = int(np.nonzero(t.coll == 0)[0][5])
    t.f[r] = (0, 0, 1 << 1)  # its filter changed: reported as new contents
    t.map.update_row(r)
    t.remove(int(small[1]))
    t.append(rng.uniform(-1, 1, (3, d)).astype(np.float32), np.array([14, 15, 0]), tags_of(np.array([14, 15, 0]), rng),
             filters_of(np.array([14, 15, 0]), rng))
    check_remap(t, gi, gs)
    t.ix.release()


@pytest.mark.parametrize("path", ("shadow", "filter"))
def test_filtered_update_equals_filtered_rebuild(knn_lib, path):
    rng = np.random.default_rng(7 if path == "shadow" else 8)
    n, d = 2500, 128
    t, gi, gs = base_graph(rng, n, d, "cosine", "f32", path)
    add = np.concatenate([t.ix.read_rows(5, 20) + 1e-3, rng.uniform(-1, 1, (30, d)).astype(np.float32)])
    ac = rng.choice(15, 50)
    t.append(add, ac, tags_of(ac, rng), filters_of(ac, rng))
    for r in (3, 40, 41):
        t.rewrite(r, rng.uniform(-1, 1, d).astype(np.float32))
    t.retag(100, 4, np.uint64(1 << 4), np.array([0, 0, 1 << 4], np.uint64))
    t.retag(101, 14, np.uint64(1 << 14), np.array([0, 1 << 16, 1 << 14], np.uint64))
    check_update(t, gi, gs, n)
    # unfiltered update of an unfiltered graph through filters=None is update_knn_graph as before
    t.ix.release()


@pytest.mark.parametrize("path", ("shadow", "filter"))
def test_row_side_filter_keeps_refused_rows_out(knn_lib, path):
    """New rows that beat the k-th entry of many lists whose filters refuse them: the reverse scan must not offer them."""
    rng = np.random.default_rng(55)
    n, d = 2000, 64
    rows = rng.uniform(-1, 1, (n, d)).astype(np.float32)
    coll = (np.arange(n) % 2).astype(np.int64)  # collections 0 and 1, interleaved
    tags = (np.uint64(1) << coll.astype(np.uint64))
    f = np.zeros((n, 3), np.uint64)
    f[:, 2] = tags  # same collection only
    ix = make_index(rows, "cosine", "f32", path)
    ix.set_row_tags(tags)
    t = Tracked(ix, coll, tags, f)
    gi, gs = ix.search_rows(np.arange(n), K, filters=f)
    # near copies of collection-0 rows, tagged collection 1: they would top their originals' lists
    src = np.arange(0, 200, 2)
    add = rows[src] + 1e-4
    t.append(add, np.ones(len(src), np.int64), np.full(len(src), 2, np.uint64), np.tile(np.array([0, 0, 2], np.uint64), (len(src), 1)))
    want = check_update(t, gi, gs, n)
    new_ids = np.arange(n, n + len(src))
    assert not np.isin(want[0][src], new_ids).any()  # collection-0 lists do not list collection-1 rows
    # and the same rows tagged collection 0 do enter them
    ix.set_row_tags(np.ones(len(src), np.uint64), first_row=n)
    t.f[n:] = (0, 0, 1)
    want2 = check_update(t, gi, gs, n)
    assert np.isin(want2[0][src], new_ids).any(axis=1).all()
    ix.release()


def test_filtered_graph_refusals_write_nothing(knn_lib):
    from nornicdb_b200.knn import KnnError
    rng = np.random.default_rng(9)
    n, d = 500, 64
    t, gi, gs = base_graph(rng, n, d, "cosine", "f32", "shadow")
    with pytest.raises(KnnError):
        t.ix.remap_knn_graph(gi, gs, n, t.map, filters=t.f[:-1])  # one filter short
    with pytest.raises(KnnError):
        t.ix.update_knn_graph(gi, gs, n, filters=t.f[:-1])
    src = t.map.src_of_row
    src[3] = src[4]
    with pytest.raises(KnnError):
        t.ix.remap_knn_graph(gi, gs, n, src, filters=t.f)  # repeated source
    with pytest.raises(KnnError):
        t.ix.update_knn_graph(gi, gs, n, changed=[n + 5], filters=t.f)  # not an old row
    t.ix.set_path("simt")
    with pytest.raises(KnnError):
        t.ix.update_knn_graph(gi, gs, n, filters=t.f)
    t.ix.release()
