"""Filtered k-NN graphs without a GPU: a numpy restatement, in exact arithmetic, of nk_knn_graph_remap_filtered's host logic
equals a brute-force filtered rebuild (each row's list bounded by its own tag filter) after appends, rewrites, removals and
retags; the rows it searches again and the rows it offers new rows to are the expected ones; and the KnnIndex wrappers pass
filters through, or refuse before the library writes anything."""
import ctypes as C

import numpy as np
import pytest

PAD = 0xFFFFFFFF
NEW = 0xFFFFFFFF
NONE = (0xFFFFFFFFFFFFFFFF, 0xFFFFFFFFFFFFFFFF, 0)


def admits(tag, f):
    a, n, s = (int(x) for x in f)
    tag = int(tag)
    return (tag & a) == a and (tag & n) == 0 and (s == 0 or (tag & s) != 0)


def key(entry):
    return (entry[0], -entry[1])


def knn_list(X, tags, f, r, k, mask, floor):
    """nk_search_rows_filtered's list of row r: nk_search_filtered's best k' = min(k + 1, rows passing the mask) rows that r's
    filter admits, at or above the floor, then r itself dropped, or the last slot if r is not among them"""
    s = X @ X[r]
    n_adm = int(mask.sum())
    js = [j for j in np.nonzero(mask & (s >= floor))[0] if admits(tags[j], f[r])]
    js = sorted(js, key=lambda j: (-s[j], j))
    top = [(float(s[j]), int(j)) for j in js[:min(k + 1, n_adm)]]
    if any(j == r for _, j in top):
        top = [e for e in top if e[1] != r]
    elif len(top) == min(k + 1, n_adm):
        top = top[:-1]
    return top[:min(k, n_adm)]


def rebuild(X, tags, f, k, mask, floor):
    return [knn_list(X, tags, f, r, k, mask, floor) for r in range(len(X))]


def reverse_merge(X, tags, f, old, r, C_, k, mask, floor, row_side=True):
    """r's list after the reverse scan: the rows of C that r's filter admits (row_side) and that beat its k-th entry, or reach
    the floor if the list is short, merged with the old entries in key space"""
    s = X @ X[r]
    full = len(old) == k
    kth = key(old[-1]) if full else None
    entrants = [(float(s[q]), q) for q in C_ if q != r and mask[q] and s[q] >= floor and (not row_side or admits(tags[q], f[r]))
                and (not full or key((s[q], q)) > kth)]
    if not entrants:
        return old
    return sorted([(float(s[j]), j) for _, j in old] + entrants, key=key, reverse=True)[:k]


def plan(graph, src, k, mask):
    """(R, C): the rows searched again and the new or moved rows, as knn_graph_remap_locked decides them"""
    N = len(src)
    now_at = {o: f for f, o in enumerate(src) if o != NEW}
    C_ = [f for f in range(N) if src[f] != f]
    full = any(len(lst) == k for lst in graph)
    still = sum(1 for f in range(N) if src[f] != NEW and mask[f])
    everything = mask.sum() <= k or (not full and still <= k)
    R = set(C_) | {f for f in range(N) if src[f] == f and (everything or any(now_at.get(j) != j for _, j in graph[f]))}
    return R, C_


def remap(X, tags, f, graph, src, k, mask, floor, row_side=True):
    R, C_ = plan(graph, src, k, mask)
    return [knn_list(X, tags, f, r, k, mask, floor) if r in R else reverse_merge(X, tags, f, graph[r], r, C_, k, mask, floor, row_side)
            for r in range(len(X))]


class Store:
    """rows, tags, filters and the GraphRowMap of one filtered graph, changed together"""

    def __init__(self, X, tags, f, k, mask=None, floor=-np.inf):
        from nornicdb_b200.knn import GraphRowMap
        self.X, self.tags, self.f, self.k, self.floor = X.copy(), tags.copy(), f.copy(), k, floor
        self.mask = np.ones(len(X), bool) if mask is None else mask.copy()
        self.graph = rebuild(self.X, self.tags, self.f, k, self.mask, floor)
        self.map = GraphRowMap(len(X))

    def remove(self, r):
        for name in ("X", "tags", "f", "mask"):
            a = getattr(self, name)
            a[r] = a[-1]
            setattr(self, name, a[:-1].copy())
        self.map.remove_swap(r)

    def append(self, rows, tags, f, keep=True):
        self.X = np.concatenate([self.X, rows])
        self.tags = np.concatenate([self.tags, tags])
        self.f = np.concatenate([self.f, f])
        self.mask = np.concatenate([self.mask, np.full(len(rows), keep)])
        self.map.append(len(rows))

    def rewrite(self, r, v):
        self.X[r] = v
        self.map.update_row(r)

    def retag(self, r, tag, filt=None):
        """a new tag (and filter): reported with GraphRowMap.update_row, as a rewrite"""
        self.tags[r] = tag
        if filt is not None:
            self.f[r] = filt
        self.map.update_row(r)

    def got(self, **kw):
        return remap(self.X, self.tags, self.f, self.graph, self.map.src_of_row.tolist(), self.k, self.mask, self.floor, **kw)

    def want(self):
        return rebuild(self.X, self.tags, self.f, self.k, self.mask, self.floor)


def corpus(rng, n, d, lo=-3, hi=4):
    return rng.integers(lo, hi, (n, d)).astype(np.float64)


def tagged(rng, n, n_coll=6):
    """collection bit per row (Zipf-ish), filters "same collection" with some any_of / none_of / all_of variants"""
    coll = rng.choice(n_coll, n, p=np.array([0.45, 0.25, 0.15, 0.1, 0.05, 0.0]))
    tags = (1 << coll) | (rng.integers(0, 4, n) << 8)
    f = np.zeros((n, 3), np.uint64)
    f[:, 2] = (1 << coll).astype(np.uint64)
    kind = rng.integers(0, 10, n)
    f[kind == 1, 1] = 1 << 8
    f[kind == 2, 2] |= np.uint64(1 << 1)
    f[kind == 3] = (0, 0, 1 << 5)  # the empty collection
    f[kind == 4] = NONE
    f[kind == 5] = (1 << 9, 0, 0)
    return tags.astype(np.uint64), f


def store(seed, n=300, d=6, k=6, **kw):
    rng = np.random.default_rng(seed)
    tags, f = tagged(rng, n)
    return rng, Store(corpus(rng, n, d), tags, f, k, **kw)


def test_filtered_lists_respect_their_own_filter():
    _, st = store(1)
    for r, lst in enumerate(st.graph):
        assert all(admits(st.tags[j], st.f[r]) and j != r for _, j in lst)
    assert any(len(lst) == 0 for lst in st.graph)  # the filters that admit nothing, or the empty collection
    assert any(len(lst) == st.k for lst in st.graph)


def test_mixed_changes_equal_a_filtered_rebuild():
    rng, st = store(2)
    for step in range(80):
        op = step % 4
        if op == 0:
            st.remove(int(rng.integers(len(st.X))))
        elif op == 1:
            t, f = tagged(rng, 2)
            st.append(corpus(rng, 2, 6), t, f)
        elif op == 2:
            st.rewrite(int(rng.integers(len(st.X))), corpus(rng, 1, 6)[0])
        else:
            t, f = tagged(rng, 1)
            st.retag(int(rng.integers(len(st.X))), t[0], f[0])
    assert st.got() == st.want()


def test_which_rows_are_searched_again_and_which_are_offered_new_rows():
    rng, st = store(3, n=200)
    gone = 10
    listed_gone = {r for r, lst in enumerate(st.graph) if any(j == gone for _, j in lst)}
    last = len(st.X) - 1
    listed_last = {r for r, lst in enumerate(st.graph) if any(j == last for _, j in lst)}
    st.remove(gone)  # the last row moves into `gone`
    t, f = tagged(rng, 3)
    st.append(corpus(rng, 3, 6), t, f)
    st.retag(50, st.tags[50] ^ np.uint64(1 << 9))
    listed_50 = {r for r, lst in enumerate(st.graph) if any(j == 50 for _, j in lst)}
    R, C_ = plan(st.graph, st.map.src_of_row.tolist(), st.k, st.mask)
    assert C_ == [gone, 50] + list(range(len(st.X) - 3, len(st.X)))
    # searched again: new and moved rows, and kept rows whose list held the gone, moved or retagged row
    assert R == set(C_) | ((listed_gone | listed_last | listed_50) - {last})
    # every other row is offered C through the reverse scan, bounded by its own filter
    assert st.got() == st.want()


def test_retag_is_handled_as_a_rewrite():
    """A row that moves to another collection leaves the lists of its old collection and enters those of the new one; not
    reporting it leaves both stale"""
    rng, st = store(4, n=250)
    r = next(i for i in range(len(st.X)) if st.f[i][2] == 1 and st.tags[i] & 1)  # collection 0, "same collection"
    holders = [q for q, lst in enumerate(st.graph) if any(j == r for _, j in lst)]
    assert holders
    st.tags[r] = np.uint64(1 << 1)
    st.f[r] = (0, 0, 1 << 1)
    unreported = st.got()
    assert unreported != st.want()
    st.map.update_row(r)
    assert st.got() == st.want()


def test_short_lists_take_new_rows_at_the_floor():
    """A list short because few rows pass its filter has the floor as its threshold: a new row of its collection enters it
    through the reverse scan, with no special case"""
    rng = np.random.default_rng(5)
    n, k = 200, 6
    tags, f = tagged(rng, n)
    tags[:3] = 1 << 4 | 1 << 8
    tags[3:][(tags[3:] & (1 << 4)) != 0] = 1 << 0
    f[:3] = (0, 0, 1 << 4)
    st = Store(corpus(rng, n, 6), tags, f, k, floor=-1e9)
    assert all(len(st.graph[r]) == 2 for r in range(3))
    st.append(corpus(rng, 2, 6), np.array([1 << 4, 1 << 4], np.uint64), np.array([[0, 0, 1 << 4]] * 2, np.uint64))
    R, _ = plan(st.graph, st.map.src_of_row.tolist(), k, st.mask)
    assert not {0, 1, 2} & R  # the short lists go through the reverse scan
    got = st.got()
    assert got == st.want() and all(len(got[r]) == 4 for r in range(3))


def test_row_side_predicate_is_needed():
    """New rows beating the k-th entry of lists whose filters refuse them: without the row-side predicate the reverse scan
    lets them in"""
    rng = np.random.default_rng(6)
    n, k = 120, 5
    X = corpus(rng, n, 6)
    tags = np.where(np.arange(n) % 2 == 0, 1, 2).astype(np.uint64)
    f = np.zeros((n, 3), np.uint64)
    f[:, 2] = tags
    st = Store(X, tags, f, k)
    st.append(X[0:40:2] * 3, np.full(20, 2, np.uint64), np.array([[0, 0, 2]] * 20, np.uint64))  # collection-1 copies of 0-rows
    assert st.got() == st.want()
    assert st.got(row_side=False) != st.want()


@pytest.mark.parametrize("how", ["shrink", "few_admissible"])
def test_no_more_than_k_rows_pass_the_mask(how):
    rng = np.random.default_rng(7)
    k = 6
    if how == "shrink":
        _, st = store(7, n=k + 4, k=k)
        for _ in range(5):
            st.remove(int(rng.integers(len(st.X))))
    else:
        mask = np.zeros(60, bool)
        mask[[2, 9, 30, 41, 55]] = True
        _, st = store(8, n=60, k=k, mask=mask)
        st.remove(20)
        t, f = tagged(rng, 4)
        st.append(corpus(rng, 4, 6), t, f)
    assert st.got() == st.want()


def test_mask_and_floor():
    rng, st = store(9, n=300, k=8, mask=np.random.default_rng(90).random(300) > 0.25, floor=6.0)
    for r in (3, 100, 250):
        st.remove(r)
    t, f = tagged(rng, 5)
    st.append(corpus(rng, 5, 6), t, f, keep=False)
    t, f = tagged(rng, 5)
    st.append(corpus(rng, 5, 6), t, f, keep=True)
    assert st.got() == st.want()


# ---- the wrappers over a stand-in of the C calls ------------------------------------------------------------------------
class FakeLib:
    """records the filtered calls' arguments, refuses what the library refuses, else returns min(k, rows)"""

    def __init__(self, rows):
        self.rows, self.calls = rows, []

    def nk_index_rows(self, ptr):
        return self.rows

    def _filters(self, fp):
        return np.ctypeslib.as_array(C.cast(fp, C.POINTER(C.c_uint64)), (self.rows, 3)).copy()

    def nk_knn_graph_remap_filtered(self, ptr, k, n_old, src, fp, gi_in, gs_in, gi, gs, n_changed_out):
        s = np.ctypeslib.as_array(C.cast(src, C.POINTER(C.c_uint32)), (self.rows,)).copy()
        self.calls.append(("remap", k, n_old, s, self._filters(fp)))
        named = s[s != NEW]
        if k == 0 or k > 191 or (named >= n_old).any() or len(np.unique(named)) != len(named):
            return -1
        return min(k, self.rows)

    def nk_knn_graph_update_filtered(self, ptr, k, n_old, ch, n_ch, fp, gi, gs, n_changed_out):
        c = np.ctypeslib.as_array(C.cast(ch, C.POINTER(C.c_uint32)), (n_ch,)).copy() if n_ch else np.empty(0, np.uint32)
        self.calls.append(("update", k, n_old, c, self._filters(fp)))
        if k == 0 or k > 191 or (c >= n_old).any():
            return -1
        return min(k, self.rows)

    def nk_search_rows_filtered(self, ptr, rows, fp, Q, k, idx, sc):
        f = np.ctypeslib.as_array(C.cast(fp, C.POINTER(C.c_uint64)), (Q, 3)).copy()
        self.calls.append(("rows", Q, k, f))
        out = np.ctypeslib.as_array(C.cast(idx, C.POINTER(C.c_uint32)), (Q, k))
        out[:] = PAD
        np.ctypeslib.as_array(C.cast(sc, C.POINTER(C.c_float)), (Q, k))[:] = 0
        return min(k, self.rows)


def fake_index(rows):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex.__new__(KnnIndex)
    ix.lib, ix.ptr = FakeLib(rows), 1
    return ix


def test_wrappers_pass_filters_through():
    from nornicdb_b200.knn import GraphRowMap
    ix = fake_index(5)
    f = np.arange(15, dtype=np.uint64).reshape(5, 3)
    gi = np.full((5, 2), PAD, np.uint32)
    gs = np.zeros((5, 2), np.float32)
    m = GraphRowMap(5)
    m.update_row(2)  # a retag
    ix.remap_knn_graph(gi, gs, 5, m, k=3, filters=f)
    what, k, n_old, s, fc = ix.lib.calls[-1]
    assert (what, k, n_old, s.tolist()) == ("remap", 3, 5, [0, 1, NEW, 3, 4]) and (fc == f).all()
    ix.update_knn_graph(gi, gs, 5, changed=[2], filters=f.tolist())
    what, k, n_old, c, fc = ix.lib.calls[-1]
    assert (what, c.tolist()) == ("update", [2]) and (fc == f).all()
    i, s_ = ix.search_rows([0, 4], 3, filters=[(1, 2, 3), (4, 5, 6)])
    assert ix.lib.calls[-1][0] == "rows" and ix.lib.calls[-1][3].tolist() == [[1, 2, 3], [4, 5, 6]] and i.shape == (2, 3)


def test_refusals_before_the_library_writes():
    from nornicdb_b200.knn import KnnError
    ix = fake_index(5)
    gi = np.zeros((5, 2), np.uint32)
    gs = np.zeros((5, 2), np.float32)
    f = np.zeros((5, 3), np.uint64)
    for bad in (f[:4], np.zeros((6, 3), np.uint64), np.zeros(10, np.uint64)):
        with pytest.raises(KnnError):
            ix.remap_knn_graph(gi, gs, 5, list(range(5)), filters=bad)
        with pytest.raises(KnnError):
            ix.update_knn_graph(gi, gs, 5, filters=bad)
    with pytest.raises(KnnError):
        ix.search_rows([0, 1, 2], 3, filters=f[:2])
    assert ix.lib.calls == []
    with pytest.raises(KnnError):  # the library's own refusals raise
        ix.remap_knn_graph(gi, gs, 5, [0, 1, 1, 3, 4], filters=f)
    with pytest.raises(KnnError):
        ix.update_knn_graph(gi, gs, 5, changed=[7], filters=f)
