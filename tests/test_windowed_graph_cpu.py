"""Windowed k-NN graphs without a GPU: a numpy restatement, in exact arithmetic, of nk_knn_graph_remap_windowed's host logic
equals a brute-force windowed rebuild (each row's list bounded by its own value window, and its tag filter) after appends,
rewrites, re-valued rows, window changes and removals; the row-side window test of the reverse scan is needed; short lists
take new in-window rows at the floor; window edges are inclusive at every key; and the KnnIndex wrappers pass windows
through, or refuse before the library writes anything."""
import ctypes as C

import numpy as np
import pytest

from nornicdb_b200.knn import EMPTY_WINDOW, band_windows

PAD = 0xFFFFFFFF
NEW = 0xFFFFFFFF
TOP = 0xFFFFFFFFFFFFFFFF


def admits(tag, f):
    a, n, s = (int(x) for x in f)
    tag = int(tag)
    return (tag & a) == a and (tag & n) == 0 and (s == 0 or (tag & s) != 0)


def in_window(v, w):
    return int(w[0]) <= int(v) <= int(w[1])


def key(entry):
    return (entry[0], -entry[1])


def ok(st, r, j):
    """may row j appear in row r's list: r's filter admits j's tag and r's window admits j's value key"""
    return admits(st.tags[j], st.f[r]) and in_window(st.keys[j], st.w[r])


def knn_list(st, r):
    """nk_search_rows_windowed's list of row r: nk_search_windowed's best k' = min(k + 1, rows passing the mask) rows that r's
    filter and window admit, at or above the floor, then r itself dropped, or the last slot if r is not among them"""
    s = st.X @ st.X[r]
    n_adm = int(st.mask.sum())
    js = [j for j in np.nonzero(st.mask & (s >= st.floor))[0] if ok(st, r, j)]
    js = sorted(js, key=lambda j: (-s[j], j))
    top = [(float(s[j]), int(j)) for j in js[:min(st.k + 1, n_adm)]]
    if any(j == r for _, j in top):
        top = [e for e in top if e[1] != r]
    elif len(top) == min(st.k + 1, n_adm):
        top = top[:-1]
    return top[:min(st.k, n_adm)]


def reverse_merge(st, old, r, C_, row_side):
    """r's list after the reverse scan: the rows of C that r's filter and (row_side) r's window admit, and that beat its k-th
    entry, or reach the floor if the list is short, merged with the old entries in key space"""
    s = st.X @ st.X[r]
    full = len(old) == st.k
    kth = key(old[-1]) if full else None
    entrants = [(float(s[q]), q) for q in C_ if q != r and st.mask[q] and s[q] >= st.floor and admits(st.tags[q], st.f[r])
                and (not row_side or in_window(st.keys[q], st.w[r])) and (not full or key((s[q], q)) > kth)]
    if not entrants:
        return old
    return sorted([(float(s[j]), j) for _, j in old] + entrants, key=key, reverse=True)[:st.k]


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


class Store:
    """rows, tags, filters, value keys, windows and the GraphRowMap of one windowed graph, changed together.  gap: the band
    half-width of band windows (None: the windows are given and kept as they are)"""

    def __init__(self, X, tags, f, keys, w, k, mask=None, floor=-np.inf, gap=None):
        from nornicdb_b200.knn import GraphRowMap
        self.X, self.tags, self.f, self.keys, self.w = X.copy(), tags.copy(), f.copy(), keys.copy(), w.copy()
        self.k, self.floor, self.gap = k, floor, gap
        self.mask = np.ones(len(X), bool) if mask is None else mask.copy()
        self.graph = self.want()
        self.map = GraphRowMap(len(X))

    def remove(self, r):
        for name in ("X", "tags", "f", "keys", "w", "mask"):
            a = getattr(self, name)
            a[r] = a[-1]
            setattr(self, name, a[:-1].copy())
        self.map.remove_swap(r)

    def append(self, rows, keys, tags=None, f=None, keep=True):
        n = len(rows)
        self.X = np.concatenate([self.X, rows])
        self.tags = np.concatenate([self.tags, np.zeros(n, np.uint64) if tags is None else tags])
        self.f = np.concatenate([self.f, np.zeros((n, 3), np.uint64) if f is None else f])
        self.keys = np.concatenate([self.keys, np.asarray(keys, np.uint64)])
        self.w = np.concatenate([self.w, band_windows(keys, self.gap) if self.gap is not None else np.tile(self.w[:1], (n, 1))])
        self.mask = np.concatenate([self.mask, np.full(n, keep)])
        self.map.append(n)

    def rewrite(self, r, v):
        self.X[r] = v
        self.map.update_row(r)

    def revalue(self, r, key, report=True):
        """a new value key (a band window moves with it): reported with GraphRowMap.update_row, as a rewrite"""
        self.keys[r] = key
        if self.gap is not None:
            self.w[r] = band_windows([key], self.gap)[0]
        if report:
            self.map.update_row(r)

    def rewindow(self, r, w):
        self.w[r] = w
        self.map.update_row(r)

    def got(self, row_side=True):
        R, C_ = plan(self.graph, self.map.src_of_row.tolist(), self.k, self.mask)
        return [knn_list(self, r) if r in R else reverse_merge(self, self.graph[r], r, C_, row_side) for r in range(len(self.X))]

    def want(self):
        return [knn_list(self, r) for r in range(len(self.X))]


def corpus(rng, n, d, lo=-3, hi=4):
    return rng.integers(lo, hi, (n, d)).astype(np.float64)


DAY = 86_400


def stamps(rng, n, span=60 * DAY):
    """timestamps over two months (1 s units), a few rows without a value (key 0)"""
    k = rng.integers(1, span, n).astype(np.uint64)
    k[rng.random(n) < 0.03] = 0
    return k


def store(seed, n=300, d=6, k=6, filtered=False, **kw):
    rng = np.random.default_rng(seed)
    keys = stamps(rng, n)
    tags = np.zeros(n, np.uint64)
    f = np.zeros((n, 3), np.uint64)
    if filtered:
        coll = rng.integers(0, 3, n)
        tags = (1 << coll).astype(np.uint64)
        f[:, 2] = tags
        f[rng.random(n) < 0.2] = 0
    return rng, Store(corpus(rng, n, d), tags, f, keys, band_windows(keys, 4 * DAY), k, gap=4 * DAY, **kw)


def test_windowed_lists_respect_their_own_window():
    _, st = store(1)
    for r, lst in enumerate(st.graph):
        assert all(in_window(st.keys[j], st.w[r]) and j != r for _, j in lst)
    assert any(len(lst) == 0 for lst in st.graph)  # the rows without a value: their window admits nothing
    assert any(len(lst) == st.k for lst in st.graph)


@pytest.mark.parametrize("filtered", [False, True])
def test_mixed_changes_equal_a_windowed_rebuild(filtered):
    rng, st = store(2, filtered=filtered)
    for step in range(100):
        op = step % 5
        r = int(rng.integers(len(st.X)))
        if op == 0:
            st.remove(r)
        elif op == 1:
            st.append(corpus(rng, 2, 6), stamps(rng, 2), st.tags[:2].copy(), st.f[:2].copy())
        elif op == 2:
            st.rewrite(r, corpus(rng, 1, 6)[0])
        elif op == 3:
            st.revalue(r, int(st.keys[r]) + 7 * DAY)
        else:
            st.rewindow(r, (int(st.w[r][0]), int(st.w[r][1]) + 10 * DAY))
    assert st.got() == st.want()


def test_revalue_must_be_reported():
    """A row moved by a week leaves the lists of its old neighbourhood in time and enters those of its new one; not reporting
    it leaves both stale"""
    rng, st = store(3, n=250)
    r = next(i for i, lst in enumerate(st.graph) if lst and any(any(j == i for _, j in o) for o in st.graph))
    st.revalue(r, int(st.keys[r]) + 7 * DAY, report=False)
    assert st.got() != st.want()
    st.map.update_row(r)
    assert st.got() == st.want()


def test_row_side_predicate_is_needed():
    """Near copies of old rows keyed outside their originals' windows: they beat those lists' k-th entries, yet must not
    enter.  Without the row-side window test the reverse scan lets them in.  Re-valued into the windows and reported, they
    enter."""
    rng = np.random.default_rng(6)
    n, k = 150, 5
    X = corpus(rng, n, 6)
    keys = np.arange(1, n + 1, dtype=np.uint64) * np.uint64(DAY)
    st = Store(X, np.zeros(n, np.uint64), np.zeros((n, 3), np.uint64), keys, band_windows(keys, 10 * DAY), k, gap=10 * DAY)
    far = keys[0:40:2] + np.uint64(30 * DAY)
    st.append(X[0:40:2] * 3, far)
    got = st.got()
    assert got == st.want()
    assert st.got(row_side=False) != st.want()
    for i in range(20):
        assert all(j != n + i for _, j in got[2 * i])  # no copy entered its original's list
    st.graph, st.map = got, type(st.map)(len(st.X))
    for i in range(20):
        st.revalue(n + i, int(keys[2 * i]))
    got = st.got()
    assert got == st.want()
    assert sum(any(j == n + i for _, j in got[2 * i]) for i in range(20)) >= 15


def test_short_lists_take_new_in_window_rows_at_the_floor():
    """A list short because its window holds fewer than k other rows has the floor as its threshold: a new row inside the
    window enters it through the reverse scan, with no special case"""
    rng = np.random.default_rng(5)
    n, k = 200, 6
    keys = (np.arange(n, dtype=np.uint64) + np.uint64(1)) * np.uint64(DAY)
    keys[:3] = [10_000 * DAY, 10_000 * DAY + 1, 10_000 * DAY + 2]  # three rows far from the rest
    st = Store(corpus(rng, n, 6), np.zeros(n, np.uint64), np.zeros((n, 3), np.uint64), keys, band_windows(keys, DAY // 2), k,
               floor=-1e9, gap=DAY // 2)
    assert all(len(st.graph[r]) == 2 for r in range(3))
    st.append(corpus(rng, 2, 6), [10_000 * DAY + 3, 10_000 * DAY - 5])
    R, _ = plan(st.graph, st.map.src_of_row.tolist(), k, st.mask)
    assert not {0, 1, 2} & R  # the short lists go through the reverse scan
    got = st.got()
    assert got == st.want() and all(len(got[r]) == 4 for r in range(3))


def test_window_edges_and_extreme_keys():
    """Inclusive edges, key 0, empty windows (lo > hi) and keys at 1 and 2^64 - 1"""
    rng = np.random.default_rng(8)
    n, k = 60, 4
    X = corpus(rng, n, 5)
    keys = rng.integers(2, 1000, n).astype(np.uint64)
    keys[:6] = [0, 1, TOP, TOP - 1, 500, 0]
    w = np.tile(np.array([[1, TOP]], np.uint64), (n, 1))
    w[10] = (500, 500)              # exactly one key
    w[11] = (1, 1)                  # only key 1
    w[12] = (TOP, TOP)              # only the top key
    w[13] = EMPTY_WINDOW            # lo > hi: nothing
    w[14] = (0, TOP)                # every key, 0 included
    w[15] = (0, 0)                  # only rows without a value
    st = Store(X, np.zeros(n, np.uint64), np.zeros((n, 3), np.uint64), keys, w, k)
    assert {j for _, j in st.graph[10]} <= {j for j in range(n) if keys[j] == 500}
    assert {j for _, j in st.graph[11]} == {1}
    assert {j for _, j in st.graph[12]} == {2}
    assert st.graph[13] == []
    assert {j for _, j in st.graph[15]} == {0, 5}
    # new rows at every edge
    st.append(X[[10, 11, 12, 14, 15, 20]] * 2, [500, 1, TOP, 0, 0, 499], keep=True)
    assert st.got() == st.want()
    got = st.got()
    assert {j for _, j in got[11]} == {1, n + 1} and {j for _, j in got[12]} == {2, n + 2} and got[13] == []
    assert {n + 3, n + 4} <= {j for _, j in got[15]}
    assert n + 5 not in {j for _, j in got[10]}


def test_band_windows_at_the_ends_of_the_key_space():
    w = band_windows(np.array([1, 2, TOP, TOP - 1, 0], np.uint64), 3)
    assert w[:4].tolist() == [[1, 4], [1, 5], [TOP - 3, TOP], [TOP - 4, TOP]]
    assert int(w[4][0]) > int(w[4][1])  # key 0: the empty window


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
        st.append(corpus(rng, 4, 6), stamps(rng, 4))
    assert st.got() == st.want()


def test_mask_and_floor():
    rng, st = store(9, n=300, k=8, mask=np.random.default_rng(90).random(300) > 0.25, floor=6.0)
    for r in (3, 100, 250):
        st.remove(r)
    st.append(corpus(rng, 5, 6), stamps(rng, 5), keep=False)
    st.append(corpus(rng, 5, 6), stamps(rng, 5), keep=True)
    assert st.got() == st.want()


# ---- the wrappers over a stand-in of the C calls ------------------------------------------------------------------------
class FakeLib:
    """records the windowed calls' arguments, refuses what the library refuses, else returns min(k, rows)"""

    def __init__(self, rows):
        self.rows, self.calls = rows, []

    def nk_index_rows(self, ptr):
        return self.rows

    def _arr(self, p, cols):
        return None if p is None else np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint64)), (self.rows, cols)).copy()

    def nk_knn_graph_remap_windowed(self, ptr, k, n_old, src, fp, wp, gi_in, gs_in, gi, gs, n_changed_out):
        s = np.ctypeslib.as_array(C.cast(src, C.POINTER(C.c_uint32)), (self.rows,)).copy()
        self.calls.append(("remap", k, n_old, s, self._arr(fp, 3), self._arr(wp, 2)))
        named = s[s != NEW]
        if k == 0 or k > 191 or (named >= n_old).any() or len(np.unique(named)) != len(named):
            return -1
        return min(k, self.rows)

    def nk_knn_graph_update_windowed(self, ptr, k, n_old, ch, n_ch, fp, wp, gi, gs, n_changed_out):
        c = np.ctypeslib.as_array(C.cast(ch, C.POINTER(C.c_uint32)), (n_ch,)).copy() if n_ch else np.empty(0, np.uint32)
        self.calls.append(("update", k, n_old, c, self._arr(fp, 3), self._arr(wp, 2)))
        if k == 0 or k > 191 or (c >= n_old).any():
            return -1
        return min(k, self.rows)

    def nk_knn_graph_remap_filtered(self, ptr, k, n_old, src, fp, gi_in, gs_in, gi, gs, n_changed_out):
        self.calls.append(("remap_filtered",))
        return min(k, self.rows)

    def nk_knn_graph_update_filtered(self, ptr, k, n_old, ch, n_ch, fp, gi, gs, n_changed_out):
        self.calls.append(("update_filtered",))
        return min(k, self.rows)


def fake_index(rows):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex.__new__(KnnIndex)
    ix.lib, ix.ptr = FakeLib(rows), 1
    return ix


def test_wrappers_pass_windows_through():
    from nornicdb_b200.knn import GraphRowMap
    ix = fake_index(5)
    w = band_windows(np.arange(1, 6, dtype=np.uint64) * np.uint64(10), 5)
    f = np.arange(15, dtype=np.uint64).reshape(5, 3)
    gi = np.full((5, 2), PAD, np.uint32)
    gs = np.zeros((5, 2), np.float32)
    m = GraphRowMap(5)
    m.update_row(2)  # a re-valued row
    ix.remap_knn_graph(gi, gs, 5, m, k=3, windows=w)
    what, k, n_old, s, fc, wc = ix.lib.calls[-1]
    assert (what, k, n_old, s.tolist(), fc) == ("remap", 3, 5, [0, 1, NEW, 3, 4], None) and (wc == w).all()
    ix.update_knn_graph(gi, gs, 5, changed=[2], filters=f, windows=w.tolist())
    what, k, n_old, c, fc, wc = ix.lib.calls[-1]
    assert (what, c.tolist()) == ("update", [2]) and (fc == f).all() and (wc == w).all()
    # windows=None: the filtered calls, as before
    ix.remap_knn_graph(gi, gs, 5, m, filters=f)
    ix.update_knn_graph(gi, gs, 5, filters=f)
    assert [c[0] for c in ix.lib.calls[-2:]] == ["remap_filtered", "update_filtered"]


def test_refusals_before_the_library_writes():
    from nornicdb_b200.knn import KnnError
    ix = fake_index(5)
    gi = np.zeros((5, 2), np.uint32)
    gs = np.zeros((5, 2), np.float32)
    w = np.zeros((5, 2), np.uint64)
    for bad in (w[:4], np.zeros((6, 2), np.uint64), np.zeros(10, np.uint64), np.zeros((5, 3), np.uint64), w[0]):
        with pytest.raises(KnnError):
            ix.remap_knn_graph(gi, gs, 5, list(range(5)), windows=bad)
        with pytest.raises(KnnError):
            ix.update_knn_graph(gi, gs, 5, windows=bad)
    assert ix.lib.calls == []
    with pytest.raises(KnnError):  # the library's own refusals raise
        ix.remap_knn_graph(gi, gs, 5, [0, 1, 1, 3, 4], windows=w)
    with pytest.raises(KnnError):
        ix.update_knn_graph(gi, gs, 5, changed=[7], windows=w)
