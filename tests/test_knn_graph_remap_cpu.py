"""The k-NN graph remap without a GPU: a numpy restatement of nk_knn_graph_remap's algorithm with exact arithmetic equals a
rebuild after removals (swap with the last row), appends and rewrites; GraphRowMap follows the index's renumbering; and
KnnIndex.remap_knn_graph's argument handling over a stand-in of the C call."""
import ctypes as C

import numpy as np
import pytest

from fake_knn import FakeKnnIndex

PAD = 0xFFFFFFFF
NEW = 0xFFFFFFFF


# ---- the algorithm, restated with exact keys ---------------------------------------------------------------------------
# Integer-valued vectors and the dot product in fp64 make every score exact, so equal scores are true ties, broken by row id
# as the library's keys break them.
def key(entry):
    return (entry[0], -entry[1])


def knn_list(X, r, k, mask, floor):
    """nk_search_rows' list of row r: the scan's best k' = min(k + 1, admissible) rows at or above the floor, then r itself
    dropped, or the last slot if r is not among them; min(k, admissible) slots"""
    s = X @ X[r]
    n_adm = int(mask.sum())
    js = np.nonzero(mask & (s >= floor))[0]
    top = [(float(s[j]), int(j)) for j in js[np.lexsort((js, -s[js]))][:min(k + 1, n_adm)]]
    if any(j == r for _, j in top):
        top = [e for e in top if e[1] != r]
    elif len(top) == min(k + 1, n_adm):
        top = top[:-1]
    return top[:min(k, n_adm)]


def rebuild(X, k, mask, floor):
    return [knn_list(X, r, k, mask, floor) for r in range(len(X))]


def reverse_merge(X, old, r, C, k, mask, floor):
    """r's list after the reverse scan: the rows of C that beat its k-th entry (or reach the floor if it is short), merged
    with the old entries in key space"""
    s = X @ X[r]
    full = len(old) == k
    kth = key(old[-1]) if full else None
    entrants = [(float(s[q]), q) for q in C if q != r and mask[q] and s[q] >= floor and (not full or key((s[q], q)) > kth)]
    if not entrants:
        return old
    return sorted([(float(s[j]), j) for _, j in old] + entrants, key=key, reverse=True)[:k]


def remap(X, graph, src, k, mask, floor):
    """nk_knn_graph_remap: search again the new and moved rows and the kept rows whose list holds a row no longer at its
    id; reverse-scan the new and moved rows for every other kept row"""
    N, n_old = len(X), len(graph)
    now_at = {o: f for f, o in enumerate(src) if o != NEW}
    C = [f for f in range(N) if src[f] != f]
    full = any(len(lst) == k for lst in graph)
    still = sum(1 for f in range(N) if src[f] != NEW and mask[f])
    everything = mask.sum() <= k or (not full and still <= k)
    R = set(C) | {f for f in range(N) if src[f] == f and (everything or any(now_at.get(j) != j for _, j in graph[f]))}
    out = [None] * N
    for f in range(N):
        out[f] = knn_list(X, f, k, mask, floor) if f in R else reverse_merge(X, graph[f], f, C, k, mask, floor)
    assert n_old >= max([o for o in src if o != NEW], default=-1) + 1
    return out


def remap_by_relabelling(X, graph, src, k, mask, floor):
    """The tempting shortcut: a moved row keeps its old list, entries renamed to the rows' new ids, and only new rows are
    offered to the others.  It misses that a moved row's tie-break key changes with its id."""
    N = len(X)
    now_at = {o: f for f, o in enumerate(src) if o != NEW}
    C = [f for f in range(N) if src[f] == NEW]
    out = []
    for f in range(N):
        o = src[f]
        if o == NEW or any(j not in now_at for _, j in graph[o]):
            out.append(knn_list(X, f, k, mask, floor))
        else:
            out.append(reverse_merge(X, [(s, now_at[j]) for s, j in graph[o]], f, C, k, mask, floor))
    return out


class Store:
    """The index's rows and the GraphRowMap of one graph, changed together"""

    def __init__(self, X, k, mask=None, floor=-np.inf):
        from nornicdb_b200.knn import GraphRowMap
        self.X, self.k, self.floor = X.copy(), k, floor
        self.mask = np.ones(len(X), bool) if mask is None else mask.copy()
        self.graph = rebuild(self.X, k, self.mask, floor)
        self.map = GraphRowMap(len(X))

    def remove(self, r):
        self.X[r], self.mask[r] = self.X[-1], self.mask[-1]
        self.X, self.mask = self.X[:-1].copy(), self.mask[:-1].copy()
        self.map.remove_swap(r)

    def append(self, rows, keep=True):
        self.X = np.concatenate([self.X, rows])
        self.mask = np.concatenate([self.mask, np.full(len(rows), keep)])
        self.map.append(len(rows))

    def rewrite(self, r, v):
        self.X[r] = v
        self.map.update_row(r)

    def check(self, fn=remap):
        got = fn(self.X, self.graph, self.map.src_of_row.tolist(), self.k, self.mask, self.floor)
        return got == rebuild(self.X, self.k, self.mask, self.floor)


def corpus(rng, n, d, lo=-3, hi=4):
    return rng.integers(lo, hi, (n, d)).astype(np.float64)


@pytest.mark.parametrize("where", ["middle", "last", "first"])
def test_single_removal(where):
    rng = np.random.default_rng(1)
    st = Store(corpus(rng, 400, 6), 8)  # few distinct values: many exact ties
    st.remove({"middle": 171, "last": 399, "first": 0}[where])
    assert st.check()


def test_moved_row_enters_its_former_neighbours_list():
    rng = np.random.default_rng(2)
    st = Store(corpus(rng, 300, 6), 6)
    last = len(st.X) - 1
    x = st.graph[last][0][1]  # the last row's best neighbour: the last row moves into its id
    st.remove(x)
    assert st.check()


def test_hub_row_removed():
    rng = np.random.default_rng(3)
    X = corpus(rng, 500, 5)
    X[7] = 20.0  # near the top of many dot-product lists
    st = Store(X, 6)
    counts = np.bincount([j for lst in st.graph for _, j in lst], minlength=len(X))
    hub = int(np.argmax(counts))
    assert counts[hub] > 50
    st.remove(hub)
    assert st.check()


def test_the_same_contents_move_twice():
    rng = np.random.default_rng(4)
    st = Store(corpus(rng, 300, 6), 7)
    n = len(st.X)
    st.remove(n - 3)  # row n-1's contents move to n-3
    st.remove(10)     # row n-2's to 10
    st.remove(20)     # row n-3 is the last row now: the first contents move again, to 20
    assert st.map.src_of_row[20] == n - 1
    assert st.check()


def test_remove_an_appended_row_and_append_after_removal():
    rng = np.random.default_rng(5)
    st = Store(corpus(rng, 300, 6), 6)
    st.append(corpus(rng, 4, 6))
    st.remove(301)  # an appended row, replaced by the last appended one
    st.remove(5)    # an old row, replaced by an appended one
    st.append(corpus(rng, 2, 6))
    assert st.check()


def test_interleaved_removals_appends_and_rewrites():
    rng = np.random.default_rng(6)
    st = Store(corpus(rng, 400, 6), 8)
    for step in range(60):
        op = step % 3
        if op == 0:
            st.remove(int(rng.integers(len(st.X))))
        elif op == 1:
            st.append(corpus(rng, 1, 6))
        else:
            st.rewrite(int(rng.integers(len(st.X))), corpus(rng, 1, 6)[0])
    assert st.check()


def test_removals_under_a_mask_and_a_floor():
    rng = np.random.default_rng(7)
    X = corpus(rng, 400, 6)
    st = Store(X, 10, mask=rng.random(400) > 0.25, floor=12.0)
    assert any(len(lst) < 10 for lst in st.graph)
    for r in (3, 100, 250):
        st.remove(r)
    st.append(corpus(rng, 5, 6), keep=False)  # masked-out new rows enter no list
    assert st.check()


@pytest.mark.parametrize("how", ["shrink", "remove_then_grow"])
def test_no_more_than_k_admissible_rows(how):
    """While no more than k rows are admissible, nk_search_rows drops a real entry from an inadmissible row's list: the
    remap searches every row again when that held before or holds now, though the rows that were removed have no mask bit"""
    rng = np.random.default_rng(8)
    k = 6
    if how == "shrink":
        st = Store(corpus(rng, k + 4, 6), k)
        for _ in range(5):
            st.remove(int(rng.integers(len(st.X))))  # k - 1 rows remain
    else:
        mask = np.zeros(60, bool)
        mask[[2, 9, 30, 41, 55]] = True  # 5 <= k admissible: every old list is short
        st = Store(corpus(rng, 60, 6), k, mask=mask)
        st.remove(20)  # an inadmissible row; the last row, also inadmissible, moves into its id
        st.append(corpus(rng, 4, 6))  # 9 admissible now: the inadmissible rows' old lists lack a real entry
    assert st.check()
    if how == "remove_then_grow":
        # without the rule the inadmissible rows keep their short old lists
        def no_rule(X, graph, src, k, mask, floor):
            N = len(X)
            now_at = {o: f for f, o in enumerate(src) if o != NEW}
            C_ = [f for f in range(N) if src[f] != f]
            R = set(C_) | {f for f in range(N) if src[f] == f and any(now_at.get(j) != j for _, j in graph[f])}
            return [knn_list(X, f, k, mask, floor) if f in R else reverse_merge(X, graph[f], f, C_, k, mask, floor) for f in range(N)]
        assert not st.check(no_rule)


def test_tie_trap_needs_the_moved_row_rule():
    """Exact duplicates A (row a) and B (the last row): in row r's list A holds the k-th slot and B, one id higher, misses it.
    Removing a row x < a moves B to id x, ahead of A: B takes the k-th slot of r's list.  No row in that list moved or went,
    so only the reverse scan of moved rows finds it."""
    rng = np.random.default_rng(9)
    k = 5
    X = corpus(rng, 200, 8, -50, 51)
    r = 17
    s = X @ X[r]
    order = [j for j in np.lexsort((np.arange(len(X)), -s)) if j != r]
    a = int(order[k - 1])  # r's k-th neighbour
    assert s[order[k - 2]] > s[a] > s[order[k]]  # its score is not tied with another row's
    X = np.concatenate([X, X[a:a + 1]])  # B = a copy of A, the last row
    st = Store(X, k)
    assert [j for _, j in st.graph[r]][-1] == a
    listed = {j for _, j in st.graph[r]}
    x = next(j for j in range(a) if j != r and j not in listed)
    st.remove(x)
    expect = rebuild(st.X, k, st.mask, st.floor)
    assert [j for _, j in expect[r]][-1] == x  # B, now at x, beats A on row id
    assert st.check()
    assert not st.check(remap_by_relabelling)


# ---- GraphRowMap against a direct simulation of swap-with-last ----------------------------------------------------------
def test_row_map_follows_swap_with_last():
    """Rows of a stand-in index carry their origin as their value (old row o: o, new contents: -1); after random appends,
    rewrites and removals the map's src_of_row is what the rows say"""
    from nornicdb_b200.knn import ROW_NEW, GraphRowMap
    rng = np.random.default_rng(10)
    n_old = 50
    ix = FakeKnnIndex(1)
    ix.upload(np.arange(n_old, dtype=np.float32).reshape(-1, 1))
    m = GraphRowMap(n_old)
    for _ in range(400):
        op = rng.integers(4)
        if op == 0 or len(ix) == 0:
            n = int(rng.integers(1, 4))
            ix.append(np.full((n, 1), -1, np.float32))
            m.append(n)
        elif op == 1:
            r = int(rng.integers(len(ix)))
            ix.update_row(r, np.array([-1], np.float32))
            m.update_row(r)
        else:
            r = int(rng.integers(len(ix)))
            ix.remove_swap(r)
            m.remove_swap(r)
        v = ix.read_rows(0, len(ix))[:, 0].astype(np.int64)
        expect = np.where(v < 0, ROW_NEW, v).astype(np.uint32)
        assert len(m) == len(ix) and (m.src_of_row == expect).all()
    assert m.n_old == n_old


def test_row_map_refuses_rows_out_of_range():
    from nornicdb_b200.knn import GraphRowMap, KnnError
    m = GraphRowMap(3)
    for bad in (3, -1):
        with pytest.raises(KnnError):
            m.remove_swap(bad)
        with pytest.raises(KnnError):
            m.update_row(bad)


# ---- KnnIndex.remap_knn_graph over a stand-in of the C call -------------------------------------------------------------
class FakeLib:
    """nk_knn_graph_remap's contract on the host: records the arguments, refuses what the library refuses, else returns
    min(k, rows) and writes row f's first slot as f."""

    def __init__(self, rows, max_k=191):
        self.rows, self.max_k, self.calls = rows, max_k, []

    def nk_index_rows(self, ptr):
        return self.rows

    def nk_knn_graph_remap(self, ptr, k, n_old, src, gi_in, gs_in, gi, gs, n_changed_out):
        s = np.ctypeslib.as_array(C.cast(src, C.POINTER(C.c_uint32)), (self.rows,)).copy() if src else None
        ii = np.ctypeslib.as_array(C.cast(gi_in, C.POINTER(C.c_uint32)), (n_old, k)).copy()
        si = np.ctypeslib.as_array(C.cast(gs_in, C.POINTER(C.c_float)), (n_old, k)).copy()
        idx = np.ctypeslib.as_array(C.cast(gi, C.POINTER(C.c_uint32)), (self.rows, k))
        self.calls.append((k, n_old, s, ii, si))
        if k == 0 or k > self.max_k or (s is None and self.rows):
            return -1
        named = s[s != NEW]
        if (named >= n_old).any() or len(np.unique(named)) != len(named):
            return -1
        if ((ii != PAD) & (ii >= n_old)).any():
            return -1
        idx[:, 0] = np.arange(self.rows)
        n_changed_out._obj.value = 2
        return min(k, self.rows)


def fake_index(rows):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex.__new__(KnnIndex)
    ix.lib, ix.ptr = FakeLib(rows), 1
    return ix


def test_remap_pads_narrow_graphs_and_takes_a_row_map():
    from nornicdb_b200.knn import GraphRowMap
    ix = fake_index(4)
    m = GraphRowMap(5)
    m.remove_swap(1)
    m.append(1)
    m.remove_swap(4)  # the appended row removed again
    m.remove_swap(0)
    assert m.src_of_row.tolist() == [3, 4, 2]
    ix.lib.rows = len(m)
    gi = np.full((5, 3), PAD, np.uint32)
    gi[:, :2] = 1
    gs = np.ones((5, 3), np.float32)
    ui, us, n = ix.remap_knn_graph(gi, gs, 5, m, k=6)
    k, n_old, src, ii, si = ix.lib.calls[-1]
    assert (k, n_old, src.tolist()) == (6, 5, m.src_of_row.tolist())
    assert (ii[:, :3] == gi).all() and (ii[:, 3:] == PAD).all() and (si[:, :3] == 1).all() and (si[:, 3:] == 0).all()
    assert ui.shape == (3, 3) and us.shape == (3, 3) and n == 2  # k' = min(k, rows)
    assert ui[:, 0].tolist() == [0, 1, 2] and (ui[:, 1:] == PAD).all() and (us == 0).all()


def test_remap_argument_errors():
    from nornicdb_b200.knn import KnnError
    ix = fake_index(4)
    gi = np.zeros((5, 3), np.uint32)
    gs = np.zeros((5, 3), np.float32)
    src = [0, 1, 2, 3]
    with pytest.raises(KnnError):
        ix.remap_knn_graph(gi, gs[:, :2], 5, src)  # shapes differ
    with pytest.raises(KnnError):
        ix.remap_knn_graph(gi, gs, 4, src)  # n_old is not the graph's row count
    with pytest.raises(KnnError):
        ix.remap_knn_graph(gi, gs, 5, src, k=2)  # k narrower than the graph
    with pytest.raises(KnnError):
        ix.remap_knn_graph(gi, gs, 5, src[:3])  # one entry per current row
    with pytest.raises(KnnError):
        ix.remap_knn_graph(gi, gs, 5, [0, 1, -2, 3])
    assert ix.lib.calls == []


@pytest.mark.parametrize("case", ["k_too_big", "src_not_old", "src_repeated", "entry_not_old"])
def test_every_library_refusal_raises(case):
    from nornicdb_b200.knn import KnnError
    ix = fake_index(4)
    gi = np.zeros((5, 3), np.uint32)
    gs = np.zeros((5, 3), np.float32)
    src = [0, 1, 2, NEW]
    kw = {}
    if case == "k_too_big":
        kw["k"] = 192
    elif case == "src_not_old":
        src[3] = 5
    elif case == "src_repeated":
        src[3] = 1
    else:
        gi[1, 1] = 5
    with pytest.raises(KnnError):
        ix.remap_knn_graph(gi, gs, 5, src, **kw)
    assert len(ix.lib.calls) == 1
