"""The k-NN graph update without a GPU: a numpy restatement of nk_knn_graph_update's algorithm with exact arithmetic equals a
rebuild, and KnnIndex.update_knn_graph's argument handling over a stand-in of the C call."""
import ctypes as C

import numpy as np
import pytest

PAD = 0xFFFFFFFF


# ---- the algorithm, restated with exact keys ---------------------------------------------------------------------------
# Integer-valued vectors and the dot product in fp64 make every score exact, so equal scores are true ties, broken by row id
# as the library's keys break them.  A NaN score ranks as -inf, as warp_exact_score makes it.
def scores(X, r):
    with np.errstate(invalid="ignore"):
        s = X @ X[r]
    return np.where(np.isnan(s), -np.inf, s)


def knn_list(X, r, k, mask, floor):
    """search_rows' list of row r: the best k other admissible rows at or above the floor, by (score desc, row asc)"""
    s = scores(X, r)
    ok = mask & (s >= floor)
    ok[r] = False
    js = np.nonzero(ok)[0]
    order = np.lexsort((js, -s[js]))[:k]
    return [(float(s[js[i]]), int(js[i])) for i in order]


def rebuild(X, k, mask, floor):
    return [knn_list(X, r, k, mask, floor) for r in range(len(X))]


def key(entry):
    return (entry[0], -entry[1])


def update(X, graph, n_old, changed, k, mask, floor):
    """Steps 1-4: search R again, reverse-scan the other old rows with their own thresholds, merge in key space."""
    N = len(X)
    ch = set(int(c) for c in changed)
    C = sorted(ch) + list(range(n_old, N))
    R = set(C) | {r for r in range(n_old) if any(j in ch for _, j in graph[r])}
    out = list(graph) + [None] * (N - n_old)
    for r in R:
        out[r] = knn_list(X, r, k, mask, floor)
    for r in range(n_old):
        if r in R:
            continue
        s = scores(X, r)
        full = len(graph[r]) == k
        kth = key(graph[r][-1]) if full else None
        entrants = [(float(s[q]), q) for q in C if q != r and mask[q] and s[q] >= floor and (not full or key((s[q], q)) > kth)]
        if entrants:
            old = [(float(s[j]), j) for _, j in graph[r]]  # the old entries' keys, recomputed
            out[r] = sorted(old + entrants, key=key, reverse=True)[:k]
    return out


def corpus(rng, n, d, lo=-3, hi=4):
    return rng.integers(lo, hi, (n, d)).astype(np.float64)


@pytest.mark.parametrize("n_new", [1, 5, 1500])
def test_appends_equal_a_rebuild(n_new):
    rng = np.random.default_rng(n_new)
    n_old, k = 600, 8
    X = corpus(rng, n_old + n_new, 6)  # few distinct values: many exact ties
    mask = np.ones(len(X), bool)
    g = rebuild(X[:n_old], k, mask[:n_old], -np.inf)
    assert update(X, g, n_old, [], k, mask, -np.inf) == rebuild(X, k, mask, -np.inf)


def test_rewritten_rows_in_many_lists():
    rng = np.random.default_rng(1)
    n_old, k = 500, 6
    X = corpus(rng, n_old + 20, 5)
    mask = np.ones(len(X), bool)
    g = rebuild(X[:n_old], k, mask[:n_old], -np.inf)
    X[7] = 20.0  # a row of large entries is near the top of many dot-product lists before and after the rewrite
    g = rebuild(X[:n_old], k, mask[:n_old], -np.inf)
    counts = np.bincount([j for lst in g for _, j in lst], minlength=n_old)
    hubs = np.argsort(-counts)[:3]
    assert counts[hubs[0]] > 50
    for h in hubs:
        X[h] = rng.integers(-3, 4, 5)
    X[11] = X[11] * 3
    changed = list(hubs) + [11, 11]
    assert update(X, g, n_old, changed, k, mask, -np.inf) == rebuild(X, k, mask, -np.inf)


def test_a_copy_of_the_kth_neighbour_loses_the_tie_on_row_id():
    rng = np.random.default_rng(2)
    n_old, k = 300, 5
    X = corpus(rng, n_old + 1, 8)
    mask = np.ones(len(X), bool)
    g = rebuild(X[:n_old], k, mask[:n_old], -np.inf)
    X[n_old] = X[g[0][-1][1]]
    new = update(X, g, n_old, [], k, mask, -np.inf)
    assert new == rebuild(X, k, mask, -np.inf)
    assert n_old not in [j for _, j in new[0]]  # same score as the k-th entry, higher row id


def test_short_lists_under_a_floor_and_masked_new_rows():
    rng = np.random.default_rng(3)
    n_old, k = 400, 10
    X = corpus(rng, n_old + 60, 6)
    mask = rng.random(len(X)) > 0.25
    floor = 12.0
    g = rebuild(X[:n_old], k, mask[:n_old], floor)
    assert any(len(lst) < k for lst in g)
    new = update(X, g, n_old, [4], k, mask, floor)
    assert new == rebuild(X, k, mask, floor)
    masked_new = {q for q in range(n_old, len(X)) if not mask[q]}
    assert masked_new and not any(j in masked_new for lst in new for _, j in lst)


def test_nan_rows_old_and_new():
    rng = np.random.default_rng(4)
    n_old, k = 300, 6
    X = corpus(rng, n_old + 10, 6)
    X[5, 2] = np.nan
    X[n_old + 3, 0] = np.nan
    mask = np.ones(len(X), bool)
    g = rebuild(X[:n_old], k, mask[:n_old], -np.inf)
    X[9, 1] = np.nan
    assert update(X, g, n_old, [9], k, mask, -np.inf) == rebuild(X, k, mask, -np.inf)


# ---- KnnIndex.update_knn_graph over a stand-in of the C call -------------------------------------------------------------
class FakeLib:
    """nk_knn_graph_update's contract on the host: records the arguments, refuses what the library refuses, else returns
    min(k, rows) and writes row r's first slot as r."""

    def __init__(self, rows, max_k=191):
        self.rows, self.max_k, self.calls = rows, max_k, []

    def nk_index_rows(self, ptr):
        return self.rows

    def nk_knn_graph_update(self, ptr, k, n_old, changed, n_changed, gi, gs, n_changed_out):
        ch = np.ctypeslib.as_array(C.cast(changed, C.POINTER(C.c_uint32)), (n_changed,)).copy() if n_changed else np.empty(0, np.uint32)
        idx = np.ctypeslib.as_array(C.cast(gi, C.POINTER(C.c_uint32)), (self.rows, k))
        sc = np.ctypeslib.as_array(C.cast(gs, C.POINTER(C.c_float)), (self.rows, k))
        self.calls.append((k, n_old, ch, idx.copy(), sc.copy()))
        if k == 0 or k > self.max_k or n_old > self.rows or (ch >= n_old).any():
            return -1
        bad = idx[:n_old]
        if ((bad != PAD) & (bad >= n_old)).any():
            return -1
        idx[:, 0] = np.arange(self.rows)
        n_changed_out._obj.value = 3
        return min(k, self.rows)


def fake_index(rows):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex.__new__(KnnIndex)
    ix.lib, ix.ptr = FakeLib(rows), 1
    return ix


def test_update_pads_narrow_graphs_and_returns_k_prime_columns():
    ix = fake_index(7)
    gi = np.full((5, 3), PAD, np.uint32)
    gi[:, :2] = 1
    gs = np.ones((5, 3), np.float32)
    ui, us, n = ix.update_knn_graph(gi, gs, 5, changed=[2, 2], k=6)
    k, n_old, ch, idx, sc = ix.lib.calls[-1]
    assert (k, n_old, ch.tolist()) == (6, 5, [2, 2])
    assert (idx[:5, :3] == gi).all() and (idx[:5, 3:] == PAD).all() and (idx[5:] == PAD).all()
    assert (sc[:5, :3] == 1).all() and (sc[:5, 3:] == 0).all() and (sc[5:] == 0).all()
    assert ui.shape == (7, 6) and us.shape == (7, 6) and n == 3
    assert ui[:, 0].tolist() == list(range(7))


def test_update_argument_errors():
    from nornicdb_b200.knn import KnnError
    ix = fake_index(7)
    gi = np.zeros((5, 3), np.uint32)
    gs = np.zeros((5, 3), np.float32)
    with pytest.raises(KnnError):
        ix.update_knn_graph(gi, gs[:, :2], 5)  # shapes differ
    with pytest.raises(KnnError):
        ix.update_knn_graph(gi, gs, 4)  # n_old is not the graph's row count
    with pytest.raises(KnnError):
        ix.update_knn_graph(gi, gs, 5, k=2)  # k narrower than the graph
    with pytest.raises(KnnError):
        ix.update_knn_graph(gi, gs, 5, changed=[-1])
    assert ix.lib.calls == []


@pytest.mark.parametrize("case", ["k_too_big", "changed_not_old", "entry_not_old", "n_old_past_end"])
def test_every_library_refusal_raises(case):
    from nornicdb_b200.knn import KnnError
    ix = fake_index(7)
    gi = np.zeros((5, 3), np.uint32)
    gs = np.zeros((5, 3), np.float32)
    kw = {}
    if case == "k_too_big":
        kw["k"] = 192
    elif case == "changed_not_old":
        kw["changed"] = [5]
    elif case == "entry_not_old":
        gi[1, 1] = 6
    if case == "n_old_past_end":
        ix.lib.rows = 4
        gi, gs = gi[:5], gs[:5]
    with pytest.raises(KnnError):
        ix.update_knn_graph(gi, gs, 5, **kw)
