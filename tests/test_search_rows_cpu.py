"""CPU checks of search by stored row (nk_search_rows) without a GPU.

The self rule restated in numpy: search every query row for k' = min(k+1, N) and drop the query's own row from its list,
or the last slot when the row is not in it.  It must equal an fp64 brute force over the admissible rows other than the
query's own, on the cases where the rule could go wrong: exact duplicates ranked ahead of self, dot product (self is not
its own best match), euclidean, a masked-out self, a score floor, k >= N, N = 1 and repeated ids.  Also: KnnIndex.search_rows
over a numpy stand-in of the C call, and EmbeddingIndex.SearchSimilar over an fp64 fake index."""
import ctypes as C

import numpy as np
import pytest

from fake_knn import FakeKnnIndex
from nornicdb_b200.knn import KnnError, KnnIndex

PAD = 0xFFFFFFFF


def keys64(rows, queries, metric):
    """fp64 key per (query, row), larger = better: cosine / dot score, euclidean -distance."""
    x, q = np.asarray(rows, np.float64), np.asarray(queries, np.float64)
    if metric == "euclidean":
        return -np.sqrt(np.maximum((q * q).sum(1)[:, None] + (x * x).sum(1)[None, :] - 2.0 * q @ x.T, 0.0))
    s = q @ x.T
    if metric == "cosine":
        den = np.linalg.norm(q, axis=1)[:, None] * np.linalg.norm(x, axis=1)[None, :]
        s = np.where(den > 0, s / np.where(den > 0, den, 1.0), 0.0)
    return s


def ranked(key, admissible, floor, metric):
    """Admissible rows meeting the floor, in (key desc, row asc) order."""
    ok = admissible.copy()
    if floor is not None:
        ok &= (-key <= floor) if metric == "euclidean" else (key >= floor)
    r = np.flatnonzero(ok)
    return r[np.lexsort((r, -key[r]))]


def api_score(key, metric):
    return -key if metric == "euclidean" else key


def search64(rows, queries, k, metric, mask=None, floor=None):
    """nk_search in fp64: [Q x min(k, N)], N = rows passing the mask; slots the floor leaves empty hold PAD / 0."""
    n = len(rows)
    adm = np.ones(n, bool) if mask is None else np.asarray(mask, bool)
    ke = min(k, int(adm.sum()))
    key = keys64(rows, queries, metric)
    idx = np.full((len(queries), ke), PAD, np.uint32)
    sc = np.zeros((len(queries), ke))
    for q in range(len(queries)):
        r = ranked(key[q], adm, floor, metric)[:ke]
        idx[q, :len(r)], sc[q, :len(r)] = r, api_score(key[q, r], metric)
    return idx, sc


def drop_self(idx, sc, ids, k):
    """The self rule on a k'-list per query: drop the query's own row, else the last slot; keep min(k, k')."""
    Q, kk = idx.shape
    ke = min(k, kk)
    out_i = np.full((Q, ke), PAD, np.uint32)
    out_s = np.zeros((Q, ke), sc.dtype)
    for q in range(Q):
        hit = np.flatnonzero(idx[q] == ids[q])
        keep = np.delete(np.arange(kk), hit[0] if hit.size else kk - 1)[:ke]
        out_i[q, :len(keep)], out_s[q, :len(keep)] = idx[q, keep], sc[q, keep]
    return out_i, out_s


def search_rows_by_rule(rows, ids, k, metric, mask=None, floor=None):
    n_adm = len(rows) if mask is None else int(np.sum(mask))
    idx, sc = search64(rows, rows[ids], min(k + 1, n_adm), metric, mask, floor)
    return drop_self(idx, sc, ids, k)


def others64(rows, ids, k, metric, mask=None, floor=None):
    """Brute force: the top k of the admissible rows other than the query's own, padded to min(k, N)."""
    n = len(rows)
    adm = np.ones(n, bool) if mask is None else np.asarray(mask, bool)
    ke = min(k, int(adm.sum()))
    key = keys64(rows, rows[ids], metric)
    idx = np.full((len(ids), ke), PAD, np.uint32)
    sc = np.zeros((len(ids), ke))
    for q, self_row in enumerate(ids):
        a = adm.copy()
        a[self_row] = False
        r = ranked(key[q], a, floor, metric)[:ke]
        idx[q, :len(r)], sc[q, :len(r)] = r, api_score(key[q, r], metric)
    return idx, sc


def assert_rule_matches(rows, ids, k, metric, mask=None, floor=None):
    ids = np.asarray(ids, np.int64)
    gi, gs = search_rows_by_rule(rows, ids, k, metric, mask, floor)
    oi, os_ = others64(rows, ids, k, metric, mask, floor)
    assert (gi == oi).all(), (gi, oi)
    assert (gs == os_).all()
    assert not (gi == ids[:, None]).any(), "a query returned its own row"
    return gi, gs


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_rule_equals_brute_force_without_self(metric):
    rng = np.random.default_rng(11)
    rows = rng.standard_normal((300, 16)).astype(np.float32)
    for k in (1, 5, 40):
        assert_rule_matches(rows, np.arange(300), k, metric)


def test_exact_duplicates_with_lower_ids_push_self_out_of_the_list():
    """k+1 copies of a row with lower ids tie with it (cosine 1) and win the tie: self is not in the k'-list, so the last
    slot goes and the k lowest copies remain."""
    rng = np.random.default_rng(12)
    k = 4
    rows = rng.standard_normal((50, 8)).astype(np.float32)
    rows[: k + 2] = rows[k + 1]          # rows 0 .. k+1 identical; the query is the highest of them
    ids = np.array([k + 1, 0, 3])
    idx, _ = search64(rows, rows[ids], k + 1, "cosine")
    assert k + 1 not in idx[0].tolist()  # self really is outside the k'-list
    gi, _ = assert_rule_matches(rows, ids, k, "cosine")
    assert gi[0].tolist() == list(range(k))
    assert gi[1].tolist() == [1, 2, 3, 4] and gi[2].tolist() == [0, 1, 2, 4]


def test_dot_product_self_is_not_the_best_match():
    rng = np.random.default_rng(13)
    rows = rng.standard_normal((40, 8)).astype(np.float32)
    rows[7] = rows[3] * 3.0  # row 7 beats row 3 on row 3's own query
    idx, _ = search64(rows, rows[[3]], 3, "dot")
    assert idx[0, 0] == 7 and idx[0, 0] != 3
    gi, _ = assert_rule_matches(rows, [3, 7], 2, "dot")
    assert gi[0, 0] == 7


def test_masked_out_self_and_score_floor():
    rng = np.random.default_rng(14)
    rows = rng.standard_normal((60, 8)).astype(np.float32)
    mask = np.ones(60, bool)
    mask[::3] = False
    ids = np.array([0, 3, 1, 2, 59])      # 0 and 3 are masked out, still queries
    assert_rule_matches(rows, ids, 6, "cosine", mask=mask)
    for metric, floor in (("cosine", 0.3), ("dot", 1.0), ("euclidean", 3.0)):
        gi, _ = assert_rule_matches(rows, np.arange(60), 10, metric, mask=mask, floor=floor)
        assert (gi == PAD).any()           # the floor leaves slots empty
    gi, _ = assert_rule_matches(rows, np.arange(60), 60, "cosine", floor=0.99)
    assert (gi == PAD).all()


def test_k_at_or_above_n_and_a_single_row():
    rng = np.random.default_rng(15)
    rows = rng.standard_normal((7, 4)).astype(np.float32)
    gi, _ = assert_rule_matches(rows, np.arange(7), 6, "euclidean")
    assert gi.shape == (7, 6) and (gi != PAD).all()
    for k in (7, 20):
        gi, _ = assert_rule_matches(rows, np.arange(7), k, "euclidean")
        assert gi.shape == (7, 7) and (gi[:, 6] == PAD).all() and (gi[:, :6] != PAD).all()
    one = rows[:1]
    gi, gs = assert_rule_matches(one, [0, 0], 3, "cosine")
    assert gi.tolist() == [[PAD], [PAD]] and gs.tolist() == [[0.0], [0.0]]


def test_repeated_ids_give_repeated_answers():
    rng = np.random.default_rng(16)
    rows = rng.standard_normal((80, 8)).astype(np.float32)
    gi, gs = assert_rule_matches(rows, [5, 9, 5, 5, 9], 8, "dot")
    assert (gi[0] == gi[2]).all() and (gi[0] == gi[3]).all() and (gi[1] == gi[4]).all()


class FakeRowsLib:
    """numpy stand-in of nk_search_rows: the self rule over fp64 scores, the C call's return value and padding."""

    def __init__(self, rows, metric):
        self.rows, self.metric, self.calls = np.asarray(rows, np.float32), metric, []

    def nk_search_rows(self, ptr, ids_p, Q, k, idx_p, sc_p):
        ids = np.ctypeslib.as_array(C.cast(ids_p, C.POINTER(C.c_uint32)), (Q,)).astype(np.int64)
        self.calls.append((Q, k))
        if (ids >= len(self.rows)).any():
            return -1
        gi, gs = search_rows_by_rule(self.rows, ids, k, self.metric)
        idx = np.ctypeslib.as_array(C.cast(idx_p, C.POINTER(C.c_uint32)), (Q, k))
        sc = np.ctypeslib.as_array(C.cast(sc_p, C.POINTER(C.c_float)), (Q, k))
        idx[:, :gi.shape[1]], sc[:, :gi.shape[1]] = gi, gs
        return gi.shape[1]

    def nk_last_error(self):
        return b"row out of range"


def test_knn_index_search_rows_wrapper(monkeypatch):
    from nornicdb_b200 import _lib
    rng = np.random.default_rng(17)
    rows = rng.standard_normal((30, 8)).astype(np.float32)
    lib = FakeRowsLib(rows, "cosine")
    monkeypatch.setattr(_lib, "load", lambda: lib)
    ix = KnnIndex.__new__(KnnIndex)
    ix.lib, ix.dim, ix.ptr, ix.metric = lib, 8, None, "cosine"
    idx, sc = ix.search_rows([4, 2, 4], 5)
    assert idx.shape == (3, 5) and idx.dtype == np.uint32 and sc.dtype == np.float32
    oi, _ = others64(rows, np.array([4, 2, 4]), 5, "cosine")
    assert (idx == oi).all()
    idx, _ = ix.search_rows(np.arange(30), 100)  # k >= N: min(k, N) columns, the last one padding
    assert idx.shape == (30, 30) and (idx[:, -1] == PAD).all()
    assert ix.search_rows([], 3)[0].shape == (0, 0) and ix.search_rows([1], 0)[0].shape == (1, 0)
    n_calls = len(lib.calls)
    with pytest.raises(KnnError):
        ix.search_rows([-1], 3)              # rejected before the C call
    with pytest.raises(KnnError):
        ix.search_rows([2 ** 32], 3)
    assert len(lib.calls) == n_calls
    with pytest.raises(KnnError, match="out of range"):
        ix.search_rows([30], 3)


class FakeRowsKnnIndex(FakeKnnIndex):
    """FakeKnnIndex with search_rows: fp64 search of the rows as stored, k+1, self rule."""

    def search_rows(self, rows, k):
        ids = np.asarray(rows, np.int64).reshape(-1)
        if len(ids) == 0 or k <= 0:
            return np.empty((len(ids), 0), np.uint32), np.empty((len(ids), 0), np.float32)
        idx, sc = self.search(self.read_rows(0, len(self))[ids], k + 1)
        return drop_self(idx, sc, ids, k)


@pytest.fixture()
def fake_device(monkeypatch, oracle_mod):
    import nornicdb_b200.embedding_index as ei
    monkeypatch.setattr(ei, "KnnIndex", FakeRowsKnnIndex)
    return oracle_mod


def test_search_similar_maps_ids_both_ways(fake_device):
    from nornicdb_b200.embedding_index import EmbeddingIndex
    ei = EmbeddingIndex(4)
    assert ei.SearchSimilar(["a"], 3) == [[]]                      # empty index
    ei.AddBatch(["a", "b", "c", "d"], [[1, 0, 0, 0], [0.9, 0.1, 0, 0], [0, 1, 0, 0], [1, 0, 0, 0]])
    res = ei.SearchSimilar(["a", "missing", "c", "a"], 2)
    assert [[r.ID for r in lst] for lst in res] == [["d", "b"], [], ["b", "a"], ["d", "b"]]
    assert abs(res[0][0].Score - 1.0) < 1e-6 and abs(res[0][0].Distance) < 1e-6
    assert ei.SearchSimilar(["missing"], 2) == [[]] and ei.SearchSimilar(["a"], 0) == [[]]
    assert [r.ID for r in ei.SearchSimilar(["b"], 10)[0]] == ["a", "d", "c"]  # k > others: every other node
    ei.Remove("a")                                                  # swap-remove: d moves into a's row
    assert [[r.ID for r in lst] for lst in ei.SearchSimilar(["d", "a"], 1)] == [["b"], []]
