"""CPU checks of range search (nk_search_range) without a GPU: the threshold conversion per metric restated in numpy, the
CSR layout and snprintf-like size protocol on a numpy stand-in of the C call, and KnnIndex.search_range's resize-and-retry."""
import ctypes as C

import numpy as np
import pytest

from nornicdb_b200.knn import KnnIndex, admits


def key_threshold(t, metric, floor=None):
    """The library's key-space threshold (score; euclidean -distance^2) of an API threshold, the index floor folded in."""
    t = np.float32(t)
    if metric == "euclidean":
        if t < 0:
            key = np.float32(np.inf)
        elif np.isinf(t):
            key = np.float32(-np.inf)
        else:
            with np.errstate(over="ignore"):
                d = np.float32(t * t)
                while np.isfinite(d) and np.sqrt(np.nextafter(d, np.float32(np.inf))) <= t:
                    d = np.nextafter(d, np.float32(np.inf))
            while d > 0 and np.sqrt(d) > t:
                d = np.nextafter(d, np.float32(0))
            key = -d
        fl = np.float32(-np.inf) if floor is None or not (0 <= floor < np.inf) else -np.float32(floor) * np.float32(floor)
    else:
        key = t
        fl = np.float32(-np.inf) if floor is None else np.float32(floor)
    return np.float32(max(key, fl))


def qualifies(key_scores, thr_key):
    """Exact fp32 key scores -> returned?  NaN and -inf never are."""
    k = np.asarray(key_scores, dtype=np.float32)
    return (k > -np.inf) & (k >= thr_key)


def test_cosine_dot_threshold_is_a_minimum_score_and_the_floor_wins_when_stricter():
    for metric in ("cosine", "dot"):
        assert key_threshold(0.8, metric) == np.float32(0.8)
        assert key_threshold(0.8, metric, floor=0.9) == np.float32(0.9)
        assert key_threshold(0.8, metric, floor=0.5) == np.float32(0.8)
        assert key_threshold(-np.inf, metric) == -np.inf
        s = np.array([0.81, 0.8, 0.79, np.nan, -np.inf], np.float32)
        assert qualifies(s, key_threshold(0.8, metric)).tolist() == [True, True, False, False, False]


@pytest.mark.parametrize("t", [0.0, 1e-20, 0.3, 1.0, 2.5, 17.25, 1234.5, 3e19])
def test_euclidean_threshold_admits_exactly_the_distances_reported_at_or_below_it(t):
    """A row qualifies iff sqrtf(d) <= t, d the fp32 squared distance: the largest such d is the key threshold's magnitude."""
    t = np.float32(t)
    key = key_threshold(t, "euclidean")
    dmax = -key
    assert np.sqrt(dmax) <= t
    with np.errstate(over="ignore"):
        nxt = np.nextafter(dmax, np.float32(np.inf))
    assert not np.sqrt(nxt) <= t
    # a threshold taken from a reported distance admits the row it came from
    for d in np.float32([0.0, 0.09, 6.25, 1.5e6]) * np.float32(1.0001):
        assert -d >= key_threshold(np.sqrt(d), "euclidean")


def test_euclidean_threshold_edges_and_floor():
    assert key_threshold(-1.0, "euclidean") == np.inf  # no distance is negative
    assert key_threshold(np.inf, "euclidean") == -np.inf  # every finite distance
    assert key_threshold(5.0, "euclidean", floor=2.0) == np.float32(-4.0)  # the floor (a maximum distance) is stricter
    assert key_threshold(1.0, "euclidean", floor=3.0) == key_threshold(1.0, "euclidean")
    assert not qualifies(np.float32([-np.inf]), key_threshold(np.inf, "euclidean"))[0]  # infinite distance: never


class FakeRangeLib:
    """numpy stand-in of nk_search_range over a tiny fp64-scored corpus (cosine): CSR + the size protocol."""

    def __init__(self, rows, tags=None):
        self.rows = np.asarray(rows, np.float32)
        self.tags = tags
        self.calls = []

    def nk_search_range(self, ptr, q_p, t_p, f_p, Q, capacity, off_p, idx_p, sc_p, total_ref):
        d = self.rows.shape[1]
        q = np.ctypeslib.as_array(C.cast(q_p, C.POINTER(C.c_float)), (Q, d))
        t = np.ctypeslib.as_array(C.cast(t_p, C.POINTER(C.c_float)), (Q,))
        f = None if f_p is None else np.ctypeslib.as_array(C.cast(f_p, C.POINTER(C.c_uint64)), (Q, 3))
        off = np.ctypeslib.as_array(C.cast(off_p, C.POINTER(C.c_uint64)), (Q + 1,))
        self.calls.append(int(capacity))
        x = self.rows.astype(np.float64)
        s = (q.astype(np.float64) @ x.T) / np.linalg.norm(q, axis=1)[:, None] / np.linalg.norm(x, axis=1)[None, :]
        lists = []
        for qi in range(Q):
            ok = s[qi] >= t[qi]
            if f is not None:
                ok &= admits(self.tags, *[int(v) for v in f[qi]])
            r = np.flatnonzero(ok)
            o = np.lexsort((r, -s[qi, r]))
            lists.append((r[o], s[qi, r[o]]))
        off[0] = 0
        for qi in range(Q):
            off[qi + 1] = off[qi] + len(lists[qi][0])
        total = int(off[Q])
        C.cast(total_ref, C.POINTER(C.c_uint64))[0] = total
        if total > capacity:
            return 0  # nothing but the offsets and the total
        idx = np.ctypeslib.as_array(C.cast(idx_p, C.POINTER(C.c_uint32)), (max(total, 1),))
        sc = np.ctypeslib.as_array(C.cast(sc_p, C.POINTER(C.c_float)), (max(total, 1),))
        for qi, (r, v) in enumerate(lists):
            idx[off[qi]:off[qi + 1]] = r
            sc[off[qi]:off[qi + 1]] = v
        return 0


def fake_index(lib, dim):
    ix = KnnIndex.__new__(KnnIndex)
    ix.lib, ix.dim, ix.ptr, ix.metric = lib, dim, None, "cosine"
    return ix


def test_wrapper_resizes_from_the_reported_total_and_splits_the_csr():
    rng = np.random.default_rng(3)
    rows = rng.standard_normal((200, 8)).astype(np.float32)
    q = rng.standard_normal((4, 8)).astype(np.float32)
    lib = FakeRangeLib(rows)
    ix = fake_index(lib, 8)
    thr = np.array([0.5, -2.0, 0.2, 1.5], np.float32)
    res = ix.search_range(q, thr)
    assert lib.calls[0] == 0 and len(lib.calls) == 2 and lib.calls[1] == sum(len(i) for i, _ in res)
    assert len(res[1][0]) == 200 and len(res[3][0]) == 0
    for (idx, sc), t in zip(res, thr):
        assert idx.dtype == np.uint32 and sc.dtype == np.float32
        assert np.all(sc >= t - 1e-6) and np.all(np.diff(sc) <= 0)
    # the grown capacity is kept: an equal or smaller answer needs one call
    lib.calls.clear()
    ix.search_range(q, thr + 0.1)
    assert len(lib.calls) == 1
    # a larger answer grows again
    lib.calls.clear()
    ix.search_range(q, np.full(4, -2.0, np.float32))
    assert len(lib.calls) == 2 and lib.calls[1] == 800


def test_wrapper_passes_filters_and_broadcasts_a_scalar_threshold():
    rng = np.random.default_rng(4)
    rows = rng.standard_normal((100, 8)).astype(np.float32)
    tags = np.arange(100, dtype=np.uint64) % 4
    lib = FakeRangeLib(rows, tags)
    ix = fake_index(lib, 8)
    q = rng.standard_normal((3, 8)).astype(np.float32)
    res = ix.search_range(q, -2.0, filters=[(1, 0, 0), (0, 1, 0), (0, 0, 0)])
    assert [len(i) for i, _ in res] == [50, 50, 100]
    assert np.all(tags[res[0][0]] & 1) and not np.any(tags[res[1][0]] & 1)
    assert ix.search_range(np.empty((0, 8), np.float32), []) == []
