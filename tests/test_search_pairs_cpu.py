"""CPU checks of the similarity self-join (nk_search_pairs) without a GPU.

A numpy stand-in of the C call follows the header's contract literally: range search of the stripe's rows, each list cut to
the rows above its own query row and emptied for inadmissible left rows, CSR over the stripe and the snprintf-like size
protocol.  KnnIndex.search_pairs runs over it; the pairs it returns are checked against a brute force over every unordered
pair (each pair once, under its lower row), with the row mask and a tag filter, on stripes, and at the argument errors."""
import ctypes as C

import numpy as np
import pytest

from nornicdb_b200.knn import KnnError, KnnIndex, admits


def cosine64(rows):
    x = np.asarray(rows, np.float64)
    n = np.linalg.norm(x, axis=1)
    den = n[:, None] * n[None, :]
    return np.where(den > 0, (x @ x.T) / np.where(den > 0, den, 1.0), 0.0)


class FakePairsLib:
    """numpy stand-in of nk_search_pairs over an fp64-scored cosine corpus, with an optional row mask and tag words."""

    def __init__(self, rows, mask=None, tags=None):
        self.rows = np.asarray(rows, np.float32)
        self.n = len(self.rows)
        self.mask = np.ones(self.n, bool) if mask is None else np.asarray(mask, bool)
        self.tags = np.zeros(self.n, np.uint64) if tags is None else np.asarray(tags, np.uint64)
        self.s = cosine64(self.rows)
        self.calls = []
        self.err = b""

    def nk_search_pairs(self, ptr, first, n_rows, t, f_p, capacity, off_p, idx_p, sc_p, total_ref):
        self.calls.append(int(capacity))
        if t != t:
            self.err = b"nk_search_pairs: threshold is NaN"
            return -1
        if first > self.n or n_rows > self.n - first:
            self.err = b"nk_search_pairs: rows past the end of the index"
            return -1
        f = None if f_p is None else [int(v) for v in np.ctypeslib.as_array(C.cast(f_p, C.POINTER(C.c_uint64)), (3,))]
        adm = self.mask & (admits(self.tags, *f) if f is not None else True)
        off = np.ctypeslib.as_array(C.cast(off_p, C.POINTER(C.c_uint64)), (n_rows + 1,))
        lists = []
        for i in range(first, first + n_rows):
            # range search of row i (admissible rows meeting t, score desc / row asc), cut to rows above i
            r = np.flatnonzero(adm & (self.s[i] >= t))
            r = r[np.lexsort((r, -self.s[i, r]))]
            lists.append(r[r > i] if adm[i] else r[:0])
        off[0] = 0
        for k, r in enumerate(lists):
            off[k + 1] = off[k] + len(r)
        total = int(off[n_rows])
        C.cast(total_ref, C.POINTER(C.c_uint64))[0] = total
        if total > capacity:
            return 0
        idx = np.ctypeslib.as_array(C.cast(idx_p, C.POINTER(C.c_uint32)), (max(total, 1),))
        sc = np.ctypeslib.as_array(C.cast(sc_p, C.POINTER(C.c_float)), (max(total, 1),))
        for k, (i, r) in enumerate(zip(range(first, first + n_rows), lists)):
            idx[off[k]:off[k + 1]] = r
            sc[off[k]:off[k + 1]] = self.s[i, r]
        return 0

    def nk_index_rows(self, ptr):
        return self.n

    def nk_last_error(self):
        return self.err


@pytest.fixture()
def fake(monkeypatch):
    from nornicdb_b200 import _lib

    def make(rows, mask=None, tags=None):
        lib = FakePairsLib(rows, mask, tags)
        monkeypatch.setattr(_lib, "load", lambda: lib)
        ix = KnnIndex.__new__(KnnIndex)
        ix.lib, ix.dim, ix.ptr, ix.metric = lib, rows.shape[1], None, "cosine"
        return ix, lib

    return make


def brute_pairs(rows, t, adm=None):
    """Every unordered pair {i, j} of admissible rows with cosine >= t, as (lower, higher)."""
    s = cosine64(rows)
    n = len(rows)
    adm = np.ones(n, bool) if adm is None else adm
    i, j = np.triu_indices(n, 1)
    ok = adm[i] & adm[j] & (s[i, j] >= t)
    return set(zip(i[ok].tolist(), j[ok].tolist()))


def as_pairs(off, idx, first=0):
    out = []
    for r in range(len(off) - 1):
        out += [(first + r, int(j)) for j in idx[int(off[r]):int(off[r + 1])]]
    return out


def corpus(seed, n=120, d=8):
    rng = np.random.default_rng(seed)
    rows = rng.standard_normal((n, d)).astype(np.float32)
    if n > 90:
        rows[40] = rows[7]      # exact duplicates: cosine 1 between them
        rows[90] = rows[7]
    return rows


def test_csr_layout_each_pair_once_under_its_lower_row(fake):
    rows = corpus(1)
    ix, lib = fake(rows)
    off, idx, sc = ix.search_pairs(0.3)
    assert off.dtype == np.uint64 and idx.dtype == np.uint32 and sc.dtype == np.float32
    assert len(off) == len(rows) + 1 and off[0] == 0 and off[-1] == len(idx) == len(sc)
    assert np.all(np.diff(off.astype(np.int64)) >= 0)
    pairs = as_pairs(off, idx)
    assert len(pairs) == len(set(pairs)) and set(pairs) == brute_pairs(rows, 0.3)
    assert all(i < j for i, j in pairs), "a pair under its higher row"
    assert {(7, 40), (7, 90), (40, 90)} <= set(pairs)
    for r in range(len(rows)):  # each list in search()'s order: score desc, ties by row asc
        a, b = int(off[r]), int(off[r + 1])
        s_, j = sc[a:b], idx[a:b].astype(np.int64)
        assert np.all((s_[:-1] > s_[1:]) | ((s_[:-1] == s_[1:]) & (j[:-1] < j[1:])))
    assert off[-2] == off[-1], "the last row has no higher row"


def test_size_protocol_capacity_zero_exact_and_one_short(fake):
    rows = corpus(2)
    ix, lib = fake(rows)
    _, idx, _ = ix.search_pairs(0.2)
    total = len(idx)
    assert lib.calls == [0, total], "first call sizes, second call writes"
    lib.calls.clear()
    ix.search_pairs(0.2)                     # the grown capacity is kept: one call
    assert lib.calls == [total]
    ix._pairs_cap = total - 1                # one short: nothing written, then the exact size
    lib.calls.clear()
    off, idx2, _ = ix.search_pairs(0.2)
    assert lib.calls == [total - 1, total] and np.array_equal(idx2, idx)
    # at the C level: one short writes only the offsets and the total
    off = np.zeros(len(rows) + 1, np.uint64)
    sent_i = np.full(total, 0xDEADBEEF, np.uint32)
    sent_s = np.full(total, 7.0, np.float32)
    tot = C.c_uint64(0)
    args = lambda cap: (None, 0, len(rows), 0.2, None, cap, off.ctypes.data_as(C.c_void_p), sent_i.ctypes.data_as(C.c_void_p),
                        sent_s.ctypes.data_as(C.c_void_p), C.byref(tot))
    assert lib.nk_search_pairs(*args(total - 1)) == 0 and tot.value == total and off[-1] == total
    assert (sent_i == 0xDEADBEEF).all() and (sent_s == 7.0).all()
    assert lib.nk_search_pairs(*args(total)) == 0 and np.array_equal(sent_i, idx)


def test_mask_and_filter_apply_to_both_sides_and_empty_inadmissible_left_rows(fake):
    rows = corpus(3)
    n = len(rows)
    mask = np.ones(n, bool)
    mask[[7, 55]] = False                    # row 7 has duplicates above it: its list must be empty anyway
    tags = (np.arange(n) % 3).astype(np.uint64)
    ix, lib = fake(rows, mask, tags)
    flt = (0, 2, 0)                          # none_of bit 1: rows with tag 2 are inadmissible
    off, idx, _ = ix.search_pairs(0.1, filter=flt)
    adm = mask & admits(tags, *flt)
    pairs = as_pairs(off, idx)
    assert set(pairs) == brute_pairs(rows, 0.1, adm)
    for r in np.flatnonzero(~adm):
        assert off[r] == off[r + 1], f"inadmissible left row {r} has a list"
    assert not np.isin(idx.astype(np.int64), np.flatnonzero(~adm)).any()


def test_stripes_union_to_the_whole_index_and_empty_stripes(fake):
    rows = corpus(4)
    n = len(rows)
    ix, lib = fake(rows)
    off, idx, _ = ix.search_pairs(0.25)
    whole = as_pairs(off, idx)
    got = []
    for first, cnt in ((0, 33), (33, 1), (34, 50), (84, n - 84)):
        o, i, _ = ix.search_pairs(0.25, first, cnt)
        assert len(o) == cnt + 1
        got += as_pairs(o, i, first)
    assert got == whole
    o, i, s = ix.search_pairs(0.25, 17, 0)   # an empty stripe, also at the end
    assert o.tolist() == [0] and len(i) == 0 and len(s) == 0
    o, i, _ = ix.search_pairs(0.25, n)
    assert o.tolist() == [0] and len(i) == 0
    o, i, _ = ix.search_pairs(2.0)           # no pair reaches it
    assert int(o[-1]) == 0 and len(i) == 0


def test_argument_errors(fake):
    rows = corpus(5, n=20)
    ix, lib = fake(rows)
    n_calls = len(lib.calls)
    with pytest.raises(KnnError):
        ix.search_pairs(0.5, first_row=-1)   # rejected before the C call
    with pytest.raises(KnnError):
        ix.search_pairs(0.5, 3, -2)
    assert len(lib.calls) == n_calls
    with pytest.raises(KnnError, match="past the end"):
        ix.search_pairs(0.5, 15, 6)
    with pytest.raises(KnnError, match="past the end"):
        ix.search_pairs(0.5, 21)
    with pytest.raises(KnnError, match="NaN"):
        ix.search_pairs(float("nan"))
    with pytest.raises(KnnError):
        ix.search_pairs(0.5, filter=[(1, 0, 0), (2, 0, 0)])  # one filter for the whole join
