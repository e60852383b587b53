"""The self-join kept current, without a GPU: a numpy restatement of nk_pairs_remap (carry the pairs whose two ends kept their
id, drop the rest, add the pairs incident to the new and moved rows under their lower end, merge in key space) equals a fresh
join after appends, rewrites, swap-with-last removals and retags; the C++ mirror's SimilarPairs bookkeeping; and KnnIndex.search_pairs_rows / remap_pairs' argument
handling and size protocol over a stand-in of the C calls."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

NEW = 0xFFFFFFFF


# ---- the algorithm, restated with exact keys ---------------------------------------------------------------------------
# Integer-valued vectors and the dot product in fp64 make every score exact (and the same in both orientations), so equal
# scores are true ties, broken by row id as the library's keys break them.
def key(entry):
    return (entry[0], -entry[1])


def join(X, t, adm):
    """The whole-index self-join: row i lists every admissible j > i with X[i].X[j] >= t, best key first."""
    s = X @ X.T
    return [sorted([(float(s[i, j]), j) for j in range(i + 1, len(X)) if adm[i] and adm[j] and s[i, j] >= t], key=key, reverse=True)
            for i in range(len(X))]


def incident(X, rows, t, adm):
    """nk_search_pairs_rows: for each listed c, every pair {c, j} of the join, j == c and listed j < c dropped"""
    s = X @ X.T
    listed = set(rows)
    out = []
    for c in rows:
        lst = [(float(s[c, j]), j) for j in range(len(X))
               if j != c and not (j in listed and j < c) and adm[c] and adm[j] and s[c, j] >= t]
        out.append(sorted(lst, key=key, reverse=True))
    return out


def remap(old, src, X, t, adm):
    """nk_pairs_remap's steps -> (pairs, n_dropped, n_found)"""
    N, n_old = len(X), len(old)
    kept = lambda o: o < N and src[o] == o
    C_rows = [f for f in range(N) if src[f] != f]
    new = [[] for _ in range(N)]
    carried = 0
    for o in range(n_old):
        if not kept(o):
            continue
        new[o] = [(sc, j) for sc, j in old[o] if kept(j)]
        carried += len(new[o])
    found = 0
    for c, lst in zip(C_rows, incident(X, C_rows, t, adm)):
        for sc, j in lst:
            new[min(c, j)].append((sc, max(c, j)))
            found += 1
    n_dropped = sum(len(lst) for lst in old) - carried
    return [sorted(lst, key=key, reverse=True) for lst in new], n_dropped, found


class Store:
    """An index, its row map since the last join and the stored join, mutated the way the library's index is"""

    def __init__(self, X, t, tags=None, flt=None):
        self.X, self.t = X.copy(), t
        self.tags = np.zeros(len(X), np.int64) if tags is None else tags.copy()
        self.flt = flt
        self.pairs = join(self.X, t, self.adm())
        self.src = list(range(len(X)))

    def adm(self):
        return np.ones(len(self.X), bool) if self.flt is None else (self.tags & self.flt) == 0

    def append(self, rows):
        self.X = np.concatenate([self.X, rows])
        self.tags = np.concatenate([self.tags, np.zeros(len(rows), np.int64)])
        self.src += [NEW] * len(rows)

    def update(self, r, v):
        self.X[r] = v
        self.src[r] = NEW

    def retag(self, r, tag):
        self.tags[r] = tag
        self.src[r] = NEW

    def remove(self, r):
        self.X[r], self.tags[r], self.src[r] = self.X[-1], self.tags[-1], self.src[-1]
        self.X, self.tags, self.src = self.X[:-1].copy(), self.tags[:-1].copy(), self.src[:-1]

    def check(self):
        got, dropped, found = remap(self.pairs, self.src, self.X, self.t, self.adm())
        want = join(self.X, self.t, self.adm())
        assert got == want
        changed = [f for f in range(len(self.X)) if self.src[f] != f]
        assert found == sum(len(lst) for lst in incident(self.X, changed, self.t, self.adm()))
        assert sum(len(lst) for lst in self.pairs) - dropped == sum(len(lst) for lst in want) - found
        self.pairs, self.src = want, list(range(len(self.X)))
        return dropped, found


def corpus(rng, n, d):
    return rng.integers(-3, 4, size=(n, d)).astype(np.float64)


def test_incident_of_every_row_is_the_join():
    rng = np.random.default_rng(1)
    X = corpus(rng, 60, 6)
    adm = np.ones(60, bool)
    assert incident(X, list(range(60)), 6.0, adm) == join(X, 6.0, adm)


@pytest.mark.parametrize("seed", range(6))
def test_mutation_sequences(seed):
    rng = np.random.default_rng(100 + seed)
    X = corpus(rng, 80, 6)
    st = Store(X, 6.0, tags=rng.integers(0, 4, 80), flt=2 if seed % 2 else None)
    for _ in range(10):
        for _ in range(int(rng.integers(1, 6))):
            op = rng.integers(4)
            if op == 0:
                st.append(corpus(rng, int(rng.integers(1, 5)), 6))
            elif op == 1:
                st.update(int(rng.integers(len(st.X))), corpus(rng, 1, 6)[0])
            elif op == 2 and len(st.X) > 5:
                st.remove(int(rng.integers(len(st.X))))
            else:
                st.retag(int(rng.integers(len(st.X))), int(rng.integers(0, 4)))
        st.check()


def test_a_moved_row_changes_the_orientation_by_id():
    """Row 60 (the last) duplicates row 30.  Removing row 10 moves it to id 10, below row 30: the pair {30, 60} stored under 30
    must come back under 10, and pairs of the moved row with rows between 10 and 60 change their owner too."""
    rng = np.random.default_rng(7)
    X = corpus(rng, 61, 6)
    X[60] = X[30]
    st = Store(X, 6.0)
    assert (float(X[30] @ X[30]), 60) in st.pairs[30]
    st.remove(10)
    assert st.src[10] == 60
    dropped, found = st.check()
    assert (float(X[30] @ X[30]), 30) in st.pairs[10]
    assert all(j != 10 for lst in st.pairs[11:] for _, j in lst) and dropped > 0 and found > 0


def test_remove_down_to_a_few_rows_and_append_again():
    rng = np.random.default_rng(8)
    st = Store(corpus(rng, 40, 5), 4.0)
    while len(st.X) > 3:
        st.remove(int(rng.integers(len(st.X))))
    st.check()
    st.append(corpus(rng, 20, 5))
    st.check()


# ---- KnnIndex.search_pairs_rows / remap_pairs over a stand-in of the C calls --------------------------------------------
class FakeLib:
    """The C calls' size protocol on the host: records the arguments, and gives every row `per_row` pairs (other end: the
    row's id + 1, score 0.5), offsets and total always written.  It refuses nothing: the library's own refusals are tested
    against the library (tests/test_gpu_pairs_update.py); here only what the Python layer refuses before calling it."""

    def __init__(self, rows, per_row=2):
        self.rows, self.per_row, self.calls = rows, per_row, []

    def nk_index_rows(self, ptr):
        return self.rows

    def _write(self, n, cap, off, idx, sc, total):
        o = np.ctypeslib.as_array(C.cast(off, C.POINTER(C.c_uint64)), (n + 1,))
        o[:] = np.arange(n + 1) * self.per_row
        total._obj.value = n * self.per_row
        if n * self.per_row <= cap and n:
            np.ctypeslib.as_array(C.cast(idx, C.POINTER(C.c_uint32)), (n * self.per_row,))[:] = np.repeat(np.arange(1, n + 1), self.per_row)
            np.ctypeslib.as_array(C.cast(sc, C.POINTER(C.c_float)), (n * self.per_row,))[:] = 0.5
        return 0

    def nk_search_pairs_rows_windowed(self, ptr, rows, n, t, f, w, gap, cap, off, idx, sc, total):
        r = np.ctypeslib.as_array(C.cast(rows, C.POINTER(C.c_uint32)), (n,)).copy() if n else np.empty(0, np.uint32)
        self.calls.append(("rows", r, t, f is not None, w is not None, gap, cap))
        return self._write(n, cap, off, idx, sc, total)

    def nk_pairs_remap(self, ptr, t, f, w, gap, n_old, src, oo, oi, osc, cap, off, idx, sc, total, dropped, found):
        s = np.ctypeslib.as_array(C.cast(src, C.POINTER(C.c_uint32)), (self.rows,)).copy()
        self.calls.append(("remap", n_old, s, t, f is not None, w is not None, gap, cap))
        dropped._obj.value, found._obj.value = 3, 4
        return self._write(self.rows, cap, off, idx, sc, total)


def fake_index(rows):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex.__new__(KnnIndex)
    ix.lib, ix.ptr = FakeLib(rows), 1
    ix.__dict__.pop("_pairs_cap", None)
    return ix


def test_search_pairs_rows_sizes_itself_and_passes_the_arguments():
    from nornicdb_b200.knn import NO_GAP
    ix = fake_index(10)
    off, idx, sc = ix.search_pairs_rows([4, 2, 9], 0.5)
    calls = ix.lib.calls
    assert len(calls) == 2 and calls[0][6] == 0 and calls[1][6] == 6, "one call to size, one to fill"
    assert calls[0][1].tolist() == [4, 2, 9] and calls[0][5] == NO_GAP and not calls[0][3] and not calls[0][4]
    assert off.tolist() == [0, 2, 4, 6] and idx.tolist() == [1, 1, 2, 2, 3, 3] and np.all(sc == 0.5)
    ix.search_pairs_rows([1], 0.5, filter=(1, 0, 0), window=(5, 9), max_gap=3)
    assert calls[-1][3] and calls[-1][4] and calls[-1][5] == 3 and len(calls) == 3, "the grown buffer is kept"
    off, idx, sc = ix.search_pairs_rows([], 0.5)
    assert off.tolist() == [0] and idx.size == 0


def test_search_pairs_rows_refuses_before_calling_the_library():
    from nornicdb_b200.knn import KnnError
    ix = fake_index(10)
    for bad in ([-1], [2 ** 32]):
        with pytest.raises(KnnError, match="row ids"):
            ix.search_pairs_rows(bad, 0.5)
    with pytest.raises(KnnError):
        ix.search_pairs_rows([1], 0.5, max_gap=-1)
    with pytest.raises(KnnError):
        ix.search_pairs_rows([1], 0.5, filter=[(0, 0, 0), (1, 1, 1)])
    assert not ix.lib.calls, "refused before the library is called"


def test_remap_pairs_takes_a_row_map_and_checks_shapes():
    from nornicdb_b200.knn import GraphRowMap, KnnError
    ix = fake_index(4)
    m = GraphRowMap(5)
    m.remove_swap(1)
    m.append(1)
    m.remove_swap(0)
    assert len(m) == 4
    old = (np.array([0, 1, 1, 2, 2, 2], np.uint64), np.array([3, 4], np.uint32), np.array([0.9, 0.8], np.float32))
    off, idx, sc, dropped, found = ix.remap_pairs(old, 5, m, 0.5, window=(1, 2))
    assert ix.lib.calls[-1][0] == "remap" and ix.lib.calls[-1][2].tolist() == m.src_of_row.tolist() and ix.lib.calls[-1][5]
    assert off.tolist() == [0, 2, 4, 6, 8] and (dropped, found) == (3, 4)
    n_calls = len(ix.lib.calls)
    with pytest.raises(KnnError, match="CSR"):
        ix.remap_pairs((old[0][:-1], old[1], old[2]), 5, m, 0.5)
    with pytest.raises(KnnError, match="CSR"):
        ix.remap_pairs((old[0], old[1], old[2][:1]), 5, m, 0.5)
    with pytest.raises(KnnError, match="entries"):
        ix.remap_pairs(old, 5, m.src_of_row[:3], 0.5)
    with pytest.raises(KnnError, match="ROW_NEW"):
        ix.remap_pairs(old, 5, [0, 1, 2, -3], 0.5)
    assert len(ix.lib.calls) == n_calls, "refused before the library is called"


# ---- the C++ mirror's SimilarPairs bookkeeping, linked against a stand-in of the C calls ------------------------------------
def test_similar_pairs_bookkeeping_in_the_cpp_mirror(tmp_path):
    src = os.path.join(ROOT, "tests", "cpp", "pairs_bookkeeping_test.cpp")
    out = str(tmp_path / "pairs_bookkeeping_test")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-I", ROOT, src, "-o", out], check=True, cwd=ROOT)
    res = subprocess.run([out], capture_output=True, text=True, timeout=60)
    assert res.returncode == 0 and "pairs bookkeeping ok" in res.stdout, res.stdout + res.stderr
