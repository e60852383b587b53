"""Value windows for search by stored row and for the self-join (nk_search_rows_windowed, nk_search_pairs_windowed).

search_rows(windows=...) must equal nk_search_windowed over the stored rows with k' = min(k + 1, rows passing the mask) and the
self rule, bit for bit, per block of 1024 queries; search_pairs(window=, max_gap=) must equal the unwindowed join with the
out-of-window and out-of-band pairs dropped, bit for bit (offsets, rows and scores)."""
import numpy as np
import pytest

from test_gpu_filtered import check_filtered
from test_gpu_filtered_graph import BLOCK, K, PAD, assert_same, collections, filters_of, make_index, stored_f32, tags_of

pytestmark = pytest.mark.gpu

ALL = 0xFFFFFFFFFFFFFFFF


def by_search_windowed(ix, ids, filters, windows, k, n_adm):
    """the contract: nk_search_windowed(stored rows, filters, windows, k' = min(k + 1, n_adm)) per block of 1024, the query's
    own row dropped (or the last slot where it is not in the list), padded back to min(k, n_adm) columns"""
    x = stored_f32(ix)
    kk, ke = min(k + 1, n_adm), min(k, n_adm)
    oi, osc = [], []
    for b in range(0, len(ids), BLOCK):
        bid = ids[b:b + BLOCK]
        ri, rs = ix.search_windowed(x[bid], kk, windows[b:b + BLOCK], None if filters is None else filters[b:b + BLOCK])
        for q, self_row in enumerate(bid):
            li, ls = list(ri[q]), list(rs[q])
            drop = li.index(self_row) if self_row in li else len(li) - 1
            del li[drop], ls[drop]
            li, ls = li[:ke] + [PAD] * (ke - len(li[:ke])), ls[:ke] + [0.0] * (ke - len(ls[:ke]))
            oi.append(np.array(li, np.uint32))
            osc.append(np.array(ls, np.float32))
    return np.stack(oi), np.stack(osc)


def timestamps(rng, n):
    """int64 'seconds' in row order over a year, a few rows without a value (key 0)"""
    from nornicdb_b200.knn import value_keys
    t = np.sort(rng.integers(0, 365 * 86_400, n))
    keys = value_keys(t)
    keys[rng.choice(n, n // 50, replace=False)] = 0
    return keys


def mixed_row_windows(rng, keys, ids):
    """per query: mostly +-1 day around its own key (band_windows), some one-sided, some all-admitting, some empty"""
    from nornicdb_b200.knn import EMPTY_WINDOW, band_windows
    w = band_windows(keys[ids], 86_400)
    kind = rng.integers(0, 10, len(ids))
    w[kind == 1] = band_windows(keys[ids], 7 * 86_400, 0)[kind == 1]
    w[kind == 2] = (0, ALL)
    w[kind == 3] = EMPTY_WINDOW
    w[kind == 4] = (1, ALL)
    return np.ascontiguousarray(w)


def paths_for(dtype):
    return ("auto", "simt", "shadow") + (("filter",) if dtype == "f32" else ())


CASES = [(dtype, metric, path) for dtype in ("f32", "f16", "bf16") for metric in ("cosine", "dot", "euclidean")
         for path in paths_for(dtype)]


@pytest.mark.parametrize("dtype,metric,path", CASES)
def test_search_rows_windowed_equals_search_windowed(knn_lib, dtype, metric, path):
    from nornicdb_b200.knn import KnnError, admits, window_admits
    rng = np.random.default_rng(100 + CASES.index((dtype, metric, path)))
    n, d = 3000, 64
    rows = rng.standard_normal((n, d)).astype(np.float32)
    rows[100:104] = rows[50]  # duplicates
    keys = timestamps(rng, n)
    coll = collections(rng, n)
    tags = tags_of(coll, rng)
    ix = make_index(rows, metric, dtype, path)
    ix.set_row_tags(tags)
    ix.set_row_values(keys)
    ids = np.concatenate([rng.choice(n, 1200, replace=False), [50, 100, 101]])  # two blocks
    w = mixed_row_windows(rng, keys, ids)
    f = filters_of(coll[ids], rng)
    for k in (1, K, 192):
        for filt in (None, f):
            try:
                want = by_search_windowed(ix, ids, filt, w, k, n)
            except KnnError:
                with pytest.raises(KnnError):
                    ix.search_rows(ids, k, filters=filt, windows=w)
                continue
            got = ix.search_rows(ids, k, filters=filt, windows=w)
            assert_same(got, want, f"k={k} filters={filt is not None}")
            for q in range(0, len(ids), 89):  # every listed row is admitted by the query's window (and filter)
                li = got[0][q][got[0][q] != PAD].astype(np.int64)
                assert window_admits(keys[li], int(w[q][0]), int(w[q][1])).all() and (li != ids[q]).all()
                if filt is not None:
                    assert admits(tags[li], *[int(x) for x in f[q]]).all()
    # windows=None is search_rows_filtered / search_rows; all-admitting windows give the filtered result
    assert_same(ix.search_rows(ids, K, filters=f, windows=None), ix.search_rows(ids, K, filters=f))
    assert_same(ix.search_rows(ids, K, windows=(0, ALL)), ix.search_rows(ids, K))
    ix.release()


@pytest.mark.parametrize("path", ["simt", "shadow", "filter", "auto"])
def test_search_rows_best_rows_outside_the_window(knn_lib, path):
    """Each query row's 200 nearest other rows get keys outside its window: the list must be the exact top k of the rest."""
    from nornicdb_b200.knn import value_keys
    rng = np.random.default_rng(7)
    n, d, k = 6000, 64, 10
    rows = rng.standard_normal((n, d)).astype(np.float32)
    ids = np.arange(0, n, 5)[:1100]
    ix = make_index(rows, "cosine", "f32", path)
    x = stored_f32(ix)
    xn = x / np.linalg.norm(x, axis=1, keepdims=True)
    v = rng.integers(1000, 2000, n)
    for q in ids[:300]:
        s = xn @ xn[q]
        s[q] = -np.inf
        v[np.argsort(-s)[:200]] = 10  # below every window
    keys = value_keys(v)
    ix.set_row_values(keys)
    w = np.tile(np.array([int(value_keys(np.int64(1000))), int(value_keys(np.int64(1999)))], np.uint64), (len(ids), 1))
    gi, gs = ix.search_rows(ids, k, windows=w)
    assert_same((gi, gs), by_search_windowed(ix, ids, None, w, k, n))
    adm = (v >= 1000)[None, :].repeat(len(ids), 0)
    adm[np.arange(len(ids)), ids] = False
    check_filtered(x, x[ids], k, "cosine", gi, gs, adm)
    ix.release()


def test_search_rows_windowed_mask_floor_and_two_devices(knn_lib):
    from nornicdb_b200 import cuda
    rng = np.random.default_rng(9)
    n, d = 4000, 64
    rows = rng.standard_normal((n, d)).astype(np.float32)
    keys = timestamps(rng, n)
    ids = rng.choice(n, 1500, replace=False)
    w = mixed_row_windows(rng, keys, ids)
    keep = rng.random(n) > 0.3
    devs = [(0,)] + ([(0, 1)] if cuda.DeviceCount() >= 2 else [])
    for devices in devs:
        ix = make_index(rows, "dot", "f32", "auto", devices=devices)
        ix.set_row_values(keys)
        ix.set_row_mask(keep)
        ix.set_min_score(0.0)
        got = ix.search_rows(ids, K, windows=w)
        assert_same(got, by_search_windowed(ix, ids, None, w, K, int(keep.sum())), str(devices))
        li = got[0][got[0] != PAD].astype(np.int64)
        assert keep[li].all()
        ix.release()


def test_search_rows_windowed_refusals(knn_lib):
    from nornicdb_b200.knn import KnnError
    rng = np.random.default_rng(3)
    ix = make_index(rng.standard_normal((100, 16)).astype(np.float32), "cosine")
    with pytest.raises(KnnError):
        ix.search_rows([1, 2, 3], 5, windows=np.zeros((2, 2), np.uint64))
    with pytest.raises(KnnError):
        ix.search_rows([1, 200], 5, windows=(0, ALL))
    w = np.zeros((1, 2), np.uint64)
    assert ix.lib.nk_search_rows_windowed(ix.ptr, None, None, w.ctypes.data, 1, 5, None, None) == -1
    ix.release()


# ---- the self-join ------------------------------------------------------------------------------------------------------

def drop_pairs(res, first, keys, lo, hi, gap):
    """the contract: the unwindowed join's CSR with the pairs the window or the band refuses dropped"""
    from nornicdb_b200.knn import NO_GAP
    off, idx, sc = res
    left = first + np.repeat(np.arange(len(off) - 1), np.diff(off.astype(np.int64)))
    ki, kj = keys[left], keys[idx.astype(np.int64)]
    lo, hi = np.uint64(lo), np.uint64(hi)
    keep = (ki >= lo) & (ki <= hi) & (kj >= lo) & (kj <= hi)
    if gap != NO_GAP:
        diff = np.where(ki > kj, ki - kj, kj - ki)
        keep &= (ki != 0) & (kj != 0) & (diff <= np.uint64(gap))
    kept = np.concatenate([[0], np.cumsum(keep)]).astype(np.uint64)
    return kept[off.astype(np.int64)], idx[keep], sc[keep]


PAIR_CASES = [(dtype, metric, path) for dtype in ("f32", "f16", "bf16") for metric in ("cosine", "dot", "euclidean")
              for path in paths_for(dtype)]
THRESHOLD = {"cosine": 0.25, "dot": 14.0, "euclidean": 9.0}


@pytest.mark.parametrize("dtype,metric,path", PAIR_CASES)
def test_pairs_windowed_equal_the_join_with_pairs_dropped(knn_lib, dtype, metric, path):
    from nornicdb_b200.knn import NO_GAP
    rng = np.random.default_rng(200 + PAIR_CASES.index((dtype, metric, path)))
    n, d = 2600, 64
    rows = rng.standard_normal((n, d)).astype(np.float32)
    keys = timestamps(rng, n)
    ix = make_index(rows, metric, dtype)
    ix.set_path(path)
    ix.set_row_values(keys)
    t = THRESHOLD[metric]
    lo, hi = int(keys[keys != 0].min()) + 30 * 86_400, int(keys.max()) - 30 * 86_400
    for first, n_rows in ((0, n), (700, 1500)):  # the whole index (three blocks), and a stripe off the 256-row tiles
        base = ix.search_pairs(t, first, n_rows)
        assert base[1].size > 100
        for window, gap in (((lo, hi), NO_GAP), (None, 3 * 86_400), ((lo, hi), 86_400), (None, 0)):
            got = ix.search_pairs(t, first, n_rows, window=window, max_gap=None if gap == NO_GAP else gap)
            w = (0, ALL) if window is None else window
            assert_pairs(got, drop_pairs(base, first, keys, w[0], w[1], gap), f"{first} {window} {gap}")
    ix.release()


def assert_pairs(a, b, what=""):
    assert np.array_equal(a[0], b[0]), f"{what}: offsets"
    assert np.array_equal(a[1], b[1]), f"{what}: rows"
    assert np.array_equal(a[2].view(np.uint32), b[2].view(np.uint32)), f"{what}: scores"


def test_pairs_band_at_the_key_extremes_and_without_values(knn_lib):
    """Keys at 1 .. 4 and 2^64 - 4 .. 2^64 - 1 (saturation at both ends), rows without a value, a filter and a row mask."""
    from nornicdb_b200.knn import NO_GAP
    rng = np.random.default_rng(11)
    n, d = 1500, 32
    rows = (rng.standard_normal((1, d)) + 0.3 * rng.standard_normal((n, d))).astype(np.float32)  # every pair similar
    keys = np.zeros(n, np.uint64)
    keys[: n // 3] = rng.integers(1, 5, n // 3).astype(np.uint64)
    keys[n // 3: 2 * n // 3] = np.uint64(ALL) - rng.integers(0, 4, n // 3).astype(np.uint64)
    tags = rng.integers(0, 2, n).astype(np.uint64)
    keep = rng.random(n) > 0.1
    ix = make_index(rows, "cosine")
    ix.set_row_values(keys)
    ix.set_row_tags(tags)
    ix.set_row_mask(keep)
    filt = (1, 0, 0)
    base = ix.search_pairs(0.5, filter=filt)
    for window, gap in ((None, 2), (None, 0), ((1, 3), 1), ((ALL - 2, ALL), 5), ((0, ALL), NO_GAP - 1), ((0, 2), NO_GAP)):
        got = ix.search_pairs(0.5, filter=filt, window=window, max_gap=None if gap == NO_GAP else gap)
        w = (0, ALL) if window is None else window
        want = drop_pairs(base, 0, keys, w[0], w[1], gap)
        assert_pairs(got, want, f"{window} {gap}")
        off, idx, _ = got
        left = np.repeat(np.arange(n), np.diff(off.astype(np.int64)))
        if gap != NO_GAP:
            assert (keys[left] != 0).all() and (keys[idx.astype(np.int64)] != 0).all()
    # two blocks of the same stripe both near 1 and near 2^64 - 1 pair only within their own end under a small band
    off, idx, _ = ix.search_pairs(0.5, max_gap=10)
    left = np.repeat(np.arange(n), np.diff(off.astype(np.int64)))
    assert ((keys[left] < 10) == (keys[idx.astype(np.int64)] < 10)).all()
    ix.release()


def test_pairs_windowed_two_shards(knn_lib):
    from nornicdb_b200 import cuda
    if cuda.DeviceCount() < 2:
        pytest.skip("one device")
    rng = np.random.default_rng(12)
    n, d = 3000, 64
    rows = rng.standard_normal((n, d)).astype(np.float32)
    keys = timestamps(rng, n)
    ix = make_index(rows, "cosine", devices=(0, 1))
    ix.set_row_values(keys)
    base = ix.search_pairs(0.25, 1000, 1024)  # one block straddling the two shards
    got = ix.search_pairs(0.25, 1000, 1024, max_gap=5 * 86_400)
    assert_pairs(got, drop_pairs(base, 1000, keys, 0, ALL, 5 * 86_400))
    ix.release()


def test_pairs_windowed_refusals(knn_lib):
    import ctypes as C
    from nornicdb_b200.knn import NO_GAP, KnnError
    rng = np.random.default_rng(13)
    ix = make_index(rng.standard_normal((300, 16)).astype(np.float32), "cosine")
    with pytest.raises(KnnError):
        ix.search_pairs(float("nan"), max_gap=3)
    with pytest.raises(KnnError):
        ix.search_pairs(0.5, 200, 200, max_gap=3)
    with pytest.raises(KnnError):
        ix.search_pairs(0.5, max_gap=-1)
    ix.set_path("tensor")
    with pytest.raises(KnnError):
        ix.search_pairs(0.5, window=(0, ALL))
    ix.set_path("auto")
    off = np.full(301, 7, np.uint64)
    total = C.c_uint64(99)
    w = np.array([0, ALL], np.uint64)
    assert ix.lib.nk_search_pairs_windowed(ix.ptr, 0, 300, C.c_float(-1.0), None, w.ctypes.data, NO_GAP, 0, off.ctypes.data, None,
                                           None, C.byref(total)) == 0
    assert total.value == off[-1] and total.value > 0  # sizes only: nothing else written with capacity 0
    ix.release()
