"""CPU tests of value windows for search by stored row and for the self-join: band_windows at the ends of the key space, the
band width argument, and a host restatement of the left-row windows of nk_search_pairs_windowed checked against the pair
predicate it must implement (window on both sides, band |key[i] - key[j]| <= max_gap between rows that have a value)."""
import numpy as np
import pytest

from nornicdb_b200.knn import ALL_BITS, EMPTY_WINDOW, NO_GAP, KnnError, _gap_keys, as_windows, band_windows, value_keys


def test_band_windows_saturate_at_both_ends():
    keys = np.array([0, 1, 2, 5, 1000, ALL_BITS - 5, ALL_BITS - 1, ALL_BITS], dtype=np.uint64)
    w = band_windows(keys, 3)
    assert w.dtype == np.uint64 and w.shape == (8, 2) and w.flags.c_contiguous
    want = [EMPTY_WINDOW, (1, 4), (1, 5), (2, 8), (997, 1003), (ALL_BITS - 8, ALL_BITS - 2), (ALL_BITS - 4, ALL_BITS),
            (ALL_BITS - 3, ALL_BITS)]
    assert [tuple(int(x) for x in r) for r in w] == [tuple(x) for x in want]
    # asymmetric: the last 7 days before each row and nothing after it
    w = band_windows(keys, 7, 0)
    assert [int(x) for x in w[4]] == [993, 1000] and [int(x) for x in w[7]] == [ALL_BITS - 7, ALL_BITS]


def test_band_windows_gap_zero_and_rows_without_a_value():
    keys = np.array([0, 7, 7, 0, 9], dtype=np.uint64)
    w = band_windows(keys, 0)
    assert [tuple(int(x) for x in r) for r in w] == [EMPTY_WINDOW, (7, 7), (7, 7), EMPTY_WINDOW, (9, 9)]
    # the widest band still never admits key 0
    w = band_windows(keys, NO_GAP - 1)
    assert all(int(r[0]) >= 1 for r in w)
    assert [tuple(int(x) for x in r) for r in w[[1, 4]]] == [(1, ALL_BITS), (1, ALL_BITS)]


def test_band_windows_of_datetimes_take_timedeltas_in_ns():
    t = np.array(["2026-01-01T00:00", "2026-01-02T12:00"], dtype="datetime64[ns]")
    keys = value_keys(t)
    w = band_windows(keys, np.timedelta64(1, "D"))
    day = 86_400 * 10 ** 9
    assert [int(x) for x in w[0]] == [int(keys[0]) - day, int(keys[0]) + day]
    assert not (int(w[0][0]) <= int(keys[1]) <= int(w[0][1]))  # 36 h apart
    assert int(w[1][0]) <= int(keys[1]) <= int(w[1][1])


@pytest.mark.parametrize("bad", [-1, NO_GAP, NO_GAP + 1, 1.5, "3", True, np.bool_(False), np.timedelta64("NaT")])
def test_gap_is_refused_outside_its_range(bad):
    with pytest.raises(KnnError):
        _gap_keys(bad)


def test_gap_conversions():
    import datetime as dt
    assert _gap_keys(0) == 0 and _gap_keys(np.int64(5)) == 5 and _gap_keys(NO_GAP - 1) == NO_GAP - 1
    assert _gap_keys(np.timedelta64(2, "s")) == 2 * 10 ** 9
    assert _gap_keys(dt.timedelta(hours=1)) == 3600 * 10 ** 9


def test_window_shapes():
    assert as_windows((1, 2), 3).shape == (3, 2)
    with pytest.raises(KnnError):
        as_windows(np.zeros((2, 2), np.uint64), 3)


# ---- the self-join's admission ------------------------------------------------------------------------------------------

def left_windows(keys, lo, hi, gap):
    """What nk::row_windows gives each left row (admissible by mask and filter): [lo, hi], narrowed to band_windows(keys, gap)
    under a band; the window that admits no row where the row's own key is outside [lo, hi] or, under a band, 0."""
    k = np.asarray(keys, np.uint64)
    w = np.tile(np.array([lo, hi], np.uint64), (k.size, 1))
    if gap != NO_GAP:
        b = band_windows(k, gap)
        w[:, 0] = np.maximum(w[:, 0], b[:, 0])
        w[:, 1] = np.minimum(w[:, 1], b[:, 1])
    own = (k >= np.uint64(lo)) & (k <= np.uint64(hi)) & ((k != 0) if gap != NO_GAP else True)
    w[~own] = EMPTY_WINDOW
    return w


def pair_admitted(ki, kj, lo, hi, gap):
    """The contract, on Python ints: both keys in [lo, hi]; under a band both set and at most gap apart."""
    ok = lo <= ki <= hi and lo <= kj <= hi
    if gap != NO_GAP:
        ok = ok and ki != 0 and kj != 0 and abs(ki - kj) <= gap
    return ok


@pytest.mark.parametrize("lo,hi", [(0, ALL_BITS), (1, ALL_BITS), (3, ALL_BITS - 3), (ALL_BITS, 0), (50, 60)])
@pytest.mark.parametrize("gap", [NO_GAP, 0, 1, 4, 10, ALL_BITS - 1])
def test_left_row_windows_equal_the_pair_predicate(lo, hi, gap):
    keys = np.array([0, 0, 1, 2, 3, 5, 50, 55, 60, 61, 1 << 63, ALL_BITS - 4, ALL_BITS - 1, ALL_BITS, ALL_BITS],
                    dtype=np.uint64)
    w = left_windows(keys, lo, hi, gap)
    n = keys.size
    for i in range(n):
        for j in range(n):
            ki, kj = int(keys[i]), int(keys[j])
            scanned = int(w[i][0]) <= kj <= int(w[i][1])
            assert scanned == pair_admitted(ki, kj, lo, hi, gap), (i, j, ki, kj, w[i])
            # symmetric: the lower id's window decides, whichever row that is
            assert scanned == (int(w[j][0]) <= ki <= int(w[j][1])), (i, j)
