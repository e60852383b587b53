"""Value keys and windows on the host (knn.value_keys / window / window_admits): the encodings keep number order, refuse the
values that have no key, and window() turns every combination of Qdrant Range bounds into the closed key window that admits
exactly the numbers the bounds admit."""
import datetime
import itertools

import numpy as np
import pytest

from nornicdb_b200.knn import (ALL_BITS, EMPTY_WINDOW, KnnError, admits, as_windows, value_keys, window,
                               window_admits)

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def test_int64_keys_keep_order_over_random_and_edge_values():
    rng = np.random.default_rng(1)
    v = np.concatenate([rng.integers(I64_MIN + 1, I64_MAX, 5000, dtype=np.int64, endpoint=True),
                        np.array([I64_MIN + 1, -1, 0, 1, I64_MAX, I64_MAX - 1], dtype=np.int64)])
    k = value_keys(v)
    assert k.dtype == np.uint64 and (k != 0).all()
    order = np.argsort(v, kind="stable")
    assert (k[order][1:] >= k[order][:-1]).all()
    assert ((v[:, None] < v[None, :]) == (k[:, None] < k[None, :])).all()
    assert int(value_keys(np.int64(I64_MAX))) == ALL_BITS and int(value_keys(np.int64(I64_MIN + 1))) == 1


def test_float_keys_keep_order_over_random_and_edge_values():
    rng = np.random.default_rng(2)
    tiny = np.finfo(np.float64).tiny
    edge = np.array([-np.inf, -np.finfo(np.float64).max, -1.0, -tiny, -tiny / 2 ** 20, -5e-324, -0.0, 0.0, 5e-324, tiny / 2 ** 20,
                     tiny, 1.0, np.finfo(np.float64).max, np.inf])
    v = np.concatenate([rng.standard_normal(3000) * 10.0 ** rng.integers(-300, 300, 3000), edge])
    k = value_keys(v)
    assert (k != 0).all()
    # strict order where the numbers differ, equal keys where they are equal (-0.0 == +0.0)
    lt_v = v[:, None] < v[None, :]
    eq_v = v[:, None] == v[None, :]
    lt_k = k[:, None] < k[None, :]
    eq_k = k[:, None] == k[None, :]
    assert (lt_v == lt_k).all() and (eq_v == eq_k).all()
    assert value_keys(np.array([-0.0]))[0] == value_keys(np.array([0.0]))[0]


def test_float32_is_widened_exactly():
    rng = np.random.default_rng(3)
    f = np.concatenate([rng.standard_normal(2000).astype(np.float32),
                        np.array([np.float32(1e-45), -np.float32(1e-45), np.float32(3.4e38), -np.inf, np.inf], dtype=np.float32)])
    assert (value_keys(f) == value_keys(f.astype(np.float64))).all()


def test_datetime_keys_are_nanosecond_integers():
    t = np.array(["1969-12-31T23:59:59.999999999", "1970-01-01", "2024-02-29T12:00:00.000000001", "2262-04-11"],
                 dtype="datetime64[ns]")
    assert (value_keys(t) == value_keys(t.astype(np.int64))).all()
    kt = value_keys(t)
    assert (kt[1:] > kt[:-1]).all()
    d = np.array(["2024-01-01", "2024-01-02"], dtype="datetime64[D]")  # coarser units convert to ns first
    assert (value_keys(d) == value_keys(d.astype("datetime64[ns]").astype(np.int64))).all()


@pytest.mark.parametrize("bad", [np.array([1.0, np.nan]), np.array([np.nan], dtype=np.float32), np.array([I64_MIN], dtype=np.int64),
                                 np.array(["NaT"], dtype="datetime64[ns]"), np.array([1 << 63], dtype=np.uint64)])
def test_values_without_a_key_are_refused(bad):
    with pytest.raises(KnnError):
        value_keys(bad)


def _predicate(v, gt, gte, lt, lte):
    ok = np.ones(len(v), dtype=bool)
    if gt is not None:
        ok &= v > gt
    if gte is not None:
        ok &= v >= gte
    if lt is not None:
        ok &= v < lt
    if lte is not None:
        ok &= v <= lte
    return ok


@pytest.mark.parametrize("kind", ["int", "float"])
def test_window_matches_every_bound_combination(kind):
    rng = np.random.default_rng(4)
    if kind == "int":
        v = np.concatenate([rng.integers(-50, 50, 400), [I64_MIN + 1, I64_MAX, I64_MAX - 1, I64_MIN + 2]]).astype(np.int64)
        probes = [I64_MIN + 1, I64_MIN + 2, -7, 0, 3, 49, I64_MAX - 1, I64_MAX]
    else:
        v = np.concatenate([np.round(rng.standard_normal(400) * 4, 1), [-np.inf, np.inf, -0.0, 0.0, 5e-324, -5e-324]])
        probes = [-np.inf, -1.5, -0.0, 0.0, 5e-324, 2.3, np.inf]
    keys = value_keys(v)
    for gt, gte, lt, lte in itertools.product([None] + probes[::2], [None] + probes[1::2], [None] + probes[::3], [None] + probes[1::3]):
        lo, hi = window(gt=gt, gte=gte, lt=lt, lte=lte, kind=kind)
        got = window_admits(keys, lo, hi)
        assert (got == _predicate(v, gt, gte, lt, lte)).all(), (gt, gte, lt, lte, lo, hi)
        assert lo >= 1  # rows without a value (key 0) never match


def test_window_empty_at_both_ends_and_kind_inference():
    assert window(gt=np.int64(I64_MAX)) == EMPTY_WINDOW
    assert window(lt=np.int64(I64_MIN + 1)) == EMPTY_WINDOW
    assert window(gt=5, lt=6) == EMPTY_WINDOW
    assert window(gte=6, lte=5) == EMPTY_WINDOW
    assert window(gte=5, lte=5) == (int(value_keys(np.int64(5))), int(value_keys(np.int64(5))))
    assert window() == (1, ALL_BITS)
    lo, hi = EMPTY_WINDOW
    assert lo > hi and not window_admits(value_keys(np.arange(-5, 5)), lo, hi).any()
    # a Python float bound encodes as a float; kind="float" makes integer bounds filter a float column
    assert window(gte=2.0) == window(gte=2, kind="float") != window(gte=2)
    when = datetime.datetime(2024, 5, 1, 12, 30)
    assert window(gte=when) == window(gte=np.datetime64(when, "ns")) == (int(value_keys(np.datetime64(when, "ns"))), ALL_BITS)
    with pytest.raises(KnnError):
        window(gte=1, kind="decimal")


def test_as_windows_layout():
    w = as_windows([(1, 2), (3, 4)], 2)
    assert w.dtype == np.uint64 and w.flags.c_contiguous and w.shape == (2, 2)
    assert (as_windows((5, 9), 3) == np.array([[5, 9]] * 3, dtype=np.uint64)).all()  # one window for every query
    with pytest.raises(KnnError):
        as_windows([(1, 2), (3, 4)], 3)


def test_combined_predicate_restated_per_row():
    """The admissibility of a windowed search, restated row by row in plain Python: row mask AND tag filter AND lo <= key <= hi
    (unsigned), the numpy helpers the GPU tests check against agree with it."""
    rng = np.random.default_rng(5)
    n = 500
    tags = rng.integers(0, 1 << 6, n).astype(np.uint64)
    keys = value_keys(rng.integers(-20, 20, n))
    keys[::9] = 0  # rows without a value
    mask = rng.random(n) < 0.8
    cases = [((0, 0, 0), (0, ALL_BITS)), ((1, 0, 0), (1, ALL_BITS)), ((0, 2, 0), window(gte=-3, lt=7)),
             ((0, 0, 12), window(gt=0, kind="int")), ((3, 4, 0), EMPTY_WINDOW), ((0, 0, 0), (0, int(value_keys(np.int64(0)))))]
    for (a, no, an), (lo, hi) in cases:
        want = [bool(mask[r]) and (int(tags[r]) & a) == a and (int(tags[r]) & no) == 0 and (an == 0 or (int(tags[r]) & an) != 0)
                and lo <= int(keys[r]) <= hi for r in range(n)]
        got = mask & admits(tags, a, no, an) & window_admits(keys, lo, hi)
        assert got.tolist() == want, ((a, no, an), (lo, hi))


def test_fractional_and_infinite_bounds_on_an_int_column():
    """Qdrant Range bounds are doubles: on an int column a fractional bound rounds inward (gte=2.5 admits 3, lt=2.5 admits
    2), infinite and out-of-range bounds open or empty the window, and a NaN bound is refused."""
    v = np.concatenate([np.arange(-6, 7), [I64_MIN + 1, I64_MAX]]).astype(np.int64)
    keys = value_keys(v)
    probes = [-np.inf, -1e30, -2.5, -2.0, -0.5, 0.0, 0.5, 2.0, 2.5, 1e30, np.inf]
    for op in ("gt", "gte", "lt", "lte"):
        for x in probes:
            lo, hi = window(**{op: x}, kind="int")
            # (the float64 images of the int64 extremes stay on the right side of every probe)
            want = _predicate(v.astype(np.float64), *[x if o == op else None for o in ("gt", "gte", "lt", "lte")])
            assert (window_admits(keys, lo, hi) == want).all(), (op, x, lo, hi)
    assert window(gte=2.5, kind="int") == window(gte=3, kind="int")
    assert window(lt=2.5, kind="int") == window(lte=2, kind="int")
    assert window(gt=np.inf, kind="int") == EMPTY_WINDOW and window(lt=-np.inf, kind="int") == EMPTY_WINDOW
    with pytest.raises(KnnError):
        window(gte=float("nan"), kind="int")
