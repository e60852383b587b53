"""GPU tests of per-query value windows (nk_search_windowed, nk_search_range_windowed): one value key per row, a [lo, hi] key
window per query, evaluated inside every scan kernel next to the tag filters.  Each test mirrors its counterpart in
test_gpu_filtered.py: every result is checked against an fp64 brute force over each query's admissible rows, and the
thresholds the kernels prune with are attacked directly (a query's true best rows given values outside its window)."""
import numpy as np
import pytest

from parity import exact_scores_for
from test_gpu_filtered import _near_tie_corpus, admissible, check_filtered, fp64_scores, make_tags, mixed_filters, rows_of

pytestmark = pytest.mark.gpu

PAD = 0xFFFFFFFF
ALL = 0xFFFFFFFFFFFFFFFF


def make_values(n, seed):
    """Value keys of n rows: int64 values in [-10^6, 10^6) (value_keys), every 10th row without a value (key 0)."""
    from nornicdb_b200.knn import value_keys
    v = value_keys(np.random.default_rng(seed).integers(-10 ** 6, 10 ** 6, n))
    v[::10] = 0
    return v


def mixed_windows(Q, keys):
    """The window kinds a mixed batch carries, cycled over the queries (7 kinds against the filters' 8: every pairing occurs)."""
    from nornicdb_b200.knn import EMPTY_WINDOW
    u = np.unique(keys[keys != 0])
    m = len(u)
    kinds = [
        (0, ALL),                                  # admits every row, with or without a value
        EMPTY_WINDOW,                              # admits none
        (int(u[m // 2]), int(u[m // 2 + m // 300])),  # < 1%, lo and hi existing keys
        (int(u[100]), int(u[102])),                # 3 values: fewer admissible rows than k
        (1, ALL),                                  # every row with a value
        (int(u[m // 4]) + 1, int(u[3 * m // 4]) - 1),  # ~50%, bounds between keys
        (0, int(u[m // 3])),                       # rows without a value and the lowest third
    ]
    return np.array([kinds[q % len(kinds)] for q in range(Q)], dtype=np.uint64)


def in_windows(keys, windows):
    from nornicdb_b200.knn import window_admits
    return np.stack([window_admits(keys, int(lo), int(hi)) for lo, hi in windows])


CASES = ([("simt", 3, m, "f32") for m in ("cosine", "dot", "euclidean")]
         + [("shadow", 40, m, dt) for m in ("cosine", "dot", "euclidean") for dt in ("f32", "f16", "bf16")]
         + [("filter", 40, m, "f32") for m in ("cosine", "dot", "euclidean")]
         + [("tensor", 40, m, "f32") for m in ("cosine", "dot")]
         + [("auto", 300, m, "f32") for m in ("cosine", "dot", "euclidean")]
         + [("int8", 40, m, "f32") for m in ("cosine", "dot", "euclidean")])


def _index(monkeypatch, d, metric, dtype, path):
    from nornicdb_b200.knn import KnnIndex
    if path == "int8":
        monkeypatch.setenv("NK_SHADOW", "int8")  # read at creation: the int8 image is the shard's only image
    ix = KnnIndex(d, metric=metric, dtype=dtype)
    ix.set_path("shadow" if path == "int8" else path)
    return ix


@pytest.mark.parametrize("path,Q,metric,dtype", CASES)
def test_windowed_parity_every_path(knn_lib, oracle_mod, monkeypatch, path, Q, metric, dtype):
    """Mixed windows (every row, none, < 1%, fewer than k, lo / hi on existing keys, rows without a value) alone and together
    with mixed tag filters, on every path: exact results over each query's admissible rows, padding past them."""
    n, d, k = 20_000, 128, 10
    rows = oracle_mod.fill_uniform(n, d, 11)
    q = oracle_mod.fill_uniform(Q, d, 12)
    tags, keys = make_tags(n, 5), make_values(n, 6)
    filters, windows = mixed_filters(Q), mixed_windows(Q, keys)
    ix = _index(monkeypatch, d, metric, dtype, path)
    try:
        ix.upload(rows)
        ix.set_row_tags(tags)
        ix.set_row_values(keys)
        wi, ws = ix.search_windowed(q, k, windows)
        bi, bs = ix.search_windowed(q, k, windows, filters)
        if path != "auto":
            assert ix.last_path() == ("shadow" if path == "int8" else path)
        assert ix.debug_flags()[0] == 0
        held = rows_of(ix, rows)
    finally:
        ix.release()
    win = in_windows(keys, windows)
    check_filtered(held, q, k, metric, wi, ws, win)
    check_filtered(held, q, k, metric, bi, bs, win & admissible(tags, filters))


@pytest.mark.parametrize("path,Q", [("simt", 3), ("shadow", 40), ("filter", 40), ("tensor", 40), ("auto", 300), ("int8", 40)])
def test_best_rows_outside_the_window_never_raise_a_threshold(knn_lib, oracle_mod, monkeypatch, path, Q):
    """Each query's true top 300 rows get values below every window.  If a sample, prune, publish or flood step let one of them
    raise a threshold, admissible rows would be lost."""
    from nornicdb_b200.knn import value_keys
    n, d, k = 30_000, 128, 10
    metric = "dot" if path == "tensor" else "cosine"
    rows = oracle_mod.fill_uniform(n, d, 21)
    q = oracle_mod.fill_uniform(Q, d, 22)
    S = fp64_scores(rows, q, metric)
    v = np.random.default_rng(23).integers(1000, 2000, n)
    for qi in range(Q):
        v[np.argsort(-S[qi], kind="stable")[:300]] = qi % 1000  # below every window
    keys = value_keys(v)
    windows = np.array([(int(value_keys(np.int64(1000))), int(value_keys(np.int64(2000 - qi % 500)))) for qi in range(Q)], dtype=np.uint64)
    ix = _index(monkeypatch, d, metric, "f32", path)
    try:
        ix.upload(rows)
        ix.set_row_values(keys)
        gi, gs = ix.search_windowed(q, k, windows)
        assert ix.debug_flags()[0] == 0
    finally:
        ix.release()
    check_filtered(rows, q, k, metric, gi, gs, in_windows(keys, windows))


@pytest.mark.parametrize("path", ["simt", "shadow", "filter", "tensor"])
def test_same_window_everywhere_equals_row_mask(knn_lib, oracle_mod, path):
    """One window for the whole batch gives bit-identical results to nk_search under the equivalent row mask; {0, ~0} windows
    give search_filtered's results and windows=None search's / search_filtered's, bit for bit."""
    from nornicdb_b200.knn import KnnIndex, window_admits
    n, d, k, Q = 20_000, 256, 10, (3 if path == "simt" else 40)
    rows = oracle_mod.fill_uniform(n, d, 31)
    q = oracle_mod.fill_uniform(Q, d, 32)
    tags, keys = make_tags(n, 6), make_values(n, 7)
    u = np.unique(keys[keys != 0])
    w = (int(u[len(u) // 5]), int(u[len(u) // 2]))
    filters = mixed_filters(Q)
    ix = KnnIndex(d, metric="dot" if path == "tensor" else "cosine")
    try:
        ix.upload(rows)
        ix.set_row_tags(tags)
        ix.set_row_values(keys)
        ix.set_path(path)
        wi, ws = ix.search_windowed(q, k, w)
        ai, as_ = ix.search_windowed(q, k, (0, ALL), filters)
        fi, fs = ix.search_filtered(q, k, filters)
        ni, ns = ix.search_windowed(q, k, None)
        nfi, nfs = ix.search_windowed(q, k, None, filters)
        pi, ps = ix.search(q, k)
        ix.set_row_mask(window_admits(keys, *w))
        mi, ms = ix.search(q, k)
    finally:
        ix.release()
    assert (wi == mi).all() and (ws.view(np.uint32) == ms.view(np.uint32)).all()
    assert (ai == fi).all() and (as_.view(np.uint32) == fs.view(np.uint32)).all()
    assert (nfi == fi).all() and (nfs.view(np.uint32) == fs.view(np.uint32)).all()
    assert (ni == pi).all() and (ns.view(np.uint32) == ps.view(np.uint32)).all()


@pytest.mark.parametrize("path,metric", [("simt", "cosine"), ("shadow", "dot"), ("filter", "euclidean")])
def test_windowed_range_equals_range_under_row_mask(knn_lib, oracle_mod, path, metric):
    """nk_search_range_windowed with one window for every query equals nk_search_range under the equivalent row mask, bit for
    bit; windows=None is nk_search_range; mixed windows and filters keep exactly the admissible rows above the threshold."""
    from nornicdb_b200.knn import KnnIndex, window_admits
    n, d, Q = 20_000, 128, (3 if path == "simt" else 40)
    rows = oracle_mod.fill_uniform(n, d, 61)
    q = oracle_mod.fill_uniform(Q, d, 62)
    tags, keys = make_tags(n, 8), make_values(n, 9)
    u = np.unique(keys[keys != 0])
    w = (int(u[len(u) // 3]), ALL)
    thr = {"cosine": 0.1, "dot": 1.5, "euclidean": 9.0}[metric]
    filters, windows = mixed_filters(Q), mixed_windows(Q, keys)
    ix = KnnIndex(d, metric=metric)
    try:
        ix.upload(rows)
        ix.set_row_tags(tags)
        ix.set_row_values(keys)
        ix.set_path(path)
        got = ix.search_range(q, thr, windows=w)
        plain = ix.search_range(q, thr)
        none = ix.search_range(q, thr, windows=None)
        mixed = ix.search_range(q, thr, filters, windows)
        ix.set_row_mask(window_admits(keys, *w))
        want = ix.search_range(q, thr)
    finally:
        ix.release()
    for qi in range(Q):
        assert (got[qi][0] == want[qi][0]).all() and (got[qi][1].view(np.uint32) == want[qi][1].view(np.uint32)).all(), qi
        assert (none[qi][0] == plain[qi][0]).all() and (none[qi][1].view(np.uint32) == plain[qi][1].view(np.uint32)).all(), qi
    S = fp64_scores(rows, q, metric)
    adm = admissible(tags, filters) & in_windows(keys, windows)
    ok = S >= (-thr if metric == "euclidean" else thr)
    for qi in range(Q):
        expect = set(np.flatnonzero(adm[qi] & ok[qi]).tolist())
        gotset = set(mixed[qi][0].tolist())
        # rows whose fp64 score sits within rounding of the threshold may fall either way
        edge = set(np.flatnonzero(adm[qi] & (np.abs(S[qi] - (-thr if metric == "euclidean" else thr)) < 1e-5)).tolist())
        assert gotset - edge == expect - edge, qi
        assert adm[qi][mixed[qi][0].astype(np.int64)].all(), qi


@pytest.mark.parametrize("api", ["host", "device"])
@pytest.mark.parametrize("path,n,noise,metric", [
    pytest.param(path, n, noise, metric, id=f"{path}-{n}-{noise}" + ("" if metric == "cosine" else f"-{metric}"))
    for path, n, noise in [("filter", 20_000, 1e-5), ("shadow", 160_000, 1e-4)] for metric in ("cosine", "dot", "euclidean")])
def test_retry_and_exact_tail_honour_the_windows(knn_lib, oracle_mod, api, path, n, noise, metric):
    """The near-tie corpora of test_retry_and_exact_tail_honour_the_filters overflow the filter stages; the retry / exact
    kernels (deferred by the host API, queued blindly by the device API) must apply the same windows and filters."""
    import torch
    from nornicdb_b200.knn import KnnIndex
    rows, q = _near_tie_corpus(oracle_mod, n, noise, 1 if path == "shadow" else 0)
    Q, k = q.shape[0], 10
    tags, keys = make_tags(n, 8), make_values(n, 10)
    filters, windows = mixed_filters(Q), mixed_windows(Q, keys)
    filters[::2] = 0  # unfiltered queries keep the margin buffers overflowing
    windows[::4] = (0, ALL)
    ix = KnnIndex(128, metric=metric)
    try:
        ix.upload(rows)
        ix.set_row_tags(tags)
        ix.set_row_values(keys)
        ix.set_path(path)
        if api == "host":
            gi, gs = ix.search_windowed(q, k, windows, filters)
        else:
            qd = torch.from_numpy(q).cuda()
            fd = torch.from_numpy(filters.view(np.int64)).cuda()
            wd = torch.from_numpy(windows.view(np.int64)).cuda()
            oi = torch.empty((Q, k), dtype=torch.int32, device="cuda")
            os_ = torch.empty((Q, k), dtype=torch.float32, device="cuda")
            ix.search_windowed_device(qd.data_ptr(), fd.data_ptr(), wd.data_ptr(), Q, k, oi.data_ptr(), os_.data_ptr(), 0)
            ix.status(0)
            gi, gs = oi.cpu().numpy().view(np.uint32), os_.cpu().numpy()
        flags = ix.debug_flags()
    finally:
        ix.release()
    assert flags[0] == 0
    if path == "shadow" and api == "host":
        assert flags[3] == 1, flags  # the 16-bit stage overflowed; the TF32 stage re-ran the search
    else:
        assert flags[1] != 0, flags  # a stage overflowed; the exact kernels answered
    check_filtered(rows, q, k, metric, gi, gs, admissible(tags, filters) & in_windows(keys, windows), swap_eps=5e-6)


def test_device_api_windows_without_filters(knn_lib, oracle_mod):
    """nk_search_windowed_device with filters_dev NULL: the library stages the admit-all filters itself."""
    import torch
    from nornicdb_b200.knn import KnnIndex
    n, d, Q, k = 20_000, 128, 40, 10
    rows = oracle_mod.fill_uniform(n, d, 71)
    q = oracle_mod.fill_uniform(Q, d, 72)
    keys = make_values(n, 73)
    windows = mixed_windows(Q, keys)
    ix = KnnIndex(d, metric="cosine")
    try:
        ix.upload(rows)
        ix.set_row_values(keys)
        ix.set_path("shadow")
        qd = torch.from_numpy(q).cuda()
        wd = torch.from_numpy(windows.view(np.int64)).cuda()
        oi = torch.empty((Q, k), dtype=torch.int32, device="cuda")
        os_ = torch.empty((Q, k), dtype=torch.float32, device="cuda")
        ix.search_windowed_device(qd.data_ptr(), 0, wd.data_ptr(), Q, k, oi.data_ptr(), os_.data_ptr(), 0)
        ix.status(0)
        gi, gs = oi.cpu().numpy().view(np.uint32), os_.cpu().numpy()
        hi, hs = ix.search_windowed(q, k, windows)
    finally:
        ix.release()
    check_filtered(rows, q, k, "cosine", gi, gs, in_windows(keys, windows))
    assert (gi == hi).all() and (gs.view(np.uint32) == hs.view(np.uint32)).all()


@pytest.mark.parametrize("devices", [(0,), (0, 0)])
def test_values_follow_the_rows(knn_lib, oracle_mod, devices):
    """set_row_values on partial ranges (spanning shards), append, update_row, remove_swap, reset by upload."""
    from nornicdb_b200.knn import KnnIndex, value_keys, window
    d = 64
    rows = oracle_mod.fill_uniform(600, d, 51)
    extra = oracle_mod.fill_uniform(50, d, 52)
    q = oracle_mod.fill_uniform(3, d, 53)
    V = int(value_keys(np.int64(7)))
    win = np.array([window(gte=7, lte=7), (0, V - 1), (0, ALL)], dtype=np.uint64)  # value 7 / no value or below 7 / every row
    ix = KnnIndex(d, metric="dot", devices=devices)
    ix.set_path("simt")
    try:
        ix.upload(rows)
        keys = np.zeros(600, dtype=np.uint64)
        keys[250:350] = V                      # a range crossing the shard boundary of (0, 0)
        ix.set_row_values(keys[250:350], first_row=250)
        keys[10] = V
        ix.set_row_values(np.array([7]), first_row=10)  # numbers are encoded on the way in
        cur = rows.copy()

        def check():
            gi, gs = ix.search_windowed(q, 1024, win)
            adm = in_windows(keys, win)
            for qi in range(3):
                got = gi[qi][gi[qi] != PAD]
                assert sorted(got.tolist()) == np.flatnonzero(adm[qi]).tolist(), qi
            check_filtered(cur, q, gi.shape[1], "dot", gi, gs, adm)

        check()
        ix.append(extra)                       # appended rows: key 0
        keys = np.concatenate([keys, np.zeros(50, dtype=np.uint64)])
        cur = np.concatenate([cur, extra])
        check()
        ix.update_row(300, q[0] * 4.0)         # row keeps its key
        cur[300] = q[0] * 4.0
        check()
        keys[-1] = V
        ix.set_row_values(keys[-1:], first_row=len(keys) - 1)
        ix.remove_swap(20)                     # the last row (with a value) moves into slot 20 with its key
        keys[20] = keys[-1]; keys = keys[:-1]
        cur[20] = cur[-1]; cur = cur[:-1]
        check()
        ix.remove_swap(280)                    # a row without a value moves into a valued slot: the slot's key becomes 0
        keys[280] = keys[-1]; keys = keys[:-1]
        cur[280] = cur[-1]; cur = cur[:-1]
        check()
        ix.upload(rows)                        # every key back to 0
        keys = np.zeros(600, dtype=np.uint64)
        cur = rows.copy()
        check()
    finally:
        ix.release()


def test_large_k_multi_pass(knn_lib, oracle_mod):
    """k > NK_MAX_K: the multi-pass CUDA-core route applies the windows in every pass, including windows with fewer
    admissible rows than k."""
    from nornicdb_b200.knn import NK_MAX_K, KnnIndex
    n, d, Q, k = 20_000, 64, 6, NK_MAX_K + 500
    rows = oracle_mod.fill_uniform(n, d, 81)
    q = oracle_mod.fill_uniform(Q, d, 82)
    keys = make_values(n, 83)
    windows = mixed_windows(Q + 1, keys)[[0, 2, 3, 4, 5, 6]]
    ix = KnnIndex(d, metric="cosine")
    try:
        ix.upload(rows)
        ix.set_row_values(keys)
        gi, gs = ix.search_windowed(q, k, windows)
        assert ix.last_path() == "simt"
    finally:
        ix.release()
    check_filtered(rows, q, k, "cosine", gi, gs, in_windows(keys, windows))


def test_headline_shape_last_window_planted(knn_lib, oracle_mod):
    """N=10M d=1024 fp32 Q=64 k=10 cosine, row values are timestamps: each query asks for the last window of its own length,
    with a planted near-copy inside it (must come first) and a closer one just before it (must never appear); every returned
    row lies in the window and every score is recomputed in fp64."""
    from nornicdb_b200.knn import KnnIndex, value_keys, window, window_admits
    n, d, Q, k = 10_000_000, 1024, 64, 10
    now = np.datetime64("2026-01-01T00:00:00", "ns")
    rng = np.random.default_rng(9)
    ts = now - rng.integers(0, 365 * 86400, n).astype("timedelta64[s]")  # one year of timestamps
    ix = KnnIndex(d, metric="cosine")
    try:
        ix.fill_uniform(n, 42)
        q = oracle_mod.fill_uniform(Q, d, 1337)
        days = [1, 7, 30, 90]
        wins = [window(gte=now - np.timedelta64(days[qi % 4], "D"), lte=now) for qi in range(Q)]
        picks = rng.choice(n, size=2 * Q, replace=False)
        good = {qi: int(picks[2 * qi]) for qi in range(Q)}
        bad = {qi: int(picks[2 * qi + 1]) for qi in range(Q)}
        for qi in range(Q):
            ix.update_row(good[qi], (q[qi] * 1.5).astype(np.float32))
            ts[good[qi]] = now - np.timedelta64(3600, "s")                        # inside every window
            ix.update_row(bad[qi], (q[qi] * 1.7).astype(np.float32))
            ts[bad[qi]] = now - np.timedelta64(days[qi % 4], "D") - np.timedelta64(1, "ns")  # one ns before the window
        keys = value_keys(ts)
        ix.set_row_values(keys)
        gi, gs = ix.search_windowed(q, k, np.array(wins, dtype=np.uint64))
        assert ix.last_path() == "shadow" and ix.debug_flags()[0] == 0
        for qi in range(Q):
            assert window_admits(keys[gi[qi].astype(np.int64)], *wins[qi]).all(), qi
            assert gi[qi][0] == good[qi], (qi, gi[qi][:3], good[qi])
            assert bad[qi] not in gi[qi].tolist(), qi
            r = np.stack([ix.read_rows(int(x), 1)[0] for x in gi[qi]])
            ex = exact_scores_for(r, q[qi], np.arange(k), "cosine")
            assert np.allclose(gs[qi], ex, rtol=1e-4, atol=1e-6), qi
            assert (np.diff(gs[qi].astype(np.float64)) <= 1e-7).all()
    finally:
        ix.release()
