"""GPU tests of range search (nk_search_range): every admissible row whose exact fp32 score meets the query's threshold.

Results are checked against fp64: rows farther than 2e-6 * scale from the threshold must be returned iff they meet it,
rows inside that band may go either way (counted and reported).  Every path (16-bit, TF32 filter, CUDA cores) must return
bit-identical lists, and a threshold set to the k-th score of nk_search must reproduce nk_search's list bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PATHS_BY_DTYPE = {"f32": ("shadow", "filter", "simt"), "f16": ("shadow", "simt"), "bf16": ("shadow", "simt")}
BAND = 2e-6


def rounded(rows, dtype):
    from nornicdb_b200.knn import from_bf16_bits, to_bf16_bits
    if dtype == "f16":
        return rows.astype(np.float16).astype(np.float32)
    if dtype == "bf16":
        return from_bf16_bits(to_bf16_bits(rows))
    return rows


def fp64_keys(rows, q, metric):
    """fp64 score in key space (cosine / dot: score; euclidean: -distance^2) and the band's scale per (query, row)."""
    x = np.asarray(rows, dtype=np.float64)
    qq = np.asarray(q, dtype=np.float64)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        s = qq @ x.T
        xn, qn = np.linalg.norm(x, axis=1)[None, :], np.linalg.norm(qq, axis=1)[:, None]
        if metric == "cosine":
            den = qn * xn
            return np.where(den > 0, s / den, 0.0), np.ones_like(s)
        if metric == "dot":
            return s, np.maximum(qn * xn, 1.0)
        return -np.maximum(qn ** 2 + xn ** 2 - 2.0 * s, 0.0), np.maximum(qn ** 2 + xn ** 2, 1.0)


def key_threshold(t, metric):
    return -(t * t) if metric == "euclidean" else t


def check_range(res, keys, scale, thr, metric, adm=None):
    """res: search_range output; keys / scale [Q, n] from fp64_keys; thr: API thresholds [Q].  Returns rows in the band."""
    band_rows = 0
    for qi, (idx, sc) in enumerate(res):
        k = keys[qi]
        tk = key_threshold(float(thr[qi]), metric)
        ok = np.isfinite(k) & (k >= tk)
        if adm is not None:
            ok &= adm[qi]
        in_band = np.isfinite(k) & (np.abs(k - tk) <= BAND * scale[qi])
        got = np.zeros(len(k), dtype=bool)
        got[idx.astype(np.int64)] = True
        assert len(np.unique(idx)) == len(idx), f"query {qi}: duplicate rows"
        missing = ok & ~got & ~in_band
        extra = got & ~ok & ~in_band
        if adm is not None:
            assert adm[qi][idx.astype(np.int64)].all(), f"query {qi}: inadmissible row returned"
        assert not missing.any(), f"query {qi}: rows meeting the threshold not returned: {np.flatnonzero(missing)[:8]}"
        assert not extra.any(), f"query {qi}: rows below the threshold returned: {np.flatnonzero(extra)[:8]}"
        band_rows += int((in_band & (got != ok)).sum())
        if len(idx):
            ref = k[idx.astype(np.int64)]
            ref_sc = np.sqrt(-ref) if metric == "euclidean" else ref
            assert np.all(np.abs(sc - ref_sc) <= 1e-4 * np.maximum(np.abs(ref_sc), 1.0)), f"query {qi}: scores off fp64"
            # order: score desc, ties by row asc; euclidean: by the exact squared distance, so the returned distances (its
            # sqrtf) only never decrease
            r = idx.astype(np.int64)
            if metric == "euclidean":
                assert np.all(sc[:-1] <= sc[1:]), f"query {qi}: order"
            else:
                assert np.all((sc[:-1] > sc[1:]) | ((sc[:-1] == sc[1:]) & (r[:-1] < r[1:]))), f"query {qi}: order"
    return band_rows


def thresholds_at_ranks(keys, ranks, metric):
    """API thresholds = the fp64 score of each query's ranks[q]-th best row (euclidean: as a distance)."""
    t = np.empty(keys.shape[0], dtype=np.float32)
    for qi in range(keys.shape[0]):
        v = np.sort(keys[qi][np.isfinite(keys[qi])])[::-1]
        kk = v[min(ranks[qi % len(ranks)], len(v)) - 1]
        t[qi] = np.sqrt(-kk) if metric == "euclidean" else kk
    return t


def make_index(rows, metric, dtype, devices=(0,)):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex(rows.shape[1], metric=metric, dtype=dtype, devices=devices)
    ix.upload_from_f32(rows)
    return ix


@pytest.mark.parametrize("dtype", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_range_against_fp64_every_path(knn_lib, oracle_mod, metric, dtype):
    """Step 1 and 2: every path against fp64, and every path bit-identical to every other."""
    n, d, Q = 20_000, 128, 8
    rows = oracle_mod.fill_uniform(n, d, 11)
    q = oracle_mod.fill_uniform(Q, d, 12)
    r = rounded(rows, dtype)
    keys, scale = fp64_keys(r, q, metric)
    thr = thresholds_at_ranks(keys, [10, 500, 5000, 1], metric)
    ix = make_index(rows, metric, dtype)
    outs = {}
    for path in PATHS_BY_DTYPE[dtype]:
        ix.set_path(path)
        res = ix.search_range(q, thr)
        assert ix.last_path() == path
        band = check_range(res, keys, scale, thr, metric)
        print(f"{metric} {dtype} {path}: {sum(len(i) for i, _ in res)} results, {band} rows inside the band")
        outs[path] = res
    ref = outs[PATHS_BY_DTYPE[dtype][0]]
    for path, res in outs.items():
        for qi in range(Q):
            assert np.array_equal(res[qi][0], ref[qi][0]) and np.array_equal(res[qi][1].view(np.uint32), ref[qi][1].view(np.uint32)), (path, qi)
    ix.release()


@pytest.mark.parametrize("path", ["shadow", "filter", "simt"])
def test_mixed_batch_long_lists_filters_mask_floor_nan(knn_lib, oracle_mod, path):
    """Step 3: one query matching nothing, one matching > 200 000 rows (long-list sort, list retry on a fresh index), the
    rest in between; per-query tag filters, the row mask and the score floor together; rows with a NaN score (an Inf
    component: inf / inf) never returned.  A NaN component scores 0 under cosine (the zero-vector rule of nk_search), so
    those rows follow their threshold like any other."""
    from nornicdb_b200.knn import admits, synthetic_tags
    n, d, Q = 300_000, 64, 8
    rows = oracle_mod.fill_uniform(n, d, 21)
    bad = np.arange(7, n, 50_001)
    rows[bad[::2], 3] = np.nan
    rows[bad[1::2], 5] = np.inf
    q = oracle_mod.fill_uniform(Q, d, 22)
    tags = synthetic_tags(n, 5) & np.uint64(0xF)
    filters = np.array([(0, 0, 0), (1, 0, 0), (0, 2, 0), (0, 0, 12), (0, 0, 0), (3, 0, 0), (0, 0, 0), (0, 1, 0)], dtype=np.uint64)
    keep = np.ones(n, dtype=bool)
    keep[::97] = False
    floor = -0.3
    ix = make_index(rows, "cosine", "f32")
    ix.set_row_tags(tags)
    ix.set_row_mask(keep)
    ix.set_min_score(floor)
    ix.set_path(path)
    keys, scale = fp64_keys(rows, q, "cosine")
    thr = np.array([2.0, -1.0, 0.1, 0.2, -np.inf, 0.05, 0.3, 0.15], dtype=np.float32)
    res = ix.search_range(q, thr, filters)
    adm = np.stack([admits(tags, *[int(v) for v in f]) for f in filters]) & keep[None, :]
    eff = np.maximum(thr, floor)
    band = check_range(res, keys, scale, eff, "cosine", adm)
    assert len(res[0][0]) == 0
    assert len(res[4][0]) > 200_000
    for idx, _ in res:
        assert not np.isin(idx.astype(np.int64), bad[1::2]).any(), "a row with a NaN score was returned"
    print(f"{path}: counts {[len(i) for i, _ in res]}, {band} rows inside the band")
    ix.release()


@pytest.mark.parametrize("path", ["shadow", "filter", "simt"])
@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_threshold_at_kth_score_reproduces_search(knn_lib, oracle_mod, path, metric):
    """Step 4 (small): threshold = the k-th score of nk_search -> the first k entries are nk_search's, bit for bit, and every
    further entry scores exactly the threshold."""
    n, d, Q, k = 50_000, 128, 16, 100
    rows = oracle_mod.fill_uniform(n, d, 31)
    q = oracle_mod.fill_uniform(Q, d, 32)
    ix = make_index(rows, metric, "f32")
    ix.set_path(path)
    gi, gs = ix.search(q, k)
    res = ix.search_range(q, gs[:, k - 1])
    for qi, (idx, sc) in enumerate(res):
        assert np.array_equal(idx[:k], gi[qi]) and np.array_equal(sc[:k].view(np.uint32), gs[qi].view(np.uint32)), qi
        assert np.all(sc[k:].view(np.uint32) == gs[qi, k - 1].view(np.uint32)), qi
    ix.release()


def test_size_protocol_empty_q0_and_two_shards(knn_lib, oracle_mod):
    """Step 5: capacity too small writes only the offsets and the total; exact capacity writes the results; an empty index
    and Q = 0; two shards on one device merge to the one-shard result."""
    import ctypes as C
    from nornicdb_b200.knn import KnnIndex
    n, d, Q = 30_000, 64, 6
    rows = oracle_mod.fill_uniform(n, d, 41)
    q = oracle_mod.fill_uniform(Q, d, 42)
    thr = np.array([0.3, 0.2, 0.25, 2.0, 0.1, 0.35], dtype=np.float32)
    one = make_index(rows, "cosine", "f32")
    lib = one.lib
    off = np.zeros(Q + 1, dtype=np.uint64)
    total = C.c_uint64(0)
    sentinel_i = np.full(8, 0xDEADBEEF, dtype=np.uint32)
    sentinel_s = np.full(8, 7.0, dtype=np.float32)
    qq = np.ascontiguousarray(q)
    args = lambda cap, oi, os_: (one.ptr, qq.ctypes.data_as(C.c_void_p), thr.ctypes.data_as(C.c_void_p), None, Q, cap,
                                 off.ctypes.data_as(C.c_void_p), oi.ctypes.data_as(C.c_void_p), os_.ctypes.data_as(C.c_void_p), C.byref(total))
    assert lib.nk_search_range(*args(8, sentinel_i, sentinel_s)) == 0
    need = total.value
    assert need > 8 and off[-1] == need and off[0] == 0
    assert (sentinel_i == 0xDEADBEEF).all() and (sentinel_s == 7.0).all(), "nothing but the sizes may be written"
    off_small = off.copy()
    oi = np.empty(need, dtype=np.uint32)
    os_ = np.empty(need, dtype=np.float32)
    assert lib.nk_search_range(*args(need, oi, os_)) == 0
    assert total.value == need and np.array_equal(off, off_small)
    ref = one.search_range(q, thr)
    for qi in range(Q):
        assert np.array_equal(oi[int(off[qi]):int(off[qi + 1])], ref[qi][0])
    assert len(ref[3][0]) == 0
    assert one.search_range(np.empty((0, d), np.float32), []) == []
    two = make_index(rows, "cosine", "f32", devices=(0, 0))
    for path in ("shadow", "simt"):
        one.set_path(path)
        two.set_path(path)
        a, b = one.search_range(q, thr), two.search_range(q, thr)
        for qi in range(Q):
            assert np.array_equal(a[qi][0], b[qi][0]) and np.array_equal(a[qi][1], b[qi][1]), (path, qi)
    empty = KnnIndex(d)
    assert all(len(i) == 0 for i, _ in empty.search_range(q, thr))
    with pytest.raises(Exception):
        one.search_range(q, np.full(Q, np.nan, np.float32))
    for ix in (one, two, empty):
        ix.release()


@pytest.fixture(scope="module")
def big_index(knn_lib):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex(1024, metric="cosine")
    ix.fill_uniform(10_000_000, 42)
    yield ix
    ix.release()


def test_10m_threshold_at_kth_score_reproduces_search(big_index, oracle_mod):
    """Step 4 at N = 10M, d = 1024, Q = 64 (filled on the device): no fp64 oracle needed."""
    q = oracle_mod.fill_uniform(64, 1024, 1337)
    k = 100
    gi, gs = big_index.search(q, k)
    res = big_index.search_range(q, gs[:, k - 1])
    assert big_index.last_path() == "shadow"
    for qi, (idx, sc) in enumerate(res):
        assert np.array_equal(idx[:k], gi[qi]) and np.array_equal(sc[:k].view(np.uint32), gs[qi].view(np.uint32)), qi
        assert np.all(sc[k:].view(np.uint32) == gs[qi, k - 1].view(np.uint32)), qi


def test_10m_about_1e5_rows_per_query_against_torch_fp64(big_index, oracle_mod):
    """Step 6: thresholds yielding ~10^5 rows per query at N = 10M, against an fp64 count on the same GPU (rows regenerated
    slice by slice with the index's generator, scored in torch fp64) outside the band."""
    import torch
    from nornicdb_b200.knn import fill_uniform_device
    n, d, Q = 10_000_000, 1024, 16
    q = oracle_mod.fill_uniform(Q, d, 2024)
    thr = np.full(Q, 0.0728, dtype=np.float32) + np.linspace(-0.004, 0.004, Q, dtype=np.float32)
    res = big_index.search_range(q, thr)
    counts = [len(i) for i, _ in res]
    assert min(counts) > 50_000 and max(counts) < 200_000, counts
    got = torch.zeros((Q, n), dtype=torch.bool, device="cuda")
    for qi, (idx, _) in enumerate(res):
        got[qi, torch.from_numpy(idx.astype(np.int64)).cuda()] = True
    q64 = torch.from_numpy(q.astype(np.float64)).cuda()
    q64 = q64 / q64.norm(dim=1, keepdim=True)
    t64 = torch.from_numpy(thr.astype(np.float64)).cuda()[:, None]
    band = 0
    step = 500_000
    for lo in range(0, n, step):
        x = torch.empty((step, d), dtype=torch.float32, device="cuda")
        fill_uniform_device(0, x.data_ptr(), step, d, 42, lo, 0)
        torch.cuda.synchronize()
        x64 = x.double()
        s = (q64 @ x64.T) / x64.norm(dim=1)[None, :]
        ok = s >= t64
        in_band = (s - t64).abs() <= BAND
        g = got[:, lo:lo + step]
        assert not (ok & ~g & ~in_band).any(), f"slice {lo}: rows meeting the threshold not returned"
        assert not (g & ~ok & ~in_band).any(), f"slice {lo}: rows below the threshold returned"
        band += int((in_band & (g != ok)).sum())
        del x, x64, s
    print(f"10M range: counts {counts}, {band} rows inside the band")
