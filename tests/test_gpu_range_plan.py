"""Range search, the self-join and the incident pairs at the list, sort, batch and launch sizes where their plan changes.

The sizes come from tests/range_plan.py, which reads the library's constants and restates its rules.  Each case runs on a
planted corpus: every query has an exact, chosen number of rows above its own threshold and a gap on both sides of it many
times wider than any filter's error bound, so on every path the list fill equals the survivor count, no row falls in the
band of tests/test_gpu_range.py, and the paths and shard layouts must agree bit for bit.  The plan that ran is observed,
not assumed: last_path(), the scan passes from NkStats::bytes_scanned (a list capacity retry scans twice), and each call's
NkStats::kernel_launches against range_plan.range_launches (the scan launch split, the query blocks, the merge passes)."""
import ctypes as C

import numpy as np
import pytest

import range_plan as rp
from test_gpu_pairs_update import check_incident
from test_gpu_range import check_range, fp64_keys, rounded
from test_gpu_search_pairs import assert_same, by_range

pytestmark = pytest.mark.gpu

# (dtype, path, NK_SHADOW): every path a d = 64 shape admits; the fp32 16-bit pass over the BF16 shadow or the int8 image
PATHS = [("f32", "simt", None), ("f32", "filter", None), ("f32", "shadow", "bf16"), ("f32", "shadow", "int8"),
         ("f16", "simt", None), ("f16", "shadow", None), ("bf16", "simt", None), ("bf16", "shadow", None)]

# (a) list capacity: one query's fill on a fresh index
CAP_FILLS = [rp.LIST0 - 1, rp.LIST0, rp.LIST0 + 1]
# (b) re-scoring CTAs, compaction CTAs, run sort and merge passes: survivors per query
R = rp.RUN
SURVIVORS = [0, 1, rp.CP_THREADS - 1, rp.CP_THREADS, rp.CP_THREADS + 1, rp.RS_ENTRIES - 1, rp.RS_ENTRIES, rp.RS_ENTRIES + 1,
             R - 1, R, R + 1, 2 * R - 1, 2 * R, 2 * R + 1, 4 * R, 4 * R + 1]
# (c) the query blocks of MAX_GRID_Y
BLOCK_QS = [rp.MAX_GRID_Y, rp.MAX_GRID_Y + 1, rp.MAX_GRID_Y + 65]
BLOCK_N, BLOCK_D = 10_000, 32
# (d) the scan launch plan
PLAN_QS = [64, 65, 128, 129, 384, 385, 512, 513, 640, 641]
PLAN_GRIDS = [rp.NUM_SMS_H100, 8, 7, 6, 4, 3, 1]
SIMT_QS = [1, 2, 3, 4, 5, 8, 9, 13]
SATURATE_Q, SATURATE_N = 641, 8 * rp.ROWS - 37
# (e) the self-join: stripes starting 1, 2, 3 and 4 tiles in plus 44 rows, and a cluster whose lowest row pairs with every
# other member
PAIRS_N, PAIRS_STARTS, PAIRS_CLUSTER, PAIRS_LOW = 6000, [300, 556, 812, 1068], R + 2, 310


# ---- helpers ------------------------------------------------------------------------------------------------------------
def make(monkeypatch, rows, metric, dtype="f32", image=None, devices=(0,)):
    """a fresh index; image: the one image fp32 shards keep (NK_SHADOW, read at creation), None: the default"""
    from nornicdb_b200.knn import KnnIndex
    if image is None:
        monkeypatch.delenv("NK_SHADOW", raising=False)
    else:
        monkeypatch.setenv("NK_SHADOW", image)
    ix = KnnIndex(rows.shape[1], metric=metric, dtype=dtype, devices=devices)
    ix.upload_from_f32(rows)
    return ix


def search_once(ix, path, q, thr, cap, filters=None, windows=None):
    """one nk_search_range_windowed call with room for `cap` results, so the stats deltas are one call's
    -> (results as search_range returns them, kernel_launches delta, bytes_scanned delta)"""
    from nornicdb_b200.knn import _check, as_filters, as_windows
    ix.set_path(path)
    q = np.ascontiguousarray(q, dtype=np.float32)
    Q = len(q)
    t = np.ascontiguousarray(thr, dtype=np.float32)
    f = None if filters is None else as_filters(filters, Q)
    w = None if windows is None else as_windows(windows, Q)
    off = np.zeros(Q + 1, dtype=np.uint64)
    idx = np.empty(max(cap, 1), dtype=np.uint32)
    sc = np.empty(max(cap, 1), dtype=np.float32)
    total = C.c_uint64(0)
    vp = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    before = ix.stats()
    _check(ix.lib.nk_search_range_windowed(ix.ptr, vp(q), vp(t), vp(f), vp(w), Q, cap, vp(off), vp(idx), vp(sc), C.byref(total)),
           "nk_search_range_windowed")
    after = ix.stats()
    assert ix.last_path() == path, (path, ix.last_path())
    assert total.value <= cap, f"{total.value} results, room for {cap}"
    o = off.astype(np.int64)
    res = [(idx[o[i]:o[i + 1]].copy(), sc[o[i]:o[i + 1]].copy()) for i in range(Q)]
    return res, after["kernel_launches"] - before["kernel_launches"], after["bytes_scanned"] - before["bytes_scanned"]


def passes(dbytes, path, n, d, dtype, image, Q):
    one = rp.scan_bytes(path, n, rp.row_bytes(path, d, dtype, image or "bf16"), Q, 1)
    assert dbytes % one == 0 and dbytes // one in (1, 2), (dbytes, one)
    return dbytes // one


def same_bits(a, b, what):
    assert len(a) == len(b), what
    for qi, ((ia, sa), (ib, sb)) in enumerate(zip(a, b)):
        assert np.array_equal(ia, ib) and np.array_equal(sa.view(np.uint32), sb.view(np.uint32)), f"{what}: query {qi}"


def check_planted(res, p, metric, admitted=None, what="", dtype="f32"):
    """every query returns exactly its planted (admitted) rows, in nk_search's order, scored as fp64 scores the stored rows"""
    x = rounded(p.rows, dtype).astype(np.float64)
    for qi, (idx, sc) in enumerate(res):
        want = p.expected(qi, None if admitted is None else admitted[qi % len(admitted)])
        got = np.sort(idx.astype(np.int64))
        assert np.array_equal(got, want), f"{what}: query {qi}: {len(got)} rows, want {len(want)}"
        if len(idx) == 0:
            continue
        k, _ = rp.keys64(x[idx.astype(np.int64)], p.queries[qi:qi + 1], metric)
        ref = np.sqrt(-k[0]) if metric == "euclidean" else k[0]
        assert np.all(np.abs(sc - ref) <= 1e-4 * np.maximum(np.abs(ref), 1.0)), f"{what}: query {qi}: scores off fp64"
        r = idx.astype(np.int64)
        if metric == "euclidean":
            assert np.all(sc[:-1] <= sc[1:]), f"{what}: query {qi}: order"
        else:
            assert np.all((sc[:-1] > sc[1:]) | ((sc[:-1] == sc[1:]) & (r[:-1] < r[1:]))), f"{what}: query {qi}: order"


def check_fp64(res, p, metric, dtype):
    """check_range against fp64 of the stored rows: no row may fall in the band"""
    keys, scale = fp64_keys(rounded(p.rows, dtype), p.queries, metric)
    assert check_range(res, keys, scale, p.thr, metric) == 0


def bounds_torch(rows, queries, owner, metric, chunk=4096):
    """range_plan.bounds_np in fp64 on the device, query slice by query slice"""
    import torch
    x = torch.from_numpy(rows.astype(np.float64)).cuda()
    own = torch.from_numpy(owner).cuda()
    xn = x.norm(dim=1)[None, :]
    out = [np.full(len(queries), np.nan) for _ in range(4)]
    for c in range(0, len(queries), chunk):
        q = torch.from_numpy(queries[c:c + chunk].astype(np.float64)).cuda()
        qn = q.norm(dim=1)[:, None]
        s = q @ x.T
        k, sc = (s / (qn * xn), torch.ones_like(s)) if metric == "cosine" else (s, qn * xn) if metric == "dot" else \
            (-(qn ** 2 + xn ** 2 - 2.0 * s), qn ** 2 + xn ** 2)
        mine = own[None, :] == torch.arange(c, c + len(q), device="cuda")[:, None]
        kb = torch.where(mine, torch.full_like(k, -np.inf), k)
        kp = torch.where(mine, k, torch.full_like(k, np.inf))
        ib, ip = kb.argmax(1), kp.argmin(1)
        r = torch.arange(len(q), device="cuda")
        has = mine.any(1)
        nan = torch.full((len(q),), np.nan, dtype=torch.float64, device="cuda")
        for o, v in zip(out, (kb[r, ib], torch.where(has, kp[r, ip], nan), sc[r, ib], torch.where(has, sc[r, ip], nan))):
            o[c:c + len(q)] = v.cpu().numpy()
        del s, k, sc, mine, kb, kp
    return tuple(out)


# ---- (a) list capacity and its one retry ------------------------------------------------------------------------------
@pytest.mark.parametrize("fill", CAP_FILLS)
def test_list_capacity_and_its_one_retry(knn_lib, monkeypatch, fill):
    """one query with `fill` survivors next to small ones: a fresh index scans once up to LIST0 and twice past it; the same
    call again scans once (the lists kept their size); an index that ran a kNN search first returns the same bits"""
    n, d, metric = 12_000, 64, "cosine"
    counts = np.array([3, fill, 0, 17, 1], dtype=np.int64)
    p = rp.planted(counts, d, metric, n, 1000 + fill)
    assert p.gap > 3 * rp.MIN_GAP
    first = {}
    for dtype, path, image in PATHS:
        what = f"{dtype} {path} {image}"
        ix = make(monkeypatch, p.rows, metric, dtype, image)
        res, dl, db = search_once(ix, path, p.queries, p.thr, int(counts.sum()))
        retried = fill > rp.LIST0
        assert passes(db, path, n, d, dtype, image, len(counts)) == (2 if retried else 1), what
        assert dl == rp.range_launches(path, len(counts), n, counts, retried, d, dtype), what
        check_fp64(res, p, metric, dtype)
        check_planted(res, p, metric, what=what, dtype=dtype)
        again, dl2, db2 = search_once(ix, path, p.queries, p.thr, int(counts.sum()))
        same_bits(again, res, f"{what}: again")
        assert passes(db2, path, n, d, dtype, image, len(counts)) == 1, what
        assert dl2 == rp.range_launches(path, len(counts), n, counts, False, d, dtype), what
        ix.release()
        used = make(monkeypatch, p.rows, metric, dtype, image)
        used.set_path(path)
        used.search(p.queries, 10)
        same_bits(search_once(used, path, p.queries, p.thr, int(counts.sum()))[0], res, f"{what}: after a kNN search")
        used.release()
        if dtype in first:
            same_bits(res, first[dtype], f"{what} vs the first {dtype} path")
        first.setdefault(dtype, res)


def test_two_shards_one_retries(knn_lib, monkeypatch):
    """two shards on one device, every planted row in the first: it scans twice, the other once, and the merged result is
    the one-shard index's"""
    n, d, metric = 12_000, 64, "dot"
    counts = np.array([rp.LIST0 + 1, 5, 0, rp.LIST0 - 1], dtype=np.int64)
    p = rp.planted(counts, d, metric, n, 7)
    order = np.argsort(p.owner < 0, kind="stable")  # planted rows first: all inside the first shard's n // 2 rows
    p.rows, p.owner = p.rows[order], p.owner[order]
    assert (p.owner[n // 2:] < 0).all()
    Q = len(counts)
    for path, image in (("simt", None), ("filter", None), ("shadow", "bf16"), ("shadow", "int8")):
        one = make(monkeypatch, p.rows, metric, "f32", image)
        two = make(monkeypatch, p.rows, metric, "f32", image, devices=(0, 0))
        a = search_once(one, path, p.queries, p.thr, int(counts.sum()))[0]
        b, dl, db = search_once(two, path, p.queries, p.thr, int(counts.sum()))
        rb = rp.row_bytes(path, d, "f32", image or "bf16")
        n0, n1 = n // 2, n - n // 2
        assert db == rp.scan_bytes(path, n0, rb, Q, 2) + rp.scan_bytes(path, n1, rb, Q, 1), (path, image)
        assert dl == rp.range_launches(path, Q, n0, counts, True) + rp.range_launches(path, Q, n1, [0] * Q, False), (path, image)
        same_bits(b, a, f"{path} {image}: two shards vs one")
        check_planted(b, p, metric, what=f"{path} {image}")
        one.release()
        two.release()


# ---- (b) re-scoring, compaction, sort and merge ----------------------------------------------------------------------
def survivor_counts(seed):
    """SURVIVORS shuffled, an empty query before each and after the last"""
    s = np.random.default_rng(seed).permutation(SURVIVORS)
    out = np.zeros(2 * len(s) + 1, dtype=np.int64)
    out[1::2] = s
    return out


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_rescore_compact_sort_merge(knn_lib, monkeypatch, metric):
    """one call whose queries sit on both sides of every re-scoring, compaction, run and merge edge, half of each long list
    one row copied (thousands of equal scores across the run and merge boundaries): every path against fp64, every launch
    the plan names counted, the paths bit for bit"""
    counts = survivor_counts(11)
    n, d, Q = int(counts.sum()) + 15_000, 64, len(counts)
    p = rp.planted(counts, d, metric, n, 12)
    assert p.gap > 3 * rp.MIN_GAP
    first = {}
    for dtype, path, image in PATHS:
        what = f"{metric} {dtype} {path} {image}"
        ix = make(monkeypatch, p.rows, metric, dtype, image)
        res, dl, db = search_once(ix, path, p.queries, p.thr, int(counts.sum()))
        assert passes(db, path, n, d, dtype, image, Q) == 2, what  # the longest list is past LIST0
        assert dl == rp.range_launches(path, Q, n, counts, True, d, dtype), what
        assert rp.merge_passes(int(counts.max())) == 3
        check_fp64(res, p, metric, dtype)
        check_planted(res, p, metric, what=what, dtype=dtype)
        ix.release()
        if dtype in first:
            same_bits(res, first[dtype], f"{what} vs the first {dtype} path")
        first.setdefault(dtype, res)


# ---- (c) the MAX_GRID_Y query blocks ----------------------------------------------------------------------------------
def block_counts(Q):
    """planted rows per query: distinct counts (0 and more than RUN among them) at the queries around the block boundary,
    a few elsewhere"""
    c = np.zeros(Q, dtype=np.int64)
    c[[0, 1000, 40_000]] = [7, rp.CP_THREADS + 1, 2]
    b = rp.MAX_GRID_Y
    for q, v in zip(range(b - 2, b + 3), [R + 5, 0, 1, 300, 2]):
        if q < Q:
            c[q] = v
    if Q > b + 60:
        c[b + 60] = 9
    return c


@pytest.fixture(scope="module")
def block_corpus(knn_lib):
    Qmax = max(BLOCK_QS)
    p = rp.planted(block_counts(Qmax), BLOCK_D, "cosine", BLOCK_N, 21, bounds=bounds_torch)
    assert p.gap > 2 * rp.MIN_GAP, p.gap
    return p


@pytest.mark.parametrize("Q", BLOCK_QS)
def test_query_blocks(block_corpus, monkeypatch, Q):
    """Q at and past MAX_GRID_Y: re-scoring, compaction and sort run once per query block (q_base > 0 in the second), the
    merge over every query at once; CUDA-core lists (count only) and the TF32 filter's (re-scored)"""
    p = block_corpus
    counts = block_counts(max(BLOCK_QS))[:Q]
    q, thr = p.queries[:Q], p.thr[:Q]
    out = {}
    for path in ("simt", "filter"):
        ix = make(monkeypatch, p.rows, "cosine")
        res, dl, db = search_once(ix, path, q, thr, int(counts.sum()))
        assert passes(db, path, BLOCK_N, BLOCK_D, "f32", None, Q) == 2, path
        assert dl == rp.range_launches(path, Q, BLOCK_N, counts, True, BLOCK_D), path
        check_planted(res, p, "cosine", what=f"Q={Q} {path}")
        out[path] = res
        ix.release()
    same_bits(out["filter"], out["simt"], f"Q={Q}: filter vs simt")


# ---- (d) the scan launch plan in the range modes ---------------------------------------------------------------------
def plan_rows(grid):
    return 40_000 if grid == rp.NUM_SMS_H100 else grid * rp.ROWS - 37


def plan_counts(Q, n):
    """0, 1 or 2 planted rows per query, alternating, at most about n / 2 rows in all"""
    step = 3 if n >= 4 * Q else 8
    c = np.zeros(Q, dtype=np.int64)
    c[1::step] = 1
    c[1::2 * step] = 2
    return c


@pytest.mark.parametrize("grid", PLAN_GRIDS)
def test_scan_launch_plan(knn_lib, monkeypatch, grid):
    """Q on both sides of every launch edge over shards of `grid` tiles, in the plain, tag-filtered and windowed range modes
    on both tensor paths: the launch count is plan_launches', and every query returns its own planted rows (each query has
    its own threshold; neighbouring queries alternate filters and windows, so a launch serving the wrong queries shows)"""
    from nornicdb_b200.knn import value_keys, window, window_admits
    n, d, metric = plan_rows(grid), 64, "cosine"
    assert rp.grid(n) == grid
    Qmax = max(PLAN_QS)
    counts = plan_counts(Qmax, n)
    p = rp.planted(counts, d, metric, n, 100 + grid)
    assert p.gap > 3 * rp.MIN_GAP
    rng = np.random.default_rng(grid)
    tags = (np.uint64(1) << rng.integers(0, 4, size=n).astype(np.uint64)).astype(np.uint64)
    vals = rng.integers(0, 1000, size=n)
    keys = value_keys(vals)
    filters = np.array([(0, 0, 0), (0, 0, 0b0101)] * (Qmax // 2 + 1), dtype=np.uint64)[:Qmax]
    fadm = [np.ones(n, dtype=bool), (tags & np.uint64(0b0101)) != 0]
    wins = np.array([window(gte=0, lte=499), window(gte=500, lte=999)] * (Qmax // 2 + 1), dtype=np.uint64)[:Qmax]
    wadm = [window_admits(keys, *[int(v) for v in wins[0]]), window_admits(keys, *[int(v) for v in wins[1]])]
    ix = make(monkeypatch, p.rows, metric)
    ix.set_row_tags(tags)
    ix.set_row_values(keys)
    for Q in PLAN_QS:
        c = counts[:Q]
        for mode, kw, adm in (("plain", {}, None), ("tags", {"filters": filters[:Q]}, fadm),
                              ("window", {"windows": wins[:Q]}, wadm)):
            got = {}
            for path in rp.TENSOR_PATHS:
                what = f"grid {grid} Q={Q} {mode} {path}"
                res, dl, db = search_once(ix, path, p.queries[:Q], p.thr[:Q], int(c.sum()), **kw)
                assert passes(db, path, n, d, "f32", None, Q) == 1, what
                assert dl == rp.range_launches(path, Q, n, c if adm is None else
                                               np.array([len(p.expected(i, adm[i % 2])) for i in range(Q)]), False, d), what
                check_planted(res, p, metric, adm, what)
                got[path] = res
            same_bits(got["shadow"], got["filter"], f"grid {grid} Q={Q} {mode}: shadow vs filter")
    ix.release()


def test_saturated_buffers(knn_lib, monkeypatch):
    """every row reaches every threshold: each CTA's per-query buffer flushes on every tile of every query group (Q > 384
    over 8 tiles: 4 groups), every list is past LIST0 on a fresh index"""
    n, d, Q = SATURATE_N, 64, SATURATE_Q
    assert rp.grid(n) == 8 and {l[3] for l in rp.tensor_launches(Q, 8)} == {4, 2}
    rng = np.random.default_rng(5)
    rows = rng.standard_normal((n, d)).astype(np.float32)
    q = rng.standard_normal((Q, d)).astype(np.float32)
    thr = np.full(Q, -2.0, dtype=np.float32)
    keys, scale = fp64_keys(rows, q, "cosine")
    out = {}
    for path in ("shadow", "filter", "simt"):
        ix = make(monkeypatch, rows, "cosine")
        res, dl, db = search_once(ix, path, q, thr, n * Q)
        assert passes(db, path, n, d, "f32", None, Q) == 2, path
        assert dl == rp.range_launches(path, Q, n, [n] * Q, True, d), path
        assert all(len(i) == n for i, _ in res)
        assert check_range(res, keys, scale, thr, "cosine") == 0
        out[path] = res
        ix.release()
    same_bits(out["shadow"], out["filter"], "shadow vs filter")
    same_bits(out["shadow"], out["simt"], "shadow vs simt")


@pytest.mark.parametrize("d", [64, 66])
def test_simt_groups(knn_lib, monkeypatch, d):
    """the CUDA-core split into groups of 8 / 4 / 2 / 1 (vector loads, d = 64) and 4 / 1 (scalar loads, d = 66)"""
    n, metric = 5000, "euclidean"
    Qmax = max(SIMT_QS)
    counts = np.arange(Qmax, dtype=np.int64) % 3 + (np.arange(Qmax) % 5 == 0) * 40
    p = rp.planted(counts, d, metric, n, 300 + d)
    assert p.gap > 3 * rp.MIN_GAP
    ix = make(monkeypatch, p.rows, metric)
    for Q in SIMT_QS:
        c = counts[:Q]
        res, dl, db = search_once(ix, "simt", p.queries[:Q], p.thr[:Q], int(c.sum()))
        assert passes(db, "simt", n, d, "f32", None, Q) == 1
        assert dl == rp.range_launches("simt", Q, n, c, False, d), (d, Q, rp.simt_range_groups(Q, rp.simt_vec(d), d))
        check_planted(res, p, metric, what=f"d={d} Q={Q}")
    ix.release()


# ---- (e) the self-join and the incident pairs ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pairs_corpus():
    """PAIRS_N rows, d = 64; PAIRS_CLUSTER of them (PAIRS_LOW the lowest) near-copies of one direction, so that every pair of
    the cluster reaches the threshold and no other pair comes near it (asserted in fp64)"""
    n, d = PAIRS_N, 64
    rng = np.random.default_rng(31)
    g = rng.standard_normal((n, d))
    x = g / np.linalg.norm(g, axis=1, keepdims=True) * rng.uniform(0.5, 1.0, size=(n, 1))
    members = np.r_[PAIRS_LOW, PAIRS_LOW + 1 + rng.permutation(n - PAIRS_LOW - 1)[:PAIRS_CLUSTER - 1]]
    h = rng.standard_normal(d)
    h /= np.linalg.norm(h)
    u = rng.standard_normal((PAIRS_CLUSTER, d))
    x[members] = h + rp.EPS * u / np.linalg.norm(u, axis=1, keepdims=True)
    rows = x.astype(np.float32)
    inc = np.zeros(n, dtype=bool)
    inc[members] = True
    k, _ = rp.keys64(rows, rows, "cosine")
    both = inc[:, None] & inc[None, :]
    np.fill_diagonal(both, False)
    other = ~(inc[:, None] & inc[None, :])
    np.fill_diagonal(other, False)
    lo, hi = k[both].min(), k[other].max()
    t = np.float32((lo + hi) / 2)
    assert lo - t > 3 * rp.MIN_GAP and t - hi > 3 * rp.MIN_GAP, (lo, hi)
    return rows, t, np.sort(members)


def pairs_once(ix, t, first, n_rows, cap):
    """one nk_search_pairs call with room for `cap` pairs -> (offsets, idx, score), bytes_scanned delta"""
    from nornicdb_b200.knn import _check
    off = np.zeros(n_rows + 1, dtype=np.uint64)
    idx = np.empty(cap, dtype=np.uint32)
    sc = np.empty(cap, dtype=np.float32)
    total = C.c_uint64(0)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    before = ix.stats()["bytes_scanned"]
    _check(ix.lib.nk_search_pairs(ix.ptr, first, n_rows, float(t), None, cap, vp(off), vp(idx), vp(sc), C.byref(total)), "nk_search_pairs")
    assert total.value <= cap
    return (off, idx[:total.value].copy(), sc[:total.value].copy()), ix.stats()["bytes_scanned"] - before


def stripe_bytes(path, n, first, d):
    """bytes_scanned of one pass of every 1024-row block of the stripe [first, n) (one shard: each block scans its window
    from its first row rounded down to the scan tile) -> (all blocks, the first block)"""
    out = []
    for b in range(0, n - first, rp.SEARCH_ROWS_BLOCK):
        frm = (first + b) // rp.SCAN_TILE_ROWS * rp.SCAN_TILE_ROWS
        out.append(rp.scan_bytes(path, n - frm, rp.row_bytes(path, d), min(rp.SEARCH_ROWS_BLOCK, n - first - b), 1))
    return sum(out), out[0]


@pytest.mark.parametrize("path", ["shadow", "filter", "simt"])
def test_pairs_stripes_at_the_edges(pairs_corpus, monkeypatch, path):
    """stripes whose 1024-row blocks scan windows of odd, 2 mod 4 and 0 mod 4 tiles, down to 1; the cluster's lowest row
    pairs with more than RUN rows, and the first block on a fresh index has lists longer than LIST0 (it scans twice): each
    stripe equals the range-search contract, the planted pairs, and a slice of the whole-index join"""
    rows, t, members = pairs_corpus
    n, d = rows.shape
    cap = PAIRS_CLUSTER * PAIRS_CLUSTER // 2
    ix = make(monkeypatch, rows, "cosine")
    ix.set_path(path)
    stripes = []
    for i, s in enumerate(PAIRS_STARTS):
        st, db = pairs_once(ix, t, s, n - s, cap)
        assert ix.last_path() == path
        if i == 0:  # the fresh index: the first block's lists outgrow LIST0
            once, first_block = stripe_bytes(path, n, s, d)
            assert db >= once + first_block, (db, once, first_block)
        stripes.append(st)
    whole = pairs_once(ix, t, 0, n, cap)[0]
    assert_same(whole, by_range(ix, t, 0, n), f"{path}: whole join vs range")
    o = whole[0].astype(np.int64)
    inc = np.zeros(n, dtype=bool)
    inc[members] = True
    for i in range(n):
        want = members[members > i] if inc[i] else np.empty(0, np.int64)
        assert np.array_equal(np.sort(whole[1][o[i]:o[i + 1]].astype(np.int64)), want), f"{path}: row {i}"
    assert o[PAIRS_LOW + 1] - o[PAIRS_LOW] == PAIRS_CLUSTER - 1 > rp.RUN
    for s, st in zip(PAIRS_STARTS, stripes):
        want = (whole[0][s:] - whole[0][s], whole[1][o[s]:], whole[2][o[s]:])
        assert_same(st, want, f"{path}: stripe from {s}")
    ix.release()


def test_pairs_paths_agree_and_incident_rows(pairs_corpus, monkeypatch):
    """the join bit for bit on every path; a listed row that pairs with RUN + 1 rows, and the cluster's lowest row, through
    search_pairs_rows against the whole join regrouped"""
    rows, t, members = pairs_corpus
    got = {}
    for path in ("shadow", "filter", "simt"):
        ix = make(monkeypatch, rows, "cosine")
        ix.set_path(path)
        got[path] = ix.search_pairs(t)
        if path != "simt":
            mid = int(members[len(members) // 2])
            for listed in ([mid], [mid, PAIRS_LOW, 0, len(rows) - 1]):
                res = check_incident(ix, t, np.array(listed, np.uint32), "cosine", f"{path}: {listed}")
                o = res[0].astype(np.int64)
                if len(listed) == 1:
                    assert o[1] - o[0] == PAIRS_CLUSTER - 1
                else:  # both ends listed: the pair goes under the lower row, PAIRS_LOW
                    assert o[1] - o[0] == PAIRS_CLUSTER - 2 and o[2] - o[1] == PAIRS_CLUSTER - 1
        ix.release()
    assert_same(got["filter"], got["shadow"], "filter vs shadow")
    assert_same(got["simt"], got["shadow"], "simt vs shadow")
