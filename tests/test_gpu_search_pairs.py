"""GPU tests of the similarity self-join (nk_search_pairs): every pair of stored rows within a threshold, each pair once.

The contract: nk_search_pairs equals nk_search_range(the stripe's rows read back and widened to fp32, the threshold, the filter
for every query) with each list cut to the rows above its own query row and emptied for inadmissible left rows, bit for bit,
on every forced path, metric and corpus dtype.  The corpora have a few thousand rows, so the whole-index join runs several
1024-row blocks, and a stripe starting at row 700 puts the scan window at offsets that are not multiples of 256.  The pair set
is also checked against an fp64 brute force over all pairs: a pair may differ only where its fp64 score is within fp32
rounding of the threshold (the band of tests/test_gpu_range.py)."""
import numpy as np
import pytest

from test_gpu_range import BAND, fp64_keys, key_threshold, rounded
from test_gpu_search_rows import stored_f32

pytestmark = pytest.mark.gpu

PATHS = {"f32": ("auto", "shadow", "filter", "simt"), "f16": ("auto", "shadow", "simt"), "bf16": ("auto", "shadow", "simt")}


def make_index(rows, metric, dtype="f32", devices=(0,)):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex(rows.shape[1], metric=metric, dtype=dtype, devices=devices)
    ix.upload_from_f32(rows)
    return ix


def by_range(ix, t, first, n_rows, filt=None, left_adm=None, chunk=4096):
    """The contract: range search of the stripe's stored rows, each list cut to rows above its query row, emptied for
    inadmissible left rows (left_adm: bool per index row, None = all admissible).  -> CSR (offsets, idx, score)."""
    x = stored_f32(ix)[first:first + n_rows]
    off, idx, sc = [0], [], []
    for c in range(0, n_rows, chunk):
        q = x[c:c + chunk]
        res = ix.search_range(q, t, None if filt is None else np.tile(np.asarray(filt, np.uint64), (len(q), 1)))
        for qi, (i, s) in enumerate(res):
            row = first + c + qi
            keep = i.astype(np.int64) > row
            if left_adm is not None and not left_adm[row]:
                keep[:] = False
            idx.append(i[keep])
            sc.append(s[keep])
            off.append(off[-1] + int(keep.sum()))
    cat = lambda a, dt: np.concatenate(a).astype(dt) if a else np.empty(0, dt)
    return np.asarray(off, np.uint64), cat(idx, np.uint32), cat(sc, np.float32)


def assert_same(a, b, what=""):
    assert np.array_equal(a[0], b[0]), f"{what}: offsets"
    assert np.array_equal(a[1], b[1]), f"{what}: rows"
    assert np.array_equal(a[2].view(np.uint32), b[2].view(np.uint32)), f"{what}: scores"


def as_matrix(res, n, first=0):
    off, idx, _ = res
    got = np.zeros((n, n), dtype=bool)
    for r in range(len(off) - 1):
        got[first + r, idx[int(off[r]):int(off[r + 1])].astype(np.int64)] = True
    return got


def check_fp64(res, rows_f32, t, metric, adm=None):
    """The pair set against fp64 over every pair j > i of admissible rows, outside the band.  Returns pairs in the band."""
    n = len(rows_f32)
    keys, scale = fp64_keys(rows_f32, rows_f32, metric)
    tk = key_threshold(float(t), metric)
    upper = np.triu(np.ones((n, n), dtype=bool), 1)
    ok = upper & np.isfinite(keys) & (keys >= tk)
    if adm is not None:
        ok &= adm[:, None] & adm[None, :]
    in_band = np.isfinite(keys) & (np.abs(keys - tk) <= BAND * scale)
    got = as_matrix(res, n)
    assert not (got & ~upper).any(), "a pair under its higher row, or a row paired with itself"
    assert not (ok & ~got & ~in_band).any(), f"pairs meeting the threshold not returned: {np.argwhere(ok & ~got & ~in_band)[:4]}"
    assert not (got & ~ok & ~in_band).any(), f"pairs below the threshold returned: {np.argwhere(got & ~ok & ~in_band)[:4]}"
    return int((in_band & (got != ok)).sum())


def threshold_for(rows_f32, metric, per_row):
    """An API threshold that gives about per_row pairs per row (fp64 quantile of the off-diagonal keys)."""
    keys, _ = fp64_keys(rows_f32, rows_f32, metric)
    n = len(rows_f32)
    k = keys[~np.eye(n, dtype=bool)]
    tk = np.quantile(k[np.isfinite(k)], 1.0 - 2.0 * per_row / n)
    return np.float32(np.sqrt(-tk) if metric == "euclidean" else tk)


@pytest.mark.parametrize("dtype", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_contract_every_path_and_fp64(knn_lib, oracle_mod, metric, dtype):
    n, d = 3037, 64
    rows = oracle_mod.fill_uniform(n, d, 101)
    r = rounded(rows, dtype)
    t = threshold_for(r, metric, 12)
    ix = make_index(rows, metric, dtype)
    first = None
    for path in PATHS[dtype]:
        ix.set_path(path)
        whole = ix.search_pairs(t)
        if path != "auto":
            assert ix.last_path() == path
        assert_same(whole, by_range(ix, t, 0, n), f"{path} whole")
        stripe = ix.search_pairs(t, 700, 1500)
        assert_same(stripe, by_range(ix, t, 700, 1500), f"{path} stripe")
        if first is None:
            first = whole
            band = check_fp64(whole, r, t, metric)
            print(f"{metric} {dtype}: {int(whole[0][-1])} pairs, {band} inside the band")
        assert_same(whole, first, f"{path} vs {PATHS[dtype][0]}")
        o = whole[0].astype(np.int64)
        assert np.array_equal(stripe[1], whole[1][o[700]:o[2200]]), "a stripe is a slice of the whole-index result"
    ix.release()


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_duplicates_at_the_threshold_nan_inf_and_zero_rows(knn_lib, oracle_mod, metric):
    """Exact duplicate rows whose pair score is the threshold exactly; a NaN and an Inf component; a zero row."""
    n, d = 2600, 64
    rows = oracle_mod.fill_uniform(n, d, 102)
    dups = [5, 300, 1500, 2599]
    rows[dups] = rows[5]
    rows[800, 3] = np.nan
    rows[900, 7] = np.inf
    rows[1000] = 0.0
    ix = make_index(rows, metric)
    t = threshold_for(np.delete(rows, [800, 900], axis=0), metric, 8)
    for path in ("auto", "shadow", "filter", "simt"):
        ix.set_path(path)
        assert_same(ix.search_pairs(t), by_range(ix, t, 0, n), path)
    ix.set_path("auto")
    off, idx, sc = ix.search_pairs(t)
    o = off.astype(np.int64)
    t_dup = sc[o[5]:o[6]][idx[o[5]:o[6]] == 300][0]  # the duplicates' own score (euclidean: their distance)
    res = ix.search_pairs(t_dup)
    assert_same(res, by_range(ix, t_dup, 0, n), "threshold = the duplicates' score")
    got = as_matrix(res, n)
    for a in range(len(dups)):
        for b in range(a + 1, len(dups)):
            i, j = dups[a], dups[b]
            assert got[i, j] and not got[j, i], (i, j)
            k = res[1][int(res[0][i]):int(res[0][i + 1])].tolist().index(j)
            assert res[2][int(res[0][i]) + k].view(np.uint32) == t_dup.view(np.uint32)
    assert not got[:, 900].any() and not got[900].any(), "a row with a NaN score (Inf component) was paired"
    assert not np.isnan(sc).any()
    if metric == "cosine":  # the zero row scores 0 against every row: t = -0.5 pairs it with every finite row above it
        z = ix.search_pairs(-0.5, 1000, 1)
        assert_same(z, by_range(ix, -0.5, 1000, 1), "zero row")
        assert np.all(z[2] == 0.0) and int(z[0][-1]) >= n - 1001 - 1
    ix.release()


def test_mask_floor_filter_and_stripes(knn_lib, oracle_mod):
    from nornicdb_b200.knn import admits, synthetic_tags
    n, d = 3100, 64
    rows = oracle_mod.fill_uniform(n, d, 103)
    rows[[7, 1200]] = rows[1900]            # duplicates of a row above them; 7 is masked out, so it has no pairs at all
    tags = synthetic_tags(n, 9) & np.uint64(0xF)
    tags[[1200, 1900]] = 1                  # both pass the filter below
    keep = np.ones(n, dtype=bool)
    keep[::53] = False
    keep[7] = False
    flt = (0, 2, 0)
    adm = keep & admits(tags, *flt)
    t = threshold_for(rows, "cosine", 20)
    floor = np.float32(t + 0.02)
    ix = make_index(rows, "cosine")
    ix.set_row_tags(tags)
    ix.set_row_mask(keep)
    ix.set_min_score(float(floor))
    for path in PATHS["f32"]:
        ix.set_path(path)
        res = ix.search_pairs(t, filter=flt)
        assert_same(res, by_range(ix, t, 0, n, flt, adm), path)
        o = res[0].astype(np.int64)
        for r in np.flatnonzero(~adm):
            assert o[r] == o[r + 1], f"{path}: inadmissible left row {r} has pairs"
        assert adm[res[1].astype(np.int64)].all(), f"{path}: an inadmissible row was paired"
        assert np.all(res[2] >= floor)
    band = check_fp64(res, rows, floor, "cosine", adm)
    assert as_matrix(res, n)[1200, 1900]
    # stripes whose union is the whole result
    parts = [ix.search_pairs(t, a, b - a, filter=flt) for a, b in ((0, 1000), (1000, 1037), (1037, 2090), (2090, n))]
    assert np.array_equal(np.concatenate([p[1] for p in parts]), res[1])
    assert np.array_equal(np.concatenate([p[2] for p in parts]).view(np.uint32), res[2].view(np.uint32))
    # the mask alone (no filter): masked-out left rows still get empty lists
    ix.set_min_score(None)
    assert_same(ix.search_pairs(t), by_range(ix, t, 0, n, None, keep), "mask only")
    print(f"mask + floor + filter: {len(res[1])} pairs, {band} inside the band")
    ix.release()


def test_two_shards_and_a_straddling_stripe(knn_lib, oracle_mod):
    n, d = 4100, 64
    rows = oracle_mod.fill_uniform(n, d, 104)
    t = threshold_for(rows, "dot", 10)
    one = make_index(rows, "dot")
    two = make_index(rows, "dot", devices=(0, 0))
    for path in ("shadow", "filter", "simt"):
        one.set_path(path)
        two.set_path(path)
        a, b = one.search_pairs(t), two.search_pairs(t)
        assert_same(a, b, f"{path}: two shards")
        assert_same(b, by_range(two, t, 0, n), f"{path}: two shards vs range")
        s = two.search_pairs(t, n // 2 - 300, 600)  # straddles the shard boundary at n // 2
        assert_same(s, by_range(two, t, n // 2 - 300, 600), f"{path}: straddling stripe")
        assert_same(s, one.search_pairs(t, n // 2 - 300, 600), f"{path}: straddling stripe vs one shard")
    one.release()
    two.release()


def test_rows_changed_just_before_the_call_and_3xtf32_refused(knn_lib, oracle_mod):
    from nornicdb_b200.knn import KnnError
    n, d = 2200, 64
    rows = oracle_mod.fill_uniform(n, d, 105)
    t = threshold_for(rows, "cosine", 10)
    ix = make_index(rows, "cosine")
    ix.search_pairs(t)
    ix.update_row(10, rows[2000])            # row 10 becomes a duplicate of row 2000
    ix.remove_swap(500)                      # the last row moves into row 500
    assert len(ix) == n - 1
    res = ix.search_pairs(t)
    assert_same(res, by_range(ix, t, 0, n - 1), "after update_row / remove_swap")
    assert as_matrix(res, n - 1)[10, 2000]
    ix.set_path("tensor")
    with pytest.raises(KnnError, match="3xTF32"):
        ix.search_pairs(t)
    ix.release()


def test_200k_whole_index_against_the_range_contract(knn_lib):
    from nornicdb_b200.knn import KnnIndex
    n, d = 200_000, 128
    ix = KnnIndex(d, metric="cosine")
    ix.fill_uniform(n, 77)
    x = stored_f32(ix)
    _, s = ix.search(x[:256], 21)              # ~10 pairs per row: the 20th other row's score
    t = np.float32(np.median(s[:, 20]))
    before = ix.debug_counters()
    res = ix.search_pairs(t)
    after = ix.debug_counters()
    total = int(res[0][-1])
    assert 2 * n < total < 40 * n, total
    assert_same(res, by_range(ix, t, 0, n, chunk=16384), "200k")
    assert after["bf16_stage_retries"] == before["bf16_stage_retries"] == 0
    assert after["exact_stage_runs"] == before["exact_stage_runs"] == 0
    print(f"200k: {total} pairs at t = {t}, path {ix.last_path()}")
    ix.release()
