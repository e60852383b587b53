"""GPU tests of search by stored row (nk_search_rows): the k nearest OTHER rows of stored rows, up to the whole k-NN graph.

The contract: nk_search_rows(ids, k) equals nk_search(the rows read back and widened to fp32, k+1) with each query's own row
dropped (or the last slot, when its row is not in the list), bit for bit, on every forced path, metric and corpus dtype and
for the same blocks of 1024 queries.  Full graphs and a 1M-row clustered corpus are checked against an fp64 brute force that
excludes self, with the parity rule of tests/parity.py."""
import numpy as np
import pytest

from parity import check_parity
from test_search_rows_cpu import PAD, drop_self

pytestmark = pytest.mark.gpu

BLOCK = 1024


def paths_for(dtype, metric):
    if dtype != "f32":
        return ("simt", "shadow")
    return ("simt", "filter", "shadow") + (() if metric == "euclidean" else ("tensor",))


def make_index(rows, metric, dtype="f32", devices=(0,)):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex(rows.shape[1], metric=metric, dtype=dtype, devices=devices)
    ix.upload_from_f32(rows)
    return ix


def stored_f32(ix):
    """Every row as stored, widened exactly to fp32."""
    from nornicdb_b200.knn import from_bf16_bits
    a = ix.read_rows(0, len(ix))
    return from_bf16_bits(a) if ix.dtype == 2 else a.astype(np.float32)


def by_search(ix, ids, k):
    """nk_search(stored rows, k+1) per block of 1024 queries, with the self rule."""
    x = stored_f32(ix)
    outs = [drop_self(*ix.search(x[ids[b:b + BLOCK]], k + 1), ids[b:b + BLOCK], k) for b in range(0, len(ids), BLOCK)]
    return np.concatenate([o[0] for o in outs]), np.concatenate([o[1] for o in outs])


def assert_same(a, b, what=""):
    (ai, as_), (bi, bs) = a, b
    assert ai.shape == bi.shape, (what, ai.shape, bi.shape)
    assert np.array_equal(ai, bi), what
    assert np.array_equal(as_.view(np.uint32), bs.view(np.uint32)), what


def others64_torch(rows_of_slice, n, ids, queries, k, metric, slice_rows, q_chunk=4096):
    """fp64 brute force on the GPU (torch) of the k best rows other than each query's own, (score desc, row asc) /
    (distance asc, row asc).  rows_of_slice(lo, cnt) -> float32 cuda tensor [cnt, d].  -> (idx int64 [Q, k], score [Q, k])."""
    import torch
    Q = len(ids)
    out_i, out_s = np.empty((Q, k), np.int64), np.empty((Q, k), np.float64)
    for q0 in range(0, Q, q_chunk):
        q64 = torch.from_numpy(np.asarray(queries[q0:q0 + q_chunk], np.float64)).cuda()
        me = torch.from_numpy(np.asarray(ids[q0:q0 + q_chunk], np.int64)).cuda()
        qn = q64.norm(dim=1)
        best_s = best_i = None
        for lo in range(0, n, slice_rows):
            cnt = min(slice_rows, n - lo)
            x = rows_of_slice(lo, cnt).double()
            s = q64 @ x.T  # [q, cnt]
            if metric == "cosine":
                den = qn[:, None] * x.norm(dim=1)[None, :]
                s = torch.where(den > 0, s / den, torch.zeros_like(s))
            elif metric == "euclidean":
                s = -((q64 * q64).sum(1)[:, None] + (x * x).sum(1)[None, :] - 2.0 * s)
            loc = me - lo
            inside = ((loc >= 0) & (loc < cnt)).nonzero().squeeze(1)
            s[inside, loc[inside]] = -float("inf")  # the query's own row
            v, i = torch.topk(s, min(k + 8, cnt), dim=1)
            i = i + lo
            if best_s is not None:
                v, i = torch.cat([best_s, v], dim=1), torch.cat([best_i, i], dim=1)
                keep = torch.topk(v, min(k + 8, v.shape[1]), dim=1).indices
                v, i = torch.gather(v, 1, keep), torch.gather(i, 1, keep)
            best_s, best_i = v, i
            del x, s
        bs, bi = best_s.cpu().numpy(), best_i.cpu().numpy()
        o = np.lexsort((bi, -bs), axis=1)[:, :k]
        bs, bi = np.take_along_axis(bs, o, 1), np.take_along_axis(bi, o, 1)
        out_i[q0:q0 + len(bi)] = bi
        out_s[q0:q0 + len(bi)] = np.sqrt(np.maximum(-bs, 0.0)) if metric == "euclidean" else bs
    return out_i, out_s


@pytest.mark.parametrize("n,d", [(3000, 64), (2000, 1024)])
@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
@pytest.mark.parametrize("dtype", ["f32", "f16", "bf16"])
def test_equals_search_k_plus_one_with_self_dropped(knn_lib, dtype, metric, n, d):
    rng = np.random.default_rng(n + d)
    rows = rng.standard_normal((n, d)).astype(np.float32)
    rows[100:104] = rows[50]  # exact duplicates around query rows 50 and 101
    ix = make_index(rows, metric, dtype)
    ids = np.concatenate([rng.integers(0, n, 37), [50, 101, 103, 50]]).astype(np.int64)
    k = 10
    for path in paths_for(dtype, metric):
        ix.set_path(path)
        got = ix.search_rows(ids, k)
        assert ix.last_path() == path
        ref = by_search(ix, ids, k)
        assert ix.last_path() == path
        assert_same(got, ref, path)
        assert not (got[0] == ids[:, None]).any()
        assert (got[0] != PAD).all()
    ix.release()


@pytest.mark.parametrize("n,d,metric", [(50_000, 256, "cosine"), (8192, 1024, "dot")])
def test_full_graph_against_fp64(knn_lib, n, d, metric):
    import torch
    rng = np.random.default_rng(5)
    rows = rng.standard_normal((n, d)).astype(np.float32)
    ix = make_index(rows, metric)
    k = 10
    ids = np.arange(n)
    gi, gs = ix.search_rows(ids, k)
    path = ix.last_path()
    ix.release()
    dev = torch.from_numpy(rows).cuda()
    oi, os_ = others64_torch(lambda lo, cnt: dev[lo:lo + cnt], n, ids, rows, k, metric, slice_rows=n)
    swaps = check_parity(rows, rows, k, metric, gi, gs, oi, os_)
    print(f"full graph n={n} d={d} {metric}: path {path}, boundary swaps {swaps}")
    assert swaps <= 8


def test_clustered_1m_rows_4096_queries_fp64(knn_lib):
    """The near-tie and near-duplicate case: 1000 centres, sigma 0.1, N=1M d=1024, 4096 stored rows as queries."""
    import torch
    from nornicdb_b200.knn import KnnIndex
    n, d, Q, k = 1_000_000, 1024, 4096, 10
    ix = KnnIndex(d, metric="cosine")
    ix.fill_clustered(n, 42, n_centres=1000, sigma=0.1)
    host = np.concatenate([ix.read_rows(lo, 100_000) for lo in range(0, n, 100_000)])
    ids = np.random.default_rng(9).choice(n, Q, replace=False)
    gi, gs = ix.search_rows(ids, k)
    path, flags, counters = ix.last_path(), ix.debug_flags(), ix.debug_counters()
    ix.release()
    print(f"clustered 1M: path {path}, retry counters {counters}")
    assert flags[0] == 0
    oi, os_ = others64_torch(lambda lo, cnt: torch.from_numpy(host[lo:lo + cnt]).cuda(), n, ids, host[ids], k, "cosine",
                             slice_rows=62_500)
    check_parity(host, host[ids], k, "cosine", gi, gs, oi, os_, swap_eps=5e-6)


def test_duplicates_mask_floor_and_small_k(knn_lib):
    rng = np.random.default_rng(21)
    rows = rng.standard_normal((500, 64)).astype(np.float32)
    rows[[10, 20, 30]] = rows[40]
    ix = make_index(rows, "cosine")
    gi, _ = ix.search_rows([40, 10, 20, 30], 2)
    assert gi.tolist() == [[10, 20], [20, 30], [10, 30], [10, 20]]  # equal copies rank by row; never the query itself
    gi, _ = ix.search_rows([40], 3)
    assert gi.tolist() == [[10, 20, 30]]
    keep = np.ones(500, bool)
    keep[[10, 40, 7]] = False
    ix.set_row_mask(keep)
    ids = np.array([40, 10, 20, 7, 99, 499])                  # masked-out rows may still be queries
    got = ix.search_rows(ids, 5)
    assert_same(got, by_search(ix, ids, 5), "row mask")
    assert not np.isin(got[0], [10, 40, 7]).any() and got[0][0].tolist()[:2] == [20, 30]
    ix.set_min_score(0.35)
    got = ix.search_rows(ids, 5)
    assert_same(got, by_search(ix, ids, 5), "row mask + floor")
    assert (got[0] == PAD).any() and (got[1][got[0] != PAD] >= 0.35).all()
    ix.set_min_score(None)
    ix.set_row_mask(None)
    ix.release()
    small = make_index(rows[:20], "euclidean")
    gi, gs = small.search_rows(np.arange(20), 50)             # k >= N: N columns, the last one padding
    assert gi.shape == (20, 20) and (gi[:, -1] == PAD).all() and (gs[:, -1] == 0).all()
    for q in range(20):
        assert sorted(gi[q, :-1].tolist()) == [r for r in range(20) if r != q]
    small.release()


def test_trivial_calls_and_errors(knn_lib):
    from nornicdb_b200.knn import KnnError, KnnIndex
    rows = np.random.default_rng(22).standard_normal((100, 32)).astype(np.float32)
    ix = make_index(rows, "dot")
    assert ix.search_rows([], 5)[0].shape == (0, 0)
    assert ix.search_rows([3, 4], 0)[0].shape == (2, 0)
    with pytest.raises(KnnError, match="out of range"):
        ix.search_rows([3, 100], 5)
    with pytest.raises(KnnError, match="NK_MAX_K_TOTAL"):
        ix.search_rows([3], 65536)
    n = ix.lib.nk_search_rows(ix.ptr, None, 1, 5, None, None)
    assert n == -1 and "null" in ix.lib.nk_last_error().decode()
    empty = KnnIndex(32, metric="cosine")
    assert empty.search_rows([0, 1], 5)[0].shape == (2, 0)
    empty.release()
    ix.release()


def test_many_blocks_equal_the_same_blocks_through_search(knn_lib):
    rng = np.random.default_rng(23)
    rows = rng.standard_normal((20_000, 128)).astype(np.float32)
    ix = make_index(rows, "cosine")
    ids = rng.integers(0, 20_000, 2500)
    got = ix.search_rows(ids, 16)
    path = ix.last_path()
    assert_same(got, by_search(ix, ids, 16), "Q=2500")
    assert ix.last_path() == path == "shadow"
    ix.release()


def test_results_follow_append_update_and_remove(knn_lib):
    rng = np.random.default_rng(24)
    rows = rng.standard_normal((300, 64)).astype(np.float32)
    ix = make_index(rows, "cosine")
    ix.append(rng.standard_normal((5, 64)).astype(np.float32))
    ix.update_row(7, rows[200] * 2.0)                          # row 7 now points where row 200 does
    ids = np.arange(305)
    got = ix.search_rows(ids, 4)
    assert_same(got, by_search(ix, ids, 4), "after append + update_row")
    assert got[0][7, 0] == 200 and got[0][200, 0] == 7
    assert (got[0][300:] < 305).all()
    moved = ix.read_rows(304, 1)[0]
    ix.remove_swap(3)                                          # row 304 moves to 3
    assert np.array_equal(ix.read_rows(3, 1)[0], moved)
    ids = np.arange(304)
    after = ix.search_rows(ids, 4)
    assert_same(after, by_search(ix, ids, 4), "after remove_swap")
    assert (after[0] < 304).all() and after[0][7, 0] == 200
    ix.release()


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_two_shards_bit_identical_to_one(knn_lib, metric):
    rng = np.random.default_rng(25)
    rows = rng.standard_normal((6000, 128)).astype(np.float32)
    one, two = make_index(rows, metric), make_index(rows, metric, devices=(0, 0))
    ids = rng.integers(0, 6000, 2500)                          # every block holds rows of both shards
    for path in ("shadow", "simt"):
        one.set_path(path)
        two.set_path(path)
        assert_same(one.search_rows(ids, 10), two.search_rows(ids, 10), path)
    two.set_path("auto")
    assert_same(two.search_rows(ids, 10), by_search(two, ids, 10), "two shards vs nk_search")
    one.release()
    two.release()


def test_only_ids_cross_pcie_on_one_device(knn_lib):
    rows = np.random.default_rng(26).standard_normal((4000, 256)).astype(np.float32)
    ix = make_index(rows, "cosine")
    before = ix.stats()
    ix.search_rows(np.arange(2100), 10)
    after = ix.stats()
    assert after["bytes_h2d"] - before["bytes_h2d"] == 4 * 2100
    assert after["searches"] - before["searches"] == 1 and after["queries"] - before["queries"] == 2100
    ix.release()


def test_search_similar_python_mirror(knn_lib):
    from nornicdb_b200.embedding_index import EmbeddingIndex
    ei = EmbeddingIndex(4)
    ei.AddBatch(["a", "b", "c", "d"], [[1, 0, 0, 0], [0.9, 0.1, 0, 0], [0, 1, 0, 0], [1, 0, 0, 0]])
    res = ei.SearchSimilar(["a", "missing", "c"], 2)
    assert [[r.ID for r in lst] for lst in res] == [["d", "b"], [], ["b", "a"]]
    assert [r.ID for r in ei.SearchSimilar(["b"], 10)[0]] == ["a", "d", "c"]
    ei.Release()
