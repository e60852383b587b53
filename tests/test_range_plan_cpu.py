"""The range pipeline's plan without a GPU: the constants tests/range_plan.py reads from the sources, the rule changing across
every edge it names, the GPU tests covering every edge on both sides, the planted corpora's exact fp64 counts and gaps, and
range_merge_kernel's placement formula restated in numpy."""
import numpy as np
import pytest

import range_plan as rp
import test_gpu_range_plan as g


def test_constants_parse():
    """each constant is found once; the sizes may move, the relations the pipeline relies on may not"""
    for v in (rp.LIST0, rp.RS_ENTRIES, rp.CP_THREADS, rp.RUN, rp.ROWS, rp.QT_BIG, rp.SEARCH_ROWS_BLOCK):
        assert v > 0 and v & (v - 1) == 0, v
    assert rp.MAX_GRID_Y == 65535  # CUDA's grid.y limit
    assert rp.CP_THREADS % 32 == 0 and rp.RUN >= rp.CP_THREADS
    assert rp.SCAN_TILE_ROWS == rp.ROWS  # the self-join's windows start on scan tiles


def test_tensor_launches_cover_every_query_once():
    for grid in rp.edges()["tensor grid (tiles)"]:
        for Q in range(1, 1400):
            ls = rp.tensor_launches(Q, grid)
            assert [l[1] for l in ls] == list(np.cumsum([0] + [l[2] for l in ls[:-1]])), (Q, grid)
            assert sum(l[2] for l in ls) == Q
            for qt, q0, nq, groups in ls:
                assert nq <= qt * groups and (qt == 64) == (Q - q0 <= 64)
                assert groups == 1 or grid % groups == 0


@pytest.mark.parametrize("edge", ["tensor columns (Q)", "2 query groups (Q)", "4 query groups (Q)", "one 4-group launch (Q)",
                                  "4-group launch and a tail (Q)"])
def test_tensor_split_changes_across_each_query_edge(edge):
    a, b = rp.edges()[edge]
    changed = [grid for grid in rp.edges()["tensor grid (tiles)"] if rp.tensor_launches(a, grid) != rp.tensor_launches(b, grid)]
    assert changed, edge
    shape = lambda Q, grid: [(qt, groups) for qt, _, _, groups in rp.tensor_launches(Q, grid)]
    assert any(shape(a, grid) != shape(b, grid) for grid in changed), f"{edge}: only the query counts change"


def test_grid_changes_the_groups():
    groups = {grid: {l[3] for l in rp.tensor_launches(641, grid)} for grid in rp.edges()["tensor grid (tiles)"]}
    assert groups[rp.NUM_SMS_H100] == groups[8] == {4, 2}  # 4 groups, then the 129-query tail in 2
    assert groups[7] == groups[3] == groups[1] == {1}
    assert groups[6] == groups[4] == {2}
    assert rp.grid(rp.ROWS * 7) == 7 and rp.grid(rp.ROWS * 7 + 1) == 8 and rp.grid(10 ** 6) == rp.NUM_SMS_H100
    # max_groups = 1: the same queries in more launches
    assert len(rp.tensor_launches(641, 8, max_groups=1)) > len(rp.tensor_launches(641, 8))


def test_simt_groups():
    assert rp.simt_range_groups(13, True) == [8, 8] and rp.simt_range_groups(13, False) == [4, 4, 4, 1]
    assert rp.simt_range_groups(2, True) == [2] and rp.simt_range_groups(2, False) == [1, 1]
    assert rp.simt_range_groups(5, True) == [8] and rp.simt_range_groups(5, False) == [4, 1]
    assert rp.simt_vec(64) and not rp.simt_vec(66)
    qs = rp.edges()["CUDA-core groups (Q)"]
    for vec in (True, False):
        for Q in qs:
            assert sum(min(a, b) for a, b in zip(rp.simt_range_groups(Q, vec), np.cumsum([Q] + [-x for x in rp.simt_range_groups(Q, vec)]))) == Q
    # every group size of each load kind starts a launch somewhere in the tested counts
    assert {qt for Q in qs for qt in rp.simt_range_groups(Q, True)} == {8, 4, 2, 1}
    assert {qt for Q in qs for qt in rp.simt_range_groups(Q, False)} == {4, 1}


def test_merge_passes_and_launch_counts():
    R = rp.RUN
    assert [rp.merge_passes(x) for x in (0, 1, R, R + 1, 2 * R, 2 * R + 1, 4 * R, 4 * R + 1)] == [0, 0, 0, 1, 1, 2, 2, 3]
    assert rp.query_blocks(rp.MAX_GRID_Y) == 1 and rp.query_blocks(rp.MAX_GRID_Y + 1) == 2
    # nothing listed: the scan alone; a list but no survivor cannot happen on a planted corpus, so survivors drive both
    assert rp.range_launches("simt", 9, 5000, [0] * 9, False) == 2
    assert rp.range_launches("filter", 9, 5000, [0] * 9, False) == 2
    assert rp.range_launches("filter", 9, 5000, [0] * 8 + [1], False) == 2 + 1 + 2
    assert rp.range_launches("shadow", 9, 5000, [R + 1] + [0] * 8, True) == 2 * 2 + 1 + 2 + 1
    Q = rp.MAX_GRID_Y + 1
    assert rp.range_launches("simt", Q, 100, [1] * Q, False) == len(rp.simt_range_groups(Q, True)) + 2 + 4


def test_scan_bytes():
    assert rp.row_bytes("shadow", 64) == 128 and rp.row_bytes("shadow", 64, image="int8") == 128
    assert rp.row_bytes("shadow", 66) == 256 and rp.row_bytes("shadow", 132, image="int8") == 256
    assert rp.row_bytes("shadow", 64, "f16") == 128 and rp.row_bytes("filter", 64) == 256 and rp.row_bytes("simt", 66) == 264
    assert rp.scan_bytes("simt", 1000, 256, 9, 2) == 1000 * 256 * 2 * 2
    assert rp.scan_bytes("filter", 1000, 256, 129, 1) == 1000 * 256 * 2


def test_gpu_cases_cover_every_edge():
    """every size of every edge appears in the GPU file's parametrizations"""
    e = rp.edges()
    fills = set(g.CAP_FILLS) | set(g.SURVIVORS)
    for name in ("list capacity (fill)",):
        assert set(e[name]) <= set(g.CAP_FILLS), name
    for name in ("re-scoring CTA (fill)", "compaction CTA (fill)", "sort run (survivors)", "second merge pass (survivors)",
                 "third merge pass (survivors)"):
        assert set(e[name]) <= set(g.SURVIVORS), name
        assert set(e[name]) <= fills
    assert set(e["query blocks (Q)"]) <= set(g.BLOCK_QS) and max(g.BLOCK_QS) > rp.MAX_GRID_Y + 1
    for name in ("tensor columns (Q)", "2 query groups (Q)", "4 query groups (Q)", "one 4-group launch (Q)",
                 "4-group launch and a tail (Q)"):
        assert set(e[name]) <= set(g.PLAN_QS), name
    assert set(e["tensor grid (tiles)"]) <= set(g.PLAN_GRIDS)
    assert set(e["CUDA-core groups (Q)"]) <= set(g.SIMT_QS)
    assert g.SATURATE_Q > 3 * 128 and rp.grid(g.SATURATE_N) >= 8 and rp.grid(g.SATURATE_N) % 4 == 0
    # the queries around the block boundary have distinct counts, among them 0 and more than RUN
    c = g.block_counts(max(g.BLOCK_QS))
    near = c[rp.MAX_GRID_Y - 2: rp.MAX_GRID_Y + 3]
    assert len(set(near.tolist())) == 5 and 0 in near and near.max() > rp.RUN and g.BLOCK_N >= c.sum()
    # the self-join's stripes scan windows whose grids are odd, 2 mod 4 and 0 mod 4, and one of them small
    grids = {rp.grid(g.PAIRS_N - (s + b) // rp.SCAN_TILE_ROWS * rp.SCAN_TILE_ROWS)
             for s in g.PAIRS_STARTS for b in range(0, g.PAIRS_N - s, rp.SEARCH_ROWS_BLOCK)}
    assert {x % 4 for x in grids} == {0, 1, 2, 3} and min(grids) < 4
    assert all(s % rp.SCAN_TILE_ROWS for s in g.PAIRS_STARTS)
    assert g.PAIRS_CLUSTER - 1 > rp.RUN and g.PAIRS_CLUSTER - 1 > rp.LIST0


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_planted_counts_are_exact_in_fp64(metric):
    counts = np.array([0, 3, 0, 1, 300, 0, rp.RUN + 1, 7], dtype=np.int64)
    p = rp.planted(counts, 64, metric, 20_000, 5)
    assert p.gap > 3 * rp.MIN_GAP, p.gap
    k, _ = rp.keys64(p.rows, p.queries, metric)
    tk = -(p.thr.astype(np.float64) ** 2) if metric == "euclidean" else p.thr.astype(np.float64)
    got = k >= tk[:, None]
    assert np.array_equal(got.sum(1), counts)
    for qi in range(len(counts)):
        assert np.array_equal(np.flatnonzero(got[qi]), p.expected(qi))
    # half of the long list is one row, copied
    mine = p.rows[p.owner == 6]
    assert (np.unique(mine, axis=0).shape[0]) == len(mine) - len(mine) // 2 + 1


def test_planted_d32_many_queries():
    counts = np.zeros(3000, dtype=np.int64)
    counts[[5, 1000, 2999]] = [rp.RUN + 3, 1, 17]
    p = rp.planted(counts, 32, "cosine", 8000, 6)
    assert p.gap > 2 * rp.MIN_GAP, p.gap
    k, _ = rp.keys64(p.rows, p.queries, "cosine")
    assert np.array_equal((k >= p.thr.astype(np.float64)[:, None]).sum(1), counts)


def merge_all(keys, off):
    a = rp.sort_runs(keys, off)
    longest = int(np.diff(off).max())
    w = rp.RUN
    passes = 0
    while w < longest:
        a = rp.merge_pass(a, off, w)
        w *= 2
        passes += 1
    assert passes == rp.merge_passes(longest)
    return a


def test_merge_placement_sorts_at_the_edges_with_empty_segments_and_ties():
    """segments of 0, 1, 2, 3 and 5 runs and at the merge edges, empty segments between them; thousands of keys share one
    score, so (score desc, row asc) rests on the row bits"""
    R = rp.RUN
    lens = [0, 2 * R, 0, 2 * R + 1, 1, 0, 4 * R, 4 * R + 1, 0, 3 * R - 7, 5 * R, 0, R + 1]
    rng = np.random.default_rng(3)
    off = np.zeros(len(lens) + 1, dtype=np.uint64)
    off[1:] = np.cumsum(lens)
    keys = np.empty(int(off[-1]), dtype=np.uint64)
    for q, n in enumerate(lens):
        rows = rng.permutation(200_000)[:n]
        sc = rng.choice(np.float32([0.25, -0.5, 0.9, 0.125]), size=n) if q % 2 else rng.standard_normal(n).astype(np.float32)
        if n > 8:
            sc[: n // 2] = np.float32(0.75)  # one score across every run and merge boundary
        keys[int(off[q]):int(off[q + 1])] = rp.make_keys(sc, rows)
    out = merge_all(keys, off)
    for q in range(len(lens)):
        seg = out[int(off[q]):int(off[q + 1])]
        assert np.array_equal(seg, np.sort(keys[int(off[q]):int(off[q + 1])])[::-1]), q


def test_make_keys_order():
    k = rp.make_keys(np.float32([0.5, 0.5, -1.0, 2.0, -0.0]), np.array([7, 3, 1, 9, 4]))
    assert list(np.argsort(k)[::-1]) == [3, 1, 0, 4, 2]
