"""CPU companion of tests/test_gpu_index_lifecycle.py: the fp64 model's bookkeeping, the scripts' reach, and the harness end to
end with the model answering as the device."""
import numpy as np
import pytest

from test_gpu_index_lifecycle import CASES, Case, Lifecycle, Model, ModelIndex, build_script, required_edges


def test_model_remove_swap_agrees_with_graph_row_map():
    """The model's remove_swap moves the last row's contents, tag and key into the slot, as GraphRowMap says it does."""
    from nornicdb_b200.knn import ROW_NEW, GraphRowMap
    rng = np.random.default_rng(1)
    n, d = 60, 8
    m = Model(d, "f32", "cosine", 3)
    m.upload(rng.standard_normal((n, d)).astype(np.float32), np.ones(n, bool))
    m.set_row_tags(0, np.arange(n, dtype=np.uint64) + 1)   # the tag of each original row names it
    m.set_row_values(0, np.arange(n, dtype=np.uint64) + 1)
    gm = GraphRowMap(n)
    for _ in range(200):
        u = rng.random()
        if u < 0.5 and len(m) > 1:
            r = int(rng.integers(len(m)))
            m.remove_swap(r)
            gm.remove_swap(r)
        elif u < 0.8:
            m.append(rng.standard_normal((2, d)).astype(np.float32), np.ones(2, bool))
            gm.append(2)
        else:
            r = int(rng.integers(len(m)))
            m.update_row(r, rng.standard_normal(d).astype(np.float32))
            m.set_row_tags(r, np.zeros(1, np.uint64))
            gm.update_row(r)
        src = gm.src_of_row
        assert len(src) == len(m) == sum(m.shard_n)
        old = src != ROW_NEW
        assert (m.tags[old] == src[old] + 1).all() and (m.keys[old] == src[old] + 1).all()
        assert (m.tags[~old] == 0).all()  # appended or rewritten rows


def test_model_follows_the_repartition_rule():
    m = Model(4, "f32", "dot", 3)
    m.upload(np.zeros((10, 4), np.float32), np.ones(10, bool))
    assert m.shard_n == [3, 3, 4] and m.shard_cap == [16, 16, 16]
    m.upload(np.zeros((100, 4), np.float32), np.ones(100, bool))
    assert m.shard_n == [33, 33, 34] and m.shard_of(66) == (2, 0) and m.shard_of(65) == (1, 32)
    m.append(np.zeros((1, 4), np.float32), [True])
    assert "regrow" in m.edges and m.shard_cap[2] == 51
    m.remove_swap(0)  # the last row, in shard 2, moves into shard 0
    assert "cross_shard_move" in m.edges and m.shard_n == [33, 33, 34]


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_each_script_reaches_its_edges(case):
    """Computed from the layout rules alone: a regrowth, an append that fits, the first / last row of every shard rewritten,
    a cross-shard move, an emptied trailing shard and an append into it, straddling tag and value ranges, and the mask, the
    floor and the metric set after mutations."""
    steps, m = build_script(case)
    missing = required_edges(case) - m.edges
    assert not missing, missing
    assert sum(m.shard_n) == len(m)
    if case.big:  # AUTO keeps serving k <= 16 from the int8 image: >= 64 MB of fp32 rows after every step
        n = case.n
        for step in steps[1:]:
            for a in step:
                n += len(a[1]) if a[0] == "append" else -1 if a[0] == "remove" else 0
                assert n * case.dim * 4 >= 64 << 20


def test_scripts_are_seeded():
    case = CASES[2]
    (a, _), (b, _) = build_script(case), build_script(case)
    for sa, sb in zip(a, b):
        assert len(sa) == len(sb)
        for x, y in zip(sa, sb):
            assert x[0] == y[0] and all(np.array_equal(np.asarray(u), np.asarray(v)) for u, v in zip(x[1:], y[1:]))


@pytest.mark.parametrize("devices,dtype,dim,metric,big", [((0,), "f32", 36, "cosine", False), ((0, 0, 0), "f32", 40, "euclidean", False),
                                                         ((0, 0, 0), "bf16", 16, "dot", False), ((0,), "f16", 24, "euclidean", False),
                                                         ((0,), "f32", 32, "dot", True)])
def test_harness_runs_end_to_end_on_the_model(devices, dtype, dim, metric, big):
    """Every step and every check of the GPU test, at a tiny size, with ModelIndex in place of KnnIndex (big: the large
    case's shape of the script and its self-join stripe)."""
    case = Case("tiny", dtype, None, devices, dim, 90, metric, big)
    run = Lifecycle(case, lambda devs, met: ModelIndex(dim, met, dtype, devs))
    run.run()
    assert required_edges(case) <= run.model.edges
    assert big or (run.graph is not None and len(run.graph[1]) == len(run.model))
