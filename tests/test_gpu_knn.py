"""GPU parity tests proper: the fused CUDA path, called through the C ABI, against the CPU oracle on the same
seeded inputs (sizes the oracle finishes in seconds), plus the reference's edge cases."""
import json
import os

import numpy as np
import pytest

from parity import check_parity

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_case(oracle, n, d, Q, k, metric, dtype="f32", seed=42, path="auto", devices=(0,), mutate=None):
    from nornicdb_b200.knn import KnnIndex
    rows = oracle.fill_uniform(n, d, seed, dtype=dtype)
    q = oracle.fill_uniform(Q, d, seed + 1295)
    if mutate:
        rows, q = mutate(rows, q)
    ix = KnnIndex(d, metric=metric, dtype=dtype, devices=devices)
    try:
        ix.set_path(path)
        ix.upload(rows)
        gi, gs = ix.search(q, k)
    finally:
        ix.release()
    oi, os_ = oracle.knn_exact64(rows, q, k, metric)
    assert gi.shape == (Q, min(k, n))
    return check_parity(rows, q, k, metric, gi, gs, oi, os_)


# BASELINE.json configs[0]: N=100k d=128 fp32 Q=1 k=10 cosine — the reference's own CPU-runnable case.
def test_config1_correctness_reference(knn_lib, oracle_mod):
    assert run_case(oracle_mod, 100_000, 128, 1, 10, "cosine") == 0


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
@pytest.mark.parametrize("Q", [1, 2, 3, 5, 8, 9, 17])
def test_query_group_sizes(knn_lib, oracle_mod, metric, Q):
    run_case(oracle_mod, 5000, 256, Q, 10, metric)


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
@pytest.mark.parametrize("d", [1, 3, 7, 33, 130, 384, 768, 1024, 1536])
def test_dims_vector_and_scalar_paths(knn_lib, oracle_mod, metric, d):
    run_case(oracle_mod, 3001, d, 4, 10, metric)


@pytest.mark.parametrize("k", [1, 2, 10, 100, 257, 1024])
def test_k_values(knn_lib, oracle_mod, k):
    run_case(oracle_mod, 20_000, 64, 3, k, "cosine")
    run_case(oracle_mod, 20_000, 64, 3, k, "euclidean")


@pytest.mark.parametrize("n", [1, 2, 31, 255, 256, 257, 1000, 65_537])
def test_ragged_row_counts_and_k_clamp(knn_lib, oracle_mod, n):
    # k > n -> n results (cuda_bridge.go:647-649)
    run_case(oracle_mod, n, 48, 2, 10, "cosine")
    run_case(oracle_mod, n, 48, 2, 10, "dot")


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_fp16_corpus(knn_lib, oracle_mod, metric):
    # BASELINE.json configs[3] shape (d=768 fp16 Q=1 k=10 L2) at an oracle-sized N; scalar path via d=50
    run_case(oracle_mod, 30_000, 768, 1, 10, metric, dtype="f16")
    run_case(oracle_mod, 2000, 50, 3, 10, metric, dtype="f16")


def test_zero_vectors_score_zero(knn_lib, oracle_mod):
    # zero corpus rows and a zero query -> cosine 0 (simd_amd64.go:31-35: NaN -> 0), never NaN
    def mutate(rows, q):
        rows[5] = 0.0
        rows[77] = 0.0
        q[1] = 0.0
        return rows, q
    run_case(oracle_mod, 1000, 64, 2, 1000, "cosine", mutate=mutate)


def test_ties_lowest_index_first(knn_lib, oracle_mod):
    # duplicate rows: among equal scores the lowest row index wins and comes first (cuda_bridge.go:356-371)
    from nornicdb_b200.knn import KnnIndex
    base = oracle_mod.fill_uniform(16, 32, 5)
    rows = np.tile(base, (64, 1))  # row r == row r % 16
    q = base[3:4].copy()
    for metric in ("cosine", "dot", "euclidean"):
        ix = KnnIndex(32, metric=metric)
        ix.upload(rows)
        gi, gs = ix.search(q, 20)
        ix.release()
        assert gi[0].tolist() == [3 + 16 * j for j in range(20)], metric
        assert np.ptp(gs[0]) == 0.0


def test_all_equal_scores(knn_lib):
    from nornicdb_b200.knn import KnnIndex
    rows = np.ones((5000, 8), np.float32)
    ix = KnnIndex(8, metric="dot")
    ix.upload(rows)
    gi, gs = ix.search(np.ones((3, 8), np.float32), 100)
    ix.release()
    assert (gi == np.arange(100)[None, :]).all() and (gs == 8.0).all()


def test_adversarial_ascending_scores(knn_lib, oracle_mod):
    # every row beats all earlier rows: worst case for the threshold filter (every row is buffered)
    from nornicdb_b200.knn import KnnIndex
    n, d = 50_000, 16
    rows = np.zeros((n, d), np.float32)
    rows[:, 0] = np.arange(n, dtype=np.float32)
    q = np.zeros((2, d), np.float32)
    q[0, 0], q[1, 0] = 1.0, -1.0
    ix = KnnIndex(d, metric="dot")
    ix.upload(rows)
    gi, gs = ix.search(q, 100)
    ix.release()
    assert gi[0].tolist() == list(range(n - 1, n - 101, -1))
    assert gi[1].tolist() == list(range(100))


def test_empty_index_and_zero_k(knn_lib):
    from nornicdb_b200.knn import KnnIndex, KnnError
    ix = KnnIndex(4)
    gi, gs = ix.search(np.ones((2, 4), np.float32), 5)  # empty index -> no results (gpu.go:1540-1542)
    assert gi.shape == (2, 0)
    ix.upload(np.eye(4, dtype=np.float32))
    gi, gs = ix.search(np.ones((2, 4), np.float32), 0)  # k == 0 -> nil (cuda_bridge.go:644-646)
    assert gi.shape == (2, 0)
    with pytest.raises(KnnError):  # ErrInvalidDimensions (gpu.go:1533-1535)
        ix.search(np.ones((1, 5), np.float32), 1)
    ix.release()


def test_k_above_max_clamps_to_n_first(knn_lib):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex(4)
    ix.upload(np.eye(4, dtype=np.float32))
    gi, _ = ix.search(np.ones((1, 4), np.float32), 5000)
    assert gi.shape == (1, 4)
    ix.release()


def test_embedding_index_kat(knn_lib, kats):
    from nornicdb_b200.knn import KnnIndex
    for t in [t for t in kats if t["op"] == "gpu.embedding_index_search"]:
        ix = KnnIndex(len(t["query"]))
        ix.upload(np.asarray(t["vectors"], np.float32))
        gi, gs = ix.search(np.asarray([t["query"]], np.float32), t["k"])
        ix.release()
        assert [t["ids"][i] for i in gi[0]] == t["want_ids"]
        assert gs[0, 0] >= t["want_first_score_ge"]


def test_append_update_remove(knn_lib, oracle_mod):
    # EmbeddingIndex.Add / update-in-place / Remove (swap with last), gpu.go:1378-1471 — without re-upload
    from nornicdb_b200.knn import KnnIndex
    rows = oracle_mod.fill_uniform(1000, 64, 9)
    q = oracle_mod.fill_uniform(3, 64, 10)
    ix = KnnIndex(64, metric="cosine")
    ix.upload(rows[:600])
    ix.append(rows[600:])
    assert len(ix) == 1000
    assert (ix.read_rows(0, 1000) == rows).all()
    gi, gs = ix.search(q, 10)
    oi, os_ = oracle_mod.knn_exact64(rows, q, 10, "cosine")
    check_parity(rows, q, 10, "cosine", gi, gs, oi, os_)
    host = rows.copy()
    host[17] = q[0] * 2.0  # now the best match of query 0
    ix.update_row(17, host[17])
    victim = int(oi[1, 0])
    host[victim] = host[-1]
    host = host[:-1]
    ix.remove_swap(victim)
    assert len(ix) == 999
    gi, gs = ix.search(q, 10)
    oi, os_ = oracle_mod.knn_exact64(host, q, 10, "cosine")
    check_parity(host, q, 10, "cosine", gi, gs, oi, os_)
    assert gi[0, 0] == 17
    ix.release()


def test_score_subset(knn_lib, kats, oracle_mod):
    from nornicdb_b200.knn import KnnIndex
    for t in [t for t in kats if t["op"] == "gpu.score_subset"]:
        ix = KnnIndex(3)
        ix.upload(np.asarray(t["vectors"], np.float32))
        pos = {name: i for i, name in enumerate(t["ids"])}
        subset = [pos[s] for s in t["subset"] if s in pos]  # missing ids ignored (gpu.go:1566-1571)
        gi, _ = ix.score_subset(t["query"], subset)
        ix.release()
        assert [t["ids"][i] for i in gi] == t["want_ids"]
    rows = oracle_mod.fill_uniform(5000, 96, 21)
    q = oracle_mod.fill_uniform(1, 96, 22)[0]
    subset = np.random.default_rng(3).choice(5000, 700, replace=False).astype(np.uint32)
    ix = KnnIndex(96)
    ix.upload(rows)
    before = ix.stats()["bytes_scanned"]
    gi, gs = ix.score_subset(q, subset)
    assert ix.stats()["bytes_scanned"] - before == 700 * 96 * 4  # the subset rows, one CUDA-core pass
    ix.release()
    ex = oracle_mod.scores_exact64(rows[subset], q, "cosine")
    order = np.argsort(-ex, kind="stable")
    assert (gi == subset[order]).all()
    assert np.allclose(gs, ex[order], rtol=1e-4, atol=1e-6)


def test_golden_fixture(knn_lib, oracle_mod):
    """Committed golden fixture (tests/golden/knn_small.json, generated by make_knn_fixture.py from the oracle)."""
    from nornicdb_b200.knn import KnnIndex
    with open(os.path.join(ROOT, "tests", "golden", "knn_small.json")) as f:
        fx = json.load(f)
    for case in fx["cases"]:
        rows = oracle_mod.fill_uniform(case["n"], case["d"], case["seed"], dtype=case["dtype"])
        q = oracle_mod.fill_uniform(case["Q"], case["d"], case["qseed"])
        ix = KnnIndex(case["d"], metric=case["metric"], dtype=case["dtype"])
        ix.upload(rows)
        gi, gs = ix.search(q, case["k"])
        ix.release()
        assert gi.tolist() == case["idx"], case
        assert np.allclose(gs, case["score"], rtol=1e-4, atol=1e-6)


def test_stats_and_device_api(knn_lib, oracle_mod):
    import torch
    from nornicdb_b200.knn import KnnIndex, merge_keys_device
    n, d, Q, k = 20_000, 128, 6, 10
    ix = KnnIndex(d, metric="cosine")
    ix.fill_uniform(n, 42)
    rows = oracle_mod.fill_uniform(n, d, 42)
    assert (ix.read_rows(100, 50) == rows[100:150]).all()  # device generator == oracle generator
    q = oracle_mod.fill_uniform(Q, d, 1337)
    qd = torch.from_numpy(q).cuda()
    oi_d = torch.empty((Q, k), dtype=torch.int32, device="cuda")
    os_d = torch.empty((Q, k), dtype=torch.float32, device="cuda")
    stream = torch.cuda.Stream()  # an explicit stream: handle 0 means "the index's own stream" to the C ABI
    torch.cuda.current_stream().synchronize()
    st = stream.cuda_stream
    assert ix.search_device(qd.data_ptr(), Q, k, oi_d.data_ptr(), os_d.data_ptr(), st) == k
    torch.cuda.synchronize()
    gi, gs = ix.search(q, k)
    assert (oi_d.cpu().numpy().view(np.uint32) == gi).all() and (os_d.cpu().numpy() == gs).all()
    oi, os_ = oracle_mod.knn_exact64(rows, q, k, "cosine")
    check_parity(rows, q, k, "cosine", gi, gs, oi, os_)
    # two half shards (row_base) + key merge == the full search (row-sharding is result-invariant, §8e)
    keys = torch.empty((2, Q, k), dtype=torch.int64, device="cuda")
    halves = []
    for g in range(2):
        h = KnnIndex(d, metric="cosine")
        h.set_row_base(g * n // 2)
        h.fill_uniform(n // 2, 42)
        h.search_keys_device(qd.data_ptr(), Q, k, keys[g].data_ptr(), st)
        halves.append(h)
    merge_keys_device(0, keys.data_ptr(), 2, Q, k, "cosine", oi_d.data_ptr(), os_d.data_ptr(), st)
    torch.cuda.synchronize()
    assert (oi_d.cpu().numpy().view(np.uint32) == gi).all() and (os_d.cpu().numpy() == gs).all()
    for h in halves:
        h.release()
    s = ix.stats()
    assert s["rows"] == n and s["searches"] >= 2 and s["kernel_launches"] > 0 and s["bytes_scanned"] >= n * d * 4
    ix.release()


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_k_beyond_one_pass(knn_lib, oracle_mod, metric):
    # the reference accepts any k (cuda_bridge.go:327-375): k > NK_MAX_K is served by repeated bounded passes
    rows_n, d = 9000, 48
    run_case(oracle_mod, rows_n, d, 3, 2500, metric)
    run_case(oracle_mod, rows_n, d, 1, rows_n, metric)  # full ranking, k == n


def test_legacy_topk_any_k(gpu_device, oracle_mod):
    rng = np.random.default_rng(5)
    scores = rng.integers(-500, 500, 20000).astype(np.float32) / 16.0
    s = gpu_device.NewBuffer(scores)
    idx, sc = gpu_device.TopK(s, 20000, 3000)
    oi, os_ = oracle_mod.topk_insertion(scores, 3000)
    assert (idx == oi).all() and (sc == os_).all()
    s.Release()


def test_score_subset_large(knn_lib, oracle_mod):
    from nornicdb_b200.knn import KnnIndex
    rows = oracle_mod.fill_uniform(8000, 64, 31)
    q = oracle_mod.fill_uniform(1, 64, 32)[0]
    subset = np.random.default_rng(4).choice(8000, 3000, replace=False).astype(np.uint32)
    ix = KnnIndex(64)
    ix.upload(rows)
    before = ix.stats()["bytes_scanned"]
    gi, gs = ix.score_subset(q, subset)  # ranks all 3000 candidates (> NK_MAX_K)
    assert ix.stats()["bytes_scanned"] - before == 3 * 3000 * 64 * 4  # the subset rows, once per NK_MAX_K pass
    ix.release()
    ex = oracle_mod.scores_exact64(rows[subset], q, "cosine")
    order = np.argsort(-ex, kind="stable")
    assert (gi == subset[order]).all()


def test_multi_device_index_in_one_process(knn_lib, oracle_mod):
    """nk_index_create over several GPUs of this process: rows are range-sharded, every shard scans asynchronously,
    the Q*k candidate keys come back over PCIe and are merged on the host (SURVEY.md §8e, small-Q form)."""
    from nornicdb_b200 import cuda
    from nornicdb_b200.knn import KnnIndex
    G = min(cuda.DeviceCount(), 4)
    if G < 2:
        pytest.skip("needs >= 2 GPUs in this process")
    n, d, Q, k = 30_001, 128, 20, 25
    rows = oracle_mod.fill_uniform(n, d, 42)
    q = oracle_mod.fill_uniform(Q, d, 1337)
    for metric in ("cosine", "euclidean"):
        ix = KnnIndex(d, metric=metric, devices=tuple(range(G)))
        ix.upload(rows)
        assert len(ix) == n and (ix.read_rows(n // 2 - 3, 6) == rows[n // 2 - 3:n // 2 + 3]).all()
        gi, gs = ix.search(q, k)
        oi, os_ = oracle_mod.knn_exact64(rows, q, k, metric)
        check_parity(rows, q, k, metric, gi, gs, oi, os_)
        one = KnnIndex(d, metric=metric, devices=(0,))
        one.upload(rows)
        si, ss = one.search(q, k)
        assert (si == gi).all() and np.allclose(ss, gs, rtol=2e-6, atol=1e-6)  # independent of the sharding
        # append goes to the last shard; remove swaps across shards
        extra = oracle_mod.fill_uniform(50, d, 99)
        ix.append(extra)
        ix.remove_swap(5)
        host = np.concatenate([rows, extra])
        host[5] = host[-1]
        host = host[:-1]
        gi, gs = ix.search(q, k)
        oi, os_ = oracle_mod.knn_exact64(host, q, k, metric)
        check_parity(host, q, k, metric, gi, gs, oi, os_)
        ix.release(); one.release()
    ix = KnnIndex(d, metric="cosine", devices=tuple(range(G)))
    ix.fill_uniform(n, 42)  # device-side generation is shard-aware: same global stream
    assert (ix.read_rows(0, n) == rows).all()
    ix.release()


@pytest.mark.parametrize("path,Q", [("simt", 3), ("shadow", 40), ("filter", 40), ("tensor", 40), ("auto", 300)])
@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_row_mask_filters_inside_every_kernel(knn_lib, oracle_mod, path, Q, metric):
    """nk_index_set_row_mask (label filter of queryNodes, call_vector.go:177-193): masked search == search over the kept rows."""
    from nornicdb_b200.knn import KnnIndex
    if path == "tensor" and metric == "euclidean":
        pytest.skip("exact 3xTF32 path: cosine / dot only")
    n, d, k = 7_000, 64, 10
    rows = oracle_mod.fill_uniform(n, d, 11)
    q = oracle_mod.fill_uniform(Q, d, 12)
    keep = np.random.default_rng(4).random(n) < 0.3
    keep[:40] = False
    ix = KnnIndex(d, metric=metric)
    ix.upload(rows)
    ix.set_path(path)
    ix.set_row_mask(keep)
    gi, gs = ix.search(q, k)
    kept = np.nonzero(keep)[0]
    oi, os_ = oracle_mod.knn_exact64(rows[kept], q, k, metric)
    check_parity(rows, q, k, metric, gi, gs, kept[oi].astype(np.uint32), os_)
    assert keep[gi].all()
    # fewer kept rows than k: k is clamped to the number of set bits
    few = np.zeros(n, dtype=bool)
    few[[5, 77, 6_999]] = True
    ix.set_row_mask(few)
    gi, gs = ix.search(q[:2], k)
    assert gi.shape == (2, 3) and sorted(gi[0].tolist()) == [5, 77, 6_999]
    ix.set_row_mask(None)  # cleared: the full corpus again
    gi, gs = ix.search(q, k)
    oi, os_ = oracle_mod.knn_exact64(rows, q, k, metric)
    check_parity(rows, q, k, metric, gi, gs, oi, os_)
    ix.set_row_mask(keep)
    ix.append(rows[:3])    # a row-count change drops the mask
    gi, _ = ix.search(q[:1], k)
    assert gi.shape == (1, k)
    ix.release()
