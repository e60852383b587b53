"""GPU parity tests of the wgmma / TMA scan (path="tensor") against the fp64 oracle."""
import numpy as np
import pytest

from parity import check_parity

pytestmark = pytest.mark.gpu


def run_tc(oracle, n, d, Q, k, metric, seed=7, mutate=None, path="tensor"):
    from nornicdb_b200.knn import KnnIndex
    rows = oracle.fill_uniform(n, d, seed)
    q = oracle.fill_uniform(Q, d, seed + 999)
    if mutate:
        rows, q = mutate(rows, q)
    ix = KnnIndex(d, metric=metric)
    try:
        ix.set_path(path)
        ix.upload(rows)
        gi, gs = ix.search(q, k)
        assert ix.last_path() == path
        # the CUDA-core scan on the same index must agree (two independent kernels)
        ix.set_path("simt")
        si, ss = ix.search(q, k)
    finally:
        ix.release()
    oi, os_ = oracle.knn_exact64(rows, q, k, metric)
    swaps = check_parity(rows, q, k, metric, gi, gs, oi, os_)
    check_parity(rows, q, k, metric, si, ss, oi, os_)
    return swaps


@pytest.mark.parametrize("metric", ["cosine", "dot"])
def test_tensor_small(knn_lib, oracle_mod, metric):
    run_tc(oracle_mod, 5000, 256, 64, 10, metric)


@pytest.mark.parametrize("Q", [1, 17, 64, 65, 130])
def test_tensor_query_counts(knn_lib, oracle_mod, Q):
    run_tc(oracle_mod, 3000, 128, Q, 10, "cosine")


@pytest.mark.parametrize("n", [1, 100, 255, 256, 257, 511, 513, 40_000])
def test_tensor_ragged_rows(knn_lib, oracle_mod, n):
    run_tc(oracle_mod, n, 64, 8, 10, "dot")


@pytest.mark.parametrize("d", [32, 36, 100, 768, 1024, 1536])
def test_tensor_dims(knn_lib, oracle_mod, d):
    run_tc(oracle_mod, 4000, d, 32, 10, "cosine")


@pytest.mark.parametrize("k", [1, 100, 255])
def test_tensor_k(knn_lib, oracle_mod, k):
    run_tc(oracle_mod, 30_000, 64, 16, k, "cosine")


def test_tensor_config2_shape_subsampled(knn_lib, oracle_mod):
    # BASELINE.json configs[1] shape (d=1024 Q=64 k=10 cosine) at an oracle-sized N
    assert run_tc(oracle_mod, 60_000, 1024, 64, 10, "cosine") <= 2


def test_tensor_zero_vectors_and_ties(knn_lib, oracle_mod):
    def mutate(rows, q):
        rows[3] = 0.0
        rows[300] = 0.0
        rows[700] = rows[10]  # duplicate row: tie broken by lowest index
        q[2] = 0.0
        return rows, q
    run_tc(oracle_mod, 2000, 96, 5, 200, "cosine", mutate=mutate)
    from nornicdb_b200.knn import KnnIndex
    base = oracle_mod.fill_uniform(16, 64, 5)
    rows = np.tile(base, (64, 1))
    ix = KnnIndex(64, metric="dot")
    ix.set_path("tensor")
    ix.upload(rows)
    gi, gs = ix.search(base[3:4], 20)
    ix.release()
    assert gi[0].tolist() == [3 + 16 * j for j in range(20)]


def test_tensor_unsupported_shapes_fail_loudly(knn_lib, oracle_mod):
    from nornicdb_b200.knn import KnnIndex, KnnError
    ix = KnnIndex(30, metric="cosine")  # dim % 4 != 0 -> no TMA path
    ix.set_path("tensor")
    ix.upload(oracle_mod.fill_uniform(100, 30, 1))
    with pytest.raises(KnnError):
        ix.search(oracle_mod.fill_uniform(1, 30, 2), 5)
    ix.release()


# ---- filter mode: 1xTF32 prefilter with rigorous margins + exact fp32 rescoring --------------------------------
@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
@pytest.mark.parametrize("shape", [(5000, 256, 64, 10), (3000, 128, 17, 10), (40_000, 64, 8, 100), (257, 100, 3, 10),
                                   (60_000, 1024, 64, 10), (20_000, 768, 130, 10), (100, 32, 5, 192), (30_000, 128, 520, 10), (9_000, 64, 300, 50)])
def test_filter_parity(knn_lib, oracle_mod, metric, shape):
    n, d, Q, k = shape
    assert run_tc(oracle_mod, n, d, Q, k, metric, path="filter") == 0  # exact fp32 rescoring: no boundary swaps expected


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
@pytest.mark.parametrize("shape", [(20_000, 768, 130, 10), (30_000, 128, 520, 10), (9_000, 64, 300, 50), (50_000, 96, 1024, 100),
                                   (3_000, 1024, 257, 10)])
def test_filter_parity_big_batches_tf32_groups(knn_lib, oracle_mod, metric, shape):
    """Q > 128: the TF32 kernel's query groups (2 / 4 blocks of 128 queries per launch share corpus tiles through L2)."""
    n, d, Q, k = shape
    # exact fp32 rescoring; fp32-vs-fp64 boundary swaps (scores equal to ~1e-7) appear once Q*k reaches ~1e5 results
    assert run_tc(oracle_mod, n, d, Q, k, metric, path="filter") <= Q * k // 2000


# ---- shadow mode: the same filter over the BF16 shadow corpus, exact fp32 rescoring from the fp32 rows ----------------
@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
@pytest.mark.parametrize("shape", [(5000, 256, 64, 10), (3000, 128, 17, 10), (40_000, 64, 8, 100), (257, 100, 3, 10),
                                   (60_000, 1024, 64, 10), (20_000, 768, 130, 10), (100, 32, 5, 192), (30_000, 132, 520, 10),
                                   (9_000, 36, 300, 50), (50_000, 128, 1024, 100), (3_000, 1024, 257, 10)])
def test_shadow_parity(knn_lib, oracle_mod, metric, shape):
    """path="shadow": 64 / 128 query columns, 1 / 2 / 4 query groups, ragged tiles, dims that are not multiples of 64."""
    n, d, Q, k = shape
    assert run_tc(oracle_mod, n, d, Q, k, metric, path="shadow") <= Q * k // 2000


@pytest.mark.parametrize("path", ["filter", "shadow"])
def test_filter_equals_simt_bitwise_on_indices(knn_lib, oracle_mod, path):
    """Final scores come from exact fp32 rescoring, so the filter paths and the CUDA-core scan agree on every index."""
    from nornicdb_b200.knn import KnnIndex
    rows = oracle_mod.fill_uniform(30_000, 512, 3)
    q = oracle_mod.fill_uniform(64, 512, 4)
    ix = KnnIndex(512, metric="cosine")
    ix.upload(rows)
    ix.set_path(path)
    fi, fs = ix.search(q, 10)
    flags = ix.debug_flags()
    assert flags[:2] == [0, 0] and flags[3] == 0, flags  # ordinary data: no overflow, no retry, no fallback
    ix.set_path("simt")
    si, ss = ix.search(q, 10)
    ix.release()
    assert (fi == si).all()
    assert np.allclose(fs, ss, rtol=2e-6, atol=1e-7)


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_filter_margin_overflow_falls_back_on_device(knn_lib, oracle_mod, metric):
    """Adversarial near-ties: thousands of rows within the TF32 margin of the k-th best overflow the margin buffers; the
    device-side flag makes the exact kernels queued behind redo the search — results still match the oracle."""
    from nornicdb_b200.knn import KnnIndex
    rng = np.random.default_rng(0)
    base = oracle_mod.fill_uniform(1, 128, 9)[0]
    rows = np.tile(base, (20_000, 1)) + rng.standard_normal((20_000, 128)).astype(np.float32) * 1e-5
    rows[::7] = oracle_mod.fill_uniform(len(rows[::7]), 128, 10)
    q = (base[None, :] + rng.standard_normal((20, 128)).astype(np.float32) * 1e-3).astype(np.float32)
    ix = KnnIndex(128, metric=metric)
    ix.upload(rows)
    ix.set_path("filter")
    gi, gs = ix.search(q, 10)
    flags = ix.debug_flags()
    ix.release()
    assert flags[0] == 0 and flags[1] != 0, flags  # a margin buffer / list did overflow (bit = which); the exact fallback answered
    oi, os_ = oracle_mod.knn_exact64(rows, q, 10, metric)
    check_parity(rows, q, 10, metric, gi, gs, oi, os_, swap_eps=5e-6)


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_shadow_margin_overflow_retries_with_tf32_then_exact(knn_lib, oracle_mod, metric):
    """Adversarial near-ties: the BF16 shadow stage overflows, the TF32 filter queued behind retries on the device (and,
    if that overflows too, the exact kernels); results still match the oracle."""
    from nornicdb_b200.knn import KnnIndex
    rng = np.random.default_rng(1)
    base = oracle_mod.fill_uniform(1, 128, 9)[0]
    # 160k near-copies: > 768 rows inside the 16-bit margin per CTA — more than a 1024-slot buffer can hold between prunes
    # (a few thousand near-copies are simply re-scored in rounds by the finish step: test_gpu_round2.py)
    rows = np.tile(base, (160_000, 1)) + rng.standard_normal((160_000, 128)).astype(np.float32) * 1e-4
    rows[::7] = oracle_mod.fill_uniform(len(rows[::7]), 128, 10)
    q = (base[None, :] + rng.standard_normal((40, 128)).astype(np.float32) * 1e-3).astype(np.float32)
    ix = KnnIndex(128, metric=metric)
    ix.upload(rows)
    ix.set_path("shadow")
    gi, gs = ix.search(q, 10)
    flags = ix.debug_flags()
    ix.release()
    assert flags[0] == 0 and flags[3] == 1, flags  # the shadow stage did overflow; the TF32 stage re-ran the search
    oi, os_ = oracle_mod.knn_exact64(rows, q, 10, metric)
    check_parity(rows, q, 10, metric, gi, gs, oi, os_, swap_eps=5e-6)


@pytest.mark.parametrize("path", ["filter", "shadow"])
def test_filter_ties_and_zero_vectors(knn_lib, oracle_mod, path):
    from nornicdb_b200.knn import KnnIndex
    base = oracle_mod.fill_uniform(16, 64, 5)
    rows = np.tile(base, (64, 1))
    rows[5] = 0.0
    for metric in ("cosine", "dot", "euclidean"):
        ix = KnnIndex(64, metric=metric)
        ix.set_path(path)
        ix.upload(rows)
        gi, gs = ix.search(base[3:4], 20)
        ix.release()
        assert gi[0].tolist() == [3 + 16 * j for j in range(20)], metric


def test_shadow_follows_incremental_updates(knn_lib, oracle_mod):
    """append / update_row / remove_swap keep the BF16 shadow (and its per-row norms) in step with the fp32 rows."""
    from nornicdb_b200.knn import KnnIndex
    d, k = 96, 10
    rows = oracle_mod.fill_uniform(3000, d, 3)
    extra = oracle_mod.fill_uniform(1500, d, 4)
    q = oracle_mod.fill_uniform(9, d, 5)
    ix = KnnIndex(d, metric="cosine")
    ix.set_path("shadow")
    ix.upload(rows)
    ix.append(extra[:700])          # fits or regrows the shard: either way the shadow must cover the new rows
    ix.append(extra[700:])
    cur = np.concatenate([rows, extra])
    new_row = q[4] * 3.0            # becomes the best match of query 4
    ix.update_row(1234, new_row)
    cur[1234] = new_row
    ix.remove_swap(7)               # last row moves into slot 7
    cur[7] = cur[-1]
    cur = cur[:-1]
    ix.update_row(len(cur) - 1, q[2] * 0.5)
    cur[-1] = q[2] * 0.5
    gi, gs = ix.search(q, k)
    assert ix.last_path() == "shadow"
    ix.release()
    oi, os_ = oracle_mod.knn_exact64(cur, q, k, "cosine")
    check_parity(cur, q, k, "cosine", gi, gs, oi, os_)
    assert gi[4][0] == 1234 and gi[2][0] == len(cur) - 1


def test_auto_dispatch(knn_lib, oracle_mod):
    from nornicdb_b200.knn import KnnIndex
    rows = oracle_mod.fill_uniform(2000, 128, 1)
    ix = KnnIndex(128, metric="cosine")
    ix.upload(rows)
    ix.search(oracle_mod.fill_uniform(4, 128, 2), 5)
    assert ix.last_path() == "simt"       # Q <= 4: CUDA-core scan
    ix.search(oracle_mod.fill_uniform(40, 128, 2), 5)
    assert ix.last_path() == "shadow"     # Q >= 5: tensor cores over the BF16 shadow
    q = oracle_mod.fill_uniform(40, 128, 2)
    gi, gs = ix.search(q, 500)
    assert ix.last_path() == "simt"       # k beyond the tensor paths
    ix.release()
    oi, os_ = oracle_mod.knn_exact64(rows, q, 500, "cosine")
    check_parity(rows, q, 500, "cosine", gi, gs, oi, os_)
