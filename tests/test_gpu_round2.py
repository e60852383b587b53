"""GPU parity tests of the round-2 features, all through the C ABI against the CPU oracle:
sampled initial thresholds, score floor inside the kernels, NaN / Inf rows on every path, fp16 / bf16 corpora on the
tensor cores, attached rows + refresh_shadow, the clustered (near-tie) corpus, best-of-chunks group search, the
peer-memory exchange, big survivor lists in the finish step."""
import numpy as np
import pytest

from parity import check_parity, exact_scores_for

pytestmark = pytest.mark.gpu

PATHS_F32 = ["simt", "tensor", "filter", "shadow"]


def _index(rows, metric, dtype="f32", path="auto"):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex(rows.shape[1], metric=metric, dtype=dtype)
    ix.upload(rows)
    ix.set_path(path)
    return ix


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
@pytest.mark.parametrize("path", ["filter", "shadow"])
def test_sampled_initial_threshold_matches_oracle(knn_lib, oracle_mod, metric, path):
    """n >= 4096 and Q <= 128: the prep kernel seeds every query's threshold from a sample (no flood tiles)."""
    n, d, Q, k = 150_000, 128, 37, 10
    rows = oracle_mod.fill_uniform(n, d, 42)
    q = oracle_mod.fill_uniform(Q, d, 77)
    ix = _index(rows, metric, path=path)
    gi, gs = ix.search(q, k)
    assert ix.last_path() == path
    fl = ix.debug_flags()
    ix.release()
    assert fl[0] == 0 and fl[3] == 0, fl  # no overflow, no retry on uniform data
    oi, os_ = oracle_mod.knn_exact64(rows, q, k, metric)
    check_parity(rows, q, k, metric, gi, gs, oi, os_)


def test_sampled_threshold_with_row_mask_and_large_k(knn_lib, oracle_mod):
    n, d = 40_000, 64
    rows = oracle_mod.fill_uniform(n, d, 5)
    q = oracle_mod.fill_uniform(9, d, 6)
    keep = np.zeros(n, dtype=bool)
    keep[::3] = True
    ix = _index(rows, "cosine", path="shadow")
    ix.set_row_mask(keep)
    for k in (1, 10, 150):
        gi, gs = ix.search(q, k)
        sub = np.where(keep)[0]
        oi, os_ = oracle_mod.knn_exact64(rows[sub], q, k, "cosine")
        check_parity(rows, q, k, "cosine", gi, gs, sub[oi], os_)
    ix.release()


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
@pytest.mark.parametrize("path", PATHS_F32)
def test_score_floor_inside_kernels(knn_lib, oracle_mod, metric, path):
    """nk_index_set_min_score = VectorIndex.Search's minSimilarity cut (vector_index.go:339-352), evaluated on the device."""
    if path == "tensor" and metric == "euclidean":
        pytest.skip("3xTF32 exact kernel has no euclidean mode")
    n, d, Q, k = 30_000, 128, 11, 20
    rows = oracle_mod.fill_uniform(n, d, 8)
    q = oracle_mod.fill_uniform(Q, d, 9)
    oi, os_ = oracle_mod.knn_exact64(rows, q, k, metric)
    # a floor that cuts most queries' lists somewhere in the middle
    floor = float(np.median(os_[:, k // 2]))
    ix = _index(rows, metric, path=path)
    ix.set_min_score(floor)
    gi, gs = ix.search(q, k)
    ix.set_min_score(None)
    gi_all, _ = ix.search(q, k)
    ix.release()
    assert (gi_all == oi).all()
    for qi in range(Q):
        ok = os_[qi] <= floor if metric == "euclidean" else os_[qi] >= floor
        # rows within fp32 noise of the floor may fall on either side
        noise = np.abs(os_[qi] - floor) <= 2e-6 * max(1.0, abs(floor))
        want = oi[qi][ok & ~noise]
        got = gi[qi][gi[qi] != 0xFFFFFFFF]
        must = set(want.tolist())
        may = set(oi[qi][ok | noise].tolist())
        assert must <= set(got.tolist()) <= may, (metric, path, qi, got, want)
        assert (gi[qi][len(got):] == 0xFFFFFFFF).all()  # unused slots are marked


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
@pytest.mark.parametrize("path", PATHS_F32)
@pytest.mark.parametrize("Q", [3, 16])
def test_nan_and_inf_rows_on_every_path(knn_lib, oracle_mod, metric, path, Q):
    """Rows holding NaN (score NaN -> ranked last) must not disturb the other rows' ranking on any path (advisor finding:
    the TF32 filter used to return empty results once one row's |x|^2 was NaN)."""
    if path == "tensor" and metric == "euclidean":
        pytest.skip("3xTF32 exact kernel has no euclidean mode")
    n, d, k = 6000, 64, 10
    rows = oracle_mod.fill_uniform(n, d, 21)
    q = oracle_mod.fill_uniform(Q, d, 22)
    bad = np.array([0, 17, 255, 256, 3000, 5999])
    rows[bad[:4], 5] = np.nan
    if metric != "dot":
        rows[bad[4:], 7] = np.inf  # cosine: inf/inf = NaN; euclidean: distance inf -> last
    else:
        rows[bad[4:], 7] = np.nan  # dot with +inf would legitimately rank first
    good = np.setdiff1d(np.arange(n), bad)
    ix = _index(rows, metric, path=path)
    gi, gs = ix.search(q, k)
    fl = ix.debug_flags()
    ix.release()
    assert fl[0] == 0
    oi, os_ = oracle_mod.knn_exact64(rows[good], q, k, metric)
    check_parity(rows, q, k, metric, gi, gs, good[oi], os_)


def test_k_or_more_nan_rows_fall_back_to_exact(knn_lib, oracle_mod):
    """k or more NaN rows give the filters k undecidable (+inf) bounds: they must escalate to the exact stage instead of
    dropping every finite row."""
    n, d, k = 5000, 64, 5
    rows = oracle_mod.fill_uniform(n, d, 31)
    q = oracle_mod.fill_uniform(8, d, 32)
    bad = np.arange(100, 120)
    rows[bad, 3] = np.nan
    good = np.setdiff1d(np.arange(n), bad)
    for path in ("filter", "shadow"):
        for metric in ("cosine", "dot", "euclidean"):
            ix = _index(rows, metric, path=path)
            gi, gs = ix.search(q, k)
            ix.release()
            oi, os_ = oracle_mod.knn_exact64(rows[good], q, k, metric)
            check_parity(rows, q, k, metric, gi, gs, good[oi], os_)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
@pytest.mark.parametrize("Q,d", [(1, 768), (3, 50), (16, 768), (64, 256), (130, 128)])
def test_16bit_corpora_cuda_and_tensor_paths(knn_lib, oracle_mod, metric, dtype, Q, d):
    """fp16 / bf16 corpora: CUDA-core scan for Q <= 4, the 16-bit tensor pass IN PLACE (no shadow) from 5 queries on."""
    from nornicdb_b200.knn import KnnIndex, from_bf16_bits, to_bf16_bits
    n, k = 20_000, 10
    f32 = oracle_mod.fill_uniform(n, d, 51)
    if dtype == "f16":
        rows = f32.astype(np.float16)
        exact = rows  # the oracle widens fp16 exactly
    else:
        rows = to_bf16_bits(f32)
        exact = from_bf16_bits(rows)  # exactly widened bf16 values
    q = oracle_mod.fill_uniform(Q, d, 52)
    ix = KnnIndex(d, metric=metric, dtype=dtype)
    ix.upload(rows)
    gi, gs = ix.search(q, k)
    path = ix.last_path()
    back = ix.read_rows(0, 4)
    ix.release()
    assert (np.asarray(back).view(np.uint16) == np.asarray(rows[:4]).view(np.uint16)).all()
    assert path == ("shadow" if Q >= 5 and d % 8 == 0 else "simt"), path
    oi, os_ = oracle_mod.knn_exact64(exact, q, k, metric)
    check_parity(exact, q, k, metric, gi, gs, oi, os_)


def test_bf16_upload_from_f32_converts_on_device(knn_lib, oracle_mod):
    from nornicdb_b200.knn import KnnIndex, to_bf16_bits
    n, d = 3000, 96
    f32 = oracle_mod.fill_uniform(n, d, 61)
    ix = KnnIndex(d, metric="cosine", dtype="bf16")
    ix.upload_from_f32(f32)
    got = ix.read_rows(0, n)
    ix.release()
    assert (got == to_bf16_bits(f32)).all()


# ---------------------------------------------------------------------------------------------------------------------
def test_attached_rows_get_the_shadow_path_after_refresh(knn_lib, oracle_mod):
    """INTEGRATION.md step 2: caller-owned device rows (cuda.Buffer) + nk_index_refresh_shadow -> the fast filter path."""
    from nornicdb_b200 import cuda
    from nornicdb_b200.knn import KnnIndex
    n, d, Q, k = 30_000, 128, 16, 10
    rows = oracle_mod.fill_uniform(n, d, 71)
    q = oracle_mod.fill_uniform(Q, d, 72)
    dev = cuda.NewDevice(0)
    buf = dev.NewBuffer(rows.reshape(-1))
    ix = KnnIndex(d, metric="cosine")
    ix.attach_device_rows(buf.DataPtr(), n)
    gi0, gs0 = ix.search(q, k)
    assert ix.last_path() == "filter"  # no shadow yet: TF32 filter over the fp32 rows
    dev.NormalizeVectors(buf, n, d)    # the reference normalises its buffer in place (gpu.go:2100-2106)
    ix.refresh_shadow()
    gi, gs = ix.search(q, k)
    assert ix.last_path() == "shadow"
    ix.release()
    buf.Release()
    dev.Release()
    oi, os_ = oracle_mod.knn_exact64(rows, q, k, "cosine")  # cosine is scale-invariant: same ranking before / after
    check_parity(rows, q, k, "cosine", gi0, gs0, oi, os_)
    check_parity(rows, q, k, "cosine", gi, gs, oi, os_, swap_eps=5e-6)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_clustered_corpus_parity_and_retry_counters(knn_lib, oracle_mod, metric):
    """SURVEY.md 8(d)'s Gaussian mixture (near-ties): generated on the device, read back for the fp64 oracle."""
    from nornicdb_b200.knn import KnnIndex
    n, d, Q, k = 120_000, 256, 32, 10
    ix = KnnIndex(d, metric=metric)
    ix.fill_clustered(n, 4242, n_centres=40, sigma=0.1)
    rows = ix.read_rows(0, n)
    # queries: fresh members of some clusters = corpus rows plus a little noise
    rng = np.random.default_rng(3)
    q = (rows[rng.integers(0, n, Q)] + rng.standard_normal((Q, d)).astype(np.float32) * 0.05).astype(np.float32)
    res = {}
    for path in ("simt", "filter", "shadow"):
        ix.set_path(path)
        res[path] = ix.search(q, k)
    counters = ix.debug_counters()
    assert ix.debug_flags()[0] == 0
    ix.release()
    assert counters["bf16_stage_retries"] >= 0
    oi, os_ = oracle_mod.knn_exact64(rows, q, k, metric)
    for path, (gi, gs) in res.items():
        check_parity(rows, q, k, metric, gi, gs, oi, os_, swap_eps=5e-6)
    assert (res["shadow"][0] == res["filter"][0]).all()  # both re-score the same survivors exactly


def test_clustered_unit_norm_mode_rows_are_normalised(knn_lib):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex(128, metric="cosine")
    ix.fill_clustered(2000, 7, n_centres=20, sigma=0.15, unit_norm=True)  # cmd/kmeans-test-data's recipe
    rows = ix.read_rows(0, 2000)
    ix.release()
    assert np.allclose(np.linalg.norm(rows.astype(np.float64), axis=1), 1.0, atol=1e-5)


def test_finish_handles_thousands_of_rows_inside_the_margin(knn_lib, oracle_mod):
    """Near-duplicates: several thousand rows inside the 16-bit margin of the k-th bound.  The finish step re-scores them
    in rounds instead of overflowing (FINISH_CAP used to force a retry)."""
    from nornicdb_b200.knn import KnnIndex
    rng = np.random.default_rng(11)
    n, d, k = 300_000, 64, 10
    base = oracle_mod.fill_uniform(1, d, 9)[0]
    rows = oracle_mod.fill_uniform(n, d, 10)
    dup = rng.choice(n, 9000, replace=False)
    rows[dup] = base[None, :] + rng.standard_normal((9000, d)).astype(np.float32) * 2e-3
    q = (base[None, :] + rng.standard_normal((6, d)).astype(np.float32) * 1e-3).astype(np.float32)
    ix = KnnIndex(d, metric="cosine")
    ix.upload(rows)
    ix.set_path("shadow")
    gi, gs = ix.search(q, k)
    ix.release()
    oi, os_ = oracle_mod.knn_exact64(rows, q, k, "cosine")
    check_parity(rows, q, k, "cosine", gi, gs, oi, os_, swap_eps=5e-6)


# ---------------------------------------------------------------------------------------------------------------------
def _group_reference(rows, q, group, metric, keep=None, floor=None):
    s = exact_scores_for(rows, q, np.arange(len(rows)), metric)  # euclidean: distance
    key = -s if metric == "euclidean" else s
    best = {}
    for r in range(len(rows)):
        if keep is not None and not keep[r]:
            continue
        if floor is not None and key[r] < floor:
            continue
        g = int(group[r])
        if g not in best or key[r] > key[best[g]]:
            best[g] = r
    order = sorted(best.items(), key=lambda t: (-key[t[1]], t[1]))
    return [g for g, _ in order], [r for _, r in order], [s[r] for _, r in order]


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
def test_group_search_best_of_chunks(knn_lib, oracle_mod, metric):
    """db.index.vector.queryNodes: per-node best-of-chunks (call_vector.go:217-247) as a device segment-max."""
    rng = np.random.default_rng(5)
    n, d, nodes, k = 12_000, 96, 900, 25
    rows = oracle_mod.fill_uniform(n, d, 81)
    group = rng.integers(0, nodes, n).astype(np.uint32)
    q = oracle_mod.fill_uniform(1, d, 82)[0]
    ix = _index(rows, metric)
    ix.set_row_groups(group, nodes)
    g, r, s = ix.search_groups(q, k)
    wg, wr, ws = _group_reference(rows, q, group, metric)
    assert g.tolist() == wg[:k] and r.tolist() == wr[:k]
    assert np.allclose(s, ws[:k], rtol=1e-4, atol=1e-6)
    # label filter (row mask) + "bestScore >= 0" (score floor 0)
    keep = rng.random(n) < 0.3
    ix.set_row_mask(keep)
    ix.set_row_groups(group, nodes)  # the mask call does not clear groups, a row-count change would
    if metric != "euclidean":
        ix.set_min_score(0.0)
    g, r, s = ix.search_groups(q, k)
    wg, wr, ws = _group_reference(rows, q, group, metric, keep=keep, floor=0.0 if metric != "euclidean" else None)
    assert g.tolist() == wg[:k] and r.tolist() == wr[:k]
    # fewer admissible nodes than k
    ix.set_row_mask(np.arange(n) < 3)
    ix.set_row_groups(group, nodes)
    ix.set_min_score(None)
    g, r, s = ix.search_groups(q, k)
    wg, wr, ws = _group_reference(rows, q, group, metric, keep=np.arange(n) < 3)
    assert g.tolist() == wg and r.tolist() == wr
    ix.release()


# ---------------------------------------------------------------------------------------------------------------------
def _sharded_search(world, devices, rows, q, k, metric):
    """`world` single-device indexes (one rank each) + the peer-memory exchange; returns every rank's result."""
    import torch
    from nornicdb_b200.knn import Comm, KnnIndex
    from nornicdb_b200.sharding import shard_range
    n, d = rows.shape
    Q = q.shape[0]
    ixs, comms, outs, qd = [], [], [], []
    for r in range(world):
        lo, hi = shard_range(n, world, r)
        ix = KnnIndex(d, metric=metric, devices=(devices[r],))
        ix.set_row_base(lo)
        ix.upload(rows[lo:hi])
        ixs.append(ix)
        comms.append(Comm(devices[r], r, world, Q * k * 8))
        dev = torch.device("cuda", devices[r])
        qd.append(torch.from_numpy(q).to(dev))
        outs.append((torch.empty((Q, k), dtype=torch.int32, device=dev), torch.empty((Q, k), dtype=torch.float32, device=dev)))
    Comm.connect_local(comms)
    results = []
    for rep in range(3):  # several epochs: both parities of the slots get reused
        for r in range(world):
            ixs[r].search_sharded_device(comms[r], qd[r].data_ptr(), Q, k, outs[r][0].data_ptr(), outs[r][1].data_ptr())
        for r in range(world):
            comms[r].status()
            ixs[r].status()
    for r in range(world):
        torch.cuda.synchronize(devices[r])
        results.append((outs[r][0].cpu().numpy().view(np.uint32), outs[r][1].cpu().numpy()))
        comms[r].release()
        ixs[r].release()
    return results


@pytest.mark.parametrize("metric,near_tie", [
    pytest.param(metric, near_tie, id=metric + ("-near-tie" if near_tie else ""))
    for near_tie in (False, True) for metric in ("cosine", "dot", "euclidean") if near_tie or metric != "dot"])
def test_exchange_two_ranks_on_one_device(knn_lib, oracle_mod, metric, near_tie):
    """The exchange kernels (peer push + fused wait/merge/decode) with both ranks living on cuda:0, also on the near-tie
    corpus of test_gpu_tensor.py, where each rank's filter meets thousands of rows inside its margins."""
    if near_tie:
        from test_gpu_filtered import _near_tie_corpus
        rows, q = _near_tie_corpus(oracle_mod, 20_000, 1e-5, 0)
    else:
        rows = oracle_mod.fill_uniform(50_000, 128, 91)
        q = oracle_mod.fill_uniform(16, 128, 92)
    k = 10
    res = _sharded_search(2, (0, 0), rows, q, k, metric)
    oi, os_ = oracle_mod.knn_exact64(rows, q, k, metric)
    for gi, gs in res:
        check_parity(rows, q, k, metric, gi, gs, oi, os_, swap_eps=5e-6 if near_tie else 2e-6)
    assert (res[0][0] == res[1][0]).all()


def test_exchange_across_gpus_in_one_process(knn_lib, oracle_mod):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    world = min(torch.cuda.device_count(), 4)
    n, d, Q, k = 80_000, 128, 16, 10
    rows = oracle_mod.fill_uniform(n, d, 93)
    q = oracle_mod.fill_uniform(Q, d, 94)
    res = _sharded_search(world, tuple(range(world)), rows, q, k, "cosine")
    oi, os_ = oracle_mod.knn_exact64(rows, q, k, "cosine")
    for gi, gs in res:
        check_parity(rows, q, k, "cosine", gi, gs, oi, os_)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "dot", "euclidean"])
@pytest.mark.parametrize("Q,k", [(256, 10), (300, 10), (520, 100), (1024, 10)])
def test_large_batches_on_cta_pairs(knn_lib, oracle_mod, metric, Q, k):
    """Q >= 256 (the name dates from the Blackwell CTA-pair kernel; the test ids are kept so that the large-batch cases
    stay comparable across versions): the 16-bit pass runs in blocks of 128 query columns with 2 / 4 query groups per
    launch, the remainder in a 64-column launch; results must match the fp64 oracle like every other path."""
    n, d = 70_000, 128
    rows = oracle_mod.fill_uniform(n, d, 101)
    q = oracle_mod.fill_uniform(Q, d, 102)
    ix = _index(rows, metric, path="shadow")
    gi, gs = ix.search(q, k)
    fl = ix.debug_flags()
    ix.release()
    assert fl[0] == 0
    oi, os_ = oracle_mod.knn_exact64(rows, q, k, metric)
    check_parity(rows, q, k, metric, gi, gs, oi, os_)


def test_cta_pairs_fp16_corpus_and_ragged_rows(knn_lib, oracle_mod):
    """fp16 corpus, Q=512, a row count that is not a multiple of the 256-row tile, on the 16-bit pass (name: see above)."""
    from nornicdb_b200.knn import KnnIndex
    n, d, Q, k = 33_333, 256, 512, 10  # n not a multiple of the 256-row tile
    rows = oracle_mod.fill_uniform(n, d, 103).astype(np.float16)
    q = oracle_mod.fill_uniform(Q, d, 104)
    ix = KnnIndex(d, metric="cosine", dtype="f16")
    ix.upload(rows)
    gi, gs = ix.search(q, k)
    assert ix.last_path() == "shadow"
    ix.release()
    oi, os_ = oracle_mod.knn_exact64(rows, q, k, "cosine")
    check_parity(rows, q, k, "cosine", gi, gs, oi, os_)


def test_16bit_index_maintenance_keeps_norms_in_step(knn_lib, oracle_mod):
    """append / update_row / remove_swap on fp16 and bf16 indexes: the per-row |x|^2 array of the in-place tensor pass must
    follow every mutation (a stale norm would silently mis-rank under cosine / euclidean), and the device generator of bf16
    rows must equal round-to-nearest-even of the fp32 stream."""
    from nornicdb_b200.knn import KnnIndex, from_bf16_bits, to_bf16_bits
    d, k = 64, 8
    base = oracle_mod.fill_uniform(6000, d, 111)
    extra = oracle_mod.fill_uniform(3000, d, 112) * 3.0
    q = oracle_mod.fill_uniform(12, d, 113)
    for dtype in ("f16", "bf16"):
        conv = (lambda a: a.astype(np.float16)) if dtype == "f16" else to_bf16_bits
        wide = (lambda a: a.astype(np.float32)) if dtype == "f16" else from_bf16_bits
        for metric in ("cosine", "euclidean"):
            ix = KnnIndex(d, metric=metric, dtype=dtype)
            ix.upload(conv(base))
            ix.append(conv(extra))                      # norms of the appended rows
            ix.update_row(17, conv(extra[5] * 2.0))     # one row rewritten in place
            ix.remove_swap(100)                         # last row moves into slot 100
            host = np.concatenate([wide(conv(base)), wide(conv(extra))])
            host[17] = wide(conv(extra[5] * 2.0))
            host[100] = host[-1]
            host = host[:-1]
            gi, gs = ix.search(q, k)                    # Q >= 5: the 16-bit tensor pass
            assert ix.last_path() == "shadow"
            ix.release()
            oi, os_ = oracle_mod.knn_exact64(host, q, k, metric)
            check_parity(host, q, k, metric, gi, gs, oi, os_)
    ix = KnnIndex(d, metric="dot", dtype="bf16")
    ix.fill_uniform(4000, 42)
    got = ix.read_rows(0, 4000)
    ix.release()
    assert (got == to_bf16_bits(oracle_mod.fill_uniform(4000, d, 42))).all()
