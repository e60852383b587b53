"""Parity at BASELINE.json's full sizes.  configs[1] (N=1M, d=1024, Q=64) is checked against the full fp64 oracle (the GPU
box has the cores for it); the 10M-row configs through size-independent properties: planted neighbours, exact
re-computation of every returned score from the rows read back, sortedness / uniqueness, agreement of the three
independent kernels (CUDA-core, 3xTF32 tensor, 1xTF32-filter + rescoring), and invariance under row sharding."""
import numpy as np
import pytest

from parity import check_parity, exact_scores_for

pytestmark = pytest.mark.gpu


def _basic_properties(idx, sc, metric):
    for q in range(idx.shape[0]):
        assert len(set(idx[q].tolist())) == idx.shape[1]
        d = np.diff(sc[q].astype(np.float64))
        assert (d >= -1e-7).all() if metric == "euclidean" else (d <= 1e-7).all()


def _recompute_scores(ix, queries, idx, sc, metric):
    """Every returned score equals the fp64 score of that row (rows read back from HBM) within 1e-4 relative."""
    for q in range(idx.shape[0]):
        rows = np.stack([ix.read_rows(int(r), 1)[0] for r in idx[q]])
        ex = exact_scores_for(rows, queries[q], np.arange(len(rows)), metric)
        assert np.allclose(sc[q], ex, rtol=1e-4, atol=1e-6), (q, sc[q], ex)


def test_config2_full_size_against_oracle(knn_lib, oracle_mod):
    # BASELINE.json configs[1]: N=1M d=1024 fp32 Q=64 k=10 cosine, every kernel, full fp64 oracle
    from nornicdb_b200.knn import KnnIndex
    n, d, Q, k = 1_000_000, 1024, 64, 10
    ix = KnnIndex(d, metric="cosine")
    ix.fill_uniform(n, 42)
    rows = oracle_mod.fill_uniform(n, d, 42)
    q = oracle_mod.fill_uniform(Q, d, 1337)
    oi, os_ = oracle_mod.knn_exact64(rows, q, k, "cosine")
    swaps = {}
    for path in ("shadow", "filter", "tensor", "simt"):
        ix.set_path(path)
        gi, gs = ix.search(q, k)
        assert ix.last_path() == path
        swaps[path] = check_parity(rows, q, k, "cosine", gi, gs, oi, os_)
    assert ix.debug_flags()[0] == 0
    ix.release()
    assert swaps["shadow"] == 0 and swaps["filter"] == 0 and swaps["simt"] == 0 and swaps["tensor"] <= 2, swaps


@pytest.mark.parametrize("metric,k", [("cosine", 10), ("dot", 100)])
def test_10m_rows_properties(knn_lib, oracle_mod, metric, k):
    # headline shape (N=10M d=1024 Q=64 k=10 cosine) and configs[2]'s k=100 inner product, 64 of its queries
    from nornicdb_b200.knn import KnnIndex
    n, d, Q = 10_000_000, 1024, 64
    ix = KnnIndex(d, metric=metric)
    ix.fill_uniform(n, 42)
    q = oracle_mod.fill_uniform(Q, d, 1337)
    # plant an (almost) exact copy of query j at a known row: it must come back first
    planted = {}
    for j in range(0, Q, 8):
        row = 1_000_003 * (j + 1) % n
        v = (q[j] * 1.5).astype(np.float32)
        ix.update_row(row, v)
        planted[j] = row
    ix.set_path("shadow")
    hi, hs = ix.search(q, k)
    fl = ix.debug_flags()
    assert fl[:2] == [0, 0] and fl[3] == 0, fl   # no retry stage was needed
    ix.set_path("filter")
    fi, fs = ix.search(q, k)
    assert ix.debug_flags()[:2] == [0, 0]
    # BF16-shadow filter and TF32 filter re-score the same survivors exactly: bit-identical results
    assert (hi == fi).all() and (hs == fs).all()
    ix.set_path("simt")
    si, ss = ix.search(q[:8], k)
    _basic_properties(fi, fs, metric)
    for j, row in planted.items():
        assert fi[j, 0] == row
        if metric == "cosine":
            assert abs(fs[j, 0] - 1.0) < 1e-5
    # two independent kernels agree on every index (filter results are exact fp32 re-scores)
    assert (fi[:8] == si).all()
    assert np.allclose(fs[:8], ss, rtol=2e-6, atol=1e-6)
    _recompute_scores(ix, q[:4], fi[:4], fs[:4], metric)
    if k <= 10:
        ix.set_path("tensor")
        ti, ts = ix.search(q, k)
        same = (ti == fi).all(axis=1)
        assert same.sum() >= Q - 2  # 3xTF32 may swap a boundary pair
        assert np.allclose(ts, fs, rtol=1e-4, atol=1e-6)
    ix.release()


def test_row_sharding_invariance_full_size(knn_lib, oracle_mod):
    # SURVEY.md §8e: the result must not depend on how rows are partitioned (4 shards of 2.5M rows vs one index)
    import torch
    from nornicdb_b200.knn import KnnIndex, merge_keys_device
    n, d, Q, k, G = 10_000_000, 1024, 64, 10, 4
    q = oracle_mod.fill_uniform(Q, d, 1337)
    qd = torch.from_numpy(q).cuda()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        full = KnnIndex(d, metric="cosine")
        full.fill_uniform(n, 42)
        oi = torch.empty((Q, k), dtype=torch.int32, device="cuda")
        os_ = torch.empty((Q, k), dtype=torch.float32, device="cuda")
        full.search_device(qd.data_ptr(), Q, k, oi.data_ptr(), os_.data_ptr(), st.cuda_stream)
        st.synchronize()
        full.release()
        keys = torch.empty((G, Q, k), dtype=torch.int64, device="cuda")
        shards = []
        for g in range(G):
            s = KnnIndex(d, metric="cosine")
            s.set_row_base(g * n // G)
            s.fill_uniform(n // G, 42)
            s.search_keys_device(qd.data_ptr(), Q, k, keys[g].data_ptr(), st.cuda_stream)
            shards.append(s)
        mi = torch.empty((Q, k), dtype=torch.int32, device="cuda")
        ms = torch.empty((Q, k), dtype=torch.float32, device="cuda")
        merge_keys_device(0, keys.data_ptr(), G, Q, k, "cosine", mi.data_ptr(), ms.data_ptr(), st.cuda_stream)
        st.synchronize()
        for s in shards:
            s.release()
    assert (mi.cpu().numpy() == oi.cpu().numpy()).all()
    assert (ms.cpu().numpy() == os_.cpu().numpy()).all()


def test_config4_fp16_l2_full_size(knn_lib, oracle_mod):
    # BASELINE.json configs[3]: N=10M d=768 fp16 Q=1 k=10 L2 — fp64 oracle over all rows (one query)
    from nornicdb_b200.knn import KnnIndex
    n, d, k = 10_000_000, 768, 10
    ix = KnnIndex(d, metric="euclidean", dtype="f16")
    ix.fill_uniform(n, 42)
    q = oracle_mod.fill_uniform(1, d, 1337)
    gi, gs = ix.search(q, k)
    ix.release()
    best = None
    step = 2_000_000  # regenerate the corpus in slices: 15 GB of fp16 need not sit in host memory at once
    for lo in range(0, n, step):
        rows = oracle_mod.fill_uniform(step, d, 42, row_base=lo, dtype="f16")
        dist = oracle_mod.scores_exact64(rows, q[0], "euclidean")
        part = np.argpartition(dist, 4 * k)[: 4 * k]
        cand = [(dist[i], lo + int(i)) for i in part]
        best = sorted((best or []) + cand)[: 4 * k]
    want_idx = [r for _, r in best[:k]]
    want_dist = np.array([x for x, _ in best[:k]])
    assert gi[0].tolist() == want_idx
    assert np.allclose(gs[0], want_dist, rtol=1e-4)


def _torch_fp64_topk(n, d, q, k, metric, slice_rows, rows_of_slice):
    """Exact fp64 brute force at full size ON THE GPU (torch, fp64 matmul over row slices) — an arithmetic completely
    independent of the kernels under test.  rows_of_slice(lo, cnt) -> float32 cuda tensor [cnt, d].  Returns (idx [Q, k]
    int64 cpu, score [Q, k] float64 cpu) under the (score desc, row asc) / (distance asc, row asc) order."""
    import torch
    q64 = torch.from_numpy(np.asarray(q, dtype=np.float64)).cuda()
    qn = q64.norm(dim=1)
    best_s = best_i = None
    for lo in range(0, n, slice_rows):
        cnt = min(slice_rows, n - lo)
        x = rows_of_slice(lo, cnt).double()
        s = x @ q64.T  # [cnt, Q]
        if metric == "cosine":
            den = x.norm(dim=1)[:, None] * qn[None, :]
            s = torch.where(den > 0, s / den, torch.zeros_like(s))
        elif metric == "euclidean":
            s = -((x * x).sum(1)[:, None] + (q64 * q64).sum(1)[None, :] - 2.0 * s)
        kk = min(k + 8, cnt)
        v, i = torch.topk(s, kk, dim=0)  # [kk, Q]
        i = i + lo
        if best_s is None:
            best_s, best_i = v, i
        else:
            best_s, best_i = torch.cat([best_s, v]), torch.cat([best_i, i])
            keep = torch.topk(best_s, min(k + 8, best_s.shape[0]), dim=0).indices
            best_s, best_i = torch.gather(best_s, 0, keep), torch.gather(best_i, 0, keep)
        del x, s
    # final order: score desc, row asc
    bs, bi = best_s.T.cpu().numpy(), best_i.T.cpu().numpy()
    out_i = np.empty((bs.shape[0], k), dtype=np.int64)
    out_s = np.empty((bs.shape[0], k), dtype=np.float64)
    for r in range(bs.shape[0]):
        order = np.lexsort((bi[r], -bs[r]))[:k]
        out_i[r], out_s[r] = bi[r][order], bs[r][order]
    if metric == "euclidean":
        out_s = np.sqrt(np.maximum(-out_s, 0.0))
    return out_i, out_s


def test_config3_full_size_all_queries_fp64(knn_lib, oracle_mod):
    """BASELINE.json configs[2] at FULL size: N=10M d=1024 fp32, ALL 1024 queries, k=100, inner product (the 16-bit
    pass with 4 query groups per launch), against an fp64 brute force over all 10^7 x 1024 (row, query) pairs computed slice by slice with torch on the
    same GPU (round-1 VERDICT: only 64 of these queries had ever been checked)."""
    import torch
    from nornicdb_b200.knn import KnnIndex, fill_uniform_device
    n, d, Q, k = 10_000_000, 1024, 1024, 100
    ix = KnnIndex(d, metric="dot")
    ix.fill_uniform(n, 42)
    q = oracle_mod.fill_uniform(Q, d, 1337)
    gi, gs = ix.search(q, k)
    assert ix.last_path() == "shadow" and ix.debug_flags()[0] == 0

    def rows_of_slice(lo, cnt):
        x = torch.empty((cnt, d), dtype=torch.float32, device="cuda")
        fill_uniform_device(0, x.data_ptr(), cnt, d, 42, lo, 0)  # the same counter-based generator as the index
        torch.cuda.synchronize()
        return x

    oi, os_ = _torch_fp64_topk(n, d, q, k, "dot", 500_000, rows_of_slice)
    swaps = check_parity(lambda idx: np.stack([ix.read_rows(int(r), 1)[0] for r in idx]), q, k, "dot", gi, gs, oi, os_)
    ix.release()
    assert swaps <= 8, swaps  # boundary swaps (fp64 scores closer than fp32 summation noise) are counted, not hidden


def test_clustered_corpus_1m_rows_fp64(knn_lib, oracle_mod):
    """SURVEY.md 8(d)'s Gaussian-mixture corpus (1000 centres, sigma 0.1) at N=1M d=1024: near-ties by construction.  Rows
    are generated on the device, read back, and checked against the fp64 torch brute force; the 16-bit filter must not
    need its retry stage."""
    import torch
    from nornicdb_b200.knn import KnnIndex
    n, d, Q, k = 1_000_000, 1024, 64, 10
    ix = KnnIndex(d, metric="cosine")
    ix.fill_clustered(n, 42, n_centres=1000, sigma=0.1)
    host = np.concatenate([ix.read_rows(lo, 100_000) for lo in range(0, n, 100_000)])
    rng = np.random.default_rng(7)
    q = np.concatenate([oracle_mod.fill_uniform(Q // 2, d, 1337),                                   # unrelated directions
                        host[rng.integers(0, n, Q // 2)] + rng.standard_normal((Q // 2, d)).astype(np.float32) * 0.05])  # cluster members
    q = np.ascontiguousarray(q, dtype=np.float32)
    res = {}
    for path in ("shadow", "filter"):
        ix.set_path(path)
        res[path] = ix.search(q, k)
        assert ix.debug_flags()[0] == 0
    counters = ix.debug_counters()
    ix.release()
    oi, os_ = _torch_fp64_topk(n, d, q, k, "cosine", 250_000, lambda lo, cnt: torch.from_numpy(host[lo:lo + cnt]).cuda())
    for path, (gi, gs) in res.items():
        check_parity(host, q, k, "cosine", gi, gs, oi, os_, swap_eps=5e-6)
    assert (res["shadow"][0] == res["filter"][0]).all()
    assert counters["bf16_stage_retries"] == 0, counters
