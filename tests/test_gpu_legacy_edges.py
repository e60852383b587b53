"""The legacy boundary (include/nornic_knn.h part 1) at special values and size edges, against the reference's own arithmetic
(tests/legacy_model.py), through the mirror of its Go API (nornicdb_b200.cuda).

  * cuda_topk equals topk_model bit for bit, indices and score bits, on every mix of special scores at the sizes where the
    launch changes (one interval, two per SM, the 32-bit row range) and the k where the passes change (NK_MAX_K, and
    every multiple of it up to NK_MAX_K_TOTAL), with admissible counts and runs of ties on both sides of each.
  * cuda_compute_norms is within (d + 2) u of the fp64 norm for rows from 1e-30 to FLT_MAX / sqrt(d), and inf / NaN exactly
    where the model is; cuda_normalize_vectors equals normalize_model with the library's own norms, bit for bit.
  * cuda_cosine_similarity is within the a-priori bound of a d-term fp32 dot product of the fp64 value."""
import numpy as np
import pytest

import legacy_model as lm

pytestmark = pytest.mark.gpu

F32 = np.float32


@pytest.fixture(scope="module")
def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _topk_sizes(num_sms):
    two_per_sm = 2 * num_sms * lm.TOPK_IV  # from here on every CTA of the grid takes a second interval
    return {"1": 1, "2": 2, "iv-1": lm.TOPK_IV - 1, "iv": lm.TOPK_IV, "iv+1": lm.TOPK_IV + 1,
            "2sm_iv-1": two_per_sm - 1, "2sm_iv+1": two_per_sm + 1, "300001": 300001}


K_EDGES = (1, 2, 7, lm.NK_MAX_K, lm.NK_MAX_K + 1, 2 * lm.NK_MAX_K, 2 * lm.NK_MAX_K + 1, lm.NK_MAX_K_TOTAL)


def _ks(n):
    """the k edges that fit in n, and k = n and k = n + 1 (clamped to n) where n itself is a k the call serves"""
    return sorted({k for k in K_EDGES if k <= n} | ({n, n + 1} if n <= lm.NK_MAX_K_TOTAL else set()))


def _assert_topk(dev, buf, s, n, ks, what):
    """cuda_topk over the first n scores of buf (which hold s) equals topk_model for every k in ks"""
    want_i, want_s = lm.topk_model(s[:n], max(ks))  # a shorter k is a prefix of it
    for k in ks:
        idx, sc = dev.TopK(buf, n, k)
        kk = min(k, n)
        wi, ws = want_i[:kk], want_s[:kk]
        assert idx.shape == (k,) and sc.shape == (k,)
        bad = np.flatnonzero((idx[:kk] != wi) | (sc[:kk].view(np.uint32) != ws.view(np.uint32)))
        assert bad.size == 0, (what, n, k, bad[:5], idx[bad[:5]], wi[bad[:5]], sc[bad[:5]], ws[bad[:5]])


@pytest.mark.parametrize("mix", lm.MIXES)
@pytest.mark.parametrize("size", ["1", "2", "iv-1", "iv", "iv+1", "2sm_iv-1", "2sm_iv+1", "300001"])
def test_topk_special_scores(gpu_device, num_sms, size, mix):
    n = _topk_sizes(num_sms)[size]
    s = lm.special_scores(n, mix, 7)
    buf = gpu_device.NewBuffer(s)
    try:
        _assert_topk(gpu_device, buf, s, n, _ks(n), mix)
    finally:
        buf.Release()


@pytest.mark.parametrize("n", [5000, 300001])
def test_topk_admissible_count_at_pass_edges(gpu_device, n):
    """exactly count admissible scores for counts on both sides of k and of each pass boundary: a pass that runs dry
    leaves padding, never stale keys of an earlier pass"""
    M = lm.NK_MAX_K
    for k in (7, M, M + 1, 2 * M, 2 * M + 1):
        for count in sorted({k - 1, k, k + 1, M - 1, M, M + 1} & set(range(0, min(n, 3 * M)))):
            s = lm.short_admissible(n, count, k)
            buf = gpu_device.NewBuffer(s)
            try:
                _assert_topk(gpu_device, buf, s, n, [k], f"admissible={count}")
            finally:
                buf.Release()


@pytest.mark.parametrize("zeros", [False, True], ids=["ties", "signed_zeros"])
def test_topk_runs_straddle_k(gpu_device, num_sms, zeros):
    """runs of equal scores (the last of them -0.0 / +0.0) across rank k and across every multiple of NK_MAX_K below it"""
    M = lm.NK_MAX_K
    n = 2 * num_sms * lm.TOPK_IV + 1
    cases = [([7], 5), ([2 * M], 3001), ([4 * M], 4001), ([M, 2 * M, 3 * M, 4 * M], 1001), ([M * m for m in range(1, 9)], 301)]
    for edges, run in cases:
        s = lm.straddle(n, edges, run, 3, zeros=zeros)
        buf = gpu_device.NewBuffer(s)
        try:
            e = edges[-1]
            _assert_topk(gpu_device, buf, s, n, sorted({e - 1, e, e + 1, edges[0], e + run}), (edges, run))
        finally:
            buf.Release()


def test_topk_refuses_k_above_total(gpu_device):
    from nornicdb_b200 import cuda
    n = lm.NK_MAX_K_TOTAL + 10
    buf = gpu_device.NewBuffer(np.zeros(n, F32))
    try:
        with pytest.raises(cuda.ErrKernelExecution, match="exceeds NK_MAX_K_TOTAL"):
            gpu_device.TopK(buf, n, lm.NK_MAX_K_TOTAL + 1)
        idx, sc = gpu_device.TopK(buf, n, lm.NK_MAX_K_TOTAL)  # the largest k still served, all ties: rows in order
        assert (idx == np.arange(lm.NK_MAX_K_TOTAL)).all() and (sc == 0).all()
    finally:
        buf.Release()


def _device_view(buf, n):
    """a torch view of the first n floats of a legacy device buffer"""
    import torch

    class _Iface:
        __cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (buf.DataPtr(), False), "version": 3}

    return torch.as_tensor(_Iface(), device="cuda:0")


def test_topk_near_the_32bit_row_limit(gpu_device, knn_lib):
    """n = 2^32 - 1 and 2^32 - 1023: every interval is launched and rows >= 2^31 decode to their own index.  The scores
    are the shared uniform stream mapped into [-2, -1], with planted maxima (a tie among them), a NaN, and -0.0 / +0.0
    above everything else, near index 2^31 and near the end."""
    import torch
    N = 2 ** 32 - 1
    if torch.cuda.mem_get_info(0)[0] < N * 4 + (1 << 30):
        pytest.skip("needs about 18 GB of free device memory")
    buf = gpu_device.NewEmptyBuffer(N)
    try:
        assert knn_lib.nk_fill_uniform_device(0, buf.DataPtr(), N, 1, 5, 0, None) == 0
        torch.cuda.synchronize()
        t = _device_view(buf, N)
        t.abs_().add_(1.0).neg_()  # [-2, -1]: below every planted score
        h = 2 ** 31
        end = 2 ** 32 - 1024  # the last row of the shorter array
        plant = {h - 3: 3.0, end - 5: 3.0, h + 11: 2.5, end: 2.0, h + 1: np.nan, end - 1: np.nan,
                 h - 1: -0.0, h + 2: 0.0, end - 7: -0.0, N - 1: 4.0, N - 500: np.nan}
        for i, v in plant.items():
            t[i] = torch.tensor(v, dtype=torch.float32)
        torch.cuda.synchronize()
        for n in (N, 2 ** 32 - 1023):
            live = {i: F32(v) for i, v in plant.items() if i < n and not np.isnan(v)}
            order = sorted(live, key=lambda i: (-float(live[i]), i))
            idx, sc = gpu_device.TopK(buf, n, len(order))
            assert idx.tolist() == order, (n, idx, order)
            assert sc.view(np.uint32).tolist() == [live[i].view(np.uint32) for i in order], (n, sc)
    finally:
        buf.Release()


# ---- norms, normalize, cosine -------------------------------------------------------------------------------------------
DIMS = (1, 2, 3, 4, 5, 31, 32, 33, 127, 128, 129, 4095, 4096, 4097)
SCALES = (1e-30, 1e-20, 1.0, 1e19, 1e25, None)  # None: FLT_MAX / sqrt(d)


def _scaled_rows(n, d, seed):
    """row r: a normal row scaled so its largest |x| is SCALES[r % 6] (FLT_MAX / sqrt(d) for None); then every 9th row from
    row 6 has one inf element, from row 7 one NaN, from row 8 is zero"""
    rng = np.random.default_rng([seed, n, d])
    x = rng.standard_normal((n, d))
    top = (np.finfo(F32).max / np.sqrt(d)) * (1 - 1e-6)
    scale = np.array([top if s is None else s for s in SCALES])[np.arange(n) % len(SCALES)]
    x = (x * (scale / np.abs(x).max(axis=1))[:, None]).astype(F32)
    col = rng.integers(0, d, n)
    for r in range(6, n, 9):
        x[r, col[r]] = np.inf
    for r in range(7, n, 9):
        x[r, col[r]] = np.nan
    x[8::9] = 0.0
    return x


def _row_counts(num_sms):
    return (37, lm.warp_sweep(num_sms) + 1)  # below one sweep of the row kernels' grid, and one row into a second sweep


@pytest.mark.parametrize("d", DIMS)
def test_norms_and_normalize(gpu_device, num_sms, d):
    for n in _row_counts(num_sms):
        x = _scaled_rows(n, d, 1)
        v, nb = gpu_device.NewBuffer(x), gpu_device.NewEmptyBuffer(n)
        try:
            gpu_device.ComputeNorms(v, nb, n, d)
            got = nb.ReadFloat32(n)
            want = lm.nrm2_model(x)
            fin = np.isfinite(want)
            assert (np.isnan(got) == np.isnan(want)).all() and (np.isinf(got) == np.isinf(want)).all(), (d, n)
            err = np.abs(got[fin].astype(np.float64) - want[fin].astype(np.float64))
            bound = (d + 2) * lm.U * want[fin].astype(np.float64)
            assert (err <= bound).all(), (d, n, np.flatnonzero(fin)[err > bound][:5])
            gpu_device.NormalizeVectors(v, n, d)
            y = v.ReadFloat32(n * d).reshape(n, d)
            w = lm.normalize_model(x, got)
            nan = np.isnan(w)
            assert (np.isnan(y) == nan).all(), (d, n)
            bad = np.flatnonzero((y.view(np.uint32) != w.view(np.uint32)) & ~nan)
            assert bad.size == 0, (d, n, bad[:5] // d, y.reshape(-1)[bad[:5]], w.reshape(-1)[bad[:5]])
        finally:
            v.Release(); nb.Release()


def test_normalize_threshold_edge(gpu_device):
    """one dimension: sqrtf(x * x) == |x|, so a row at 1e-10f is exactly at the threshold (left as it is) and its fp32
    neighbour above is scaled to +-1"""
    t = lm.NORM_FLOOR
    up = np.nextafter(t, F32(1), dtype=F32)
    x = np.array([t, -t, up, -up], F32)
    b, nb = gpu_device.NewBuffer(x), gpu_device.NewEmptyBuffer(4)
    try:
        gpu_device.ComputeNorms(b, nb, 4, 1)
        assert nb.ReadFloat32(4).tolist() == [t, t, up, up]
        gpu_device.NormalizeVectors(b, 4, 1)
        assert b.ReadFloat32(4).tolist() == [t, -t, 1.0, -1.0]
    finally:
        b.Release(); nb.Release()


@pytest.mark.parametrize("d", DIMS)
def test_cosine_similarity_error_bound(gpu_device, num_sms, d):
    """|s - s64| <= gamma_d sum |x_j q_j| for the dot (normalized = 1); for cosine (normalized = 0) the same over |x||q|
    plus the relative error of the norms and the division.  Row 5 is zero (cosine 0), row 7 has a NaN (NaN in both modes,
    that row only); a zero query gives cosine 0 everywhere."""
    rng = np.random.default_rng(d)
    for n in _row_counts(num_sms):
        x = (rng.standard_normal((n, d)) * np.exp(rng.uniform(-3, 3, (n, 1)))).astype(F32)
        x[5] = 0.0
        x[7, d // 2] = np.nan
        q = rng.standard_normal(d).astype(F32)
        e, qb, sb = gpu_device.NewBuffer(x), gpu_device.NewBuffer(q), gpu_device.NewEmptyBuffer(n)
        try:
            x64, q64 = x.astype(np.float64), q.astype(np.float64)
            dot64, absdot = x64 @ q64, np.abs(x64) @ np.abs(q64)
            nx, nq = np.sqrt((x64 * x64).sum(axis=1)), np.sqrt(q64 @ q64)
            ok = np.ones(n, bool)
            ok[7] = False
            gpu_device.CosineSimilarity(e, qb, sb, n, d, True)
            s = sb.ReadFloat32(n).astype(np.float64)
            assert np.isnan(s[7]) and not np.isnan(s[ok]).any()
            err, bound = np.abs(s - dot64)[ok], lm.gamma(d + 1) * absdot[ok]
            assert (err <= bound).all(), ("dot", d, n, np.flatnonzero(ok)[err > bound][:5])
            gpu_device.CosineSimilarity(e, qb, sb, n, d, False)
            s = sb.ReadFloat32(n).astype(np.float64)
            assert np.isnan(s[7]) and not np.isnan(s[ok]).any() and s[5] == 0.0
            with np.errstate(invalid="ignore", divide="ignore"):
                cos64 = np.where(nx > 0, dot64 / (nx * nq), 0.0)
                bound = lm.gamma(d + 8) * (np.where(nx > 0, absdot / (nx * nq), 0.0) + np.abs(cos64))
            err = np.abs(s - cos64)
            assert (err[ok] <= bound[ok]).all(), ("cosine", d, n, np.flatnonzero(ok & (err > bound))[:5])
            zq = gpu_device.NewBuffer(np.zeros(d, F32))
            try:
                gpu_device.CosineSimilarity(e, zq, sb, n, d, False)
                s = sb.ReadFloat32(n)
                assert (s[ok] == 0).all() and np.isnan(s[7])
            finally:
                zq.Release()
        finally:
            e.Release(); qb.Release(); sb.Release()
