"""GPU tests of the legacy boundary — the reference's own pkg/gpu/cuda/cuda_test.go cases, driven through the
mirror of its Go API (nornicdb_b200.cuda) over the C ABI."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _kat(kats, op):
    return [t for t in kats if t["op"] == op]


def test_device_info(gpu_device):
    from nornicdb_b200 import cuda
    assert cuda.IsAvailable() and cuda.DeviceCount() >= 1
    assert gpu_device.ID() == 0
    assert "H100" in gpu_device.Name() or gpu_device.Name()
    assert gpu_device.MemoryBytes() > 0 and gpu_device.MemoryMB() > 0
    major, minor = gpu_device.ComputeCapability()
    assert (major, minor) == (9, 0), f"this build targets sm_90a, device is {major}.{minor}"
    assert cuda.HasGPUHardware() and cuda.IsCUDACapable()
    assert cuda.GPUName() == gpu_device.Name() and cuda.GPUMemoryMB() == gpu_device.MemoryMB()


def test_buffers(gpu_device):
    from nornicdb_b200 import cuda
    data = np.array([1.0, 2.0, 3.0, 4.0, 5.0], np.float32)
    for mem in (cuda.MemoryDevice, cuda.MemoryPinned):
        b = gpu_device.NewBuffer(data, mem)
        assert b.Size() == 20
        assert (b.ReadFloat32(5) == data).all()
        assert (b.ReadFloat32(3) == data[:3]).all()
        assert b.ReadFloat32(6) is None and b.ReadFloat32(0) is None  # cuda_bridge.go:574-576
        b.Release()
        b.Release()  # idempotent
    e = gpu_device.NewEmptyBuffer(100)
    assert e.Size() == 400
    e.Release()
    with pytest.raises(cuda.CudaError):
        gpu_device.NewBuffer([], cuda.MemoryDevice)  # cuda_bridge.go:507-509


def test_normalize_vectors(gpu_device, kats):
    for t in _kat(kats, "cuda.normalize_vectors"):
        b = gpu_device.NewBuffer(t["data"])
        gpu_device.NormalizeVectors(b, t["n"], t["dims"])
        assert np.allclose(b.ReadFloat32(len(t["data"])), t["want"], atol=t["tol"])
        b.Release()
    # zero rows stay untouched (norm <= 1e-10, cuda_bridge.go:267)
    b = gpu_device.NewBuffer([0, 0, 0, 0, 5, 0, 0, 0])
    gpu_device.NormalizeVectors(b, 2, 4)
    assert np.allclose(b.ReadFloat32(8), [0, 0, 0, 0, 1, 0, 0, 0])
    b.Release()


def test_compute_norms(gpu_device):
    rng = np.random.default_rng(0)
    x = rng.standard_normal((37, 130)).astype(np.float32)
    v = gpu_device.NewBuffer(x)
    n = gpu_device.NewEmptyBuffer(37)
    gpu_device.ComputeNorms(v, n, 37, 130)
    assert np.allclose(n.ReadFloat32(37), np.linalg.norm(x.astype(np.float64), axis=1), rtol=1e-5)
    v.Release(); n.Release()


def test_cosine_similarity(gpu_device, kats, oracle_mod):
    for t in _kat(kats, "cuda.cosine_similarity"):
        e = gpu_device.NewBuffer(t["embeddings"])
        q = gpu_device.NewBuffer(t["query"])
        s = gpu_device.NewEmptyBuffer(t["n"])
        gpu_device.CosineSimilarity(e, q, s, t["n"], t["dims"], t["normalized"])
        assert np.allclose(s.ReadFloat32(t["n"]), t["want"], atol=t["tol"])
        for b in (e, q, s):
            b.Release()
    # normalized=False: true cosine of raw vectors == simd.BatchCosineSimilarity (simd.go:149-170)
    emb = oracle_mod.fill_uniform(500, 96, 3)
    emb[7] = 0.0
    qv = oracle_mod.fill_uniform(1, 96, 4)[0]
    e, q, s = gpu_device.NewBuffer(emb), gpu_device.NewBuffer(qv), gpu_device.NewEmptyBuffer(500)
    gpu_device.CosineSimilarity(e, q, s, 500, 96, False)
    assert np.allclose(s.ReadFloat32(500), oracle_mod.batch("cosine", emb, qv), rtol=1e-4, atol=1e-6)
    gpu_device.CosineSimilarity(e, q, s, 500, 96, True)
    assert np.allclose(s.ReadFloat32(500), oracle_mod.batch("dot", emb, qv), rtol=1e-4, atol=1e-5)
    for b in (e, q, s):
        b.Release()


def test_topk(gpu_device, kats, oracle_mod):
    for t in _kat(kats, "cuda.topk"):
        s = gpu_device.NewBuffer(t["scores"])
        idx, sc = gpu_device.TopK(s, len(t["scores"]), t["k"])
        assert idx.tolist() == t["want_idx"]
        assert np.allclose(sc, t["want_scores"])
        s.Release()
    # bit-exact against the reference's insertion top-k (cuda_bridge.go:327-375), ties included
    rng = np.random.default_rng(1)
    for n, k in ((1, 1), (5, 5), (1000, 10), (5000, 100), (70000, 1024), (300001, 37)):
        scores = rng.integers(-50, 50, n).astype(np.float32) / 8.0  # many ties
        s = gpu_device.NewBuffer(scores)
        idx, sc = gpu_device.TopK(s, n, k)
        oi, os_ = oracle_mod.topk_insertion(scores, k)
        assert (idx == oi).all() and (sc == os_).all(), (n, k)
        s.Release()


def test_search_kats(gpu_device, kats):
    for t in _kat(kats, "cuda.search"):
        e = gpu_device.NewBuffer(t["embeddings"])
        res = gpu_device.Search(e, t["query"], t["n"], t["dims"], t["k"], True)
        assert len(res) == t["want_len"]
        assert res[0].Index == t["want_first_idx"]
        assert abs(res[0].Score - t["want_first_score"]) <= t["tol"]
        e.Release()
    for t in _kat(kats, "cuda.search_zero_k"):
        e = gpu_device.NewBuffer(t["embeddings"])
        assert gpu_device.Search(e, t["query"], t["n"], t["dims"], t["k"], True) is None
        e.Release()
    for t in _kat(kats, "cuda.search_k_gt_n"):
        e = gpu_device.NewBuffer(t["embeddings"])
        res = gpu_device.Search(e, t["query"], t["n"], t["dims"], t["k"], True)
        assert len(res) == t["want_len"]
        e.Release()


def test_search_equals_legacy_chain(gpu_device, oracle_mod):
    """Fused Device.Search == CosineSimilarity + TopK (the chain it replaces, cuda_bridge.go:643-686)."""
    emb = oracle_mod.fill_uniform(4000, 128, 11)
    oracle_mod.batch_normalize(emb.reshape(-1), 4000, 128)
    qv = oracle_mod.fill_uniform(1, 128, 12)[0]
    e, q, s = gpu_device.NewBuffer(emb), gpu_device.NewBuffer(qv), gpu_device.NewEmptyBuffer(4000)
    gpu_device.CosineSimilarity(e, q, s, 4000, 128, True)
    idx, sc = gpu_device.TopK(s, 4000, 10)
    res = gpu_device.Search(e, qv, 4000, 128, 10, True)
    assert [r.Index for r in res] == idx.tolist()
    assert np.allclose([r.Score for r in res], sc, rtol=1e-5, atol=1e-6)
    for b in (e, q, s):
        b.Release()
