"""The device-resident search API (nk_search_device, nk_search_keys_device + nk_merge_keys_device) on every path, on data
that trips each tail stage, queued back to back without a host sync, with PDL on and off, and the call order of one
index across streams.

Every answer is checked twice: against the fp64 oracle (check_parity), and against the host API on the same index and
queries.  The host API defers the retry / exact stages until it has seen a flag; the device API queues them blindly
behind the first stage and lets a flag on the device decide, so the two take different routes to the same answer."""
import os
import subprocess
import sys

import numpy as np
import pytest

from parity import check_parity, exact_scores_for

pytestmark = pytest.mark.gpu

METRICS = ["cosine", "dot", "euclidean"]
DTYPES = ["f32", "f16", "bf16"]
SENTINEL = 0xFFFFFFFF
SLEEP_CYCLES = 200_000_000  # torch.cuda._sleep: about 0.1 s at H100 clocks


def _cast(oracle, f32, dtype):
    """(rows to upload, the exact values they hold as fp32 / fp16 for the oracle)"""
    from nornicdb_b200.knn import from_bf16_bits, to_bf16_bits
    if dtype == "f32":
        return f32, f32
    if dtype == "f16":
        h = f32.astype(np.float16)
        return h, h
    b = to_bf16_bits(f32)
    return b, from_bf16_bits(b)


def _index(rows, metric, dtype="f32", path="auto"):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex(rows.shape[1], metric=metric, dtype=dtype)
    ix.upload(rows)
    ix.set_path(path)
    return ix


class _DeviceCall:
    """One device search queued on `stream` into fresh output tensors; .result() waits and reads it back."""

    def __init__(self, ix, q, k, stream):
        import torch
        self.Q, self.k, self.stream = q.shape[0], k, stream
        self.qd = torch.from_numpy(np.ascontiguousarray(q, dtype=np.float32)).cuda()
        self.oi = torch.empty((self.Q, k), dtype=torch.int32, device="cuda")
        self.os = torch.empty((self.Q, k), dtype=torch.float32, device="cuda")
        stream.wait_stream(torch.cuda.current_stream())  # inputs are written on the current stream
        assert ix.search_device(self.qd.data_ptr(), self.Q, k, self.oi.data_ptr(), self.os.data_ptr(), stream.cuda_stream) == k

    def result(self, ix):
        ix.status(self.stream.cuda_stream)  # waits for the stream; reports an internal overflow
        return self.oi.cpu().numpy().view(np.uint32), self.os.cpu().numpy()


def _device_search(ix, q, k):
    import torch
    return _DeviceCall(ix, q, k, torch.cuda.Stream()).result(ix)


def _assert_same_as_host(gi, gs, hi, hs, exact_ties=False):
    """Device and host answers of one index: scores within 2e-6 relative rank by rank, and the same rows.  The exact twins
    sum in another order than the finish kernel, so two rows whose scores agree to within that tolerance may trade places
    (a row may also trade with one just past the end of the list).  With exact_ties every rank must hold the same row."""
    assert gi.shape == hi.shape
    assert np.allclose(gs, hs, rtol=2e-6, atol=1e-7), np.abs(gs - hs).max()
    if exact_ties:
        assert (gi == hi).all(), (gi, hi)
        return
    for qi, r in zip(*np.nonzero(gi != hi)):
        tied = np.abs(hs[qi] - hs[qi, r]) <= 2e-6 * max(1.0, abs(float(hs[qi, r])))
        at = np.nonzero(hi[qi] == gi[qi, r])[0]
        assert tied[at].all() if len(at) else tied[-1], (qi, r, gi[qi], hi[qi], gs[qi], hs[qi])


def _check(exact, q, k, metric, gi, gs, hi, hs, oracle_result=None, swap_eps=2e-6):
    """A device answer (gi, gs) against the host API's (hi, hs) on the same index, and against the fp64 oracle."""
    import oracle
    _assert_same_as_host(gi, gs, hi, hs)
    oi, os_ = oracle_result if oracle_result is not None else oracle.knn_exact64(exact, q, k, metric)
    check_parity(exact, q, k, metric, gi, gs, oi, os_, swap_eps=swap_eps)


# ---- a. parity matrix -------------------------------------------------------------------------------------------------
SHAPES = [(3, 10), (40, 10), (300, 50), (40, 600), (6, 1500)]  # (40, 600): one CUDA-core pass; (6, 1500): multi-pass + decode


def _paths(dtype, metric):
    if dtype != "f32":
        return ["auto", "shadow", "simt"]
    return ["auto", "shadow", "filter"] + ([] if metric == "euclidean" else ["tensor"]) + ["simt"]


@pytest.mark.parametrize("n,d", [(20_000, 128), (40_000, 256)])
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_device_search_parity_matrix(knn_lib, oracle_mod, dtype, metric, n, d):
    from nornicdb_b200.knn import KnnError
    rows, exact = _cast(oracle_mod, oracle_mod.fill_uniform(n, d, 11 + d), dtype)
    qs = oracle_mod.fill_uniform(max(Q for Q, _ in SHAPES), d, 12 + d)
    ix = _index(rows, metric, dtype)
    served = {}
    try:
        for Q, k in SHAPES:
            q = qs[:Q]
            want = oracle_mod.knn_exact64(exact, q, k, metric)
            for path in _paths(dtype, metric):
                ix.set_path(path)
                try:
                    hi, hs = ix.search(q, k)
                except KnnError as e:
                    assert path not in ("auto", "simt"), e  # a forced tensor path may not serve this shape ...
                    with pytest.raises(KnnError):           # ... and then neither API serves it
                        _device_search(ix, q, k)
                    continue
                gi, gs = _device_search(ix, q, k)
                served[path, Q, k] = ix.last_path()
                _check(exact, q, k, metric, gi, gs, hi, hs, oracle_result=want)
    finally:
        ix.release()
    assert all(("auto", Q, k) in served and ("simt", Q, k) in served for Q, k in SHAPES)
    assert served["auto", 6, 1500] == "simt" and served["auto", 300, 50] == "shadow"


# ---- b. the blind tail on data that trips each stage -------------------------------------------------------------------
NEAR_TIES = {"filter-20k": ("filter", 20_000, 1e-5, 0), "shadow-160k": ("shadow", 160_000, 1e-4, 1)}


def _near_ties(oracle, corpus, dtype):
    from test_gpu_filtered import _near_tie_corpus
    path, n, noise, seed = NEAR_TIES[corpus]
    f32, q = _near_tie_corpus(oracle, n, noise, seed)
    rows, exact = _cast(oracle, f32, dtype)
    return rows, exact, q, (path if dtype == "f32" else "shadow")  # 16-bit rows: the 16-bit pass is the only filter


def _tail_case(oracle, corpus, dtype, metric):
    """The device search of one near-tie case: (index, exact rows, queries, result, flags); the caller releases."""
    rows, exact, q, path = _near_ties(oracle, corpus, dtype)
    ix = _index(rows, metric, dtype, path)
    gi, gs = _device_search(ix, q, 10)
    return ix, exact, q, (gi, gs), ix.debug_flags()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("corpus", list(NEAR_TIES))
def test_blind_tail_on_near_ties(knn_lib, oracle_mod, corpus, dtype, metric):
    """At these noise levels most fp16 / bf16 rows are exact copies of the base vector: the lowest-row rule is tested at
    scale.  On fp32 rows the first stage always overflows (test_gpu_tensor.py), on 16-bit rows the 160k corpus does; the
    device API then goes straight to the exact twin (3xTF32, or the gated CUDA-core scan for euclidean and 16-bit rows)."""
    ix, exact, q, (gi, gs), flags = _tail_case(oracle_mod, corpus, dtype, metric)
    try:
        assert flags[0] == 0, flags
        if dtype == "f32" or corpus == "shadow-160k":
            assert flags[1] != 0, flags  # a first-stage buffer overflowed; the exact stage answered
        hi, hs = ix.search(q, 10)
        assert ix.last_path() == (NEAR_TIES[corpus][0] if dtype == "f32" else "shadow")
        _check(exact, q, 10, metric, gi, gs, hi, hs, swap_eps=5e-6)
    finally:
        ix.release()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_exact_duplicates_keep_the_lowest_rows(knn_lib, oracle_mod, metric, dtype):
    """Every row is one of 16 vectors: each rank is an exact tie, broken by the lowest row, on both APIs."""
    base = oracle_mod.fill_uniform(16, 128, 5)
    rows, exact = _cast(oracle_mod, np.tile(base, (2048, 1)), dtype)
    q = exact[[3, 7, 12]].astype(np.float32)
    ix = _index(rows, metric, dtype)
    try:
        gi, gs = _device_search(ix, q, 20)
        hi, hs = ix.search(q, 20)
    finally:
        ix.release()
    for j, b in enumerate((3, 7, 12)):
        assert gi[j].tolist() == [b + 16 * i for i in range(20)], (j, gi[j])
    _assert_same_as_host(gi, gs, hi, hs, exact_ties=True)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("path", ["filter", "shadow"])
def test_k_or_more_nan_rows_on_the_device(knn_lib, oracle_mod, path, metric):
    """20 NaN rows and k = 5: k undecidable bounds.  The filters keep them with bound +inf and do not count them when they
    pick the k-th bound (DESIGN.md §3.3), so NaN rows must neither evict a finite row nor stall the device API."""
    n, d, k = 5000, 64, 5
    rows = oracle_mod.fill_uniform(n, d, 31)
    q = oracle_mod.fill_uniform(8, d, 32)
    bad = np.arange(100, 120)
    rows[bad, 3] = np.nan
    good = np.setdiff1d(np.arange(n), bad)
    ix = _index(rows, metric, path=path)
    try:
        gi, gs = _device_search(ix, q, k)
        flags = ix.debug_flags()
        hi, hs = ix.search(q, k)
    finally:
        ix.release()
    assert flags[0] == 0, flags
    assert not np.isin(gi, bad).any(), gi
    _assert_same_as_host(gi, gs, hi, hs)
    oi, os_ = oracle_mod.knn_exact64(rows[good], q, k, metric)
    check_parity(rows, q, k, metric, gi, gs, good[oi], os_)


@pytest.mark.parametrize("metric", METRICS)
def test_exact_twin_honours_row_mask_and_floor(knn_lib, oracle_mod, metric):
    rows, exact, q, path = _near_ties(oracle_mod, "filter-20k", "f32")
    n, k = rows.shape[0], 10
    keep = np.arange(n) % 3 != 1
    sub = np.nonzero(keep)[0]
    oi, os_ = oracle_mod.knn_exact64(rows[sub], q, k, metric)
    floor = float(np.median(os_[:, k // 2]))  # cuts most lists in the middle
    ix = _index(rows, metric, path=path)
    try:
        ix.set_row_mask(keep)
        ix.set_min_score(floor)
        gi, gs = _device_search(ix, q, k)
        flags = ix.debug_flags()
        hi, hs = ix.search(q, k)
    finally:
        ix.release()
    assert flags[0] == 0 and flags[1] != 0, flags
    _assert_same_as_host(gi, gs, hi, hs)
    eucl = metric == "euclidean"
    for qi in range(q.shape[0]):
        got = gi[qi][gi[qi] != SENTINEL]
        assert (gi[qi][len(got):] == SENTINEL).all()
        assert keep[got].all(), got
        ex = exact_scores_for(rows, q[qi], got, metric)
        tol = 5e-6 * max(1.0, abs(floor))
        assert (ex <= floor + tol).all() if eucl else (ex >= floor - tol).all(), (qi, ex, floor)
        want = os_[qi][os_[qi] <= floor] if eucl else os_[qi][os_[qi] >= floor]
        undecided = int((np.abs(os_[qi] - floor) <= tol).sum())  # rows within fp32 noise of the floor fall either side
        assert abs(len(got) - len(want)) <= undecided, (qi, got, want)
        m = min(len(got), len(want))
        assert np.allclose(ex[:m], want[:m], rtol=0, atol=5e-6 * max(1.0, float(np.abs(want).max(initial=0.0))))


# ---- c. keys + merge, and the exchange, on data that overflows ---------------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
def test_keys_of_two_half_shards_merge_to_the_full_search(knn_lib, oracle_mod, metric):
    import torch
    from nornicdb_b200.knn import merge_keys_device
    rows, exact, q, path = _near_ties(oracle_mod, "filter-20k", "f32")
    n, Q, k = rows.shape[0], q.shape[0], 10
    full = _index(rows, metric, path=path)
    halves = []
    try:
        hi, hs = full.search(q, k)
        st = torch.cuda.Stream()
        qd = torch.from_numpy(q).cuda()
        keys = torch.empty((2, Q, k), dtype=torch.int64, device="cuda")
        mi = torch.empty((Q, k), dtype=torch.int32, device="cuda")
        ms = torch.empty((Q, k), dtype=torch.float32, device="cuda")
        st.wait_stream(torch.cuda.current_stream())
        for g in range(2):
            h = _index(rows[g * n // 2:(g + 1) * n // 2], metric, path=path)
            h.set_row_base(g * n // 2)
            halves.append(h)
            assert h.search_keys_device(qd.data_ptr(), Q, k, keys[g].data_ptr(), st.cuda_stream) == k
        merge_keys_device(0, keys.data_ptr(), 2, Q, k, metric, mi.data_ptr(), ms.data_ptr(), st.cuda_stream)
        for h in halves:
            h.status(st.cuda_stream)
        flags = [h.debug_flags() for h in halves]
        gi, gs = mi.cpu().numpy().view(np.uint32), ms.cpu().numpy()
    finally:
        full.release()
        for h in halves:
            h.release()
    assert all(f[0] == 0 for f in flags) and any(f[1] != 0 for f in flags), flags
    _assert_same_as_host(gi, gs, hi, hs)
    oi, os_ = oracle_mod.knn_exact64(rows, q, k, metric)
    check_parity(rows, q, k, metric, gi, gs, oi, os_, swap_eps=5e-6)


# ---- d. back to back on one stream, one sync -----------------------------------------------------------------------------
def _back_to_back(oracle, sync_each=False):
    """Six device searches over three indexes, queued on one stream with no host sync in between (sync_each: with one
    after each call): uniform; near-tie queries on the near-tie corpus (its first stage overflows); >= k NaN rows; uniform
    queries on the near-tie corpus; then uniform and NaN again with larger Q and k, which grows the workspaces while the
    earlier searches may still be queued.  Returns the indexes, the (index, queries, k) of each call, and the device
    results."""
    import torch
    from test_gpu_filtered import _near_tie_corpus
    uni = oracle.fill_uniform(20_000, 128, 41)
    tie, tq = _near_tie_corpus(oracle, 20_000, 1e-5, 0)
    nan = oracle.fill_uniform(5000, 64, 31)
    nan[100:120, 3] = np.nan
    ixs = {"uniform": _index(uni, "cosine"), "near-tie": _index(tie, "cosine", path="filter"), "nan": _index(nan, "dot", path="shadow")}
    calls = [("uniform", oracle.fill_uniform(8, 128, 42), 10), ("near-tie", tq[:20], 10), ("nan", oracle.fill_uniform(8, 64, 32), 5),
             ("near-tie", oracle.fill_uniform(200, 128, 43), 60), ("uniform", oracle.fill_uniform(300, 128, 44), 100),
             ("nan", oracle.fill_uniform(64, 64, 33), 20)]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    queued = []
    for name, q, k in calls:
        queued.append(_DeviceCall(ixs[name], q, k, st))
        if sync_each:
            st.synchronize()
    st.synchronize()
    results = [(c.oi.cpu().numpy().view(np.uint32), c.os.cpu().numpy()) for c in queued]
    return ixs, calls, results


def _exact_runs(ixs):
    for ix in ixs.values():
        ix.status()
    return {name: ix.debug_counters()["exact_stage_runs"] for name, ix in ixs.items()}


def test_back_to_back_device_searches_on_one_stream(knn_lib, oracle_mod):
    """State one search leaves to the next (a sticky flag, a stale threshold or list fill) would change an answer or send
    a search to the exact stage that the same search, run on its own, does not take."""
    ixs, calls, results = _back_to_back(oracle_mod)
    alone, _, alone_results = _back_to_back(oracle_mod, sync_each=True)
    try:
        exact_runs, alone_runs = _exact_runs(ixs), _exact_runs(alone)
        for (name, q, k), (gi, gs), (ai, as_) in zip(calls, results, alone_results):
            assert np.array_equal(gi, ai) and np.array_equal(gs.view(np.uint32), as_.view(np.uint32)), name
            hi, hs = ixs[name].search(q, k)
            _assert_same_as_host(gi, gs, hi, hs)
    finally:
        for ix in list(ixs.values()) + list(alone.values()):
            ix.release()
    assert exact_runs == alone_runs, (exact_runs, alone_runs)
    assert exact_runs["uniform"] == 0 and exact_runs["near-tie"] >= 1, exact_runs


# ---- f. PDL off: the same answers, bit for bit ---------------------------------------------------------------------------
def _pdl_sensitive_results(oracle):
    """Device results of the tail cases (b) and the back-to-back queue (d), by name."""
    out = {}
    for corpus in NEAR_TIES:
        for dtype in DTYPES:
            for metric in METRICS:
                ix, _, _, (gi, gs), _ = _tail_case(oracle, corpus, dtype, metric)
                ix.release()
                out[f"tail-{corpus}-{dtype}-{metric}-idx"], out[f"tail-{corpus}-{dtype}-{metric}-score"] = gi, gs
    ixs, _, results = _back_to_back(oracle)
    for ix in ixs.values():
        ix.release()
    for i, (gi, gs) in enumerate(results):
        out[f"queue-{i}-idx"], out[f"queue-{i}-score"] = gi, gs
    return out


def test_pdl_off_gives_bit_identical_results(knn_lib, oracle_mod, tmp_path):
    """NK_PDL is read once per process: run the same searches in a child process with programmatic dependent launch off."""
    here = os.path.dirname(os.path.abspath(__file__))
    out = tmp_path / "pdl_off.npz"
    script = ("import sys, numpy as np; sys.path[:0] = [sys.argv[1], sys.argv[2]]\n"
              "import oracle, test_gpu_device_api as t\n"
              "oracle.build()\n"
              "np.savez(sys.argv[3], **t._pdl_sensitive_results(oracle))\n")
    env = dict(os.environ, NK_PDL="0")
    run = subprocess.run([sys.executable, "-s", "-c", script, here, os.path.dirname(here), str(out)], env=env,
                         capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stdout[-3000:] + run.stderr[-3000:]
    on = _pdl_sensitive_results(oracle_mod)
    off = np.load(out)
    assert sorted(off.files) == sorted(on)
    for name, a in on.items():
        assert np.array_equal(a.view(np.uint32), off[name].view(np.uint32)), name


# ---- e. one index, several streams: the calls take effect in call order ----------------------------------------------------
def _delayed_search(ix, q, k):
    """A device search queued on a fresh stream behind about 0.1 s of device sleep: still queued when the call returns."""
    import torch
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(st):
        torch.cuda._sleep(SLEEP_CYCLES)
    return _DeviceCall(ix, q, k, st)


def test_device_search_then_mutation_sees_the_old_rows(knn_lib, oracle_mod):
    """update_row, remove_swap and set_row_mask called after a device search must not change what it returns, however
    long the search stays queued on its stream; a host search afterwards must see them."""
    n, d, k = 30_000, 128, 10
    rows = oracle_mod.fill_uniform(n, d, 51)
    q = oracle_mod.fill_uniform(8, d, 52)
    ix = _index(rows, "cosine")
    try:
        before_i, before_s = ix.search(q, k)
        # update: row r (not among q[0]'s answers) becomes q[0]'s best match
        r = 12_345
        assert r not in before_i[0]
        call = _delayed_search(ix, q, k)
        ix.update_row(r, 4.0 * q[0])
        gi, gs = call.result(ix)
        assert r not in gi[0], gi[0]
        assert (gi == before_i).all() and np.allclose(gs, before_s, rtol=2e-6, atol=1e-7)
        assert ix.search(q, k)[0][0, 0] == r
        rows[r] = 4.0 * q[0]
        # remove_swap: q[0]'s best row is overwritten by the last row
        before_i, before_s = ix.search(q, k)
        call = _delayed_search(ix, q, k)
        ix.remove_swap(r)
        gi, gs = call.result(ix)
        assert gi[0, 0] == r and (gi == before_i).all() and np.allclose(gs, before_s, rtol=2e-6, atol=1e-7)
        rows[r] = rows[-1]
        rows = rows[:-1]
        # row mask: a mask already set (so the search reads the mask buffer), then one that drops q[1]'s best row
        keep = np.ones(len(rows), dtype=bool)
        ix.set_row_mask(keep)
        before_i, before_s = ix.search(q, k)
        best = before_i[1, 0]
        keep[best] = False
        call = _delayed_search(ix, q, k)
        ix.set_row_mask(keep)
        gi, gs = call.result(ix)
        assert gi[1, 0] == best and (gi == before_i).all() and np.allclose(gs, before_s, rtol=2e-6, atol=1e-7)
        after_i, after_s = ix.search(q, k)
        assert best not in after_i[1]
        oi, os_ = oracle_mod.knn_exact64(rows[keep], q, k, "cosine")
        check_parity(rows, q, k, "cosine", after_i, after_s, np.nonzero(keep)[0][oi], os_)
    finally:
        ix.release()


@pytest.fixture(scope="module")
def big_index(knn_lib):
    """2M x 256 fp32 rows generated on the device: each scan takes milliseconds, long enough for two to overlap."""
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex(256, metric="cosine")
    ix.fill_uniform(2_000_000, 61)
    yield ix
    ix.release()


def test_two_streams_one_index(knn_lib, oracle_mod, big_index):
    import torch
    ix, k = big_index, 10
    qa, qb = oracle_mod.fill_uniform(64, 256, 62), oracle_mod.fill_uniform(64, 256, 63)
    want_a, want_b = ix.search(qa, k), ix.search(qb, k)  # also sizes the workspace: the searches below grow nothing
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    for st in (a, b):
        with torch.cuda.stream(st):
            torch.cuda._sleep(SLEEP_CYCLES)
    ca, cb = _DeviceCall(ix, qa, k, a), _DeviceCall(ix, qb, k, b)
    for c, (hi, hs) in ((ca, want_a), (cb, want_b)):
        gi, gs = c.result(ix)
        _assert_same_as_host(gi, gs, hi, hs)


def test_device_search_then_host_search(knn_lib, oracle_mod, big_index):
    import torch
    ix, k = big_index, 10
    qa, qb = oracle_mod.fill_uniform(64, 256, 64), oracle_mod.fill_uniform(64, 256, 65)
    want_a, want_b = ix.search(qa, k), ix.search(qb, k)
    ca = _DeviceCall(ix, qa, k, torch.cuda.Stream())
    hi, hs = ix.search(qb, k)  # at once, on the index's own stream, while the device search runs
    gi, gs = ca.result(ix)
    _assert_same_as_host(gi, gs, *want_a)
    _assert_same_as_host(hi, hs, *want_b, exact_ties=True)
    # the large-corpus answers themselves, on a sample of queries, against the fp64 oracle
    sample = [0, 31, 63]
    rows = ix.read_rows(0, 2_000_000)
    oi, os_ = oracle_mod.knn_exact64(rows, qa[sample], k, "cosine")
    check_parity(rows, qa[sample], k, "cosine", gi[sample], gs[sample], oi, os_)
