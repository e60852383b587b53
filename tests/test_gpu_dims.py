"""Every search path at the dimensions d where its plan changes, on both sides of each edge, against fp64.

The edges come from tests/dims.py, which computes them from the rules the library applies (slab and pad widths, the
CUDA-core scan's 96 KB group budget, the 48 KB default and the opt-in shared memory, the finish kernel's windows and the
filters' admission limit).  At each d: AUTO and every forced path the shape admits (`simt`, `filter`, `tensor`, `shadow`
over the BF16 shadow or the rows in place, `shadow` over the int8 image), with `last_path()` asserted; every path the
shape does not admit must refuse.  Results follow tests/parity.py against an fp64 brute force; the int8 image and the BF16
shadow must agree bit for bit.  Row counts are >= 4 099 and ragged, so the sampled initial threshold and a partial last
tile both run."""
import numpy as np
import pytest

import dims
from parity import check_parity

pytestmark = pytest.mark.gpu

PAD = 0xFFFFFFFF
METRICS = ("cosine", "dot", "euclidean")
N = 4099
Q = 13  # CUDA-core groups of 8 + 4 + 1; every filter path from 5 queries on


# ---- helpers ------------------------------------------------------------------------------------------------------------
def scores64(x, q, metric):
    """fp64 scores [Q x n] (euclidean: distances) of the exact rows x against the queries q"""
    x64, q64 = np.asarray(x, np.float64), np.asarray(q, np.float64).reshape(-1, x.shape[1])
    dots = q64 @ x64.T
    if metric == "dot":
        return dots
    xn = np.sqrt((x64 * x64).sum(1))[None, :]
    qn = np.sqrt((q64 * q64).sum(1))[:, None]
    if metric == "cosine":
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.where(xn * qn > 0, dots / (xn * qn), 0.0)
    return np.sqrt(np.maximum(xn ** 2 + qn ** 2 - 2.0 * dots, 0.0))


def ranked(s, metric, k, allowed=None):
    """(idx, score) of the k best columns of each row of s, best first, ties by ascending row"""
    key = s if metric == "euclidean" else -s
    if allowed is not None:
        key = np.where(allowed[None, :], key, np.inf)
    o = np.lexsort((np.broadcast_to(np.arange(s.shape[1]), s.shape), key), axis=1)[:, :k]
    return o, np.take_along_axis(s, o, 1)


def cast(f32, dtype):
    """(rows to upload, the exact values they hold as fp32)"""
    from nornicdb_b200.knn import from_bf16_bits, to_bf16_bits
    if dtype == "f32":
        return f32, f32
    if dtype == "f16":
        h = f32.astype(np.float16)
        return h, h.astype(np.float32)
    b = to_bf16_bits(f32)
    return b, from_bf16_bits(b)


def corpus(n, d, seed):
    """rows and queries uniform on [-0.5, 1.5): the scores do not cancel, so at d in the tens of thousands fp32 summation
    stays far inside the parity rule's 1e-4 relative (sign-symmetric data leaves scores of ~1/sqrt(d) of |x||q|, whose
    fp32 rounding alone reaches 1e-4 of them there)"""
    rng = np.random.default_rng(seed)
    return (rng.random((n, d), dtype=np.float32) * 2 - 0.5), (rng.random((Q, d), dtype=np.float32) * 2 - 0.5)


def index(monkeypatch, rows, metric, dtype="f32", image=None):
    """image: None keeps every image the library builds by default; "int8" the int8 image of fp32 shards alone"""
    from nornicdb_b200.knn import KnnIndex
    if image is None:
        monkeypatch.delenv("NK_SHADOW", raising=False)
    else:
        monkeypatch.setenv("NK_SHADOW", image)  # read at creation
    ix = KnnIndex(rows.shape[1], metric=metric, dtype=dtype)
    ix.upload(rows)
    return ix


def admitted_paths(dtype, d, metric, k=10):
    """the forced paths the library serves at this shape"""
    f32_tc = dtype == "f32" and d >= 32 and d % 4 == 0
    out = {"simt"}
    if f32_tc and d <= dims.FILTER_MAX_DIM and k <= 192:
        out.add("filter")
    if f32_tc and metric != "euclidean" and k <= 255 and d <= dims.TENSOR_EXACT_MAX_DIM:
        out.add("tensor")
    if dims.filter_admits(d, dtype) and k <= 192:
        out.add("shadow")
    return out


def auto_path(paths):
    for p in ("shadow", "filter", "tensor", "simt"):
        if p in paths:
            return p


def run(ix, path, q, k):
    ix.set_path(path)
    gi, gs = ix.search(q, k)
    assert ix.last_path() == path, (path, ix.last_path())
    return gi, gs


def parity(what, exact, q, k, metric, got, want):
    try:
        check_parity(exact, q, k, metric, got[0], got[1], want[0], want[1])
    except AssertionError as e:
        raise AssertionError(f"{what}: {e}") from None


def same_bits(a, b, what):
    assert np.array_equal(a[0], b[0]), (what, np.argwhere(a[0] != b[0])[:4].tolist())
    assert np.array_equal(np.asarray(a[1]).view(np.uint32), np.asarray(b[1]).view(np.uint32)), what


def check_every_path(monkeypatch, dtype, d, k=10, n=N, seed=None, metrics=METRICS):
    """AUTO and every forced path at (dtype, d, k) on every metric; the paths the shape does not admit refuse; on fp32 the
    int8 image's results equal the BF16 shadow's bit for bit."""
    from nornicdb_b200.knn import KnnError
    f32, q = corpus(n, d, d if seed is None else seed)
    rows, exact = cast(f32, dtype)
    int8_ix = None
    ix = index(monkeypatch, rows, metrics[0], dtype)
    try:
        if dtype == "f32" and dims.filter_admits(d):
            int8_ix = index(monkeypatch, rows, metrics[0], dtype, image="int8")
        for metric in metrics:
            ix.set_metric(metric)
            want = ranked(scores64(exact, q, metric), metric, k)
            paths = admitted_paths(dtype, d, metric, k)
            for path in ("simt", "filter", "tensor", "shadow"):
                what = f"{dtype} d={d} k={k} {metric} {path}"
                if path not in paths:
                    ix.set_path(path)
                    with pytest.raises(KnnError):
                        ix.search(q, k)
                    continue
                got = run(ix, path, q, k)
                parity(what, exact, q, k, metric, got, want)
                if path == "shadow" and int8_ix is not None:
                    int8_ix.set_metric(metric)
                    same_bits(run(int8_ix, "shadow", q, k), got, what + " int8 image vs BF16 shadow")
            ix.set_path("auto")
            got = ix.search(q, k)
            assert ix.last_path() == auto_path(paths), (dtype, d, metric, ix.last_path())
            parity(f"{dtype} d={d} {metric} auto", exact, q, k, metric, got, want)
    finally:
        ix.release()
        if int8_ix is not None:
            int8_ix.release()


@pytest.fixture(scope="module")
def statics(knn_lib):
    return {"finish": dims.kernel_static("scan_tensor", r"filter_finish_kernel"),
            "simt": dims.kernel_static("scan_simt", r"knn_scan_simt_kernel")}


# ---- small d: the tensor-path floor, the ragged TF32 slab, the BF16 / int8 pads, the 16-bit box tails -------------------
SMALL = sorted({("f32", d) for d in (4, 30, 31, 32, 33, 36, 60, 64, 68, 100, 124, 128, 132)} |
               {(dt, d) for dt in ("f16", "bf16") for d in (36, 40, 56, 64, 72)})


@pytest.mark.parametrize("dtype,d", SMALL)
def test_small_dims_every_path(knn_lib, monkeypatch, dtype, d):
    check_every_path(monkeypatch, dtype, d)


# ---- the CUDA-core scan's query groups: each d where qt halves, in each candidate-buffer band ----------------------------
SIMT_EDGES = [(k, qt, d) for k in (10, 256, 800) for qt, e in dims.simt_group_edges(k).items() for d in (e, e + 4)]


@pytest.mark.parametrize("k,qt,d", SIMT_EDGES)
def test_simt_group_edges(knn_lib, monkeypatch, k, qt, d):
    groups = dims.simt_groups(d, k, Q)
    assert groups[0] == (qt if d == dims.simt_group_edges(k)[qt] else qt // 2), groups
    f32, q = corpus(N, d, d + k)
    ix = index(monkeypatch, f32, "cosine")
    try:
        for metric in METRICS:
            ix.set_metric(metric)
            got = run(ix, "simt", q, k)
            parity(f"simt d={d} k={k} {metric} groups {groups}", f32, q, k, metric, got, ranked(scores64(f32, q, metric), metric, k))
    finally:
        ix.release()


# ---- shared-memory edges: the prep kernel's opt-in, the 4d-byte query opt-in, the finish windows, the admission limit ---
def test_prep_opt_in_at_the_largest_sample(knn_lib, monkeypatch):
    """k = 192 at Q <= 128 samples 2048 rows: the prep kernel crosses 48 KB between these two d"""
    lo = (dims.DEFAULT_SMEM - 2048 * 8) // 4
    hi = lo + 4
    assert dims.prep_sample(192, Q, N) == 2048
    for d in (lo, hi):
        check_every_path(monkeypatch, "f32", d, k=192, metrics=("cosine", "euclidean"))


def large_dims(statics):
    e = dims.edges(statics)
    return sorted(set(e["4d-byte query opt-in"] + [24_704, 25_000] + e["finish window"] + e["filter admission"]))


def test_large_dims_every_path(knn_lib, monkeypatch, statics):
    """Both sides of the 48 KB query opt-in (12 288 / 12 292), the finish kernel's window edge (24 704 fits the larger
    window under either static figure, 25 000 under neither) and the filters' admission limit (32 768 / 32 772)."""
    for d in large_dims(statics):
        check_every_path(monkeypatch, "f32", d)
    for dtype in ("f16", "bf16"):
        check_every_path(monkeypatch, dtype, dims.FILTER_MAX_DIM, metrics=("cosine", "euclidean"))


@pytest.mark.parametrize("d", [12_292, 25_000, 32_768])
def test_calls_that_reuse_the_scans(knn_lib, monkeypatch, d):
    """search_filtered / search_windowed (one tag filter, one value window), search_range, search_rows, search_pairs,
    search_groups and score_subset on AUTO, against fp64."""
    f32, q = corpus(N, d, d + 1)
    f32[N - 8:] = f32[:8] + 0.01 * f32[N - 16:N - 8]  # eight planted near-duplicate pairs for the self-join
    tags = np.where(np.arange(N) % 3 == 0, 1, 2).astype(np.uint64)
    values = np.arange(1, N + 1, dtype=np.uint64)
    ix = index(monkeypatch, f32, "cosine")
    try:
        ix.set_row_tags(tags)
        ix.set_row_values(values)
        for metric in ("cosine", "euclidean"):
            ix.set_metric(metric)
            s = scores64(f32, q, metric)
            what = f"d={d} {metric}"
            allowed = tags == 1
            parity(what + " filtered", f32, q, 10, metric, ix.search_filtered(q, 10, [(1, 0, 0)] * Q), ranked(s, metric, 10, allowed))
            assert ix.last_path() == "shadow", ix.last_path()
            allowed = (values >= 1001) & (values <= 3000)
            parity(what + " windowed", f32, q, 10, metric, ix.search_windowed(q, 10, (1001, 3000)), ranked(s, metric, 10, allowed))
            # range: a threshold midway between the fp64 20th and 21st best of each query
            r = ranked(s, metric, 21)[1]
            thr = (r[:, 19] + r[:, 20]) / 2
            for qi, (gi, gs) in enumerate(ix.search_range(q, thr.astype(np.float32))):
                want = ranked(s[qi:qi + 1], metric, 20)
                parity(f"{what} range q{qi}", f32, q[qi:qi + 1], 20, metric, (gi[None, :], gs[None, :]), want)
            # search by stored row: the k nearest other rows
            sel = np.array([0, 5, 1234, N - 1])
            gi, gs = ix.search_rows(sel, 10)
            so = scores64(f32, f32[sel], metric)
            so[np.arange(len(sel)), sel] = np.inf if metric == "euclidean" else -np.inf
            parity(what + " search_rows", f32, f32[sel], 10, metric, (gi, gs), ranked(so, metric, 10))
            # the self-join over the stripe of the first 8 rows: exactly the planted pairs
            pthr = 0.99 if metric == "cosine" else float(np.sqrt(d) * 0.02)
            off, pi, ps = ix.search_pairs(pthr, 0, 8)
            for r0 in range(8):
                got = pi[int(off[r0]):int(off[r0 + 1])]
                sr = scores64(f32, f32[r0:r0 + 1], metric)[0]
                hit = (sr <= pthr) if metric == "euclidean" else (sr >= pthr)
                hit[:r0 + 1] = False
                assert sorted(got.tolist()) == np.nonzero(hit)[0].tolist() == [N - 8 + r0], (what, r0, got)
            # score_subset: the listed rows, best first
            sub = np.arange(7, N, 11)
            gi, gs = ix.score_subset(q[0], sub, 10)
            want = ranked(s[:1, sub], metric, 10)
            parity(what + " score_subset", f32, q[:1], 10, metric, (gi[None, :], gs[None, :]), (sub[want[0]], want[1]))
            # best-of-chunks: groups of 4 rows, the best chunk of each
            ix.set_row_groups(np.arange(N) // 4)
            g, gr, gs = ix.search_groups(q[0], 5)
            key = s[0] if metric != "euclidean" else -s[0]
            best = np.maximum.reduceat(key, np.arange(0, N, 4))
            assert g.tolist() == np.argsort(-best, kind="stable")[:5].tolist(), (what, g)
            assert np.allclose(gs, s[0, gr], rtol=1e-4, atol=1e-6), (what, gs, s[0, gr])
            ix.set_row_groups(None)
    finally:
        ix.release()


def test_group_search_serves_16bit_rows_above_48kb(knn_lib, monkeypatch):
    d = dims.DEFAULT_SMEM // 4 + 8
    f32, q = corpus(1000, d, 3)
    for dtype in ("f16", "bf16"):
        rows, exact = cast(f32, dtype)
        ix = index(monkeypatch, rows, "cosine", dtype)
        try:
            ix.set_row_groups(np.arange(1000) // 4)
            g, gr, gs = ix.search_groups(q[0], 5)
            s = scores64(exact, q[:1], "cosine")[0]
            assert g.tolist() == np.argsort(-np.maximum.reduceat(s, np.arange(0, 1000, 4)), kind="stable")[:5].tolist()
            assert np.allclose(gs, s[gr], rtol=1e-4, atol=1e-6)
        finally:
            ix.release()


@pytest.mark.parametrize("d", [8192, dims.FILTER_MAX_DIM])
@pytest.mark.parametrize("image", ["bf16", "int8"])
def test_filter_bounds_hold_at_large_d(knn_lib, monkeypatch, image, d):
    """acc_c = d 2^-22 + 4e-6 grows with d: every estimate of the BF16 shadow / int8 image lies within its bound of fp64"""
    f32, q = corpus(N, d, d + 2)
    ix = index(monkeypatch, f32, "cosine", image=image)
    try:
        for metric in METRICS:
            ix.set_metric(metric)
            est, bnd = ix.filter_dump(q, "shadow")
            s = scores64(f32, q, metric).T
            if metric == "euclidean":
                s = -s * s  # the euclidean filter works on -dist^2
            err = np.abs(est.astype(np.float64) - s)
            assert np.isfinite(est).all() and np.isfinite(bnd).all()
            bad = np.argwhere(err > bnd)
            assert bad.size == 0, (image, d, metric, bad[:4].tolist(), float((err / bnd).max()))
    finally:
        ix.release()


@pytest.mark.parametrize("d", [dims.FILTER_MAX_DIM, dims.FILTER_MAX_DIM + 4])
def test_assign_nearest_at_the_admission_limit(knn_lib, monkeypatch, d):
    f32, _ = corpus(N, d, d + 3)
    cen = f32[::512][:8] + 0.5
    for metric in ("euclidean", "cosine"):
        ix = index(monkeypatch, f32, metric)
        try:
            assign = np.zeros(N, np.int32)
            ix.assign_nearest(cen, assign, metric=metric)
            s = scores64(cen, f32, metric)
            want = s.argmin(1) if metric == "euclidean" else s.argmax(1)
            srt = np.sort(s, 1)
            gap = srt[:, 1] - srt[:, 0] if metric == "euclidean" else srt[:, -1] - srt[:, -2]
            bad = (assign != want) & (gap > 1e-6 * np.abs(srt).max(1))
            assert not bad.any(), (metric, d, np.nonzero(bad)[0][:5])
        finally:
            ix.release()


def test_no_path_past_the_simt_refusal(knn_lib, monkeypatch, statics):
    """Past the CUDA-core scan's last d no path serves a search: a clean refusal naming d, on AUTO and forced, for one
    query and for a batch."""
    from nornicdb_b200.knn import KnnError
    lo, hi = dims.edges(statics)["SIMT refusal"]
    f32, q = corpus(600, hi, 5)
    ix = index(monkeypatch, f32, "euclidean")
    try:
        for metric in METRICS:
            ix.set_metric(metric)
            for path in ("auto", "simt"):
                ix.set_path(path)
                for nq in (1, 5):
                    with pytest.raises(KnnError, match=f"dim={hi}"):
                        ix.search(q[:nq], 10)
        ix.set_metric("cosine")
        ix.set_path("tensor")
        with pytest.raises(KnnError):
            ix.search(q[:5], 10)
    finally:
        ix.release()
    f32, q = corpus(600, lo, 6)
    ix = index(monkeypatch, f32, "euclidean")
    try:
        got = run(ix, "simt", q[:1], 10)
        parity(f"simt euclidean d={lo}", f32, q[:1], 10, "euclidean", got, ranked(scores64(f32, q[:1], "euclidean"), "euclidean", 10))
    finally:
        ix.release()
