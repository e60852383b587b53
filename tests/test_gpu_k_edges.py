"""Every search path at the k values (and batch sizes) where its internal plan changes, against a plain fp64 reference.

The plan of each path changes with k (DESIGN.md §3): the 16-bit pass (`shadow`) sizes its threshold sample as
next_pow2(8k) (k = 16/17), keeps 4 / 2 / 1 query groups per launch up to k = 128 / 160 / 192 and emits 768 instead of 512
entries per (CTA, query) above k = 160; the TF32 filter's emission k_emit = next_pow2(k + k/2 + 32) steps at k = 21/22
and 64/65 and is clamped to 256 after that; both filters stop at k = 192; the exact 3xTF32 scan serves k <= 255; the
CUDA-core scan switches its buffer from 512 to 1024 / 2048 slots at k = 256 / 768 and shrinks its query group with the
shared-memory budget; k > NK_MAX_K = 1024 runs ceil(k / 1024) CUDA-core passes, each admitting only keys below the last
key of the pass before; merging candidate lists is limited to NK_MAX_K.

References: the fp64 CPU oracle for small shapes, a float64 brute force on the device (torch, slice by slice) for the
200k-row corpora.  Row mask, score floor and tag filters are applied in the reference by selecting rows before ranking.
Results are checked with tests/parity.py (scores within 1e-4, identical index sets, boundary swaps only within fp32
noise); equal scores must come out by ascending row."""
import numpy as np
import pytest

from parity import check_parity, exact_scores_for

pytestmark = pytest.mark.gpu

PAD = 0xFFFFFFFF
METRICS = ["cosine", "dot", "euclidean"]
DTYPES = ["f32", "f16", "bf16"]
N_BIG, D_BIG, Q_BIG = 200_000, 128, 520  # large enough that every filter buffer fills

SHADOW_CASES = [(16, 64), (17, 64)] + [(k, Q) for k in (128, 129, 160, 161, 192) for Q in (64, 300, 520)]
FILTER_CASES = [(k, Q) for k in (21, 22, 64, 65, 150, 192) for Q in (5, 130, 520)]
TENSOR_CASES = [(k, Q) for k in (192, 193, 255) for Q in (5, 65, 130)]
SIMT_KS, SIMT_QS = (255, 256, 767, 768, 1024), (1, 2, 3, 8, 9, 13)
BIGK_KS, BIGK_QS = (1025, 2048, 2049, 2500), (1, 5, 13)


# ---- helpers ------------------------------------------------------------------------------------------------------------
def others64_torch(rows_of_slice, n, ids, queries, k, metric, slice_rows, q_chunk=4096):
    """fp64 brute force on the GPU (torch) of the k best rows other than each query's own, (score desc, row asc) /
    (distance asc, row asc).  rows_of_slice(lo, cnt) -> float32 cuda tensor [cnt, d]; an id of -1 excludes nothing.
    -> (idx int64 [Q, k], score [Q, k])."""
    import torch
    Q = len(ids)
    out_i, out_s = np.empty((Q, k), np.int64), np.empty((Q, k), np.float64)
    for q0 in range(0, Q, q_chunk):
        q64 = torch.from_numpy(np.asarray(queries[q0:q0 + q_chunk], np.float64)).cuda()
        me = torch.from_numpy(np.asarray(ids[q0:q0 + q_chunk], np.int64)).cuda()
        qn = q64.norm(dim=1)
        best_s = best_i = None
        for lo in range(0, n, slice_rows):
            cnt = min(slice_rows, n - lo)
            x = rows_of_slice(lo, cnt).double()
            s = q64 @ x.T  # [q, cnt]
            if metric == "cosine":
                den = qn[:, None] * x.norm(dim=1)[None, :]
                s = torch.where(den > 0, s / den, torch.zeros_like(s))
            elif metric == "euclidean":
                s = -((q64 * q64).sum(1)[:, None] + (x * x).sum(1)[None, :] - 2.0 * s)
            loc = me - lo
            inside = ((loc >= 0) & (loc < cnt)).nonzero().squeeze(1)
            s[inside, loc[inside]] = -float("inf")  # the query's own row
            v, i = torch.topk(s, min(k + 8, cnt), dim=1)
            i = i + lo
            if best_s is not None:
                v, i = torch.cat([best_s, v], dim=1), torch.cat([best_i, i], dim=1)
                keep = torch.topk(v, min(k + 8, v.shape[1]), dim=1).indices
                v, i = torch.gather(v, 1, keep), torch.gather(i, 1, keep)
            best_s, best_i = v, i
            del x, s
        bs, bi = best_s.cpu().numpy(), best_i.cpu().numpy()
        o = np.lexsort((bi, -bs), axis=1)[:, :k]
        bs, bi = np.take_along_axis(bs, o, 1), np.take_along_axis(bi, o, 1)
        out_i[q0:q0 + len(bi)] = bi
        out_s[q0:q0 + len(bi)] = np.sqrt(np.maximum(-bs, 0.0)) if metric == "euclidean" else bs
    return out_i, out_s


def knn64_torch(exact, queries, k, metric):
    """fp64 top k of every query over the exact fp32 rows `exact` (host), brute force on the device."""
    import torch
    dev = torch.from_numpy(np.ascontiguousarray(exact, dtype=np.float32)).cuda()
    out = others64_torch(lambda lo, cnt: dev[lo:lo + cnt], len(exact), np.full(len(queries), -1), queries, k, metric,
                         slice_rows=100_000)
    del dev
    torch.cuda.empty_cache()
    return out


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


def make_index(rows, metric, dtype="f32", devices=(0,)):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex(rows.shape[1], metric=metric, dtype=dtype, devices=devices)
    ix.upload(rows)
    return ix


def search(ix, path, q, k):
    """One forced-path search -> (idx, score, retry / exact-stage counts of this search, fatal flag)."""
    ix.set_path(path)
    c0 = ix.debug_counters()
    gi, gs = ix.search(q, k)
    assert ix.last_path() == path, (path, ix.last_path(), q.shape[0], k)
    c1 = ix.debug_counters()
    tail = (c1["bf16_stage_retries"] - c0["bf16_stage_retries"], c1["exact_stage_runs"] - c0["exact_stage_runs"])
    return gi, gs, tail, ix.debug_flags()[0]


def parity(what, rows, q, k, metric, gi, gs, oi, os_, swap_eps=2e-6):
    try:
        return check_parity(rows, q, k, metric, gi, gs, oi, os_, swap_eps=swap_eps)
    except AssertionError as e:
        raise AssertionError(f"{what}: {e}") from None


def assert_ties_by_row(rows, q, metric, gi, what=""):
    """Rows whose fp64 scores are exactly equal (exact copies) come out by ascending row; check_parity accepts any order
    inside such a tie.  (Equal returned euclidean distances do not mean a tie: sqrtf maps neighbouring squares together.)"""
    for qi in range(gi.shape[0]):
        g = gi[qi][gi[qi] != PAD].astype(np.int64)
        ex = exact_scores_for(rows, q[qi], g, metric)
        bad = (ex[1:] == ex[:-1]) & (g[1:] <= g[:-1])
        assert not bad.any(), (what, qi, np.nonzero(bad)[0][:5])


def same_bits(a, b, what=""):
    (ai, as_), (bi, bs) = a, b
    assert ai.shape == bi.shape, (what, ai.shape, bi.shape)
    assert np.array_equal(ai, bi), what
    assert np.array_equal(np.asarray(as_).view(np.uint32), np.asarray(bs).view(np.uint32)), what


_CORPORA = {}


def uniform_corpus(dtype, n=N_BIG, d=D_BIG, seed=7):
    """(rows to upload, exact fp32 values) of the uniform corpus, generated once per module."""
    import oracle
    key = (dtype, n, d, seed)
    if key not in _CORPORA:
        _CORPORA[key] = cast(oracle.fill_uniform(n, d, seed), dtype)
    return _CORPORA[key]


# ---- a + b. single-pass regimes of the filter and tensor paths, no retries on uniform data ------------------------------
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_shadow_at_its_plan_changes(knn_lib, oracle_mod, dtype, metric):
    """The 16-bit pass over a BF16 shadow (fp32) or the fp16 / bf16 rows themselves: sample size (k = 16/17 at Q = 64),
    4 / 2 / 1 query groups (k = 128/129/160/161 at Q = 300 and 520) and the 768-entry emission (k > 160).  Uniform data
    must never leave the first stage."""
    rows, exact = uniform_corpus(dtype)
    q = oracle_mod.fill_uniform(Q_BIG, D_BIG, 8)
    oi, os_ = knn64_torch(exact, q, 192, metric)
    ix = make_index(rows, metric, dtype)
    try:
        for k, Q in SHADOW_CASES:
            what = f"shadow {dtype} {metric} k={k} Q={Q}"
            gi, gs, tail, fatal = search(ix, "shadow", q[:Q], k)
            assert fatal == 0 and tail == (0, 0), (what, "retry / exact-stage runs", tail)
            parity(what, exact, q[:Q], k, metric, gi, gs, oi[:Q, :k], os_[:Q, :k])
    finally:
        ix.release()


@pytest.mark.parametrize("metric", METRICS)
def test_filter_and_tensor_at_their_plan_changes(knn_lib, oracle_mod, metric):
    """TF32 filter at k_emit 64 -> 128 -> 256 (k = 21/22, 64/65) and up to k = 192, where the margin room is smallest;
    exact 3xTF32 at k = 192..255 (cosine / dot); AUTO's pick at k = 193; the refusals just past each path's limit."""
    from nornicdb_b200.knn import KnnError
    rows, exact = uniform_corpus("f32")
    q = oracle_mod.fill_uniform(Q_BIG, D_BIG, 8)
    oi, os_ = knn64_torch(exact, q, 255, metric)
    ix = make_index(rows, metric)
    try:
        for k, Q in FILTER_CASES:
            what = f"filter {metric} k={k} Q={Q}"
            gi, gs, tail, fatal = search(ix, "filter", q[:Q], k)
            assert fatal == 0 and tail == (0, 0), (what, "retry / exact-stage runs", tail)
            parity(what, exact, q[:Q], k, metric, gi, gs, oi[:Q, :k], os_[:Q, :k])
        if metric != "euclidean":
            for k, Q in TENSOR_CASES:
                gi, gs, _, fatal = search(ix, "tensor", q[:Q], k)
                assert fatal == 0
                parity(f"tensor {metric} k={k} Q={Q}", exact, q[:Q], k, metric, gi, gs, oi[:Q, :k], os_[:Q, :k])
        # AUTO: the exact 3xTF32 scan serves cosine / dot between the filters' limit and its own; euclidean goes to CUDA cores
        ix.set_path("auto")
        for Q in (5, 130):
            gi, gs = ix.search(q[:Q], 193)
            assert ix.last_path() == ("simt" if metric == "euclidean" else "tensor"), (metric, Q, ix.last_path())
            parity(f"auto {metric} k=193 Q={Q}", exact, q[:Q], 193, metric, gi, gs, oi[:Q, :193], os_[:Q, :193])
        for path, k in (("shadow", 193), ("filter", 193), ("tensor", 256)) + ((("tensor", 1),) if metric == "euclidean" else ()):
            ix.set_path(path)
            with pytest.raises(KnnError, match="does not support this shape"):
                ix.search(q[:5], k)
    finally:
        ix.release()


# ---- a. CUDA-core scan: buffer sizes and query groups --------------------------------------------------------------------
@pytest.mark.parametrize("d", [128, 130])  # 130: scalar loads (d % 4 != 0), groups of 4 / 1
@pytest.mark.parametrize("metric", METRICS)
def test_simt_buffers_and_query_groups(knn_lib, oracle_mod, metric, d):
    """P = 512 / 1024 / 2048 slots (k = 255 | 256..767 | 768..1024) with query groups of 8 / 4 / 2 / 1 (Q = 13 = 8 + 4 + 1)."""
    n = 20_000
    rows = oracle_mod.fill_uniform(n, d, 21)
    q = oracle_mod.fill_uniform(max(SIMT_QS), d, 22)
    oi, os_ = oracle_mod.knn_exact64(rows, q, max(SIMT_KS), metric)
    ix = make_index(rows, metric)
    try:
        for k in SIMT_KS:
            for Q in SIMT_QS:
                gi, gs, _, fatal = search(ix, "simt", q[:Q], k)
                assert fatal == 0
                parity(f"simt {metric} d={d} k={k} Q={Q}", rows, q[:Q], k, metric, gi, gs, oi[:Q, :k], os_[:Q, :k])
    finally:
        ix.release()


@pytest.mark.parametrize("metric", METRICS)
def test_simt_wide_rows_shrink_the_query_group(knn_lib, oracle_mod, metric):
    """d = 8192 at k = 1024: a 2048-slot buffer plus 8 query rows exceed the 96 KB budget, so the group shrinks to 2."""
    n, d, k = 3000, 8192, 1024
    rows = oracle_mod.fill_uniform(n, d, 23)
    q = oracle_mod.fill_uniform(9, d, 24)
    oi, os_ = oracle_mod.knn_exact64(rows, q, k, metric)
    ix = make_index(rows, metric)
    try:
        for Q in (1, 2, 9):
            gi, gs, _, _ = search(ix, "simt", q[:Q], k)
            parity(f"simt d=8192 {metric} Q={Q}", rows, q[:Q], k, metric, gi, gs, oi[:Q], os_[:Q])
    finally:
        ix.release()


# ---- c. near ties at the largest k: the finish kernel carries up to 192 entries between rounds ---------------------------
def _near_tie_case(corpus, metric):
    """(index, exact rows, 300 queries)"""
    from nornicdb_b200.knn import KnnIndex
    import oracle
    rng = np.random.default_rng(11)
    if corpus == "clustered":
        n, d = 200_000, 128
        ix = KnnIndex(d, metric=metric)
        ix.fill_clustered(n, 4242, n_centres=40, sigma=0.1)
        rows = ix.read_rows(0, n)
        q = (rows[rng.integers(0, n, 300)] + rng.standard_normal((300, d)).astype(np.float32) * 0.05).astype(np.float32)
        return ix, rows, q
    # thousands of near-duplicates inside the margin of the k-th bound (test_gpu_round2.py's corpus)
    n, d = 300_000, 64
    base = oracle.fill_uniform(1, d, 9)[0]
    rows = oracle.fill_uniform(n, d, 10)
    dup = rng.choice(n, 9000, replace=False)
    rows[dup] = base[None, :] + rng.standard_normal((9000, d)).astype(np.float32) * 2e-3
    q = (base[None, :] + rng.standard_normal((300, d)).astype(np.float32) * 1e-3).astype(np.float32)
    return make_index(rows, metric), rows, q


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("corpus", ["clustered", "near-duplicates"])
def test_near_ties_at_the_largest_k(knn_lib, corpus, metric):
    """Exact results whatever the retry counters show; where neither filter retried, `shadow` and `filter` re-score the
    same survivors with the same arithmetic and must agree bit for bit."""
    ix, rows, q = _near_tie_case(corpus, metric)
    try:
        oi, os_ = knn64_torch(rows, q, 192, metric)
        seen = {}
        for k in (128, 161, 192):
            for Q in (6, 300):
                res = {}
                for path in ("shadow", "filter"):
                    gi, gs, tail, fatal = search(ix, path, q[:Q], k)
                    assert fatal == 0
                    parity(f"{corpus} {path} {metric} k={k} Q={Q}", rows, q[:Q], k, metric, gi, gs, oi[:Q, :k], os_[:Q, :k],
                           swap_eps=5e-6)
                    res[path] = (gi, gs, tail)
                    seen[f"{path} k={k} Q={Q}"] = tail
                if res["shadow"][2] == (0, 0) and res["filter"][2] == (0, 0):
                    same_bits(res["shadow"][:2], res["filter"][:2], f"{corpus} {metric} k={k} Q={Q}: shadow vs filter")
        print(f"\n{corpus} {metric}: (bf16-stage retries, exact-stage runs) per search: {seen}")
    finally:
        ix.release()


# ---- d. k > NK_MAX_K: several CUDA-core passes ----------------------------------------------------------------------------
def _dup7_corpus(dtype, d=64, m=715, seed=31):
    """n = 7m rows, every row one of m vectors, the copies scattered: every rank block is an exact 7-way tie, so the ties
    straddle rank 1024 (1024 % 7 = 2) and 2048 (2048 % 7 = 4) for every query."""
    import oracle
    base = oracle.fill_uniform(m, d, seed)
    f32 = base[np.random.default_rng(seed).permutation(7 * m) % m]
    return cast(f32, dtype)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_passes_continue_ties_by_row(knn_lib, oracle_mod, dtype, metric):
    rows, exact = _dup7_corpus(dtype)
    n, d = exact.shape
    q = oracle_mod.fill_uniform(max(BIGK_QS), d, 32)
    oi, os_ = oracle_mod.knn_exact64(exact, q, n, metric)
    ix = make_index(rows, metric, dtype)
    try:
        for k in BIGK_KS + (n,):
            for Q in BIGK_QS:
                what = f"{dtype} {metric} k={k} Q={Q}"
                gi, gs, _, _ = search(ix, "simt", q[:Q], k)
                assert gi.shape == (Q, k), what
                parity(what, exact, q[:Q], k, metric, gi, gs, oi[:Q, :k], os_[:Q, :k])
                assert_ties_by_row(exact, q, metric, gi, what)
        ix.set_path("auto")
        gi, _ = ix.search(q, 2049)
        assert ix.last_path() == "simt"
    finally:
        ix.release()


def _nan_tail_ok(gi, gs, good_count, bad, metric, what):
    """NaN rows rank after every finite row, by ascending row, with score -inf (distance +inf)."""
    tail_i, tail_s = gi[:, good_count:], gs[:, good_count:]
    want = np.sort(bad)[:tail_i.shape[1]]
    assert (tail_i == want[None, :]).all(), (what, tail_i[:, :8], want[:8])
    assert (tail_s == (np.inf if metric == "euclidean" else -np.inf)).all(), (what, tail_s[:, :8])


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("dtype", ["f32", "f16"])
def test_passes_rank_nan_rows_last(knn_lib, oracle_mod, dtype, metric):
    """4100 rows, 30 of them NaN.  dot / euclidean: ranks 4070..4099 hold the NaN rows, across the pass boundary at 4096.
    Cosine maps a NaN similarity to 0 (as for zero vectors): the NaN rows tie at 0, by row, in the middle of the ranking."""
    n, d = 4100, 64
    f32 = oracle_mod.fill_uniform(n, d, 41)
    bad = np.sort(np.random.default_rng(41).choice(n, 30, replace=False))
    f32[bad, 5] = np.nan
    rows, exact = cast(f32, dtype)
    good = np.setdiff1d(np.arange(n), bad)
    q = oracle_mod.fill_uniform(max(BIGK_QS), d, 42)
    oi, os_ = oracle_mod.knn_exact64(exact[good], q, len(good), metric)
    oi = good[oi]
    if metric == "cosine":  # the NaN rows join the ranking with score 0
        Qn = q.shape[0]
        oi = np.concatenate([oi, np.broadcast_to(bad, (Qn, len(bad)))], axis=1)
        os_ = np.concatenate([os_, np.zeros((Qn, len(bad)))], axis=1)
        o = np.lexsort((oi, -os_), axis=1)
        oi, os_ = np.take_along_axis(oi, o, 1), np.take_along_axis(os_, o, 1)
    ix = make_index(rows, metric, dtype)
    try:
        for k in (2500, 4080, n):
            for Q in BIGK_QS:
                what = f"NaN {dtype} {metric} k={k} Q={Q}"
                gi, gs, _, _ = search(ix, "simt", q[:Q], k)
                m = k if metric == "cosine" else min(k, len(good))
                parity(what, exact, q[:Q], m, metric, gi[:, :m], gs[:, :m], oi[:Q, :m], os_[:Q, :m])
                assert_ties_by_row(exact, q, metric, gi, what)
                if metric != "cosine":
                    _nan_tail_ok(gi, gs, m, bad, metric, what)
    finally:
        ix.release()


@pytest.mark.parametrize("metric", METRICS)
def test_passes_with_row_mask_floor_and_tag_filters(knn_lib, oracle_mod, metric):
    """Every pass honours the row mask, the score floor and the per-query tag filters; the count is min(k, rows passing
    the mask) and slots past a query's admissible rows hold 0xffffffff / 0."""
    from nornicdb_b200.knn import ADMIT_NONE, synthetic_tags, admits
    n, d = 6000, 64
    rows = oracle_mod.fill_uniform(n, d, 51)
    q = oracle_mod.fill_uniform(13, d, 52)
    rng = np.random.default_rng(51)
    ix = make_index(rows, metric)
    try:
        # row mask: 2700 rows pass; k = 1500 (two passes over the masked rows) and k = 4000 (count = 2700)
        keep = np.zeros(n, bool)
        keep[rng.choice(n, 2700, replace=False)] = True
        kept = np.nonzero(keep)[0]
        ix.set_row_mask(keep)
        oi, os_ = oracle_mod.knn_exact64(rows[kept], q, len(kept), metric)
        for k in (1500, 2048, 2049, 4000):
            for Q in BIGK_QS:
                what = f"mask {metric} k={k} Q={Q}"
                gi, gs, _, _ = search(ix, "simt", q[:Q], k)
                m = min(k, len(kept))
                assert gi.shape == (Q, m), what
                parity(what, rows, q[:Q], m, metric, gi, gs, kept[oi[:Q, :m]], os_[:Q, :m])
        ix.set_row_mask(None)

        # score floor: every query keeps at least its best 1800 rows (the floor cuts inside the second pass or later); rows
        # within fp32 noise of the floor may fall either side
        oi, os_ = oracle_mod.knn_exact64(rows, q, 2500, metric)
        floor = float(os_[:, 1800].max() if metric == "euclidean" else os_[:, 1800].min())
        ix.set_min_score(floor)
        gi, gs, _, _ = search(ix, "simt", q, 2500)
        ix.set_min_score(None)
        assert gi.shape == (13, 2500) and (gi == PAD).any()
        for qi in range(13):
            ok = os_[qi] <= floor if metric == "euclidean" else os_[qi] >= floor
            noise = np.abs(os_[qi] - floor) <= 2e-6 * max(1.0, abs(floor))
            got = gi[qi][gi[qi] != PAD]
            assert (gi[qi][len(got):] == PAD).all() and (gs[qi][len(got):] == 0).all(), qi
            assert len(got) > 1024, (qi, len(got))  # the floor cuts inside the second pass
            assert set(oi[qi][ok & ~noise].tolist()) <= set(got.tolist()) <= set(oi[qi][ok | noise].tolist()), qi
            m = len(got)
            parity(f"floor {metric} q{qi}", rows, q[qi:qi + 1], m, metric, gi[qi:qi + 1, :m], gs[qi:qi + 1, :m],
                   oi[qi:qi + 1, :m], os_[qi:qi + 1, :m])

        # per-query tag filters: ~1/2, ~1/4 (< k), none, no filter, admit none
        tags = synthetic_tags(n, 53)
        ix.set_row_tags(tags)
        pattern = [(1, 0, 0), (3, 0, 0), (0, 4, 0), (0, 0, 0), ADMIT_NONE]
        filters = np.array([pattern[i % len(pattern)] for i in range(13)], dtype=np.uint64)
        for k in (1025, 2500):
            gi, gs = ix.search_filtered(q, k, filters)
            assert gi.shape == (13, k)
            for qi in range(13):
                adm = np.nonzero(admits(tags, *[int(v) for v in filters[qi]]))[0]
                m = min(k, len(adm))
                what = f"tags {metric} k={k} q{qi} admitted={len(adm)}"
                assert (gi[qi, m:] == PAD).all() and (gs[qi, m:] == 0).all(), what
                if m == 0:
                    continue
                oi, os_ = oracle_mod.knn_exact64(rows[adm], q[qi:qi + 1], m, metric)
                parity(what, rows, q[qi:qi + 1], m, metric, gi[qi:qi + 1, :m], gs[qi:qi + 1, :m], adm[oi], os_)
    finally:
        ix.release()


# ---- e. entry points at the same edges ------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
def test_search_rows_across_the_filter_and_pass_limits(knn_lib, metric):
    """k + 1 crosses the filters' limit (191 -> 192 | 193) and the one-pass limit (1023 -> 1024 | 1025)."""
    import oracle
    import torch
    n, d = 20_000, 128
    rows = oracle.fill_uniform(n, d, 61)
    ids = np.random.default_rng(61).choice(n, 40, replace=False)
    ix = make_index(rows, metric)
    dev = torch.from_numpy(rows).cuda()
    try:
        oi, os_ = others64_torch(lambda lo, cnt: dev[lo:lo + cnt], n, ids, rows[ids], 1024, metric, slice_rows=n)
        for k in (191, 192, 1023, 1024):
            gi, gs = ix.search_rows(ids, k)
            assert not (gi == ids[:, None]).any()
            parity(f"search_rows {metric} k={k} ({ix.last_path()})", rows, rows[ids], k, metric, gi, gs, oi[:, :k], os_[:, :k])
    finally:
        ix.release()


def _device_call(ix, q, k, filters=None):
    import torch
    Q = q.shape[0]
    st = torch.cuda.Stream()
    qd = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    fd = None if filters is None else torch.from_numpy(filters.view(np.int64)).cuda()
    oi = torch.empty((Q, k), dtype=torch.int32, device="cuda")
    os_ = torch.empty((Q, k), dtype=torch.float32, device="cuda")
    st.wait_stream(torch.cuda.current_stream())
    if fd is None:
        assert ix.search_device(qd.data_ptr(), Q, k, oi.data_ptr(), os_.data_ptr(), st.cuda_stream) == k
    else:
        assert ix.search_filtered_device(qd.data_ptr(), fd.data_ptr(), Q, k, oi.data_ptr(), os_.data_ptr(), st.cuda_stream) == k
    ix.status(st.cuda_stream)
    return oi.cpu().numpy().view(np.uint32), os_.cpu().numpy()


@pytest.mark.parametrize("metric", METRICS)
def test_device_api_at_the_limits(knn_lib, oracle_mod, metric):
    """search_device / search_filtered_device at k = 192 | 193 and 1024 | 1025: bit-identical to the host call on the
    same path, and right."""
    from nornicdb_b200.knn import ADMIT_NONE, admits, synthetic_tags
    n, d, Q = 30_000, 128, 13
    rows = oracle_mod.fill_uniform(n, d, 71)
    q = oracle_mod.fill_uniform(Q, d, 72)
    tags = synthetic_tags(n, 73)
    pattern = [(0, 0, 0), (1, 0, 0), (2, 1, 0), ADMIT_NONE]
    filters = np.array([pattern[i % len(pattern)] for i in range(Q)], dtype=np.uint64)
    oi, os_ = oracle_mod.knn_exact64(rows, q, 1025, metric)
    ix = make_index(rows, metric)
    ix.set_row_tags(tags)
    try:
        for k in (192, 193, 1024, 1025):
            for path in ("auto", "simt"):
                ix.set_path(path)
                host = ix.search(q, k)
                used = ix.last_path()
                dev = _device_call(ix, q, k)
                assert ix.last_path() == used
                same_bits(dev, host, f"search_device {metric} k={k} {path} ({used})")
                parity(f"search_device {metric} k={k} {used}", rows, q, k, metric, *dev, oi[:, :k], os_[:, :k])
                host = ix.search_filtered(q, k, filters)
                dev = _device_call(ix, q, k, filters)
                same_bits(dev, host, f"search_filtered_device {metric} k={k} {path} ({ix.last_path()})")
                for qi in range(Q):
                    adm = np.nonzero(admits(tags, *[int(v) for v in filters[qi]]))[0]
                    m = min(k, len(adm))
                    assert (dev[0][qi, m:] == PAD).all()
                    if m:
                        ri, rs = oracle_mod.knn_exact64(rows[adm], q[qi:qi + 1], m, metric)
                        parity(f"filtered {metric} k={k} q{qi}", rows, q[qi:qi + 1], m, metric, dev[0][qi:qi + 1, :m],
                               dev[1][qi:qi + 1, :m], adm[ri], rs)
    finally:
        ix.release()


def test_score_subset_around_the_pass_limit(knn_lib, oracle_mod):
    n, d = 12_000, 64
    rows = oracle_mod.fill_uniform(n, d, 81)
    q = oracle_mod.fill_uniform(1, d, 82)[0]
    rng = np.random.default_rng(81)
    ix = make_index(rows, "cosine")
    try:
        for size in (1024, 1025, 2049, 6000):
            subset = rng.choice(n, size, replace=False).astype(np.uint32)
            ex = oracle_mod.scores_exact64(rows[subset], q, "cosine")
            order = np.lexsort((subset, -ex))
            for k in (1024, 1025, 2048, 5000):
                kk = min(k, size)
                gi, gs = ix.score_subset(q, subset, k)
                assert gi.shape == (kk,)
                parity(f"score_subset size={size} k={k}", rows, q[None], kk, "cosine", gi[None], gs[None],
                       subset[order][None, :kk], ex[order][None, :kk])
    finally:
        ix.release()


@pytest.mark.parametrize("metric", METRICS)
def test_search_groups_at_the_merge_width(knn_lib, oracle_mod, metric):
    """k = 1024 best nodes out of 2500 (each node's best chunk against the fp64 reference); k = 1025 is refused."""
    from nornicdb_b200.knn import KnnError
    n, d, G = 12_000, 96, 2500
    rows = oracle_mod.fill_uniform(n, d, 91)
    q = oracle_mod.fill_uniform(1, d, 92)[0]
    group = np.random.default_rng(91).integers(0, G, n).astype(np.uint32)
    s = exact_scores_for(rows, q, np.arange(n), metric)
    key = -s if metric == "euclidean" else s
    order = np.lexsort((np.arange(n), -key))               # best chunk first, lowest row on ties
    _, first = np.unique(group[order], return_index=True)  # each node's best chunk
    best = order[np.sort(first)]                           # in ranking order
    ix = make_index(rows, metric)
    try:
        ix.set_row_groups(group, G)
        g, r, sc = ix.search_groups(q, 1024)
        assert len(g) == 1024 and (group[r] == g).all()
        parity(f"groups {metric}", rows, q[None], 1024, metric, r[None], sc[None], best[None, :1024], s[best][None, :1024])
        with pytest.raises(KnnError, match="exceeds NK_MAX_K"):
            ix.search_groups(q, 1025)
    finally:
        ix.release()


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_in_process_shards_equal_one_shard(knn_lib, oracle_mod, metric):
    """devices = (0, 0) and (0, 0, 0): 3000 / 2000 rows per shard, so k = 2500 exceeds a shard; bit-identical to one shard."""
    n, d, Q = 6000, 64, 7
    rows = oracle_mod.fill_uniform(n, d, 101)
    q = oracle_mod.fill_uniform(Q, d, 102)
    oi, os_ = oracle_mod.knn_exact64(rows, q, 2500, metric)
    ixs = [make_index(rows, metric, devices=dv) for dv in ((0,), (0, 0), (0, 0, 0))]
    try:
        for k in (192, 1024, 1025, 2500):
            for path in ("auto", "simt") + (("shadow",) if k <= 192 else ()):
                res = []
                for ix in ixs:
                    ix.set_path(path)
                    res.append(ix.search(q, k))
                parity(f"shards {metric} k={k} {path}", rows, q, k, metric, *res[0], oi[:, :k], os_[:, :k])
                for shards, r in zip((2, 3), res[1:]):
                    same_bits(r, res[0], f"{shards} shards {metric} k={k} {path}")
    finally:
        for ix in ixs:
            ix.release()


# ---- §2. merging is limited to NK_MAX_K, and refused before any work -----------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
def test_keys_of_two_halves_merge_at_the_merge_width(knn_lib, oracle_mod, metric):
    import torch
    from nornicdb_b200.knn import KnnError, merge_keys_device
    n, d, Q = 20_000, 128, 9
    rows = oracle_mod.fill_uniform(n, d, 111)
    q = oracle_mod.fill_uniform(Q, d, 112)
    full = make_index(rows, metric)
    halves = []
    try:
        qd = torch.from_numpy(q).cuda()
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        for g in range(2):
            h = make_index(rows[g * n // 2:(g + 1) * n // 2], metric)
            h.set_row_base(g * n // 2)
            halves.append(h)
        for k in (1024, 1025):
            keys = torch.empty((2, Q, k), dtype=torch.int64, device="cuda")
            mi = torch.empty((Q, k), dtype=torch.int32, device="cuda")
            ms = torch.empty((Q, k), dtype=torch.float32, device="cuda")
            for g, h in enumerate(halves):  # one shard's keys are served up to NK_MAX_K_TOTAL
                assert h.search_keys_device(qd.data_ptr(), Q, k, keys[g].data_ptr(), st.cuda_stream) == k
            if k > 1024:
                with pytest.raises(KnnError, match="NK_MAX_K"):
                    merge_keys_device(0, keys.data_ptr(), 2, Q, k, metric, mi.data_ptr(), ms.data_ptr(), st.cuda_stream)
                continue
            merge_keys_device(0, keys.data_ptr(), 2, Q, k, metric, mi.data_ptr(), ms.data_ptr(), st.cuda_stream)
            for h in halves:
                h.status(st.cuda_stream)
            got = (mi.cpu().numpy().view(np.uint32), ms.cpu().numpy())
            full.set_path("simt")
            same_bits(got, full.search(q, k), f"merged halves {metric} k={k}")
            oi, os_ = oracle_mod.knn_exact64(rows, q, k, metric)
            parity(f"merged halves {metric} k={k}", rows, q, k, metric, *got, oi, os_)
    finally:
        full.release()
        for h in halves:
            h.release()


class _TwoRanks:
    """Two single-device indexes (one rank each) on cuda:0, connected for the peer-memory exchange."""

    def __init__(self, rows, metric, q, ks, slot_k):
        import torch
        from nornicdb_b200.knn import Comm
        from nornicdb_b200.sharding import shard_range
        n, d = rows.shape
        self.metric, self.ixs, self.comms = metric, [], []
        for r in range(2):
            lo, hi = shard_range(n, 2, r)
            ix = make_index(rows[lo:hi], metric)
            ix.set_row_base(lo)
            # A workspace that grows waits for the whole device first, and with both ranks on one device that includes the
            # other rank's merge, which waits for this rank's push: size every workspace before the first exchange.
            for k in ks:
                ix.search(q, k)
            self.ixs.append(ix)
            self.comms.append(Comm(0, r, 2, q.shape[0] * slot_k * 8))
        Comm.connect_local(self.comms)
        # one stream per rank, as separate processes would have: a rank's merge waits on the device for the other's push
        self.streams = [torch.cuda.Stream() for _ in range(2)]

    def search(self, q, k, ranks=(0, 1)):
        import torch
        Q = q.shape[0]
        qd = torch.from_numpy(q).cuda()
        outs = [(torch.empty((Q, k), dtype=torch.int32, device="cuda"), torch.empty((Q, k), dtype=torch.float32, device="cuda"))
                for _ in ranks]
        for r, (oi, os_) in zip(ranks, outs):
            st = self.streams[r]
            st.wait_stream(torch.cuda.current_stream())
            self.ixs[r].search_sharded_device(self.comms[r], qd.data_ptr(), Q, k, oi.data_ptr(), os_.data_ptr(), st.cuda_stream)
        for r in ranks:
            self.comms[r].status(self.streams[r].cuda_stream)
            self.ixs[r].status(self.streams[r].cuda_stream)
        return [(oi.cpu().numpy().view(np.uint32), os_.cpu().numpy()) for oi, os_ in outs]

    def release(self):
        for st in self.streams:
            st.synchronize()
        for c in self.comms:
            c.release()
        for ix in self.ixs:
            ix.release()


@pytest.mark.parametrize("metric", METRICS)
def test_exchange_at_the_merge_width_and_refusal_above(knn_lib, oracle_mod, metric):
    """Two ranks on one device: k = 1024 is exact; k = 1025 is refused by nk_search_sharded_device and by
    nk_comm_exchange_merge on ONE rank each, before the exchange epoch advances or a peer buffer is written, so both
    ranks' next exchanges still pair up and return the right result."""
    import torch
    from nornicdb_b200.knn import KnnError, METRICS as METRIC_IDS
    n, d, Q = 30_000, 128, 6
    rows = oracle_mod.fill_uniform(n, d, 121)
    q = oracle_mod.fill_uniform(Q, d, 122)
    ranks = _TwoRanks(rows, metric, q, (1024, 10), 1025)  # slots hold Q * 1025 keys: only the k limit can refuse k = 1025
    try:
        oi, os_ = oracle_mod.knn_exact64(rows, q, 1024, metric)
        res = ranks.search(q, 1024)
        for gi, gs in res:
            parity(f"exchange {metric} k=1024", rows, q, 1024, metric, gi, gs, oi, os_)
        same_bits(res[0], res[1], "both ranks")
        with pytest.raises(KnnError, match="NK_MAX_K"):
            ranks.search(q, 1025, ranks=(0,))
        keys = torch.zeros((Q, 1025), dtype=torch.int64, device="cuda")
        out_i = torch.empty((Q, 1025), dtype=torch.int32, device="cuda")
        out_s = torch.empty((Q, 1025), dtype=torch.float32, device="cuda")
        c1 = ranks.comms[1]
        rc = c1.lib.nk_comm_exchange_merge(c1.ptr, keys.data_ptr(), Q, 1025, METRIC_IDS[metric], out_i.data_ptr(),
                                           out_s.data_ptr(), ranks.streams[1].cuda_stream)
        assert rc == -1 and "NK_MAX_K" in c1.lib.nk_last_error().decode()
        for k in (10, 1024):
            res = ranks.search(q, k)
            for gi, gs in res:
                parity(f"exchange {metric} k={k} after the refusals", rows, q, k, metric, gi, gs, oi[:, :k], os_[:, :k])
    finally:
        ranks.release()
