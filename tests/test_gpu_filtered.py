"""GPU tests of per-query tag filters (nk_search_filtered): one corpus pass for a batch whose queries carry different
filters.  Every result is checked against an fp64 brute force over each query's admissible rows; the thresholds the
kernels prune with are attacked directly (a query's true unfiltered best rows made inadmissible)."""
import numpy as np
import pytest

from parity import check_parity, exact_scores_for

pytestmark = pytest.mark.gpu

PAD = 0xFFFFFFFF
ALL = 0xFFFFFFFFFFFFFFFF
RARE_BIT = 1 << 40  # set on only a handful of rows: fewer admissible rows than k


def mixed_filters(Q):
    """The filter kinds a mixed batch carries, cycled over the queries (tags: bits 0..15 random with p = 1/2)."""
    kinds = [
        (0, 0, 0),                  # no filter
        (1 << 0, 0, 0),             # all_of, ~50%
        (0, 1 << 1, 0),             # none_of, ~50%
        (0, 0, (1 << 2) | (1 << 3)),  # any_of, ~75%
        (0b1111111 << 4, 0, 0),     # all_of 7 bits, < 1%
        (RARE_BIT, 0, 0),           # fewer admissible rows than k
        (ALL, ALL, 0),              # admits no row
        ((1 << 5) | (1 << 6), 1 << 7, (1 << 8) | (1 << 9)),  # all three
    ]
    return np.array([kinds[q % len(kinds)] for q in range(Q)], dtype=np.uint64)


def make_tags(n, seed):
    from nornicdb_b200.knn import synthetic_tags
    t = synthetic_tags(n, seed) & np.uint64(0xFFFF)
    t[np.arange(3, n, max(n // 5, 1))[:5]] |= np.uint64(RARE_BIT)
    return t


def admissible(tags, filters):
    from nornicdb_b200.knn import admits
    return np.stack([admits(tags, *[int(v) for v in f]) for f in filters])


def fp64_scores(rows, q, metric):
    x = np.asarray(rows, dtype=np.float64)
    qq = np.asarray(q, dtype=np.float64)
    s = qq @ x.T
    if metric == "cosine":
        den = np.linalg.norm(qq, axis=1)[:, None] * np.linalg.norm(x, axis=1)[None, :]
        with np.errstate(invalid="ignore", divide="ignore"):
            s = np.where(den > 0, s / den, 0.0)
    elif metric == "euclidean":
        s = -np.sqrt(np.maximum((qq * qq).sum(1)[:, None] + (x * x).sum(1)[None, :] - 2.0 * s, 0.0))
    return s


def check_filtered(rows, q, k, metric, gi, gs, adm, swap_eps=2e-6):
    """gi / gs [Q, k'] against the fp64 top-k of each query's admissible rows (adm [Q, n]); slots past a query's admissible
    rows must be padding."""
    Q = q.shape[0]
    S = fp64_scores(rows, q, metric)
    swaps = 0
    for qi in range(Q):
        cand = np.flatnonzero(adm[qi])
        m = min(k, len(cand), gi.shape[1])
        got = gi[qi].astype(np.int64)
        assert (got[m:] == PAD).all() and (gs[qi][m:] == 0).all(), (qi, got, gs[qi])
        assert adm[qi][got[:m]].all(), f"query {qi}: inadmissible row returned {got[:m][~adm[qi][got[:m]]]}"
        if m == 0:
            continue
        sc = S[qi, cand]
        order = np.lexsort((cand, -sc))[:m]
        oi = cand[order][None, :]
        os_ = sc[order][None, :]
        if metric == "euclidean":
            os_ = -os_
        swaps += check_parity(rows, q[qi:qi + 1], m, metric, got[None, :m], gs[qi:qi + 1, :m], oi, os_, swap_eps=swap_eps)
    return swaps


def rows_of(ix, rows):
    """What the device holds (16-bit corpora: the rounded rows), as fp32."""
    from nornicdb_b200.knn import from_bf16_bits
    back = ix.read_rows(0, len(rows))
    return from_bf16_bits(back) if ix.dtype == 2 else back.astype(np.float32)


CASES = ([("simt", 3, m, "f32") for m in ("cosine", "dot", "euclidean")]
         + [("shadow", 40, m, dt) for m in ("cosine", "dot", "euclidean") for dt in ("f32", "f16", "bf16")]
         + [("filter", 40, m, "f32") for m in ("cosine", "dot", "euclidean")]
         + [("tensor", 40, m, "f32") for m in ("cosine", "dot")]
         + [("auto", 300, m, "f32") for m in ("cosine", "dot", "euclidean")])


@pytest.mark.parametrize("path,Q,metric,dtype", CASES)
def test_filtered_parity_every_path(knn_lib, oracle_mod, path, Q, metric, dtype):
    """Mixed batch ({0,0,0}, all_of, none_of, any_of, < 1%, fewer than k, none admissible) on every path: exact results
    over each query's admissible rows, padding where a query has fewer than k."""
    from nornicdb_b200.knn import KnnIndex
    n, d, k = 20_000, 128, 10
    rows = oracle_mod.fill_uniform(n, d, 11)
    q = oracle_mod.fill_uniform(Q, d, 12)
    tags = make_tags(n, 5)
    filters = mixed_filters(Q)
    ix = KnnIndex(d, metric=metric, dtype=dtype)
    try:
        ix.upload(rows)
        ix.set_row_tags(tags)
        ix.set_path(path)
        gi, gs = ix.search_filtered(q, k, filters)
        if path != "auto":
            assert ix.last_path() == path
        assert ix.debug_flags()[0] == 0
        held = rows_of(ix, rows)
    finally:
        ix.release()
    check_filtered(held, q, k, metric, gi, gs, admissible(tags, filters))


@pytest.mark.parametrize("path,Q", [("simt", 3), ("shadow", 40), ("filter", 40), ("tensor", 40), ("auto", 300)])
def test_inadmissible_best_rows_never_raise_a_threshold(knn_lib, oracle_mod, path, Q):
    """Each query's true unfiltered top 300 rows carry a bit the query excludes (none_of).  If a sample, prune, publish or
    flood step let one of them raise a threshold, admissible rows would be lost."""
    from nornicdb_b200.knn import KnnIndex
    n, d, k = 30_000, 128, 10
    metric = "dot" if path == "tensor" else "cosine"
    rows = oracle_mod.fill_uniform(n, d, 21)
    q = oracle_mod.fill_uniform(Q, d, 22)
    S = fp64_scores(rows, q, metric)
    tags = np.zeros(n, dtype=np.uint64)
    filters = np.zeros((Q, 3), dtype=np.uint64)
    for qi in range(Q):
        bit = np.uint64(1 << (qi % 64))
        top = np.argsort(-S[qi], kind="stable")[:300]
        tags[top] |= bit
        filters[qi, 1] = bit
    ix = KnnIndex(d, metric=metric)
    try:
        ix.upload(rows)
        ix.set_row_tags(tags)
        ix.set_path(path)
        gi, gs = ix.search_filtered(q, k, filters)
    finally:
        ix.release()
    check_filtered(rows, q, k, metric, gi, gs, admissible(tags, filters))


@pytest.mark.parametrize("path", ["simt", "shadow", "filter", "tensor"])
def test_same_filter_everywhere_equals_row_mask(knn_lib, oracle_mod, path):
    """One filter for the whole batch gives bit-identical results to nk_search under the equivalent row mask, and {0,0,0}
    queries bit-identical results to plain nk_search (exact re-scoring: the same arithmetic picks the same rows)."""
    from nornicdb_b200.knn import KnnIndex, admits
    n, d, k, Q = 20_000, 256, 10, (3 if path == "simt" else 40)
    rows = oracle_mod.fill_uniform(n, d, 31)
    q = oracle_mod.fill_uniform(Q, d, 32)
    tags = make_tags(n, 6)
    f = ((1 << 0) | (1 << 1), 1 << 2, 0)
    ix = KnnIndex(d, metric="dot" if path == "tensor" else "cosine")
    try:
        ix.upload(rows)
        ix.set_row_tags(tags)
        ix.set_path(path)
        fi, fs = ix.search_filtered(q, k, np.tile(np.array(f, dtype=np.uint64), (Q, 1)))
        zi, zs = ix.search_filtered(q, k, np.zeros((Q, 3), dtype=np.uint64))
        pi, ps = ix.search(q, k)
        ix.set_row_mask(admits(tags, *f))
        mi, ms = ix.search(q, k)
    finally:
        ix.release()
    assert (fi == mi).all() and (fs.view(np.uint32) == ms.view(np.uint32)).all()
    assert (zi == pi).all() and (zs.view(np.uint32) == ps.view(np.uint32)).all()


@pytest.mark.parametrize("path,metric", [("simt", "cosine"), ("shadow", "cosine"), ("filter", "euclidean"), ("auto", "dot")])
def test_filters_combine_with_row_mask_and_score_floor(knn_lib, oracle_mod, path, metric):
    from nornicdb_b200.knn import KnnIndex
    n, d, k = 20_000, 128, 20
    Q = 3 if path == "simt" else 160
    rows = oracle_mod.fill_uniform(n, d, 41)
    q = oracle_mod.fill_uniform(Q, d, 42)
    tags = make_tags(n, 7)
    filters = mixed_filters(Q)
    mask = (np.arange(n) % 3) != 0
    floor = {"cosine": 0.05, "dot": 2.0, "euclidean": 9.0}[metric]
    ix = KnnIndex(d, metric=metric)
    try:
        ix.upload(rows)
        ix.set_row_tags(tags)
        ix.set_path(path)
        ix.set_row_mask(mask)
        ix.set_min_score(floor)
        gi, gs = ix.search_filtered(q, k, filters)
    finally:
        ix.release()
    S = fp64_scores(rows, q, metric)
    ok = S >= (-floor if metric == "euclidean" else floor)  # euclidean: S = -distance, the floor a maximum distance
    adm = admissible(tags, filters) & mask[None, :] & ok
    check_filtered(rows, q, k, metric, gi, gs, adm)


def _near_tie_corpus(oracle, n, noise, seed):
    rng = np.random.default_rng(seed)
    base = oracle.fill_uniform(1, 128, 9)[0]
    rows = np.tile(base, (n, 1)) + rng.standard_normal((n, 128)).astype(np.float32) * noise
    rows[::7] = oracle.fill_uniform(len(rows[::7]), 128, 10)
    q = (base[None, :] + rng.standard_normal((40, 128)).astype(np.float32) * 1e-3).astype(np.float32)
    return rows, q


@pytest.mark.parametrize("api", ["host", "device"])
@pytest.mark.parametrize("path,n,noise,metric", [
    pytest.param(path, n, noise, metric, id=f"{path}-{n}-{noise}" + ("" if metric == "cosine" else f"-{metric}"))
    for path, n, noise in [("filter", 20_000, 1e-5), ("shadow", 160_000, 1e-4)] for metric in ("cosine", "dot", "euclidean")])
def test_retry_and_exact_tail_honour_the_filters(knn_lib, oracle_mod, api, path, n, noise, metric):
    """The near-tie corpora of test_gpu_tensor.py overflow the filter stages; the retry / exact kernels (deferred by the
    host API, queued blindly by the device API: 3xTF32, or the CUDA-core scan for euclidean) must apply the same filters."""
    import torch
    from nornicdb_b200.knn import KnnIndex
    rows, q = _near_tie_corpus(oracle_mod, n, noise, 1 if path == "shadow" else 0)
    Q, k = q.shape[0], 10
    tags = make_tags(n, 8)
    filters = mixed_filters(Q)
    filters[::2] = 0  # unfiltered queries keep the margin buffers overflowing
    ix = KnnIndex(128, metric=metric)
    try:
        ix.upload(rows)
        ix.set_row_tags(tags)
        ix.set_path(path)
        if api == "host":
            gi, gs = ix.search_filtered(q, k, filters)
        else:
            qd = torch.from_numpy(q).cuda()
            fd = torch.from_numpy(filters.view(np.int64)).cuda()
            oi = torch.empty((Q, k), dtype=torch.int32, device="cuda")
            os_ = torch.empty((Q, k), dtype=torch.float32, device="cuda")
            ix.search_filtered_device(qd.data_ptr(), fd.data_ptr(), Q, k, oi.data_ptr(), os_.data_ptr(), 0)
            ix.status(0)
            gi, gs = oi.cpu().numpy().view(np.uint32), os_.cpu().numpy()
        flags = ix.debug_flags()
    finally:
        ix.release()
    assert flags[0] == 0
    if path == "shadow" and api == "host":
        assert flags[3] == 1, flags  # the 16-bit stage overflowed; the TF32 stage re-ran the search
    else:
        assert flags[1] != 0, flags  # a stage overflowed; the exact kernels answered
    check_filtered(rows, q, k, metric, gi, gs, admissible(tags, filters), swap_eps=5e-6)


@pytest.mark.parametrize("devices", [(0,), (0, 0)])
def test_tags_follow_the_rows(knn_lib, oracle_mod, devices):
    """set_row_tags on partial ranges (spanning shards), append, update_row, remove_swap, reset by upload."""
    from nornicdb_b200.knn import KnnIndex
    d = 64
    rows = oracle_mod.fill_uniform(600, d, 51)
    extra = oracle_mod.fill_uniform(50, d, 52)
    q = oracle_mod.fill_uniform(3, d, 53)
    B = 1 << 9
    flt = np.array([(B, 0, 0), (0, B, 0), (0, 0, 0)], dtype=np.uint64)
    ix = KnnIndex(d, metric="dot", devices=devices)
    ix.set_path("simt")
    try:
        ix.upload(rows)
        tags = np.zeros(600, dtype=np.uint64)
        tags[250:350] = B                      # a range crossing the shard boundary of (0, 0)
        ix.set_row_tags(tags[250:350], first_row=250)
        tags[10] = B
        ix.set_row_tags(tags[10:11], first_row=10)
        cur = rows.copy()

        def check():
            gi, gs = ix.search_filtered(q, 1024, flt)
            adm = admissible(tags, flt)
            for qi in range(3):
                got = gi[qi][gi[qi] != PAD]
                assert sorted(got.tolist()) == np.flatnonzero(adm[qi]).tolist(), qi
            check_filtered(cur, q, gi.shape[1], "dot", gi, gs, adm)

        check()
        ix.append(extra)                       # appended rows: tag 0
        tags = np.concatenate([tags, np.zeros(50, dtype=np.uint64)])
        cur = np.concatenate([cur, extra])
        check()
        ix.update_row(300, q[0] * 4.0)         # row keeps its tag
        cur[300] = q[0] * 4.0
        check()
        tags[-1] = B
        ix.set_row_tags(tags[-1:], first_row=len(tags) - 1)
        ix.remove_swap(20)                     # the last row (tagged) moves into slot 20 with its tag
        tags[20] = tags[-1]; tags = tags[:-1]
        cur[20] = cur[-1]; cur = cur[:-1]
        check()
        ix.remove_swap(280)                    # an untagged row moves into a tagged slot: the slot's tag becomes 0
        tags[280] = tags[-1]; tags = tags[:-1]
        cur[280] = cur[-1]; cur = cur[:-1]
        check()
        ix.upload(rows)                        # every tag back to 0
        tags = np.zeros(600, dtype=np.uint64)
        cur = rows.copy()
        check()
    finally:
        ix.release()


def test_headline_shape_mixed_filters_planted(knn_lib, oracle_mod):
    """N=10M d=1024 fp32 Q=64 k=10 cosine, mixed filters: planted near-copies the query admits come back first, planted ones
    it rejects never come back, every returned row is admissible and every score is recomputed in fp64."""
    from nornicdb_b200.knn import KnnIndex, admits, synthetic_tags
    n, d, Q, k = 10_000_000, 1024, 64, 10
    ix = KnnIndex(d, metric="cosine")
    try:
        ix.fill_uniform(n, 42)
        q = oracle_mod.fill_uniform(Q, d, 1337)
        tags = synthetic_tags(n, 3)
        ms = [0, 1, 3, 7, 10]
        filters = np.zeros((Q, 3), dtype=np.uint64)
        for qi in range(Q):
            filters[qi, 0] = (1 << ms[qi % 5]) - 1
        rows = np.random.default_rng(5).choice(n, size=2 * Q, replace=False)
        good = {qi: int(rows[2 * qi]) for qi in range(Q)}
        bad = {qi: int(rows[2 * qi + 1]) for qi in range(Q) if filters[qi, 0]}
        for qi in range(Q):
            ix.update_row(good[qi], (q[qi] * 1.5).astype(np.float32))
            tags[good[qi]] |= filters[qi, 0]           # admitted by its query
            if qi in bad:                              # the same near-copy, rejected: bit 0 (in every non-empty all_of) cleared
                ix.update_row(bad[qi], (q[qi] * 1.7).astype(np.float32))
                tags[bad[qi]] &= ~np.uint64(1)
        ix.set_row_tags(tags)
        gi, gs = ix.search_filtered(q, k, filters)
        assert ix.last_path() == "shadow" and ix.debug_flags()[0] == 0
        for qi in range(Q):
            f = [int(v) for v in filters[qi]]
            assert admits(tags[gi[qi].astype(np.int64)], *f).all(), qi
            assert gi[qi][0] == good[qi], (qi, gi[qi][:3], good[qi])
            if qi in bad:
                assert bad[qi] not in gi[qi].tolist(), qi
            r = np.stack([ix.read_rows(int(x), 1)[0] for x in gi[qi]])
            ex = exact_scores_for(r, q[qi], np.arange(k), "cosine")
            assert np.allclose(gs[qi], ex, rtol=1e-4, atol=1e-6), qi
            assert (np.diff(gs[qi].astype(np.float64)) <= 1e-7).all()
    finally:
        ix.release()


def test_q1024_mixed_filters_against_torch_fp64(knn_lib, oracle_mod):
    """Q=1024 (4 query groups per launch) with mixed filters: an fp64 brute force, slice by slice with torch on the same GPU,
    over the admissible rows of a sample of queries."""
    import torch
    from nornicdb_b200.knn import KnnIndex, fill_uniform_device, synthetic_tags
    n, d, Q, k = 10_000_000, 1024, 1024, 10
    ix = KnnIndex(d, metric="dot")
    try:
        ix.fill_uniform(n, 42)
        tags = synthetic_tags(n, 4)
        ix.set_row_tags(tags)
        q = oracle_mod.fill_uniform(Q, d, 1337)
        ms = [0, 1, 3, 7, 10]
        filters = np.zeros((Q, 3), dtype=np.uint64)
        for qi in range(Q):
            filters[qi, 0] = (1 << ms[qi % 5]) - 1
        gi, gs = ix.search_filtered(q, k, filters)
        assert ix.last_path() == "shadow" and ix.debug_flags()[0] == 0
        sample = list(range(0, Q, 37))
        tg = torch.from_numpy(tags.view(np.int64)).cuda()
        q64 = torch.from_numpy(q[sample].astype(np.float64)).cuda()
        fl = torch.from_numpy(filters[sample, 0].view(np.int64)).cuda()
        best_s = best_i = None
        for lo in range(0, n, 250_000):
            cnt = min(250_000, n - lo)
            x = torch.empty((cnt, d), dtype=torch.float32, device="cuda")
            fill_uniform_device(0, x.data_ptr(), cnt, d, 42, lo, 0)
            torch.cuda.synchronize()
            s = x.double() @ q64.T
            ok = (tg[lo:lo + cnt, None] & fl[None, :]) == fl[None, :]
            s = torch.where(ok, s, torch.full_like(s, -np.inf))
            v, i = torch.topk(s, k + 8, dim=0)
            i = i + lo
            best_s = v if best_s is None else torch.cat([best_s, v])
            best_i = i if best_i is None else torch.cat([best_i, i])
            keep = torch.topk(best_s, k + 8, dim=0).indices
            best_s, best_i = torch.gather(best_s, 0, keep), torch.gather(best_i, 0, keep)
        bs, bi = best_s.T.cpu().numpy(), best_i.T.cpu().numpy()
        for j, qi in enumerate(sample):
            order = np.lexsort((bi[j], -bs[j]))[:k]
            oi, os_ = bi[j][order][None, :], bs[j][order][None, :]
            check_parity(lambda idx: np.stack([ix.read_rows(int(r), 1)[0] for r in idx]), q[qi:qi + 1], k, "dot",
                         gi[qi:qi + 1], gs[qi:qi + 1], oi, os_)
    finally:
        ix.release()
