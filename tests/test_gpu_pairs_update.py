"""GPU tests of the self-join kept current: nk_search_pairs_rows (the pairs of the whole-index join incident to listed rows) and
nk_pairs_remap (a stored join brought up to date after appends, rewrites, removals, retags and re-valued rows).

The contract of the incident call: the whole-index nk_search_pairs[_windowed] with the same arguments, on the graph path,
restricted to the pairs with a listed end and grouped by that end (a pair with both ends listed under the lower one), bit
for bit: ids, scores, order and offsets.  The remap must equal a fresh whole-index join with the path forced, bit for bit."""
import zlib

import numpy as np
import pytest

from test_gpu_search_pairs import assert_same, threshold_for
from test_gpu_search_rows import stored_f32

pytestmark = pytest.mark.gpu


def make_index(rows, metric, dtype="f32", devices=(0,), path="shadow"):
    from nornicdb_b200.knn import KnnIndex
    ix = KnnIndex(rows.shape[1], metric=metric, dtype=dtype, devices=devices)
    ix.upload_from_f32(rows)
    ix.set_path(path)
    return ix


def restrict(whole, listed, metric):
    """The whole-index join's pairs with an end in `listed`, grouped by that end (both ends listed: the lower one), each list
    in nk_search's order -> CSR.  Under euclidean two keys can decode to one distance, so there the order within equal
    distances is taken by row (the caller compares sorted lists)."""
    off, idx, sc = whole
    o = off.astype(np.int64)
    n = len(o) - 1
    listed = np.asarray(listed, dtype=np.int64)
    is_listed = np.zeros(n, dtype=bool)
    is_listed[listed] = True
    lists = {int(c): ([], []) for c in listed}
    for i in range(n):
        js = idx[o[i]:o[i + 1]].astype(np.int64)
        ss = sc[o[i]:o[i + 1]]
        if is_listed[i]:
            lists[i][0].extend(js.tolist())
            lists[i][1].extend(ss.tolist())
        for j, s in zip(js, ss):
            if is_listed[j] and not is_listed[i]:
                lists[int(j)][0].append(i)
                lists[int(j)][1].append(s)
    out_off, out_idx, out_sc = [0], [], []
    for c in listed:
        j = np.asarray(lists[int(c)][0], dtype=np.int64)
        s = np.asarray(lists[int(c)][1], dtype=np.float32)
        order = np.lexsort((j, s if metric == "euclidean" else -s))
        out_idx.append(j[order])
        out_sc.append(s[order])
        out_off.append(out_off[-1] + len(j))
    cat = lambda a, dt: np.concatenate(a).astype(dt) if a else np.empty(0, dt)
    return np.asarray(out_off, np.uint64), cat(out_idx, np.uint32), cat(out_sc, np.float32)


def sorted_lists(res, metric):
    """Each list sorted by (score desc / distance asc, row asc): the order of restrict()."""
    off, idx, sc = res
    o = off.astype(np.int64)
    ii, ss = idx.copy(), sc.copy()
    for r in range(len(o) - 1):
        j, s = idx[o[r]:o[r + 1]], sc[o[r]:o[r + 1]]
        order = np.lexsort((j, s if metric == "euclidean" else -s))
        ii[o[r]:o[r + 1]], ss[o[r]:o[r + 1]] = j[order], s[order]
    return off, ii, ss


def check_incident(ix, t, listed, metric, what, **kw):
    """search_pairs_rows against restrict(search_pairs).  Under euclidean the lists are compared after sorting by (distance,
    row): two squared distances one ulp apart decode to one distance and are ordered by their keys, not by row, and the
    decoded join cannot say which comes first.  So there only the ascending distances and the pair sets are checked here; the
    full order under euclidean is checked by the remap test, whose two sides both come from keys."""
    whole = ix.search_pairs(t, **kw)
    want = restrict(whole, listed, metric)
    got = ix.search_pairs_rows(listed, t, **kw)
    if metric == "euclidean":
        o = got[0].astype(np.int64)
        for r in range(len(o) - 1):
            assert np.all(np.diff(got[2][o[r]:o[r + 1]]) >= 0), f"{what}: list {r} out of order"
        got = sorted_lists(got, metric)
    assert_same(got, want, what)
    return got


def listed_sets(n, seed):
    rng = np.random.default_rng(seed)
    a = rng.choice(n, size=min(n, 1500), replace=False)  # two blocks of queries, many pairs between listed rows
    return {"random": a.astype(np.uint32), "few": np.array([n - 1, 3, 700], np.uint32),
            "tail": np.arange(n - 300, n, dtype=np.uint32)}


CASES = [("cosine", "f32", "shadow", None), ("dot", "f32", "shadow", None), ("euclidean", "f32", "shadow", None),
         ("cosine", "f32", "shadow", "int8"), ("euclidean", "f32", "shadow", "int8"), ("cosine", "f32", "filter", None),
         ("dot", "f32", "filter", None), ("cosine", "f16", "shadow", None), ("euclidean", "f16", "shadow", None),
         ("cosine", "bf16", "shadow", None), ("dot", "bf16", "shadow", None)]


@pytest.mark.parametrize("metric,dtype,path,image", CASES)
def test_incident_equals_whole_join(knn_lib, oracle_mod, monkeypatch, metric, dtype, path, image):
    if image:
        monkeypatch.setenv("NK_SHADOW", image)
    n, d = 3100, 64
    rows = oracle_mod.fill_uniform(n, d, 201)
    t = threshold_for(rows, metric, 12)
    ix = make_index(rows, metric, dtype, path=path)
    for name, listed in listed_sets(n, 202).items():
        check_incident(ix, t, listed, metric, f"{metric} {dtype} {path} {image}: {name}")
    # AUTO runs the graph path: the same result as the forced one
    ix.set_path("auto")
    listed = listed_sets(n, 202)["random"]
    auto = ix.search_pairs_rows(listed, t)
    ix.set_path(path)
    assert_same(auto, ix.search_pairs_rows(listed, t), "AUTO")
    ix.release()


def test_every_row_is_the_join_regrouped_and_the_empty_set(knn_lib, oracle_mod):
    n, d = 2100, 64
    rows = oracle_mod.fill_uniform(n, d, 203)
    t = threshold_for(rows, "cosine", 10)
    ix = make_index(rows, "cosine")
    every = ix.search_pairs_rows(np.arange(n), t)
    assert_same(every, ix.search_pairs(t), "every row listed, in order: the join itself")
    rev = np.arange(n)[::-1].astype(np.uint32)
    check_incident(ix, t, rev, "cosine", "every row, reversed")
    off, idx, sc = ix.search_pairs_rows([], t)
    assert off.tolist() == [0] and idx.size == 0 and sc.size == 0
    ix.release()


def test_two_shards(knn_lib, oracle_mod):
    n, d = 4100, 64
    rows = oracle_mod.fill_uniform(n, d, 204)
    t = threshold_for(rows, "dot", 10)
    one = make_index(rows, "dot")
    two = make_index(rows, "dot", devices=(0, 0))
    listed = np.r_[np.arange(n // 2 - 200, n // 2 + 200), [0, n - 1]].astype(np.uint32)  # straddles the shard boundary
    for path in ("shadow", "filter"):
        one.set_path(path)
        two.set_path(path)
        got = check_incident(two, t, listed, "dot", f"{path}: two shards")
        assert_same(got, one.search_pairs_rows(listed, t), f"{path}: two shards vs one")
    one.release()
    two.release()


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_mask_filter_nan_inf_zero_and_duplicates(knn_lib, oracle_mod, metric):
    from nornicdb_b200.knn import synthetic_tags
    n, d = 2600, 64
    rows = oracle_mod.fill_uniform(n, d, 205)
    dups = [5, 300, 1500, 2599]
    rows[dups] = rows[5]
    rows[800, 3] = np.nan
    rows[900, 7] = np.inf
    rows[1000] = 0.0
    t = threshold_for(np.delete(rows, [800, 900], axis=0), metric, 8)
    ix = make_index(rows, metric)
    listed = np.array(dups + [800, 900, 1000, 17, 2000], np.uint32)
    check_incident(ix, t, listed, metric, "nan / inf / zero rows")
    whole = ix.search_pairs(t)
    o = whole[0].astype(np.int64)
    t_dup = whole[2][o[5]:o[6]][whole[1][o[5]:o[6]] == 300][0]  # the duplicates' own score: pairs exactly at the threshold
    got = check_incident(ix, t_dup, listed, metric, "threshold = the duplicates' score")
    g = got[0].astype(np.int64)
    assert sorted(got[1][g[0]:g[1]].tolist()) == [300, 1500, 2599], "row 5 lists the other duplicates"
    assert g[4] == g[5] and g[5] == g[6], "rows with a NaN or an Inf component pair with nothing"
    if metric == "cosine":
        z = ix.search_pairs_rows([1000], -0.5)
        assert_same(z, restrict(ix.search_pairs(-0.5), [1000], metric), "zero row")
        assert np.all(z[2] == 0.0) and z[1].size >= n - 3
    # mask and a tag filter: masked and refused listed rows have no pairs, and no pair reaches them
    tags = synthetic_tags(n, 9) & np.uint64(0xF)
    keep = np.ones(n, dtype=bool)
    keep[::41] = False
    ix.set_row_tags(tags)
    ix.set_row_mask(keep)
    flt = (0, 2, 0)
    listed = np.r_[np.arange(0, n, 7), [41, 82]].astype(np.uint32)
    listed = np.unique(listed)
    got = check_incident(ix, t, listed, metric, "mask + filter", filter=flt)
    adm = keep & ((tags & np.uint64(2)) == 0)
    g = got[0].astype(np.int64)
    for r, c in enumerate(listed):
        if not adm[c]:
            assert g[r] == g[r + 1], f"inadmissible listed row {c} has pairs"
    assert adm[got[1].astype(np.int64)].all()
    ix.release()


def test_refusals(knn_lib, oracle_mod):
    from nornicdb_b200.knn import KnnError
    n, d = 600, 32
    rows = oracle_mod.fill_uniform(n, d, 206)
    ix = make_index(rows, "cosine")
    with pytest.raises(KnnError, match="listed twice"):
        ix.search_pairs_rows([3, 9, 3], 0.1)
    with pytest.raises(KnnError, match="out of range"):
        ix.search_pairs_rows([3, n], 0.1)
    with pytest.raises(KnnError, match="NaN"):
        ix.search_pairs_rows([3], float("nan"))
    for p in ("simt", "tensor"):
        ix.set_path(p)
        with pytest.raises(KnnError, match="filter paths"):
            ix.search_pairs_rows([3], 0.1)
        with pytest.raises(KnnError, match="filter paths"):
            ix.remap_pairs((np.zeros(n + 1, np.uint64), [], []), n, np.arange(n), 0.1)
    ix.release()


def test_library_refusals_through_the_c_abi(knn_lib, oracle_mod):
    """The C calls' own refusals, past the Python layer's checks: a null pointer with n > 0 and an old CSR that is not one
    (offsets not starting at 0 or decreasing, an entry that is not an old row above its owner, a repeated source row).
    Nothing is written to the output offsets on a refusal."""
    import ctypes as C
    from nornicdb_b200.knn import NO_GAP
    n, d = 300, 32
    rows = oracle_mod.fill_uniform(n, d, 210)
    ix = make_index(rows, "cosine")
    lib = ix.lib
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    total = C.c_uint64(7)
    off = np.full(n + 1, 99, np.uint64)
    rows_ok = np.array([3, 5], np.uint32)
    assert lib.nk_search_pairs_rows(ix.ptr, None, 2, C.c_float(0.1), None, 0, vp(off), None, None, C.byref(total)) == -1
    assert "null" in lib.nk_last_error().decode()
    assert lib.nk_search_pairs_rows(ix.ptr, vp(rows_ok), 2, C.c_float(0.1), None, 0, None, None, None, C.byref(total)) == -1
    assert lib.nk_search_pairs_rows(ix.ptr, vp(rows_ok), 2, C.c_float(0.1), None, 0, vp(off), None, None, None) == -1
    assert lib.nk_search_pairs_rows(ix.ptr, vp(np.array([3, 3], np.uint32)), 2, C.c_float(0.1), None, 0, vp(off), None, None,
                                    C.byref(total)) == -1
    assert "listed twice" in lib.nk_last_error().decode()
    assert (off == 99).all() and total.value == 7, "a refused call wrote its outputs"

    src = np.arange(n, dtype=np.uint32)
    o_idx = np.array([2], np.uint32)
    o_sc = np.array([0.5], np.float32)

    def remap(old_off, old_idx=o_idx, s=src):
        return lib.nk_pairs_remap(ix.ptr, C.c_float(0.1), None, None, NO_GAP, n, vp(s), vp(old_off), vp(old_idx), vp(o_sc), 0, vp(off),
                                  None, None, C.byref(total), None, None)

    good = np.zeros(n + 1, np.uint64)
    good[1:] = 1  # row 0 lists row 2
    assert remap(good) == 0 and total.value > 0
    off[:] = 99
    total.value = 7
    bad = good.copy()
    bad[0] = 1
    assert remap(bad) == -1 and "old_offsets[0]" in lib.nk_last_error().decode()
    bad = good.copy()
    bad[5] = 0
    assert remap(bad) == -1 and "decrease" in lib.nk_last_error().decode()
    below = good.copy()
    below[:4] = 0  # row 3 lists row 2: not above its owner
    assert remap(below) == -1 and "above" in lib.nk_last_error().decode()
    assert remap(good, np.array([n + 5], np.uint32)) == -1 and "not an old row" in lib.nk_last_error().decode()
    rep = src.copy()
    rep[4] = 3
    assert remap(good, s=rep) == -1 and "source of rows" in lib.nk_last_error().decode()
    assert lib.nk_pairs_remap(ix.ptr, C.c_float(0.1), None, None, NO_GAP, n, vp(src), vp(good), None, None, 0, vp(off), None, None,
                              C.byref(total), None, None) == -1, "null old pairs with old_offsets[n_old] > 0"
    assert (off == 99).all() and total.value == 7, "a refused call wrote its outputs"
    ix.release()


def test_orientation_trap_cosine(knn_lib, oracle_mod):
    """Pairs whose two orientations give different fp32 cosines: the incident call, listing only the higher row, must score the
    pair with the lower row as the query.  At a threshold equal to the higher of the two scores the pair appears iff the
    lower-row orientation meets it."""
    n, d = 1500, 100
    rows = oracle_mod.fill_uniform(n, d, 207)
    ix = make_index(rows, "cosine")
    x = stored_f32(ix)
    t0 = threshold_for(x, "cosine", 30)
    S = {}
    for b in range(0, n, 500):
        for qi, (i, s) in enumerate(ix.search_range(x[b:b + 500], t0 - 0.05)):
            for j, v in zip(i.tolist(), s.tolist()):
                S[(b + qi, j)] = np.float32(v)
    traps = [(i, j) for (i, j), v in S.items() if i < j and (j, i) in S and S[(j, i)].view(np.uint32) != v.view(np.uint32)]
    assert len(traps) >= 4, f"only {len(traps)} pairs whose orientations round differently"
    lower_wins = upper_wins = 0
    for i, j in traps[:40]:
        lo, hi = S[(i, j)], S[(j, i)]  # lo: row i (the lower) as the query, as the join scores the pair
        t = max(lo, hi)
        off, idx, sc = ix.search_pairs_rows([j], float(t))
        present = i in idx.tolist()
        assert present == (lo >= t), (i, j, lo, hi)
        if present:
            assert sc[idx.tolist().index(i)].view(np.uint32) == lo.view(np.uint32)
            lower_wins += 1
        else:
            upper_wins += 1
        assert_same((off, idx, sc), restrict(ix.search_pairs(float(t)), [j], "cosine"), f"trap {(i, j)}")
    assert lower_wins and upper_wins, (lower_wins, upper_wins)
    ix.release()


def test_windowed_and_filtered(knn_lib, oracle_mod):
    from nornicdb_b200.knn import synthetic_tags
    n, d = 3000, 64
    rows = oracle_mod.fill_uniform(n, d, 208)
    rng = np.random.default_rng(208)
    keys = rng.integers(1, 1000, size=n).astype(np.uint64)
    keys[::97] = 0  # rows without a value
    tags = synthetic_tags(n, 3) & np.uint64(0x7)
    t = threshold_for(rows, "cosine", 40)
    ix = make_index(rows, "cosine")
    ix.set_row_values(keys)
    ix.set_row_tags(tags)
    listed = np.unique(rng.choice(n, size=1200, replace=False)).astype(np.uint32)
    for kw in ({"window": (100, 800)}, {"max_gap": 50}, {"window": (0, 600), "max_gap": 20, "filter": (0, 4, 0)},
               {"filter": (1, 0, 0)}):
        check_incident(ix, t, listed, "cosine", f"{kw}", **kw)
    # rows re-valued across the band: listed rows and rows they pair with
    moved = listed[:50]
    keys[moved] = (keys[moved] + 500) % 999 + 1
    keys[listed[50:60]] = 0
    ix.set_row_values(keys)
    check_incident(ix, t, listed, "cosine", "re-valued", max_gap=50)
    check_incident(ix, t, moved, "cosine", "re-valued, listed alone", window=(100, 900), max_gap=30)
    ix.release()


@pytest.mark.parametrize("metric,dtype,devices,windowed", [("cosine", "f32", (0,), False), ("euclidean", "f32", (0, 0), False),
                                                          ("dot", "f16", (0,), True), ("cosine", "bf16", (0, 0), True)])
def test_remap_follows_mutation_sequences(knn_lib, oracle_mod, metric, dtype, devices, windowed):
    from nornicdb_b200.knn import GraphRowMap, KnnIndex
    n0, d = 1800, 64
    rng = np.random.default_rng(zlib.crc32(f"{metric} {dtype} {windowed}".encode()))
    rows = oracle_mod.fill_uniform(n0 + 2000, d, 209)
    t = threshold_for(rows[:n0], metric, 10)
    ix = KnnIndex(d, metric=metric, dtype=dtype, devices=devices)
    ix.upload_from_f32(rows[:n0])
    ix.set_path("shadow")
    keys = rng.integers(1, 500, size=n0).astype(np.uint64)
    tags = (rng.integers(0, 4, size=n0)).astype(np.uint64)
    kw = {"window": (20, 480), "max_gap": 40, "filter": (0, 2, 0)} if windowed else {}
    if windowed:
        ix.set_row_values(keys)
        ix.set_row_tags(tags)
    pairs = ix.search_pairs(t, **kw)
    spare = n0
    for step in range(6):
        n_old = len(ix)
        m = GraphRowMap(n_old)
        ops = rng.choice(["append", "update", "remove", "retag", "revalue"], size=8)
        for op in ops:
            n = len(ix)
            if op == "append":
                a = int(rng.integers(1, 300))
                ix.append(rows[spare:spare + a])
                spare = (spare + a) % (n0 + 1500)
                m.append(a)
                if windowed:
                    keys = np.r_[keys, rng.integers(1, 500, size=a).astype(np.uint64)]
                    tags = np.r_[tags, rng.integers(0, 4, size=a).astype(np.uint64)]
                    ix.set_row_values(keys[n:], n)
                    ix.set_row_tags(tags[n:], n)
            elif op == "update":
                r = int(rng.integers(0, n))
                ix.update_row(r, rows[int(rng.integers(0, n0))])
                m.update_row(r)
            elif op == "remove" and n > 40:
                for _ in range(int(rng.integers(1, 60 if step < 5 else n - 5))):
                    r = int(rng.integers(0, len(ix)))
                    ix.remove_swap(r)
                    m.remove_swap(r)
                    if windowed:
                        keys[r], tags[r] = keys[-1], tags[-1]
                        keys, tags = keys[:-1], tags[:-1]
            elif op == "retag" and windowed:
                r = rng.integers(0, n, size=5)
                tags[r] = rng.integers(0, 4, size=5).astype(np.uint64)
                ix.set_row_tags(tags)
                for x in r:
                    m.update_row(int(x))
            elif op == "revalue" and windowed:
                r = rng.integers(0, n, size=5)
                keys[r] = rng.integers(1, 500, size=5).astype(np.uint64)
                ix.set_row_values(keys)
                for x in r:
                    m.update_row(int(x))
        off, idx, sc, dropped, found = ix.remap_pairs(pairs, n_old, m, t, **kw)
        fresh = ix.search_pairs(t, **kw)
        assert_same((off, idx, sc), fresh, f"step {step} ({list(ops)}): remap vs fresh join")
        src = m.src_of_row
        changed = np.flatnonzero(src != np.arange(len(src)))
        n_inc = int(ix.search_pairs_rows(changed, t, **kw)[0][-1]) if changed.size else 0
        assert found == n_inc, (found, n_inc)
        assert int(pairs[0][-1]) - dropped == int(fresh[0][-1]) - found, "carried pairs: old - dropped = new - found"
        pairs = fresh
    ix.release()
