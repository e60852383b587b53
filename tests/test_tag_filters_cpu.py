"""Per-query tag filters without a GPU: the admissibility predicate restated in numpy, the label helper of knn.py and the
C ABI declarations / bindings of nk_index_set_row_tags, nk_search_filtered and nk_search_filtered_device."""
import os
import re

import numpy as np
import pytest

from nornicdb_b200.knn import ADMIT_NONE, ALL_BITS, KnnError, Labels, admits, as_filters, synthetic_tags

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def admits_py(tag, all_of, none_of, any_of):
    return (tag & all_of) == all_of and (tag & none_of) == 0 and (any_of == 0 or (tag & any_of) != 0)


def test_predicate_matches_its_definition():
    rng = np.random.default_rng(0)
    tags = rng.integers(0, 2**63, size=400, dtype=np.uint64) | (rng.integers(0, 2, size=400, dtype=np.uint64) << np.uint64(63))
    tags[:4] = [0, ALL_BITS, 1, 1 << 63]
    filters = [(0, 0, 0), ADMIT_NONE, (1, 0, 0), (0, 1, 0), (0, 0, 1), (1 << 63, 0, 0), (0, 0, (1 << 63) | 1)]
    for _ in range(60):
        a, n, s = (int(rng.integers(0, 2**63)) & int(rng.integers(0, 2**63)) for _ in range(3))
        filters.append((a, n & ~a, s))
    for f in filters:
        want = np.array([admits_py(int(t), *f) for t in tags])
        assert (admits(tags, *f) == want).all(), f


def test_predicate_edge_cases():
    tags = np.array([0, 1, 2, 3, ALL_BITS], dtype=np.uint64)
    assert admits(tags, 0, 0, 0).all()                          # {0,0,0} admits every row, untagged ones included
    assert not admits(tags, *ADMIT_NONE).any()                  # all_of = none_of = ~0 admits nothing
    assert admits(tags, 1, 0, 0).tolist() == [False, True, False, True, True]
    assert admits(tags, 0, 1, 0).tolist() == [True, False, True, False, False]
    assert admits(tags, 0, 0, 3).tolist() == [False, True, True, True, True]


def test_filtered_topk_needs_thresholds_over_admissible_pairs_only():
    """The keep rule in numpy: a running threshold built from admissible pairs only returns the filtered top-k; one that
    also counted inadmissible pairs (what a missed predicate in a prune / sample step would do) loses admissible rows."""
    rng = np.random.default_rng(1)
    n, k = 5000, 10
    s = rng.standard_normal(n)
    tags = synthetic_tags(n, 9)
    best = np.argsort(-s)[:300]
    tags[best] |= np.uint64(1 << 5)
    adm = admits(tags, 0, 1 << 5, 0)
    want = np.flatnonzero(adm)[np.argsort(-s[adm], kind="stable")[:k]]

    def scan(count_inadmissible):
        tau, buf = -np.inf, []
        for lo in range(0, n, 256):
            r = np.arange(lo, min(n, lo + 256))
            ok = (s[r] >= tau) & (adm[r] | count_inadmissible)
            buf.extend(r[ok].tolist())
            if len(buf) > k:
                buf = sorted(buf, key=lambda i: (-s[i], i))
                tau = s[buf[k - 1]]
                buf = buf[:k]
        return [i for i in sorted(buf, key=lambda i: (-s[i], i)) if adm[i]][:k]

    assert scan(False) == want.tolist()
    assert scan(True) != want.tolist()


def test_labels_map_names_to_bits():
    lab = Labels(["Person"])
    t = lab.row_tags([["Person"], ["Person", "Admin"], [], ["Doc"]])
    assert t.dtype == np.uint64 and t.tolist() == [1, 3, 0, 4]
    assert lab.filter() == (0, 0, 0)
    assert lab.filter(must=["Person"], must_not=["Admin"]) == (1, 2, 0)
    assert lab.filter(should=["Admin", "Doc"]) == (0, 0, 6)
    f = lab.filter(must=["Person"], must_not=["Admin"])
    assert admits(t, *f).tolist() == [True, False, False, False]


def test_labels_unknown_names():
    lab = Labels(["A", "B"])
    assert lab.filter(must=["A", "nope"]) == ADMIT_NONE           # a condition no row can meet
    assert lab.filter(must_not=["nope"]) == (0, 0, 0)             # excluding an absent label excludes nothing
    assert lab.filter(should=["nope", "B"]) == (0, 0, 2)          # unknown should names are ignored ...
    assert lab.filter(should=["nope", "zilch"]) == ADMIT_NONE     # ... unless all of them are unknown
    assert "nope" not in lab.bits                                 # filters never assign bits


def test_labels_hold_64_names_and_refuse_the_65th():
    lab = Labels([f"l{i}" for i in range(64)])
    assert lab.bit("l63") == 1 << 63
    t = lab.row_tags([[f"l{i}" for i in range(64)]])
    assert int(t[0]) == ALL_BITS
    with pytest.raises(KnnError):
        lab.bit("l64")
    with pytest.raises(KnnError):
        lab.row_tags([["l64"]])


def test_filter_array_layout():
    f = as_filters([(1, 2, 3), (4, 5, 6)], 2)
    assert f.dtype == np.uint64 and f.flags.c_contiguous and f.shape == (2, 3)
    assert f.tobytes() == np.array([1, 2, 3, 4, 5, 6], dtype="<u8").tobytes()  # NkFilter { all_of, none_of, any_of }
    with pytest.raises(KnnError):
        as_filters([(1, 2, 3)], 2)


def test_synthetic_tags_are_deterministic_fair_bits():
    t = synthetic_tags(100_000, 7)
    assert (t == synthetic_tags(100_000, 7)).all() and not (t == synthetic_tags(100_000, 8)).all()
    assert (synthetic_tags(10, 7, row_base=50_000) == t[50_000:50_010]).all()
    bits = ((t[:, None] >> np.arange(64, dtype=np.uint64)[None, :]) & np.uint64(1)).mean(0)
    assert np.abs(bits - 0.5).max() < 0.01


def test_abi_declares_and_binds_the_filtered_calls():
    from nornicdb_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "nornic_knn.h")).read(), flags=re.S)
    m = re.search(r"typedef struct NkFilter \{(.*?)\} NkFilter;", src, flags=re.S)
    assert m and re.sub(r"\s+", " ", m.group(1)).strip() == "uint64_t all_of, none_of, any_of;"
    for name, nargs in (("nk_index_set_row_tags", 4), ("nk_search_filtered", 7), ("nk_search_filtered_device", 8)):
        decl = re.search(name + r"\s*\(([^)]*)\)", src)
        assert decl, name
        assert len(decl.group(1).split(",")) == nargs, name
        res, args = _lib.SIGNATURES[name]
        assert len(args) == nargs, name
