"""The dimension edges of tests/dims.py and the shared memory each d-dependent launch requests, without a GPU.

Static shared memory is read from the built objects with `cuobjdump -res-usage` (static + the 1 KB per-block reservation,
the figure the library also counts); the opt-in limit is an H100's.  For every d a path admits, its launches must fit:
otherwise the planner promises a shape that cudaFuncSetAttribute then refuses."""
import pytest

import dims


@pytest.fixture(scope="module")
def statics(knn_lib):
    return {
        "finish": dims.kernel_static("scan_tensor", r"filter_finish_kernel"),
        "prep": dims.kernel_static("scan_tensor", r"filter_prep_kernel"),
        "rescore": dims.kernel_static("range", r"range_rescore\w*_kernel"),
        "group": dims.kernel_static("rowops", r"group_best_kernel"),
        "simt": dims.kernel_static("scan_simt", r"knn_scan_simt_kernel"),
    }


def test_each_edge_has_both_neighbours_and_the_rule_changes_across_it(statics):
    e = dims.edges(statics)
    for name, ds in e.items():
        assert len(ds) >= 2 and ds == sorted(set(ds)), (name, ds)
    # the rule each edge names does change between its two sides
    lo, hi = e["filter admission"]
    assert dims.filter_admits(lo) and not dims.filter_admits(hi)
    lo, hi = e["finish window"]
    big, small = dims.finish_windows()[:2]
    assert dims.finish_window(lo, statics["finish"]) == big and dims.finish_window(hi, statics["finish"]) == small
    lo, hi = e["prep opt-in at the largest sample"]
    assert dims.prep_smem(lo, 2048) <= dims.DEFAULT_SMEM < dims.prep_smem(hi, 2048)
    assert dims.prep_sample(192, 128, 4099) == 2048
    lo, hi = e["4d-byte query opt-in"]
    assert lo * 4 <= dims.DEFAULT_SMEM < hi * 4
    lo, hi = e["SIMT refusal"]
    P = dims.simt_cap_for_k(10)
    assert P * 8 + lo * 4 + statics["simt"] <= dims.OPTIN_H100 < P * 8 + hi * 4 + 1024
    assert dims.filter_admits(31) is False and dims.filter_admits(32) and not dims.filter_admits(33)
    assert dims.filter_admits(40, "bf16") and not dims.filter_admits(36, "f16")
    for name, ds in e.items():
        if name.startswith("SIMT group"):
            qt, k = int(name.split()[2]), int(name.split("k=")[1])
            lo, hi = ds
            # Q = 13 runs every group size the budget leaves at lo; one past the edge the first group is halved
            assert dims.simt_groups(lo, k, 13)[0] == qt and dims.simt_groups(hi, k, 13)[0] == qt // 2, (name, ds)
    # the three P bands
    assert [dims.simt_cap_for_k(k) for k in (255, 256, 767, 768, 1024)] == [512, 1024, 1024, 2048, 2048]
    # the pads
    assert e["BF16 pad"] == [60, 64, 68] and e["int8 pad"] == [124, 128, 132] and e["ragged TF32 slab"] == [100, 124]


def test_every_admitted_d_fits_the_shared_memory_it_requests(statics):
    """Every d the filters admit gets a finish window that fits; the prep kernel at the largest sample, range re-scoring and
    group search fit there too; the headline d = 1024 keeps the larger window."""
    windows = dims.finish_windows()
    optin = dims.OPTIN_H100
    for dtype in ("f32", "bf16"):
        for d in range(32, dims.FILTER_MAX_DIM + 8, 4):
            if not dims.filter_admits(d, dtype):
                continue
            fits = [w for w in windows if dims.finish_smem(w, d) + statics["finish"] <= optin]
            assert fits, (f"d={d}: the filter admits it but no finish window fits: "
                          f"{[(w, dims.finish_smem(w, d) + statics['finish']) for w in windows]} B > {optin} B")
            assert dims.prep_smem(d, 2048) + statics["prep"] <= optin, d
            assert d * 4 + statics["rescore"] <= optin, d
    assert dims.finish_window(1024, statics["finish"]) == windows[0] == 16384
    # group search and the CUDA-core scan serve every d up to the CUDA-core refusal
    d = dims.simt_max_dim(10, statics["simt"])
    assert d * 4 + statics["group"] <= optin and dims.simt_cap_for_k(10) * 8 + d * 4 + statics["simt"] <= optin
