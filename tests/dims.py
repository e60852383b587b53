"""The dimensions d where a kernel's plan changes, computed from the rules the library applies, so that a test names each
edge by its rule rather than by a number.  Shared by tests/test_dims_cpu.py (the rules and the shared-memory sizes, no GPU)
and tests/test_gpu_dims.py (every path on both sides of every edge, against fp64).

The rules, and where the library applies them:
  * TF32 filter and 3xTF32 scans: 32-float K-slabs (tc::BK); fp32 rows need d % 4 == 0 and d >= 32, else CUDA cores.
    The 3xTF32 scan also stops at TENSOR_EXACT_MAX_DIM, where its accumulation error reaches the parity rule.
  * BF16 shadow rows are padded to a multiple of 64 columns, the int8 image's to a multiple of 128; fp16 / bf16 rows are
    scanned in place in 64-column boxes and need d % 8 == 0.
  * Filters: d <= FILTER_MAX_DIM (kernels.cuh), and a query row that fits the finish kernel's shared memory beside one of its
    cached-score windows (FINISH_HI / FINISH_HI_SMALL in scan_tensor.cu).
  * The query prep stages 4 ceil4(d) + 8 sample bytes; sample = clamp(next_pow2(8k), 128, 2048) for Q <= 128 on n >= 4096.
  * CUDA-core scan: query groups of 8 / 4 / 2 / 1 (4 / 1 on the scalar path) shrink while P*8 + qt*d*4 passes 96 KB,
    P = simt_cap_for_k(k); it refuses once one query row no longer fits the device.
  * Range re-scoring and group search stage the query in 4d bytes: opted in above 48 KB.
Shared memory counted as `cuobjdump -res-usage` counts it (static + the 1 KB per-block reservation), as the library does."""
from __future__ import annotations

import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "nornicdb_b200", "build")
CSRC = os.path.join(ROOT, "nornicdb_b200", "csrc")
CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")

OPTIN_H100 = 232_448        # cudaDeviceProp::sharedMemPerBlockOptin of an H100
DEFAULT_SMEM = 48 * 1024    # dynamic shared memory a launch gets without opting in
FILTER_MAX_DIM = 32_768
TENSOR_EXACT_MAX_DIM = 12_288  # the exact 3xTF32 scan (kernels.cuh)
BK = 32                     # TF32 K-slab (floats)
SHADOW_PAD = 64             # BF16 shadow row pad; 16-bit in-place box width
INT8_PAD = 128              # int8 image row pad
SIMT_BUDGET = 96 * 1024
SIMT_RT = 256
FINISH_CAP = 4096


def next_pow2(x: int) -> int:
    p = 1
    while p < x:
        p <<= 1
    return p


def simt_cap_for_k(k: int) -> int:
    return max(512, next_pow2(k + SIMT_RT + 1))


def simt_groups(d: int, k: int, Q: int, vec: bool = True) -> list:
    """query-group sizes of the CUDA-core scan's launches, in order (scan_simt)"""
    P, out, left = simt_cap_for_k(k), [], Q
    while left:
        qt = 8 if left >= 5 else 4 if left >= 3 else 2 if left == 2 else 1
        if not vec:
            qt = 4 if left >= 3 else 1
        while qt > 1 and P * 8 + qt * d * 4 > SIMT_BUDGET:
            qt = qt // 2 if vec else 1
        out.append(qt)
        left -= min(left, qt)
    return out


def simt_group_edges(k: int) -> dict:
    """qt -> the largest d (multiple of 4) at which a full group of qt queries still runs; past it the group halves"""
    P = simt_cap_for_k(k)
    return {qt: (SIMT_BUDGET - P * 8) // (qt * 4) // 4 * 4 for qt in (8, 4, 2)}


def simt_max_dim(k: int, static: int, optin: int = OPTIN_H100) -> int:
    """largest d (multiple of 4) the CUDA-core scan serves: one query row and the candidate buffer fit the device"""
    return (optin - static - simt_cap_for_k(k) * 8) // 4 // 4 * 4


def prep_sample(k: int, Q: int, n: int) -> int:
    if Q > 128 or n < 4096:
        return 0
    return min(max(next_pow2(8 * k), 128), 2048)


def prep_smem(d: int, sample: int) -> int:
    return (d + 3) // 4 * 4 * 4 + sample * 8


def finish_smem(window: int, d: int) -> int:
    return window * 4 + FINISH_CAP * 16 + d * 4


def finish_windows() -> list:
    """the finish kernel's cached-score windows, largest first, as scan_tensor.cu declares them"""
    src = open(os.path.join(CSRC, "scan_tensor.cu")).read()
    return sorted((int(v) for v in re.findall(r"constexpr int FINISH_HI\w* = (\d+);", src)), reverse=True)


def finish_window(d: int, static: int, optin: int = OPTIN_H100):
    """the window the filter plans at d (the largest that fits), None if none fits"""
    for w in finish_windows():
        if finish_smem(w, d) + static <= optin:
            return w
    return None


def finish_edge(window: int, static: int, optin: int = OPTIN_H100) -> int:
    """largest d (multiple of 4) whose finish launch fits beside `window`"""
    return (optin - static - finish_smem(window, 0)) // 4 // 4 * 4


def filter_admits(d: int, dtype: str = "f32") -> bool:
    return 32 <= d <= FILTER_MAX_DIM and d % (4 if dtype == "f32" else 8) == 0


def static_smem(obj: str) -> dict:
    """mangled kernel name -> static shared memory in bytes as `cuobjdump -res-usage` reports it (no GPU needed)"""
    out = subprocess.run([CUOBJDUMP, "-res-usage", obj], capture_output=True, text=True, check=True).stdout
    return {m.group(1): int(m.group(2)) for m in re.finditer(r"Function (\S+):\s*\n\s*REG:\d+ STACK:\d+ SHARED:(\d+)", out)}


def kernel_static(obj: str, pattern: str) -> int:
    """the largest static shared memory among the kernels of build/<obj>.o whose mangled name matches pattern"""
    found = [v for k, v in static_smem(os.path.join(BUILD, obj + ".o")).items() if re.search(pattern, k)]
    assert found, f"no kernel matching {pattern!r} in {obj}.o"
    return max(found)


def edges(statics: dict) -> dict:
    """edge name -> the d values on both sides of it.  statics: 'finish', 'simt' -> static shared memory (bytes)."""
    fin = statics["finish"]
    big = finish_windows()[0]
    e = {
        "tensor floor": [4, 28, 30, 31, 32, 33, 36],
        "ragged TF32 slab": [BK * 3 + 4, BK * 4 - 4],
        "BF16 pad": [SHADOW_PAD - 4, SHADOW_PAD, SHADOW_PAD + 4],
        "int8 pad": [INT8_PAD - 4, INT8_PAD, INT8_PAD + 4],
        "16-bit box tail": [36, 40, SHADOW_PAD - 8, SHADOW_PAD, SHADOW_PAD + 8],
        "prep opt-in at the largest sample": [(DEFAULT_SMEM - 2048 * 8) // 4, (DEFAULT_SMEM - 2048 * 8) // 4 + 4],
        "4d-byte query opt-in": [DEFAULT_SMEM // 4, DEFAULT_SMEM // 4 + 4],
        "finish window": [finish_edge(big, fin), finish_edge(big, fin) + 4],
        "filter admission": [FILTER_MAX_DIM, FILTER_MAX_DIM + 4],
        # served by every instantiation / refused by any (the least static figure is the 1 KB reservation alone)
        "SIMT refusal": [simt_max_dim(10, statics["simt"]), simt_max_dim(10, 1024) + 4],
    }
    for k in (10, 256, 800):
        for qt, d in simt_group_edges(k).items():
            e[f"SIMT group {qt} at k={k}"] = [d, d + 4]
    return e
