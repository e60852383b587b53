"""CPU-side checks of the drop-in boundary: the C-ABI library builds for sm_90a, loads, and exports every
symbol include/nornic_knn.h declares, with the binding table in lock-step.  No compute calls (no GPU here)."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "nornic_knn.h")


def declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = re.findall(r"\b((?:cuda|nk)_[a-z0-9_]+)\s*\(", src)
    return sorted(set(names))


def test_header_declares_the_reference_legacy_symbols():
    # Exactly the C functions of the cgo preamble, pkg/gpu/cuda/cuda_bridge.go:20-375.
    legacy = {
        "cuda_set_error", "cuda_get_last_error", "cuda_clear_error", "cuda_get_device_count", "cuda_is_available",
        "cuda_create_device", "cuda_release_device", "cuda_device_name", "cuda_device_memory",
        "cuda_device_compute_capability", "cuda_create_buffer", "cuda_release_buffer", "cuda_buffer_data",
        "cuda_buffer_size", "cuda_buffer_copy_to_host", "cuda_compute_norms", "cuda_normalize_vectors",
        "cuda_cosine_similarity", "cuda_topk",
    }
    assert legacy <= set(declared_symbols())


def test_library_exports_every_declared_symbol(knn_lib):
    from nornicdb_b200 import _lib
    syms = declared_symbols()
    assert len(syms) >= 40
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    missing = [s for s in syms if s not in exported]
    assert not missing, f"declared in nornic_knn.h but not exported: {missing}"
    # binding table covers the header, and nothing else
    assert sorted(_lib.SIGNATURES) == syms


def test_library_is_sm90a_and_self_contained(knn_lib):
    from nornicdb_b200 import _lib
    out = subprocess.run(["cuobjdump", "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    ldd = subprocess.run(["ldd", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "cublas" not in ldd and "torch" not in ldd  # plain C ABI: cudart (static) only


def test_error_convention_without_gpu(knn_lib):
    """0/-1 + thread-local message, NULL pointers on failure (cuda_bridge.go:20-33 convention)."""
    import ctypes as C
    from nornicdb_b200 import cuda
    if cuda.IsAvailable():
        pytest.skip("GPU present: covered by the -m gpu tests")
    assert cuda.DeviceCount() == 0
    with pytest.raises(cuda.ErrCUDANotAvailable):
        cuda.NewDevice(0)
    ids = (C.c_int * 1)(0)
    assert not knn_lib.nk_index_create(ids, 1, 8, 0, 0)
    assert knn_lib.nk_last_error()
    knn_lib.cuda_set_error(b"boom")
    assert knn_lib.cuda_get_last_error() == b"boom"
    knn_lib.cuda_clear_error()
    assert knn_lib.cuda_get_last_error() == b""
    assert cuda.GPUName() == "" and cuda.GPUMemoryMB() == 0


def test_product_package_never_imports_the_oracle():
    """The oracle is test infrastructure; a product path that routes through it voids parity claims."""
    pkg = os.path.join(ROOT, "nornicdb_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".hpp", ".cpp")):
                text = open(os.path.join(dirpath, f), errors="replace").read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, flags=re.M), f
                assert "liboracle" not in text, f


def test_blob_vectors_walks_the_id_table_without_a_gpu():
    """nk_blob_vectors (host-only): locates the fp32 payload of EmbeddingIndex.Serialize's format (gpu.go:2373-2412)."""
    import struct

    import numpy as np
    from nornicdb_b200.knn import KnnError, blob_vectors
    ids = ["a", "node-22", "", "ünïcode"]
    dims = 3
    vec = np.arange(len(ids) * dims, dtype="<f4")
    blob = struct.pack("<II", dims, len(ids))
    for s in ids:
        b = s.encode("utf-8")
        blob += struct.pack("<I", len(b)) + b
    off = len(blob)
    blob += vec.tobytes()
    assert blob_vectors(blob) == (dims, len(ids), off)
    assert off % 4 != 0  # the payload really is unaligned in this example
    for bad in (blob[:7], blob[:off - 3], blob[:-1]):
        with pytest.raises(KnnError):
            blob_vectors(bad)
