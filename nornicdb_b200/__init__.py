"""nornicdb_b200 — H100-native brute-force vector kNN behind NornicDB's pkg/gpu/cuda boundary.

Contents (only what the hot path needs; see DESIGN.md):
  csrc/      hand-written sm_90a CUDA kernels + the C ABI (include/nornic_knn.h)
  _lib       ctypes binding of libnornic_knn.so (fails loudly if the library is missing)
  cuda       mirror of the reference's Go package pkg/gpu/cuda (Device / Buffer / Search)
  knn        KnnIndex: the fused batched search API (nk_*)
  build      in-tree nvcc build of the shared library
"""
__version__ = "0.1.0"
