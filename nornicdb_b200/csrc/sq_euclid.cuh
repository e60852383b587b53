// sq_euclid.cuh — squaredEuclidean (kmeans.go:430-454, oracle orc_sq_euclid64) bit for bit, shared by the k-means
// assignment fix-up (assign_tensor.cu) and the k-means++ seeding passes (kmeanspp.cu).
#pragma once
#include <stdint.h>

namespace nk {

// fp32 differences, fp64 squares in four interleaved sums (element j into s[j % 4]), the tail past the last whole group
// of four into s0, then ((s0 + s1) + s2) + s3.  Explicit round-to-nearest intrinsics: nvcc would contract a * b + c into
// an fma and change the rounding.  A caller that streams a row in pieces calls sq_add4 / sq_add_tail on the groups in
// ascending order and gets sq_euclid64's sums.
__device__ __forceinline__ void sq_add4(double &s0, double &s1, double &s2, double &s3, float x0, float x1, float x2, float x3,
                                        float c0, float c1, float c2, float c3) {
    const double d0 = (double)__fsub_rn(x0, c0), d1 = (double)__fsub_rn(x1, c1);
    const double d2 = (double)__fsub_rn(x2, c2), d3 = (double)__fsub_rn(x3, c3);
    s0 = __dadd_rn(s0, __dmul_rn(d0, d0)); s1 = __dadd_rn(s1, __dmul_rn(d1, d1));
    s2 = __dadd_rn(s2, __dmul_rn(d2, d2)); s3 = __dadd_rn(s3, __dmul_rn(d3, d3));
}
__device__ __forceinline__ void sq_add_tail(double &s0, float x, float c) {
    const double d = (double)__fsub_rn(x, c);
    s0 = __dadd_rn(s0, __dmul_rn(d, d));
}
__device__ __forceinline__ double sq_total(double s0, double s1, double s2, double s3) {
    return __dadd_rn(__dadd_rn(__dadd_rn(s0, s1), s2), s3);
}

__device__ __forceinline__ double sq_euclid64(const float *x, const float *c, uint32_t dim) {
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
    uint32_t j = 0;
    for (; j + 4 <= dim; j += 4) sq_add4(s0, s1, s2, s3, x[j], x[j + 1], x[j + 2], x[j + 3], c[j], c[j + 1], c[j + 2], c[j + 3]);
    for (; j < dim; ++j) sq_add_tail(s0, x[j], c[j]);
    return sq_total(s0, s1, s2, s3);
}

}  // namespace nk
