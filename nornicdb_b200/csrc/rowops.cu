// rowops.cu — one-pass row kernels behind the legacy ABI and index maintenance.
//
//   row_norms       replaces n x cublasSnrm2                  (cuda_bridge.go:231-246), overflow- and underflow-safe like it
//   normalize_rows  replaces n x cublasSnrm2 + D2H + n x cublasSscal (cuda_bridge.go:249-284)
//   row_scores      replaces cublasSgemv                      (cuda_bridge.go:290-318)
//   fill_uniform / fill_clustered   synthetic corpora generated in HBM (bench / tests); the uniform one is bit-identical
//                   to the oracle's, the Gaussian mixture is SURVEY.md §8(d)'s near-tie corpus
//   gather_rows     row gather for ScoreSubset (gpu.go:1578-1589 does this on the host + re-upload)
//   row_filters     left-row admission of the self-join (nk_search_pairs): one thread per row, not warp-per-row
//   row_sqnorms16   |x|^2 per row of an fp16 / bf16 corpus (the 16-bit tensor pass scans such a corpus in place)
//   group_best      best-of-chunks per node for db.index.vector.queryNodes (call_vector.go:217-240)
// All are warp-per-row, lanes striding the row in 16-byte vectors where the layout allows (one 512 B coalesced segment per
// step; the scalar path serves dim % 4 != 0 or unaligned buffers), 64-bit row offsets (the reference's orphan kernels
// overflow uint32 at n*dim >= 2^32, cuda_kernels.cu:195,274,298).  Grids are sized from the device's SM count.
// HBM-bound; algorithmic bytes: norms / scores n*dim*4 (read once), normalize 2*n*dim*4 (read + write; the row is re-read
// from L1/L2 for the scaling pass).
#include <float.h>
#include <type_traits>

#include "kernels.cuh"

namespace nk {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

static int sm_count() {
    static int sms[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (!sms[dev]) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
        sms[dev] = v;
    }
    return sms[dev];
}
// persistent-style grid: `per_sm` CTAs of 256 threads per SM, never more CTAs than there are 8-row groups
static inline unsigned warp_grid(uint64_t n, int per_sm = 16) {
    uint64_t blocks = (n + 7) / 8;  // 8 warps per 256-thread block
    const uint64_t cap = (uint64_t)sm_count() * per_sm;
    if (blocks > cap) blocks = cap;
    if (blocks == 0) blocks = 1;
    return (unsigned)blocks;
}
// Norm of a row whose fp32 sum of squares `a` (the warp-uniform result of the fast path) is not finite, or below 2^-100
// where subnormal squares lose precision: elements beyond ~1e19 overflow it, elements below ~1e-19 underflow it; cublasSnrm2,
// which the reference calls, does neither.  As BLAS nrm2 does, the row is summed again scaled by the power of two that
// brings its largest |x| into [0.5, 1), and the root scaled back.  Rows of ordinary magnitude never get here, so they keep
// the fast path's bits.  A NaN element gives NaN, an inf element inf, a zero row 0.
__device__ __noinline__ float scaled_row_norm(const float *p, uint32_t dim, uint32_t lane, float a) {
    if (a != a) return a;
    float m = 0.0f;
    for (uint32_t j = lane; j < dim; j += 32) m = fmaxf(m, fabsf(p[j]));
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (m == 0.0f || isinf(m)) return m;
    int e;
    frexpf(m, &e);
    float t = 0.0f;
    for (uint32_t j = lane; j < dim; j += 32) {
        const float x = scalbnf(p[j], -e);
        t = fmaf(x, x, t);
    }
    return scalbnf(sqrtf(warp_sum(t)), e);
}
__device__ __forceinline__ bool needs_scaling(float a) { return !(a >= 0x1p-100f && a <= FLT_MAX); }

static inline bool vec4_ok(const void *p, uint32_t dim) { return dim % 4 == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <bool VEC>
__global__ void row_norms_kernel(const float *rows, float *norms, uint32_t n, uint32_t dim) {
    uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t r = warp; r < n; r += nwarps) {
        const float *p = rows + (size_t)r * dim;
        float a = 0.0f;
        if (VEC) {
            const float4 *p4 = reinterpret_cast<const float4 *>(p);
            for (uint32_t j = lane; j < dim / 4; j += 32) {
                const float4 v = __ldg(p4 + j);
                a = fmaf(v.x, v.x, a); a = fmaf(v.y, v.y, a); a = fmaf(v.z, v.z, a); a = fmaf(v.w, v.w, a);
            }
        } else {
            for (uint32_t j = lane; j < dim; j += 32) {
                float x = __ldg(p + j);
                a = fmaf(x, x, a);
            }
        }
        a = warp_sum(a);
        const float nrm = needs_scaling(a) ? scaled_row_norm(p, dim, lane, a) : sqrtf(a);
        if (lane == 0) norms[r] = nrm;
    }
}

template <bool VEC>
__global__ void normalize_rows_kernel(float *rows, uint32_t n, uint32_t dim) {
    uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t r = warp; r < n; r += nwarps) {
        float *p = rows + (size_t)r * dim;
        float a = 0.0f;
        if (VEC) {
            float4 *p4 = reinterpret_cast<float4 *>(p);
            for (uint32_t j = lane; j < dim / 4; j += 32) {
                const float4 v = p4[j];
                a = fmaf(v.x, v.x, a); a = fmaf(v.y, v.y, a); a = fmaf(v.z, v.z, a); a = fmaf(v.w, v.w, a);
            }
            a = warp_sum(a);
            const float nrm = needs_scaling(a) ? scaled_row_norm(p, dim, lane, a) : sqrtf(a);
            if (nrm > 1e-10f) {  // cuda_bridge.go:267: rows with norm <= 1e-10 are left untouched
                const float inv = 1.0f / nrm;
                for (uint32_t j = lane; j < dim / 4; j += 32) {
                    float4 v = p4[j];
                    v.x *= inv; v.y *= inv; v.z *= inv; v.w *= inv;
                    p4[j] = v;
                }
            }
        } else {
            for (uint32_t j = lane; j < dim; j += 32) a = fmaf(p[j], p[j], a);
            a = warp_sum(a);
            const float nrm = needs_scaling(a) ? scaled_row_norm(p, dim, lane, a) : sqrtf(a);
            if (nrm > 1e-10f) {
                const float inv = 1.0f / nrm;
                for (uint32_t j = lane; j < dim; j += 32) p[j] *= inv;
            }
        }
    }
}

template <bool VEC>
__global__ void row_scores_kernel(const float *rows, const float *query, float *scores, uint32_t n, uint32_t dim,
                                  int normalized) {
    uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    float qq = 0.0f;
    if (!normalized) {
        for (uint32_t j = lane; j < dim; j += 32) qq = fmaf(query[j], query[j], qq);
        qq = warp_sum(qq);
    }
    for (uint32_t r = warp; r < n; r += nwarps) {
        const float *p = rows + (size_t)r * dim;
        float d = 0.0f, xx = 0.0f;
        if (VEC) {
            const float4 *p4 = reinterpret_cast<const float4 *>(p), *q4 = reinterpret_cast<const float4 *>(query);
            for (uint32_t j = lane; j < dim / 4; j += 32) {
                const float4 v = __ldg(p4 + j), u = __ldg(q4 + j);
                d = fmaf(v.x, u.x, d); xx = fmaf(v.x, v.x, xx);
                d = fmaf(v.y, u.y, d); xx = fmaf(v.y, v.y, xx);
                d = fmaf(v.z, u.z, d); xx = fmaf(v.z, v.z, xx);
                d = fmaf(v.w, u.w, d); xx = fmaf(v.w, v.w, xx);
            }
        } else {
            for (uint32_t j = lane; j < dim; j += 32) {
                float x = __ldg(p + j);
                d = fmaf(x, __ldg(query + j), d);
                xx = fmaf(x, x, xx);
            }
        }
        d = warp_sum(d);
        xx = warp_sum(xx);
        if (lane == 0) {
            if (normalized) {
                scores[r] = d;
            } else {
                float den = sqrtf(xx * qq);
                scores[r] = den == 0.0f ? 0.0f : d / den;  // 0 for a zero row or query; a NaN element stays NaN
            }
        }
    }
}

template <typename T> __device__ __forceinline__ T from_float(float v);
template <> __device__ __forceinline__ float from_float<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_float<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_float<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <typename T>
__global__ void fill_uniform_kernel(T *out, uint64_t total, uint32_t dim, uint64_t seed, uint64_t row_base) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (; i < total; i += stride) out[i] = from_float<T>(uniform_at(seed, row_base * dim + i));
}

// Gaussian-mixture corpus (SURVEY.md §8(d): "1000 centres, sigma = 0.1", the shape of cmd/kmeans-test-data's clusters
// mode, main.go:231-283): row r belongs to centre hash(r) % C (the reference shuffles its rows), centre c is U[-1,1)^dim,
// element = centre + sigma * N(0,1) by Box-Muller over the counter-based generator.  unit != 0 follows the reference tool
// to the letter: centres normalised to unit length first, rows normalised after the noise.  Device-only (fast-math log /
// cos): tests read the rows back for the oracle instead of regenerating them on the host.
template <typename T>
__global__ void fill_clustered_kernel(T *out, uint64_t n_rows, uint32_t dim, uint64_t seed, uint64_t row_base, uint32_t centres, float sigma,
                                      int unit) {
    const int lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t r = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n_rows; r += warps) {
        const uint64_t g = row_base + r;
        const uint64_t c = mix64(g * 0x9E3779B97F4A7C15ULL + seed) % centres;
        float cn = 1.0f;
        if (unit) {
            float a = 0.0f;
            for (uint32_t j = lane; j < dim; j += 32) { const float v = uniform_at(seed ^ 0xC3A5C85C97CB3127ULL, c * dim + j); a = fmaf(v, v, a); }
            a = warp_sum(a);
            cn = a > 0.0f ? rsqrtf(a) : 0.0f;
        }
        float xx = 0.0f;
        for (uint32_t j = lane; j < dim; j += 32) {
            const float u1 = (uniform_at(seed ^ 0x5851F42D4C957F2DULL, g * dim + j) + 1.0f) * 0.5f;  // [0,1)
            const float u2 = (uniform_at(seed ^ 0x14057B7EF767814FULL, g * dim + j) + 1.0f) * 0.5f;
            const float z = sqrtf(-2.0f * __logf(fmaxf(u1, 5.9604645e-8f))) * __cosf(6.2831853f * u2);
            const float v = uniform_at(seed ^ 0xC3A5C85C97CB3127ULL, c * dim + j) * cn + sigma * z;
            xx = fmaf(v, v, xx);
            if (!unit) out[r * dim + j] = from_float<T>(v);
        }
        if (unit) {  // second pass: regenerate and scale (the generator is a pure function of (seed, row, column))
            xx = warp_sum(xx);
            const float inv = xx > 0.0f ? rsqrtf(xx) : 0.0f;
            for (uint32_t j = lane; j < dim; j += 32) {
                const float u1 = (uniform_at(seed ^ 0x5851F42D4C957F2DULL, g * dim + j) + 1.0f) * 0.5f;
                const float u2 = (uniform_at(seed ^ 0x14057B7EF767814FULL, g * dim + j) + 1.0f) * 0.5f;
                const float z = sqrtf(-2.0f * __logf(fmaxf(u1, 5.9604645e-8f))) * __cosf(6.2831853f * u2);
                out[r * dim + j] = from_float<T>((uniform_at(seed ^ 0xC3A5C85C97CB3127ULL, c * dim + j) * cn + sigma * z) * inv);
            }
        }
    }
}

// O == T: a copy; O == float with 16-bit rows: the exact widening (every fp16 / bf16 value is an fp32 value)
template <typename T, typename O>
__global__ void gather_rows_kernel(const T *rows, uint32_t dim, const uint32_t *idx, uint32_t n_idx, O *out) {
    uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t r = warp; r < n_idx; r += nwarps) {
        const T *src = rows + (size_t)idx[r] * dim;
        O *dst = out + (size_t)r * dim;
        for (uint32_t j = lane; j < dim; j += 32) {
            if constexpr (std::is_same<T, O>::value) dst[j] = src[j];
            else if constexpr (std::is_same<T, __half>::value) dst[j] = __half2float(src[j]);
            else dst[j] = __bfloat162float(src[j]);
        }
    }
}

__global__ void row_filters_kernel(const uint32_t *idx, uint32_t n_idx, const uint32_t *mask, const uint64_t *tags, NkFilter f,
                                   NkFilter *out) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_idx) return;
    const uint32_t row = idx[r];
    const bool in_mask = !mask || ((mask[row >> 5] >> (row & 31)) & 1u);
    const uint64_t tag = tags ? tags[row] : 0ull;
    out[r] = in_mask && tag_admits(tag, f.all_of, f.none_of, f.any_of) ? f : NkFilter{~0ull, ~0ull, 0ull};
}

__global__ void row_windows_kernel(const uint32_t *idx, uint32_t n_idx, const uint32_t *mask, const uint64_t *tags, const uint64_t *values,
                                   NkFilter f, NkWindow w, uint64_t gap, NkWindow *out) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_idx) return;
    const uint32_t row = idx[r];
    const bool in_mask = !mask || ((mask[row >> 5] >> (row & 31)) & 1u);
    const uint64_t tag = tags ? tags[row] : 0ull;
    const uint64_t v = values ? values[row] : 0ull;
    const bool band = gap != NK_NO_GAP;
    NkWindow o{~0ull, 0ull};  // admits no row
    if (in_mask && tag_admits(tag, f.all_of, f.none_of, f.any_of) && window_admits(v, w.lo, w.hi) && (!band || v != 0)) {
        o = w;
        if (band) {  // [v - gap, v + gap], saturating, without key 0 (a row without a value is in no band)
            const uint64_t lo = v > gap ? v - gap : 1ull, hi = v > ~0ull - gap ? ~0ull : v + gap;
            o.lo = o.lo > lo ? o.lo : lo;
            o.hi = o.hi < hi ? o.hi : hi;
        }
    }
    out[r] = o;
}

// |x|^2 per row of a 16-bit corpus (fp32 accumulation of the exactly widened elements)
template <typename T>
__global__ void row_sqnorms16_kernel(const T *rows, uint64_t n, uint32_t dim, float *out) {
    const int lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t r = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n; r += warps) {
        const T *x = rows + r * dim;
        float a = 0.0f;
        for (uint32_t j = lane; j < dim; j += 32) {
            float v;
            if constexpr (sizeof(T) == 2 && std::is_same<T, __half>::value) v = __half2float(x[j]);
            else v = __bfloat162float(x[j]);
            a = fmaf(v, v, a);
        }
        a = warp_sum(a);
        if (lane == 0) out[r] = a;
    }
}

// ---- k-means update step (pkg/gpu/kmeans.go:585-618) -------------------------------------------------------------
// Per-cluster float64 sums of the member rows: one warp per row, lanes stride the dimensions, fp64 atomic adds (the
// K x dim accumulator is spread over L2, so contention is low; fp64 keeps the sum order-independent to ~1e-16, far
// below the float32 the mean is rounded to).  Rows whose assignment is outside [0, K) are skipped.
__global__ void cluster_sums_kernel(const float *rows, uint64_t n, uint32_t dim, const int32_t *assign, uint32_t K, double *sums,
                                    unsigned long long *counts) {
    const int lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t row = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < n; row += warps) {
        const int32_t c = assign[row];
        if (c < 0 || (uint32_t)c >= K) continue;
        const float *x = rows + row * dim;
        double *dst = sums + (size_t)c * dim;
        for (uint32_t j = lane; j < dim; j += 32) atomicAdd(dst + j, (double)x[j]);
        if (lane == 0) atomicAdd(counts + c, 1ull);
    }
}
template <typename T>
__global__ void convert_f32_kernel(const float *src, T *dst, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = from_float<T>(src[i]);
}
// changed += (a[i] != b[i])
__global__ void count_changed_kernel(const int32_t *a, const uint32_t *b, uint64_t n, unsigned long long *changed) {
    unsigned long long mine = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        mine += a[i] != (int32_t)b[i];
    mine = __reduce_add_sync(0xffffffffu, (unsigned)mine);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(changed, mine);
}

// ---- best-of-chunks per node (db.index.vector.queryNodes, call_vector.go:217-247) ---------------------------------
// Every row is one chunk embedding of node group[row]; a node's score is the BEST score over its chunks.  One pass over
// the rows (HBM-bound, n*dim*sizeof(elem) bytes): warp per row, exact fp32 score, then a 64-bit atomicMax of the packed
// (score, row) key into the node's slot — the segment-max.  best[] is zeroed by the caller; nodes whose best stays 0
// have no admissible chunk (masked, or below min_score: the reference keeps a node only if bestScore >= 0).
template <typename T>
__global__ void group_best_kernel(const T *rows, uint64_t n, uint32_t dim, uint64_t row_base, const float *query, int metric,
                                  const uint32_t *group, const uint32_t *mask, float min_score, unsigned long long *best) {
    extern __shared__ __align__(16) float gq[];
    __shared__ float s_qq;
    for (uint32_t j = threadIdx.x; j < dim; j += blockDim.x) gq[j] = query[j];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    if (threadIdx.x < 32) {
        float a = 0.0f;
        for (uint32_t j = lane; j < dim; j += 32) a = fmaf(gq[j], gq[j], a);
        a = warp_sum(a);
        if (lane == 0) s_qq = a;
    }
    __syncthreads();
    const float qq = s_qq;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t r = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n; r += warps) {
        if (mask && !((__ldg(mask + (r >> 5)) >> (r & 31)) & 1u)) continue;
        const T *x = rows + r * dim;
        float d = 0.0f, xx = 0.0f;
        for (uint32_t j = lane; j < dim; j += 32) {
            float v;
            if constexpr (sizeof(T) == 4) v = __ldg(reinterpret_cast<const float *>(x) + j);
            else if constexpr (std::is_same<T, __half>::value) v = __half2float(x[j]);
            else v = __bfloat162float(x[j]);
            if (metric == NK_METRIC_EUCLIDEAN) { const float t = v - gq[j]; d = fmaf(t, t, d); }
            else { d = fmaf(v, gq[j], d); xx = fmaf(v, v, xx); }
        }
        d = warp_sum(d);
        xx = warp_sum(xx);
        if (lane == 0) {
            float sc = d;
            if (metric == NK_METRIC_EUCLIDEAN) sc = -d;
            else if (metric == NK_METRIC_COSINE) { const float den = sqrtf(xx * qq); sc = den > 0.0f ? d / den : 0.0f; }
            if (sc == sc && sc >= min_score) atomicMax(best + group[r], (unsigned long long)make_key(sc, (uint32_t)(row_base + r)));
        }
    }
}

// ---- launchers --------------------------------------------------------------------------------------------------------
int row_norms(const float *rows, float *norms, uint32_t n, uint32_t dim, cudaStream_t s) {
    if (n == 0) return 0;
    if (vec4_ok(rows, dim)) row_norms_kernel<true><<<warp_grid(n), 256, 0, s>>>(rows, norms, n, dim);
    else row_norms_kernel<false><<<warp_grid(n), 256, 0, s>>>(rows, norms, n, dim);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}
int normalize_rows(float *rows, uint32_t n, uint32_t dim, cudaStream_t s) {
    if (n == 0) return 0;
    if (vec4_ok(rows, dim)) normalize_rows_kernel<true><<<warp_grid(n), 256, 0, s>>>(rows, n, dim);
    else normalize_rows_kernel<false><<<warp_grid(n), 256, 0, s>>>(rows, n, dim);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}
int row_scores(const float *rows, const float *query, float *scores, uint32_t n, uint32_t dim, int normalized,
               cudaStream_t s) {
    if (n == 0) return 0;
    if (vec4_ok(rows, dim) && (reinterpret_cast<uintptr_t>(query) & 15) == 0)
        row_scores_kernel<true><<<warp_grid(n), 256, 0, s>>>(rows, query, scores, n, dim, normalized);
    else
        row_scores_kernel<false><<<warp_grid(n), 256, 0, s>>>(rows, query, scores, n, dim, normalized);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}
int fill_uniform(void *out, int dtype, uint64_t n_rows, uint32_t dim, uint64_t seed, uint64_t row_base, cudaStream_t s) {
    uint64_t total = n_rows * dim;
    if (total == 0) return 0;
    const unsigned grid = (unsigned)sm_count() * 16;
    if (dtype == NK_DTYPE_F16) fill_uniform_kernel<__half><<<grid, 256, 0, s>>>((__half *)out, total, dim, seed, row_base);
    else if (dtype == NK_DTYPE_BF16) fill_uniform_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>((__nv_bfloat16 *)out, total, dim, seed, row_base);
    else fill_uniform_kernel<float><<<grid, 256, 0, s>>>((float *)out, total, dim, seed, row_base);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}
int fill_clustered(void *out, int dtype, uint64_t n_rows, uint32_t dim, uint64_t seed, uint64_t row_base, uint32_t centres, float sigma,
                   int unit, cudaStream_t s) {
    if (n_rows == 0 || dim == 0) return 0;
    if (centres == 0) centres = 1;
    const unsigned grid = warp_grid(n_rows);
    if (dtype == NK_DTYPE_F16) fill_clustered_kernel<__half><<<grid, 256, 0, s>>>((__half *)out, n_rows, dim, seed, row_base, centres, sigma, unit);
    else if (dtype == NK_DTYPE_BF16) fill_clustered_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>((__nv_bfloat16 *)out, n_rows, dim, seed, row_base, centres, sigma, unit);
    else fill_clustered_kernel<float><<<grid, 256, 0, s>>>((float *)out, n_rows, dim, seed, row_base, centres, sigma, unit);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}
int row_sqnorms16(const void *rows, int dtype, uint64_t first, uint64_t count, uint32_t dim, float *out, cudaStream_t s) {
    if (count == 0) return 0;
    if (dtype == NK_DTYPE_F16)
        row_sqnorms16_kernel<__half><<<warp_grid(count), 256, 0, s>>>(static_cast<const __half *>(rows) + first * dim, count, dim, out + first);
    else
        row_sqnorms16_kernel<__nv_bfloat16><<<warp_grid(count), 256, 0, s>>>(static_cast<const __nv_bfloat16 *>(rows) + first * dim, count, dim, out + first);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}
int cluster_sums(const float *rows, uint64_t n, uint32_t dim, const int32_t *assign, uint32_t K, double *sums,
                 unsigned long long *counts, cudaStream_t s) {
    if (n == 0) return 0;
    cluster_sums_kernel<<<warp_grid(n, 8), 256, 0, s>>>(rows, n, dim, assign, K, sums, counts);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}
int convert_f32_to_16(const float *src, void *dst, int dtype, size_t n, cudaStream_t s) {
    if (n == 0) return 0;
    const unsigned grid = (unsigned)sm_count() * 8;
    if (dtype == NK_DTYPE_BF16) convert_f32_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(src, static_cast<__nv_bfloat16 *>(dst), n);
    else convert_f32_kernel<__half><<<grid, 256, 0, s>>>(src, static_cast<__half *>(dst), n);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}
int count_changed(const int32_t *a, const uint32_t *b, uint64_t n, unsigned long long *changed, cudaStream_t s) {
    if (n == 0) return 0;
    count_changed_kernel<<<(unsigned)sm_count() * 4, 256, 0, s>>>(a, b, n, changed);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}
int gather_rows(const void *rows, int dtype, uint32_t dim, const uint32_t *idx, uint32_t n_idx, void *out, bool out_f32,
                cudaStream_t s) {
    if (n_idx == 0) return 0;
    if (dtype == NK_DTYPE_F32)
        gather_rows_kernel<float, float><<<warp_grid(n_idx), 256, 0, s>>>((const float *)rows, dim, idx, n_idx, (float *)out);
    else if (!out_f32)  // fp16 / bf16: a 2-byte copy either way
        gather_rows_kernel<__half, __half><<<warp_grid(n_idx), 256, 0, s>>>((const __half *)rows, dim, idx, n_idx, (__half *)out);
    else if (dtype == NK_DTYPE_F16)
        gather_rows_kernel<__half, float><<<warp_grid(n_idx), 256, 0, s>>>((const __half *)rows, dim, idx, n_idx, (float *)out);
    else
        gather_rows_kernel<__nv_bfloat16, float><<<warp_grid(n_idx), 256, 0, s>>>((const __nv_bfloat16 *)rows, dim, idx, n_idx, (float *)out);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}
int row_filters(const uint32_t *idx, uint32_t n_idx, const uint32_t *mask, const uint64_t *tags, NkFilter f, NkFilter *out,
                cudaStream_t s) {
    if (n_idx == 0) return 0;
    row_filters_kernel<<<(n_idx + 255) / 256, 256, 0, s>>>(idx, n_idx, mask, tags, f, out);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}
int row_windows(const uint32_t *idx, uint32_t n_idx, const uint32_t *mask, const uint64_t *tags, const uint64_t *values, NkFilter f,
                NkWindow w, uint64_t gap, NkWindow *out, cudaStream_t s) {
    if (n_idx == 0) return 0;
    row_windows_kernel<<<(n_idx + 255) / 256, 256, 0, s>>>(idx, n_idx, mask, tags, values, f, w, gap, out);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}
int group_best(const DeviceInfo &di, const void *rows, int dtype, uint64_t n, uint32_t dim, uint64_t row_base, const float *query,
               int metric, const uint32_t *group, const uint32_t *mask, float min_score, unsigned long long *best, cudaStream_t s) {
    if (n == 0) return 0;
    const size_t smem = (size_t)dim * 4;
    const unsigned grid = warp_grid(n);
    const void *kern = dtype == NK_DTYPE_F16    ? reinterpret_cast<const void *>(group_best_kernel<__half>)
                       : dtype == NK_DTYPE_BF16 ? reinterpret_cast<const void *>(group_best_kernel<__nv_bfloat16>)
                                                : reinterpret_cast<const void *>(group_best_kernel<float>);
    if (ensure_smem(di, kern, smem, "group search", dim)) return -1;
    if (dtype == NK_DTYPE_F16)
        group_best_kernel<__half><<<grid, 256, smem, s>>>((const __half *)rows, n, dim, row_base, query, metric, group, mask, min_score, best);
    else if (dtype == NK_DTYPE_BF16)
        group_best_kernel<__nv_bfloat16><<<grid, 256, smem, s>>>((const __nv_bfloat16 *)rows, n, dim, row_base, query, metric, group, mask, min_score, best);
    else
        group_best_kernel<float><<<grid, 256, smem, s>>>((const float *)rows, n, dim, row_base, query, metric, group, mask, min_score, best);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace nk
