// kmeanspp.cu — k-means++ seeding over every row of a shard (initCentroidsKMeansPlusPlus, kmeans.go:364-426; DESIGN §7
// item 3).  One pass per seed: kmeanspp_step_kernel brings every row's D² (squared distance to its nearest seed) up to date
// with the newest seed in the reference's arithmetic (sq_euclid.cuh) and writes the sequential fp64 sum of each chunk of
// 256 rows; the host (nk_index_kmeanspp) draws the next seed from those sums.  A row the triangle inequality proves
// unchanged is skipped without reading its contents.
#include "kernels.cuh"
#include "sq_euclid.cuh"

namespace nk {

namespace kmpp {
constexpr int CHUNK = KMPP_CHUNK;  // rows per chunk = threads per CTA: one thread per row
constexpr int COLS = 32;           // columns of a row per stage
constexpr int PITCH = COLS + 4;    // floats per staged row: 9 16-byte units, odd, so the rows' float4 reads are conflict-free
constexpr int STAGES = 2;
constexpr int STAGE_FLOATS = CHUNK * PITCH;
constexpr size_t SMEM = (size_t)STAGES * STAGE_FLOATS * 4;
constexpr int CTAS_PER_SM = 3;
}  // namespace kmpp

// delta[j] = sq_euclid64(seed c, seed j) for every earlier seed j < c (seeds: the shard's [K x dim] seed list).
__global__ void kmeanspp_delta_kernel(const float *seeds, uint32_t dim, uint32_t c, double *delta) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < c) delta[j] = sq_euclid64(seeds + (size_t)c * dim, seeds + (size_t)j * dim, dim);
}

__device__ __forceinline__ void cp_async16(float *dst, const float *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async4(float *dst, const float *src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_one() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }

struct KmppStepParams {
    const float *rows;
    uint64_t n;
    uint32_t dim;
    const float *seed;      // seed c, [dim]
    const double *delta;    // [c]: sq_euclid64(seed c, seed j)
    uint32_t c;
    int prune;
    double *d2;             // [n] in / out
    uint32_t *near;         // [n] in / out: the seed that set d2
    double *chunk_sum;      // [ceil(n / CHUNK)] out
    unsigned long long *rows_read;
};

// One CTA per chunk of 256 rows (grid-stride), one thread per row.  The rows a pass computes are staged through a
// two-deep shared-memory ring COLS columns at a time: VEC (4 dim a multiple of 16 bytes, 16-byte aligned rows) with
// 16-byte cp.async copies, eight threads per 128-byte row segment; otherwise 4-byte copies.  Each thread then adds its
// row's columns in ascending order, so the sums are sq_euclid64's.  The chunk's sum is added sequentially by one thread.
template <bool VEC>
__global__ void __launch_bounds__(kmpp::CHUNK, kmpp::CTAS_PER_SM) kmeanspp_step_kernel(KmppStepParams p) {
    using namespace kmpp;
    extern __shared__ float4 kmpp_smem[];
    float *stage = reinterpret_cast<float *>(kmpp_smem);
    __shared__ unsigned char take[CHUNK];
    const uint32_t t = threadIdx.x, dim = p.dim;
    const uint32_t nslice = (dim + COLS - 1) / COLS;
    constexpr uint32_t UNIT = VEC ? 4 : 1;            // floats per copy
    constexpr uint32_t UNITS = COLS / UNIT;           // copies per row segment
    constexpr uint32_t PER_THREAD = UNITS;            // CHUNK * UNITS copies per stage over CHUNK threads
    const uint64_t nchunk = (p.n + CHUNK - 1) / CHUNK;
    unsigned long long read = 0;
    for (uint64_t ch = blockIdx.x; ch < nchunk; ch += gridDim.x) {
        const uint64_t r0 = ch * CHUNK, i = r0 + t;
        const uint32_t rows_in = p.n - r0 < (uint64_t)CHUNK ? (uint32_t)(p.n - r0) : (uint32_t)CHUNK;
        const bool live = t < rows_in;
        double m = 0.0;
        bool compute = live;
        if (live && p.c > 0) {
            m = p.d2[i];
            // Triangle inequality (DESIGN §7 item 3): with a = near[i], delta_a >= 4 m (1 + 2^-18) proves that the new seed's
            // computed distance is >= the computed m, so kmeans.go's strict < would keep m.  NaN m or delta: computed.
            const double da = p.prune ? p.delta[p.near[i]] : 0.0;
            if (p.prune && dim <= 32768u && da < INFINITY && da >= 4.0 * m * (1.0 + 0x1p-18)) compute = false;
        }
        take[t] = compute;
        const int count = __syncthreads_count(compute);
        read += (unsigned long long)count;
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
        if (count) {
            const float *base = p.rows + r0 * dim;
            auto load = [&](uint32_t s) {
                float *dst = stage + (s % STAGES) * STAGE_FLOATS;
                const uint32_t c0 = s * COLS, w = min(dim - c0, (uint32_t)COLS);
#pragma unroll
                for (uint32_t k = 0; k < PER_THREAD; ++k) {
                    const uint32_t item = t + k * CHUNK, r = item / UNITS, u = item % UNITS;
                    if (r < rows_in && take[r] && u * UNIT < w) {
                        const float *src = base + (size_t)r * dim + c0 + u * UNIT;
                        if (VEC) cp_async16(dst + r * PITCH + u * UNIT, src);
                        else cp_async4(dst + r * PITCH + u, src);
                    }
                }
                cp_async_commit();
            };
            load(0);
            for (uint32_t s = 0; s < nslice; ++s) {
                if (s + 1 < nslice) load(s + 1);
                else cp_async_commit();
                cp_async_wait_one();
                __syncthreads();
                if (compute) {
                    const float *x = stage + (s % STAGES) * STAGE_FLOATS + t * PITCH;
                    const uint32_t c0 = s * COLS, w = min(dim - c0, (uint32_t)COLS);
                    if (VEC) {
                        const float4 *x4 = reinterpret_cast<const float4 *>(x);
                        const float4 *s4 = reinterpret_cast<const float4 *>(p.seed + c0);
#pragma unroll
                        for (uint32_t u = 0; u < COLS / 4; ++u) {
                            if (u * 4 < w) {
                                const float4 a = x4[u], b = __ldg(s4 + u);
                                sq_add4(s0, s1, s2, s3, a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w);
                            }
                        }
                    } else {
                        for (uint32_t e = 0; e < w; e += 4) {
                            if (c0 + e + 4 <= dim) {
                                sq_add4(s0, s1, s2, s3, x[e], x[e + 1], x[e + 2], x[e + 3], __ldg(p.seed + c0 + e), __ldg(p.seed + c0 + e + 1),
                                         __ldg(p.seed + c0 + e + 2), __ldg(p.seed + c0 + e + 3));
                            } else {
                                for (uint32_t f = e; f < w; ++f) sq_add_tail(s0, x[f], __ldg(p.seed + c0 + f));
                            }
                        }
                    }
                }
                __syncthreads();  // the stage is refilled by the next iteration's load
            }
        }
        double wgt = m;
        if (compute) {
            const double d = sq_total(s0, s1, s2, s3);
            if (p.c == 0) {  // kmeans.go:379-384: assigned, so a NaN distance stays NaN
                wgt = d;
                p.d2[i] = d; p.near[i] = 0;
            } else if (d < m) {  // kmeans.go:418
                wgt = d;
                p.d2[i] = d; p.near[i] = p.c;
            }
        }
        double *w = reinterpret_cast<double *>(stage);  // the ring is idle here: every read of it is behind the last barrier
        if (live) w[t] = wgt;
        __syncthreads();
        if (t == 0) {
            double S = 0.0;
            for (uint32_t r = 0; r < rows_in; ++r) S = __dadd_rn(S, w[r]);
            p.chunk_sum[ch] = S;
        }
        __syncthreads();
    }
    if (t == 0 && read) atomicAdd(p.rows_read, read);
}

int kmeanspp_pass(const DeviceInfo &di, const float *rows, uint64_t n, uint32_t dim, const float *seeds, uint32_t c, double *delta,
                  bool prune, double *d2, uint32_t *near, double *chunk_sum, unsigned long long *rows_read, cudaStream_t stream,
                  uint64_t *launches) {
    using namespace kmpp;
    if (n == 0) return 0;
    if (c > 0) kmeanspp_delta_kernel<<<(c + 63) / 64, 64, 0, stream>>>(seeds, dim, c, delta);
    KmppStepParams p;
    p.rows = rows; p.n = n; p.dim = dim; p.seed = seeds + (size_t)c * dim; p.delta = delta; p.c = c; p.prune = prune ? 1 : 0;
    p.d2 = d2; p.near = near; p.chunk_sum = chunk_sum; p.rows_read = rows_read;
    const uint64_t nchunk = (n + CHUNK - 1) / CHUNK;
    const uint64_t full = (uint64_t)di.num_sms * CTAS_PER_SM;
    const uint32_t grid = (uint32_t)(nchunk < full ? nchunk : full);
    const bool vec = dim % 4 == 0 && (reinterpret_cast<uintptr_t>(rows) & 15) == 0;
    const void *kern = vec ? reinterpret_cast<const void *>(kmeanspp_step_kernel<true>) : reinterpret_cast<const void *>(kmeanspp_step_kernel<false>);
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM);
    if (e == cudaSuccess) {
        if (vec) kmeanspp_step_kernel<true><<<grid, CHUNK, SMEM, stream>>>(p);
        else kmeanspp_step_kernel<false><<<grid, CHUNK, SMEM, stream>>>(p);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { set_error("kmeanspp_pass: %s", cudaGetErrorString(e)); return -1; }
    if (launches) *launches += c > 0 ? 2 : 1;
    return 0;
}

}  // namespace nk
