// scan_simt.cu — fused distance + top-k scan on CUDA cores (the HBM-bound small-Q path).
//
// Replaces, in one kernel, the reference's per-query chain
//   cublasSgemv (cuda_bridge.go:302-309) -> D2H of all n scores -> host insertion top-k (cuda_bridge.go:336-371)
// and the CPU scan simd.Batch{Cosine,Dot,Euclidean} + bounded top-k (pkg/simd/simd.go:149-231).
//
// Shape of the work: every corpus byte is read from HBM exactly once per group of QT<=8 queries.
//   * a warp owns R rows at a time; lanes stride the row in 16-byte vectors (float4 / 8 halves), so a
//     warp-wide load is one fully coalesced 512 B segment per row;
//   * the QT queries of the group live in shared memory (read as conflict-free LDS.128, re-used by the
//     R rows in registers);
//   * R*QT partial dot products per lane are folded with a butterfly "reduce-scatter" (31 shuffles for
//     32 values) so each lane ends up owning one finished (row, query) score;
//   * scores never go to memory: the owner lane compares against the query's running threshold (k-th
//     best score this CTA has seen) and only then appends a packed 64-bit key to a per-(CTA, query)
//     candidate buffer; the CTA prunes a buffer with a bitonic sort when it could overflow;
//   * each CTA finally emits its best k keys per query; merge_keys() folds the per-CTA lists.
//
// Algorithmic HBM traffic per launch = n*dim*sizeof(elem) (+ QT*dim*4 of queries): DESIGN.md §Kernels.
#include <map>
#include <mutex>
#include <tuple>
#include <type_traits>

#include "kernels.cuh"

namespace nk {

constexpr int SIMT_THREADS = 256;
constexpr int SIMT_WARPS = SIMT_THREADS / 32;
constexpr int SIMT_RT = 256;  // rows a CTA scores between two prune checks

struct SimtParams {
    const void *rows;
    uint32_t n, dim;
    uint64_t row_base;
    const float *queries;  // [Q x dim], this launch handles queries q0 .. q0+nq-1
    uint32_t q0, nq, k;
    int metric;
    int P;               // candidate-buffer capacity = sort width (power of two)
    uint64_t *cand;      // [grid][QT][P]
    uint64_t *partial;   // [Q][grid][k]
    int *flags;
    const int *only_if;  // device-side conditional fallback: run only if *only_if != 0
    const uint64_t *below;  // per-query exclusive key bound (k > NK_MAX_K passes) or nullptr
    const uint32_t *mask;   // row bitmask or nullptr
    float min_score;        // caller's score floor (key space); -inf = none
    const uint64_t *row_tags;  // TAGS kernels only: tag word per local row
    const NkFilter *qfilter;   // TAGS kernels only: filter per query [Q]
};
// RANGE kernels (nk_search_range) take these on top; the top-k kernels keep their parameter block as it is.
struct SimtRangeParams : SimtParams {
    const uint32_t *range_tau;  // order-preserving bits of each query's fixed threshold [Q] (floor included)
    int *range_fill;            // list fill per query [Q], counts past list_cap
    uint32_t list_cap;          // `partial` is [Q][list_cap]
};
// WINDOW kernels (the window modes) take the value windows on top of either block, so the other kernels' parameter offsets
// stay as they are.
template <bool RANGE> struct SimtWindowParams : std::conditional_t<RANGE, SimtRangeParams, SimtParams> {
    const uint64_t *row_values;  // value key per local row
    const NkWindow *qwindow;     // window per query [Q]
};
template <bool RANGE, bool WINDOW = false>
using SimtArgs = std::conditional_t<WINDOW, SimtWindowParams<RANGE>, std::conditional_t<RANGE, SimtRangeParams, SimtParams>>;

// ---- element loaders -------------------------------------------------------------------------
template <typename T, bool VEC> struct Lane;
template <> struct Lane<float, true> {
    static constexpr int EPL = 4;
    static __device__ __forceinline__ void load(const float *p, float (&x)[4]) {
        asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                     : "=f"(x[0]), "=f"(x[1]), "=f"(x[2]), "=f"(x[3]) : "l"(p));
    }
};
template <> struct Lane<__half, true> {
    static constexpr int EPL = 8;
    static __device__ __forceinline__ void load(const __half *p, float (&x)[8]) {
        uint32_t w0, w1, w2, w3;
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                     : "=r"(w0), "=r"(w1), "=r"(w2), "=r"(w3) : "l"(p));
        float2 f;
        f = __half22float2(*reinterpret_cast<__half2 *>(&w0)); x[0] = f.x; x[1] = f.y;
        f = __half22float2(*reinterpret_cast<__half2 *>(&w1)); x[2] = f.x; x[3] = f.y;
        f = __half22float2(*reinterpret_cast<__half2 *>(&w2)); x[4] = f.x; x[5] = f.y;
        f = __half22float2(*reinterpret_cast<__half2 *>(&w3)); x[6] = f.x; x[7] = f.y;
    }
};
template <> struct Lane<__nv_bfloat16, true> {
    static constexpr int EPL = 8;
    static __device__ __forceinline__ void load(const __nv_bfloat16 *p, float (&x)[8]) {
        uint32_t w[4];
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                     : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "l"(p));
#pragma unroll
        for (int i = 0; i < 4; ++i) {  // bf16 -> fp32 is a 16-bit shift
            x[2 * i] = __uint_as_float(w[i] << 16);
            x[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
        }
    }
};
template <> struct Lane<__nv_bfloat16, false> {
    static constexpr int EPL = 1;
    static __device__ __forceinline__ void load(const __nv_bfloat16 *p, float (&x)[1]) { x[0] = __bfloat162float(*p); }
};
template <> struct Lane<float, false> {
    static constexpr int EPL = 1;
    static __device__ __forceinline__ void load(const float *p, float (&x)[1]) { x[0] = __ldg(p); }
};
template <> struct Lane<__half, false> {
    static constexpr int EPL = 1;
    static __device__ __forceinline__ void load(const __half *p, float (&x)[1]) { x[0] = __half2float(__ldg(p)); }
};

// Butterfly reduce-scatter of V per-lane partial sums across the warp.  Afterwards v[0] holds the
// finished total of value index lane / (32 / V) (every lane of that group holds the same total).
template <int V>
__device__ __forceinline__ void warp_reduce_scatter(float (&v)[V], int lane) {
#pragma unroll
    for (int s = 0; s < 5; ++s) {
        const int o = 16 >> s;
        const int c = V >> s;  // live values before this step (compile-time after unrolling)
        if (c > 1) {
            const bool up = (lane & o) != 0;
#pragma unroll
            for (int i = 0; i < (c >> 1); ++i) {
                float keep = up ? v[i + (c >> 1)] : v[i];
                float send = up ? v[i] : v[i + (c >> 1)];
                v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
            }
        } else {
            v[0] += __shfl_xor_sync(0xffffffffu, v[0], o);
        }
    }
}

// TAGS: filtered search — the owner lane also tests its (row, query) pair against the query's tag filter.
// WINDOW (with TAGS): windowed search — ... and against the query's value window.
// RANGE (nk_search_range): the owner lane appends every pair whose exact score reaches the query's fixed threshold straight to
// the query's list — no buffer, no prune, no emission, and the scores need no re-scoring.
template <typename T, bool VEC, int QT, int R, bool EUCLID, bool TAGS, bool RANGE, bool WINDOW>
__global__ void __launch_bounds__(SIMT_THREADS) knn_scan_simt_kernel(SimtArgs<RANGE, WINDOW> p) {
    pdl_trigger();  // the merge launch behind this scan may begin (it waits for this grid before reading)
    pdl_wait();     // exact-stage twin of a filter search: programmatic dependent of the finish kernel
    if (p.only_if && *p.only_if == 0) return;
    using L = Lane<T, VEC>;
    constexpr int EPL = L::EPL;
    constexpr int CH = 32 * EPL;  // elements a warp covers per step
    constexpr int V = R * QT;
    static_assert(V <= 32 && (32 % V) == 0, "R*QT must divide 32");
    constexpr int LPV = 32 / V;

    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint64_t *sbuf = reinterpret_cast<uint64_t *>(smem_raw);
    float *qs = reinterpret_cast<float *>(smem_raw + (size_t)p.P * 8);  // [QT][dim]
    __shared__ float s_qq[QT];
    __shared__ float s_tau[QT];
    __shared__ int s_cnt[QT];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t dim = p.dim, n = p.n;
    const T *rows = static_cast<const T *>(p.rows);

    // ---- stage the query group -----------------------------------------------------------------
    for (uint32_t i = tid; i < (uint32_t)QT * dim; i += SIMT_THREADS) {
        uint32_t qi = i / dim, j = i - qi * dim;
        qs[i] = qi < p.nq ? p.queries[(size_t)(p.q0 + qi) * dim + j] : 0.0f;
    }
    if (tid < QT) {
        if constexpr (RANGE) s_tau[tid] = (uint32_t)tid < p.nq ? ord_to_float(p.range_tau[p.q0 + tid]) : INFINITY;
        else s_tau[tid] = p.min_score;
        s_cnt[tid] = 0;
    }
    __syncthreads();
    for (int qi = warp; qi < QT; qi += SIMT_WARPS) {  // |q|^2 per query (cosine)
        float a = 0.0f;
        for (uint32_t j = lane; j < dim; j += 32) a = fmaf(qs[qi * dim + j], qs[qi * dim + j], a);
#pragma unroll
        for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) s_qq[qi] = a;
    }
    __syncthreads();

    uint64_t *my_cand = p.cand + (size_t)blockIdx.x * QT * p.P;
    const int prune_at = p.P - SIMT_RT;
    const uint32_t num_iv = (n + SIMT_RT - 1) / SIMT_RT;
    const uint32_t nsteps = (dim + CH - 1) / CH;

    for (uint32_t iv = blockIdx.x; iv < num_iv; iv += gridDim.x) {
        const uint32_t base = iv * SIMT_RT;
#pragma unroll 1
        for (int t = 0; t < SIMT_RT / (SIMT_WARPS * R); ++t) {
            const uint32_t row0 = base + (uint32_t)(t * SIMT_WARPS + warp) * R;
            if (row0 >= n) continue;  // warp-uniform
            const T *rp[R];
#pragma unroll
            for (int r = 0; r < R; ++r) {
                uint32_t rr = row0 + r < n ? row0 + r : n - 1;  // clamp; masked below
                rp[r] = rows + (size_t)rr * dim;
            }
            float acc[V];
            float xx[R];
#pragma unroll
            for (int i = 0; i < V; ++i) acc[i] = 0.0f;
#pragma unroll
            for (int r = 0; r < R; ++r) xx[r] = 0.0f;

#pragma unroll 2
            for (uint32_t c = 0; c < nsteps; ++c) {
                const uint32_t e = c * CH + lane * EPL;
                if (e < dim) {
                    float x[R][EPL];
#pragma unroll
                    for (int r = 0; r < R; ++r) L::load(rp[r] + e, x[r]);
#pragma unroll
                    for (int qi = 0; qi < QT; ++qi) {
                        float q[EPL];
                        if constexpr (EPL == 1) {
                            q[0] = qs[qi * dim + e];
                        } else {
#pragma unroll
                            for (int h = 0; h < EPL / 4; ++h) {
                                float4 t4 = *reinterpret_cast<const float4 *>(&qs[qi * dim + e + 4 * h]);
                                q[4 * h + 0] = t4.x; q[4 * h + 1] = t4.y; q[4 * h + 2] = t4.z; q[4 * h + 3] = t4.w;
                            }
                        }
#pragma unroll
                        for (int r = 0; r < R; ++r) {
#pragma unroll
                            for (int u = 0; u < EPL; ++u) {
                                if constexpr (EUCLID) {
                                    float d = x[r][u] - q[u];
                                    acc[r * QT + qi] = fmaf(d, d, acc[r * QT + qi]);
                                } else {
                                    acc[r * QT + qi] = fmaf(x[r][u], q[u], acc[r * QT + qi]);
                                }
                            }
                        }
                    }
                    if constexpr (!EUCLID) {
#pragma unroll
                        for (int r = 0; r < R; ++r)
#pragma unroll
                            for (int u = 0; u < EPL; ++u) xx[r] = fmaf(x[r][u], x[r][u], xx[r]);
                    }
                }
            }

            // ---- fold across lanes; lane owns (row r, query qi) -----------------------------------
            warp_reduce_scatter<V>(acc, lane);
            const int j = lane / LPV;
            const int r = j / QT, qi = j - r * QT;
            float s = acc[0];
            float xr = 0.0f;
            if constexpr (!EUCLID) {
                warp_reduce_scatter<R>(xx, lane);
                xr = __shfl_sync(0xffffffffu, xx[0], r * (32 / R));
            }
            const uint32_t row = row0 + r;
            if ((lane % LPV) == 0 && row < n && (uint32_t)qi < p.nq && (!p.mask || ((p.mask[row >> 5] >> (row & 31)) & 1u)) &&
                (!TAGS || tag_admits(__ldg(p.row_tags + row), p.qfilter + p.q0 + qi))) {
                if constexpr (WINDOW) {
                    if (!window_admits(__ldg(p.row_values + row), p.qwindow + p.q0 + qi)) continue;
                }
                if constexpr (EUCLID) {
                    s = -s;
                } else if (p.metric == NK_METRIC_COSINE) {
                    // dot / sqrt(|x|^2 |q|^2); zero vector -> 0 (simd_amd64.go:31-35 NaN -> 0)
                    float den = sqrtf(xr * s_qq[qi]);
                    s = den > 0.0f ? s / den : 0.0f;
                }
                if constexpr (RANGE) {
                    if (s > -INFINITY && s >= s_tau[qi]) {  // NaN fails both compares
                        const int pos = atomicAdd(p.range_fill + p.q0 + qi, 1);
                        if (pos < (int)p.list_cap) p.partial[(size_t)(p.q0 + qi) * p.list_cap + pos] = make_key(s, (uint32_t)(p.row_base + row));
                    }
                } else if (s != s) {
                    s = -INFINITY;
                }
                if (!RANGE && s >= s_tau[qi] && s >= p.min_score) {  // (a prune with fewer than k live keys resets tau to -inf)
                    const uint64_t key = make_key(s, (uint32_t)(p.row_base + row));
                    if (!p.below || key < p.below[p.q0 + qi]) {
                        int pos = atomicAdd(&s_cnt[qi], 1);
                        if (pos < p.P) my_cand[(size_t)qi * p.P + pos] = key;
                        else atomicExch(p.flags, 1);
                    }
                }
            }
        }
        if constexpr (RANGE) continue;
        // ---- prune any buffer that could overflow during the next interval ---------------------
        __syncthreads();
        uint32_t need = 0;
#pragma unroll
        for (int qi = 0; qi < QT; ++qi) need |= (s_cnt[qi] > prune_at ? 1u : 0u) << qi;
        __syncthreads();
        if (need && p.P == 512) {
            // k <= 255: warp w prunes query w with the register radix select (QT <= 8 queries, 8 warps: all in parallel, ~2 us)
            if (warp < QT && (need & (1u << warp)))
                warp_prune<16>(my_cand + (size_t)warp * p.P, &s_cnt[warp], &s_tau[warp], p.k, lane, nullptr, 0, false, 0.0f, (int)p.k, p.min_score);
            __syncthreads();
        } else if (need) {
#pragma unroll 1
            for (int qi = 0; qi < QT; ++qi)
                if (need & (1u << qi)) block_prune(my_cand + (size_t)qi * p.P, p.P, &s_cnt[qi], &s_tau[qi], p.k, sbuf, p.P);
        }
    }

    if constexpr (RANGE) return;
    // ---- emit this CTA's best k per query --------------------------------------------------------
    if (p.P == 512) {
        // k <= 255: one warp per query selects the best k of the (<= 512) buffered keys with the register radix select
        // (~2 us) instead of a 45-stage block bitonic sort — on small shards (configs[0]: one interval per CTA) the
        // emission sort WAS the scan time.  The list goes out unsorted; merge_keys sorts.
        __syncthreads();
        for (uint32_t qi = warp; qi < p.nq; qi += SIMT_WARPS) {
            uint64_t *dst = p.partial + ((size_t)(p.q0 + qi) * gridDim.x + blockIdx.x) * p.k;
            warp_prune<16>(my_cand + (size_t)qi * p.P, &s_cnt[qi], &s_tau[qi], p.k, lane, dst, (int)p.k, false, 0.0f, (int)p.k, p.min_score);
        }
        return;
    }
#pragma unroll 1
    for (uint32_t qi = 0; qi < p.nq; ++qi) {
        block_prune(my_cand + (size_t)qi * p.P, p.P, &s_cnt[qi], &s_tau[qi], p.k, sbuf, p.P);
        uint64_t *dst = p.partial + ((size_t)(p.q0 + qi) * gridDim.x + blockIdx.x) * p.k;
        for (uint32_t i = tid; i < p.k; i += SIMT_THREADS) dst[i] = sbuf[i];  // zeros beyond the live entries
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------
template <bool RANGE, bool WINDOW> using SimtKernelT = void (*)(SimtArgs<RANGE, WINDOW>);

template <typename T, bool VEC, bool EUCLID, bool TAGS, bool RANGE, bool WINDOW>
static SimtKernelT<RANGE, WINDOW> pick_qt(int qt) {
    if constexpr (VEC) {
        switch (qt) {
            case 8: return knn_scan_simt_kernel<T, VEC, 8, 4, EUCLID, TAGS, RANGE, WINDOW>;
            case 4: return knn_scan_simt_kernel<T, VEC, 4, 8, EUCLID, TAGS, RANGE, WINDOW>;
            case 2: return knn_scan_simt_kernel<T, VEC, 2, 8, EUCLID, TAGS, RANGE, WINDOW>;
            default: return knn_scan_simt_kernel<T, VEC, 1, 8, EUCLID, TAGS, RANGE, WINDOW>;
        }
    } else {
        switch (qt) {
            case 4: return knn_scan_simt_kernel<T, VEC, 4, 8, EUCLID, TAGS, RANGE, WINDOW>;
            default: return knn_scan_simt_kernel<T, VEC, 1, 8, EUCLID, TAGS, RANGE, WINDOW>;
        }
    }
}

template <bool TAGS, bool RANGE, bool WINDOW>
static SimtKernelT<RANGE, WINDOW> pick_kernel_t(int dtype, bool vec, bool euclid, int qt) {
    if (dtype == NK_DTYPE_F16) {
        if (vec) return euclid ? pick_qt<__half, true, true, TAGS, RANGE, WINDOW>(qt) : pick_qt<__half, true, false, TAGS, RANGE, WINDOW>(qt);
        return euclid ? pick_qt<__half, false, true, TAGS, RANGE, WINDOW>(qt) : pick_qt<__half, false, false, TAGS, RANGE, WINDOW>(qt);
    }
    if (dtype == NK_DTYPE_BF16) {
        if (vec) return euclid ? pick_qt<__nv_bfloat16, true, true, TAGS, RANGE, WINDOW>(qt) : pick_qt<__nv_bfloat16, true, false, TAGS, RANGE, WINDOW>(qt);
        return euclid ? pick_qt<__nv_bfloat16, false, true, TAGS, RANGE, WINDOW>(qt) : pick_qt<__nv_bfloat16, false, false, TAGS, RANGE, WINDOW>(qt);
    }
    if (vec) return euclid ? pick_qt<float, true, true, TAGS, RANGE, WINDOW>(qt) : pick_qt<float, true, false, TAGS, RANGE, WINDOW>(qt);
    return euclid ? pick_qt<float, false, true, TAGS, RANGE, WINDOW>(qt) : pick_qt<float, false, false, TAGS, RANGE, WINDOW>(qt);
}

// Calls run(kern, params) with the kernel of a scan in the mode a.mode — a kNN mode (RANGE = false) or a range mode (RANGE =
// true), as ScanArgs::check found — and params(p), which turns the parameter block p into the kernel's: p itself, or for
// the window modes p with the windows appended.
template <bool RANGE, class Run> static int with_simt_kernel(const ScanArgs &a, bool vec, int qt, Run run) {
    const bool euclid = a.metric == NK_METRIC_EUCLIDEAN;
    if (mode_window(a.mode))
        return run(pick_kernel_t<true, RANGE, true>(a.dtype, vec, euclid, qt), [&](const SimtArgs<RANGE> &p) {
            SimtWindowParams<RANGE> w{};
            static_cast<SimtArgs<RANGE> &>(w) = p;
            w.row_values = a.row_values; w.qwindow = a.qwindow;
            return w;
        });
    const auto same = [](const SimtArgs<RANGE> &p) { return p; };
    return mode_tags(a.mode) ? run(pick_kernel_t<true, RANGE, false>(a.dtype, vec, euclid, qt), same)
                             : run(pick_kernel_t<false, RANGE, false>(a.dtype, vec, euclid, qt), same);
}

// cudaFuncSetAttribute + occupancy query once per (kernel, device, smem) instead of once per search
static std::mutex g_simt_mu;
static std::map<std::tuple<const void *, int, size_t>, int> g_simt_occ;
static std::map<std::pair<const void *, int>, size_t> g_simt_smem;
static int simt_ensure(const void *kern, int device, size_t smem) {
    std::lock_guard<std::mutex> lk(g_simt_mu);
    size_t &cur = g_simt_smem[{kern, device}];
    if (cur < smem || cur == 0) {
        NK_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        cur = smem;
    }
    return 0;
}
static int simt_occupancy(const void *kern, int device, size_t smem) {
    std::lock_guard<std::mutex> lk(g_simt_mu);
    auto key = std::make_tuple(kern, device, smem);
    auto it = g_simt_occ.find(key);
    if (it != g_simt_occ.end()) return it->second;
    int occ = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, SIMT_THREADS, smem) != cudaSuccess) { cudaGetLastError(); occ = 1; }
    if (occ < 1) occ = 1;
    if (occ > 8) occ = 8;
    g_simt_occ[key] = occ;
    return occ;
}

int simt_cap_for_k(uint32_t k) {
    uint32_t P = next_pow2(k + SIMT_RT + 1);
    return (int)(P < 512 ? 512 : P);
}

int scan_simt(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, uint64_t *out_keys, uint64_t *launches) {
    if (a.check(false, true)) return -1;
    if (a.n == 0 || a.Q == 0 || a.k == 0) return 0;
    if (a.k > NK_MAX_K) {
        set_error("k=%u exceeds NK_MAX_K=%u", a.k, NK_MAX_K);
        return -1;
    }
    const size_t esz = a.dtype == NK_DTYPE_F32 ? 4 : 2;
    const uint32_t vec_elems = a.dtype == NK_DTYPE_F32 ? 4 : 8;
    const bool vec = (a.dim % vec_elems == 0) && ((reinterpret_cast<uintptr_t>(a.rows) & 15) == 0);
    const int P = simt_cap_for_k(a.k);
    const size_t smem_budget = 96 * 1024;  // keeps >= 2 CTAs per SM
    const uint32_t num_iv = (a.n + SIMT_RT - 1) / SIMT_RT;

    const uint32_t max_grid = (uint32_t)di.num_sms * 8;
    (void)esz;

    uint32_t grid_used = 0;
    if (a.ev_begin) NK_CUDA_OK(cudaEventRecord(a.ev_begin, a.stream));
    for (uint32_t q0 = 0; q0 < a.Q;) {
        uint32_t left = a.Q - q0;
        int qt = left >= 5 ? 8 : left >= 3 ? 4 : left == 2 ? 2 : 1;
        if (!vec) qt = left >= 3 ? 4 : 1;
        while (qt > 1 && (size_t)P * 8 + (size_t)qt * a.dim * 4 > smem_budget) qt = vec ? qt / 2 : 1;
        size_t smem = (size_t)P * 8 + (size_t)qt * a.dim * 4;
        const uint32_t nq = left < (uint32_t)qt ? left : (uint32_t)qt;
        if (with_simt_kernel<false>(a, vec, qt, [&](auto kern, auto params) -> int {
                if (!smem_fits(di, reinterpret_cast<const void *>(kern), smem)) {
                    set_error("dim=%u too large for the SIMT scan (needs %zu B shared memory)", a.dim, smem);
                    return -1;
                }
                if (simt_ensure(reinterpret_cast<const void *>(kern), di.device_id, smem)) return -1;
                int occ = simt_occupancy(reinterpret_cast<const void *>(kern), di.device_id, smem);
                // One grid for every query group of this search so the per-CTA partial lists line up.
                if (grid_used == 0) {
                    grid_used = (uint32_t)di.num_sms * (uint32_t)occ;
                    if (grid_used > num_iv) grid_used = num_iv;
                    if (grid_used > max_grid) grid_used = max_grid;
                    if (ws_reserve((void **)&ws.cand, &ws.cand_bytes, (size_t)grid_used * 8 * P * 8)) return -1;
                    if (ws_reserve((void **)&ws.partial, &ws.partial_bytes, (size_t)a.Q * grid_used * a.k * 8)) return -1;
                }
                SimtParams p;
                p.rows = a.rows; p.n = a.n; p.dim = a.dim; p.row_base = a.row_base;
                p.queries = a.queries; p.q0 = q0; p.nq = nq; p.k = a.k;
                p.metric = a.metric; p.P = P; p.cand = ws.cand; p.partial = ws.partial; p.flags = ws.flags; p.only_if = a.only_if; p.below = a.below; p.mask = a.row_mask; p.min_score = a.min_score;
                p.row_tags = a.row_tags; p.qfilter = a.qfilter;
                NK_CUDA_OK(launch_pdl(kern, dim3(grid_used), dim3(SIMT_THREADS), smem, a.stream, a.only_if != nullptr && !a.defer_tail, params(p)));
                return 0;
            }))
            return -1;
        if (launches) ++*launches;
        if (a.main_launches) ++*a.main_launches;
        q0 += nq;
    }
    if (a.ev_end) NK_CUDA_OK(cudaEventRecord(a.ev_end, a.stream));
    // Fold the per-CTA lists: list l of query q starts at partial[(q*grid + l)*k].
    // ... and, when the caller wants them, the decoded (index, score) arrays in the same launch
    if (merge_keys(ws.partial, grid_used, a.k, (size_t)grid_used * a.k, a.Q, a.k, out_keys, a.stream, a.only_if, 0, a.out_idx, a.out_score,
                   a.metric))
        return -1;
    if (launches) ++*launches;
    return 0;
}

// Range mode: one launch per query group of QT <= 8 (one corpus read each), the same grid for all.
int scan_simt_range(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, uint32_t list_cap, uint64_t *launches) {
    if (a.n == 0 || a.Q == 0) return 0;
    const uint32_t vec_elems = a.dtype == NK_DTYPE_F32 ? 4 : 8;
    const bool vec = (a.dim % vec_elems == 0) && ((reinterpret_cast<uintptr_t>(a.rows) & 15) == 0);
    const size_t smem_budget = 96 * 1024;
    const uint32_t num_iv = (a.n + SIMT_RT - 1) / SIMT_RT;
    const uint32_t QA = range_qa(a.Q);
    if (a.ev_begin) NK_CUDA_OK(cudaEventRecord(a.ev_begin, a.stream));
    for (uint32_t q0 = 0; q0 < a.Q;) {
        const uint32_t left = a.Q - q0;
        int qt = left >= 5 ? 8 : left >= 3 ? 4 : left == 2 ? 2 : 1;
        if (!vec) qt = left >= 3 ? 4 : 1;
        while (qt > 1 && (size_t)qt * a.dim * 4 > smem_budget) qt = vec ? qt / 2 : 1;
        const size_t smem = (size_t)qt * a.dim * 4;  // the queries only: no candidate buffer
        const uint32_t nq = left < (uint32_t)qt ? left : (uint32_t)qt;
        if (with_simt_kernel<true>(a, vec, qt, [&](auto kern, auto params) -> int {
                if (!smem_fits(di, reinterpret_cast<const void *>(kern), smem)) {
                    set_error("dim=%u too large for the SIMT scan (needs %zu B shared memory)", a.dim, smem);
                    return -1;
                }
                if (simt_ensure(reinterpret_cast<const void *>(kern), di.device_id, smem)) return -1;
                const int occ = simt_occupancy(reinterpret_cast<const void *>(kern), di.device_id, smem);
                uint32_t grid = (uint32_t)di.num_sms * (uint32_t)occ;
                if (grid > num_iv) grid = num_iv;
                SimtRangeParams p{};
                p.rows = a.rows; p.n = a.n; p.dim = a.dim; p.row_base = a.row_base;
                p.queries = a.queries; p.q0 = q0; p.nq = nq; p.k = 1;
                p.metric = a.metric; p.P = 0; p.partial = ws.partial; p.flags = ws.flags; p.mask = a.row_mask; p.min_score = a.min_score;
                p.row_tags = a.row_tags; p.qfilter = a.qfilter;
                p.range_tau = reinterpret_cast<const uint32_t *>(ws.keys2); p.range_fill = reinterpret_cast<int *>(ws.keys2) + QA; p.list_cap = list_cap;
                NK_CUDA_OK(launch_pdl(kern, dim3(grid), dim3(SIMT_THREADS), smem, a.stream, false, params(p)));
                return 0;
            }))
            return -1;
        if (launches) ++*launches;
        if (a.main_launches) ++*a.main_launches;
        q0 += nq;
    }
    if (a.ev_end) NK_CUDA_OK(cudaEventRecord(a.ev_end, a.stream));
    return 0;
}

}  // namespace nk
