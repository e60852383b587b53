// assign_tensor.cu — k-means assignment step on the tensor cores (pkg/gpu/kmeans.go:458-546; SURVEY.md §8(f)4).
//
// nearest centroid of every corpus row = the Q x N^T contraction of the scan with Q = #centroids and an ARGMAX over the
// centroid columns instead of a per-query top-k.  The kernel reuses the shadow scan's pipeline (scan_tensor_shared.cuh:
// TMA slabs of the BF16 shadow and of the bf16 centroids, wgmma from shared memory, accumulators in the registers of two
// consumer warpgroups; the centroids are prepared by filter_prep_kernel) with one more loop level — every corpus tile is multiplied with each block of 64 centroids in turn
// (the tile is re-read from L2, it crossed HBM once) — and a register-only epilogue: each thread keeps, for each of its
// four fragment rows, the four best UPPER bounds and the best LOWER bound over its columns of every centroid block; the
// four lanes that share a row merge their lists at the end.
//   cosine    (assignToCentroidsGPU, kmeans.go:491-546)  score = x.c/|c|            (|x| > 0 does not change the argmax)
//   euclidean (assignToCentroids,    kmeans.go:458-489)  score = 2 x.c - |c|^2      (argmin |x-c|^2)
// with the rigorous bound of scan_tensor_shadow.cu (over the BF16 shadow, or the int8 image: s8 MMAs, 128-byte slabs of
// 128 elements, the estimate scaled by the row's and the centroid's scales), widened under euclidean by the rounding of kmeans.go's own
// arithmetic (fp32 differences: 2^-22 (|x|^2 - lo), DESIGN §7 item 3).  A row whose runner-up cannot reach the winner's
// lower bound is decided; the others (near-ties) are listed with their <= 3 candidates (or ALL) and assign_fixup_kernel
// decides them with the contract's arithmetic: squaredEuclidean bit for bit, or the fp64 cosine (strict comparison in
// ascending centroid order = lowest index wins ties, kmeans.go:470-476,529-534).
#include <cuda.h>
#include <float.h>
#include <stdlib.h>

#include "kernels.cuh"
#include "ptx_sm90.cuh"
#include "scan_tensor_shared.cuh"
#include "sq_euclid.cuh"

namespace nk {

namespace asg {
using namespace tc;
constexpr int NTHREADS = 384;
constexpr int QT = 64;
constexpr int BKB = 64;
constexpr int ASTAGES = 4;
constexpr int A_BYTES = ROWS * 128;
constexpr int B_BYTES = QT * 128;
constexpr int BSTAGES = 8;
constexpr int RING_BYTES = ASTAGES * A_BYTES + BSTAGES * B_BYTES;
constexpr int EPI_WARP0 = 4;
constexpr uint32_t NONE = 0xffffffffu, ALL = 0xfffffffeu;

struct Params {
    uint32_t n, nslab, K, nqb;   // rows, 128-byte slabs per row, centroids, blocks of 64 centroids
    int metric;
    const float *qn, *qa, *qb;   // per centroid (padded): |c| (1 for cosine), bound factors
    const float *xnorm2, *dnorm2;
    const float *xscale, *qscale;  // int8 image: per row, per centroid (padded)
    uint32_t *assign;            // [n] out
    uint32_t *amb_count, *amb_rows, *amb_cand;  // near-ties: count, rows, 4 candidates each (ALL = every centroid)
    uint32_t amb_cap;
};

struct __align__(8) Shared {
    Rings<ASTAGES> ring;
};
}  // namespace asg

template <ptx::Opnd OP>
__global__ void __launch_bounds__(asg::NTHREADS, 1)
assign_scan_kernel(const __grid_constant__ CUtensorMap map_rows, const __grid_constant__ CUtensorMap map_q, asg::Params p) {
    using namespace asg;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *smem_raw = smem_dyn + ((1024u - (ptx::smem_u32(smem_dyn) & 1023u)) & 1023u);
    unsigned char *a_base = smem_raw;
    unsigned char *b_base = smem_raw + (size_t)ASTAGES * A_BYTES;
    Shared &sh = *reinterpret_cast<Shared *>(smem_raw + (size_t)RING_BYTES);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t num_tiles = (p.n + ROWS - 1) / ROWS, nslab = p.nslab, nqb = p.nqb;
    constexpr bool S8 = OP == ptx::Opnd::S8;
    constexpr uint32_t KCOLS = S8 ? 128 : BKB;  // elements per 128-byte slab row

    if (warp == 0 && lane == 0) {
        ptx::prefetch_tensormap(&map_rows);
        ptx::prefetch_tensormap(&map_q);
        sh.ring.init(BSTAGES);
    }
    __syncthreads();

    if (warp == 0) {
        // TMA producer: shadow slabs; a tile is streamed once per centroid block (first from HBM, then from L2)
        tma_producer<ASTAGES>(sh.ring.aempty, blockIdx.x, num_tiles, gridDim.x, nqb, nslab, false, [&](uint32_t s, uint32_t tile, uint32_t qbk, uint32_t j) {
            ptx::mbar_arrive_expect_tx(&sh.ring.afull[s], A_BYTES);
            ptx::tma_load_2d(&map_rows, &sh.ring.afull[s], a_base + (size_t)s * A_BYTES, (int32_t)(j * KCOLS), (int32_t)(tile * ROWS),
                             qbk + 1 == nqb ? ptx::CACHE_EVICT_FIRST : ptx::CACHE_EVICT_NORMAL);
        });
    } else if (warp == 3) {
        // TMA producer: centroid slabs (L2-resident)
        tma_producer<BSTAGES>(sh.ring.bempty, blockIdx.x, num_tiles, gridDim.x, nqb, nslab, false, [&](uint32_t s, uint32_t, uint32_t qbk, uint32_t j) {
            ptx::mbar_arrive_expect_tx(&sh.ring.bfull[s], B_BYTES);
            ptx::tma_load_2d(&map_q, &sh.ring.bfull[s], b_base + (size_t)s * B_BYTES, (int32_t)(j * KCOLS), (int32_t)(qbk * QT), ptx::CACHE_EVICT_LAST);
        });
    } else if (warp >= EPI_WARP0) {
        // consumers: warpgroup m owns rows [128 m, 128 m + 128) of the tile as two m64 halves h; thread = 4 rows
        // (rbase + 64 h + 8 r) x QT/4 centroid columns (cbase + 8 (j / 2) + j % 2) of every centroid block
        const uint32_t ewarp = warp - EPI_WARP0, m = ewarp >> 2, wq = ewarp & 3;
        const uint32_t rbase = m * 128 + wq * 16 + ((uint32_t)lane >> 2), cbase = 2u * ((uint32_t)lane & 3u);
        const bool euclid = p.metric == NK_METRIC_EUCLIDEAN;
        // score = mul * acc - (euclid ? |c|^2 : 0);  bound = ra qa[c] + rb qb[c] (+ 1e-6 |c|^2 + 2^-22 (xhi - (score - bound)))
        const float mul = euclid ? 2.0f : 1.0f;
        float acc[2][QT / 2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < QT / 2; ++i) acc[h][i] = 0.0f;
        uint32_t g = 0;
        for (uint32_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            float x2[4], ra[4], rb[4], xs[4], maxlo[4], u[4][4];
            uint32_t id[4][4];
#pragma unroll
            for (int ri = 0; ri < 4; ++ri) {
                const uint32_t row = tile * ROWS + rbase + 64 * (ri >> 1) + 8 * (ri & 1);
                x2[ri] = row < p.n ? __ldg(p.xnorm2 + row) : 0.0f;
                const float dxn = sqrtf(row < p.n ? __ldg(p.dnorm2 + row) : 0.0f) * 1.0001f;
                ra[ri] = mul * dxn;
                rb[ri] = mul * sqrtf(x2[ri]);
                xs[ri] = S8 ? mul * (row < p.n ? __ldg(p.xscale + row) : 0.0f) : mul;  // the estimate's multiplier
                maxlo[ri] = -INFINITY;
#pragma unroll
                for (int e = 0; e < 4; ++e) { u[ri][e] = -INFINITY; id[ri][e] = NONE; }
            }
            for (uint32_t qbk = 0; qbk < nqb; ++qbk) {
                for (uint32_t j = 0; j < nslab; ++j, ++g) {
                    const uint32_t sa = g % ASTAGES, sbq = g % BSTAGES;
                    ptx::mbar_wait(&sh.ring.bfull[sbq], (g / BSTAGES) & 1);
                    ptx::mbar_wait(&sh.ring.afull[sa], (g / ASTAGES) & 1);
                    const uint64_t bdesc = ptx::make_smem_desc_sw128(ptx::smem_u32(b_base + (size_t)sbq * B_BYTES));
                    const uint32_t abase = ptx::smem_u32(a_base + (size_t)sa * A_BYTES + (size_t)m * (A_BYTES / 2));
                    ptx::wgmma_fence();
#pragma unroll
                    for (uint32_t h = 0; h < 2; ++h) {
                        const uint64_t adesc = ptx::make_smem_desc_sw128(abase + h * (A_BYTES / 4));
#pragma unroll
                        for (uint32_t kk = 0; kk < 4; ++kk) ptx::wgmma_op<QT, OP>(acc[h], adesc + kk * 2, bdesc + kk * 2, (j | kk) != 0);
                    }
                    ptx::wgmma_commit();
                    ptx::wgmma_wait_all();
                    ptx::fence_acc(acc[0]);
                    ptx::fence_acc(acc[1]);
                    __syncwarp();
                    if (lane == 0) { ptx::mbar_arrive(&sh.ring.aempty[sa]); ptx::mbar_arrive(&sh.ring.bempty[sbq]); }
                }
#pragma unroll
                for (int jj = 0; jj < QT / 4; ++jj) {
                    const uint32_t ci = qbk * QT + cbase + 8 * (jj >> 1) + (jj & 1);  // centroid index, ascending in jj
                    if (ci >= p.K) continue;
                    const float qn = __ldg(p.qn + ci), qa = __ldg(p.qa + ci), qb = __ldg(p.qb + ci);
                    const float cc = euclid ? qn * qn : 0.0f;
                    const float qs = S8 ? __ldg(p.qscale + ci) : 1.0f;
#pragma unroll
                    for (int ri = 0; ri < 4; ++ri) {
                        const float av = acc[ri >> 1][(jj >> 1) * 4 + (ri & 1) * 2 + (jj & 1)];
                        const float s = fmaf(S8 ? __int2float_rn(__float_as_int(av)) * qs : av, xs[ri], -cc);
                        float bnd = fmaf(ra[ri], qa, rb[ri] * qb) + 1e-6f * cc;
                        // kmeans.go rounds every difference x_j - c_j to fp32: its squared distance is within 2^-23 (1 + 2^-15) of
                        // the exact one, which is at most |x|^2 - lo <= 1.001 xx - lo (xx: the fp32 |x|^2, relative error < 6.3e-5)
                        if (euclid) bnd = fmaf(fmaxf(fmaf(x2[ri], 1.001f, bnd - s), 0.0f), 2.384185791015625e-7f, bnd);
                        const float up = s + bnd, lo = s - bnd;
                        maxlo[ri] = fmaxf(maxlo[ri], lo);  // NaN scores never enter: such rows end up in the exact fix-up
                        if (up > u[ri][3]) {  // strict: among equal bounds the lower centroid index stays ahead
                            u[ri][3] = up; id[ri][3] = ci;
#pragma unroll
                            for (int e = 3; e > 0; --e)
                                if (u[ri][e] > u[ri][e - 1]) {
                                    const float t = u[ri][e - 1]; u[ri][e - 1] = u[ri][e]; u[ri][e] = t;
                                    const uint32_t ti = id[ri][e - 1]; id[ri][e - 1] = id[ri][e]; id[ri][e] = ti;
                                }
                        }
                    }
                }
            }
#pragma unroll
            for (int ri = 0; ri < 4; ++ri) {
                // the four lanes of a row saw disjoint columns: merge their lists, ordered by (bound desc, centroid asc) —
                // the order the strict insertion above produces over ascending centroids
#pragma unroll
                for (int o = 1; o <= 2; o <<= 1) {
                    float pu[4];
                    uint32_t pid[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        pu[e] = __shfl_xor_sync(0xffffffffu, u[ri][e], o);
                        pid[e] = __shfl_xor_sync(0xffffffffu, id[ri][e], o);
                    }
                    maxlo[ri] = fmaxf(maxlo[ri], __shfl_xor_sync(0xffffffffu, maxlo[ri], o));
#pragma unroll
                    for (int f = 0; f < 4; ++f) {
                        if (pu[f] > u[ri][3] || (pu[f] == u[ri][3] && pid[f] < id[ri][3])) {
                            u[ri][3] = pu[f]; id[ri][3] = pid[f];
#pragma unroll
                            for (int e = 3; e > 0; --e)
                                if (u[ri][e] > u[ri][e - 1] || (u[ri][e] == u[ri][e - 1] && id[ri][e] < id[ri][e - 1])) {
                                    const float t = u[ri][e - 1]; u[ri][e - 1] = u[ri][e]; u[ri][e] = t;
                                    const uint32_t ti = id[ri][e - 1]; id[ri][e - 1] = id[ri][e]; id[ri][e] = ti;
                                }
                        }
                    }
                }
                const uint32_t row = tile * ROWS + rbase + 64 * (ri >> 1) + 8 * (ri & 1);
                if ((lane & 3) != 0 || row >= p.n) continue;
                const float u1 = u[ri][1], u2 = u[ri][2], u3 = u[ri][3], ml = maxlo[ri], xx = x2[ri];
                const uint32_t i0 = id[ri][0], i1 = id[ri][1], i2 = id[ri][2];
                const bool decided = i0 != NONE && !(u1 >= ml) && xx > 0.0f && xx < INFINITY;
                if (decided) {
                    p.assign[row] = i0;
                } else {
                    // near-tie (or a zero / non-finite row): the fix-up re-scores the candidates with the contract's arithmetic
                    const uint32_t pos = atomicAdd(p.amb_count, 1u);
                    if (pos < p.amb_cap) {
                        p.amb_rows[pos] = row;
                        const bool all = i0 == NONE || u3 >= ml || !(xx > 0.0f) || !(xx < INFINITY);
                        p.amb_cand[4 * pos + 0] = all ? ALL : i0;
                        p.amb_cand[4 * pos + 1] = all ? NONE : i1;
                        p.amb_cand[4 * pos + 2] = (all || !(u2 >= ml)) ? NONE : i2;
                        p.amb_cand[4 * pos + 3] = NONE;
                    }
                    p.assign[row] = i0 == NONE ? 0u : i0;  // overwritten by the fix-up
                }
            }
        }
    }
}

// fp64 cosine of the fp32 inputs: 0 for a zero row or centroid, NaN for non-finite inputs (never wins)
__device__ __forceinline__ double cosine64(const float *x, const float *c, uint32_t dim) {
    double xc = 0.0, xx = 0.0, cc = 0.0;
    for (uint32_t j = 0; j < dim; ++j) {
        const double a = x[j], b = c[j];
        xc = fma(a, b, xc); xx = fma(a, a, xx); cc = fma(b, b, cc);
    }
    return (xx == 0.0 || cc == 0.0) ? 0.0 : xc / (sqrt(xx) * sqrt(cc));
}

// The contract's decision for the listed rows: one warp per row, lane t scores candidates t, t + 32, ... sequentially (the
// near-tie rows are few), then the warp keeps the best (score, lowest index): the strict comparison in ascending centroid
// order of kmeans.go:470-476 (dist < minDist from math.MaxFloat64) and :529-534 (sim > maxSim); NaN never wins, and a
// row no candidate beats the initial value of goes to centroid 0.
__global__ void assign_fixup_kernel(const float *rows, uint32_t dim, const float *centroids, uint32_t K, int metric,
                                    const uint32_t *amb_count, uint32_t amb_cap, const uint32_t *amb_rows, const uint32_t *amb_cand,
                                    uint32_t *assign) {
    const int lane = threadIdx.x & 31;
    uint32_t total = *amb_count;
    if (total > amb_cap) total = amb_cap;
    const uint32_t warps = gridDim.x * (blockDim.x >> 5);
    const bool euclid = metric == NK_METRIC_EUCLIDEAN;
    for (uint32_t e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); e < total; e += warps) {
        const uint32_t row = amb_rows[e];
        const float *x = rows + (size_t)row * dim;
        const bool all = amb_cand[4 * e] == asg::ALL;
        const uint32_t count = all ? K : 3u;
        // euclidean: minimise d, kept as -d so both metrics maximise; ties -> lower index
        double best = euclid ? -DBL_MAX : -INFINITY;
        uint32_t nearest = asg::NONE;
        for (uint32_t t = lane; t < count; t += 32) {
            const uint32_t ci = all ? t : amb_cand[4 * e + t];
            if (ci >= K) continue;
            const float *c = centroids + (size_t)ci * dim;
            const double sc = euclid ? -sq_euclid64(x, c, dim) : cosine64(x, c, dim);
            if (sc > best || (sc == best && ci < nearest)) { best = sc; nearest = ci; }
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, o);
            const uint32_t on = __shfl_xor_sync(0xffffffffu, nearest, o);
            if (ob > best || (ob == best && on < nearest)) { best = ob; nearest = on; }
        }
        if (lane == 0) assign[row] = nearest == asg::NONE ? 0u : nearest;
    }
}

// A centroid with a NaN or infinite element scores NaN under the contract (never wins), but filter_prep_kernel scales it to
// a zero vector under cosine (t = |c|^2 is not > 0 or 1/|c| = 0), which would score an exact 0 with a zero bound.  A NaN
// bound factor keeps such a centroid out of every row's candidates (its upper and lower bounds are NaN).
__global__ void assign_mark_nonfinite_kernel(const float *centroids, uint32_t K, uint32_t dim, float *qb) {
    const uint32_t c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (c >= K) return;
    bool bad = false;
    for (uint32_t j = lane; j < dim; j += 32) bad |= !isfinite(centroids[(size_t)c * dim + j]);
    if (__any_sync(0xffffffffu, bad) && lane == 0) qb[c] = __int_as_float(0x7fc00000);
}

bool assign_tensor_supported(const DeviceInfo &di, uint32_t dim, uint32_t K, int metric) {
    if (const char *e = getenv("NK_ASSIGN_TENSOR"))
        if (atoi(e) == 0) return false;
    return di.cc >= 90 && dim % 4 == 0 && dim >= 32 && dim <= 32768 && K >= 1 && (metric == NK_METRIC_COSINE || metric == NK_METRIC_EUCLIDEAN);
}

// rows / img: one fp32 shard and its BF16 shadow or int8 image (device pointers); centroids_dev: [K x dim] fp32 on the same
// device; assign_dev: [n].
int assign_tensor(const DeviceInfo &di, const float *rows, const RowImage &img, uint32_t n, uint32_t dim, const float *centroids_dev, uint32_t K,
                  int metric, AssignTies ties, uint32_t *assign_dev, cudaStream_t stream, uint64_t *launches, void **scratch, size_t *scratch_bytes) {
    using namespace asg;
    if (n == 0) return 0;
    if (ties.cap < n) { set_error("assign_tensor: near-tie list shorter than the shard"); return -1; }
    const uint32_t nqb = (K + QT - 1) / QT, Kpad = nqb * QT;
    const float acc_c = (float)dim * 2.384185791015625e-7f + 4e-6f;
    // scratch: bf16 (int8 image: int8) centroids [Kpad x dimpad], qn / qa / qb (/ scales) [Kpad]
    const bool s8 = img.kind == RowImage::S8;
    const uint32_t esz = img.esz(), dimpad = img.dimpad;
    const size_t off_q = 0, off_f = ((size_t)Kpad * dimpad * esz + 255) & ~(size_t)255;
    const size_t total = off_f + (size_t)4 * Kpad * 4;
    if (ws_reserve(scratch, scratch_bytes, total)) return -1;  // grow-only, reused across calls
    unsigned char *buf = static_cast<unsigned char *>(*scratch);
    float *qn = reinterpret_cast<float *>(buf + off_f), *qa = qn + Kpad, *qb = qa + Kpad, *qsc = qb + Kpad;
    uint32_t *amb_count = ties.count, *amb_rows = ties.rows, *amb_cand = ties.cand;
    int rc = 0;
    do {
        if (cudaMemsetAsync(amb_count, 0, 4, stream) != cudaSuccess) { rc = -1; break; }
        ScanArgs a;
        a.queries = centroids_dev; a.Q = K; a.dim = dim; a.metric = metric;
        PrepParams pp = prep_params(a, Kpad, dimpad);
        pp.acc_c = acc_c; pp.qnorm = qn; pp.qa = qa; pp.qb = qb;
        if (s8) { pp.qs8 = reinterpret_cast<int8_t *>(buf + off_q); pp.qscale = qsc; }
        else pp.qbf = reinterpret_cast<uint16_t *>(buf + off_q);
        if (launch_prep(di, a.mode, pp, stream, launches)) { rc = -1; break; }
        assign_mark_nonfinite_kernel<<<(K + 7) / 8, 256, 0, stream>>>(centroids_dev, K, dim, qb);
        CUtensorMap map_rows, map_q;
        if (tc_make_map(&map_rows, img.data, n, img.stride, esz, 128 / esz, ROWS, img.row_bytes())) { rc = -1; break; }
        if (tc_make_map(&map_q, buf + off_q, Kpad, dimpad, esz, 128 / esz, QT, (uint64_t)dimpad * esz)) { rc = -1; break; }
        const size_t smem = (size_t)RING_BYTES + sizeof(Shared) + 1024;
        const void *kern = s8 ? reinterpret_cast<const void *>(assign_scan_kernel<ptx::Opnd::S8>)
                              : reinterpret_cast<const void *>(assign_scan_kernel<ptx::Opnd::BF16>);
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) { rc = -1; break; }
        asg::Params p;
        p.n = n; p.nslab = dimpad * esz / 128; p.K = K; p.nqb = nqb; p.metric = metric;
        p.qn = qn; p.qa = qa; p.qb = qb; p.xnorm2 = img.xnorm2; p.dnorm2 = img.dnorm2; p.xscale = img.xscale; p.qscale = qsc;
        p.assign = assign_dev; p.amb_count = amb_count; p.amb_rows = amb_rows; p.amb_cand = amb_cand; p.amb_cap = n;
        const uint32_t num_tiles = (n + ROWS - 1) / ROWS;
        const uint32_t grid = num_tiles < (uint32_t)di.num_sms ? num_tiles : (uint32_t)di.num_sms;
        if (s8) assign_scan_kernel<ptx::Opnd::S8><<<grid, NTHREADS, smem, stream>>>(map_rows, map_q, p);
        else assign_scan_kernel<ptx::Opnd::BF16><<<grid, NTHREADS, smem, stream>>>(map_rows, map_q, p);
        assign_fixup_kernel<<<di.num_sms * 4, 256, 0, stream>>>(rows, dim, centroids_dev, K, metric, amb_count, n, amb_rows, amb_cand, assign_dev);
        if (cudaGetLastError() != cudaSuccess) { rc = -1; break; }
        if (launches) *launches += 3;
    } while (0);
    if (rc != 0) {
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) set_error("assign_tensor: %s", cudaGetErrorString(e));
    }
    cudaStreamSynchronize(stream);
    return rc;
}

// The search path's near-ties.  idx / sc: [n x k] results of a k = min(2, K) search of the rows against the centroids
// (warp_exact_score's fp32 scores, euclidean as the distance).  Each such score is within acc_c of the real cosine, or within
// acc_c d^2 of the real squared distance d^2, and kmeans.go's own arithmetic is within 2^-22 d^2 of it, so a row whose top
// two are further apart than 3 acc_c (d1^2 under euclidean) has the search's winner as the contract's; the others, and
// every row with a non-finite score or a missing result, are listed as ALL (DESIGN §7 item 3).
__global__ void assign_search_ties_kernel(const uint32_t *idx, const float *sc, uint32_t n, uint32_t k, uint32_t K, int metric,
                                          float acc_c, uint32_t *assign, uint32_t *amb_count, uint32_t *amb_rows, uint32_t *amb_cand) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const uint32_t i0 = idx[(size_t)r * k];
    assign[r] = i0 < K ? i0 : 0u;
    if (K < 2) return;  // one centroid: it is every row's
    const uint32_t i1 = idx[(size_t)r * k + 1];
    const double s0 = sc[(size_t)r * k], s1 = sc[(size_t)r * k + 1];
    bool tie = !(i0 < K && i1 < K && isfinite(s0) && isfinite(s1));
    if (!tie) {
        if (metric == NK_METRIC_EUCLIDEAN) tie = s1 * s1 - s0 * s0 <= 3.0 * acc_c * (s1 * s1);
        else tie = s0 - s1 <= 3.0 * acc_c;
    }
    if (tie) {
        const uint32_t pos = atomicAdd(amb_count, 1u);
        amb_rows[pos] = r;
        amb_cand[4 * pos] = asg::ALL;
        amb_cand[4 * pos + 1] = amb_cand[4 * pos + 2] = amb_cand[4 * pos + 3] = asg::NONE;
    }
}

int assign_from_search(const DeviceInfo &di, const float *rows, uint32_t n, uint32_t dim, const float *centroids_dev, uint32_t K, int metric,
                       const uint32_t *idx, const float *sc, uint32_t k, AssignTies ties, uint32_t *assign_dev, cudaStream_t stream,
                       uint64_t *launches) {
    if (n == 0) return 0;
    if (ties.cap < n) { set_error("assign_from_search: near-tie list shorter than the shard"); return -1; }
    const float acc_c = (float)dim * 2.384185791015625e-7f + 4e-6f;
    if (cudaMemsetAsync(ties.count, 0, 4, stream) != cudaSuccess) return -1;
    assign_search_ties_kernel<<<(n + 255) / 256, 256, 0, stream>>>(idx, sc, n, k, K, metric, acc_c, assign_dev, ties.count, ties.rows, ties.cand);
    assign_fixup_kernel<<<di.num_sms * 4, 256, 0, stream>>>(rows, dim, centroids_dev, K, metric, ties.count, n, ties.rows, ties.cand, assign_dev);
    if (launches) *launches += 2;
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("assign_from_search: %s", cudaGetErrorString(e)); return -1; }
    return 0;
}

}  // namespace nk
