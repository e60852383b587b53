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
// with the rigorous BF16 bound of scan_tensor_shadow.cu.  A row whose runner-up cannot reach the winner's lower bound is
// decided; the others (near-ties) are listed with their <= 4 candidates and assign_fixup_kernel re-scores those candidates
// exactly in fp32 (strict comparison in ascending centroid order = lowest index wins ties, kmeans.go:470-476,529-534).
#include <cuda.h>
#include <stdlib.h>

#include "kernels.cuh"
#include "ptx_sm90.cuh"
#include "scan_tensor_shared.cuh"

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
    uint32_t n, nslab, K, nqb;   // rows, 64-element slabs per row, centroids, blocks of 128 centroids
    int metric;
    const float *qn, *qa, *qb;   // per centroid (padded): |c| (1 for cosine), bound factors
    const float *xnorm2, *dnorm2;
    uint32_t *assign;            // [n] out
    uint32_t *amb_count, *amb_rows, *amb_cand;  // near-ties: count, rows, 4 candidates each (ALL = every centroid)
    uint32_t amb_cap;
};

struct __align__(8) Shared {
    Rings<ASTAGES> ring;
};
}  // namespace asg

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
            ptx::tma_load_2d(&map_rows, &sh.ring.afull[s], a_base + (size_t)s * A_BYTES, (int32_t)(j * BKB), (int32_t)(tile * ROWS),
                             qbk + 1 == nqb ? ptx::CACHE_EVICT_FIRST : ptx::CACHE_EVICT_NORMAL);
        });
    } else if (warp == 3) {
        // TMA producer: centroid slabs (L2-resident)
        tma_producer<BSTAGES>(sh.ring.bempty, blockIdx.x, num_tiles, gridDim.x, nqb, nslab, false, [&](uint32_t s, uint32_t, uint32_t qbk, uint32_t j) {
            ptx::mbar_arrive_expect_tx(&sh.ring.bfull[s], B_BYTES);
            ptx::tma_load_2d(&map_q, &sh.ring.bfull[s], b_base + (size_t)s * B_BYTES, (int32_t)(j * BKB), (int32_t)(qbk * QT), ptx::CACHE_EVICT_LAST);
        });
    } else if (warp >= EPI_WARP0) {
        // consumers: warpgroup m owns rows [128 m, 128 m + 128) of the tile as two m64 halves h; thread = 4 rows
        // (rbase + 64 h + 8 r) x QT/4 centroid columns (cbase + 8 (j / 2) + j % 2) of every centroid block
        const uint32_t ewarp = warp - EPI_WARP0, m = ewarp >> 2, wq = ewarp & 3;
        const uint32_t rbase = m * 128 + wq * 16 + ((uint32_t)lane >> 2), cbase = 2u * ((uint32_t)lane & 3u);
        const bool euclid = p.metric == NK_METRIC_EUCLIDEAN;
        // score = mul * acc - (euclid ? |c|^2 : 0);  bound = ra qa[c] + rb qb[c] (+ 1e-6 |c|^2)
        const float mul = euclid ? 2.0f : 1.0f;
        float acc[2][QT / 2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < QT / 2; ++i) acc[h][i] = 0.0f;
        uint32_t g = 0;
        for (uint32_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            float x2[4], ra[4], rb[4], maxlo[4], u[4][4];
            uint32_t id[4][4];
#pragma unroll
            for (int ri = 0; ri < 4; ++ri) {
                const uint32_t row = tile * ROWS + rbase + 64 * (ri >> 1) + 8 * (ri & 1);
                x2[ri] = row < p.n ? __ldg(p.xnorm2 + row) : 0.0f;
                const float dxn = sqrtf(row < p.n ? __ldg(p.dnorm2 + row) : 0.0f) * 1.0001f;
                ra[ri] = mul * dxn;
                rb[ri] = mul * sqrtf(x2[ri]);
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
                        for (uint32_t kk = 0; kk < 4; ++kk) ptx::wgmma_bf16_n64(acc[h], adesc + kk * 2, bdesc + kk * 2, (j | kk) != 0);
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
#pragma unroll
                    for (int ri = 0; ri < 4; ++ri) {
                        const float s = fmaf(acc[ri >> 1][(jj >> 1) * 4 + (ri & 1) * 2 + (jj & 1)], mul, -cc);
                        const float bnd = fmaf(ra[ri], qa, rb[ri] * qb) + 1e-6f * cc;
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
                    // near-tie (or a zero / non-finite row): exact fp32 re-scoring of the candidates decides
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

// Exact fp32 decision for the listed rows: one warp per row, candidates in ascending centroid order, strict comparison
// (kmeans.go:470-476: dist < minDist; :529-534: sim > maxSim), so the lowest index wins ties.
__global__ void assign_fixup_kernel(const float *rows, uint32_t dim, const float *centroids, uint32_t K, int metric,
                                    const uint32_t *amb_count, uint32_t amb_cap, const uint32_t *amb_rows, const uint32_t *amb_cand,
                                    uint32_t *assign) {
    const int lane = threadIdx.x & 31;
    uint32_t total = *amb_count;
    if (total > amb_cap) total = amb_cap;
    const uint32_t warps = gridDim.x * (blockDim.x >> 5);
    for (uint32_t e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); e < total; e += warps) {
        const uint32_t row = amb_rows[e];
        const float *x = rows + (size_t)row * dim;
        uint32_t cand[3] = {amb_cand[4 * e], amb_cand[4 * e + 1], amb_cand[4 * e + 2]};
        const bool all = cand[0] == asg::ALL;
        if (!all) {  // ascending order (3-element sorting network; NONE = 0xffffffff sorts last)
            if (cand[0] > cand[1]) { uint32_t t = cand[0]; cand[0] = cand[1]; cand[1] = t; }
            if (cand[1] > cand[2]) { uint32_t t = cand[1]; cand[1] = cand[2]; cand[2] = t; }
            if (cand[0] > cand[1]) { uint32_t t = cand[0]; cand[0] = cand[1]; cand[1] = t; }
        }
        float xx = 0.0f;
        if (metric != NK_METRIC_EUCLIDEAN) {
            for (uint32_t j = lane; j < dim; j += 32) xx = fmaf(x[j], x[j], xx);
#pragma unroll
            for (int o = 16; o; o >>= 1) xx += __shfl_xor_sync(0xffffffffu, xx, o);
        }
        float best = metric == NK_METRIC_EUCLIDEAN ? INFINITY : -INFINITY;
        uint32_t nearest = 0;
        const uint32_t count = all ? K : 3u;
        for (uint32_t t = 0; t < count; ++t) {
            const uint32_t ci = all ? t : cand[t];
            if (ci >= K) continue;
            const float *c = centroids + (size_t)ci * dim;
            float a = 0.0f, cc = 0.0f;
            if (metric == NK_METRIC_EUCLIDEAN) {
                for (uint32_t j = lane; j < dim; j += 32) { const float d = x[j] - c[j]; a = fmaf(d, d, a); }
            } else {
                for (uint32_t j = lane; j < dim; j += 32) { a = fmaf(x[j], c[j], a); cc = fmaf(c[j], c[j], cc); }
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) {
                a += __shfl_xor_sync(0xffffffffu, a, o);
                cc += __shfl_xor_sync(0xffffffffu, cc, o);
            }
            if (metric == NK_METRIC_EUCLIDEAN) {
                if (a < best) { best = a; nearest = ci; }
            } else {
                const float den = sqrtf(xx * cc);
                const float sim = den > 0.0f ? a / den : 0.0f;  // cosineSimilarityFlat: 0 for zero vectors (gpu.go:2467-2484)
                if (sim > best) { best = sim; nearest = ci; }
            }
        }
        if (lane == 0) assign[row] = nearest;
    }
}

bool assign_tensor_supported(const DeviceInfo &di, uint32_t dim, uint32_t K, int metric) {
    if (const char *e = getenv("NK_ASSIGN_TENSOR"))
        if (atoi(e) == 0) return false;
    return di.cc >= 90 && dim % 4 == 0 && dim >= 32 && dim <= 32768 && K >= 1 && (metric == NK_METRIC_COSINE || metric == NK_METRIC_EUCLIDEAN);
}

// rows / shadow / norms: one shard (device pointers); centroids_dev: [K x dim] fp32 on the same device; assign_dev: [n].
int assign_tensor(const DeviceInfo &di, const float *rows, const void *shadow, uint32_t dimpad, const float *xnorm2, const float *dnorm2,
                  uint32_t n, uint32_t dim, const float *centroids_dev, uint32_t K, int metric, uint32_t *assign_dev, cudaStream_t stream,
                  uint64_t *launches, void **scratch, size_t *scratch_bytes) {
    using namespace asg;
    if (n == 0) return 0;
    const uint32_t nqb = (K + QT - 1) / QT, Kpad = nqb * QT;
    const float acc_c = (float)dim * 2.384185791015625e-7f + 4e-6f;
    // scratch: bf16 centroids [Kpad x dimpad], qn / qa / qb [Kpad], near-tie list (every row could be one)
    const size_t off_q = 0, off_f = ((size_t)Kpad * dimpad * 2 + 255) & ~(size_t)255, off_amb = off_f + (((size_t)3 * Kpad * 4 + 255) & ~(size_t)255);
    const size_t total = off_amb + 4 + (size_t)n * 4 + (size_t)n * 16 + 64;
    if (ws_reserve(scratch, scratch_bytes, total)) return -1;  // grow-only, reused across calls
    unsigned char *buf = static_cast<unsigned char *>(*scratch);
    float *qn = reinterpret_cast<float *>(buf + off_f), *qa = qn + Kpad, *qb = qa + Kpad;
    uint32_t *amb_count = reinterpret_cast<uint32_t *>(buf + off_amb);
    uint32_t *amb_rows = amb_count + 1;
    uint32_t *amb_cand = amb_rows + n;
    int rc = 0;
    do {
        if (cudaMemsetAsync(amb_count, 0, 4, stream) != cudaSuccess) { rc = -1; break; }
        ScanArgs a;
        a.queries = centroids_dev; a.Q = K; a.dim = dim; a.metric = metric;
        PrepParams pp = prep_params(a, Kpad, dimpad);
        pp.acc_c = acc_c; pp.qbf = reinterpret_cast<uint16_t *>(buf + off_q); pp.qnorm = qn; pp.qa = qa; pp.qb = qb;
        if (launch_prep(di, pp, stream, launches)) { rc = -1; break; }
        CUtensorMap map_rows, map_q;
        if (tc_make_map(&map_rows, shadow, n, dimpad, 2, BKB, ROWS, (uint64_t)dimpad * 2)) { rc = -1; break; }
        if (tc_make_map(&map_q, buf + off_q, Kpad, dimpad, 2, BKB, QT, (uint64_t)dimpad * 2)) { rc = -1; break; }
        const size_t smem = (size_t)RING_BYTES + sizeof(Shared) + 1024;
        if (cudaFuncSetAttribute(assign_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) { rc = -1; break; }
        asg::Params p;
        p.n = n; p.nslab = dimpad / BKB; p.K = K; p.nqb = nqb; p.metric = metric;
        p.qn = qn; p.qa = qa; p.qb = qb; p.xnorm2 = xnorm2; p.dnorm2 = dnorm2;
        p.assign = assign_dev; p.amb_count = amb_count; p.amb_rows = amb_rows; p.amb_cand = amb_cand; p.amb_cap = n;
        const uint32_t num_tiles = (n + ROWS - 1) / ROWS;
        const uint32_t grid = num_tiles < (uint32_t)di.num_sms ? num_tiles : (uint32_t)di.num_sms;
        assign_scan_kernel<<<grid, NTHREADS, smem, stream>>>(map_rows, map_q, p);
        assign_fixup_kernel<<<di.num_sms * 4, 256, 0, stream>>>(rows, dim, centroids_dev, K, metric, amb_count, n, amb_rows, amb_cand, assign_dev);
        if (cudaGetLastError() != cudaSuccess) { rc = -1; break; }
        if (launches) *launches += 2;
    } while (0);
    if (rc != 0) {
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) set_error("assign_tensor: %s", cudaGetErrorString(e));
    }
    cudaStreamSynchronize(stream);
    return rc;
}

}  // namespace nk
