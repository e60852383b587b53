// scan_tensor.cu — fused distance + top-k scan over the FP32 rows on the tensor cores (wgmma + TMA + mbarrier):
// the path of shards without a BF16 shadow, the retry stage of the shadow filter (scan_tensor_shadow.cu), the exact
// 3xTF32 scan, plus the finish step and the host logic both filters share.
//
// For Q > ~16 queries the CUDA-core scan stops being HBM-bound (fp32 FMA ridge ~10 flop/byte, the batch needs
// Q/2 flop/byte), so the Q x N^T contraction moves to wgmma.  fp32 inputs on tensor cores mean TF32
// (10-bit mantissa), which by itself cannot meet "identical index sets, 1e-4".  Two modes (template NT):
//
//   NT = 3  "exact":  3xTF32 split  x*q ~= xl*qh + xh*ql + xh*qh  (xh = rn_tf32(x), xl = x - xh exactly),
//           fp32 accumulation, ~2^-21 relative per product.  Per-CTA exact top-k lists.
//   NT = 1  "filter": ONE TF32 product per element (a third of the tensor work and energy — the chip is
//           power-capped when HBM and the tensor pipes both run flat out) with a RIGOROUS error margin:
//           |s_hat - s| <= c*|x|*|q|, c = 2^-10 + d*2^-22  (rounding of both operands + fp32 accumulation), so
//           every row whose upper bound s_hat + B can still reach the running k-th best lower bound is kept.
//           The few survivors (k + a handful) are re-scored EXACTLY in fp32 by filter_finish_kernel, so final
//           scores/indices carry no TF32 error at all.  If a margin buffer overflows (adversarial near-ties) a flag
//           is raised ON DEVICE and the NT=3 kernels — enqueued behind, early-exiting when the flag is clear —
//           redo the search exactly.  No host round trip.
//
// One persistent CTA per SM, warp-specialised (12 warps):
//   warp 0      TMA producer: corpus K-slabs [256 rows x 32 floats] (128B-swizzled), ring released once the MMAs that
//               read the slab have completed (EVICT_FIRST);
//   warp 3      TMA producer: query slabs (pre-rounded hi [+ lo], [QT x 32 floats] each, L2-resident, EVICT_LAST);
//   warps 4-11  two consumer warpgroups, one per 128-row M-tile.  Per slab: split (thread = corpus row: swizzled LDS.128,
//               xh rounded in place, xl into a per-warpgroup tile, |x|^2 on the side), then wgmma.m64nQTk8.tf32 with A
//               and B from shared memory, fp32 accumulators in registers.  Per tile: scale / bound straight from the
//               accumulator registers, compare against each query's running threshold with a compact mask pass,
//               append the few survivors; warp-level register top-k prune.  Distances never go to memory.
// Exact mode: per-CTA lists are folded by merge_keys().  Filter mode: CTAs share their thresholds through a per-query
// atomic max, append their survivors to one list per query, and filter_finish_kernel (below) selects, re-scores and
// sorts.  Large batches: 2 / 4 query groups per launch share every corpus tile through L2 (Params::qgroups).
// The set-up, the producer loop and the filter epilogue are scan_tensor_shared.cuh's, shared with the 16-bit kernel.
//
// Algorithmic HBM traffic per launch: n*dim*4 (corpus, once); query re-reads are served from L2.
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <mutex>
#include <string>

#include "kernels.cuh"
#include "ptx_sm90.cuh"
#include "scan_tensor_shared.cuh"

namespace nk {

namespace tc {
constexpr int QT_MAX = 128;      // queries per launch (MMA N): 64, or 128 for large batches (filter mode)
constexpr int ASTAGES = 4;       // corpus-slab smem ring
constexpr int A_BYTES = ROWS * BK * 4;   // 32 KB
constexpr int EPI_WARP0 = 4;     // consumer warpgroups: warps 4-7 (rows 0-127), 8-11 (rows 128-255)

template <int NT, int QT> struct Cfg {
    static constexpr int PARTS = NT == 3 ? 2 : 1;          // hi (+ lo)
    static constexpr int B_BYTES = QT * BK * 4;            // one part of one query slab (8 / 16 KB)
    static constexpr int BST_BYTES = PARTS * B_BYTES;
    static constexpr int B_BUDGET = NT == 3 ? 48 * 1024 : 80 * 1024;  // exact mode also holds the xl tiles (32 KB)
    static constexpr int BSTAGES = B_BUDGET / BST_BYTES > MAX_BSTAGES ? MAX_BSTAGES : B_BUDGET / BST_BYTES;
    static constexpr int XL_BYTES = NT == 3 ? A_BYTES : 0;    // xl = x - xh of the current slab, one 16 KB tile per warpgroup
    static constexpr int RING_BYTES = ASTAGES * A_BYTES + BSTAGES * BST_BYTES + XL_BYTES;
    static_assert(BSTAGES >= 2, "ring too shallow");
};

struct __align__(8) Shared {
    Rings<ASTAGES> ring;      // corpus and query slabs in smem: TMA -> consumers -> TMA
    unsigned int maxxx;      // running max of |x|^2 (float bits) over the rows this CTA has scored
    float xx[ROWS];           // |x|^2 per row of the current tile (split step -> epilogue, same warpgroup)
    float tau[QT_MAX];
    float qn[QT_MAX];
    int cnt[QT_MAX];
};
}  // namespace tc

// Wait-time instrumentation (NK_TC_DEBUG bit 64): cycles CTA 0 spends blocked at each hand-off.
__device__ long long g_tc_prof[32];
#define TC_PROF_BEGIN() long long _t0 = prof ? clock64() : 0
#define TC_PROF_END(slot) do { if (prof) { long long _t1 = clock64(); acc_##slot += _t1 - _t0; } } while (0)

// ---------------------------------------------------------------------------------------------------
// filter_prep_kernel — everything a filter search needs before its scan, in ONE launch (one CTA per padded query row):
//   * |q|, cosine normalisation; TF32 hi / lo split (TF32 filter + exact 3xTF32 stages); BF16 copy with the measured
//     rounding residues qa = |bf16(q)|, qb = |q - bf16(q)| + acc_c |q| (shadow stage);
//   * clears the search state the scan kernels accumulate into (shared thresholds, list fills, status words 1..7) —
//     previously two cudaMemsetAsync;
//   * SAMPLED INITIAL THRESHOLD: the query's exact fp32 score against `sample` evenly spaced rows of the shard; the k-th
//     largest of their LOWER bounds (score minus the fp32 summation allowance) is a lower bound of the true k-th best
//     score, so the scan starts with a real threshold instead of buffering every (row, query) pair of its first two
//     tiles and pruning 64-128 full buffers per CTA (~25 us per launch, the largest fixed cost of a small-shard search).
// ---------------------------------------------------------------------------------------------------
constexpr int PREP_THREADS = 1024;  // 32 warps: the sample scoring is latency-bound (one 4 KB row per warp at a time)

// TAGS (filtered searches): the sample only counts rows the query admits, so a query with fewer than k admissible sample rows
// starts at the score floor.  WINDOW (windowed searches, with TAGS): admitted means by the tag filter AND the value window.
template <bool TAGS, bool WINDOW>
__global__ void __launch_bounds__(PREP_THREADS) filter_prep_kernel(PrepParams p) {
    extern __shared__ __align__(16) unsigned char prep_smem[];
    float *qs = reinterpret_cast<float *>(prep_smem);                                  // raw query [dim]
    uint64_t *skeys = reinterpret_cast<uint64_t *>(prep_smem + (size_t)((p.dim + 3) & ~3u) * 4);  // [sample]
    __shared__ float red[3][PREP_THREADS / 32];
    if (p.only_if && *p.only_if == 0) return;
    const uint32_t row = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    constexpr int NW = PREP_THREADS / 32;
    // ---- clear the search state: own entry, block 0 also the padding and the status words
    if (p.state) {
        if (tid == 0) { p.state[row] = 0u; p.state[p.QA + row] = 0u; }
        if (row == 0) {
            for (uint32_t i = p.Qpad + tid; i < p.QA; i += PREP_THREADS) { p.state[i] = 0u; p.state[p.QA + i] = 0u; }
            if (tid >= 1 && tid <= 7) p.flags[tid] = 0;
        }
    }
    float t = 0.0f;
    if (row < p.Q) {
        float a = 0.0f;
        for (uint32_t j = tid; j < p.dim; j += PREP_THREADS) {
            const float v = p.q[(size_t)row * p.dim + j];
            qs[j] = v;
            a = fmaf(v, v, a);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) red[0][w] = a;
    }
    __syncthreads();
    if (row < p.Q)
        for (int i = 0; i < NW; ++i) t += red[0][i];
    const float nrm = sqrtf(t);
    // zero query -> all cosine scores 0 (simd_amd64.go:31-35)
    const float inv = p.normalise ? (t > 0.0f ? 1.0f / nrm : 0.0f) : 1.0f;
    const float qn = p.normalise ? (t > 0.0f ? 1.0f : 0.0f) : nrm;
    if (p.qhi) {
        for (uint32_t j = tid; j < p.dim; j += PREP_THREADS) {
            const float v = row < p.Q ? qs[j] * inv : 0.0f;
            const float h = __uint_as_float(ptx::tf32_round_bits(__float_as_uint(v)));
            p.qhi[(size_t)row * p.dim + j] = h;
            if (p.qlo) p.qlo[(size_t)row * p.dim + j] = v - h;
        }
    }
    float hh = 0.0f, dd = 0.0f;
    if (p.qbf) {
        for (uint32_t j = tid; j < p.dimpad; j += PREP_THREADS) {
            const float v = (row < p.Q && j < p.dim) ? qs[j] * inv : 0.0f;
            uint16_t b;
            float vb;
            if (p.qbf_f16) {
                const __half h = __float2half_rn(v);
                b = __half_as_ushort(h);
                vb = __half2float(h);
            } else {
                b = ptx::f32_to_bf16_bits(v);
                vb = __uint_as_float((uint32_t)b << 16);
            }
            p.qbf[(size_t)row * p.dimpad + j] = b;
            hh = fmaf(vb, vb, hh);
            dd = fmaf(v - vb, v - vb, dd);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            hh += __shfl_xor_sync(0xffffffffu, hh, o);
            dd += __shfl_xor_sync(0xffffffffu, dd, o);
        }
        if (lane == 0) { red[1][w] = hh; red[2][w] = dd; }
    } else if (p.qs8) {
        // int8 image q ~ s qq, s = max|q_i| / 127 (NaN if an element is not finite: every estimate of the query is then NaN
        // and kept as +inf); qa / qb below measure |s qq| and |q - s qq| as the BF16 copy's residues are measured
        float mx = 0.0f;
        bool bad = false;
        for (uint32_t j = tid; j < p.dim; j += PREP_THREADS) {
            const float v = row < p.Q ? qs[j] * inv : 0.0f;
            mx = fmaxf(mx, fabsf(v));
            bad |= (v - v) != 0.0f;
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        bad = __any_sync(0xffffffffu, bad);
        if (lane == 0) red[1][w] = bad ? NAN : mx;
        __syncthreads();
        for (int i = 0; i < NW; ++i) { const float r = red[1][i]; mx = (mx != mx || r != r) ? NAN : fmaxf(mx, r); }  // NaN sticks
        __syncthreads();  // red[1] is reused below
        const float s = mx / 127.0f, sinv = mx > 0.0f ? 127.0f / mx : 0.0f;  // (mx NaN: s NaN, sinv 0)
        for (uint32_t j = tid; j < p.dimpad; j += PREP_THREADS) {
            const float v = (row < p.Q && j < p.dim) ? qs[j] * inv : 0.0f;
            const int iq = max(-127, min(127, __float2int_rn(v * sinv)));
            p.qs8[(size_t)row * p.dimpad + j] = (int8_t)iq;
            const float vb = s * (float)iq, e = fmaf(-s, (float)iq, v);
            hh = fmaf(vb, vb, hh);
            dd = fmaf(e, e, dd);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            hh += __shfl_xor_sync(0xffffffffu, hh, o);
            dd += __shfl_xor_sync(0xffffffffu, dd, o);
        }
        if (lane == 0) { red[1][w] = hh; red[2][w] = dd; }
        if (tid == 0) p.qscale[row] = s;
    }
    __syncthreads();
    if (tid == 0) {
        if (p.qnorm) p.qnorm[row] = qn;
        if (p.qbf || p.qs8) {
            hh = dd = 0.0f;
            for (int i = 0; i < NW; ++i) { hh += red[1][i]; dd += red[2][i]; }
            p.qa[row] = sqrtf(hh) * 1.0001f;
            p.qb[row] = (sqrtf(dd) + p.acc_c * qn) * 1.0001f;
        }
    }
    // ---- sampled initial threshold
    if (p.sample == 0 || row >= p.Q) return;
    const uint32_t S = p.sample;  // power of two
    auto sample_row = [&](uint32_t i) -> uint64_t { return p.n >= S ? (uint64_t)i * p.n / S : i; };
    auto lower_key = [&](float sc, float xx) -> uint64_t {
        // lower bound of the real-valued score: the fp32 summation allowance the filters use (acc_c |x||q|)
        const float lo = sc - (p.metric == NK_METRIC_COSINE ? p.acc_c : p.metric == NK_METRIC_DOT ? p.acc_c * sqrtf(xx * t) : p.acc_c * -sc);
        return (lo == lo && lo > -INFINITY && lo < INFINITY) ? (uint64_t)ord_bits(lo) : 0ull;
    };
    auto admissible = [&](uint64_t r) -> bool {
        return r < p.n && (!p.mask || ((__ldg(p.mask + (r >> 5)) >> (r & 31)) & 1u)) && (!TAGS || tag_admits(__ldg(p.row_tags + r), p.qfilter + row)) &&
               (!WINDOW || window_admits(__ldg(p.row_values + r), p.qwindow + row));
    };
    if (p.dtype == NK_DTYPE_F32 && p.metric != NK_METRIC_EUCLIDEAN) {
        // two rows per warp at a time: both rows' 128-bit loads are in flight together (the scoring is latency-bound:
        // one 4 KB row per warp per round trip)
        const float4 *q4 = reinterpret_cast<const float4 *>(qs);
        for (uint32_t i = 2 * w; i < S; i += 2 * NW) {
            const uint64_t r0 = sample_row(i), r1 = sample_row(i + 1);
            const bool ok0 = admissible(r0), ok1 = i + 1 < S && admissible(r1);
            const float4 *x0 = reinterpret_cast<const float4 *>(static_cast<const float *>(p.rows) + (ok0 ? r0 : 0) * p.dim);
            const float4 *x1 = reinterpret_cast<const float4 *>(static_cast<const float *>(p.rows) + (ok1 ? r1 : 0) * p.dim);
            float d0 = 0.f, d1 = 0.f, n0 = 0.f, n1 = 0.f;
#pragma unroll 4
            for (uint32_t j = lane; j < p.dim / 4; j += 32) {
                const float4 a = __ldg(x0 + j), b = __ldg(x1 + j), u = q4[j];
                d0 = fmaf(a.x, u.x, d0); n0 = fmaf(a.x, a.x, n0); d0 = fmaf(a.y, u.y, d0); n0 = fmaf(a.y, a.y, n0);
                d0 = fmaf(a.z, u.z, d0); n0 = fmaf(a.z, a.z, n0); d0 = fmaf(a.w, u.w, d0); n0 = fmaf(a.w, a.w, n0);
                d1 = fmaf(b.x, u.x, d1); n1 = fmaf(b.x, b.x, n1); d1 = fmaf(b.y, u.y, d1); n1 = fmaf(b.y, b.y, n1);
                d1 = fmaf(b.z, u.z, d1); n1 = fmaf(b.z, b.z, n1); d1 = fmaf(b.w, u.w, d1); n1 = fmaf(b.w, b.w, n1);
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) {
                d0 += __shfl_xor_sync(0xffffffffu, d0, o); n0 += __shfl_xor_sync(0xffffffffu, n0, o);
                d1 += __shfl_xor_sync(0xffffffffu, d1, o); n1 += __shfl_xor_sync(0xffffffffu, n1, o);
            }
            if (lane == 0) {
                float s0 = d0, s1 = d1;
                if (p.metric == NK_METRIC_COSINE) {
                    const float e0 = sqrtf(n0 * t), e1 = sqrtf(n1 * t);
                    s0 = e0 > 0.0f ? d0 / e0 : 0.0f;
                    s1 = e1 > 0.0f ? d1 / e1 : 0.0f;
                }
                skeys[i] = ok0 ? lower_key(s0, n0) : 0ull;
                if (i + 1 < S) skeys[i + 1] = ok1 ? lower_key(s1, n1) : 0ull;
            }
        }
    } else {
        for (uint32_t i = w; i < S; i += NW) {
            uint64_t key = 0ull;
            const uint64_t r = sample_row(i);
            if (admissible(r)) {
                float xx;
                const float sc = warp_exact_score(p.rows, p.dtype, (size_t)r, p.dim, qs, t, p.metric, lane, &xx);
                key = lower_key(sc, xx);
            }
            if (lane == 0) skeys[i] = key;
        }
    }
    __syncthreads();
    // k-th largest of the S lower bounds by counting ranks (S <= 2048: one barrier instead of a bitonic network)
    if (p.k > S) return;
    for (uint32_t i = tid; i < S; i += PREP_THREADS) {
        const uint64_t mine = skeys[i];
        if (!mine) continue;
        uint32_t greater = 0, equal_before = 0;
        for (uint32_t j = 0; j < S; ++j) {
            const uint64_t o = skeys[j];
            greater += o > mine ? 1u : 0u;
            equal_before += (o == mine && j < i) ? 1u : 0u;
        }
        if (greater + equal_before == p.k - 1) {  // exactly one entry holds rank k-1 (ties ordered by position)
            const float tau0 = fmaxf(ord_to_float((uint32_t)mine), p.min_score);
            if (tau0 > -INFINITY) p.state[row] = ord_bits(tau0);
        }
    }
}

// Score estimate of one accumulator fragment row of the TF32 scan (keep_fragment_rows):
//   cosine     acc / |x|  (queries pre-normalised)       filter bound c
//   dot        acc                                        filter bound c |x| |q|
//   euclidean  -(|x|^2 + |q|^2 - 2 acc)   (filter only)   filter bound 2c |x| |q|
// filter mode buffers the UPPER bound score + bound.
template <bool FILTER> struct Tf32Est {
    float mul, bnd, x2;
    const float *qn;
    bool euclid;
    struct Col { float qn; };  // the query's input, read once per column for all of a thread's rows
    __device__ __forceinline__ Col col(uint32_t qi) const { return {FILTER ? qn[qi] : 0.0f}; }
    __device__ __forceinline__ float upper(float v, const Col &c) const {
        float sc = v * mul;
        if (FILTER) {
            const float q = c.qn;
            if (euclid) sc -= tc::EUC_KEEP * fmaf(q, q, x2);
            sc = fmaf(bnd, q, sc);
        }
        return sc;
    }
    __device__ __forceinline__ float bound(uint32_t qi) const { return bnd * qn[qi]; }
};

// M: the scan mode (kernels.cuh).  The row-filter modes stage the launch's query tags (REVERSE_RWINDOW: and value keys) in
// shared memory past Shared.
template <int NT, int QT, ScanMode M>
__global__ void __launch_bounds__(tc::THREADS, 1)
knn_scan_tc_kernel(const __grid_constant__ CUtensorMap map_rows, const __grid_constant__ CUtensorMap map_qhi,
                   const __grid_constant__ CUtensorMap map_qlo, tc::Params p) {
    using namespace tc;
    using C = Cfg<NT, QT>;
    constexpr bool FILTER = NT == 1;
    constexpr int B_BYTES = C::B_BYTES;
    pdl_trigger();
    pdl_wait();
    if (p.only_if && *p.only_if == 0) return;  // exact fallback not needed (uniform over the grid)

    extern __shared__ unsigned char smem_dyn[];
    // 128-byte-swizzled tiles need 1024-byte alignment: align by hand (the launch reserves the slack).
    unsigned char *smem_raw = smem_dyn + ((1024u - (ptx::smem_u32(smem_dyn) & 1023u)) & 1023u);
    // layout: [ASTAGES x A 32K] [BSTAGES x (Bhi [| Blo])] [xl 2 x 16K (exact mode)] [Shared]
    unsigned char *a_base = smem_raw;
    unsigned char *b_base = smem_raw + (size_t)ASTAGES * A_BYTES;
    Shared &sh = *reinterpret_cast<Shared *>(smem_raw + (size_t)C::RING_BYTES);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t num_tiles = (p.n + ROWS - 1) / ROWS;
    const QueryGroup<QT> qg(p);
    const uint32_t sub = qg.sub, sgrid = qg.sgrid, q0 = qg.q0, qpad_off = qg.qpad_off, nq = qg.nq;
    const bool prof = (p.debug & 64) && blockIdx.x == 0;
    long long acc_a = 0, acc_b = 0;
    const long long t_start = prof ? clock64() : 0;

    if (warp == 0 && lane == 0) {
        ptx::prefetch_tensormap(&map_rows);
        ptx::prefetch_tensormap(&map_qhi);
        if (NT == 3) ptx::prefetch_tensormap(&map_qlo);
        sh.maxxx = 0u;
        sh.ring.init(C::BSTAGES);
    }
    if (tid < QT) {
        sh.tau[tid] = FILTER ? start_tau(p, q0, tid, nq) : p.min_score;
        sh.cnt[tid] = 0;
        sh.qn[tid] = (FILTER && p.qnorm) ? p.qnorm[qpad_off + tid] : 1.0f;
    }
    // row-filter modes only: the query tags [QT], then (REVERSE_RWINDOW) the query value keys [QT]
    uint64_t *qtag = reinterpret_cast<uint64_t *>(smem_raw + (size_t)C::RING_BYTES + sizeof(Shared));
    if (mode_row_filter(M) && tid < QT) qtag[tid] = (uint32_t)tid < nq ? p.qtags[q0 + tid] : 0ull;
    if constexpr (mode_row_window(M))
        if (tid < QT) qtag[QT + tid] = (uint32_t)tid < nq ? p.qvalues[q0 + tid] : 0ull;
    __syncthreads();
    const bool flood = !(FILTER && p.presampled);  // first two tiles: every (row, query) pair is placed directly
    uint64_t *my_cand = p.cand + (size_t)blockIdx.x * QT * P;
    auto prune = [&](uint32_t qi, uint64_t *out, int out_len, int max_keep, float floor_tau, int *gcount) {
        const float margin2 = !FILTER ? 0.0f : filter_margin2(p.metric, p.margin_c, __uint_as_float(sh.maxxx), sh.qn[qi]);
        warp_prune<16>(my_cand + (size_t)qi * P, &sh.cnt[qi], &sh.tau[qi], p.k, lane, out, out_len, FILTER, margin2, max_keep, floor_tau,
                       gcount, p.flags + FLAG_OVERFLOW);
    };

    if (warp == 0) {
        // ===================================== TMA producer: corpus slabs ========================
        acc_a = tma_producer<ASTAGES>(sh.ring.aempty, sub, num_tiles, sgrid, 1, p.nslab, prof, [&](uint32_t s, uint32_t tile, uint32_t, uint32_t j) {
            ptx::mbar_arrive_expect_tx(&sh.ring.afull[s], A_BYTES);
            ptx::tma_load_2d(&map_rows, &sh.ring.afull[s], a_base + (size_t)s * A_BYTES, (int32_t)(j * BK), (int32_t)(tile * ROWS), qg.a_policy);
        });
        if (prof && lane == 0) { g_tc_prof[0] = acc_a; g_tc_prof[1] = clock64() - t_start; }
    } else if (warp == 3) {
        // ===================================== TMA producer: query slabs (L2-resident) ===========
        acc_a = tma_producer<C::BSTAGES>(sh.ring.bempty, sub, num_tiles, sgrid, 1, p.nslab, prof, [&](uint32_t s, uint32_t, uint32_t, uint32_t j) {
            unsigned char *st = b_base + (size_t)s * C::BST_BYTES;
            ptx::mbar_arrive_expect_tx(&sh.ring.bfull[s], C::BST_BYTES);
            ptx::tma_load_2d(&map_qhi, &sh.ring.bfull[s], st, (int32_t)(j * BK), (int32_t)qpad_off, ptx::CACHE_EVICT_LAST);
            if (NT == 3) ptx::tma_load_2d(&map_qlo, &sh.ring.bfull[s], st + B_BYTES, (int32_t)(j * BK), (int32_t)qpad_off, ptx::CACHE_EVICT_LAST);
        });
        if (prof && lane == 0) { g_tc_prof[2] = acc_a; }
    } else if (warp >= EPI_WARP0) {
        // ===================================== consumers: split + MMA + epilogue ===================
        // warpgroup m owns rows [128 m, 128 m + 128) of the tile.  Split step: thread t rounds row 128 m + t of the slab.
        // MMA / epilogue: two m64 halves h; thread = 4 rows x QT/4 columns of the accumulator fragments: rows
        // rbase + 64 h + 8 r, columns cbase + 8 (j / 2) + j % 2.
        const uint32_t ewarp = warp - EPI_WARP0, m = ewarp >> 2, wq = ewarp & 3;
        const uint32_t srow = m * 128 + ((uint32_t)tid & 127u);  // split row
        const uint32_t rbase = m * 128 + wq * 16 + ((uint32_t)lane >> 2), cbase = 2u * ((uint32_t)lane & 3u);
        unsigned char *xl_base = smem_raw + (size_t)ASTAGES * A_BYTES + (size_t)C::BSTAGES * C::BST_BYTES + (size_t)m * (A_BYTES / 2);
        const int prune_at = P - ROWS;
        const bool cosine = p.metric == NK_METRIC_COSINE, euclid = p.metric == NK_METRIC_EUCLIDEAN;
        const float bfac = p.margin_c * (euclid ? 2.0f : 1.0f);  // bound on -dist^2 = -(|x|^2+|q|^2-2x.q) is 2c|x||q|
        float acc[2][QT / 2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < QT / 2; ++i) acc[h][i] = 0.0f;
        uint32_t g = 0, it = 0;
        for (uint32_t tile = sub; tile < num_tiles; tile += sgrid, ++it) {
            float xe = 0.0f, xo = 0.0f;  // |x|^2 of the split row: partial sums over even / odd elements
            for (uint32_t j = 0; j < p.nslab; ++j, ++g) {
                const uint32_t s = g % ASTAGES, sb = g % C::BSTAGES;
                { TC_PROF_BEGIN(); ptx::mbar_wait(&sh.ring.afull[s], (g / ASTAGES) & 1); TC_PROF_END(a); }
                if (NT == 3 && j > 0) group_sync(2 + m, 128);  // the previous slab's MMAs no longer read the xl tile
                // split: xh = rn_tf32(x) in place (the MMA's A operand), xl = x - xh (exact) into this warpgroup's xl tile,
                // |x|^2 on the side
                unsigned char *rowp = a_base + (size_t)s * A_BYTES + (size_t)srow * 128;
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    // 128B swizzle: logical 16-byte chunk c of row r sits at chunk c ^ (r & 7)
                    const uint32_t off = (uint32_t)(c ^ (int)(srow & 7)) << 4;
                    const uint4 v = *reinterpret_cast<const uint4 *>(rowp + off);
                    const uint32_t e[4] = {v.x, v.y, v.z, v.w};
                    uint32_t hi[4], lo[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const float x = __uint_as_float(e[u]);
                        if (u & 1) xo = fmaf(x, x, xo); else xe = fmaf(x, x, xe);
                        hi[u] = ptx::tf32_round_bits(e[u]);
                        lo[u] = __float_as_uint(x - __uint_as_float(hi[u]));
                    }
                    *reinterpret_cast<uint4 *>(rowp + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                    if (NT == 3) *reinterpret_cast<uint4 *>(xl_base + (size_t)(srow - m * 128) * 128 + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
                }
                if (j + 1 == p.nslab) sh.xx[srow] = xe + xo;
                ptx::fence_proxy_async_smem();
                group_sync(2 + m, 128);  // every row of this warpgroup's half of the slab is rounded
                { TC_PROF_BEGIN(); ptx::mbar_wait(&sh.ring.bfull[sb], (g / C::BSTAGES) & 1); TC_PROF_END(b); }
                const uint32_t bhi = ptx::smem_u32(b_base + (size_t)sb * C::BST_BYTES);
                const uint64_t dhi = ptx::make_smem_desc_sw128(bhi), dlo = ptx::make_smem_desc_sw128(bhi + B_BYTES);
                const uint32_t ahi = ptx::smem_u32(a_base + (size_t)s * A_BYTES + (size_t)m * (A_BYTES / 2)), alo = ptx::smem_u32(xl_base);
                ptx::wgmma_fence();
                // K advance per MMA = 8 floats = 32 B = 2 descriptor units; M-half h = 64 rows = 8 KB
#pragma unroll
                for (uint32_t kk = 0; kk < BK / 8; ++kk) {
#pragma unroll
                    for (uint32_t h = 0; h < 2; ++h) {
                        const uint64_t dah = ptx::make_smem_desc_sw128(ahi + h * (A_BYTES / 4)) + kk * 2;
                        if (NT == 3) {  // smallest terms first
                            const uint64_t dal = ptx::make_smem_desc_sw128(alo + h * (A_BYTES / 4)) + kk * 2;
                            ptx::wgmma_tf32<QT>(acc[h], dal, dhi + kk * 2, (j | kk) != 0);
                            ptx::wgmma_tf32<QT>(acc[h], dah, dlo + kk * 2, 1);
                            ptx::wgmma_tf32<QT>(acc[h], dah, dhi + kk * 2, 1);
                        } else {
                            ptx::wgmma_tf32<QT>(acc[h], dah, dhi + kk * 2, (j | kk) != 0);
                        }
                    }
                }
                ptx::wgmma_commit();
                ptx::wgmma_wait_all();
                ptx::fence_acc(acc[0]);
                ptx::fence_acc(acc[1]);
                __syncwarp();
                if (lane == 0) { ptx::mbar_arrive(&sh.ring.aempty[s]); ptx::mbar_arrive(&sh.ring.bempty[sb]); }
            }
            if (flood && it < 2 && ewarp == 0 && lane == 0)
                for (uint32_t qi = 0; qi < nq; ++qi) sh.cnt[qi] = (int)((it + 1) * ROWS);
#pragma unroll
            for (uint32_t ri = 0; ri < 4; ++ri) {
                const uint32_t rt = rbase + 64 * (ri >> 1) + 8 * (ri & 1);  // row within the tile
                const uint32_t row = tile * ROWS + rt;
                const bool alive = row_alive(p, row);
                Tf32Est<FILTER> est[1];
                Tf32Est<FILTER> &e = est[0];
                e.x2 = sh.xx[rt];
                e.qn = sh.qn;
                e.euclid = euclid;
                const float xn = sqrtf(e.x2);
                e.mul = 1.0f;
                e.bnd = 0.0f;
                if (cosine) e.mul = e.x2 > 0.0f ? 1.0f / xn : 0.0f;
                if (FILTER) {
                    e.bnd = cosine ? p.margin_c : bfac * xn;
                    if (!cosine && alive && e.x2 < INFINITY && (lane & 3) == 0) atomicMax(&sh.maxxx, __float_as_uint(e.x2));  // NaN / Inf rows: kept, judged exactly
                    if (euclid) e.mul = 2.0f;
                }
                const float rthr[1] = {mode_row_thr(M) && row < p.n ? __ldg(p.row_thr + row) : -INFINITY};
                keep_fragment_rows<QT, P, FILTER, M>(p, est, acc, ri, alive ? 1u : 0u, tile * ROWS, rbase, flood, it, cbase, q0, nq, sh.tau, sh.qn,
                                                     sh.cnt, my_cand, rthr, qtag);
            }
            // prune any buffer that could overflow during the next tile; the 8 consumer warps prune different
            // queries concurrently with a register-resident warp selection
            group_sync(EPI_BAR, EPI_THREADS);  // every push of this tile is visible
            if constexpr (mode_range(M)) flush_tile<P>(p, q0, nq, ewarp, lane, my_cand, sh.cnt);
            else prune_tile<FILTER>(p, q0, nq, ewarp, lane, sh.cnt, sh.tau, prune_at, prune_at, flood && it == 0, prune);
            group_sync(EPI_BAR, EPI_THREADS);
            if (FILTER && !mode_range(M)) adopt_shared_tau(p, q0, nq, tid - EPI_WARP0 * 32, sh.tau);
        }
    }

    // ---- emit this CTA's list per query: everything inside the margin (filter) or the best k into fixed slots (exact).
    // Every role has finished its tile loop here, so all 12 warps share the final prunes.
    __syncthreads();
    for (uint32_t qi = warp; qi < nq; qi += THREADS / 32) {
        if (mode_range(M))
            flush_query(p, q0, qi, lane, my_cand + (size_t)qi * P, sh.cnt);
        else if (FILTER)
            emit_query(p, q0, qi, lane, my_cand + (size_t)qi * P, sh.cnt, sh.tau, prune);
        else
            prune(qi, p.partial + ((size_t)(q0 + qi) * gridDim.x + blockIdx.x) * p.k_emit, (int)p.k_emit, (int)p.k_emit, p.min_score, nullptr);
    }
    if (FILTER && p.metric != NK_METRIC_COSINE && tid == 0) atomicMax(reinterpret_cast<unsigned int *>(p.flags + FLAG_MAXXX), sh.maxxx);

    if (prof && tid == EPI_WARP0 * 32) { g_tc_prof[4] = acc_a; g_tc_prof[5] = acc_b; g_tc_prof[6] = clock64() - t_start; g_tc_prof[7] = (long long)num_tiles; }
}

// ---------------------------------------------------------------------------------------------------
// Filter-mode finish (one CTA per query): the query's shared list holds every row whose upper bound reached the
// cross-CTA threshold (k plus a few dozen).  Radix-select the k-th largest bound; everything with bound >= (k-th bound -
// 2*Bmax) may belong to the true top-k: those rows are re-scored EXACTLY in fp32 with the same arithmetic as the
// CUDA-core scan (dot / sqrt(|x|^2 |q|^2) etc.), sorted by (score desc, row asc), and the best k written out — as keys
// and, when the caller wants them, already decoded (index, score), so no separate decode launch follows.  Survivor
// sets of any size are handled in rounds of FINISH_WIN list entries (near-tie data: thousands of rows inside the margin)
// with the running best k carried from round to round.
// The LAST CTA to finish does the stage bookkeeping that used to be two more launches: it turns the stage's overflow
// flag into the retry marker and, if a retry is due, wipes the shared thresholds and list fills.
// ---------------------------------------------------------------------------------------------------
constexpr int FINISH_THREADS = 1024;  // one CTA per query has an SM to itself: 32 warps for the list passes and the re-scoring
constexpr int FINISH_CAP = 4096;
constexpr int FINISH_WIN = FINISH_CAP - 256;  // list entries per round; the carried best k (<= 192) fits in the rest
constexpr int FINISH_HI = 16384;              // score words of the list cached in shared memory (longer lists: read from L2)
constexpr int FINISH_HI_SMALL = 8192;         // the same for query rows too long to fit beside FINISH_HI (make_filter_plan)
constexpr uint32_t ORD_POS_INF = 0xFF800000u;  // ord_bits(+inf): the bound of a row whose score is undecidable (NaN)
struct FinishParams {
    const void *rows;        // corpus shard (fp32, or fp16 for the fp16 tensor path)
    int dtype;
    uint32_t dim;
    uint64_t row_base;
    const float *queries;    // raw fp32 queries [Q x dim]
    const uint64_t *lists;   // [Q][list_cap] shared append lists (keys carry upper bounds)
    const int *gcount;       // [Q]
    uint32_t list_cap, k;
    int metric;
    float margin_c;          // TF32 passes: c in |s_hat - s| <= c |x||q|
    uint32_t q_big;          // queries [0, q_big) went through the BF16 / FP16 kernel: bound factors qa / qb / qn below
    const float *qa, *qb, *qn;
    int *flags;
    const int *only_if;      // retry stage: run only if *only_if != 0
    uint64_t *out;           // [Q][k] keys
    uint32_t *out_idx;       // optional fused decode (nullable): [Q][k]
    float *out_score;
    float min_score;         // caller's score floor: exact scores below it are dropped
    int mark_retry;          // first stage of a two-stage filter: overflow -> retry marker + state wipe
    uint32_t *state;         // gtau[QA] + gcount[QA]
    uint32_t state_words;
    int debug;               // NK_TC_DEBUG & 64: per-CTA phase stamps (g_fin_prof)
};

// Debug timeline of the finish kernel (NK_TC_DEBUG & 64), printed after the first-stage finish launch:
//   [0] entry  [1] list cached  [2] k-th bound selected  [3] survivors gathered  [4] re-scored  [5] ranked  [6] exit  [7] list length
__device__ unsigned long long g_fin_prof[256][8];

// HI: score words of the list cached in shared memory (FINISH_HI, or FINISH_HI_SMALL where the query row needs the room)
template <int HI>
__global__ void __launch_bounds__(FINISH_THREADS) filter_finish_kernel(FinishParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint32_t *shi = reinterpret_cast<uint32_t *>(smem_raw);                            // HI score words of the list
    uint64_t *sb = reinterpret_cast<uint64_t *>(smem_raw + HI * 4);                    // FINISH_CAP bound keys
    uint64_t *se = reinterpret_cast<uint64_t *>(smem_raw + HI * 4 + FINISH_CAP * 8);   // FINISH_CAP exact keys
    float *qs = reinterpret_cast<float *>(smem_raw + HI * 4 + FINISH_CAP * 16);        // query
    __shared__ float s_qq;
    __shared__ int s_count, s_last;
    pdl_trigger();
    pdl_wait();  // launched as a programmatic dependent of the scan (common.cuh)
    if (p.only_if && *p.only_if == 0) return;
    const uint32_t q = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool prof = p.debug && q < 256 && tid == 0;
    if (prof) g_fin_prof[q][0] = tc::globaltimer_ns();
    for (uint32_t j = tid; j < p.dim; j += FINISH_THREADS) qs[j] = p.queries[(size_t)q * p.dim + j];
    int n = p.gcount[q];
    if (tid == 0) atomicMax(p.flags + FLAG_LONGEST, n);  // diagnostics: longest shared list of this search
    if (n > (int)p.list_cap) n = (int)p.list_cap;
    const uint64_t *list = p.lists + (size_t)q * p.list_cap;
    // ONE pass over the list (L2): the score words go to shared memory — every selection pass below reads them from there
    // (the list was read five times from L2, each time a chain of dependent ~1 us loads: that, not the arithmetic, was the
    // finish step's cost).  Four independent loads per thread per iteration.
    const bool cached = n <= HI;
    uint32_t umax = 0u, umin = 0xffffffffu;
    int ninf = 0;
    for (int i0 = tid; i0 < n; i0 += 4 * FINISH_THREADS) {
        uint32_t h[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int i = i0 + u * FINISH_THREADS;
            h[u] = i < n ? (uint32_t)(__ldcg(list + i) >> 32) : 0u;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int i = i0 + u * FINISH_THREADS;
            if (i < n) {
                if (cached) shi[i] = h[u];
                umax = max(umax, h[u]);
                umin = min(umin, h[u]);
                ninf += h[u] >= ORD_POS_INF ? 1 : 0;
            }
        }
    }
    auto hi_at = [&](int i) -> uint32_t { return cached ? shi[i] : (uint32_t)(__ldcg(list + i) >> 32); };
    __syncthreads();
    if (prof) { g_fin_prof[q][1] = tc::globaltimer_ns(); g_fin_prof[q][7] = (unsigned long long)n; }
    if (warp == 0) {
        float a = 0.0f;
        for (uint32_t j = lane; j < p.dim; j += 32) a = fmaf(qs[j], qs[j], a);
#pragma unroll
        for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) s_qq = a;
    }
    // k-th largest bound by radix select over the score bits that actually vary (8 bits per pass, smem histogram), then
    // everything inside the margin below it is gathered for exact re-scoring.
    __shared__ int hist[256];
    __shared__ uint32_t s_prefix, s_red[3][FINISH_THREADS / 32];
    __shared__ int s_krem;
    // Rows with an undecidable score (NaN -> bound +inf) are always kept but say nothing about the k-th best score: the
    // threshold comes from the k-th largest FINITE bound = the (k + n_inf)-th largest overall.
    umax = __reduce_max_sync(0xffffffffu, umax);
    umin = __reduce_min_sync(0xffffffffu, umin);
    ninf = __reduce_add_sync(0xffffffffu, ninf);
    if (lane == 0) { s_red[0][warp] = umax; s_red[1][warp] = umin; s_red[2][warp] = (uint32_t)ninf; }
    if (tid == 0) s_count = 0;
    __syncthreads();
    const float maxxx = __uint_as_float((unsigned int)p.flags[FLAG_MAXXX]);
    const float margin2 = q < p.q_big ? bf16_margin2(p.metric, __uint_as_float((unsigned int)p.flags[FLAG_MAX_RA]),
                                                     __uint_as_float((unsigned int)p.flags[FLAG_MAX_RB]), maxxx, p.qa[q], p.qb[q], p.qn[q])
                                      : filter_margin2(p.metric, p.margin_c, maxxx, sqrtf(s_qq));
    ninf = 0;
#pragma unroll
    for (int w = 0; w < FINISH_THREADS / 32; ++w) { umax = max(umax, s_red[0][w]); umin = min(umin, s_red[1][w]); ninf += (int)s_red[2][w]; }
    const int k_eff = (int)p.k + ninf;
    if (tid == 0) s_krem = k_eff;
    uint64_t thr_key = 1ull;  // fewer than k decidable entries: keep them all
    if (n >= k_eff) {
        int rem = 32 - __clz(umax ^ umin);  // low bits in which the bounds differ (0: all equal)
        if (tid == 0) s_prefix = rem >= 32 ? 0u : (umax >> rem) << rem;
        __syncthreads();
        // The select stops with <= 10 low bits unresolved: the prefix (low bits zero) is then a LOWER bound of the k-th largest
        // bound, at most 2^10 ulps (~1e-4 relative) below it — far inside the filter margin subtracted next, so at most a
        // stray extra survivor is re-scored, and two of the four histogram passes (3 barriers of 1024 threads each) are gone.
        while (rem > 10) {
            const int w = rem < 8 ? rem : 8, shift = rem - w;
            if (tid < 256) hist[tid] = 0;
            __syncthreads();
            const uint32_t prefix = s_prefix;
            for (int i = tid; i < n; i += FINISH_THREADS) {
                const uint32_t hi = hi_at(i);
                if (rem >= 32 || (hi >> rem) == (prefix >> rem)) atomicAdd(&hist[(hi >> shift) & ((1u << w) - 1u)], 1);
            }
            __syncthreads();
            if (warp == 0) {  // digit holding the krem-th largest: lane l owns the 8 digits below nb - 8l, descending
                const int krem = s_krem, nb = 1 << w;
                int loc[8], sum = 0;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int dgt = nb - 1 - (lane * 8 + j);
                    loc[j] = dgt >= 0 ? hist[dgt] : 0;
                    sum += loc[j];
                }
                __syncwarp();  // every lane has read s_krem / hist before the owner lane rewrites s_krem below
                int incl = sum;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int t = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += t;
                }
                int c = incl - sum;
                if (c < krem && incl >= krem) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        if (c + loc[j] >= krem) {
                            s_prefix = prefix | ((uint32_t)(nb - 1 - (lane * 8 + j)) << shift);
                            s_krem = krem - c;
                            break;
                        }
                        c += loc[j];
                    }
                }
            }
            __syncthreads();
            rem = shift;
        }
        __syncthreads();
        const float thr = ord_to_float(s_prefix) - margin2;
        if (thr < INFINITY) {
            thr_key = (uint64_t)ord_bits(thr) << 32;
            if (thr_key == 0ull) thr_key = 1ull;
        } else if (tid == 0) {
            // k-th bound +inf / NaN (k or more NaN rows) or a non-finite margin: no threshold can be trusted -> keep every
            // listed row here and let the exact stage redo the search
            atomicOr(p.flags + FLAG_OVERFLOW, 8);
        }
    }
    // ---- how many rows are inside the margin?  Almost always a few dozen: ONE gather + re-score round.  Only adversarial
    // near-tie data (thousands of survivors) goes through the list in windows, the running best k carried over.
    const uint32_t thr_hi = (uint32_t)(thr_key >> 32);  // keys >= thr_key  <=>  score word >= thr_hi (thr_key's low word is 0 or 1)
    if (prof) g_fin_prof[q][2] = tc::globaltimer_ns();
    int mine = 0;
    for (int i = tid; i < n; i += FINISH_THREADS) mine += hi_at(i) >= thr_hi ? 1 : 0;
    mine = __reduce_add_sync(0xffffffffu, mine);
    if (lane == 0 && mine) atomicAdd(&s_count, mine);
    __syncthreads();
    const int survivors = s_count;
    const int win = survivors <= FINISH_WIN ? (n > 0 ? n : 1) : FINISH_WIN;  // whole list in one round when the survivors fit
    int carry = 0;
    for (int w0 = 0; w0 < n || w0 == 0; w0 += win) {
        __syncthreads();
        if (tid == 0) s_count = 0;
        __syncthreads();
        const int w1 = min(n, w0 + win);
        for (int i = w0 + tid; i < w1; i += FINISH_THREADS) {
            if (hi_at(i) >= thr_hi) {  // the full key is fetched only for survivors
                const uint64_t key = __ldcg(list + i);
                if (key >= thr_key) sb[atomicAdd(&s_count, 1)] = key;
            }
        }
        __syncthreads();
        if (prof && w0 == 0) g_fin_prof[q][3] = tc::globaltimer_ns();
        const int count = s_count;  // <= FINISH_WIN
        for (int i = warp; i < count; i += FINISH_THREADS / 32) {
            const uint32_t grow = key_row(sb[i]);
            const size_t local = (size_t)(grow - (uint32_t)p.row_base);
            const float sc = warp_exact_score(p.rows, p.dtype, local, p.dim, qs, s_qq, p.metric, lane);
            if (lane == 0) se[carry + i] = sc >= p.min_score ? make_key(sc, grow) : 0ull;
        }
        const int total = carry + count;
        __syncthreads();
        if (prof && w0 == 0) g_fin_prof[q][4] = tc::globaltimer_ns();
        if (total <= FINISH_THREADS) {
            // small sets (the common case): rank by counting — one barrier instead of a 15-45 stage bitonic network
            const uint64_t mykey = tid < total ? se[tid] : 0ull;
            int rank = 0;
            for (int j = 0; j < total; ++j) rank += se[j] > mykey ? 1 : 0;  // keys are unique (row in the low word) or 0
            __syncthreads();
            if (tid < total && mykey) se[rank] = mykey;
            // dropped (0) keys: fill the tail behind the live ones
            int live = __syncthreads_count(tid < total && mykey != 0ull);
            for (int i = live + tid; i < total; i += FINISH_THREADS) se[i] = 0ull;
            __syncthreads();
        } else {
            int P2 = 32;
            while (P2 < total) P2 <<= 1;
            for (int i = total + tid; i < P2; i += FINISH_THREADS) se[i] = 0ull;
            block_bitonic_sort_desc(se, P2);
        }
        carry = total < (int)p.k ? total : (int)p.k;
    }
    if (prof) g_fin_prof[q][5] = tc::globaltimer_ns();
    for (uint32_t i = tid; i < p.k; i += FINISH_THREADS) {
        const uint64_t key = (int)i < carry ? se[i] : 0ull;
        p.out[(size_t)q * p.k + i] = key;
        if (p.out_idx) {
            float sc = key_score(key);
            if (p.metric == NK_METRIC_EUCLIDEAN) sc = sqrtf(fmaxf(-sc, 0.0f));
            p.out_idx[(size_t)q * p.k + i] = key ? key_row(key) : 0xffffffffu;
            p.out_score[(size_t)q * p.k + i] = key ? sc : 0.0f;
        }
    }
    // ---- stage bookkeeping by the last CTA
    __syncthreads();
    if (tid == 0) {
        __threadfence();
        s_last = atomicAdd(p.flags + FLAG_FINISH_CTAS, 1) == (int)gridDim.x - 1;
    }
    __syncthreads();
    if (prof) g_fin_prof[q][6] = tc::globaltimer_ns();
    if (!s_last) return;
    __threadfence();
    const int ovf = atomicOr(p.flags + FLAG_OVERFLOW, 0);
    if (tid == 0 && ovf) atomicOr(p.flags + FLAG_OVF_BITS, ovf);
    if (p.mark_retry) {
        if (ovf)
            for (uint32_t i = tid; i < p.state_words; i += FINISH_THREADS) p.state[i] = 0u;
        if (tid == 0) {
            p.flags[FLAG_RETRY] = ovf != 0;
            p.flags[FLAG_OVERFLOW] = 0;
            if (ovf) atomicAdd(p.flags + FLAG_N_RETRY, 1);
        }
    } else if (tid == 0 && ovf) {
        atomicAdd(p.flags + FLAG_N_EXACT, 1);
    }
    if (tid == 0) p.flags[FLAG_FINISH_CTAS] = 0;
}

// ---------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn) return fn;
    void *p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || !p) {
        cudaGetLastError();
        return nullptr;
    }
    fn = reinterpret_cast<EncodeTiledFn>(p);
    return fn;
}

int tc_make_map(CUtensorMap *m, const void *base, uint64_t rows, uint32_t cols, uint32_t elem_bytes, uint32_t box_cols,
                uint32_t box_rows, uint64_t row_stride_bytes, int map_dtype) {
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) {
        set_error("cuTensorMapEncodeTiled entry point unavailable");
        return -1;
    }
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {(cuuint64_t)row_stride_bytes};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    const CUtensorMapDataType dt = elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                   : elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                   : map_dtype == NK_DTYPE_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    CUresult r = enc(m, dt, 2,
                     const_cast<void *>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%u", (int)r, (unsigned long long)rows, cols);
        return -1;
    }
    return 0;
}
// Tensor maps are cached per shard: cuTensorMapEncodeTiled (1-2 us of host time each, three per launch) runs only when
// the base pointer or the shape changed since the previous search.
const CUtensorMap *tc_cached_map(Workspace &ws, int slot, const void *base, uint64_t rows, uint32_t cols, uint32_t elem_bytes,
                                 uint32_t box_cols, uint32_t box_rows, uint64_t row_stride_bytes, int map_dtype) {
    static_assert(sizeof(CUtensorMap) == sizeof(ws.maps[0].bytes), "CUtensorMap is 128 bytes");
    Workspace::MapSlot &m = ws.maps[slot];
    const uint64_t key[6] = {reinterpret_cast<uint64_t>(base), rows, ((uint64_t)cols << 32) | elem_bytes,
                             ((uint64_t)box_cols << 32) | box_rows, row_stride_bytes, (uint64_t)map_dtype};
    if (!m.valid || memcmp(m.key, key, sizeof(key)) != 0) {
        if (tc_make_map(reinterpret_cast<CUtensorMap *>(m.bytes), base, rows, cols, elem_bytes, box_cols, box_rows, row_stride_bytes, map_dtype))
            return nullptr;
        memcpy(m.key, key, sizeof(key));
        m.valid = true;
    }
    return reinterpret_cast<const CUtensorMap *>(m.bytes);
}

// getenv once per variable (the search path used to call getenv per search)
int tc_env_int(const char *name, int dflt) {
    static std::mutex mu;
    static std::map<std::string, int> cache;
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find(name);
    if (it != cache.end()) return it->second;
    const char *e = getenv(name);
    const int v = e ? atoi(e) : dflt;
    cache[name] = v;
    return v;
}

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device) instead of once per launch
int tc_ensure_smem(const void *func, int device, size_t smem) {
    static std::mutex mu;
    static std::map<std::pair<const void *, int>, size_t> done;
    std::lock_guard<std::mutex> lk(mu);
    size_t &cur = done[{func, device}];
    if (cur >= smem && cur != 0) return 0;
    NK_CUDA_OK(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cur = smem;
    return 0;
}

// the prep kernel's dynamic shared memory: the query row (padded to float4) and the threshold sample's keys
static size_t prep_smem_bytes(uint32_t dim, uint32_t sample) { return (size_t)((dim + 3) & ~3u) * 4 + (size_t)sample * 8; }

size_t kernel_static_smem(const void *func) {
    static std::mutex mu;
    static std::map<const void *, size_t> known;
    std::lock_guard<std::mutex> lk(mu);
    auto it = known.find(func);
    if (it != known.end()) return it->second;
    cudaFuncAttributes fa{};
    if (cudaFuncGetAttributes(&fa, func) != cudaSuccess) {
        cudaGetLastError();
        return (size_t)1 << 40;  // unknown (not cached): nothing fits
    }
    return known[func] = fa.sharedSizeBytes + SMEM_RESERVED;
}
bool smem_fits(const DeviceInfo &di, const void *func, size_t dyn) { return dyn + kernel_static_smem(func) <= di.max_smem_optin; }
int ensure_smem(const DeviceInfo &di, const void *func, size_t dyn, const char *what, uint32_t dim) {
    if (!smem_fits(di, func, dyn)) {
        set_error("%s: dim=%u needs %zu B shared memory (> %zu)", what, dim, dyn + kernel_static_smem(func), di.max_smem_optin);
        return -1;
    }
    return dyn + kernel_static_smem(func) > 48 * 1024 ? tc_ensure_smem(func, di.device_id, dyn) : 0;
}

static bool tc_common_ok(const DeviceInfo &di, const ScanArgs &a) {
    if (di.cc < 90) return false;
    if (a.dtype != NK_DTYPE_F32) return false;                      // fp16 / bf16 corpus: 16-bit tensor pass or CUDA cores
    if (a.dim % 4 != 0 || a.dim < 32) return false;                 // TMA: 16-byte global stride
    if ((reinterpret_cast<uintptr_t>(a.rows) & 15) != 0) return false;
    if (a.n == 0 || a.k == 0) return false;
    return true;
}
// exact (3xTF32) mode: cosine / dot, k <= 255 (register-resident prune over a 512-slot buffer), d <= TENSOR_EXACT_MAX_DIM:
// its scores fall below fp64 by about 3e-9 d |x||q| (the dropped lo*lo products and the MMA's truncating fp32 adds),
// 1e-4 of a score of 0.4 |x||q| at d = 12288 (tests/test_gpu_dims.py); larger d take the CUDA-core scan
bool scan_tensor_supported(const DeviceInfo &di, const ScanArgs &a) {
    return tc_common_ok(di, a) && a.metric != NK_METRIC_EUCLIDEAN && a.k + tc::ROWS + 1 <= (uint32_t)tc::P &&
           a.dim <= TENSOR_EXACT_MAX_DIM &&
           smem_fits(di, reinterpret_cast<const void *>(filter_prep_kernel<false, false>), prep_smem_bytes(a.dim, 0));
}
// The finish launch of a filter search over rows of `dim` elements: the FINISH_HI window wherever its dynamic shared
// memory (cached score words, bound and exact keys, the query row) fits the device's opt-in limit beside the kernel's
// static shared memory, else the FINISH_HI_SMALL window (lists longer than the window are read from L2).  kern == nullptr:
// neither fits.  The planner (scan_tensor_filter_supported) and the launch (make_filter_plan) both ask here.
struct FinishLaunch {
    void (*kern)(FinishParams);
    size_t smem;
};
static size_t finish_dyn_smem(int hi, uint32_t dim) { return (size_t)hi * 4 + (size_t)FINISH_CAP * 16 + (size_t)dim * 4; }
static FinishLaunch finish_launch(const DeviceInfo &di, uint32_t dim) {
    if (smem_fits(di, reinterpret_cast<const void *>(filter_finish_kernel<FINISH_HI>), finish_dyn_smem(FINISH_HI, dim)))
        return {filter_finish_kernel<FINISH_HI>, finish_dyn_smem(FINISH_HI, dim)};
    if (smem_fits(di, reinterpret_cast<const void *>(filter_finish_kernel<FINISH_HI_SMALL>), finish_dyn_smem(FINISH_HI_SMALL, dim)))
        return {filter_finish_kernel<FINISH_HI_SMALL>, finish_dyn_smem(FINISH_HI_SMALL, dim)};
    return {nullptr, 0};
}

// filter mode (1xTF32 over fp32 rows, or the 16-bit pass over a shadow / a 16-bit corpus) + exact rescoring: all three
// metrics, k <= 192, d <= FILTER_MAX_DIM (the int8 image's exact integer accumulation, DESIGN §3.3) and a query row that
// fits the finish kernel's shared memory on this device
bool scan_tensor_filter_supported(const DeviceInfo &di, const ScanArgs &a) {
    if (a.k > 192 || a.dim > FILTER_MAX_DIM) return false;
    if (!(tc_common_ok(di, a) || shadow_pass_supported(di, a))) return false;
    return finish_launch(di, a.dim).kern != nullptr;
}

int tc_debug_flags() { return tc_env_int("NK_TC_DEBUG", 0); }

tc::Params pass_params(const ScanArgs &a, Workspace &ws, const tc::PassArgs &t) {
    tc::Params p{};
    p.n = a.n; p.dim = a.dim; p.row_base = a.row_base;
    p.q0 = t.q0; p.nq = t.nq; p.k = a.k; p.qpad_off = t.q0; p.qgroups = t.qgroups; p.list_cap = mode_range(a.mode) ? t.list_cap : t.grid * t.k_emit;
    p.metric = a.metric; p.k_emit = t.k_emit; p.qnorm = t.qnorm;
    p.cand = ws.cand; p.partial = ws.partial; p.flags = ws.flags; p.debug = tc_debug_flags(); p.mask = a.row_mask;
    p.gtau = reinterpret_cast<uint32_t *>(ws.keys2); p.gcount = reinterpret_cast<int *>(ws.keys2) + (t.Qpad + tc::QT_BIG);
    p.presampled = t.presampled; p.min_score = a.min_score;
    p.row_tags = a.row_tags; p.qfilter = a.qfilter; p.row_thr = a.row_thr; p.row_filter = a.row_filter; p.qtags = a.qtags;
    p.row_values = a.row_values; p.qwindow = a.qwindow; p.row_window = a.row_window; p.qvalues = a.qvalues;
    p.dump_est = t.dump_est; p.dump_bnd = t.dump_bnd; p.dump_ld = t.dump_ld;
    return p;
}

// Splits queries [q0, q_end) into scan launches: 128 query columns per MMA while more than 64 queries remain (twice the
// queries per corpus byte streamed), 64 for the tail.  4 query groups per launch while more than 384 queries remain and 2
// while more than 128 remain (at most max_groups, grid % G == 0): the G sibling CTAs share every corpus tile through L2.
// launch(qt, q0, nq, groups) returns nonzero on error.
template <class Launch>
static int plan_launches(uint32_t q0, uint32_t q_end, uint32_t grid, uint32_t max_groups, Launch launch) {
    while (q0 < q_end) {
        const uint32_t left = q_end - q0;
        uint32_t qt = 64, groups = 1, nq = left;
        if (left > 64) {
            if (left > 3 * 128 && max_groups >= 4 && grid % 4 == 0 && grid >= 8) groups = 4;
            else if (left > 128 && max_groups >= 2 && grid % 2 == 0 && grid >= 4) groups = 2;
            qt = 128;
            nq = left < 128u * groups ? left : 128u * groups;
        }
        if (launch(qt, q0, nq, groups)) return -1;
        q0 += nq;
    }
    return 0;
}

PrepParams prep_params(const ScanArgs &a, uint32_t Qpad, uint32_t dimpad) {
    PrepParams pp{};
    pp.q = a.queries; pp.Q = a.Q; pp.dim = a.dim; pp.dimpad = dimpad; pp.Qpad = Qpad;
    pp.normalise = a.metric == NK_METRIC_COSINE; pp.metric = a.metric;
    pp.rows = a.rows; pp.dtype = a.dtype; pp.n = a.n; pp.k = a.k; pp.mask = a.row_mask; pp.min_score = a.min_score;
    pp.row_tags = a.row_tags; pp.qfilter = a.qfilter; pp.row_values = a.row_values; pp.qwindow = a.qwindow;
    return pp;
}

int launch_prep(const DeviceInfo &di, ScanMode mode, const PrepParams &pp, cudaStream_t stream, uint64_t *launches) {
    const size_t smem = prep_smem_bytes(pp.dim, pp.sample);
    void (*kern)(PrepParams) = mode_window(mode) ? filter_prep_kernel<true, true>
                               : mode_tags(mode) ? filter_prep_kernel<true, false> : filter_prep_kernel<false, false>;
    if (ensure_smem(di, reinterpret_cast<const void *>(kern), smem, "query prep", pp.dim)) return -1;
    kern<<<pp.Qpad, PREP_THREADS, smem, stream>>>(pp);
    NK_CUDA_OK(cudaGetLastError());
    if (launches) ++*launches;
    return 0;
}

// One launch: queries [q0, q0+nq) against the whole shard, QT = 64 or 128 query columns per MMA.
struct TcPassArgs : tc::PassArgs {
    float margin_c;
    const float *qhi, *qlo;
    const int *only_if;
    bool count_main;
};
template <int NT, int QT, ScanMode M>
static int launch_pass_t(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, const TcPassArgs &t, uint64_t *launches) {
    using namespace tc;
    const CUtensorMap *map_rows = tc_cached_map(ws, 0, a.rows, a.n, a.dim, 4, (uint32_t)BK, ROWS, (uint64_t)a.dim * 4);
    // query rows past Qpad are zero-filled by TMA
    const CUtensorMap *map_qhi = tc_cached_map(ws, QT == 64 ? 1 : 2, t.qhi, t.Qpad, a.dim, 4, (uint32_t)BK, QT, (uint64_t)a.dim * 4);
    const CUtensorMap *map_qlo = NT == 3 ? tc_cached_map(ws, 3, t.qlo, t.Qpad, a.dim, 4, (uint32_t)BK, QT, (uint64_t)a.dim * 4) : map_qhi;
    if (!map_rows || !map_qhi || !map_qlo) return -1;
    const size_t smem = (size_t)Cfg<NT, QT>::RING_BYTES + sizeof(Shared) + (mode_row_filter(M) ? QT * sizeof(uint64_t) : 0) +
                        (mode_row_window(M) ? QT * sizeof(uint64_t) : 0) + 1024;
    if (smem > di.max_smem_optin) {
        set_error("tensor path needs %zu B shared memory (> %zu)", smem, di.max_smem_optin);
        return -1;
    }
    if (tc_ensure_smem(reinterpret_cast<const void *>(knn_scan_tc_kernel<NT, QT, M>), di.device_id, smem))
        return -1;
    Params p = pass_params(a, ws, t);
    p.nslab = (a.dim + BK - 1) / BK; p.margin_c = t.margin_c; p.only_if = t.only_if;
    // (asynchronous API: the early-exit retry / exact stages are programmatic dependents — their launch overlaps the kernel
    // before them.  Not for the host-synchronous API: measured 5-15 us slower per nk_search, the copy-out behind it waits longer)
    NK_CUDA_OK(launch_pdl(knn_scan_tc_kernel<NT, QT, M>, dim3(t.grid), dim3(THREADS), smem, a.stream, t.only_if != nullptr && !a.defer_tail, *map_rows, *map_qhi,
                          *map_qlo, p));
    if (launches) ++*launches;
    if (t.count_main && a.main_launches) ++*a.main_launches;
    return 0;
}
// One pass in the mode a.mode.  The exact 3xTF32 kernel serves the kNN modes only (the retry and exact stages of a filter
// search re-run its arguments); the dump mode exists at QT = 64 only.
template <int NT, int QT>
static int launch_pass(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, const TcPassArgs &t, uint64_t *launches) {
    return tc::with_scan_mode(a.mode, [&](auto mode) {
        constexpr ScanMode M = decltype(mode)::value;
        if constexpr ((NT == 1 || M == ScanMode::KNN || M == ScanMode::KNN_TAGS || M == ScanMode::KNN_WINDOW) && (QT == 64 || !mode_dump(M)))
            return launch_pass_t<NT, QT, M>(di, a, ws, t, launches);
        set_error("internal: no %s kernel for scan mode %d at %d query columns", NT == 3 ? "3xTF32" : "TF32 filter", (int)M, QT);
        return -1;
    });
}

static void fin_print_prof(cudaStream_t stream, uint32_t Q) {
    if (!(tc_debug_flags() & 64)) return;
    static unsigned long long h[256][8];
    cudaStreamSynchronize(stream);
    cudaMemcpyFromSymbol(h, g_fin_prof, sizeof(h));
    const uint32_t g = Q < 256 ? Q : 256;
    unsigned long long t0 = ~0ull, tmax = 0;
    for (uint32_t b = 0; b < g; ++b) { t0 = h[b][0] < t0 ? h[b][0] : t0; tmax = h[b][6] > tmax ? h[b][6] : tmax; }
    double a[8] = {0};
    for (uint32_t b = 0; b < g; ++b) {
        for (int i = 1; i < 7; ++i) a[i] += (double)(h[b][i] - h[b][i - 1]);
        a[0] += (double)(h[b][0] - t0);
        a[7] += (double)h[b][7];
    }
    fprintf(stderr, "[finish prof, %u CTAs] span %.1f us | entry +%.1f | list cached %.1f | k-th bound %.1f | gather %.1f | re-score %.1f | rank %.1f | write + count %.1f | "
            "list length %.0f\n", g, (tmax - t0) / 1e3, a[0] / g / 1e3, a[1] / g / 1e3, a[2] / g / 1e3, a[3] / g / 1e3, a[4] / g / 1e3, a[5] / g / 1e3, a[6] / g / 1e3, a[7] / g);
}

static void tc_print_prof(cudaStream_t stream, uint32_t num_tiles, uint32_t grid, uint32_t nslab) {
    if (!(tc_debug_flags() & 64)) return;
    long long h[32];
    cudaStreamSynchronize(stream);
    cudaMemcpyFromSymbol(h, g_tc_prof, sizeof(h));
    uint32_t slabs = ((num_tiles + grid - 1) / grid) * nslab;
    fprintf(stderr, "[tc prof CTA0, ~%u slabs] total %lld cyc (%.0f/slab)\n  tmaA wait aempty_s %lld (total %lld) | tmaB wait bempty %lld\n"
            "  consumer warpgroup 0: wait afull_s %lld, wait bfull %lld\n",
            slabs, h[6], (double)h[6] / slabs, h[0], h[1], h[2], h[4], h[5]);
}

// ---- the plan of one filter search: everything both the primary stage and the (possibly deferred) tail derive from
// (device, args).  Deterministic, so the host-driven retry of nk_search can rebuild it after the fact.
struct FilterPlan {
    uint32_t Qpad, QA, num_tiles, grid, k_emit, dimpad, sample;
    bool big;           // first stage = 16-bit / int8 pass over a.image
    bool s8;            // a.image is the int8 image
    bool stage2;        // the TF32 filter over the fp32 rows exists as the retry stage (fp32 shards with an image)
    bool can_exact_tc;  // exact stage = 3xTF32 kernel (else the CUDA-core scan)
    float acc_c, margin_tf32;
    float *qhi, *qlo, *qnorm, *qa, *qb, *qscale;
    void *qbf16;        // the queries in the image's element type: bf16 / fp16, or int8 (with qscale) for an int8 image
    uint32_t max_groups_shadow;
    FinishLaunch finish;
    // the fields every 16-bit / int8 pass of the plan shares; the caller sets the query range and the mode
    ShadowPassArgs shadow_pass() const {
        ShadowPassArgs sp{};
        sp.grid = grid; sp.k_emit = k_emit; sp.dimpad = dimpad; sp.Qpad = Qpad;
        sp.qbf16 = qbf16; sp.qnorm = qnorm; sp.qa = qa; sp.qb = qb; sp.qscale = qscale;
        return sp;
    }
};

static int make_filter_plan(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, FilterPlan *fp) {
    using namespace tc;
    FilterPlan &f = *fp;
    f.Qpad = (a.Q + 63) / 64 * 64;
    f.QA = f.Qpad + QT_BIG;  // padded per-query arrays
    f.num_tiles = (a.n + ROWS - 1) / ROWS;
    f.grid = (uint32_t)di.num_sms < f.num_tiles ? (uint32_t)di.num_sms : f.num_tiles;
    // per-CTA contribution: at most k + room for the rows inside the margin
    f.k_emit = next_pow2(a.k + a.k / 2 + 32);
    if (f.k_emit < 64) f.k_emit = 64;
    if (f.k_emit > (uint32_t)(P - ROWS)) f.k_emit = P - ROWS;
    // TF32: 2^-10 (rounding of both operands, unit roundoff 2^-11 each) + d * 2^-22 (fp32 accumulation, truncating
    // adders) + fp32 rounding of the norms.  The 16-bit kernel measures its rounding residues instead.
    f.acc_c = (float)a.dim * 2.384185791015625e-7f + 4e-6f;
    f.margin_tf32 = 9.765625e-4f + f.acc_c;
    f.big = shadow_pass_supported(di, a);
    f.s8 = a.image.kind == RowImage::S8;
    f.stage2 = f.big && a.dtype == NK_DTYPE_F32 && tc_common_ok(di, a);
    f.can_exact_tc = scan_tensor_supported(di, a);  // euclidean / 16-bit rows have no 3xTF32 twin: overflow -> CUDA-core scan
    // 16-bit margins are ~6x wider than TF32's and clustered corpora put hundreds of rows per CTA inside them: the 16-bit
    // kernel has 1024-slot buffers and emits up to 512 entries per (CTA, query) (the finish step re-scores in rounds).  The
    // int8 image's margins are ~3x the BF16 shadow's: a CTA's local top 100 of 300k uniform rows already has ~550 rows inside
    // them, so it emits up to the whole prunable buffer at every k.
    if (f.big) f.k_emit = a.k <= 160 && !f.s8 ? 512u : (uint32_t)(P_SHADOW - ROWS);
    f.dimpad = f.big ? a.image.dimpad : (a.dim + 63) / 64 * 64;
    const bool need_f32q = a.dtype == NK_DTYPE_F32;  // hi / lo arrays only serve passes over fp32 rows
    const size_t qaux_floats = (need_f32q ? (size_t)2 * f.Qpad * a.dim : 0) + (size_t)4 * f.QA;
    if (ws_reserve((void **)&ws.qaux, &ws.qaux_bytes, qaux_floats * 4 + (f.big ? (size_t)f.Qpad * f.dimpad * 2 : 0))) return -1;
    if (ws_reserve((void **)&ws.cand, &ws.cand_bytes, (size_t)f.grid * QT_MAX * (f.big ? P_SHADOW : P) * 8)) return -1;
    if (ws_reserve((void **)&ws.partial, &ws.partial_bytes, (size_t)a.Q * f.grid * f.k_emit * 8)) return -1;
    if (ws_reserve((void **)&ws.keys2, &ws.keys2_bytes, (size_t)f.QA * 8)) return -1;  // gtau[] + gcount[]
    f.qhi = need_f32q ? ws.qaux : nullptr;
    f.qlo = need_f32q ? ws.qaux + (size_t)f.Qpad * a.dim : nullptr;
    f.qnorm = ws.qaux + (need_f32q ? (size_t)2 * f.Qpad * a.dim : 0);
    f.qa = f.qnorm + f.QA;
    f.qb = f.qa + f.QA;
    f.qscale = f.s8 ? f.qb + f.QA : nullptr;
    f.qbf16 = ws.qaux + qaux_floats;
    // G query groups leave each CTA 1/G of the grid for its queries, i.e. G times the rows — and G times the rows inside
    // the BF16 margin — per (CTA, query) buffer: large k keeps fewer groups so that k + margin rows stay inside k_emit
    f.max_groups_shadow = a.k <= 128 ? 4u : a.k <= 160 ? 2u : 1u;
    // Sampled initial threshold: single-pass batches on shards with enough tiles per CTA for the flood tiles to matter.
    // (Large batches re-score the sample once per query — more L2 traffic than the flood tiles cost.)
    f.sample = 0;
    if (tc_env_int("NK_TAU_SAMPLE", 1) && a.Q <= 128 && a.n >= 4096) {
        f.sample = next_pow2(8 * a.k);  // k-th best of the sample = top k/S of the shard: ~8-12% of the rows pass at first
        if (f.sample < 128) f.sample = 128;
        if (f.sample > 2048) f.sample = 2048;
    }
    f.finish = finish_launch(di, a.dim);
    if (!f.finish.kern) {
        set_error("filter finish: dim=%u needs more shared memory than the device allows (%zu B)", a.dim, di.max_smem_optin);
        return -1;
    }
    if (tc_ensure_smem(reinterpret_cast<const void *>(f.finish.kern), di.device_id, f.finish.smem)) return -1;
    return 0;
}

// Exact 3xTF32 scan.  only_if != nullptr: every kernel early-exits unless *only_if != 0 (device-side fallback).
// prep: convert the queries here (stand-alone use); the filter path has already done it in its fused prep.
static int scan_tensor_exact(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, uint64_t *out_keys, uint64_t *launches,
                             const int *only_if, bool prep, bool count_main) {
    using namespace tc;
    const uint32_t Qpad = (a.Q + 63) / 64 * 64;
    const uint32_t num_tiles = (a.n + ROWS - 1) / ROWS;
    uint32_t grid = (uint32_t)di.num_sms;
    if (grid > num_tiles) grid = num_tiles;
    if (ws_reserve((void **)&ws.qaux, &ws.qaux_bytes, ((size_t)2 * Qpad * a.dim + Qpad + QT_MAX) * 4)) return -1;
    if (ws_reserve((void **)&ws.cand, &ws.cand_bytes, (size_t)grid * QT_MAX * P * 8)) return -1;
    if (ws_reserve((void **)&ws.partial, &ws.partial_bytes, (size_t)a.Q * grid * a.k * 8)) return -1;
    float *qhi = ws.qaux, *qlo = ws.qaux + (size_t)Qpad * a.dim;
    if (prep) {
        PrepParams pp = prep_params(a, Qpad, a.dim);
        pp.qhi = qhi; pp.qlo = qlo; pp.only_if = only_if;
        if (launch_prep(di, a.mode, pp, a.stream, launches)) return -1;
    }
    if (count_main && a.ev_begin) NK_CUDA_OK(cudaEventRecord(a.ev_begin, a.stream));
    for (uint32_t q0 = 0; q0 < a.Q; q0 += 64) {
        TcPassArgs t{};
        t.grid = grid; t.k_emit = a.k; t.Qpad = Qpad; t.q0 = q0; t.nq = a.Q - q0 < 64u ? a.Q - q0 : 64u; t.qgroups = 1;
        t.qhi = qhi; t.qlo = qlo; t.only_if = only_if; t.count_main = count_main;
        if (launch_pass<3, 64>(di, a, ws, t, launches)) return -1;
    }
    if (count_main && a.ev_end) NK_CUDA_OK(cudaEventRecord(a.ev_end, a.stream));
    // fold the per-CTA lists and, when the caller wants them, write the decoded (index, score) arrays in the same launch
    if (merge_keys(ws.partial, grid, a.k, (size_t)grid * a.k, a.Q, a.k, out_keys, a.stream, only_if, 0, a.out_idx, a.out_score, a.metric)) return -1;
    if (launches) ++*launches;
    if (count_main) tc_print_prof(a.stream, num_tiles, grid, (a.dim + BK - 1) / BK);
    return 0;
}

int scan_tensor(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, uint64_t *out_keys, uint64_t *launches) {
    if (a.n == 0 || a.Q == 0 || a.k == 0) return 0;
    if (!scan_tensor_supported(di, a)) {
        set_error("tensor path: unsupported shape");
        return -1;
    }
    return scan_tensor_exact(di, a, ws, out_keys, launches, nullptr, true, true);
}

// TF32 filter passes over all queries
static int tf32_passes(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, const FilterPlan &f, const int *only_if,
                       bool count_main, int presampled, uint64_t *launches) {
    return plan_launches(0, a.Q, f.grid, 4, [&](uint32_t qt, uint32_t q0, uint32_t nq, uint32_t groups) {
        TcPassArgs t{};
        t.grid = f.grid; t.k_emit = f.k_emit; t.Qpad = f.Qpad; t.q0 = q0; t.nq = nq; t.qgroups = groups; t.margin_c = f.margin_tf32;
        t.qhi = f.qhi; t.qnorm = f.qnorm; t.only_if = only_if; t.count_main = count_main; t.presampled = presampled;
        return qt == 128 ? launch_pass<1, 128>(di, a, ws, t, launches) : launch_pass<1, 64>(di, a, ws, t, launches);
    });
}

// The prep launch of a filter search: every query array the plan's passes read, the cleared search state, the sample.
static PrepParams filter_prep_params(const ScanArgs &a, Workspace &ws, const FilterPlan &f) {
    PrepParams pp = prep_params(a, f.Qpad, f.dimpad);
    pp.acc_c = f.acc_c; pp.qhi = f.qhi;
    pp.qbf = f.big && !f.s8 ? static_cast<uint16_t *>(f.qbf16) : nullptr; pp.qbf_f16 = a.dtype == NK_DTYPE_F16;
    pp.qs8 = f.big && f.s8 ? static_cast<int8_t *>(f.qbf16) : nullptr; pp.qscale = f.qscale;
    pp.qnorm = f.qnorm; pp.qa = f.qa; pp.qb = f.qb;
    pp.state = reinterpret_cast<uint32_t *>(ws.keys2); pp.QA = f.QA; pp.flags = ws.flags; pp.sample = f.sample;
    return pp;
}

static void fill_finish(FinishParams &fp, const ScanArgs &a, Workspace &ws, const FilterPlan &f, uint64_t *out_keys) {
    fp.rows = a.rows; fp.dtype = a.dtype; fp.dim = a.dim; fp.row_base = a.row_base; fp.queries = a.queries;
    fp.lists = ws.partial; fp.gcount = reinterpret_cast<const int *>(ws.keys2) + f.QA; fp.list_cap = f.grid * f.k_emit; fp.k = a.k;
    fp.metric = a.metric; fp.margin_c = f.margin_tf32; fp.flags = ws.flags; fp.out = out_keys;
    fp.out_idx = a.out_idx; fp.out_score = a.out_score; fp.min_score = a.min_score;
    fp.qa = f.qa; fp.qb = f.qb; fp.qn = f.qnorm;
    fp.state = reinterpret_cast<uint32_t *>(ws.keys2); fp.state_words = 2 * f.QA;
}

// The retry / exact stages of a filter search.  Every kernel returns at once unless the stage before raised its flag on
// the device, so the tail can be queued blindly behind the first stage (asynchronous API: no host round trip) — or, for
// the host-synchronous API, only after the host has seen a flag (a_defer_tail): the common case then launches nothing.
int scan_tensor_filter_tail(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, uint64_t *out_keys, uint64_t *launches) {
    using namespace tc;
    FilterPlan f;
    if (make_filter_plan(di, a, ws, &f)) return -1;
    if (f.stage2 && a.defer_tail) {
        // the same search over the fp32 rows with the (much tighter) TF32 margins, if a 16-bit margin buffer overflowed.
        // Host-driven tail only: queued blindly (asynchronous API) the stage would cost two early-exit launches on EVERY
        // search to make the rare overflow cheaper — there an overflow goes straight to the exact stage.
        if (tf32_passes(di, a, ws, f, ws.flags + FLAG_RETRY, false, 0, launches)) return -1;
        FinishParams fp{};
        fill_finish(fp, a, ws, f, out_keys);
        fp.q_big = 0; fp.only_if = ws.flags + FLAG_RETRY; fp.mark_retry = 0;
        NK_CUDA_OK(launch_pdl(f.finish.kern, dim3(a.Q), dim3(FINISH_THREADS), f.finish.smem, a.stream, !a.defer_tail, fp));
        if (launches) ++*launches;
    }
    ScanArgs b = a;
    b.ev_begin = b.ev_end = nullptr;
    b.main_launches = nullptr;
    if (f.can_exact_tc) {
        if (scan_tensor_exact(di, b, ws, out_keys, launches, ws.flags + FLAG_OVERFLOW, false, false)) return -1;
    } else {  // euclidean / large k / 16-bit rows: the CUDA-core scan is the exact twin
        b.only_if = ws.flags + FLAG_OVERFLOW;
        if (scan_simt(di, b, ws, out_keys, launches)) return -1;
    }
    return 0;  // (both exact twins write the decoded arrays from their merge launch)
}

// Filter mode: prep -> 16-bit (or 1xTF32) scan with rigorous margins -> finish (select by upper bound, exact fp32
// rescoring, decode).  Three launches in the common case; the retry / exact stages follow as scan_tensor_filter_tail.
int scan_tensor_filter(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, uint64_t *out_keys, uint64_t *launches) {
    using namespace tc;
    if (a.check(false, false)) return -1;
    if (a.n == 0 || a.Q == 0 || a.k == 0) return 0;
    if (!scan_tensor_filter_supported(di, a)) {
        set_error("tensor filter path: unsupported shape");
        return -1;
    }
    FilterPlan f;
    if (make_filter_plan(di, a, ws, &f)) return -1;
    const uint32_t q_big = f.big ? a.Q : 0;  // queries served by the 16-bit kernel in the first stage (all or none)

    PrepParams pp = filter_prep_params(a, ws, f);
    pp.qlo = f.can_exact_tc ? f.qlo : nullptr;
    if (launch_prep(di, a.mode, pp, a.stream, launches)) return -1;

    if (a.ev_begin) NK_CUDA_OK(cudaEventRecord(a.ev_begin, a.stream));
    if (plan_launches(0, q_big, f.grid, f.max_groups_shadow, [&](uint32_t qt, uint32_t q0, uint32_t nq, uint32_t groups) {
            ShadowPassArgs sp = f.shadow_pass();
            sp.q0 = q0; sp.nq = nq; sp.qgroups = groups; sp.presampled = f.sample != 0;
            return launch_shadow_pass((int)qt, di, a, ws, sp, launches);
        }))
        return -1;
    if (!f.big && tf32_passes(di, a, ws, f, nullptr, true, f.sample != 0, launches)) return -1;
    if (a.ev_end) NK_CUDA_OK(cudaEventRecord(a.ev_end, a.stream));

    FinishParams fp{};
    fill_finish(fp, a, ws, f, out_keys);
    fp.q_big = q_big; fp.only_if = nullptr; fp.mark_retry = (f.stage2 && a.defer_tail) ? 1 : 0;
    fp.debug = tc_debug_flags() & 64;
    NK_CUDA_OK(launch_pdl(f.finish.kern, dim3(a.Q), dim3(FINISH_THREADS), f.finish.smem, a.stream, !a.defer_tail, fp));
    if (launches) ++*launches;
    tc_print_prof(a.stream, f.num_tiles, f.grid, (a.dim + BK - 1) / BK);
    fin_print_prof(a.stream, a.Q);
    if (a.defer_tail) return 0;
    return scan_tensor_filter_tail(di, a, ws, out_keys, launches);
}

// Range mode (nk_search_range, range.cu): the query prep, then the 16-bit / int8 pass (a.image set) or the TF32 filter over the
// fp32 rows with FIXED thresholds: ws.keys2 holds the order-preserving bits of every query's key-space threshold where the
// filter keeps its shared thresholds (presampled: no flood tiles, nothing is published), and every pair whose upper bound
// reaches it lands in ws.partial [Q][list_cap], fill counted in the list fills next to them (range_qa).  The caller
// re-scores the lists exactly.
int scan_tensor_range(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, uint32_t list_cap, uint64_t *launches) {
    using namespace tc;
    static_assert(QT_BIG == 256, "range_qa() (kernels.cuh) mirrors the padded per-query arrays");
    ScanArgs b = a;
    b.k = 1;
    FilterPlan f;
    if (make_filter_plan(di, b, ws, &f)) return -1;
    if (ws_reserve((void **)&ws.partial, &ws.partial_bytes, (size_t)a.Q * list_cap * 8)) return -1;
    PrepParams pp = filter_prep_params(b, ws, f);
    pp.state = nullptr;  // the thresholds and list fills are the caller's
    pp.sample = 0;
    if (launch_prep(di, a.mode, pp, a.stream, launches)) return -1;
    if (a.ev_begin) NK_CUDA_OK(cudaEventRecord(a.ev_begin, a.stream));
    int rc;
    if (f.big) {
        rc = plan_launches(0, a.Q, f.grid, 4, [&](uint32_t qt, uint32_t q0, uint32_t nq, uint32_t groups) {
            ShadowPassArgs sp = f.shadow_pass();
            sp.q0 = q0; sp.nq = nq; sp.qgroups = groups; sp.presampled = 1; sp.list_cap = list_cap;
            return launch_shadow_pass((int)qt, di, b, ws, sp, launches);
        });
    } else {
        rc = plan_launches(0, a.Q, f.grid, 4, [&](uint32_t qt, uint32_t q0, uint32_t nq, uint32_t groups) {
            TcPassArgs t{};
            t.grid = f.grid; t.k_emit = f.k_emit; t.Qpad = f.Qpad; t.q0 = q0; t.nq = nq; t.qgroups = groups; t.margin_c = f.margin_tf32;
            t.qhi = f.qhi; t.qnorm = f.qnorm; t.count_main = true; t.presampled = 1; t.list_cap = list_cap;
            return qt == 128 ? launch_pass<1, 128>(di, b, ws, t, launches) : launch_pass<1, 64>(di, b, ws, t, launches);
        });
    }
    if (rc) return -1;
    if (a.ev_end) NK_CUDA_OK(cudaEventRecord(a.ev_end, a.stream));
    return 0;
}

// ---- tests only: the filters' raw score estimates and error bounds for every (row, query) pair --------------------
// which: NK_PATH_TENSOR_FILTER (1xTF32 over the fp32 rows) or NK_PATH_TENSOR_SHADOW (16-bit pass).  est / bnd: device
// [n x ld] floats.  The estimate is what the kernel compares (before adding the bound); |est - exact| <= bnd is the
// invariant the filter's soundness rests on (tests/test_gpu_error_model.py measures it against fp64).
int scan_filter_dump(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, int which, float *est, float *bnd, uint32_t ld,
                     uint64_t *launches) {
    using namespace tc;
    if (a.Q == 0 || a.Q > 64 || a.n == 0) { set_error("dump: 1 <= Q <= 64 and n > 0 required"); return -1; }
    ScanArgs b = a;
    b.k = 1; b.min_score = -INFINITY; b.defer_tail = true; b.out_idx = nullptr; b.out_score = nullptr; b.mode = ScanMode::DUMP;
    if (!scan_tensor_filter_supported(di, b)) { set_error("dump: unsupported shape"); return -1; }
    FilterPlan f;
    if (make_filter_plan(di, b, ws, &f)) return -1;
    if (which == NK_PATH_TENSOR_SHADOW && !f.big) { set_error("dump: no 16-bit pass for this shard"); return -1; }
    if (which == NK_PATH_TENSOR_FILTER && a.dtype != NK_DTYPE_F32) { set_error("dump: TF32 pass needs fp32 rows"); return -1; }
    PrepParams pp = filter_prep_params(b, ws, f);
    pp.sample = 0;
    if (launch_prep(di, b.mode, pp, b.stream, launches)) return -1;
    if (which == NK_PATH_TENSOR_SHADOW) {
        ShadowPassArgs sp = f.shadow_pass();
        sp.q0 = 0; sp.nq = b.Q; sp.qgroups = 1; sp.presampled = 0;
        sp.dump_est = est; sp.dump_bnd = bnd; sp.dump_ld = ld;
        if (launch_shadow_pass(64, di, b, ws, sp, launches)) return -1;
    } else {
        TcPassArgs t{};
        t.grid = f.grid; t.k_emit = f.k_emit; t.Qpad = f.Qpad; t.q0 = 0; t.nq = b.Q; t.qgroups = 1; t.margin_c = f.margin_tf32;
        t.qhi = f.qhi; t.qnorm = f.qnorm; t.dump_est = est; t.dump_bnd = bnd; t.dump_ld = ld;
        if (launch_pass<1, 64>(di, b, ws, t, launches)) return -1;
    }
    return 0;
}

}  // namespace nk
