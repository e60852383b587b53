// scan_tensor_shadow.cu — filter scan over the BF16 SHADOW of the corpus (wgmma / TMA / mbarrier).
//
// An fp32 shard optionally carries a bf16 copy of itself ("shadow", +50% HBM, built once at upload and kept in step by
// append / update / remove) plus two floats per row: |x|^2 and |x - bf16(x)|^2.  The filter scan streams the SHADOW —
// half the bytes of the fp32 corpus, so the HBM-bound regime (Q <= 128) runs at twice the queries per second — and
// exact fp32 re-scoring of the few survivors (filter_finish_kernel, reading the fp32 rows) makes the results identical
// to a full-precision scan.  This is the default filter where a shadow exists; the TF32 scan over the fp32 rows
// (scan_tensor.cu) is its retry stage and serves shards without a shadow (caller-owned device rows, fp16 corpora).
//
// Rigorous bound.  With x = xb + dx, q = qb + dq (xb, qb the BF16 roundings):
//     x.q - xb.qb = dx.qb + x.dq   =>   |s_hat - s| <= |dx| |qb| + |x| |dq| + acc_c |x| |q|   (fp32 accumulation)
// |dx| per row and |qb|, |dq| per query are the MEASURED rounding residues (~0.4 * 2^-8 relative for typical data, not
// the worst case 2^-8), so the margin is as tight as Cauchy-Schwarz allows.  Rows whose upper bound reaches the running
// k-th bound are kept; margin overflow raises the device flag and the TF32 filter, then the exact kernels, retry.
//
// Both operands are plain bf16 tiles in shared memory, so there is no conversion stage; the accumulators live in the
// registers of the warpgroups that issue the MMAs and score them.
//   warp 0      TMA: shadow slabs [256 rows x 64 bf16] (32 KB, 128B-swizzled), 6-stage ring at QT = 64, 5 at QT = 128;
//   warp 3      TMA: query slabs [QT x 64 bf16] (8 / 16 KB), L2-resident;
//   warps 4-11  two consumer warpgroups, one per 128-row M-tile: per slab 2 x 4 wgmma.m64nQTk16 (A and B from smem,
//               fp32 accumulators in registers), then per tile: bound / compare / push straight
//               from the accumulator registers, warp-level prunes (scan_tensor_shared.cuh, shared with the TF32 kernel).
//               The TMA rings run ahead during the epilogue.  The epilogue's global inputs (row norms, mask words, shared
//               thresholds) are loaded at the top of the tile and have landed by the time the accumulators are ready.
//   registers   setmaxnreg: TMA warpgroup 24, consumers 240 during the scan (no spills at QT = 128); all warps 160 for
//               the end-of-launch emission, the producers' increase ordered after the consumers' decrease.
// Shared-memory traffic per [256 rows x 128 queries x 64 dims]: 112 KB (A 32 w + 32 r, B 16 w + 32 r) for twice the K
// extent of a TF32 slab: half the bytes per product of the TF32 kernel, which is shared-memory-bandwidth bound at 128
// query columns.  Algorithmic HBM bytes per launch: n * dimpad * 2 (shadow) + n * 8 (norms).
//
// Int8 image (Opnd::S8; the kNN filter picks it per search, index_api.cu shard_image): rows of dimpad8 = ceil(d / 128) * 128 int8 with one fp32 scale per row, x ~ s_x xq,
// and int8 queries with one scale each.  The shared-memory layout is the same byte for byte (a 128-byte swizzle row holds 128
// int8, one m64nQTk32 s8 MMA consumes the 32 B of one bf16 k16 MMA), the slab count halves, the exact s32 accumulators are
// converted in place to float(acc) s_q and s_x joins the row's multiplier.  The bound above holds for any image xb, qb, with
// the measured int8 residues; integer accumulation adds no error.  Bytes per launch: n * dimpad8 + n * 12.
#include <cuda.h>
#include <stdlib.h>

#include "kernels.cuh"
#include "ptx_sm90.cuh"
#include "scan_tensor_shared.cuh"

namespace nk {

namespace sb {
using namespace tc;
constexpr int NTHREADS = 384;
constexpr int QT_MAX = 128;
constexpr int BKB = 64;                   // bf16 per row per slab = one 128-byte swizzle row (int8 images: 128 elements)
constexpr int ASTAGES_MAX = 6;            // deepest shadow-slab ring (Cfg<QT>::ASTAGES)
constexpr int A_BYTES = ROWS * 128;       // 32 KB
constexpr int EPI_WARP0 = 4, EPI_WARPS = 8, EPI_NT = EPI_WARPS * 32;
// Registers (setmaxnreg): the TMA warpgroup gives its share to the consumers for the scan (128 x 24 + 256 x 240 = the
// 384 x 168 of the launch); every warp has 160 for the end-of-launch emission.  The pool is handed over in two ordered
// steps: the consumers' increase can only be served by the producers' decrease (nothing else asks for registers
// then), and the producers increase again only after every consumer warp has decreased (named barrier REG_BAR).
constexpr int PRODUCER_REGS = 24, CONSUMER_REGS = 240, EMIT_REGS = 160;
constexpr int REG_BAR = 2;                // consumers arrive after releasing their scan registers, producers wait
constexpr int PB = tc::P_SHADOW;          // candidate buffer slots per (CTA, query)
constexpr int PRUNE_LANE = PB / 32;       // keys per lane of a warp prune

// The shadow-slab ring is the HBM look-ahead that keeps loads in flight while the consumers run a tile's epilogue (every
// stage it holds is ~1.3 us of one SM's share of HBM time at the headline shape; the epilogue takes longer than the ring
// covers).  The query-slab ring reads L2-resident data and only has to stay ahead of the consumers' pace: at QT = 64 three
// stages suffice, and the 24 KB this frees from six buys a sixth shadow stage.  QT = 128 (16 KB query slabs) has no room
// for one: 5 x 32 KB + 3 x 16 KB is already the shared-memory budget.
template <int QT> struct Cfg {
    static constexpr int B_BYTES = QT * 128;
    static constexpr int ASTAGES = QT == 64 ? 6 : 5;
    static constexpr int BSTAGES = QT == 64 ? 3 : (48 * 1024) / B_BYTES;
    static constexpr int RING_BYTES = ASTAGES * A_BYTES + BSTAGES * B_BYTES;
    static_assert(ASTAGES <= ASTAGES_MAX && BSTAGES <= MAX_BSTAGES, "ring deeper than its barriers");
};

struct __align__(8) Shared {
    Rings<ASTAGES_MAX> ring;                       // (QT = 128 leaves the last stage's barriers unused)
    unsigned int maxxx, max_ra, max_rb;            // running maxima (float bits) of |x|^2 and the per-row bound factors
    float tau[QT_MAX];
    float qn[QT_MAX];                              // |q| (1 for cosine)
    float qa[QT_MAX], qb[QT_MAX];                  // bound(row, q) = ra(row) qa[q] + rb(row) qb[q]
    float qs[QT_MAX];                              // int8 image: scale of the query's int8 copy
    int cnt[QT_MAX];
    uint32_t ethr[QT_MAX];                         // emission: score-word threshold per query
    int eoff[QT_MAX + 1];                          // emission: prefix of 32-entry chunk counts
};
}  // namespace sb

// fp32 rows -> bf16 shadow rows (row stride dimpad, zero padded) + |x|^2 and |x - bf16(x)|^2 per row.  One warp per row.
__global__ void build_shadow_kernel(const float *rows, uint64_t n, uint32_t dim, uint32_t dimpad, uint16_t *shadow, float *xnorm2,
                                    float *dnorm2) {
    const uint64_t row = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= n) return;
    const float *x = rows + row * dim;
    uint16_t *o = shadow + row * dimpad;
    float xx = 0.0f, dd = 0.0f;
    if ((dim & 3u) == 0 && ((reinterpret_cast<uintptr_t>(rows) & 15) == 0)) {
        for (uint32_t j = lane * 4; j < dimpad; j += 128) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (j < dim) v = __ldg(reinterpret_cast<const float4 *>(x + j));
            const uint32_t b01 = ptx::pack_bf16x2(v.x, v.y), b23 = ptx::pack_bf16x2(v.z, v.w);
            *reinterpret_cast<uint2 *>(o + j) = make_uint2(b01, b23);
            const float e0 = v.x - __uint_as_float(b01 << 16), e1 = v.y - __uint_as_float(b01 & 0xffff0000u);
            const float e2 = v.z - __uint_as_float(b23 << 16), e3 = v.w - __uint_as_float(b23 & 0xffff0000u);
            xx = fmaf(v.x, v.x, xx); xx = fmaf(v.y, v.y, xx); xx = fmaf(v.z, v.z, xx); xx = fmaf(v.w, v.w, xx);
            dd = fmaf(e0, e0, dd); dd = fmaf(e1, e1, dd); dd = fmaf(e2, e2, dd); dd = fmaf(e3, e3, dd);
        }
    } else {
        for (uint32_t j = lane; j < dimpad; j += 32) {
            const float v = j < dim ? x[j] : 0.0f;
            const uint16_t b = ptx::f32_to_bf16_bits(v);
            o[j] = b;
            const float e = v - __uint_as_float((uint32_t)b << 16);
            xx = fmaf(v, v, xx);
            dd = fmaf(e, e, dd);
        }
    }
#pragma unroll
    for (int s = 16; s; s >>= 1) {
        xx += __shfl_xor_sync(0xffffffffu, xx, s);
        dd += __shfl_xor_sync(0xffffffffu, dd, s);
    }
    if (lane == 0) { xnorm2[row] = xx; dnorm2[row] = dd; }
}

int build_shadow(const float *rows, uint64_t first, uint64_t count, uint32_t dim, uint32_t dimpad, void *shadow, float *xnorm2,
                 float *dnorm2, cudaStream_t stream) {
    if (count == 0) return 0;
    const unsigned int blocks = (unsigned int)((count + 7) / 8);
    build_shadow_kernel<<<blocks, 256, 0, stream>>>(rows + first * dim, count, dim, dimpad,
                                                    static_cast<uint16_t *>(shadow) + first * dimpad, xnorm2 + first, dnorm2 + first);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}

// fp32 rows -> int8 image rows (row stride dimpad bytes, zero padded) + per row s = max|x_i| / 127, |x|^2 and |x - s q|^2.
// One warp per row, two passes over the row (the second from L1): the maximum, then the rounding.  A row with a non-finite
// element gets s = NaN (and q = 0): its estimates are NaN and it is kept with bound +inf, as a NaN row of the BF16 shadow is.
// A zero row has s = 0, q = 0 and a zero residue.
__global__ void build_image_s8_kernel(const float *rows, uint64_t n, uint32_t dim, uint32_t dimpad, int8_t *image, float *xscale,
                                      float *xnorm2, float *dnorm2) {
    const uint64_t row = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= n) return;
    const float *x = rows + row * dim;
    const bool vec = (dim & 3u) == 0 && ((reinterpret_cast<uintptr_t>(rows) & 15) == 0);
    auto load4 = [&](uint32_t j) {
        if (j >= dim) return make_float4(0.f, 0.f, 0.f, 0.f);
        if (vec) return __ldg(reinterpret_cast<const float4 *>(x + j));
        return make_float4(__ldg(x + j), j + 1 < dim ? __ldg(x + j + 1) : 0.f, j + 2 < dim ? __ldg(x + j + 2) : 0.f, j + 3 < dim ? __ldg(x + j + 3) : 0.f);
    };
    float mx = 0.0f, xx = 0.0f;
    bool bad = false;
    for (uint32_t j = lane * 4; j < dim; j += 128) {
        const float4 v = load4(j);
        mx = fmaxf(fmaxf(mx, fmaxf(fabsf(v.x), fabsf(v.y))), fmaxf(fabsf(v.z), fabsf(v.w)));
        bad |= (v.x - v.x) != 0.0f || (v.y - v.y) != 0.0f || (v.z - v.z) != 0.0f || (v.w - v.w) != 0.0f;
        xx = fmaf(v.x, v.x, xx); xx = fmaf(v.y, v.y, xx); xx = fmaf(v.z, v.z, xx); xx = fmaf(v.w, v.w, xx);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        xx += __shfl_xor_sync(0xffffffffu, xx, o);
    }
    bad = __any_sync(0xffffffffu, bad);
    const float sc = bad ? NAN : mx / 127.0f, sinv = !bad && mx > 0.0f ? 127.0f / mx : 0.0f;
    int8_t *o = image + row * dimpad;
    float dd = 0.0f;
    for (uint32_t j = lane * 4; j < dimpad; j += 128) {
        const float4 v = load4(j);
        const float f[4] = {v.x, v.y, v.z, v.w};
        uint32_t packed = 0;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int iq = max(-127, min(127, __float2int_rn(f[e] * sinv)));
            const float r = fmaf(-sc, (float)iq, f[e]);
            dd = fmaf(r, r, dd);
            packed |= ((uint32_t)iq & 0xffu) << (8 * e);
        }
        *reinterpret_cast<uint32_t *>(o + j) = packed;
    }
#pragma unroll
    for (int s = 16; s; s >>= 1) dd += __shfl_xor_sync(0xffffffffu, dd, s);
    if (lane == 0) { xscale[row] = sc; xnorm2[row] = xx; dnorm2[row] = dd; }
}

int build_image_s8(const float *rows, uint64_t first, uint64_t count, uint32_t dim, uint32_t dimpad, void *image, float *xscale,
                   float *xnorm2, float *dnorm2, cudaStream_t stream) {
    if (count == 0) return 0;
    const unsigned int blocks = (unsigned int)((count + 7) / 8);
    build_image_s8_kernel<<<blocks, 256, 0, stream>>>(rows + first * dim, count, dim, dimpad, static_cast<int8_t *>(image) + first * dimpad,
                                                      xscale + first, xnorm2 + first, dnorm2 + first);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}

// Debug timeline (NK_TC_DEBUG & 64): per-CTA globaltimer stamps, printed by launch_shadow_pass_t after a synchronize.
//   [0] entry  [1] set-up done  [2] first accumulator ready  [3] last tile's epilogue done  [4] exit
//   [5] ns in the prune section (epilogue warp 0)  [6] tile index of the first prune  [7] ns waiting for accumulators
//   [8] all warps past the tile loop  [9] warp 0 done emitting  [10] live chunks  [11] entries emitted by warp 0
//   [12..14] emission stages.  The tile loop of epilogue thread 0, split (ns summed over its tiles): [15] tiles
//   [16] waiting for the row inputs (|x|^2, |dx|^2, scale, mask word, row threshold) after the accumulators
//   [17] int8 conversion, the rows' estimates and the keep rule  [18] the row maxima's shared atomics (one per warp and value)
//   [19] the first EPI_BAR (arrival skew)  [20] prunes / flushes  [21] the second EPI_BAR  [22] threshold adoption
__device__ unsigned long long g_sb_prof[256][24];
__device__ float g_sb_sink;  // the timeline's row-input stamp stores their sum here: the store waits until they landed

// Score estimate of one accumulator fragment row of the 16-bit scan (keep_fragment_rows): the UPPER bound of the score,
// bound(row, q) = ra qa[q] + rb qb[q]:
//   cosine     acc/|x|                        ra = |dx|/|x|   rb = 1
//   dot        acc                            ra = |dx|       rb = |x|
//   euclidean  -(|x|^2 + |q|^2 - 2 acc)        ra = 2|dx|      rb = 2|x|   (+ eps (|x|^2 + |q|^2))
struct Bf16Est {
    float mul, ra, rb, x2;
    const float *qa, *qb, *qn;
    bool euclid;
    struct Col { float qa, qb, qn; };  // the query's inputs, read once per column for all of a thread's rows
    __device__ __forceinline__ Col col(uint32_t qi) const { return {qa[qi], qb[qi], euclid ? qn[qi] : 0.0f}; }
    __device__ __forceinline__ float upper(float v, const Col &c) const {
        float sc = fmaf(v, mul, fmaf(ra, c.qa, rb * c.qb));
        if (euclid) sc -= tc::EUC_KEEP * fmaf(c.qn, c.qn, x2);
        return sc;
    }
    __device__ __forceinline__ float bound(uint32_t qi) const { return fmaf(ra, qa[qi], rb * qb[qi]); }
};

// OP: the operand type, bf16 (BF16 shadow, bf16 corpora), fp16 (an fp16 corpus scanned in place) or int8 (the int8 image of
// an fp32 shard).  M: the scan mode (kernels.cuh).  Tag filters are read through the read-only cache (shared memory is spent
// on the rings); the row-filter modes stage the launch's query tags (REVERSE_RWINDOW: and value keys) in shared memory past
// Shared.
template <int QT, ptx::Opnd OP, ScanMode M>
__global__ void __launch_bounds__(sb::NTHREADS, 1)
knn_scan_shadow_kernel(const __grid_constant__ CUtensorMap map_rows, const __grid_constant__ CUtensorMap map_q, tc::Params p) {
    using namespace sb;
    using C = Cfg<QT>;
    pdl_trigger();  // the finish kernel's launch may begin now (it waits for this grid's completion before reading anything)
    if (p.only_if && *p.only_if == 0) return;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *smem_raw = smem_dyn + ((1024u - (ptx::smem_u32(smem_dyn) & 1023u)) & 1023u);
    unsigned char *a_base = smem_raw;
    unsigned char *b_base = smem_raw + (size_t)C::ASTAGES * A_BYTES;
    Shared &sh = *reinterpret_cast<Shared *>(smem_raw + (size_t)C::RING_BYTES);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const bool prof = (p.debug & 64) && blockIdx.x < 256;
    if (prof && tid == 0) {
        g_sb_prof[blockIdx.x][0] = globaltimer_ns(); g_sb_prof[blockIdx.x][6] = ~0ull;
        for (int i = 16; i <= 22; ++i) g_sb_prof[blockIdx.x][i] = 0;
    }
    const uint32_t num_tiles = (p.n + ROWS - 1) / ROWS;
    const QueryGroup<QT> qg(p);
    const uint32_t sub = qg.sub, sgrid = qg.sgrid, q0 = qg.q0, qpad_off = qg.qpad_off, nq = qg.nq;
    const uint32_t nslab = p.nslab;  // dimpad / 64 (int8 image: dimpad / 128)
    constexpr bool S8 = OP == ptx::Opnd::S8;
    constexpr uint32_t KCOLS = S8 ? 128 : BKB;  // elements per row of a slab: 128 bytes either way

    if (warp == 0 && lane == 0) {
        ptx::prefetch_tensormap(&map_rows);
        ptx::prefetch_tensormap(&map_q);
        sh.maxxx = 0u; sh.max_ra = 0u; sh.max_rb = 0u;
        sh.ring.init(C::BSTAGES);
    }
    if (tid < QT) {
        sh.tau[tid] = start_tau(p, q0, tid, nq);
        sh.cnt[tid] = 0;
        sh.qn[tid] = p.qnorm[qpad_off + tid];
        sh.qa[tid] = p.qa[qpad_off + tid];
        sh.qb[tid] = p.qb[qpad_off + tid];
        if (S8) sh.qs[tid] = p.qscale[qpad_off + tid];
    }
    // row-filter modes only: the query tags [QT], then (REVERSE_RWINDOW) the query value keys [QT]
    uint64_t *qtag = reinterpret_cast<uint64_t *>(smem_raw + (size_t)C::RING_BYTES + sizeof(Shared));
    if (mode_row_filter(M) && tid < QT) qtag[tid] = (uint32_t)tid < nq ? p.qtags[q0 + tid] : 0ull;
    if constexpr (mode_row_window(M))
        if (tid < QT) qtag[QT + tid] = (uint32_t)tid < nq ? p.qvalues[q0 + tid] : 0ull;
    __syncthreads();
    const bool flood = !p.presampled;  // first two tiles: every (row, query) pair is placed directly
    if (prof && tid == 0) g_sb_prof[blockIdx.x][1] = globaltimer_ns();
    const bool cosine = p.metric == NK_METRIC_COSINE;
    uint64_t *my_cand = p.cand + (size_t)blockIdx.x * QT * PB;
    auto prune = [&](uint32_t qi, uint64_t *out, int out_len, int max_keep, float floor_tau, int *gcount) {
        const float margin2 = bf16_margin2(p.metric, __uint_as_float(sh.max_ra), cosine ? 1.0f : __uint_as_float(sh.max_rb),
                                           __uint_as_float(sh.maxxx), sh.qa[qi], sh.qb[qi], sh.qn[qi]);
        // the select's cost is the register-resident key count: an early-trigger prune holds ~260-300 keys, not PB
        uint64_t *c = my_cand + (size_t)qi * PB;
        const int have = sh.cnt[qi];
        if (have <= 320)
            warp_prune<10>(c, &sh.cnt[qi], &sh.tau[qi], p.k, lane, out, out_len, true, margin2, max_keep, floor_tau, gcount, p.flags + FLAG_OVERFLOW);
        else if (have <= 512)
            warp_prune<16>(c, &sh.cnt[qi], &sh.tau[qi], p.k, lane, out, out_len, true, margin2, max_keep, floor_tau, gcount, p.flags + FLAG_OVERFLOW);
        else
            warp_prune<PRUNE_LANE>(c, &sh.cnt[qi], &sh.tau[qi], p.k, lane, out, out_len, true, margin2, max_keep, floor_tau, gcount,
                                   p.flags + FLAG_OVERFLOW);
    };

    if (warp < EPI_WARP0) {
        ptx::setmaxnreg_dec<PRODUCER_REGS>();
        if (warp == 0) {
            // ===================================== TMA producer: shadow slabs =========================
            tma_producer<C::ASTAGES>(sh.ring.aempty, sub, num_tiles, sgrid, 1, nslab, false, [&](uint32_t s, uint32_t tile, uint32_t, uint32_t j) {
                ptx::mbar_arrive_expect_tx(&sh.ring.afull[s], A_BYTES);
                ptx::tma_load_2d(&map_rows, &sh.ring.afull[s], a_base + (size_t)s * A_BYTES, (int32_t)(j * KCOLS), (int32_t)(tile * ROWS), qg.a_policy);
            });
        } else if (warp == 3) {
            // ===================================== TMA producer: query slabs (L2-resident) ===========
            tma_producer<C::BSTAGES>(sh.ring.bempty, sub, num_tiles, sgrid, 1, nslab, false, [&](uint32_t s, uint32_t, uint32_t, uint32_t j) {
                ptx::mbar_arrive_expect_tx(&sh.ring.bfull[s], C::B_BYTES);
                ptx::tma_load_2d(&map_q, &sh.ring.bfull[s], b_base + (size_t)s * C::B_BYTES, (int32_t)(j * KCOLS), (int32_t)qpad_off, ptx::CACHE_EVICT_LAST);
            });
        }
        ptx::named_bar_sync(REG_BAR, NTHREADS);  // every consumer warp is back at EMIT_REGS: the pool holds what this asks for
        ptx::setmaxnreg_inc<EMIT_REGS>();
    } else {
        ptx::setmaxnreg_inc<CONSUMER_REGS>();
        // ===================================== consumers: MMA + epilogue ===========================
        // warpgroup m owns rows [128 m, 128 m + 128) of the tile as two m64 halves h; thread = 4 rows x QT/4 columns of
        // the accumulator fragments: rows rbase + 64 h + 8 r, columns cbase + 8 (j / 2) + j % 2
        const uint32_t ewarp = warp - EPI_WARP0, m = ewarp >> 2, wq = ewarp & 3;
        const uint32_t rbase = m * 128 + wq * 16 + ((uint32_t)lane >> 2), cbase = 2u * ((uint32_t)lane & 3u);
        // capacity rule: a buffer must be prunable below PB - ROWS, or the next tile could overflow it.  Prunes are TRIGGERED
        // much earlier: an early, tight threshold keeps the buffers short, so the emission at the end of the launch needs no
        // selection and the finish step reads short lists (small shards: 26 tiles per CTA at N = 1M would otherwise never
        // prune at all).
        const int prune_at = PB - ROWS;
        const int prune_trigger = min(prune_at, max(192, 4 * (int)p.k));
        const bool euclid = p.metric == NK_METRIC_EUCLIDEAN;
        const bool eprof = prof && ewarp == 0 && lane == 0;
        unsigned long long t_wait = 0, t_a = 0;
        unsigned long long *split = g_sb_prof[blockIdx.x < 256 ? blockIdx.x : 0];  // [16..22] (eprof only: no registers held)
        float acc[2][QT / 2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < QT / 2; ++i) acc[h][i] = 0.0f;
        uint32_t g = 0, it = 0;
        for (uint32_t tile = sub; tile < num_tiles; tile += sgrid, ++it) {
            if (eprof) t_a = globaltimer_ns();
            // The epilogue's row inputs, loaded before the MMAs: |x|^2, |dx|^2 (int8 image: and the row's scale), the mask word
            // and (reverse modes) the threshold of this thread's 4 rows; and the shared threshold of query etid (it only grows: an
            // earlier value is still a lower bound).
            float x2[4], d2[4], rthr[4], xs[4];
            uint32_t mword[4];
#pragma unroll
            for (uint32_t ri = 0; ri < 4; ++ri) {
                const uint32_t row = tile * ROWS + rbase + 64 * (ri >> 1) + 8 * (ri & 1);
                const bool in = row < p.n;
                x2[ri] = in ? __ldg(p.xnorm2 + row) : 0.0f;
                d2[ri] = in && p.dnorm2 ? __ldg(p.dnorm2 + row) : 0.0f;  // 16-bit corpus: no residue
                mword[ri] = in && p.mask ? __ldg(p.mask + (row >> 5)) : ~0u;
                rthr[ri] = mode_row_thr(M) && in ? __ldg(p.row_thr + row) : -INFINITY;
                xs[ri] = S8 && in ? __ldg(p.xscale + row) : 1.0f;
            }
            const uint32_t etid = tid - EPI_WARP0 * 32;  // consumer thread: one query each (QT <= EPI_NT)
            const uint32_t gt_pre = !mode_range(M) && etid < nq ? __ldcg(p.gtau + q0 + etid) : 0u;
            uint32_t prev_sa = 0, prev_sb = 0;
            for (uint32_t j = 0; j < nslab; ++j, ++g) {
                const uint32_t sa = g % C::ASTAGES, sbq = g % C::BSTAGES;
                ptx::mbar_wait(&sh.ring.bfull[sbq], (g / C::BSTAGES) & 1);
                ptx::mbar_wait(&sh.ring.afull[sa], (g / C::ASTAGES) & 1);
                const uint64_t bdesc = ptx::make_smem_desc_sw128(ptx::smem_u32(b_base + (size_t)sbq * C::B_BYTES));
                const uint32_t abase = ptx::smem_u32(a_base + (size_t)sa * A_BYTES + (size_t)m * (A_BYTES / 2));
                ptx::wgmma_fence();
                // K advance per MMA = 16 bf16 (32 int8) = 32 B = 2 descriptor units
#pragma unroll
                for (uint32_t h = 0; h < 2; ++h) {
                    const uint64_t adesc = ptx::make_smem_desc_sw128(abase + h * (A_BYTES / 4));
#pragma unroll
                    for (uint32_t kk = 0; kk < 4; ++kk) ptx::wgmma_op<QT, OP>(acc[h], adesc + kk * 2, bdesc + kk * 2, (j | kk) != 0);
                }
                ptx::wgmma_commit();
                if (j > 0) {  // the previous slab's MMAs are done while this slab's run: its stages go back to the producers
                    ptx::wgmma_wait_one();
                    __syncwarp();
                    if (lane == 0) { ptx::mbar_arrive(&sh.ring.aempty[prev_sa]); ptx::mbar_arrive(&sh.ring.bempty[prev_sb]); }
                }
                prev_sa = sa;
                prev_sb = sbq;
            }
            ptx::wgmma_wait_all();
            ptx::fence_acc(acc[0]);
            ptx::fence_acc(acc[1]);
            if (eprof) {
                const unsigned long long t = globaltimer_ns();
                t_wait += t - t_a;
                if (it == 0) g_sb_prof[blockIdx.x][2] = t;
                t_a = t;
            }
            if (eprof) {  // wait for the row inputs here, to time it
                float s = 0.0f;
#pragma unroll
                for (uint32_t ri = 0; ri < 4; ++ri) s += x2[ri] + d2[ri] + xs[ri] + rthr[ri] + (float)mword[ri];
                *(volatile float *)&g_sb_sink = s;
                const unsigned long long t = globaltimer_ns();
                split[16] += t - t_a;
                t_a = t;
            }
            if constexpr (S8) {
                // exact int32 dot products of the int8 rows -> fp32 in the same registers, times the query's scale (the
                // row's scale is part of the estimate's multiplier): acc = xq.qq s_q, the estimate (s_x xq).(s_q qq)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int i = 0; i < QT / 2; ++i)
                        acc[h][i] = __int2float_rn(__float_as_int(acc[h][i])) * sh.qs[cbase + 8 * (i >> 2) + (i & 1)];
            }
            __syncwarp();
            if (lane == 0) { ptx::mbar_arrive(&sh.ring.aempty[prev_sa]); ptx::mbar_arrive(&sh.ring.bempty[prev_sb]); }
            // the rows' estimates
            Bf16Est est[4];
            uint32_t alive = 0u;
            uint32_t mx_ra = 0u, mx_rb = 0u, mx_xx = 0u;  // maxima (float bits) of the bound factors and |x|^2 of the alive rows
#pragma unroll
            for (uint32_t ri = 0; ri < 4; ++ri) {
                const uint32_t row = tile * ROWS + rbase + 64 * (ri >> 1) + 8 * (ri & 1);
                const bool live = row < p.n && ((mword[ri] >> (row & 31)) & 1u);
                alive |= live ? 1u << ri : 0u;
                Bf16Est &e = est[ri];
                e.x2 = x2[ri];
                e.qa = sh.qa;
                e.qb = sh.qb;
                e.qn = sh.qn;
                e.euclid = euclid;
                const float xn = sqrtf(e.x2);
                const float dxn = sqrtf(d2[ri]) * 1.0001f;
                e.mul = 1.0f; e.ra = dxn; e.rb = xn;
                if (cosine) {
                    e.mul = e.x2 > 0.0f ? 1.0f / xn : 0.0f;
                    e.ra = dxn * e.mul * 1.000001f;
                    e.rb = 1.0f;
                } else if (euclid) {
                    e.mul = 2.0f; e.ra = 2.0f * dxn; e.rb = 2.0f * xn;
                }
                if (S8) e.mul *= xs[ri];  // (a NaN scale: a non-finite row, every estimate NaN -> kept)
                if (live && e.ra < INFINITY && e.rb < INFINITY) {  // NaN / Inf rows are kept anyway (score NaN -> +inf)
                    mx_ra = max(mx_ra, __float_as_uint(e.ra));
                    if (!cosine) { mx_rb = max(mx_rb, __float_as_uint(e.rb)); mx_xx = max(mx_xx, __float_as_uint(e.x2)); }
                }
            }
            if (eprof) { const unsigned long long t = globaltimer_ns(); split[17] += t - t_a; t_a = t; }
            {
                // One atomic per warp and maximum.  This tile's prunes (after the first EPI_BAR) read the maxima over every
                // row this CTA has seen, as per-row atomics would leave them.
                const uint32_t wa = __reduce_max_sync(0xffffffffu, mx_ra);
                const uint32_t wb = __reduce_max_sync(0xffffffffu, mx_rb), wx = __reduce_max_sync(0xffffffffu, mx_xx);
                if (lane == 0) {
                    atomicMax(&sh.max_ra, wa);
                    if (!cosine) { atomicMax(&sh.max_rb, wb); atomicMax(&sh.maxxx, wx); }
                }
            }
            if (eprof) { const unsigned long long t = globaltimer_ns(); split[18] += t - t_a; t_a = t; }
            if (flood && it < 2 && ewarp == 0 && lane == 0)
                for (uint32_t qi = 0; qi < nq; ++qi) sh.cnt[qi] = (int)((it + 1) * ROWS);
            keep_fragment_rows<QT, PB, true, M>(p, est, acc, 0, alive, tile * ROWS, rbase, flood, it, cbase, q0, nq, sh.tau, sh.qn, sh.cnt, my_cand,
                                                rthr, qtag);
            if (eprof) { const unsigned long long t = globaltimer_ns(); split[17] += t - t_a; t_a = t; }
            // prune any buffer that could overflow during the next tile (8 warps, different queries concurrently)
            group_sync(EPI_BAR, EPI_NT);  // every push of this tile is visible
            if (eprof) { const unsigned long long t = globaltimer_ns(); split[19] += t - t_a; t_a = t; }
            if constexpr (mode_range(M))
                flush_tile<PB>(p, q0, nq, ewarp, lane, my_cand, sh.cnt);
            else
                prune_tile<true>(p, q0, nq, ewarp, lane, sh.cnt, sh.tau, prune_trigger, prune_at, flood && it == 0,
                                 [&](uint32_t qi, uint64_t *out, int out_len, int max_keep, float floor_tau, int *gcount) {
                                     if (eprof && g_sb_prof[blockIdx.x][6] == ~0ull) g_sb_prof[blockIdx.x][6] = it;
                                     prune(qi, out, out_len, max_keep, floor_tau, gcount);
                                 });
            if (eprof) { const unsigned long long t = globaltimer_ns(); split[20] += t - t_a; t_a = t; }
            group_sync(EPI_BAR, EPI_NT);
            if (eprof) { const unsigned long long t = globaltimer_ns(); split[21] += t - t_a; t_a = t; }
            if (!mode_range(M) && etid < nq) sh.tau[etid] = raise_to_shared_tau(gt_pre, sh.tau[etid]);  // adopt the shared threshold
            if (eprof) split[22] += globaltimer_ns() - t_a;
        }
        if (eprof) {
            unsigned long long *pr = g_sb_prof[blockIdx.x];
            pr[3] = globaltimer_ns(); pr[5] = pr[20] + pr[21]; pr[7] = t_wait; pr[15] = it;
        }
        ptx::setmaxnreg_dec<EMIT_REGS>();
        ptx::named_bar_arrive(REG_BAR, NTHREADS);
    }

    // ---- emit: everything inside this CTA's margin AND above the shared threshold goes to the query's shared list.
    __syncthreads();
    if constexpr (mode_range(M)) {  // range modes: what the last flushes left, whole (no staging: one buffer per warp at a time)
        for (uint32_t qi = warp; qi < nq; qi += NTHREADS / 32) flush_query(p, q0, qi, lane, my_cand + (size_t)qi * PB, sh.cnt);
    } else {
        // Fast path (buffers with <= k_emit entries, i.e. almost always all of them): no selection, the finish kernel selects
        // globally — append what still reaches the current threshold.  The buffers live in global memory (L2); walking them
        // query by query was a chain of dependent round trips (~19 us at the end of every launch, measured).  Instead: the
        // thresholds of all queries in one round, then the live 32-entry chunks of ALL buffers as one flat work list, 16
        // independent loads in flight per warp, then the list-fill atomics of the whole batch in one more round.
        constexpr int NW = NTHREADS / 32, JQ = (QT + NW - 1) / NW;
        constexpr int STAGE_CHUNKS = Cfg<QT>::RING_BYTES / 256;  // 32-key chunks the (contiguous) operand rings hold
        if (prof && tid == 0) g_sb_prof[blockIdx.x][8] = globaltimer_ns();
        int n_emitted = 0;
        if (tid < QT) {
            // (the shared threshold is fetched asynchronously: its round trip — several microseconds while the other CTAs
            // still stream — overlaps the staging of the buffers below instead of preceding it)
            int chunks = 0;
            sh.ethr[tid] = 0u;
            if ((uint32_t)tid < nq && sh.cnt[tid] <= (int)p.k_emit) {
                asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(ptx::smem_u32(&sh.ethr[tid])), "l"(p.gtau + q0 + tid) : "memory");
                chunks = (sh.cnt[tid] + 31) >> 5;
            }
            sh.eoff[tid + 1] = chunks;
        }
        __syncthreads();
        if (warp == 0) {  // inclusive prefix of the chunk counts -> eoff[q + 1]; eoff[0] = 0
            constexpr int PERL = QT / 32;
            int loc[PERL], sum = 0;
#pragma unroll
            for (int i = 0; i < PERL; ++i) { loc[i] = sh.eoff[lane * PERL + i + 1]; sum += loc[i]; }
            int incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            int run = incl - sum;
            if (lane == 0) sh.eoff[0] = 0;
#pragma unroll
            for (int i = 0; i < PERL; ++i) { run += loc[i]; sh.eoff[lane * PERL + i + 1] = run; }
        }
        __syncthreads();
        {
            // The operand rings are idle now (every MMA has completed: the epilogue saw the last accumulator): stage the live
            // chunks there with asynchronous copies — every load of the warp in flight at once, no registers held.  Chunk
            // c of query q lands in stage slot eoff[q] + c; queries whose chunks do not fit the rings take the per-query path.
            if (prof && tid == 0) g_sb_prof[blockIdx.x][12] = globaltimer_ns();  // prefix done
            uint64_t *stage = reinterpret_cast<uint64_t *>(a_base);
            for (uint32_t qi = warp; qi < nq; qi += NW) {
                const int c0 = sh.eoff[qi], c1 = sh.eoff[qi + 1], n = sh.cnt[qi];
                if (c1 > STAGE_CHUNKS) continue;
                for (int ch = 0; ch < c1 - c0; ++ch) {
                    const int slot = (ch << 5) + lane;
                    uint64_t *dst = stage + ((size_t)(c0 + ch) << 5) + lane;
                    if (slot < n)
                        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(ptx::smem_u32(dst)), "l"(my_cand + (size_t)qi * PB + slot) : "memory");
                    else
                        *dst = 0ull;
                }
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            if (tid < QT) {  // the shared thresholds have landed too -> final score-word threshold per query
                float t = fmaxf(sh.tau[tid], p.min_score);
                const uint32_t gt = sh.ethr[tid];
                if (gt) t = fmaxf(t, ord_to_float(gt));
                sh.ethr[tid] = t > -INFINITY ? ord_bits(t) : 0u;
            }
            __syncthreads();
            if (prof && tid == 0) g_sb_prof[blockIdx.x][13] = globaltimer_ns();  // staged
            // survivors per query (pass A), ONE list-fill atomic per query — lane j owns the warp's j-th query, all of them
            // in one round trip — then the stores (pass B)
            int my = 0;
#pragma unroll
            for (int j = 0; j < JQ; ++j) {
                const uint32_t qi = warp + j * NW;
                if (qi >= nq) continue;
                const int c0 = sh.eoff[qi], c1 = sh.eoff[qi + 1];
                if (c1 > STAGE_CHUNKS) continue;
                const uint32_t th = sh.ethr[qi];
                int tot = 0;
                for (int c = c0; c < c1; ++c) {
                    const uint64_t v = stage[((size_t)c << 5) + lane];
                    tot += __popc(__ballot_sync(0xffffffffu, v != 0ull && (uint32_t)(v >> 32) >= th));
                }
                if (lane == j) my = tot;
            }
            int off = 0;
            if (my > 0) off = atomicAdd(p.gcount + q0 + warp + lane * NW, my);
            if (prof && tid == 0) g_sb_prof[blockIdx.x][14] = globaltimer_ns() + (off & 0);  // list-fill atomics answered
#pragma unroll
            for (int j = 0; j < JQ; ++j) {
                const uint32_t qi = warp + j * NW;
                int goff = __shfl_sync(0xffffffffu, off, j);
                if (qi >= nq) continue;
                const int c0 = sh.eoff[qi], c1 = sh.eoff[qi + 1];
                if (c1 > STAGE_CHUNKS) continue;
                const uint32_t th = sh.ethr[qi];
                uint64_t *out = p.partial + (size_t)(q0 + qi) * p.list_cap;
                for (int c = c0; c < c1; ++c) {
                    const uint64_t v = stage[((size_t)c << 5) + lane];
                    const bool keep = v != 0ull && (uint32_t)(v >> 32) >= th;
                    const uint32_t m = __ballot_sync(0xffffffffu, keep);
                    const int pos = goff + __popc(m & ((1u << lane) - 1u));
                    if (keep && pos < (int)p.list_cap) out[pos] = v;
                    goff += __popc(m);
                    n_emitted += __popc(m);
                }
            }
            if (prof && tid == 0) { g_sb_prof[blockIdx.x][9] = globaltimer_ns(); g_sb_prof[blockIdx.x][10] = (unsigned long long)sh.eoff[QT]; g_sb_prof[blockIdx.x][11] = (unsigned long long)n_emitted; }
        }
        for (uint32_t qi = warp; qi < nq; qi += NW) {  // buffers beyond k_emit (near-tie data): select, then emit
            if (sh.cnt[qi] <= (int)p.k_emit && sh.eoff[qi + 1] <= STAGE_CHUNKS) continue;
            emit_query(p, q0, qi, lane, my_cand + (size_t)qi * PB, sh.cnt, sh.tau, prune);  // (or did not fit the staging area)
        }
        if (tid == 0) {
            atomicMax(reinterpret_cast<unsigned int *>(p.flags + FLAG_MAXXX), sh.maxxx);
            atomicMax(reinterpret_cast<unsigned int *>(p.flags + FLAG_MAX_RA), sh.max_ra);
            atomicMax(reinterpret_cast<unsigned int *>(p.flags + FLAG_MAX_RB), cosine ? __float_as_uint(1.0f) : sh.max_rb);
        }
    }
    if (prof && tid == 0) g_sb_prof[blockIdx.x][4] = globaltimer_ns();
}

static void sb_print_prof(cudaStream_t stream, uint32_t grid) {
    static unsigned long long h[256][24];
    cudaStreamSynchronize(stream);
    cudaMemcpyFromSymbol(h, g_sb_prof, sizeof(h));
    const uint32_t g = grid < 256 ? grid : 256;
    unsigned long long t0 = ~0ull, tend_min = ~0ull, tend_max = 0, e3_max = 0;
    double setup = 0, first = 0, prune = 0, wait = 0, ends = 0, e3 = 0, ftile = 0;
    for (uint32_t b = 0; b < g; ++b) t0 = h[b][0] < t0 ? h[b][0] : t0;
    unsigned long long start_max = 0;
    for (uint32_t b = 0; b < g; ++b) {
        start_max = h[b][0] - t0 > start_max ? h[b][0] - t0 : start_max;
        setup += (double)(h[b][1] - h[b][0]); first += (double)(h[b][2] - h[b][0]); prune += (double)h[b][5]; wait += (double)h[b][7];
        ends += (double)(h[b][4] - t0); e3 += (double)(h[b][3] - t0); ftile += h[b][6] == ~0ull ? -1.0 : (double)h[b][6];
        tend_min = h[b][4] - t0 < tend_min ? h[b][4] - t0 : tend_min;
        tend_max = h[b][4] - t0 > tend_max ? h[b][4] - t0 : tend_max;
        e3_max = h[b][3] - t0 > e3_max ? h[b][3] - t0 : e3_max;
    }
    double sync_at = 0, emit_at = 0, chunks = 0, emitted = 0;
    for (uint32_t b = 0; b < g; ++b) { sync_at += (double)(h[b][8] - t0); emit_at += (double)(h[b][9] - t0); chunks += (double)h[b][10]; emitted += (double)h[b][11]; }
    double t12 = 0, t13 = 0, t14 = 0;
    for (uint32_t b = 0; b < g; ++b) { t12 += (double)(h[b][12] - t0); t13 += (double)(h[b][13] - t0); t14 += (double)(h[b][14] - t0); }
    fprintf(stderr, "[shadow prof] emission of warp 0: thresholds + prefix +%.1f | staged +%.1f | atomics answered +%.1f\n", t12 / g / 1e3, t13 / g / 1e3, t14 / g / 1e3);
    fprintf(stderr, "[shadow prof] all warps past the loop avg +%.1f | warp 0 emitted avg +%.1f | live chunks per CTA %.1f | entries emitted by warp 0 %.1f\n",
            sync_at / g / 1e3, emit_at / g / 1e3, chunks / g, emitted / g);
    fprintf(stderr, "[shadow prof, %u CTAs] span %.1f us | last CTA start +%.1f | set-up %.1f | first accumulator +%.1f | epilogue done avg +%.1f max +%.1f | "
            "exit min +%.1f avg +%.1f max +%.1f | prune section %.1f us (first at tile %.1f) | accumulator wait %.1f us\n",
            g, tend_max / 1e3, start_max / 1e3, setup / g / 1e3, first / g / 1e3, e3 / g / 1e3, e3_max / 1e3, tend_min / 1e3, ends / g / 1e3,
            tend_max / 1e3, prune / g / 1e3, ftile / g, wait / g / 1e3);
    double split[24] = {};
    for (uint32_t b = 0; b < g; ++b)
        for (int i = 15; i <= 22; ++i) split[i] += (double)h[b][i];
    fprintf(stderr, "[shadow prof] tile loop per CTA (us, epilogue thread 0, %.1f tiles): accumulator wait %.1f | row inputs %.1f | "
            "conversion + keep rule %.1f | shared atomics %.1f | barrier 1 %.1f | prunes %.1f | barrier 2 %.1f | adoption %.1f\n",
            split[15] / g, wait / g / 1e3, split[16] / g / 1e3, split[17] / g / 1e3, split[18] / g / 1e3, split[19] / g / 1e3,
            split[20] / g / 1e3, split[21] / g / 1e3, split[22] / g / 1e3);
}

// The 16-bit / int8 pass needs an image of the rows (a.image): the BF16 shadow or the int8 image of an fp32 shard, or —
// fp16 / bf16 corpora — the rows themselves (no rounding residue on the row side, only the per-row |x|^2 array).
bool shadow_pass_supported(const DeviceInfo &di, const ScanArgs &a) {
    if (di.cc < 90 || a.image.kind == RowImage::NONE || a.image.xnorm2 == nullptr || a.k > 192 || a.dim > FILTER_MAX_DIM || a.dim < 32 || a.n == 0)
        return false;
    if ((reinterpret_cast<uintptr_t>(a.rows) & 15) != 0 || (reinterpret_cast<uintptr_t>(a.image.data) & 15) != 0) return false;
    if (a.dtype == NK_DTYPE_F32) return a.dim % 4 == 0;
    return a.dim % 8 == 0;  // 16-bit rows: 16-byte TMA row stride and 128-bit exact re-scoring loads
}

template <int QT, ptx::Opnd OP, ScanMode M>
static int launch_shadow_pass_t(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, const ShadowPassArgs &sp, uint64_t *launches) {
    using namespace sb;
    const uint32_t esz = OP == ptx::Opnd::S8 ? 1 : 2, kcols = 128 / esz;  // int8 image: 1-byte elements, 128 per swizzle row
    // rows scanned in place have stride dim: the columns past dim read as zero (TMA OOB fill)
    const CUtensorMap *map_rows = tc_cached_map(ws, 4, a.image.data, a.n, a.image.stride, esz, kcols, ROWS, a.image.row_bytes(), a.dtype);
    const CUtensorMap *map_q = tc_cached_map(ws, QT == 64 ? 5 : 6, sp.qbf16, sp.Qpad, sp.dimpad, esz, kcols, QT, (uint64_t)sp.dimpad * esz,
                                             a.dtype);  // rows past Qpad: zero
    if (!map_rows || !map_q) return -1;
    const size_t smem = (size_t)Cfg<QT>::RING_BYTES + sizeof(Shared) + (mode_row_filter(M) ? QT * sizeof(uint64_t) : 0) +
                        (mode_row_window(M) ? QT * sizeof(uint64_t) : 0) + 1024;
    if (smem > di.max_smem_optin) {
        set_error("shadow tensor path needs %zu B shared memory (> %zu)", smem, di.max_smem_optin);
        return -1;
    }
    if (tc_ensure_smem(reinterpret_cast<const void *>(knn_scan_shadow_kernel<QT, OP, M>), di.device_id, smem))
        return -1;
    tc::Params p = pass_params(a, ws, sp);
    p.nslab = sp.dimpad / kcols; p.qa = sp.qa; p.qb = sp.qb; p.xnorm2 = a.image.xnorm2; p.dnorm2 = a.image.dnorm2;
    p.xscale = a.image.xscale; p.qscale = sp.qscale;
    knn_scan_shadow_kernel<QT, OP, M><<<sp.grid, NTHREADS, smem, a.stream>>>(*map_rows, *map_q, p);
    NK_CUDA_OK(cudaGetLastError());
    if (launches) ++*launches;
    if (a.main_launches) ++*a.main_launches;
    if (p.debug & 64) sb_print_prof(a.stream, sp.grid);
    return 0;
}

// One pass at qt = 64 or 128 query columns in the mode a.mode; the dump mode exists at QT = 64 only.
template <ptx::Opnd OP>
static int launch_shadow_pass_op(int qt, const DeviceInfo &di, const ScanArgs &a, Workspace &ws, const ShadowPassArgs &sp, uint64_t *launches) {
    return tc::with_scan_mode(a.mode, [&](auto mode) {
        constexpr ScanMode M = decltype(mode)::value;
        if (qt != 128) return launch_shadow_pass_t<64, OP, M>(di, a, ws, sp, launches);
        if constexpr (!mode_dump(M)) return launch_shadow_pass_t<128, OP, M>(di, a, ws, sp, launches);
        set_error("internal: no 16-bit / int8 kernel for scan mode %d at 128 query columns", (int)M);
        return -1;
    });
}

// the int8 image runs the s8 wgmma form, the BF16 shadow the bf16 one, rows scanned in place the form of their dtype
int launch_shadow_pass(int qt, const DeviceInfo &di, const ScanArgs &a, Workspace &ws, const ShadowPassArgs &sp, uint64_t *launches) {
    if (a.image.kind == RowImage::S8) return launch_shadow_pass_op<ptx::Opnd::S8>(qt, di, a, ws, sp, launches);
    return a.image.kind == RowImage::NATIVE && a.dtype == NK_DTYPE_F16 ? launch_shadow_pass_op<ptx::Opnd::F16>(qt, di, a, ws, sp, launches)
                                                                       : launch_shadow_pass_op<ptx::Opnd::BF16>(qt, di, a, ws, sp, launches);
}

}  // namespace nk
