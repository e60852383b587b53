// scan_tensor_shared.cuh — declarations shared by the tensor-core scan kernels (scan_tensor.cu: TF32 exact / filter over
// the fp32 rows, scan_tensor_shadow.cu: BF16 filter over the shadow corpus) and their common finish step.
#pragma once
#include <cuda.h>

#include "kernels.cuh"

namespace nk {

// Device status words of one shard (Workspace::flags, NK_FLAG_WORDS ints).  filter_prep_kernel clears [1..7] at the start of
// every filter search; [0] is sticky until the host reads it; [8..] are cumulative diagnostics.
enum {
    FLAG_FATAL = 0,       // candidate-buffer overflow (must stay 0)
    FLAG_OVERFLOW = 1,    // a filter stage overflowed its margin buffers / met non-finite bounds -> next stage
    FLAG_MAXXX = 2,       // float bits: max |x|^2 seen
    FLAG_FINISH_CTAS = 3, // filter_finish_kernel: CTAs done (the last one does the stage bookkeeping)
    FLAG_MAX_RA = 4,      // float bits: BF16 max ra
    FLAG_RETRY = 5,       // retry-stage marker (stage 2 runs only if set)
    FLAG_MAX_RB = 6,      // float bits: BF16 max rb
    FLAG_LONGEST = 7,     // longest shared list of this search (diagnostics)
    FLAG_N_RETRY = 8,     // cumulative: searches whose first (BF16) stage overflowed
    FLAG_N_EXACT = 9,     // cumulative: searches that fell through to the exact kernels
    FLAG_OVF_BITS = 10,   // cumulative OR of the overflow reasons seen: 1 margin buffer could not be pruned below prune_at,
                          // 2 emission cut at k_emit, 8 non-finite bound / margin
    NK_FLAG_WORDS = 16
};
namespace tc {
constexpr int THREADS = 384;
constexpr int BK = 32;           // floats per corpus K-slab = one 128-byte swizzle row
constexpr int EPI_THREADS = 256; // the two consumer warpgroups
constexpr int EPI_BAR = 1;       // named barrier of the consumers (2, 3: one per warpgroup)
constexpr int P = 512;           // candidate buffer capacity per (CTA, query) of the TF32 kernels: warp_prune<16>
constexpr int P_SHADOW = 1024;   // ... of the 16-bit kernel (wider margins, 4 query groups at k = 100): warp_prune<32>
constexpr int QT_BIG = 256;      // padding of the per-query arrays (a CTA reads up to 128 entries past the last query)
constexpr float EUC_EPS = 4e-6f;  // fp32 rounding of |x|^2 + |q|^2 in the euclidean upper bound
constexpr float EUC_KEEP = 1.0f - EUC_EPS;

struct Params {
    uint32_t n, dim, nslab;
    uint64_t row_base;
    uint32_t q0, nq, k;       // queries [q0, q0+nq) in this launch; nq <= qgroups * QT
    uint32_t qgroups;         // 1, 2 or 4 query blocks (sibling CTAs b, b+1, ..) share each corpus tile (grid % qgroups == 0)
    uint32_t list_cap;        // filter: entries per query in `partial`
    int metric;
    uint32_t k_emit;          // slots per (CTA, query) in `partial` (k for exact; k + margin room for filter)
    float margin_c;           // filter mode: c in |s_hat - s| <= c |x| |q|
    const float *qnorm;       // filter mode: |q| per query (1 for cosine), padded
    const float *qa, *qb;     // shadow kernel: per-query bound factors |bf16(q)| and |q - bf16(q)| + acc_c |q|
    const float *xnorm2, *dnorm2;  // shadow kernel: per-row |x|^2 and |x - bf16(x)|^2
    uint64_t *cand;           // [grid][QT][P]
    uint32_t qpad_off;        // row of this launch's first query inside the padded query arrays
    uint64_t *partial;        // exact: [Q][grid][k_emit] fixed slots; filter: [Q][grid*k_emit] shared append lists
    uint32_t *gtau;           // filter: [Q] cross-CTA shared threshold (order-preserving bits, atomicMax; 0 = none yet)
    int *gcount;              // filter: [Q] fill of the shared append lists
    int *flags;               // status words, layout in FLAG_* below
    const int *only_if;       // exact fallback: run only if *only_if != 0
    const uint32_t *mask;     // row bitmask (bit set = row takes part) or nullptr
    int debug;                // NK_TC_DEBUG bit 64: clock64 wait-time instrumentation of CTA 0
    int prune_trigger;        // 16-bit pass: early prune trigger override (NK_PRUNE_TRIGGER, 0 = default)
    int presampled;           // filter: gtau[] already holds a sampled lower bound of every query's k-th best score
                              // (filter_prep_kernel): no flood tiles, thresholds are adopted at kernel start
    float min_score;          // filter: caller's score floor (VectorIndex minSimilarity, vector_index.go:339-352): rows
                              // whose upper bound is below it are never buffered (-inf = none)
    float *dump_est, *dump_bnd;  // DUMP kernels only (tests): per (row, query) score estimate and error bound, [n][dump_ld]
    uint32_t dump_ld;
    int op_f16;               // 16-bit kernel: operands are fp16 (an fp16 corpus scanned in place) instead of bf16
};


}  // namespace tc

#ifdef __CUDACC__
// Filter mode: 2 x (largest possible gap between an upper bound and the true score) for rows with |x|^2 <= maxxx.
//   cosine 2c | dot 2c|x||q| | euclidean (on -dist^2) 2(2c|x||q| + eps(|x|^2+|q|^2))
__device__ __forceinline__ float filter_margin2(int metric, float c, float maxxx, float qn) {
    if (metric == NK_METRIC_COSINE) return 2.0f * c;
    const float xq = sqrtf(maxxx) * qn;
    if (metric == NK_METRIC_DOT) return 2.0f * c * xq;
    return 2.0f * (2.0f * c * xq + tc::EUC_EPS * (maxxx + qn * qn));
}
// BF16 filter: bound(row, q) = ra(row) qa[q] + rb(row) qb[q] (+ eps (|x|^2 + |q|^2) for euclidean); margin2 is twice its
// largest value over the rows seen.
__device__ __forceinline__ float bf16_margin2(int metric, float max_ra, float max_rb, float maxxx, float qa, float qb, float qn) {
    float m = 2.0f * fmaf(max_ra, qa, max_rb * qb);
    if (metric == NK_METRIC_EUCLIDEAN) m += 2.0f * tc::EUC_EPS * (maxxx + qn * qn);
    return m;
}
#endif

// 2-D row-major [rows x cols] tensor of 4-byte (fp32) or 2-byte (bf16) elements, box = [box_rows x box_cols] with
// box_cols * elem_bytes == 128 (one swizzle row), 128-byte swizzle, OOB -> 0.
// map_dtype (2-byte elements only): NK_DTYPE_F16 -> fp16 tensor, anything else -> bf16.
int tc_make_map(CUtensorMap *m, const void *base, uint64_t rows, uint32_t cols, uint32_t elem_bytes, uint32_t box_cols,
                uint32_t box_rows, uint64_t row_stride_bytes, int map_dtype = 0);
int tc_ensure_smem(const void *func, int device, size_t smem);
int tc_debug_flags();

// Cached tensor map: cuTensorMapEncodeTiled runs only when (base, shape, box) changed since the last search.
const CUtensorMap *tc_cached_map(Workspace &ws, int slot, const void *base, uint64_t rows, uint32_t cols, uint32_t elem_bytes,
                                 uint32_t box_cols, uint32_t box_rows, uint64_t row_stride_bytes, int map_dtype = 0);
int tc_env_int(const char *name, int dflt);  // getenv once per name (read at first use)

// BF16 shadow filter pass (scan_tensor_shadow.cu): queries [q0, q0+nq), nq <= qgroups * qt, qt = 64 or 128.
struct ShadowPassArgs {
    uint32_t grid, k_emit, dimpad, Qpad, q0, nq, qgroups;
    const void *qbf16;
    const float *qnorm, *qa, *qb;
    int presampled;
    float *dump_est = nullptr, *dump_bnd = nullptr;  // test-only DUMP instantiation
    uint32_t dump_ld = 0;
};
int launch_shadow_pass(int qt, const DeviceInfo &di, const ScanArgs &a, Workspace &ws, const ShadowPassArgs &sp, uint64_t *launches);
bool shadow_pass_supported(const DeviceInfo &di, const ScanArgs &a);
// stand-alone bf16 conversion of a query block (k-means assignment: centroids as "queries")
int bf16_prep_queries(const ScanArgs &a, uint32_t Qpad, uint32_t dimpad, float acc_c, void *qbf16, float *qnorm, float *qa,
                      float *qb, uint64_t *launches);
// fp32 rows [first, first+count) -> bf16 shadow rows (stride dimpad) + |x|^2, |x - bf16(x)|^2
int build_shadow(const float *rows, uint64_t first, uint64_t count, uint32_t dim, uint32_t dimpad, void *shadow, float *xnorm2,
                 float *dnorm2, cudaStream_t stream);

}  // namespace nk
