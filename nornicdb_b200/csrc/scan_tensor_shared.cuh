// scan_tensor_shared.cuh — what the tensor-core scan kernels (scan_tensor.cu: TF32 exact / filter over the fp32 rows,
// scan_tensor_shadow.cu: BF16 filter over the shadow corpus; assign_tensor.cu: k-means assignment) share: parameters,
// set-up, the TMA producer loop and the filter epilogue (keep rule, per-tile prune / publish / adopt, emission fallback).
#pragma once
#include <cuda.h>
#include <type_traits>

#include "kernels.cuh"
#ifdef __CUDACC__
#include "ptx_sm90.cuh"
#endif

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
constexpr int ROWS = 256;        // corpus rows per tile (2 M-tiles of 128)
constexpr int MAX_BSTAGES = 8;   // deepest query-slab ring
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
    const float *xnorm2, *dnorm2;  // shadow kernel: per-row |x|^2 and |x - image(x)|^2
    const float *xscale, *qscale;  // shadow kernel over an int8 image: per-row and per-query scales (image = scale * int8)
    uint64_t *cand;           // [grid][QT][P]
    uint32_t qpad_off;        // row of this launch's first query inside the padded query arrays
    uint64_t *partial;        // exact: [Q][grid][k_emit] fixed slots; filter: [Q][grid*k_emit] shared append lists
    uint32_t *gtau;           // filter: [Q] cross-CTA shared threshold (order-preserving bits, atomicMax; 0 = none yet)
    int *gcount;              // filter: [Q] fill of the shared append lists
    int *flags;               // status words, layout in FLAG_* below
    const int *only_if;       // exact fallback: run only if *only_if != 0
    const uint32_t *mask;     // row bitmask (bit set = row takes part) or nullptr
    int debug;                // NK_TC_DEBUG bit 64: clock64 wait-time instrumentation of CTA 0
    int presampled;           // filter: gtau[] already holds a sampled lower bound of every query's k-th best score
                              // (filter_prep_kernel): no flood tiles, thresholds are adopted at kernel start
    float min_score;          // filter: caller's score floor (VectorIndex minSimilarity, vector_index.go:339-352): rows
                              // whose upper bound is below it are never buffered (-inf = none)
    float *dump_est, *dump_bnd;  // dump mode only (tests): per (row, query) score estimate and error bound, [n][dump_ld]
    uint32_t dump_ld;
    const uint64_t *row_tags; // tag modes only: tag word per local row
    const NkFilter *qfilter;  // tag modes only: filter per query [Q], indexed like gtau (absolute query index)
    const float *row_thr;     // reverse modes only: key-space threshold per local row (the reverse scan of nk_knn_graph_update)
    const NkFilter *row_filter;  // row-filter modes only: the filter of each local row's own k-NN list (filtered graphs)
    const uint64_t *qtags;    // row-filter modes only: tag word per query [Q], indexed like gtau; staged in shared memory per CTA
    const uint64_t *row_values;  // window modes only: value key per local row
    const NkWindow *qwindow;     // window modes only: window per query [Q] (absolute query index; no padding, never read past Q)
    const NkWindow *row_window;  // REVERSE_RWINDOW only: the window of each local row's own k-NN list (windowed graphs)
    const uint64_t *qvalues;     // REVERSE_RWINDOW only: value key per query [Q]; staged in shared memory per CTA past the tags
};

// What one scan launch covers: queries [q0, q0+nq) in `qgroups` query groups over a `grid`-CTA launch.  Both kernels'
// launch arguments extend it; pass_params() turns it into the Params fields they share.
struct PassArgs {
    uint32_t grid, k_emit, Qpad, q0, nq, qgroups;
    const float *qnorm;
    int presampled;
    float *dump_est = nullptr, *dump_bnd = nullptr;  // read under ScanMode::DUMP only (tests)
    uint32_t dump_ld = 0;
    uint32_t list_cap = 0;    // range modes: gtau[] holds fixed thresholds, survivors go to lists of list_cap
};

// Where a scan's run-time mode becomes its kernel's template argument: launch(std::integral_constant<ScanMode, M>{}) for M = m
// (modes tried in order, DUMP last).  The launchers refuse with `if constexpr` the (kernel, mode) pairs that do not exist.
template <ScanMode M = ScanMode::KNN, class Launch> int with_scan_mode(ScanMode m, Launch &&launch) {
    if (m == M) return launch(std::integral_constant<ScanMode, M>{});
    if constexpr (M != ScanMode::DUMP) return with_scan_mode<ScanMode((int)M + 1)>(m, launch);
    set_error("internal: unknown scan mode %d", (int)m);
    return -1;
}

#ifdef __CUDACC__
// mbarriers of the two TMA rings (corpus slabs, query slabs) of a scan kernel; the first member of its shared state.
template <int ASTAGES> struct Rings {
    uint64_t afull[ASTAGES], aempty[ASTAGES];
    uint64_t bfull[MAX_BSTAGES], bempty[MAX_BSTAGES];
    // a stage is free again once every consumer warp has seen its MMAs complete
    __device__ __forceinline__ void init(int bstages) {
        for (int i = 0; i < ASTAGES; ++i) { ptx::mbar_init(&afull[i], 1); ptx::mbar_init(&aempty[i], 8); }
        for (int i = 0; i < bstages; ++i) { ptx::mbar_init(&bfull[i], 1); ptx::mbar_init(&bempty[i], 8); }
        ptx::fence_barrier_init();
    }
};

// Query groups: CTA b serves query block (b % G) over the tile subset (b / G).  The G sibling CTAs stream the SAME
// corpus tiles at the same pace, so a tile crosses HBM once and its other G-1 readers hit the 50 MB L2: large
// batches (Q > 128) stop being bound by re-reading the corpus once per 128 queries.
template <int QT> struct QueryGroup {
    uint32_t sub, sgrid, q0, qpad_off, nq;
    uint64_t a_policy;
    __device__ __forceinline__ explicit QueryGroup(const Params &p) {
        const uint32_t grp = blockIdx.x % p.qgroups;
        sub = blockIdx.x / p.qgroups;
        sgrid = gridDim.x / p.qgroups;
        q0 = p.q0 + grp * QT;
        qpad_off = p.qpad_off + grp * QT;
        nq = p.nq - grp * QT < (uint32_t)QT ? p.nq - grp * QT : (uint32_t)QT;
        a_policy = p.qgroups > 1 ? ptx::CACHE_EVICT_NORMAL : ptx::CACHE_EVICT_FIRST;
    }
};

// One TMA producer warp: for every tile of this CTA (first, first + step, ..), `reps` passes over its nslab K-slabs
// through a STAGES-deep ring.  issue(stage, tile, rep, slab) arms the stage's full barrier and starts the copies (one
// elected lane).  Returns the cycles spent waiting for free stages when prof is set (NK_TC_DEBUG bit 64).
template <int STAGES, class Issue>
__device__ __forceinline__ long long tma_producer(uint64_t *empty, uint32_t first, uint32_t num_tiles, uint32_t step, uint32_t reps,
                                                  uint32_t nslab, bool prof, Issue issue) {
    long long waited = 0;
    uint32_t g = 0;
    for (uint32_t tile = first; tile < num_tiles; tile += step)
        for (uint32_t rep = 0; rep < reps; ++rep)
            for (uint32_t j = 0; j < nslab; ++j, ++g) {
                const uint32_t s = g % STAGES;
                const long long t0 = prof ? clock64() : 0;
                ptx::mbar_wait(&empty[s], ((g / STAGES) & 1) ^ 1);
                if (prof) waited += clock64() - t0;
                if (ptx::elect_one_sync()) issue(s, tile, rep, j);
                __syncwarp();
            }
    return waited;
}

// t raised to a shared threshold word g read earlier (0 = none published yet)
__device__ __forceinline__ float raise_to_shared_tau(uint32_t g, float t) { return g ? fmaxf(t, ord_to_float(g)) : t; }
// t raised to the query's cross-CTA shared threshold, if any CTA has published one
__device__ __forceinline__ float with_shared_tau(const uint32_t *gtau_q, float t) { return raise_to_shared_tau(__ldcg(gtau_q), t); }
// Start threshold of a query: the caller's score floor and, when the prep kernel sampled the shard, a lower bound of the
// query's k-th best score (no flood tiles then).
__device__ __forceinline__ float start_tau(const Params &p, uint32_t q0, uint32_t qi, uint32_t nq) {
    return p.presampled && qi < nq ? with_shared_tau(p.gtau + q0 + qi, p.min_score) : p.min_score;
}
__device__ __forceinline__ bool row_alive(const Params &p, uint32_t row) {
    return row < p.n && (!p.mask || ((__ldg(p.mask + (row >> 5)) >> (row & 31)) & 1u));
}

// Element i of a thread's per-row array for a row index known only at run time: the register file is not indexable, so
// select by compare (an indexed local array would live in local memory).
template <class T, int N> __device__ __forceinline__ T pick_row(const T (&a)[N], uint32_t ri) {
    T v = a[0];
#pragma unroll
    for (int i = 1; i < N; ++i)
        if (ri == (uint32_t)i) v = a[i];
    return v;
}
// Accumulator value of fragment row fr (tile rows rbase + 64 (fr / 2) + 8 (fr % 2)) in column slot jj (query cbase +
// 8 (jj / 2) + jj % 2).
template <int QT> __device__ __forceinline__ float frag_at(const float (&acc)[2][QT / 2], uint32_t fr, int jj) {
    const int i = (jj >> 1) * 4 + (jj & 1);
    return fr == 0 ? acc[0][i] : fr == 1 ? acc[0][i + 2] : fr == 2 ? acc[1][i] : acc[1][i + 2];
}
// ... for a column slot c known only at run time: select by compare.
template <int QT> __device__ __forceinline__ float frag_value(const float (&acc)[2][QT / 2], uint32_t fr, uint32_t c) {
    float v = 0.0f;
#pragma unroll
    for (int jj = 0; jj < QT / 4; ++jj)
        if (c == (uint32_t)jj) v = frag_at<QT>(acc, fr, jj);
    return v;
}

// The filter's keep rule for NR of a thread's 4 accumulator fragment rows: est[ri] is fragment row fr = fr0 + ri = tile row
// rbase + 64 (fr / 2) + 8 (fr % 2) (corpus row row0 + that), QT/4 query columns cbase + 8 (j / 2) + j % 2.  Buffers every
// (row, query) pair whose score estimate can still reach the query's threshold.  The kernel supplies one estimate per row:
// est[ri].upper(v, col) is the UPPER bound of the score from accumulator value v (exact mode: the score itself) given the
// query's inputs col = est[0].col(qi), est.bound(qi) its error bound before the euclidean term (dump mode only), est.mul /
// est.x2 the row's scale and |x|^2.  alive: bit ri set = the row takes part.  The 16-bit / int8 scan passes all 4 rows at
// once (NR = 4); the TF32 kernel, whose register budget is 168 rather than 240, one row at a time (NR = 1).
//   flood (first two tiles without a sampled threshold): every pair is placed directly at slot = tile-local row, in a loop
//   over the rows that is not unrolled: it runs on two tiles of a launch at most and stays out of the hot code.
//   otherwise a compare pass over the columns reads each query's inputs and threshold from shared memory once for all NR
//   rows and builds the masks of pairs worth buffering (NaN passes); the rare pushes run in a small loop that is not
//   unrolled.
// BOUNDED: a NaN estimate is undecidable here, so it is kept as +inf and the exact re-scoring judges; exact mode: -inf.
// M (ScanMode): tag modes: a pair whose query does not admit the row's tag never enters a buffer — else the pruned and
// published thresholds would stop being lower bounds of the FILTERED k-th best score; flood tiles place it as key 0, the
// compare pass loads the row's tag only when some column passed.  Window modes: the same for the row's value key and the
// query's window, loaded and tested after the tag, and only for the columns the tag test kept (so only queries < nq: the
// window array has Q entries, no padding).  The window's query index is summed in 32 bits before the one pointer add: the
// 16-bit / int8 QT=128 instantiations then keep their register budget without spills.  Reverse modes: a pair must also reach the ROW's threshold rthr[ri] and
// (row-filter modes) be admitted by the row's own filter (qtag: the CTA's query tags), loaded only once both thresholds hold;
// REVERSE_RWINDOW: and by the row's own window (qtag[QT + qi]: the CTA's query value keys), loaded only once a column passed the
// filter.  The range modes have no later stage that could drop a pair the window refuses: this is where it is enforced.
template <int QT, int CAP, bool BOUNDED, ScanMode M, int NR, class Est>
__device__ __forceinline__ void keep_fragment_rows(const Params &p, const Est (&est)[NR], const float (&acc)[2][QT / 2], uint32_t fr0,
                                                   uint32_t alive, uint32_t row0, uint32_t rbase, bool flood, uint32_t it, uint32_t cbase,
                                                   uint32_t q0, uint32_t nq, const float *tau, const float *qn, int *cnt, uint64_t *cand,
                                                   const float (&rthr)[NR], const uint64_t *qtag = nullptr) {
    if (mode_dump(M)) {  // tests only: score estimate and error bound per (row, query)
#pragma unroll
        for (uint32_t ri = 0; ri < (uint32_t)NR; ++ri) {
            const uint32_t fr = fr0 + ri, row = row0 + rbase + 64 * (fr >> 1) + 8 * (fr & 1);
            if (row >= p.n) continue;
#pragma unroll
            for (int jj = 0; jj < QT / 4; ++jj) {
                const uint32_t qi = cbase + 8 * (jj >> 1) + (jj & 1);
                if (qi >= nq) continue;
                const float q = qn[qi];
                float e = frag_at<QT>(acc, fr, jj) * est[ri].mul, b = est[ri].bound(qi);
                if (p.metric == NK_METRIC_EUCLIDEAN) { e -= fmaf(q, q, est[ri].x2); b += EUC_EPS * fmaf(q, q, est[ri].x2); }
                p.dump_est[(size_t)row * p.dump_ld + q0 + qi] = e;
                p.dump_bnd[(size_t)row * p.dump_ld + q0 + qi] = b;
            }
        }
    }
    if (flood && it < 2) {
        // Until the first prune (after this CTA's second tile) every threshold is -inf and EVERY (row, query) pair is
        // buffered: no atomics.
#pragma unroll 1
        for (uint32_t r = 0; r < (uint32_t)NR; ++r) {
            const uint32_t ri = NR == 1 ? 0u : r;  // (one row: a constant, so the row's values stay compile-time selected)
            const uint32_t fr = fr0 + ri, rt = rbase + 64 * (fr >> 1) + 8 * (fr & 1), row = row0 + rt;
            const bool live = (alive >> ri) & 1u;
            const Est e = pick_row(est, ri);
            const uint32_t slot = it * ROWS + rt;
            const uint32_t grow = (uint32_t)(p.row_base + row);
            uint32_t admit = ~0u;  // columns whose filter admits the row
            if (mode_tags(M)) {
                admit = 0u;
                if (live) {
                    const uint64_t tag = __ldg(p.row_tags + row);
#pragma unroll 1
                    for (uint32_t c = 0; c < (uint32_t)(QT / 4); ++c) {
                        const uint32_t qi = cbase + 8 * (c >> 1) + (c & 1);
                        if (qi < nq && tag_admits(tag, p.qfilter + q0 + qi) && (!mode_row_filter(M) || tag_admits(qtag[qi], p.row_filter + row)))
                            admit |= 1u << c;
                    }
                }
            }
            if constexpr (mode_window(M)) {
                if (admit) {  // only the columns the tag loop admitted: those are queries < nq, whose windows exist
                    const uint64_t val = __ldg(p.row_values + row);
                    uint32_t chk = admit;
#pragma unroll 1
                    while (chk) {
                        const uint32_t c = (uint32_t)__ffs((int)chk) - 1u;
                        chk &= chk - 1u;
                        if (!window_admits(val, p.qwindow + (q0 + cbase + 8 * (c >> 1) + (c & 1)))) admit &= ~(1u << c);
                    }
                }
            }
            if constexpr (mode_row_window(M)) {
                if (admit) {  // only the columns the tag loop admitted (queries < nq): the row's own window against their keys
                    const NkWindow *rw = p.row_window + row;
                    const uint64_t lo = __ldg(&rw->lo), hi = __ldg(&rw->hi);
                    uint32_t chk = admit;
#pragma unroll 1
                    while (chk) {
                        const uint32_t c = (uint32_t)__ffs((int)chk) - 1u;
                        chk &= chk - 1u;
                        if (!window_admits(qtag[QT + cbase + 8 * (c >> 1) + (c & 1)], lo, hi)) admit &= ~(1u << c);
                    }
                }
            }
#pragma unroll
            for (int jj = 0; jj < QT / 4; ++jj) {
                const uint32_t qi = cbase + 8 * (jj >> 1) + (jj & 1);
                if (qi < nq) {
                    float sc = e.upper(frag_at<QT>(acc, fr, jj), e.col(qi));
                    if (sc != sc) sc = BOUNDED ? INFINITY : -INFINITY;
                    const bool keep = live && sc >= p.min_score && ((admit >> jj) & 1u);
                    cand[(size_t)qi * CAP + slot] = keep ? make_key(sc, grow) : 0ull;  // 0 = empty slot
                }
            }
        }
        return;
    }
    uint32_t pass[NR];
#pragma unroll
    for (int ri = 0; ri < NR; ++ri) pass[ri] = 0u;
#pragma unroll
    for (int jj = 0; jj < QT / 4; ++jj) {
        const uint32_t qi = cbase + 8 * (jj >> 1) + (jj & 1);
        const typename Est::Col col = est[0].col(qi);
        const float t = tau[qi];
#pragma unroll
        for (uint32_t ri = 0; ri < (uint32_t)NR; ++ri) {
            const float s0 = est[ri].upper(frag_at<QT>(acc, fr0 + ri, jj), col);
            const float tr = mode_row_thr(M) ? fmaxf(t, rthr[ri]) : t;
            pass[ri] |= (!(s0 < tr) && qi < nq) ? (1u << jj) : 0u;
        }
    }
    uint32_t any = 0u;
#pragma unroll
    for (uint32_t ri = 0; ri < (uint32_t)NR; ++ri) {
        if (!((alive >> ri) & 1u)) pass[ri] = 0u;
        any |= pass[ri];
    }
    if (!any) return;
#pragma unroll 1
    for (uint32_t r = 0; r < (uint32_t)NR; ++r) {
        const uint32_t ri = NR == 1 ? 0u : r;
        uint32_t ps = pick_row(pass, ri);
        if (!ps) continue;
        const uint32_t fr = fr0 + ri, row = row0 + rbase + 64 * (fr >> 1) + 8 * (fr & 1);
        const Est e = pick_row(est, ri);
        const float rt = mode_row_thr(M) ? pick_row(rthr, ri) : -INFINITY;
        if (mode_tags(M)) {
            const uint64_t tag = __ldg(p.row_tags + row);
            uint32_t chk = ps;
#pragma unroll 1
            while (chk) {
                const uint32_t c = (uint32_t)__ffs((int)chk) - 1u;
                chk &= chk - 1u;
                if (!tag_admits(tag, p.qfilter + q0 + cbase + 8 * (c >> 1) + (c & 1))) ps &= ~(1u << c);
            }
        }
        if constexpr (mode_window(M)) {
            if (ps) {
                const uint64_t val = __ldg(p.row_values + row);
                uint32_t chk = ps;
#pragma unroll 1
                while (chk) {
                    const uint32_t c = (uint32_t)__ffs((int)chk) - 1u;
                    chk &= chk - 1u;
                    if (!window_admits(val, p.qwindow + (q0 + cbase + 8 * (c >> 1) + (c & 1)))) ps &= ~(1u << c);
                }
            }
        }
        if (mode_row_filter(M) && ps) {
            const NkFilter *rf = p.row_filter + row;
            const uint64_t all_of = __ldg(&rf->all_of), none_of = __ldg(&rf->none_of), any_of = __ldg(&rf->any_of);
            uint32_t chk = ps;
#pragma unroll 1
            while (chk) {
                const uint32_t c = (uint32_t)__ffs((int)chk) - 1u;
                chk &= chk - 1u;
                if (!tag_admits(qtag[cbase + 8 * (c >> 1) + (c & 1)], all_of, none_of, any_of)) ps &= ~(1u << c);
            }
            if constexpr (mode_row_window(M)) {
                if (ps) {
                    const NkWindow *rw = p.row_window + row;
                    const uint64_t lo = __ldg(&rw->lo), hi = __ldg(&rw->hi);
                    chk = ps;
#pragma unroll 1
                    while (chk) {
                        const uint32_t c = (uint32_t)__ffs((int)chk) - 1u;
                        chk &= chk - 1u;
                        if (!window_admits(qtag[QT + cbase + 8 * (c >> 1) + (c & 1)], lo, hi)) ps &= ~(1u << c);
                    }
                }
            }
        }
#pragma unroll 1
        while (ps) {
            const uint32_t c = (uint32_t)__ffs((int)ps) - 1u;
            ps &= ps - 1u;
            const uint32_t qi = cbase + 8 * (c >> 1) + (c & 1);
            float sc = e.upper(frag_value<QT>(acc, fr, c), e.col(qi));
            if (sc != sc) sc = BOUNDED ? INFINITY : -INFINITY;
            if (sc >= (mode_row_thr(M) ? fmaxf(tau[qi], rt) : tau[qi])) {
                int pos = atomicAdd(&cnt[qi], 1);
                if (pos < CAP) cand[(size_t)qi * CAP + pos] = make_key(sc, (uint32_t)(p.row_base + row));
                else atomicExch(p.flags + FLAG_FATAL, 1);
            }
        }
    }
}

// End of a tile, after a barrier that makes every push visible: warp w of the consumers prunes queries w, w + 8, .. whose
// buffer holds more than `trigger` entries (never between the two flood tiles: the second one is placed by slot, behind
// the first one's 256 entries).  prune(qi, out, out_len, max_keep, floor_tau, gcount) runs the kernel's warp_prune.
// Filter mode: everything inside the margin must then fit below prune_at, or the next tile could overflow the buffer; and
// the new threshold is published: it is a lower bound on the true global k-th best score, so every CTA may filter with
// the largest one any CTA has found.
template <bool FILTER, class Prune>
__device__ __forceinline__ void prune_tile(const Params &p, uint32_t q0, uint32_t nq, uint32_t ewarp, int lane, const int *cnt,
                                           const float *tau, int trigger, int prune_at, bool between_floods, Prune prune) {
    if (between_floods) return;
    for (uint32_t qi = ewarp; qi < nq; qi += EPI_THREADS / 32)
        if (cnt[qi] > trigger) {
            prune(qi, nullptr, 0, prune_at, FILTER ? with_shared_tau(p.gtau + q0 + qi, p.min_score) : p.min_score, nullptr);
            if (FILTER && lane == 0 && cnt[qi] >= prune_at) atomicOr(p.flags + FLAG_OVERFLOW, 1);
            if (FILTER && lane == 0 && tau[qi] > -INFINITY) atomicMax(p.gtau + q0 + qi, ord_bits(tau[qi]));
        }
}
// After the prunes: adopt the shared thresholds (one L2 read per query per tile), consumer thread etid of EPI_THREADS.
__device__ __forceinline__ void adopt_shared_tau(const Params &p, uint32_t q0, uint32_t nq, uint32_t etid, float *tau) {
    for (uint32_t qi = etid; qi < nq; qi += EPI_THREADS)
        tau[qi] = with_shared_tau(p.gtau + q0 + qi, tau[qi]);
}

// Filter emission of one query by one warp: everything inside this CTA's margin AND above the shared threshold goes to the
// query's shared list.  Few entries (<= k_emit): no local selection, the finish kernel selects globally — append what still
// reaches the current threshold.  Otherwise select with the margin, and flag the exact fallback when the list was cut at
// k_emit while rows inside the margin remained.
template <class Prune>
__device__ __forceinline__ void emit_query(const Params &p, uint32_t q0, uint32_t qi, int lane, const uint64_t *cand, const int *cnt,
                                           const float *tau, Prune prune) {
    const float floor_tau = with_shared_tau(p.gtau + q0 + qi, p.min_score);
    uint64_t *list = p.partial + (size_t)(q0 + qi) * p.list_cap;
    if (cnt[qi] <= (int)p.k_emit) {
        const float t = fmaxf(tau[qi], floor_tau);
        uint64_t thr = t > -INFINITY ? (uint64_t)ord_bits(t) << 32 : 1ull;
        if (thr == 0ull) thr = 1ull;
        warp_emit_above(cand, cnt[qi], thr, lane, list, (int)p.list_cap, p.gcount + q0 + qi);
        return;
    }
    prune(qi, list, (int)p.list_cap, (int)p.k_emit, floor_tau, p.gcount + q0 + qi);
    if (lane == 0 && cnt[qi] >= (int)p.k_emit && (int)p.k_emit > (int)p.k) atomicOr(p.flags + FLAG_OVERFLOW, 2);
    if (lane == 0 && tau[qi] > -INFINITY) atomicMax(p.gtau + q0 + qi, ord_bits(tau[qi]));
}

// Range mode (nk_search_range): the threshold is fixed (gtau[] holds it from the start, presampled), so a buffer is never
// pruned: every key in it reached the threshold when it was pushed, and the buffer goes whole to the query's list and starts
// over.  The list fill counts past list_cap, so a pass whose lists were too short still knows its exact survivor count.
__device__ __forceinline__ void flush_query(const Params &p, uint32_t q0, uint32_t qi, int lane, const uint64_t *cand, int *cnt) {
    warp_emit_above(cand, cnt[qi], 1ull, lane, p.partial + (size_t)(q0 + qi) * p.list_cap, (int)p.list_cap, p.gcount + q0 + qi);
    __syncwarp();
    if (lane == 0) cnt[qi] = 0;
    __syncwarp();
}
// End of a tile in range mode (in place of prune_tile, after the same barrier): warp ewarp of the consumers flushes queries
// ewarp, ewarp + 8, .. whose buffer could overflow during the next tile (a tile pushes at most ROWS keys per query).
template <int CAP>
__device__ __forceinline__ void flush_tile(const Params &p, uint32_t q0, uint32_t nq, uint32_t ewarp, int lane, const uint64_t *cand,
                                           int *cnt) {
    for (uint32_t qi = ewarp; qi < nq; qi += EPI_THREADS / 32)
        if (cnt[qi] > CAP - ROWS) flush_query(p, q0, qi, lane, cand + (size_t)qi * CAP, cnt);
}

__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)::"memory");
    return t;
}
#endif

}  // namespace tc

#ifdef __CUDACC__
// Exact fp32 score of one corpus row against the query staged in shared memory, by one warp: the arithmetic every
// filter path re-scores its survivors with (filter_finish_kernel, range_rescore_kernel) (fp32 FMA, 128-bit loads; fp16 rows are widened exactly).  Returns the key
// score: dot | dot / sqrt(|x|^2 |q|^2) (0 for zero vectors, simd_amd64.go:31-35) | -|x - q|^2; NaN -> -inf.  *xx_out = |x|^2.
__device__ __forceinline__ float warp_exact_score(const void *rows, int dtype, size_t local, uint32_t dim, const float *qs, float qq,
                                                  int metric, int lane, float *xx_out = nullptr) {
    float d = 0.0f, xx = 0.0f;
    const float4 *q4 = reinterpret_cast<const float4 *>(qs);
    auto acc4 = [&](const float4 v, const float4 u) {
        if (metric == NK_METRIC_EUCLIDEAN) {
            float t;
            t = v.x - u.x; d = fmaf(t, t, d);
            t = v.y - u.y; d = fmaf(t, t, d);
            t = v.z - u.z; d = fmaf(t, t, d);
            t = v.w - u.w; d = fmaf(t, t, d);
            xx = fmaf(v.x, v.x, xx); xx = fmaf(v.y, v.y, xx); xx = fmaf(v.z, v.z, xx); xx = fmaf(v.w, v.w, xx);
        } else {
            d = fmaf(v.x, u.x, d); xx = fmaf(v.x, v.x, xx);
            d = fmaf(v.y, u.y, d); xx = fmaf(v.y, v.y, xx);
            d = fmaf(v.z, u.z, d); xx = fmaf(v.z, v.z, xx);
            d = fmaf(v.w, u.w, d); xx = fmaf(v.w, v.w, xx);
        }
    };
    if (dtype == NK_DTYPE_F32) {
        const float4 *x4 = reinterpret_cast<const float4 *>(static_cast<const float *>(rows) + local * dim);
#pragma unroll 8
        for (uint32_t j = lane; j < dim / 4; j += 32) acc4(__ldg(x4 + j), q4[j]);
    } else if (dtype == NK_DTYPE_F16) {  // fp16 rows, dim % 8 == 0: 8 halves per 128-bit load
        const uint4 *x8 = reinterpret_cast<const uint4 *>(static_cast<const __half *>(rows) + local * dim);
#pragma unroll 4
        for (uint32_t j = lane; j < dim / 8; j += 32) {
            const uint4 w = __ldg(x8 + j);
            const float2 f0 = __half22float2(*reinterpret_cast<const __half2 *>(&w.x)), f1 = __half22float2(*reinterpret_cast<const __half2 *>(&w.y));
            const float2 f2 = __half22float2(*reinterpret_cast<const __half2 *>(&w.z)), f3 = __half22float2(*reinterpret_cast<const __half2 *>(&w.w));
            acc4(make_float4(f0.x, f0.y, f1.x, f1.y), q4[2 * j]);
            acc4(make_float4(f2.x, f2.y, f3.x, f3.y), q4[2 * j + 1]);
        }
    } else {  // bf16 rows: widening is a 16-bit shift
        const uint4 *x8 = reinterpret_cast<const uint4 *>(static_cast<const uint16_t *>(rows) + local * dim);
#pragma unroll 4
        for (uint32_t j = lane; j < dim / 8; j += 32) {
            const uint4 w = __ldg(x8 + j);
            acc4(make_float4(__uint_as_float(w.x << 16), __uint_as_float(w.x & 0xffff0000u), __uint_as_float(w.y << 16), __uint_as_float(w.y & 0xffff0000u)), q4[2 * j]);
            acc4(make_float4(__uint_as_float(w.z << 16), __uint_as_float(w.z & 0xffff0000u), __uint_as_float(w.w << 16), __uint_as_float(w.w & 0xffff0000u)), q4[2 * j + 1]);
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        d += __shfl_xor_sync(0xffffffffu, d, o);
        xx += __shfl_xor_sync(0xffffffffu, xx, o);
    }
    float sc = d;
    if (metric == NK_METRIC_EUCLIDEAN) sc = -d;
    else if (metric == NK_METRIC_COSINE) {
        const float den = sqrtf(xx * qq);
        sc = den > 0.0f ? d / den : 0.0f;
    }
    if (sc != sc) sc = -INFINITY;
    if (xx_out) *xx_out = xx;
    return sc;
}

// |x|^2 of a row of `dtype` held widened in fp32 (xs), accumulated as warp_exact_score accumulates a STORED row's: per lane in
// chunks of 4 (fp32) or 8 (16-bit) elements, then the same butterfly.
__device__ __forceinline__ float warp_stored_sqnorm(const float *xs, int dtype, uint32_t dim, int lane) {
    const uint32_t w = dtype == NK_DTYPE_F32 ? 4 : 8;
    float xx = 0.0f;
    for (uint32_t c = lane; c < dim / w; c += 32)
        for (uint32_t e = 0; e < w; ++e) xx = fmaf(xs[c * w + e], xs[c * w + e], xx);
#pragma unroll
    for (int o = 16; o; o >>= 1) xx += __shfl_xor_sync(0xffffffffu, xx, o);
    return xx;
}

// Key score K(r, j) of the k-NN graph, by one warp: the score nk_search_rows gives stored row j in the list of query = stored
// row r, whichever of the two is at hand as the widened fp32 copy.  js = row j widened (any memory), jj = its
// warp_stored_sqnorm; r = local row of `rows`, read here.  The dot product or squared difference accumulates the same
// products in the same order whichever row warp_exact_score stages as the query (fmaf is commutative in its factors); for
// cosine the norms are not symmetric: |j|^2 is a stored row's (jj) and |r|^2 a query's, lane-strided as filter_finish_kernel
// accumulates it.  (warp_exact_score in dot mode returns the raw product with NaN -> -inf, which leaves the cosine quotient's
// result unchanged: NaN / den and -inf / den both end at -inf.)
__device__ __forceinline__ float warp_pair_score(const void *rows, int dtype, size_t r, uint32_t dim, const float *js, float jj,
                                                 int metric, int lane) {
    const float d = warp_exact_score(rows, dtype, r, dim, js, 1.0f, metric == NK_METRIC_EUCLIDEAN ? metric : NK_METRIC_DOT, lane);
    if (metric != NK_METRIC_COSINE) return d;
    float rr = 0.0f;
    for (uint32_t j = lane; j < dim; j += 32) {
        float x;
        if (dtype == NK_DTYPE_F32) x = __ldg(static_cast<const float *>(rows) + r * dim + j);
        else if (dtype == NK_DTYPE_F16) x = __half2float(static_cast<const __half *>(rows)[r * dim + j]);
        else x = __uint_as_float((uint32_t)static_cast<const uint16_t *>(rows)[r * dim + j] << 16);
        rr = fmaf(x, x, rr);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) rr += __shfl_xor_sync(0xffffffffu, rr, o);
    const float den = sqrtf(jj * rr);
    float sc = den > 0.0f ? d / den : 0.0f;
    if (sc != sc) sc = -INFINITY;
    return sc;
}

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

// 2-D row-major [rows x cols] tensor of 4-byte (fp32), 2-byte (bf16) or 1-byte (int8) elements, box = [box_rows x box_cols]
// with box_cols * elem_bytes == 128 (one swizzle row), 128-byte swizzle, OOB -> 0.
// map_dtype (2-byte elements only): NK_DTYPE_F16 -> fp16 tensor, anything else -> bf16.
int tc_make_map(CUtensorMap *m, const void *base, uint64_t rows, uint32_t cols, uint32_t elem_bytes, uint32_t box_cols,
                uint32_t box_rows, uint64_t row_stride_bytes, int map_dtype = 0);
int tc_debug_flags();

// Cached tensor map: cuTensorMapEncodeTiled runs only when (base, shape, box) changed since the last search.
const CUtensorMap *tc_cached_map(Workspace &ws, int slot, const void *base, uint64_t rows, uint32_t cols, uint32_t elem_bytes,
                                 uint32_t box_cols, uint32_t box_rows, uint64_t row_stride_bytes, int map_dtype = 0);
int tc_env_int(const char *name, int dflt);  // getenv once per name (read at first use)

// The Params fields every scan launch fills the same way (scan_tensor.cu)
tc::Params pass_params(const ScanArgs &a, Workspace &ws, const tc::PassArgs &t);

// Filter pass over a row image (scan_tensor_shadow.cu): queries [q0, q0+nq), nq <= qgroups * qt, qt = 64 or 128.  qbf16:
// the queries in the image's element type (int8 images: int8, with the per-query scales qscale).
struct ShadowPassArgs : tc::PassArgs {
    uint32_t dimpad;
    const void *qbf16;
    const float *qa, *qb, *qscale;
};
int launch_shadow_pass(int qt, const DeviceInfo &di, const ScanArgs &a, Workspace &ws, const ShadowPassArgs &sp, uint64_t *launches);

// Query preparation (filter_prep_kernel, scan_tensor.cu), one CTA per padded query row.
struct PrepParams {
    const float *q;
    uint32_t Q, dim, dimpad;
    int normalise, metric;
    float acc_c;
    float *qhi, *qlo;      // [Qpad x dim] (nullable)
    uint16_t *qbf;         // [Qpad x dimpad] (nullable); fp16 bits when qbf_f16
    int qbf_f16;
    int8_t *qs8;           // [Qpad x dimpad] int8 image q = qscale * qs8 (nullable; exclusive with qbf)
    float *qscale;         // [Qpad] with qs8
    float *qnorm, *qa, *qb;
    uint32_t *state;       // gtau[QA] then gcount[QA] (nullable)
    uint32_t Qpad, QA;
    int *flags;
    // sampled initial threshold (sample == 0: none)
    const void *rows;
    int dtype;
    uint32_t n, sample, k;
    const uint32_t *mask;
    float min_score;
    const int *only_if;
    const uint64_t *row_tags;  // the tag modes' filters: the sample counts admissible rows only
    const NkFilter *qfilter;
    const uint64_t *row_values;  // ... and the window modes' windows
    const NkWindow *qwindow;
};
// The fields taken from the search arguments: the queries, the metric and the shard (for the sample).
PrepParams prep_params(const ScanArgs &a, uint32_t Qpad, uint32_t dimpad);
// The tag and window modes run the instantiations whose sample counts only the rows each query admits.
int launch_prep(const DeviceInfo &di, ScanMode mode, const PrepParams &pp, cudaStream_t stream, uint64_t *launches);

}  // namespace nk
