// kernels.cuh — internal launcher interface between the C-ABI host code and the kernels.
#pragma once
#include <vector>

#include "common.cuh"

namespace nk {

struct DeviceInfo {
    int device_id = 0;
    int num_sms = 132;
    size_t max_smem_optin = 0;
    int cc = 0;
};
int query_device_info(int device_id, DeviceInfo *out);

// Grow-only device scratch of one shard (never freed between searches: no per-query cudaMalloc,
// unlike cuda.Device.Search, cuda_bridge.go:652-663).
struct Workspace {
    uint64_t *cand = nullptr;     size_t cand_bytes = 0;     // [grid][QT][cap] candidate buffers
    uint64_t *partial = nullptr;  size_t partial_bytes = 0;  // [Q][grid][k] per-CTA sorted lists
    uint64_t *keys = nullptr;     size_t keys_bytes = 0;     // [Q][k] merged keys
    uint64_t *below = nullptr;    size_t below_bytes = 0;    // [Q] exclusion bounds of the k > NK_MAX_K passes
    uint64_t *keys2 = nullptr;    size_t keys2_bytes = 0;    // filter mode: shared thresholds gtau[] + list fills gcount[]; big-k: per-pass keys
    float *queries = nullptr;     size_t queries_bytes = 0;  // staged queries (host API)
    uint32_t *out_idx = nullptr;  size_t out_idx_bytes = 0;
    float *out_score = nullptr;   size_t out_score_bytes = 0;
    NkFilter *qfilter = nullptr;  size_t qfilter_bytes = 0;  // staged per-query tag filters (host API, next to the queries)
    float *qaux = nullptr;        size_t qaux_bytes = 0;     // tensor path: split / normalised queries
    float *rownorm = nullptr;     size_t rownorm_bytes = 0;  // tensor path: per-row inverse norms / sq norms
    int *flags = nullptr;   // NK_FLAG_WORDS ints of device status (layout: FLAG_* in scan_tensor_shared.cuh)
    uint32_t *sub_rows = nullptr; size_t sub_rows_bytes = 0;  // nk_score_subset: row ids + gathered rows (no per-call alloc)
    void *sub_gather = nullptr;   size_t sub_gather_bytes = 0;
    void *scratch = nullptr;      size_t scratch_bytes = 0;    // k-means routing / group search scratch
    float *row_thr = nullptr;     size_t row_thr_bytes = 0;    // nk_knn_graph_update: per-row thresholds [n], then keep-mask words
    NkFilter *row_filter = nullptr; size_t row_filter_bytes = 0;  // filtered graph update: each row's own filter [n]
    uint64_t *qtags = nullptr;    size_t qtags_bytes = 0;      // ... and the tags of the reverse scan's queries [Q]
    NkWindow *row_window = nullptr; size_t row_window_bytes = 0;  // windowed graph update: each row's own window [n]
    uint64_t *qvalues = nullptr;  size_t qvalues_bytes = 0;    // ... and the value keys of the reverse scan's queries [Q]
    NkWindow *qwindow = nullptr;  size_t qwindow_bytes = 0;    // staged per-query value windows (host API, next to the filters)
    uint32_t *pair_rows = nullptr; size_t pair_rows_bytes = 0;  // nk_search_pairs_rows: listed-row bits [(n + 31) / 32], then query rows [Q]
    // cached TMA descriptors (tc_cached_map): re-encoded only when the base pointer or shape changes
    struct MapSlot {
        alignas(64) unsigned char bytes[128];
        uint64_t key[6];
        bool valid = false;
    };
    MapSlot maps[8];
    int release();
};
int ws_reserve(void **p, size_t *cur, size_t need);

// What the filter's 16-bit / int8 pass streams in place of a shard's rows (scan_tensor_shadow.cu, DESIGN §2): the BF16
// shadow or the int8 image of an fp32 shard, or the rows of an fp16 / bf16 shard scanned in place.
struct RowImage {
    enum Kind { NONE, BF16, S8, NATIVE };
    Kind kind = NONE;
    const void *data = nullptr;
    uint32_t dimpad = 0;  // columns the scan covers: dim rounded up to one 128-byte swizzle row (64 16-bit / 128 int8 elements)
    uint32_t stride = 0;  // row stride in elements: dimpad, or dim for rows scanned in place (columns past dim read as zero)
    const float *xnorm2 = nullptr;  // per row |x|^2
    const float *dnorm2 = nullptr;  // per row |x - image(x)|^2; nullptr for rows scanned in place (no residue)
    const float *xscale = nullptr;  // int8 only: per row s, x ~ s * int8 row
    RowImage() = default;
    RowImage(Kind k, const void *d, uint32_t dim, const float *x2, const float *d2 = nullptr, const float *xs = nullptr)
        : kind(k), data(d), dimpad(k == S8 ? (dim + 127) / 128 * 128 : (dim + 63) / 64 * 64), stride(k == NATIVE ? dim : dimpad),
          xnorm2(x2), dnorm2(d2), xscale(xs) {}
    uint32_t esz() const { return kind == S8 ? 1 : 2; }
    uint64_t row_bytes() const { return (uint64_t)stride * esz(); }
    // the image of rows [from, ..): the data and the per-row arrays move together
    RowImage window(uint64_t from) const {
        RowImage w = *this;
        if (kind == NONE) return w;
        w.data = static_cast<const char *>(data) + from * row_bytes();
        w.xnorm2 += from;
        if (dnorm2) w.dnorm2 += from;
        if (xscale) w.xscale += from;
        return w;
    }
};

// What a scan keeps and which filters it applies: the 10 kinds of scan.  ScanArgs::mode is set where the pointers it reads
// are attached (ScanArgs::check holds the two together); the tensor-core scan kernels take it as a template argument.
//   KNN, KNN_TAGS           the k best rows per query: running thresholds, shared between CTAs; full buffers are pruned
//   KNN_WINDOW              ... with per-query value windows on top of the tag filters
//   RANGE, RANGE_TAGS       every row that reaches a fixed per-query threshold: full buffers are flushed to the lists
//   RANGE_WINDOW            ... with per-query value windows on top of the tag filters
//   REVERSE, REVERSE_TAGS   the graph update's reverse scan: a range scan whose pairs must also reach their row's threshold (row_thr)
//   REVERSE_RFILT           ... of a filtered graph: the row's own filter (row_filter) must also admit the query's tag (qtags)
//   REVERSE_RWINDOW         ... of a windowed graph: the row's own window (row_window) must also admit the query's value key
//                           (qvalues); a row-filter mode too (the row filters of a graph without filters admit every tag)
//   DUMP                    tests only (scan_filter_dump): a kNN filter pass that also writes every pair's estimate and bound
// The *_TAGS and *_WINDOW modes and the row-filter modes apply per-query tag filters (row_tags, qfilter): a pair takes part
// only if the query admits the row's tag.  The window modes also apply per-query value windows (row_values, qwindow): a pair
// takes part only if the row's value key lies in the query's window.  The range modes (RANGE .. REVERSE_RWINDOW) and the reverse
// modes (REVERSE ..) are contiguous.  The queries' own windows play no part in a reverse scan: mode_window excludes
// REVERSE_RWINDOW.
enum class ScanMode { KNN, KNN_TAGS, KNN_WINDOW, RANGE, RANGE_TAGS, RANGE_WINDOW, REVERSE, REVERSE_TAGS, REVERSE_RFILT, REVERSE_RWINDOW, DUMP };
__host__ __device__ constexpr bool mode_window(ScanMode m) { return m == ScanMode::KNN_WINDOW || m == ScanMode::RANGE_WINDOW; }
__host__ __device__ constexpr bool mode_tags(ScanMode m) {
    return m == ScanMode::KNN_TAGS || m == ScanMode::RANGE_TAGS || m == ScanMode::REVERSE_TAGS || m == ScanMode::REVERSE_RFILT ||
           m == ScanMode::REVERSE_RWINDOW || mode_window(m);
}
__host__ __device__ constexpr bool mode_range(ScanMode m) { return m >= ScanMode::RANGE && m <= ScanMode::REVERSE_RWINDOW; }
__host__ __device__ constexpr bool mode_row_thr(ScanMode m) { return m >= ScanMode::REVERSE && m <= ScanMode::REVERSE_RWINDOW; }
__host__ __device__ constexpr bool mode_row_filter(ScanMode m) { return m == ScanMode::REVERSE_RFILT || m == ScanMode::REVERSE_RWINDOW; }
__host__ __device__ constexpr bool mode_row_window(ScanMode m) { return m == ScanMode::REVERSE_RWINDOW; }
__host__ __device__ constexpr bool mode_dump(ScanMode m) { return m == ScanMode::DUMP; }

struct ScanArgs {
    const void *rows = nullptr;  // [n x dim] row-major, fp32 or fp16
    int dtype = NK_DTYPE_F32;
    uint32_t n = 0;
    uint32_t dim = 0;
    uint64_t row_base = 0;       // global index of row 0
    const float *queries = nullptr;  // device [Q x dim] fp32
    uint32_t Q = 0;
    uint32_t k = 0;              // 1..NK_MAX_K (may exceed n: missing slots are key 0)
    int metric = NK_METRIC_COSINE;
    cudaStream_t stream = nullptr;
    // optional timing of the dominant kernel only (bench roofline): events recorded on `stream` right before the
    // first and right after the last main scan launch (query prep / list merge excluded); *main_launches += count
    cudaEvent_t ev_begin = nullptr, ev_end = nullptr;
    uint64_t *main_launches = nullptr;
    const int *only_if = nullptr;  // CUDA-core scan as a device-side conditional fallback (runs only if *only_if != 0)
    // k > NK_MAX_K is served by repeated passes: pass p only admits keys strictly below below[q] (the last key the
    // previous pass returned for query q); nullptr = no bound.  CUDA-core scan only.
    const uint64_t *below = nullptr;
    // optional row filter (label / tombstone bitmask): bit r (LSB first in 32-bit words) set = local row r takes part;
    // nullptr = every row.  Honoured by every scan kernel.
    const uint32_t *row_mask = nullptr;
    ScanMode mode = ScanMode::KNN;
    // the tag modes (mode_tags): per-query tag filters, row_tags [n] (local rows) and qfilter [Q]; a (row, query) pair takes
    // part only if tag_admits(row_tags[row], qfilter + q).  Unfiltered searches run kernels without the filter code.
    const uint64_t *row_tags = nullptr;
    const NkFilter *qfilter = nullptr;
    RowImage image;  // what the 16-bit / int8 pass streams; kind NONE = no such pass
    // optional fused decode: the final (index, score) arrays [Q x k] are written by the last kernel of the path
    uint32_t *out_idx = nullptr;
    float *out_score = nullptr;
    // caller's score floor in key space (cosine / dot: similarity; euclidean: -distance^2): lower-scoring rows are never
    // returned (VectorIndex.Search minSimilarity, vector_index.go:339-352; queryNodes bestScore >= 0, call_vector.go:243)
    float min_score = -INFINITY;
    // filter paths: do not queue the retry / exact stages; the (host-synchronous) caller inspects the status words and
    // calls scan_tensor_filter_tail only when a stage overflowed
    bool defer_tail = false;
    // the reverse modes (mode_row_thr): key-space threshold per local row [n]; a (row, query) pair is listed only if it
    // reaches both the query's threshold and the row's
    const float *row_thr = nullptr;
    // the row-filter modes (mode_row_filter): row_filter [n] (local rows) and qtags [Q]; a (row, query) pair is also listed only
    // if tag_admits(qtags[q], row_filter + row), the mirror image of row_tags / qfilter
    const NkFilter *row_filter = nullptr;
    const uint64_t *qtags = nullptr;
    // REVERSE_RWINDOW: row_window [n] (local rows) and qvalues [Q]; a (row, query) pair is also listed only if
    // window_admits(qvalues[q], row_window + row), the mirror image of row_values / qwindow
    const NkWindow *row_window = nullptr;
    const uint64_t *qvalues = nullptr;
    // the window modes (mode_window): value key per local row, row_values [n], and window per query, qwindow [Q]; a (row,
    // query) pair takes part only if window_admits(row_values[row], qwindow + q) (and the tag filter admits it)
    const uint64_t *row_values = nullptr;
    const NkWindow *qwindow = nullptr;
    // 0 if a range (else kNN) scan, on the CUDA cores (no reverse modes) or not, serves the mode and exactly the pointers the
    // mode reads are set; else set_error and -1.  No scan accepts DUMP: scan_filter_dump sets it on its own copy.
    int check(bool range, bool cuda_cores) const;
};

// Fused distance + top-k scan on CUDA cores (small Q, any dim / dtype / alignment).
// Writes per-query sorted candidate keys [Q][k] to out_keys (device).
int scan_simt(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, uint64_t *out_keys, uint64_t *launches);

// Tensor-core scans (scan_tensor.cu, scan_tensor_shadow.cu): the exact 3xTF32 scan, and the filter (TF32 over fp32 rows, or
// the 16-bit / int8 pass over a.image) with exact re-scoring.  scan_tensor_filter_tail queues the retry / exact stages a deferred
// (a.defer_tail) filter search skipped.
int scan_tensor(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, uint64_t *out_keys, uint64_t *launches);
bool scan_tensor_supported(const DeviceInfo &di, const ScanArgs &a);
int scan_tensor_filter(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, uint64_t *out_keys, uint64_t *launches);
int scan_tensor_filter_tail(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, uint64_t *out_keys, uint64_t *launches);
bool scan_tensor_filter_supported(const DeviceInfo &di, const ScanArgs &a);
bool shadow_pass_supported(const DeviceInfo &di, const ScanArgs &a);
// Largest d the filters serve: the int8 image's integer accumulation is exact while 127^2 d < 2^31 (DESIGN §3.3).
// scan_tensor_filter_supported also asks that the finish kernel's shared memory fit the device.
constexpr uint32_t FILTER_MAX_DIM = 32768;
// Largest d the exact 3xTF32 scan serves (scan_tensor_supported); above it the exact stage of a filter search, TENSOR and
// AUTO use the CUDA-core scan.
constexpr uint32_t TENSOR_EXACT_MAX_DIM = 12288;
// Tests only: the filters' score estimates and error bounds for every (row, query) pair (nk_debug_filter_dump).
int scan_filter_dump(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, int which, float *est, float *bnd, uint32_t ld, uint64_t *launches);
// fp32 rows [first, first+count) -> bf16 shadow rows (stride dimpad) + |x|^2, |x - bf16(x)|^2
int build_shadow(const float *rows, uint64_t first, uint64_t count, uint32_t dim, uint32_t dimpad, void *shadow, float *xnorm2,
                 float *dnorm2, cudaStream_t stream);
// fp32 rows [first, first+count) -> int8 image rows (stride dimpad bytes, a multiple of 128) + per-row scale s = max|x_i| / 127
// (NaN for a row with a non-finite element), |x|^2 and |x - s q|^2
int build_image_s8(const float *rows, uint64_t first, uint64_t count, uint32_t dim, uint32_t dimpad, void *image, float *xscale,
                   float *xnorm2, float *dnorm2, cudaStream_t stream);
// k-means assignment (assign_tensor.cu).  Both paths list their near-tie rows (device buffers: count, rows [cap], 4
// candidate ids per row, 0xfffffffe = every centroid) and decide them with assign_fixup_kernel's contract arithmetic; the
// list stays readable after the call (nk_debug_assign_ties).  cap >= n.
struct AssignTies {
    uint32_t *count = nullptr, *rows = nullptr, *cand = nullptr;
    uint32_t cap = 0;
};
// One pass of the 16-bit scan with an argmax epilogue.
bool assign_tensor_supported(const DeviceInfo &di, uint32_t dim, uint32_t K, int metric);
int assign_tensor(const DeviceInfo &di, const float *rows, const RowImage &img, uint32_t n, uint32_t dim, const float *centroids_dev, uint32_t K,
                  int metric, AssignTies ties, uint32_t *assign_dev, cudaStream_t stream, uint64_t *launches, void **scratch, size_t *scratch_bytes);
// From a k = min(2, K) search of the rows against the centroids (idx / sc: [n x k], euclidean scores as distances).
int assign_from_search(const DeviceInfo &di, const float *rows, uint32_t n, uint32_t dim, const float *centroids_dev, uint32_t K, int metric,
                       const uint32_t *idx, const float *sc, uint32_t k, AssignTies ties, uint32_t *assign_dev, cudaStream_t stream,
                       uint64_t *launches);

// A shard's fatal status word (FLAG_FATAL) held `flag`: clear the word on `stream` (flags == nullptr: the caller has cleared
// it), set the error message and return -1.
int fatal_overflow(int flag, int *flags, cudaStream_t stream);

// Range search (nk_search_range, range.cu).  State in the shard workspace: ws.keys2 = [range_qa(Q)] order-preserving bits of
// every query's key-space threshold (score floor included), then [range_qa(Q)] list fills; ws.partial = the lists
// [Q][list_cap].  A fill counts every survivor, also those past list_cap.  range_qa mirrors the filter's padded per-query
// arrays (Qpad + tc::QT_BIG), whose shared thresholds and fills sit at the same places.
inline uint32_t range_qa(uint32_t Q) { return (Q + 63) / 64 * 64 + 256; }
// 16-bit / int8 (a.image set) or TF32 filter scan with fixed thresholds: lists hold every pair whose UPPER bound reaches the threshold.
int scan_tensor_range(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, uint32_t list_cap, uint64_t *launches);
// CUDA-core scan: lists hold every pair whose exact score reaches the threshold.
int scan_simt_range(const DeviceInfo &di, const ScanArgs &a, Workspace &ws, uint32_t list_cap, uint64_t *launches);
// One shard's scan (tensor: the filter, else the CUDA-core scan) and exact re-scoring: survivors per query -> counts[Q] (host);
// *list_cap = the list capacity the lists were filled with; *retried = 1 if the scan ran twice.  pair_first (the self-join,
// nk_search_pairs): query q is stored row *pair_first + q (global id) and keeps only rows above it; nullptr = range search.
// incident (nk_search_pairs_rows, tensor-core lists only): query q is stored row qrow[q] (global id, device [Q]); listed (device,
// one bit per row of the shard) marks the rows listed in the call; each listed pair is kept under its lower listed end and
// scored with its lower row as the query.
struct IncidentRows {
    const uint32_t *qrow;
    const uint32_t *listed;
};
int range_scan_shard(const DeviceInfo &di, const ScanArgs &a, bool tensor, const uint32_t *thr_bits, Workspace &ws, uint64_t *launches,
                     int *counts, uint32_t *list_cap, int *retried, const uint64_t *pair_first = nullptr,
                     const IncidentRows *incident = nullptr);
// After range_scan_shard: the shard's survivors, CSR by counts[Q], each query's run sorted -> *keys (host).
int range_sorted_keys(const DeviceInfo &di, Workspace &ws, cudaStream_t stream, uint32_t Q, const int *counts, uint32_t list_cap,
                      std::vector<uint64_t> *keys, uint64_t *launches);

// nk_knn_graph_update's merge: out[i] = the key K(r, j) under which row j ranks in the k-NN list of local row rl[i] of `rows`,
// j = row js_row[i] of the widened fp32 block js (device, [.. x dim]), global id jid[i] (warp_pair_score).
int graph_pair_keys(const void *rows, int dtype, uint32_t dim, int metric, const float *js, const uint32_t *rl, const uint32_t *js_row,
                    const uint32_t *jid, uint32_t n_pairs, uint64_t *out, cudaStream_t stream);

// Merge n_lists sorted (or unsorted) key lists per query into the best k, sorted descending.
// key(list l, query q, slot i) = keys[l*list_stride + q*q_stride + i], i < list_len (0 = k).
// only_if != nullptr: the kernel returns at once unless *only_if != 0 (device-side conditional fallback).
// dec_idx / dec_score != nullptr: also write the decoded (index, score) arrays [Q x k] (fused decode_keys; dec_metric).
int merge_keys(const uint64_t *keys, uint32_t n_lists, size_t list_stride, size_t q_stride, uint32_t Q, uint32_t k,
               uint64_t *out_keys, cudaStream_t stream, const int *only_if = nullptr, uint32_t list_len = 0,
               uint32_t *dec_idx = nullptr, float *dec_score = nullptr, int dec_metric = 0, const uint32_t *wait_flags = nullptr,
               uint32_t wait_epoch = 0, int *wait_err = nullptr);
// keys [Q][k] -> idx/score [Q][k]; euclidean decodes score = sqrt(-s).
int decode_keys(const uint64_t *keys, uint32_t Q, uint32_t k, int metric, uint32_t *out_idx, float *out_score,
                cudaStream_t stream, const int *only_if = nullptr);

// Row utilities (legacy ABI + index maintenance).
int row_norms(const float *rows, float *norms, uint32_t n, uint32_t dim, cudaStream_t s);
int normalize_rows(float *rows, uint32_t n, uint32_t dim, cudaStream_t s);
int row_scores(const float *rows, const float *query, float *scores, uint32_t n, uint32_t dim, int normalized,
               cudaStream_t s);
int topk_scores(const DeviceInfo &di, const float *scores, uint32_t n, uint32_t k, Workspace &ws, uint64_t *out_keys,
                cudaStream_t s, const uint64_t *below = nullptr);
// keys [k] of topk_scores -> (row, scores[row]), and (0, -1e30f) for an empty slot: cuda_topk's output.
int decode_topk_scores(const uint64_t *keys, uint32_t k, const float *scores, uint32_t *out_idx, float *out_score, cudaStream_t s);
// below[q] = keys[q*k + k-1] (the smallest key pass p returned): the exclusion bound of pass p+1.
int update_below(const uint64_t *keys, uint32_t Q, uint32_t k, uint64_t *below, cudaStream_t s);
int fill_uniform(void *out, int dtype, uint64_t n_rows, uint32_t dim, uint64_t seed, uint64_t row_base, cudaStream_t s);
int fill_clustered(void *out, int dtype, uint64_t n_rows, uint32_t dim, uint64_t seed, uint64_t row_base, uint32_t centres, float sigma,
                   int unit, cudaStream_t s);
// |x|^2 of rows [first, first+count) of an fp16 / bf16 corpus -> out[first..]
int row_sqnorms16(const void *rows, int dtype, uint64_t first, uint64_t count, uint32_t dim, float *out, cudaStream_t s);
// best-of-chunks per node (queryNodes): best[group[r]] = max key over the node's rows; top-k over the node keys; decode
// (the query is staged in 4 dim bytes of shared memory: refused only past the device's opt-in limit)
int group_best(const DeviceInfo &di, const void *rows, int dtype, uint64_t n, uint32_t dim, uint64_t row_base, const float *query,
               int metric, const uint32_t *group, const uint32_t *mask, float min_score, unsigned long long *best, cudaStream_t s);
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device) and size (scan_tensor.cu)
int tc_ensure_smem(const void *func, int device, size_t smem);
// Shared memory a launch of func needs besides its dynamic part, counted as `cuobjdump -res-usage` counts it: the static
// shared memory plus the SMEM_RESERVED bytes the system reserves per block (so a fit errs by at most 1 KB on the safe
// side).  smem_fits: dyn + that <= the device's opt-in limit.  Every path whose dynamic shared memory grows with d asks
// here before it admits d, so the planner never promises a launch the device refuses.
constexpr size_t SMEM_RESERVED = 1024;
size_t kernel_static_smem(const void *func);
bool smem_fits(const DeviceInfo &di, const void *func, size_t dyn);
// Before a launch of func with dyn bytes of dynamic shared memory: an error naming `what` and dim if it cannot fit the
// device, else the opt-in wherever static + dynamic pass the 48 KB a launch gets by default.
int ensure_smem(const DeviceInfo &di, const void *func, size_t dyn, const char *what, uint32_t dim);
int topk_keys(const DeviceInfo &di, const unsigned long long *keys, uint32_t n, uint32_t k, Workspace &ws, uint64_t *out_keys,
              cudaStream_t s);
int decode_group_keys(const uint64_t *keys, uint32_t k, int metric, const uint32_t *group, uint64_t row_base, uint32_t *out_group,
                      uint32_t *out_row, float *out_score, cudaStream_t s);
// k-means update step on device (kmeans.go:585-618): fp64 per-cluster sums + member counts (the K x dim means are
// finished on the host); count_changed = |{i : a[i] != b[i]}| accumulated into *changed.
int cluster_sums(const float *rows, uint64_t n, uint32_t dim, const int32_t *assign, uint32_t K, double *sums,
                 unsigned long long *counts, cudaStream_t s);
int count_changed(const int32_t *a, const uint32_t *b, uint64_t n, unsigned long long *changed, cudaStream_t s);
// k-means++ seeding (kmeanspp.cu): the pass of seed c (row c of the shard's [K x dim] seed list `seeds`) over a shard.  c = 0
// sets d2 (and near = 0); c > 0 first computes delta[j] = sq_euclid64(seed c, seed j) for j < c, then lowers d2[i] (near[i]
// = c) where the new distance is strictly smaller; rows the triangle inequality proves unchanged are skipped when `prune`.
// chunk_sum[j] = sequential fp64 sum of d2 over rows [KMPP_CHUNK j, KMPP_CHUNK (j + 1)); *rows_read += rows computed.
constexpr uint32_t KMPP_CHUNK = 256;
int kmeanspp_pass(const DeviceInfo &di, const float *rows, uint64_t n, uint32_t dim, const float *seeds, uint32_t c, double *delta,
                  bool prune, double *d2, uint32_t *near, double *chunk_sum, unsigned long long *rows_read, cudaStream_t stream,
                  uint64_t *launches);
int convert_f32_to_16(const float *src, void *dst, int dtype, size_t n, cudaStream_t s);  // fp16 / bf16, round to nearest even like the host's astype
// out[r] = rows[idx[r]]: in the rows' dtype, or (out_f32) widened exactly to fp32
int gather_rows(const void *rows, int dtype, uint32_t dim, const uint32_t *idx, uint32_t n_idx, void *out, bool out_f32,
                cudaStream_t s);
// Left-row admission of a self-join (nk_search_pairs): out[r] = f if local row idx[r] passes the row mask (nullptr = every
// row) and f admits its tag (tags nullptr = tag 0), else the filter that admits no row (all_of = none_of = ~0).
int row_filters(const uint32_t *idx, uint32_t n_idx, const uint32_t *mask, const uint64_t *tags, NkFilter f, NkFilter *out,
                cudaStream_t s);
// Left-row windows of a windowed self-join (nk_search_pairs_windowed): out[r] = w, narrowed to [v - gap, v + gap] (saturating,
// and never below key 1) where gap != NK_NO_GAP, if local row idx[r] passes the row mask and f, and its value key v (values
// nullptr = key 0) lies in w and, under a band, is not 0; else the window that admits no row (lo = ~0, hi = 0).
int row_windows(const uint32_t *idx, uint32_t n_idx, const uint32_t *mask, const uint64_t *tags, const uint64_t *values, NkFilter f,
                NkWindow w, uint64_t gap, NkWindow *out, cudaStream_t s);

}  // namespace nk
