/*
 * nornic_knn.h — C ABI of libnornic_knn.so, the H100-native brute-force kNN engine that sits behind
 * NornicDB's GPU boundary.
 *
 * Part 1 re-exports, symbol for symbol, the C functions of the cgo preamble in the reference's
 * pkg/gpu/cuda/cuda_bridge.go (lines cited per function) so that file can link this library instead
 * of carrying its own cuBLAS code (INTEGRATION.md shows the two-line change).  Part 2 is the fused,
 * batched API the Go host calls after a one-function change in cuda.Device.Search.
 *
 * Conventions (same as the reference, cuda_bridge.go:20-33,452-453): int returns are 0 = ok, -1 =
 * failure with a message retrievable through cuda_get_last_error() / nk_last_error(); pointer
 * returns are NULL on failure.  Unlike the reference's process-global buffer, the message is
 * thread-local.  Every entry point binds its CUDA device itself (cudaSetDevice per call), so
 * callers may migrate between OS threads (goroutines) freely.  Host pointers are only borrowed for
 * the duration of a call; every host-pointer entry point is synchronous.
 *
 * No torch / C++ types cross this boundary: plain pointers and sizes only.
 */
#ifndef NORNIC_KNN_H
#define NORNIC_KNN_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ======================================================================================
 * Part 1 — legacy ABI (drop-in for the cgo preamble of pkg/gpu/cuda/cuda_bridge.go)
 * ====================================================================================== */

/* cuda_bridge.go:36-40.  Opaque to Go (only ever held as *C.CudaDevice).  The reference's struct
 * carries a cuBLAS handle; this library has no cuBLAS dependency. */
typedef struct CudaDevice CudaDevice;

/* cuda_bridge.go:132-136.  Field layout kept identical (data, size in BYTES, memory_type). */
typedef struct CudaBuffer {
    float *data;
    size_t size;
    int memory_type; /* 0 = device, 1 = pinned host */
} CudaBuffer;

void cuda_set_error(const char *msg);  /* cuda_bridge.go:23 */
const char *cuda_get_last_error(void); /* cuda_bridge.go:27 */
void cuda_clear_error(void);           /* cuda_bridge.go:31 */

int cuda_get_device_count(void);                     /* cuda_bridge.go:42  (-1 on error) */
int cuda_is_available(void);                         /* cuda_bridge.go:52  (1/0) */
CudaDevice *cuda_create_device(int device_id);       /* cuda_bridge.go:56  (NULL on error) */
void cuda_release_device(CudaDevice *dev);           /* cuda_bridge.go:94  (NULL-safe) */
const char *cuda_device_name(int device_id);         /* cuda_bridge.go:102 ("Unknown" on error) */
size_t cuda_device_memory(int device_id);            /* cuda_bridge.go:113 (bytes, 0 on error) */
int cuda_device_compute_capability(int device_id);   /* cuda_bridge.go:122 (major*10+minor; H100 = 90) */

/* cuda_bridge.go:138.  count is in floats; host_data may be NULL (uninitialised buffer); the copy
 * is synchronous.  memory_type 0 = device, 1 = pinned host. */
CudaBuffer *cuda_create_buffer(CudaDevice *dev, float *host_data, size_t count, int memory_type);
void cuda_release_buffer(CudaBuffer *buf);           /* cuda_bridge.go:184 (NULL-safe) */
void *cuda_buffer_data(CudaBuffer *buf);             /* cuda_bridge.go:197 */
size_t cuda_buffer_size(CudaBuffer *buf);            /* cuda_bridge.go:201 */
/* cuda_bridge.go:205.  Copies min(count*4, size) bytes; 0 / -1. */
int cuda_buffer_copy_to_host(CudaBuffer *buf, float *host_data, size_t count);

/* cuda_bridge.go:231.  norms[i] = ||vectors[i]||2.  One kernel (the reference issues n cublasSnrm2 calls).  Like
 * cublasSnrm2 it neither overflows nor underflows in between: a row whose fp32 sum of squares is not finite or below 2^-100
 * is summed again scaled by a power of two, so rows of elements near 1e25 or 1e-30 get a finite, accurate norm.  A NaN
 * element gives NaN, an inf element inf. */
int cuda_compute_norms(CudaDevice *dev, CudaBuffer *vectors, CudaBuffer *norms, unsigned int n, unsigned int dims);
/* cuda_bridge.go:249.  In place; rows with norm <= 1e-10 are left untouched (cuda_bridge.go:267). */
int cuda_normalize_vectors(CudaDevice *dev, CudaBuffer *vectors, unsigned int n, unsigned int dims);
/* cuda_bridge.go:290.  scores[i] = embeddings[i] . query when normalized != 0 (what the reference's
 * sgemv computes for every input, cuda_bridge.go:293-309); when normalized == 0 the true cosine
 * dot/(|e||q|) with 0 for zero vectors (the case the reference leaves as a TODO). */
int cuda_cosine_similarity(CudaDevice *dev, CudaBuffer *embeddings, CudaBuffer *query, CudaBuffer *scores,
                           unsigned int n, unsigned int dims, int normalized);
/* cuda_bridge.go:327.  out_indices/out_scores are HOST arrays of length k; k is clamped to n; result
 * sorted by score descending, ties by lowest index first (the strict '>' forward scan of
 * cuda_bridge.go:356-371).  As in that scan, only scores > -1e30f enter: NaN, -inf and anything at or below -1e30f never
 * do, and slots no score reached are (0, -1e30f).  -0.0 and +0.0 are equal (ties by index); each score is returned with
 * its own bits.  Any n up to 2^32 - 1.  Selection runs on the device; only k pairs cross PCIe. */
int cuda_topk(CudaDevice *dev, CudaBuffer *scores, unsigned int *out_indices, float *out_scores, unsigned int n,
              unsigned int k);

/* ======================================================================================
 * Part 2 — fused batched kNN API (what cuda.Device.Search / gpu.EmbeddingIndex call instead of
 * NewBuffer + CosineSimilarity + TopK; SURVEY.md §8b)
 * ====================================================================================== */

/* Metric enum = vectorspace.DistanceMetric, pkg/vectorspace/registry.go:27-31. */
enum { NK_METRIC_COSINE = 0, NK_METRIC_DOT = 1, NK_METRIC_EUCLIDEAN = 2 };
/* Corpus element type held in HBM.  Queries and scores are always fp32.  fp16 / bf16 corpora (SURVEY.md §8(f)3 "fp16/bf16
 * down-conversion at load") are half the bytes; batches of >= 5 queries scan them IN PLACE on the tensor cores
 * (fp16 or bf16 wgmma operands — no shadow copy, no row-side rounding residue). */
enum { NK_DTYPE_F32 = 0, NK_DTYPE_F16 = 1, NK_DTYPE_BF16 = 2 };
/* Kernel selection for nk_index_set_path (diagnostics / tests); AUTO picks by Q, dim and dtype. */
/* TENSOR = exact 3xTF32 tensor-core scan; TENSOR_FILTER = 1xTF32 prefilter over the fp32 rows with rigorous margins +
 * exact fp32 rescoring (device-side fallback to the exact scan on margin overflow); TENSOR_SHADOW = the same filter
 * streaming a BF16 shadow copy of the shard (half the HBM bytes; built at upload for library-owned fp32 shards unless
 * NK_SHADOW=0, +50% device memory; plus an int8 copy with one scale per row, +25%, a quarter of the fp32 bytes, which
 * serves k <= 16 on large shards), exact fp32 rescoring from the fp32 rows, device-side retry through TENSOR_FILTER
 * and then the exact scan.  All paths return identical index sets.
 * Dimensions each path serves (the shared-memory limits as on an H100, 232 448 B per block):
 *   SIMT           any d up to about 56 800 (the query row and the candidate buffer in shared memory);
 *   TENSOR         fp32, cosine / dot, 32 <= d <= 12288, d % 4 == 0 (its accumulation error grows with d);
 *   TENSOR_FILTER  fp32, 32 <= d <= 32768, d % 4 == 0;
 *   TENSOR_SHADOW  32 <= d <= 32768, d % 4 == 0 for fp32 rows (BF16 shadow or int8 image), d % 8 == 0 for fp16 / bf16;
 *   group search (nk_search_groups) up to about 57 800.
 * A forced path that does not serve the shape fails; AUTO picks among the paths that do, and the filters' exact stage
 * runs on SIMT where TENSOR does not serve.  Past the SIMT limit no path serves d: a search fails with nk_last_error
 * naming d (DESIGN.md §3.5g). */
enum { NK_PATH_AUTO = 0, NK_PATH_SIMT = 1, NK_PATH_TENSOR = 2, NK_PATH_TENSOR_FILTER = 3, NK_PATH_TENSOR_SHADOW = 4 };

/* k up to NK_MAX_K is one fused pass; larger k (the reference accepts any k) is served by ceil(k/NK_MAX_K) passes
 * of the CUDA-core scan, up to NK_MAX_K_TOTAL results per query.  Merging candidate lists (nk_merge_keys_device,
 * nk_comm_exchange_merge, nk_search_sharded_device) is limited to k <= NK_MAX_K. */
#define NK_MAX_K 1024u
#define NK_MAX_K_TOTAL 65536u

typedef struct NkIndex NkIndex;
/* Exchange context of one rank of a row-sharded, one-rank-per-GPU search (see "Row-sharded search" below). */
typedef struct NkComm NkComm;
#define NK_COMM_HANDLE_BYTES 64 /* sizeof(cudaIpcMemHandle_t) */

typedef struct NkStats {
    uint64_t rows;            /* total rows resident */
    uint64_t searches;        /* nk_search* calls */
    uint64_t queries;         /* queries answered */
    uint64_t kernel_launches; /* kernels launched by this index */
    uint64_t bytes_h2d;       /* host->device bytes moved by this index */
    uint64_t bytes_d2h;
    uint64_t bytes_scanned;   /* corpus bytes streamed from HBM by search kernels */
    uint32_t n_devices;
    uint32_t dim;
} NkStats;

const char *nk_last_error(void);
const char *nk_version(void);

/* An index = one row-major [N x dim] corpus, row-sharded by contiguous ranges over n_devices GPUs of
 * this process (shard g holds rows [base_g, base_g + n_g)).  gpu.EmbeddingIndex storage, gpu.go:1224-1260.  Any dim is
 * accepted; which search paths serve it is listed with NK_PATH_* above. */
NkIndex *nk_index_create(const int *device_ids, int n_devices, uint32_t dim, int dtype, int metric);
void nk_index_release(NkIndex *ix); /* NULL-safe */

/* Replace the corpus with n_rows host rows (dtype of the index), split evenly over the devices.
 * Replaces syncToCUDA's NewBuffer + NormalizeVectors (gpu.go:2073-2118): rows are stored RAW; cosine
 * normalisation happens inside the search kernel, so device rows always equal host rows. */
int nk_index_upload(NkIndex *ix, const void *rows_host, uint64_t n_rows);
/* The same from fp32 host rows whatever the dtype of the index: an fp16 index converts on the device while loading
 * (round to nearest even).  Uploads stream through two pinned staging buffers, so pageable or unaligned sources load
 * at the PCIe / host-memcpy rate. */
int nk_index_upload_from_f32(NkIndex *ix, const float *rows_host_f32, uint64_t n_rows);
/* Locate the vectors inside a serialized index (EmbeddingIndex.Serialize, gpu.go:2373-2412: LE [dims u32][count u32]
 * [count x (len u32, id bytes)][count x dims fp32]) so that they can be fed straight to nk_index_upload_from_f32 —
 * the ids are the host language's business.  vec_offset has no alignment guarantee.  0 / -1 ("gpu: invalid
 * serialized data" for blobs shorter than the header, gpu.go:2419-2421). */
int nk_blob_vectors(const void *blob, size_t blob_bytes, uint32_t *dims, uint32_t *count, size_t *vec_offset);
/* Append rows to the last shard without re-uploading the rest (EmbeddingIndex.Add, gpu.go:1378-1434). */
int nk_index_append(NkIndex *ix, const void *rows_host, uint64_t n_rows);
/* Overwrite row `row` (global index) in place (EmbeddingIndex.Add on an existing id, gpu.go:1391-1399). */
int nk_index_update_row(NkIndex *ix, uint64_t row, const void *row_host);
/* Swap-with-last removal (EmbeddingIndex.Remove, gpu.go:1437-1471): row `row` takes the contents of the
 * last row and the corpus shrinks by one. */
int nk_index_remove_swap(NkIndex *ix, uint64_t row);
/* Row filter for subsequent searches — the label / type filter of db.index.vector.queryNodes (call_vector.go:177-193) as
 * a row bitmask, also usable for tombstones: bit r of mask_words (LSB first in 32-bit words, n_bits = rows of the index)
 * set = row r may be returned; k is clamped to the number of set bits.  NULL clears the filter.  Honoured inside every
 * scan kernel (no over-fetch).  upload / append / remove_swap / fill / attach clear it. */
int nk_index_set_row_mask(NkIndex *ix, const uint32_t *mask_words, uint64_t n_bits);
/* Fill the index with n_rows synthetic rows generated ON DEVICE by the counter-based generator shared
 * with the oracle (oracle/knn_oracle.c orc_fill_uniform): U[-1,1), element (r,j) depends only on
 * (seed, r, j).  Used by bench.py and the large-shape tests so 40 GB corpora never cross PCIe. */
int nk_index_fill_uniform(NkIndex *ix, uint64_t n_rows, uint64_t seed);
/* The Gaussian-mixture corpus of SURVEY.md §8(d) ("1000 centres, sigma = 0.1", the shape of cmd/kmeans-test-data's
 * clusters mode, main.go:231-283), generated ON DEVICE: row r = centre[hash(r) % n_centres] + sigma * N(0,1) per element,
 * centres U[-1,1)^dim.  unit_norm != 0 follows the reference tool to the letter (unit-length centres, rows normalised after
 * the noise).  The near-tie stress case of the filter paths; device-only generator — tests read the rows back. */
int nk_index_fill_clustered(NkIndex *ix, uint64_t n_rows, uint64_t seed, uint32_t n_centres, float sigma, int unit_norm);
/* Single-device index only: this process owns rows [row_base, row_base+n) of a larger corpus
 * (multi-process sharding, one rank per GPU).  Emitted indices are global.  Also offsets the synthetic
 * generator so rank g's rows equal rows row_base.. of the global stream. */
int nk_index_set_row_base(NkIndex *ix, uint64_t row_base);
/* Adopt caller-owned device memory as the (single) shard; not freed by nk_index_release.  The rows may still change behind
 * the library's back (the reference normalises its buffer right after creating it, gpu.go:2100-2106), so no BF16 shadow is
 * built until the caller says the rows are final: nk_index_refresh_shadow. */
int nk_index_attach_device_rows(NkIndex *ix, void *rows_dev, uint64_t n_rows);
/* (Re)build the 16-bit image the fast filter path streams (BF16 shadow + norms of fp32 rows; |x|^2 of fp16 / bf16 rows) from
 * the rows as they are NOW.  For attached rows this is what gives the documented drop-in route (INTEGRATION.md step 2) the
 * headline path; call it again whenever the caller rewrites its buffer. */
int nk_index_refresh_shadow(NkIndex *ix);
/* Change the metric of subsequent searches (rows are stored raw and the shadow is metric-independent: nothing is rebuilt). */
int nk_index_set_metric(NkIndex *ix, int metric);
/* Score floor of subsequent searches, evaluated INSIDE the kernels (it seeds every query's running threshold, so it also
 * prunes): cosine / dot — rows scoring below min_score are never returned (VectorIndex.Search minSimilarity,
 * vector_index.go:339-352; queryNodes keeps a node only if bestScore >= 0, call_vector.go:243); euclidean — the value is a
 * MAXIMUM distance.  Queries with fewer than k admissible rows return 0xffffffff / 0 in the unused slots.  -INFINITY
 * (euclidean: +INFINITY or any negative value) clears it. */
int nk_index_set_min_score(NkIndex *ix, float min_score);
int nk_index_set_path(NkIndex *ix, int path);
uint64_t nk_index_rows(const NkIndex *ix);
int nk_index_stats(const NkIndex *ix, NkStats *out);
/* Diagnostics: copies the device status words of shard 0 after synchronising: out[0] = candidate-buffer overflow
 * (always 0 in a correct run), out[1] != 0 if the last filter stage overflowed its margin buffers and the exact kernels
 * queued behind it produced the result, out[2] = bit pattern of max |x|^2 seen by that search, out[3] = 1 if the BF16
 * shadow stage overflowed and the TF32 filter over the fp32 rows re-ran the search. */
int nk_index_debug_flags(NkIndex *ix, int out[4]);
/* Cumulative diagnostics of shard 0: out[0] = filter searches whose first (16-bit) stage overflowed its margin buffers and
 * re-ran through the TF32 filter, out[1] = filter searches that fell through to the exact kernels, out[2] = longest
 * per-query survivor list of the last filter search, out[3] = OR of the overflow reasons seen so far (1 = a margin buffer
 * could not be pruned below its refill mark, 2 = a CTA's emission was cut at its slot count, 8 = non-finite bound).
 * (Retry rate of a corpus = out[0..1] / searches.) */
int nk_index_debug_counters(NkIndex *ix, uint64_t out[4]);
/* Tests only: the raw score estimate and the error bound the filter kernels compare with, for EVERY (row, query) pair of
 * a single-device index: est_host / bnd_host are [rows x Q] floats (row-major, Q <= 64).  which = NK_PATH_TENSOR_FILTER
 * (1xTF32 pass over fp32 rows) or NK_PATH_TENSOR_SHADOW (16-bit pass).  The filters are sound iff |est - exact| <= bnd;
 * tests/test_gpu_error_model.py measures the worst err / bnd ratio against fp64 on adversarial data. */
int nk_debug_filter_dump(NkIndex *ix, const float *queries_host, uint32_t Q, int which, float *est_host, float *bnd_host);
/* Tests only: run nk_index_assign_nearest on a single-device index (from a zero assignment, result discarded) and return
 * how many rows it listed as near-ties, i.e. rows whose centroid the exact fix-up decided rather than the assignment's error
 * bound.  The first min(count, cap) such rows go to rows_out and their 4 candidate ids each to cand_out ([cap x 4]; 0xfffffffe
 * = every centroid, 0xffffffff = no candidate).  Rows not listed were decided by the bound. */
int nk_debug_assign_ties(NkIndex *ix, const float *centroids_host, uint32_t K, int metric, uint32_t *rows_out, uint32_t *cand_out,
                         uint32_t cap);
/* Device-resident searches return before the device has run: this waits for `stream` (and the index's own streams), reads
 * and clears the sticky internal-overflow word nk_search checks on every call, and returns 0 / -1 with that message. */
int nk_index_status(NkIndex *ix, void *stream);
/* Which kernel the last search used: NK_PATH_SIMT / _TENSOR / _TENSOR_FILTER / _TENSOR_SHADOW (-1: null index). */
int nk_index_last_path(const NkIndex *ix);
/* Device-side timing of the dominant kernel (bench.py roofline): when enabled, the main scan launches of
 * every search (CUDA-core or tensor-core scan; query prep and list merge excluded) are bracketed by CUDA
 * events on their stream.  nk_index_scan_time_ms synchronises, returns the summed duration and the number
 * of main scan launches since the last call, and resets the counters. */
int nk_index_enable_timing(NkIndex *ix, int enabled);
int nk_index_scan_time_ms(NkIndex *ix, double *total_ms, uint64_t *scan_launches);
/* Copy n_rows rows starting at global row `row` back to the host (tests / Serialize). */
int nk_index_read_rows(NkIndex *ix, uint64_t row, uint64_t n_rows, void *rows_host);

/* Batched fused search.  queries_host: [Q x dim] fp32.  out_idx/out_score: caller-owned [Q x k]
 * (row stride k).  Returns the number of results per query, min(k, N) (cuda_bridge.go:647-649;
 * 0 for k == 0 or an empty index, cuda_bridge.go:644-646, gpu.go:1540-1542), or -1 on error.
 * Order: cosine/dot — score descending, ties by row index ascending; euclidean — distance ascending,
 * ties by row index ascending, out_score = the distance (callers apply 1/(1+d), similarity.go:152-158).
 * Synchronous: inputs are consumed and outputs complete on return. */
int nk_search(NkIndex *ix, const float *queries_host, uint32_t Q, uint32_t k, uint32_t *out_idx, float *out_score);

/* Same, single-device index, everything device-resident and asynchronous on `stream` (a cudaStream_t,
 * NULL = the index's own stream).  queries_dev [Q x dim] fp32; out_idx_dev/out_score_dev [Q x k].
 * Call order: the calls on one index take effect in the order they are made, on any mix of streams and threads.  A device
 * search still queued on a busy stream sees the rows, mask and tags as they were when it was called, not a later
 * nk_index_update_row / remove_swap / set_row_mask; two device searches on two streams, or a device search and a host
 * search, run one after the other on the device (they share the shard's workspace).  Each shard keeps one event for this:
 * every call makes its stream wait on it and records it again afterwards.  Nothing waits on the host. */
int nk_search_device(NkIndex *ix, const float *queries_dev, uint32_t Q, uint32_t k, uint32_t *out_idx_dev,
                     float *out_score_dev, void *stream);

/* Per-query tag filters: one corpus pass for a batch whose queries carry different label filters (Qdrant SearchBatch with
 * a Filter per request, search.Service Types, one queryNodes label per vector index).
 * Every row carries a 64-bit tag word whose bits the caller assigns (labels, types, collection, keyword values); rows that
 * were never tagged have tag 0.  Each query carries an NkFilter; row r is ADMISSIBLE for the query iff
 *     (tag[r] & all_of) == all_of  &&  (tag[r] & none_of) == 0  &&  (any_of == 0 || (tag[r] & any_of) != 0)
 * (Qdrant's must / must_not / should over bit conditions).  {0,0,0} admits every row, so filtered and unfiltered queries
 * share a batch; all_of = none_of = ~0 admits no row.  The predicate is evaluated inside the scan kernels, before a pair can
 * enter a candidate buffer: results are exact (every returned score re-scored in fp32), with nk_search's order and ties.
 * The index-wide row mask and score floor still apply.  Returns min(k, rows passing the row mask), like nk_search; a query
 * with fewer admissible rows gets 0xffffffff / 0 in its unused slots.  filters == NULL: no filter.
 * Tags live per shard in device memory (8 B per row) and follow the rows: append gives new rows tag 0, update_row keeps the
 * tag, remove_swap moves the last row's tag with its row; upload, upload_from_f32, fill_* and attach_device_rows reset every
 * tag to 0.
 * Not filtered: nk_search_groups, nk_score_subset, nk_search_keys_device, nk_search_sharded_device and the k-means calls.
 * Not windowed (value windows, below): nk_search_groups, nk_score_subset, nk_search_keys_device, nk_search_sharded_device,
 * the exchange calls and the k-means calls (search by stored row, the self-join and the graph calls have windowed forms:
 * nk_search_rows_windowed, nk_search_pairs_windowed, nk_knn_graph_update_windowed, nk_knn_graph_remap_windowed). */
typedef struct NkFilter {
    uint64_t all_of, none_of, any_of;
} NkFilter;
/* Tags of rows [first_row, first_row + n_rows) (global, relative to the index's first row); may span shards. */
int nk_index_set_row_tags(NkIndex *ix, uint64_t first_row, const uint64_t *tags_host, uint64_t n_rows);
/* nk_search with one filter per query (filters_host [Q], NULL = none).  Synchronous, any number of devices. */
int nk_search_filtered(NkIndex *ix, const float *queries_host, const NkFilter *filters_host, uint32_t Q, uint32_t k,
                       uint32_t *out_idx, float *out_score);
/* nk_search_device with one filter per query: filters_dev [Q] device memory (NULL = none) that must stay valid until `stream`
 * has run the search. */
int nk_search_filtered_device(NkIndex *ix, const float *queries_dev, const NkFilter *filters_dev, uint32_t Q, uint32_t k,
                              uint32_t *out_idx_dev, float *out_score_dev, void *stream);

/* Per-query value windows: numeric range conditions (Qdrant Range / DatetimeRange, "the last 7 days", "under a price")
 * evaluated inside the scan, in the same corpus pass as the tag filters.
 * Every row carries one 64-bit VALUE KEY; rows that were never given a value have key 0.  Keys are compared as unsigned
 * integers only: the caller encodes its numbers so that key order is number order (nornicdb_b200.knn.value_keys: int64
 * v ^ 2^63; doubles by their order-preserving bit pattern; key 0 is kept for "no value").  Each query carries an NkWindow;
 * row r is admissible for the query iff  lo <= value[r] <= hi  AND the query's tag filter admits tag[r] (NULL filters: every
 * tag), with the row mask and the score floor as in nk_search_filtered.  {0, ~0} admits every row; lo > hi admits none; a
 * window with lo >= 1 never admits a row without a value.
 * Results, order, ties, padding (0xffffffff / 0), return values and the k clamp: those of nk_search_filtered /
 * nk_search_filtered_device; the range call's size protocol: that of nk_search_range.  windows == NULL: each call IS its
 * counterpart (same kernels, bit-identical output).  Any number of devices, as for the counterparts.
 * Values live per shard in device memory (8 B per row) and follow the rows exactly as tags do: append gives new rows key 0,
 * update_row keeps the key, remove_swap moves the last row's key with its row; upload, upload_from_f32, fill_* and
 * attach_device_rows reset every key to 0. */
typedef struct NkWindow {
    uint64_t lo, hi; /* row r admissible iff lo <= value[r] <= hi (unsigned) */
} NkWindow;
/* Value keys of rows [first_row, first_row + n_rows) (global, relative to the index's first row); may span shards. */
int nk_index_set_row_values(NkIndex *ix, uint64_t first_row, const uint64_t *keys_host, uint64_t n_rows);
/* nk_search_filtered with one value window per query (windows_host [Q], NULL = none; filters_host NULL = no tag filter). */
int nk_search_windowed(NkIndex *ix, const float *queries_host, const NkFilter *filters_host, const NkWindow *windows_host,
                       uint32_t Q, uint32_t k, uint32_t *out_idx, float *out_score);
/* nk_search_filtered_device with one value window per query: windows_dev [Q] device memory (NULL = none) that, like
 * filters_dev, must stay valid until `stream` has run the search. */
int nk_search_windowed_device(NkIndex *ix, const float *queries_dev, const NkFilter *filters_dev, const NkWindow *windows_dev,
                              uint32_t Q, uint32_t k, uint32_t *out_idx_dev, float *out_score_dev, void *stream);

/* ---- Search by stored row ----------------------------------------------------------------------------------------------
 * The k nearest OTHER rows of stored rows ("which nodes are like this node?", FindSimilar, OnStore's related-node search, the
 * k-NN graph of the whole index).  rows_host [Q]: row ids relative to the index's first row (< nk_index_rows; duplicates
 * allowed).  Query q is row rows_host[q] as stored NOW, widened exactly to fp32 for fp16 / bf16 indexes, read on the device
 * that holds it (on a single device only the ids cross PCIe).  Result: the top k, in nk_search's order and ties, of the
 * admissible rows other than rows_host[q] itself: row mask and score floor apply as in nk_search, and a masked-out row may
 * still be a query.  out_idx / out_score: [Q x k] (row stride k), global row ids.  Returns min(k, rows passing the row mask);
 * a query with fewer admissible other rows gets 0xffffffff / 0 in its unused slots.  Any Q, including every row of the index
 * (the k-NN graph): queries run in blocks of 1024, so the device workspace stays bounded; any number of devices.
 * k <= NK_MAX_K_TOTAL - 1.  Out-of-range ids, a null pointer with Q > 0, or a larger k return -1; k == 0, Q == 0 or no
 * admissible row return 0.  Synchronous, and it holds the index lock throughout: a whole-index graph call blocks every
 * other call on the index for its duration.
 * Equals nk_search(the rows read back and widened, k + 1) with the query's own row removed from each list (or, where it is
 * not in the list, the last entry), bit for bit, for the same blocks of 1024 queries. */
int nk_search_rows(NkIndex *ix, const uint32_t *rows_host, uint32_t Q, uint32_t k, uint32_t *out_idx, float *out_score);
/* nk_search_rows with one tag filter per query (filters_host [Q], NULL = none: then nk_search_rows bit for bit), e.g. "the k
 * nearest rows of the same collection".  Query q gets the top k of the rows other than rows_host[q] that filters_host[q]
 * admits (nk_search_filtered's predicate), with the row mask and the score floor as in nk_search_rows.  The query row itself
 * may be inadmissible (masked out, or refused by its own filter).  Return value, padding, blocks of 1024, devices, k limit,
 * locking and refusals: those of nk_search_rows.
 * Equals nk_search_filtered(the rows read back and widened, filters_host, k' = min(k + 1, rows passing the row mask)) with the
 * query's own row removed from each list (or, where it is not in the list, the last entry), bit for bit, for the same blocks
 * of 1024 queries. */
int nk_search_rows_filtered(NkIndex *ix, const uint32_t *rows_host, const NkFilter *filters_host, uint32_t Q, uint32_t k,
                            uint32_t *out_idx, float *out_score);
/* nk_search_rows_filtered with one value window per query (windows_host [Q], NULL = none: then nk_search_rows_filtered bit for
 * bit), e.g. "nodes like this one from the last 7 days".  Query q gets the top k of the rows other than rows_host[q] that
 * filters_host[q] (NULL = every tag) and windows_host[q] admit (nk_search_windowed's predicate), with the row mask and the score
 * floor as in nk_search_rows.  The query row itself may lie outside its own window.  Return value, padding, blocks of 1024,
 * devices, k limit, locking and refusals: those of nk_search_rows.
 * Equals nk_search_windowed(the rows read back and widened, filters_host, windows_host, k' = min(k + 1, rows passing the row
 * mask)) with the query's own row removed from each list (or, where it is not in the list, the last entry), bit for bit, for
 * the same blocks of 1024 queries. */
int nk_search_rows_windowed(NkIndex *ix, const uint32_t *rows_host, const NkFilter *filters_host, const NkWindow *windows_host,
                            uint32_t Q, uint32_t k, uint32_t *out_idx, float *out_score);

/* ---- Range search ------------------------------------------------------------------------------------------------------
 * Every admissible row whose score reaches the query's threshold (Cypher WHERE vector.similarity.* >= t, auto-links above a
 * similarity threshold, near-duplicate checks): no k.  thresholds_host [Q]: cosine / dot a minimum score, euclidean a
 * maximum distance (rows whose returned distance, sqrtf of the fp32 squared distance, is <= t; t < 0 admits none).  filters_host: NULL or [Q] NkFilters
 * (nk_search_filtered).  The row mask and the score floor apply too; where floor and threshold disagree the stricter wins.
 * Row r is returned for query q iff it is admissible and its exact fp32 score (the arithmetic of nk_search) meets the
 * threshold; a NaN or -inf score (euclidean: NaN or infinite distance) never does.
 * Results in CSR layout: query q's are [out_offsets[q], out_offsets[q+1]) of out_idx (global row ids) / out_score
 * (euclidean: the distance), in nk_search's order (score desc / distance asc, ties by row asc).
 * Size protocol (like snprintf): out_offsets [Q+1] and *out_total are always written and exact; if *out_total > capacity
 * nothing else is written and the call returns 0 — allocate *out_total and call again.  Returns 0, or -1 with
 * nk_last_error (NaN threshold, no device memory for the survivors, ...).  Synchronous, any number of devices. */
int nk_search_range(NkIndex *ix, const float *queries_host, const float *thresholds_host, const NkFilter *filters_host,
                    uint32_t Q, uint64_t capacity, uint64_t *out_offsets, uint32_t *out_idx, float *out_score,
                    uint64_t *out_total);
/* nk_search_range with one value window per query (windows_host [Q], NULL = none: then nk_search_range bit for bit). */
int nk_search_range_windowed(NkIndex *ix, const float *queries_host, const float *thresholds_host, const NkFilter *filters_host,
                             const NkWindow *windows_host, uint32_t Q, uint64_t capacity, uint64_t *out_offsets,
                             uint32_t *out_idx, float *out_score, uint64_t *out_total);

/* ---- Similarity self-join ----------------------------------------------------------------------------------------------
 * Every pair of stored rows whose similarity reaches one threshold (near-duplicate detection, threshold auto-linking of a
 * graph, MATCH (a),(b) WHERE vector.similarity.cosine(a.e, b.e) >= t), each unordered pair scanned and returned once.
 * Left rows: the stripe i in [first_row, first_row + n_rows), ids relative to the index's first row as in nk_search_rows;
 * first_row = 0, n_rows = nk_index_rows(ix) is the whole index.  Left row i gets every row j with a higher global id such that
 *   - j is admissible: it passes the row mask and `filter` (one NkFilter, NULL = none, the predicate of nk_search_filtered);
 *   - i itself passes the row mask and `filter` (otherwise i's list is empty);
 *   - the exact fp32 score of row j against the query "row i as stored, widened to fp32" meets `threshold` with the score
 *     floor folded in: the arithmetic and threshold of nk_search_range (cosine / dot a minimum score, euclidean a maximum
 *     distance; a NaN score never qualifies).
 * So every unordered pair {i, j} appears exactly once when the stripe covers both rows: under the lower id, scored with the
 * lower row as the query.
 * Results in CSR layout over the stripe: left row first_row + r owns [out_offsets[r], out_offsets[r+1]) of out_idx (global
 * row ids) / out_score (euclidean: the distance), out_offsets [n_rows + 1], each list in nk_search's order (score desc /
 * distance asc, ties by row asc).
 * Size protocol (nk_search_range's): out_offsets and *out_total are always written and exact; if *out_total > capacity
 * nothing else is written and the call returns 0.  Returns 0, or -1 with nk_last_error for a NaN threshold, a stripe past
 * the end, a null pointer with n_rows > 0 or the exact 3xTF32 path forced.  Any number of devices.  Synchronous, and it holds
 * the index lock throughout, like nk_search_rows.
 * Costs: the result is staged in host memory during the call, 8 B per pair.  A call that overflows `capacity` has done the
 * whole join, and the retry does it again: callers of a whole-index job should work in stripes.
 * Equals, bit for bit, nk_search_range(queries = the stripe's rows read back and widened, thresholds = threshold, filters =
 * filter for every query) with each list cut to the rows above its own query row, and emptied for inadmissible left rows. */
int nk_search_pairs(NkIndex *ix, uint64_t first_row, uint64_t n_rows, float threshold, const NkFilter *filter, uint64_t capacity,
                    uint64_t *out_offsets, uint32_t *out_idx, float *out_score, uint64_t *out_total);
/* nk_search_pairs with value conditions on both sides (near-duplicates within the same hour, auto-links only between rows close
 * in time).  A pair {i, j} is returned iff nk_search_pairs returns it and
 *   - `window` (one NkWindow, NULL = none) admits value[i] and value[j];
 *   - max_gap != NK_NO_GAP (a BAND): value[i] != 0, value[j] != 0 and |value[i] - value[j]| <= max_gap.  max_gap is in key
 *     units, which are value units for int64 and datetime64 (ns) columns encoded by nornicdb_b200.knn.value_keys.
 * Both conditions are symmetric, so each unordered pair still appears once, under its lower id.  Left row i scans with the
 * window [max(lo, value[i] - max_gap, 1), min(hi, value[i] + max_gap)] (saturating; without a band, [lo, hi]), computed on the
 * device that holds it; a left row that fails the row mask, `filter`, `window` or the band's value rule gets the window that
 * admits no row.  The scans run in the windowed range mode, so out-of-window pairs are never staged.
 * Arguments, CSR layout, size protocol, refusals, locking and costs: those of nk_search_pairs.  window == NULL and max_gap ==
 * NK_NO_GAP: nk_search_pairs, bit for bit (same kernels).
 * Equals nk_search_pairs with the out-of-window and out-of-band pairs dropped, bit for bit (scores, order and CSR). */
#define NK_NO_GAP 0xffffffffffffffffull
int nk_search_pairs_windowed(NkIndex *ix, uint64_t first_row, uint64_t n_rows, float threshold, const NkFilter *filter,
                             const NkWindow *window, uint64_t max_gap, uint64_t capacity, uint64_t *out_offsets, uint32_t *out_idx,
                             float *out_score, uint64_t *out_total);

/* ---- k-NN graph update -------------------------------------------------------------------------------------------------
 * Keeps the k-NN graph of nk_search_rows exact across nk_index_append and nk_index_update_row without an O(N^2) rebuild.
 * graph_idx / graph_score: host arrays [nk_index_rows(ix) x k], row stride k.  On entry rows [0, n_old) hold what
 * nk_search_rows(rows 0 .. n_old-1, k) returned before the changes, unused slots 0xffffffff / 0.  Rows [n_old, N) are the
 * rows appended since; changed_rows [n_changed] the old rows rewritten since (ids < n_old, repeats allowed).  On return every
 * row holds, bit for bit, what nk_search_rows(rows 0 .. N-1, k) returns now (order, ties, scores), slots past a list 0xffffffff
 * / 0; *n_lists_changed (nullable) = how many old rows' lists changed.  Ids are global (row_base included), as returned.
 * New and rewritten rows, and the old rows that list a rewritten row, are searched again; every other old row's list only
 * takes in new or rewritten rows that beat its k-th entry, found by one scan of those rows with per-row thresholds.
 * Preconditions (not checked): the metric and the score floor are unchanged since the graph was built, every old row keeps
 * its row-mask bit (nk_index_append clears the mask: set it again), and the graph was built on the graph path — TENSOR_SHADOW
 * or TENSOR_FILTER forced, or under AUTO the 16-bit pass where every live shard has a 16-bit image and the TF32 filter
 * otherwise.  (AUTO runs blocks of <= 4 rows on a shard under 64 MB on the CUDA cores, whose arithmetic differs: build a graph
 * that will be updated with the path set.)  This call runs on that path whatever AUTO would pick.
 * Returns min(k, admissible rows), the entries a list can hold (nk_search_rows' return value), or -1 with nk_last_error,
 * before the arrays are touched, for: the SIMT or 3xTF32 path forced, k == 0 or
 * k > NK_GRAPH_MAX_K, a shape without a filter path, n_old > N, a changed id >= n_old, a graph entry of rows [0, n_old) that is
 * neither an old row nor 0xffffffff, or a null pointer.  nk_index_remove_swap renumbers rows: use nk_knn_graph_remap below.
 * NaN rows: a search block with a NaN query falls through to the exact stage, whose cosine / dot arithmetic differs, so
 * nk_search_rows itself depends on the block there; the guarantee covers the rows of rebuild blocks without a NaN query, and
 * a NaN row's own list holds the right rows with its stage's scores.
 * Synchronous, and it holds the index lock throughout, like nk_search_rows.  It is nk_knn_graph_remap with old rows kept at
 * their ids, changed_rows and rows >= n_old NK_ROW_NEW, done in place. */
#define NK_GRAPH_MAX_K 191u /* nk_search_rows asks the scan for k + 1; the filter paths stop at 192 */
int nk_knn_graph_update(NkIndex *ix, uint32_t k, uint64_t n_old, const uint32_t *changed_rows, uint32_t n_changed,
                        uint32_t *graph_idx, float *graph_score, uint64_t *n_lists_changed);

/* Keeps the same graph exact across any mix of nk_index_append, nk_index_update_row and nk_index_remove_swap (which moves the
 * last row into the removed row's id), given where each current row's contents came from.
 * src_of_row [N], N = nk_index_rows(ix) now: the old row (relative id < n_old) whose contents current row f holds unchanged
 * since the graph was built, or NK_ROW_NEW if f holds contents the old graph never saw (appended, rewritten).  Non-NEW values
 * must be distinct.  Old rows named by no entry are gone (removed, or overwritten by a move or a rewrite).
 * graph_idx_in / graph_score_in [n_old x k]: what nk_search_rows(rows 0 .. n_old-1, k) returned when the graph was built,
 * unused slots 0xffffffff / 0.  graph_idx_out / graph_score_out [N x k], which must not overlap the input: on return,
 * bit for bit, what nk_search_rows(rows 0 .. N-1, k) returns now (order, ties, scores), slots past a list 0xffffffff / 0.
 * *n_lists_changed (nullable) = how many rows f with src_of_row[f] == f got a list that differs from their old one.
 * New and moved rows, and the rows at unchanged ids whose old list holds a gone or moved row (a moved row's tie-break key
 * changes with its id), are searched again; every other row only takes in new or moved rows that beat its k-th entry, found
 * by one scan of those rows with per-row thresholds.
 * Preconditions, return value, NaN caveat and refusals: those of nk_knn_graph_update, with "old rows keep their mask bit"
 * read as "every kept old row has, at its new id, the mask bit it had when the graph was built".  Also refused, before any
 * output is written: a src_of_row value >= n_old other than NK_ROW_NEW, a repeated non-NEW value, a null src_of_row with
 * N > 0, and output arrays that overlap the input.  (n_old may exceed N: rows were removed.) */
#define NK_ROW_NEW 0xffffffffu
int nk_knn_graph_remap(NkIndex *ix, uint32_t k, uint64_t n_old, const uint32_t *src_of_row,
                       const uint32_t *graph_idx_in, const float *graph_score_in,
                       uint32_t *graph_idx_out, float *graph_score_out, uint64_t *n_lists_changed);

/* Filtered k-NN graphs: one graph per collection (or any tag predicate) of a shared index.  filters_host [N], N =
 * nk_index_rows(ix) now: the filter of each current row's list (NULL = none: then nk_knn_graph_update / nk_knn_graph_remap bit
 * for bit).  The graph is what nk_search_rows_filtered(rows 0 .. N-1, filters_host, k) returns: row r's list holds only rows
 * r's filter admits.  On entry the old graph is what nk_search_rows_filtered(rows 0 .. n_old-1, the filters of that time, k)
 * returned.  Arguments, return value, refusals and every other precondition: those of the unfiltered call.
 * One more precondition (not checked): every kept row (nk_knn_graph_update_filtered: an old row not in changed_rows;
 * nk_knn_graph_remap_filtered: src_of_row[f] != NK_ROW_NEW) has the tag and the filter its contents had when the graph was
 * built.  Report a row whose tag or filter changed as new contents, exactly like a rewritten row (a changed row, or
 * NK_ROW_NEW): lists that held it are searched again and every other list is offered it.
 * Each list holds only rows its own filter admits: rows searched again are searched with their own filter, and the scan of
 * new and moved rows also holds each pair (row r, new row c) to r's filter admitting c's tag, inside the scan kernel. */
int nk_knn_graph_update_filtered(NkIndex *ix, uint32_t k, uint64_t n_old, const uint32_t *changed_rows, uint32_t n_changed,
                                 const NkFilter *filters_host, uint32_t *graph_idx, float *graph_score, uint64_t *n_lists_changed);
int nk_knn_graph_remap_filtered(NkIndex *ix, uint32_t k, uint64_t n_old, const uint32_t *src_of_row, const NkFilter *filters_host,
                                const uint32_t *graph_idx_in, const float *graph_score_in, uint32_t *graph_idx_out,
                                float *graph_score_out, uint64_t *n_lists_changed);

/* Windowed k-NN graphs: time-local graphs ("related events in the same week") kept exact across updates.  windows_host [N]:
 * the value window of each current row's list, in current row order (knn.band_windows gives each row its own +-delta band);
 * NULL = none: then the _filtered call bit for bit, running the same kernels.  filters_host [N] as in the _filtered calls
 * (NULL = no tag filter).  The graph is what nk_search_rows_windowed(rows 0 .. N-1, filters_host, windows_host, k) returns,
 * bit for bit (order, ties, scores, padding): row r's list holds only rows whose value key r's window admits.  On entry the
 * old graph is that call's result at the time it was built.  Arguments, return value, refusals, the NaN caveat, locking and
 * every other precondition: those of the unfiltered calls.
 * One more precondition (not checked): every kept row has the tag, value key, filter and window its contents had when the
 * graph was built.  Report a row whose value key or window changed as new contents, exactly like a rewritten row (a changed
 * row, or NK_ROW_NEW).  A band window moves with its row's key, so re-valuing a row is such a report.
 * Rows searched again are searched with their own filter and window, and the scan of new and moved rows also holds each
 * pair (row r, new row c) to r's window admitting c's value key, inside the scan kernel. */
int nk_knn_graph_update_windowed(NkIndex *ix, uint32_t k, uint64_t n_old, const uint32_t *changed_rows, uint32_t n_changed,
                                 const NkFilter *filters_host, const NkWindow *windows_host,
                                 uint32_t *graph_idx, float *graph_score, uint64_t *n_lists_changed);
int nk_knn_graph_remap_windowed(NkIndex *ix, uint32_t k, uint64_t n_old, const uint32_t *src_of_row,
                                const NkFilter *filters_host, const NkWindow *windows_host,
                                const uint32_t *graph_idx_in, const float *graph_score_in,
                                uint32_t *graph_idx_out, float *graph_score_out, uint64_t *n_lists_changed);

/* ---- Self-join kept current --------------------------------------------------------------------------------------------
 * The pairs of the whole-index self-join incident to a set of rows: on a write, every pair the changed rows now form (the
 * edges to create; the edges to delete are those touching the changed or removed rows, which the caller knows).
 * rows_host [n]: distinct relative ids.  Take nk_search_pairs_windowed(first_row = 0, n_rows = nk_index_rows(ix), threshold,
 * filter, window, max_gap) on the graph path, keep its pairs {i, j} with at least one end listed, and group them by that
 * listed end (a pair with both ends listed goes under the lower one): listed row rows_host[r] owns [out_offsets[r],
 * out_offsets[r+1]) of out_idx (global ids of the other ends) / out_score, out_offsets [n + 1].  The result equals that, bit
 * for bit: each score is the join's, with the lower row of the pair as the query (under cosine the two orientations can
 * round differently), and each list is in nk_search's order.  Size protocol: nk_search_pairs'.
 * The call runs on the graph path (nk_knn_graph_update) whatever AUTO would pick: every score is warp_exact_score's, so it
 * equals the join run with TENSOR_SHADOW or TENSOR_FILTER forced (AUTO may run small joins on the CUDA cores).  Each block of
 * 1024 listed rows scans every shard whole: about n / 1024 full-index range scans.
 * Returns 0, or -1 with nk_last_error, before any work, for: a repeated or out-of-range id, a NaN threshold, a null pointer
 * with n > 0, the SIMT or 3xTF32 path forced, or a shape without a filter path.  Synchronous; holds the index lock.
 * nk_search_pairs_rows is the _windowed call with window == NULL and max_gap == NK_NO_GAP. */
int nk_search_pairs_rows(NkIndex *ix, const uint32_t *rows_host, uint32_t n, float threshold, const NkFilter *filter, uint64_t capacity,
                         uint64_t *out_offsets, uint32_t *out_idx, float *out_score, uint64_t *out_total);
int nk_search_pairs_rows_windowed(NkIndex *ix, const uint32_t *rows_host, uint32_t n, float threshold, const NkFilter *filter,
                                  const NkWindow *window, uint64_t max_gap, uint64_t capacity, uint64_t *out_offsets, uint32_t *out_idx,
                                  float *out_score, uint64_t *out_total);

/* Brings a stored self-join up to date after any mix of append, update_row, remove_swap, retags and re-valued rows.
 * src_of_row [N] as for nk_knn_graph_remap: NK_ROW_NEW marks a row appended, rewritten, retagged or re-valued since.
 * old_offsets [n_old + 1] / old_idx / old_score: what nk_search_pairs_windowed over the whole index (rows [0, n_old)) returned
 * with the same threshold, filter, window and max_gap.  out_offsets [N + 1] / out_idx / out_score: on return, bit for bit, what
 * that call over the whole index returns now on the graph path, under nk_search_pairs' size protocol.  *n_dropped (nullable):
 * old pairs with an end that is gone, moved or NK_ROW_NEW; *n_found (nullable): pairs incident to the new and moved rows.
 * Old pairs with both ends kept at their id are carried; every other old pair is dropped (a moved row counts as new: its id
 * decides the orientation and the tie order); nk_search_pairs_rows_windowed of the new and moved rows adds the rest; each
 * owner's list is merged in key space.  The merge is host C++, O(pairs) time and memory.  This is the verification and
 * convenience path: a database that keeps the pairs as edges calls nk_search_pairs_rows_windowed on each write.
 * Preconditions (not checked): the metric and the score floor are unchanged, and every kept row has its mask bit, tag and
 * value key.  Refused before any output is written: those of nk_search_pairs_rows, a src_of_row value >= n_old other than
 * NK_ROW_NEW or repeated, an old entry that is not an old row above its owner, old_offsets not starting at 0 or decreasing. */
int nk_pairs_remap(NkIndex *ix, float threshold, const NkFilter *filter, const NkWindow *window, uint64_t max_gap, uint64_t n_old,
                   const uint32_t *src_of_row, const uint64_t *old_offsets, const uint32_t *old_idx, const float *old_score,
                   uint64_t capacity, uint64_t *out_offsets, uint32_t *out_idx, float *out_score, uint64_t *out_total,
                   uint64_t *n_dropped, uint64_t *n_found);

/* Multi-process sharding (one rank per GPU): emit this shard's sorted candidate list as packed 64-bit
 * keys [Q x k] (order-preserving score bits << 32 | ~row index; larger key = better), to be exchanged
 * (e.g. ncclAllGather of Q*k*8 bytes per rank) and merged with nk_merge_keys_device.  k <= NK_MAX_K_TOTAL: one shard's
 * keys are useful on their own, but only lists of k <= NK_MAX_K can be merged. */
int nk_search_keys_device(NkIndex *ix, const float *queries_dev, uint32_t Q, uint32_t k, uint64_t *out_keys_dev,
                          void *stream);
/* Merge n_lists candidate lists laid out [n_lists][Q][k] into final [Q x k] idx/score on the current
 * device of `device_id`.  metric selects the score decoding (euclidean: distance).  With a stream the call is
 * asynchronous on it (the searches that produced the keys must be ordered before it on that stream); with
 * stream == NULL it synchronises the device first and returns after the merge has completed.  k > NK_MAX_K (the merge
 * width) returns -1 before any work. */
int nk_merge_keys_device(int device_id, const uint64_t *keys_dev, uint32_t n_lists, uint32_t Q, uint32_t k,
                         int metric, uint32_t *out_idx_dev, float *out_score_dev, void *stream);

/* Best-of-chunks per node — the scoring loop of db.index.vector.queryNodes (call_vector.go:177-256) on the device.  Rows are
 * chunk embeddings; group_of_row[r] in [0, n_groups) is the node row r belongs to (host array, one entry per row; NULL
 * clears; cleared by row-count changing mutations like the row mask).  nk_search_groups scores ONE query against every
 * admissible row (row mask = label filter, score floor = "bestScore >= 0"), keeps each node's best chunk with a per-node
 * atomic max (segment-max) and returns the k best nodes: out_group / out_row / out_score [k] = node id, row of its best
 * chunk, that chunk's score (euclidean: distance), ordered by (score desc, row asc).  Returns the number of nodes found.
 * Exact fp32 arithmetic, no over-select loop.  Single-device indexes. */
int nk_index_set_row_groups(NkIndex *ix, const uint32_t *group_of_row, uint64_t n_rows, uint32_t n_groups);
int nk_search_groups(NkIndex *ix, const float *query_host, uint32_t k, uint32_t *out_group, uint32_t *out_row, float *out_score);

/* Row-sharded search, one rank per GPU, exchange BEHIND the ABI (SURVEY.md §8e; the reference has a single DeviceID,
 * gpu.go:218).  Each rank owns rows [row_base, row_base + n) (nk_index_set_row_base).  The only data that crosses GPUs is
 * every rank's Q*k candidate keys, pushed with plain peer stores over NVLink into a small buffer each rank exports through
 * CUDA IPC — no NCCL, no host hop, two launches (csrc/exchange.cu):
 *   c = nk_comm_create(device, rank, world, slot_bytes >= max Q*k*8);  nk_comm_export(c, handle[64]);
 *   (the host exchanges the world handles by any transport);  nk_comm_connect(c, all_handles = world x 64 B in rank order);
 *   nk_search_sharded_device(ix, c, queries_dev, Q, k, out_idx_dev, out_score_dev, stream)  on every rank, same sequence.
 * Ranks living in ONE process (several single-device indexes) use nk_comm_connect_local instead of export / connect.
 * nk_comm_status synchronises the stream and reports a peer that never arrived (the device-side wait is bounded: 2 s).
 * k <= NK_MAX_K (the merge width): a larger k returns -1 before the scan, before the exchange epoch advances and before
 * anything is written to a peer, so every rank's next call works as if the failed one had never been made. */
NkComm *nk_comm_create(int device_id, int rank, int world, size_t slot_bytes);
int nk_comm_export(NkComm *c, void *handle_out);
int nk_comm_connect(NkComm *c, const void *handles);
int nk_comm_connect_local(NkComm **comms, int world);
int nk_comm_status(NkComm *c, void *stream);
void nk_comm_release(NkComm *c);
/* The exchange step alone: keys_dev = this rank's [Q x k] keys (e.g. from nk_search_keys_device, ordered before on
 * `stream`); writes the merged, decoded result. */
int nk_comm_exchange_merge(NkComm *c, const uint64_t *keys_dev, uint32_t Q, uint32_t k, int metric, uint32_t *out_idx_dev,
                           float *out_score_dev, void *stream);
int nk_search_sharded_device(NkIndex *ix, NkComm *comm, const float *queries_dev, uint32_t Q, uint32_t k, uint32_t *out_idx_dev,
                             float *out_score_dev, void *stream);

/* Score an explicit subset of rows (global indices) against one query and return them sorted
 * (EmbeddingIndex.ScoreSubset gpu.go:1552-1616, ClusterIndex.SearchCandidates kmeans.go:839-895).
 * out arrays have length min(k, n_rows_subset) per query; returns that length or -1. */
int nk_score_subset(NkIndex *ix, const float *query_host, const uint32_t *rows_host, uint32_t n_subset, uint32_t k,
                    uint32_t *out_idx, float *out_score);

/* k-means routing on device (pkg/gpu/kmeans.go, SURVEY.md §8(f)4) for fp32 indexes.
 * nk_index_assign_nearest = assignToCentroids (kmeans.go:458-489, metric NK_METRIC_EUCLIDEAN: nearest by squared
 * distance) / assignToCentroidsGPU (kmeans.go:491-546, NK_METRIC_COSINE: highest cosine): the fused scan with the roles
 * swapped — the K centroids (host, [K x dim]) are the corpus, the index's rows are the queries, read in place.
 * assign_io (host, [rows], int32) holds the previous assignment on entry (any value, e.g. 0 as in Go) and the new one
 * on return; *changed (nullable) = how many differ.  The result is exact, on every path (DESIGN §7 item 3):
 *   euclidean: kmeans.go's assignment row for row (squaredEuclidean: fp32 differences, fp64 sums; lowest index on ties);
 *   cosine: the argmax of the fp64 cosine of the fp32 inputs, lowest index among equal scores; a zero row or a zero
 *   centroid scores 0 and NaN never wins.  This equals cosineSimilarityFlat's choice wherever its own fp32 rounding cannot
 *   flip the order, and departs from it where its sqrt32 has not converged (|c|^2 far outside about [1e-4, 1e5]).
 * A row no centroid scores (all NaN) goes to centroid 0.
 * nk_index_cluster_means = updateCentroidsWithBuffer (kmeans.go:585-618): centroids_io (host, [K x dim]) <- float32 of the
 * float64 mean of each cluster's rows; clusters without members keep their value; counts_out (nullable, [K]). */
int nk_index_assign_nearest(NkIndex *ix, const float *centroids_host, uint32_t K, int metric, int32_t *assign_io,
                            uint64_t *changed);
int nk_index_cluster_means(NkIndex *ix, const int32_t *assign_host, uint32_t K, float *centroids_io, uint32_t *counts_out);
/* nk_index_kmeanspp = initCentroidsKMeansPlusPlus (kmeans.go:364-426) over every row of an fp32 index, on the device.
 * The caller owns the randomness: first_row plays rand.Intn(n), u_host [K-1] (each in [0, 1); nullable when K == 1) plays
 * rand.Float64() for seeds 1 .. K-1.  Outputs: seeds_out [K] row ids (relative to the index's first row);
 * centroids_out (nullable) [K x dim] those rows; potential_out (nullable) [K]: the sum of every row's D² after seeds
 * 0..c (the total seed c+1 is drawn from; the last entry is the k-means++ cost); min_d2_out (nullable) [rows]: each
 * row's D² to its nearest seed; *rows_read (nullable): rows whose contents the passes read.  D² is squaredEuclidean
 * bit for bit; seed 0 assigns it (a NaN stays NaN), later seeds lower it only where strictly smaller.  The pick: target
 * = u T, where the weights are summed sequentially in chunks of 256 rows from each shard's first row, and the chunk sums
 * sequentially in row order (P_j inclusive prefixes, T the total); seed = the first row i of the first chunk j with
 * P_j >= target such that P_{j-1} + (the chunk's partial sum up to i) >= target, or the last row if no chunk qualifies
 * (NaN).  This equals kmeans.go's pick except where target lies within the rounding of the running sums, and exactly
 * where every sum is exact; the number of devices enters only through the chunk boundaries.  NK_KMPP_PRUNE=0 (read per
 * call) computes every row of every pass instead of skipping the rows the triangle inequality proves unchanged: same
 * outputs.  The row mask, tags and score floor are ignored.  Synchronous; -1 before any work for a null ix / seeds_out
 * (/ u_host when K > 1), a non-fp32 index, K == 0 or K > rows, first_row >= rows, or any u that is NaN or outside [0, 1). */
int nk_index_kmeanspp(NkIndex *ix, uint32_t K, uint64_t first_row, const double *u_host, uint32_t *seeds_out, float *centroids_out,
                      double *potential_out, double *min_d2_out, uint64_t *rows_read);

/* Synthetic fp32 query block from the shared generator, on the device of a single-device index. */
int nk_fill_uniform_device(int device_id, float *out_dev, uint64_t n_rows, uint32_t dim, uint64_t seed,
                           uint64_t row_base, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NORNIC_KNN_H */
