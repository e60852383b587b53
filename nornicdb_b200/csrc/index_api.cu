// index_api.cu — the fused batched kNN API (Part 2 of include/nornic_knn.h).
//
// NkIndex is the device-side half of gpu.EmbeddingIndex (pkg/gpu/gpu.go:1224-1260): a flat row-major
// [N x dim] corpus resident in HBM, row-sharded by contiguous ranges over the GPUs of this process.
// nk_search replaces cuda.Device.Search (pkg/gpu/cuda/cuda_bridge.go:643-686: NewBuffer + NewEmptyBuffer
// + CosineSimilarity + TopK, with a cudaMalloc/cudaFree pair and an n-float D2H per query) by one
// fused scan per shard + a candidate merge; nothing is allocated per query and only Q*k results leave
// the device.
#include <algorithm>
#include <functional>
#include <map>
#include <mutex>
#include <stdlib.h>
#include <string.h>
#include <thread>
#include <vector>

#include "kernels.cuh"
#include "scan_tensor_shared.cuh"

// The images of a shard that the filter scans instead of its rows (nk::RowImage, shard_image): the BF16 shadow (+ |x -
// bf16(x)|^2 per row) and the int8 image (+ per-row scale s and |x - s xq|^2) of an owned fp32 shard, either or both; a
// 16-bit shard (fp16 / bf16) is scanned in place and only carries |x|^2, which all images share.  Rows [0, n) are
// converted; capacity in rows.
struct ShardImages {
    void *bf16 = nullptr, *s8 = nullptr;
    float *xnorm2 = nullptr, *bf16_dnorm2 = nullptr, *s8_dnorm2 = nullptr, *s8_scale = nullptr;
    uint64_t cap = 0, n = 0;
    bool attached = false;  // caller-owned rows: images built on request (nk_index_refresh_shadow)
    // The int8 image is dropped from the kNN filter of this shard once a search on it overflowed its margin buffers (a
    // near-tie-heavy corpus: its ~3x wider margins send such searches to the slower retry stages).  The overflow counters
    // are copied to pinned memory behind every int8 search and read, without waiting, when the next search is planned.
    mutable bool s8_off = false;
    mutable cudaEvent_t s8_ev = nullptr;
    mutable int *s8_h = nullptr;      // pinned: FLAG_N_RETRY, FLAG_N_EXACT after the last int8 search
    mutable int64_t s8_seen = 0;      // their sum when last read
    nk::RowImage bf16_image(uint32_t dim) const { return nk::RowImage(nk::RowImage::BF16, bf16, dim, xnorm2, bf16_dnorm2); }
    nk::RowImage s8_image(uint32_t dim) const { return nk::RowImage(nk::RowImage::S8, s8, dim, xnorm2, s8_dnorm2, s8_scale); }
    bool current(uint64_t rows) const { return xnorm2 && n == rows; }  // are all `rows` rows converted?
    // Free the int8 image alone (s8_only) or every buffer.  The overflow watch stays: a shard that left the int8 image stays off it.
    void release(bool s8_only = false) {
        cudaFree(s8); cudaFree(s8_scale); cudaFree(s8_dnorm2);
        s8 = nullptr; s8_scale = s8_dnorm2 = nullptr;
        if (s8_only) return;
        cudaFree(bf16); cudaFree(bf16_dnorm2); cudaFree(xnorm2);
        bf16 = nullptr; bf16_dnorm2 = xnorm2 = nullptr;
        cap = n = 0;
    }
};

struct NkShard {
    int device = 0;
    nk::DeviceInfo di;
    cudaStream_t stream = nullptr;
    cudaEvent_t last = nullptr;  // the end of the last work any call queued on this shard, on whichever stream (ShardOrder)
    void *rows = nullptr;
    bool owns = true;
    uint64_t n = 0, cap = 0, base = 0;
    ShardImages img;
    uint32_t *group = nullptr;  // node id per row (nk_index_set_row_groups), local rows
    size_t group_bytes = 0;
    bool group_on = false;
    nk::Workspace ws;
    uint64_t *h_keys = nullptr;  // pinned staging for multi-shard host merge
    size_t h_keys_bytes = 0;
    unsigned char *h_res = nullptr;  // pinned staging of a single-shard result: [idx][score][status words] in ONE sync
    size_t h_res_bytes = 0;
    // cold-start feed: two pinned staging buffers + their "copy drained" events (stream_h2d)
    void *stage[2] = {nullptr, nullptr};
    cudaEvent_t stage_ev[2] = {nullptr, nullptr};
    void *cvt = nullptr;  // device scratch for fp32 -> fp16 conversion at load
    uint32_t *mask = nullptr;  // optional row filter (nk_index_set_row_mask): bit = local row
    size_t mask_bytes = 0;
    bool mask_on = false;
    // tag word per local row (nk_index_set_row_tags), grow-only; tags_on = false: every tag is 0 and the array may be stale
    uint64_t *tags = nullptr;
    uint64_t tags_cap = 0;
    bool tags_on = false;
    // value key per local row (nk_index_set_row_values), kept exactly like the tags; values_on = false: every key is 0
    uint64_t *values = nullptr;
    uint64_t values_cap = 0;
    bool values_on = false;
    size_t cvt_bytes = 0;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> timing;  // pending scan-kernel event pairs
    std::vector<uint64_t> timing_launches;
};

struct NkIndex {
    uint32_t dim = 0;
    int dtype = NK_DTYPE_F32;
    int metric = NK_METRIC_COSINE;
    int path = NK_PATH_AUTO;
    // The image kinds shards keep (bit 1 << nk::RowImage::Kind), NK_SHADOW at creation: unset / 1 both the BF16 shadow (+50%
    // HBM) and the int8 image (+25%; the int8 image alone is dropped when its memory cannot be had) of fp32 shards, bf16 the
    // BF16 shadow only, int8 the int8 image only; 16-bit shards are scanned in place unless NK_SHADOW is 0, which keeps none
    unsigned images = 1u << nk::RowImage::BF16 | 1u << nk::RowImage::S8 | 1u << nk::RowImage::NATIVE;
    bool keeps(nk::RowImage::Kind k) const { return images >> k & 1u; }
    bool timing_on = false;
    int last_path = NK_PATH_SIMT;
    uint64_t row_base = 0;
    std::vector<NkShard> shards;
    uint64_t mask_alive = 0;  // rows that pass the row mask (all shards); meaningful while a mask is set
    bool mask_on = false;
    float min_score = -INFINITY;  // score floor of subsequent searches, in the API's score domain (nk_index_set_min_score)
    uint32_t n_groups = 0;        // nk_index_set_row_groups
    float *h_qrows = nullptr;     // pinned: a block of nk_search_rows queries assembled from several shards, + gather staging
    size_t h_qrows_bytes = 0;
    NkStats stats{};
    std::mutex mu;
    size_t esz() const { return dtype == NK_DTYPE_F32 ? 4 : 2; }
    // the floor in key space: euclidean keys are -distance^2 and the API's floor is a maximum distance
    float key_floor() const {
        if (metric == NK_METRIC_EUCLIDEAN) return (min_score >= 0.0f && min_score < INFINITY) ? -(min_score * min_score) : -INFINITY;
        return min_score > -INFINITY ? min_score : -INFINITY;
    }
    uint64_t rows() const {
        uint64_t t = 0;
        for (auto &s : shards) t += s.n;
        return t;
    }
    uint64_t returnable_rows() const { return mask_on ? mask_alive : rows(); }  // rows that can be returned
    uint64_t first_row(const NkShard &s) const { return s.base - row_base; }    // of a shard, relative to the index's first row
};

// An NVTX range (NK_RANGE_PUSH) that lasts to the end of the scope.
struct ScopedRange {
    explicit ScopedRange(const char *name) { NK_RANGE_PUSH(name); }
    ~ScopedRange() { NK_RANGE_POP(); }
    ScopedRange(const ScopedRange &) = delete;
    ScopedRange &operator=(const ScopedRange &) = delete;
};

// ---- call order (include/nornic_knn.h, "Call order") ------------------------------------------------------------------
// The calls on one index take effect in call order, whatever streams they run on: the device searches run on the caller's
// stream, everything else on the shard's own non-blocking stream, and all of them share the shard's rows, masks, tags and
// workspace.  A call holds a ShardOrder, under the index lock, for every shard it queues work on: its stream first waits on
// the shard's event, which marks the end of the last call's work, and when the call is done the event is recorded on its
// stream.  One wait and one record per shard and call; no host synchronisation.
class ShardOrder {
  public:
    explicit ShardOrder(NkIndex *ix) {  // every shard, each on its own stream
        for (auto &s : ix->shards) enter(s, s.stream);
    }
    ShardOrder(NkShard &s, cudaStream_t st) { enter(s, st); }
    ~ShardOrder() {
        for (auto &h : held_) {
            cudaSetDevice(h.first->device);
            cudaEventRecord(h.first->last, h.second);
        }
    }
    ShardOrder(const ShardOrder &) = delete;
    ShardOrder &operator=(const ShardOrder &) = delete;
    bool failed() const { return failed_; }

  private:
    void enter(NkShard &s, cudaStream_t st) {
        cudaError_t e = cudaSetDevice(s.device);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(st, s.last, 0);
        if (e != cudaSuccess) {
            nk::set_error("cannot order the call after earlier work on device %d: %s", s.device, cudaGetErrorString(e));
            failed_ = true;
            return;
        }
        held_.emplace_back(&s, st);
    }
    std::vector<std::pair<NkShard *, cudaStream_t>> held_;
    bool failed_ = false;
};

// Block until every call queued on the shard so far has run, and this call's work on the shard's own stream too: before a
// buffer that earlier work, on any stream, may still read is freed or replaced.
static int shard_drain(NkShard &s) {
    NK_CUDA_OK(cudaEventSynchronize(s.last));
    NK_CUDA_OK(cudaStreamSynchronize(s.stream));
    return 0;
}

// Row-count changing mutations invalidate the row mask (its bits are positions).
static void drop_row_mask(NkIndex *ix) {
    ix->mask_on = false;
    ix->n_groups = 0;
    for (auto &s : ix->shards) { s.mask_on = false; s.group_on = false; }
}

// Global row ids are 32-bit on this boundary (SearchResult.Index uint32, cuda_bridge.go:425-428): may the index hold `rows`?
static int check_row_limit(const NkIndex *ix, uint64_t rows) {
    if (ix->row_base + rows > 0xfffffff0ull) { nk::set_error("index exceeds 2^32 rows (row ids are uint32)"); return -1; }
    return 0;
}

static std::vector<NkShard *> live_shards(NkIndex *ix) {  // the non-empty shards
    std::vector<NkShard *> live;
    for (auto &s : ix->shards)
        if (s.n) live.push_back(&s);
    return live;
}

// Grow-only pinned host staging (25% headroom, like the device workspace).
static int pinned_reserve(void **p, size_t *cur, size_t need) {
    if (*cur >= need) return 0;
    if (*p) cudaFreeHost(*p);
    *p = nullptr; *cur = 0;
    NK_CUDA_OK(cudaMallocHost(p, need + need / 4));
    *cur = need + need / 4;
    return 0;
}

// A result key -> (global row, score in the API's domain: euclidean keys are -distance^2).
static void decode_key(int metric, uint64_t key, uint32_t *row, float *score) {
    const float sc = nk::key_score(key);
    *row = nk::key_row(key);
    *score = metric == NK_METRIC_EUCLIDEAN ? sqrtf(std::max(-sc, 0.0f)) : sc;
}

// ---- per-row tag words (nk_search_filtered) and value keys (nk_search_windowed) -------------------------------------
// One 64-bit word per row, in a shard array (words, cap, on) = (tags, tags_cap, tags_on) or (values, values_cap, values_on).
// The array follows the rows: rows [old_n, s.n) are new and get word 0; the capacity follows the row capacity.  Synchronous,
// so a search on any stream may read the array afterwards.
static int shard_words_grow(NkShard &s, uint64_t *&words, uint64_t &words_cap, uint64_t old_n) {
    if (words_cap < s.n) {
        const uint64_t cap = std::max<uint64_t>(std::max(s.cap, s.n), 16);
        uint64_t *p = nullptr;
        NK_CUDA_OK(cudaMalloc((void **)&p, cap * 8));
        if (words && old_n) NK_CUDA_OK(cudaMemcpyAsync(p, words, old_n * 8, cudaMemcpyDeviceToDevice, s.stream));
        if (shard_drain(s)) return -1;
        if (words) NK_CUDA_OK(cudaFree(words));
        words = p;
        words_cap = cap;
    }
    if (s.n > old_n) NK_CUDA_OK(cudaMemsetAsync(words + old_n, 0, (s.n - old_n) * 8, s.stream));
    NK_CUDA_OK(cudaStreamSynchronize(s.stream));
    return 0;
}
// Make the array real (all zero if its words were never set since the last reset).
static int shard_words_on(NkShard &s, uint64_t *&words, uint64_t &words_cap, bool &on) {
    if (on) return 0;
    if (shard_words_grow(s, words, words_cap, 0)) return -1;
    on = true;
    return 0;
}
static int shard_tags_grow(NkShard &s, uint64_t old_n) { return shard_words_grow(s, s.tags, s.tags_cap, old_n); }
static int shard_tags_on(NkShard &s) { return shard_words_on(s, s.tags, s.tags_cap, s.tags_on); }
static int shard_values_on(NkShard &s) { return shard_words_on(s, s.values, s.values_cap, s.values_on); }

// Convert rows [first, first+count) into every image the shard has (one launch counted): the int8 image and / or the BF16
// shadow with their norms (fp32 shards), or the |x|^2 array (16-bit shards).
static int shard_image_build(NkIndex *ix, NkShard &s, uint64_t first, uint64_t count) {
    const ShardImages &m = s.img;
    ix->stats.kernel_launches++;
    if (ix->dtype != NK_DTYPE_F32) return nk::row_sqnorms16(s.rows, ix->dtype, first, count, ix->dim, m.xnorm2, s.stream);
    const float *rows = static_cast<const float *>(s.rows);
    if (m.s8 && nk::build_image_s8(rows, first, count, ix->dim, m.s8_image(ix->dim).dimpad, m.s8, m.s8_scale, m.xnorm2, m.s8_dnorm2, s.stream))
        return -1;
    return m.bf16 ? nk::build_shadow(rows, first, count, ix->dim, m.bf16_image(ix->dim).dimpad, m.bf16, m.xnorm2, m.bf16_dnorm2, s.stream) : 0;
}

// Bring the images of a shard up to date with rows [0, s.n) (converting only what is missing).  They are an optimisation: if
// their memory cannot be had the shard simply goes without (TF32 filter / CUDA-core scan over the rows).
static int shard_sync_shadow(NkIndex *ix, NkShard &s) {
    ShardImages &m = s.img;
    const bool f32 = ix->dtype == NK_DTYPE_F32;
    const bool bf = f32 && ix->keeps(nk::RowImage::BF16), s8 = f32 && ix->keeps(nk::RowImage::S8);
    const bool wanted = (f32 ? bf || s8 : ix->keeps(nk::RowImage::NATIVE)) && (s.owns || m.attached) && ix->dim >= 32 && s.n > 0 &&
                        (f32 ? ix->dim % 4 == 0 : ix->dim % 8 == 0);
    if (!wanted) {
        m.n = 0;
        return 0;
    }
    if (m.cap < s.n) {
        if (shard_drain(s)) return -1;
        m.release();
        const uint64_t cap = s.cap > s.n ? s.cap : s.n;
        cudaError_t e = cudaMalloc((void **)&m.xnorm2, cap * 4);
        if (e == cudaSuccess && bf) e = cudaMalloc(&m.bf16, cap * m.bf16_image(ix->dim).row_bytes());
        if (e == cudaSuccess && bf) e = cudaMalloc((void **)&m.bf16_dnorm2, cap * 4);
        if (e == cudaSuccess && s8) {
            e = cudaMalloc(&m.s8, cap * m.s8_image(ix->dim).row_bytes());
            if (e == cudaSuccess) e = cudaMalloc((void **)&m.s8_scale, cap * 4);
            if (e == cudaSuccess) e = cudaMalloc((void **)&m.s8_dnorm2, cap * 4);
            if (e != cudaSuccess && bf) {  // the shard keeps its BF16 shadow and goes without the int8 image
                cudaGetLastError();
                m.release(true);
                e = cudaSuccess;
            }
        }
        if (e != cudaSuccess) {
            cudaGetLastError();
            m.release();
            return 0;
        }
        m.cap = cap;
    }
    if (m.n < s.n && shard_image_build(ix, s, m.n, s.n - m.n)) return -1;
    m.n = s.n;
    return 0;
}

// ---- cold-start feed (SURVEY.md §8(f)3) ---------------------------------------------------------------------------
// Host rows -> device through two pinned staging buffers: while chunk i crosses PCIe by DMA the CPU copies chunk i+1
// into the other buffer, so pageable (and unaligned: the vectors of a serialized index start at an arbitrary byte
// offset) sources load at the slower of the host memcpy and the PCIe rate instead of the driver's pageable path.
// cvt_f32_to_f16: the source is fp32 and the destination rows are fp16 (down-conversion at load, on the device).
constexpr size_t STAGE_BYTES = 32u << 20;

// one core copies ~11 GB/s, a x16 Gen5 link moves ~50: split the staging copy over a few threads
static void parallel_memcpy(void *dst, const void *src, size_t bytes) {
    constexpr int T = 6;
    if (bytes < (4u << 20)) {
        memcpy(dst, src, bytes);
        return;
    }
    std::thread th[T - 1];
    const size_t part = (bytes / T + 63) & ~(size_t)63;
    for (int t = 1; t < T; ++t) {
        const size_t lo = std::min(bytes, part * t), hi = t == T - 1 ? bytes : std::min(bytes, part * (t + 1));
        th[t - 1] = std::thread([=] { if (hi > lo) memcpy(static_cast<char *>(dst) + lo, static_cast<const char *>(src) + lo, hi - lo); });
    }
    memcpy(dst, src, std::min(bytes, part));
    for (auto &t : th) t.join();
}

static int stream_h2d(NkShard &s, void *dst_dev, const void *src_host, size_t bytes, bool cvt_f32_to_f16 = false, int cvt_dtype = NK_DTYPE_F16) {
    if (bytes == 0) return 0;
    for (int i = 0; i < 2; ++i) {
        if (!s.stage[i]) NK_CUDA_OK(cudaHostAlloc(&s.stage[i], STAGE_BYTES, cudaHostAllocDefault));
        if (!s.stage_ev[i]) NK_CUDA_OK(cudaEventCreateWithFlags(&s.stage_ev[i], cudaEventDisableTiming));
    }
    if (cvt_f32_to_f16 && nk::ws_reserve(&s.cvt, &s.cvt_bytes, 2 * STAGE_BYTES)) return -1;
    size_t done = 0;
    for (int i = 0; done < bytes; ++i) {
        const int b = i & 1;
        const size_t chunk = std::min(STAGE_BYTES, bytes - done);
        if (i >= 2) NK_CUDA_OK(cudaEventSynchronize(s.stage_ev[b]));  // the DMA that last read this buffer has drained
        parallel_memcpy(s.stage[b], static_cast<const char *>(src_host) + done, chunk);
        if (cvt_f32_to_f16) {
            float *scratch = reinterpret_cast<float *>(static_cast<char *>(s.cvt) + (size_t)b * STAGE_BYTES);
            NK_CUDA_OK(cudaMemcpyAsync(scratch, s.stage[b], chunk, cudaMemcpyHostToDevice, s.stream));
            if (nk::convert_f32_to_16(scratch, static_cast<char *>(dst_dev) + done / 2, cvt_dtype, chunk / 4, s.stream)) return -1;
        } else {
            NK_CUDA_OK(cudaMemcpyAsync(static_cast<char *>(dst_dev) + done, s.stage[b], chunk, cudaMemcpyHostToDevice, s.stream));
        }
        NK_CUDA_OK(cudaEventRecord(s.stage_ev[b], s.stream));
        done += chunk;
    }
    return 0;
}

static int shard_reserve_rows(NkIndex *ix, NkShard &s, uint64_t need_rows, bool keep) {
    if (need_rows <= s.cap && s.rows) return 0;
    if (!s.owns) {
        nk::set_error("cannot grow attached (caller-owned) device rows");
        return -1;
    }
    uint64_t cap = keep ? std::max<uint64_t>(need_rows, s.cap + s.cap / 2) : need_rows;
    if (cap < 16) cap = 16;
    void *p = nullptr;
    size_t rb = (size_t)ix->dim * ix->esz();
    NK_CUDA_OK(cudaMalloc(&p, cap * rb));
    if (s.rows) {
        if (keep && s.n) NK_CUDA_OK(cudaMemcpyAsync(p, s.rows, s.n * rb, cudaMemcpyDeviceToDevice, s.stream));
        if (shard_drain(s)) return -1;
        NK_CUDA_OK(cudaFree(s.rows));
    }
    s.rows = p;
    s.cap = cap;
    return 0;
}

static void rebase(NkIndex *ix) {
    uint64_t b = ix->row_base;
    for (auto &s : ix->shards) {
        s.base = b;
        b += s.n;
    }
    ix->stats.rows = ix->rows();
}

// Locate the shard holding global row `row` (relative to row_base).
static NkShard *find_shard(NkIndex *ix, uint64_t row, uint64_t *local) {
    for (auto &s : ix->shards)
        if (row >= ix->first_row(s) && row < ix->first_row(s) + s.n) {
            *local = row - ix->first_row(s);
            return &s;
        }
    return nullptr;
}

// The plain kNN scan (ScanMode::KNN) of Q device queries over shard s as it stands: its rows, the row mask and the score floor.
static nk::ScanArgs shard_scan_args(const NkIndex *ix, const NkShard &s, const float *q_dev, uint32_t Q, uint32_t k, cudaStream_t stream) {
    nk::ScanArgs a;
    a.rows = s.rows; a.dtype = ix->dtype; a.n = (uint32_t)s.n; a.dim = ix->dim; a.row_base = s.base;
    a.queries = q_dev; a.Q = Q; a.k = k; a.metric = ix->metric; a.stream = stream;
    a.row_mask = s.mask_on ? s.mask : nullptr; a.min_score = ix->key_floor();
    return a;
}

// Give *a mode m and what m reads on shard s: the shard's tag and value arrays (turned on by whoever staged the predicates); the
// per-query filters and windows staged in the workspace (stage_predicates), or the caller's own device arrays qfilter /
// qwindow where given (the device API); and for the reverse modes each row's threshold with the keep mask behind them, which
// takes the place of the row mask, each row's own filter and window and the queries' tags and value keys (graph_reverse_scan).
static void set_scan_mode(const NkShard &s, nk::ScanMode m, nk::ScanArgs *a, const NkFilter *qfilter = nullptr,
                          const NkWindow *qwindow = nullptr) {
    a->mode = m;
    if (nk::mode_tags(m)) { a->row_tags = s.tags; a->qfilter = qfilter ? qfilter : s.ws.qfilter; }
    if (nk::mode_window(m)) { a->row_values = s.values; a->qwindow = qwindow ? qwindow : s.ws.qwindow; }
    if (nk::mode_row_thr(m)) { a->row_thr = s.ws.row_thr; a->row_mask = reinterpret_cast<const uint32_t *>(s.ws.row_thr + s.n); }
    if (nk::mode_row_filter(m)) { a->row_filter = s.ws.row_filter; a->qtags = s.ws.qtags; }
    if (nk::mode_row_window(m)) { a->row_window = s.ws.row_window; a->qvalues = s.ws.qvalues; }
}

// Has a search on the shard's int8 image overflowed its margin buffers since the last look?  Reads the counters copied
// behind the last int8 search if they have landed (never waits); once true, the shard's kNN filter keeps to the BF16 shadow.
static bool shard_s8_off(const NkShard &s) {
    const ShardImages &m = s.img;
    if (!m.s8_off && m.s8_ev && cudaEventQuery(m.s8_ev) == cudaSuccess) {
        const int64_t seen = (int64_t)m.s8_h[0] + m.s8_h[1];
        if (seen > m.s8_seen) m.s8_off = true;
        m.s8_seen = seen;
    }
    return m.s8_off;
}

// The image a scan of shard s streams, if the shard has an up-to-date one (else kind NONE): a 16-bit shard's own rows, or
// the int8 image or the BF16 shadow of an fp32 shard.  knn: a kNN filter search for the k best.  The int8 image serves it
// where it wins: a shard large enough for the scan to be bound by HBM bytes (the same 64 MB as AUTO's), k <= S8_MAX_K, and
// no earlier overflow on it.  Its margins are ~3x the BF16 shadow's, so at larger k every CTA emits several times more rows
// for exact re-scoring (Q = 1024, k = 100: 5.6x slower, DESIGN §3.3), range searches would list more rows and k-means
// assignment would leave more near-ties to its fix-up; those keep to the BF16 shadow where the shard has one.
constexpr uint32_t S8_MAX_K = 16;
static nk::RowImage shard_image(const NkIndex *ix, const NkShard &s, bool knn, uint32_t k) {
    const ShardImages &m = s.img;
    if (!m.current(s.n)) return {};
    if (ix->dtype != NK_DTYPE_F32) return nk::RowImage(nk::RowImage::NATIVE, s.rows, ix->dim, m.xnorm2);
    const bool s8 = m.s8 && (!m.bf16 || (knn && k <= S8_MAX_K && (uint64_t)s.n * ix->dim * 4 >= (64ull << 20) && !shard_s8_off(s)));
    return s8 ? m.s8_image(ix->dim) : m.bf16_image(ix->dim);
}

// Behind a search on the int8 image: copy the shard's overflow counters to pinned memory (read by shard_s8_off).
static int shard_s8_watch(NkShard &s, cudaStream_t stream) {
    ShardImages &m = s.img;
    if (!m.s8_ev) {
        if (cudaEventCreateWithFlags(&m.s8_ev, cudaEventDisableTiming) != cudaSuccess ||
            cudaMallocHost((void **)&m.s8_h, 2 * sizeof(int)) != cudaSuccess) {
            nk::set_error("int8 image: event / pinned counters unavailable");
            return -1;
        }
    }
    NK_CUDA_OK(cudaMemcpyAsync(m.s8_h, s.ws.flags + nk::FLAG_N_RETRY, 2 * sizeof(int), cudaMemcpyDeviceToHost, stream));
    NK_CUDA_OK(cudaEventRecord(m.s8_ev, stream));
    return 0;
}

// The path a scan of *a over shard s takes when the call asks for `path` (the index's setting, nk_index_set_path, or the
// one a graph call chose): the forced one (an error if it cannot serve the shape), or AUTO's pick.  *a gets
// the shard's image (shard_image) attached if the path is the 16-bit / int8 pass.  Range searches have no exact 3xTF32 mode.
// AUTO: CUDA cores keep Q <= 4 (the single-kernel scan already streams the fewest bytes), tensor cores from 5 queries on.
// With a BF16 shadow the filter streams half the bytes of the fp32 rows, so it serves every batch size once the shard is
// large enough for bytes (not launches) to matter; small shards keep the CUDA-core scan at Q <= 4.  16-bit shards: the
// 16-bit tensor pass from 5 queries on.
static int plan_path(const NkIndex *ix, const NkShard &s, int path, bool range, nk::ScanArgs *a) {
    if (range && path == NK_PATH_TENSOR) {
        nk::set_error("nk_search_range: the exact 3xTF32 path has no range mode (use AUTO, SIMT, TENSOR_FILTER or TENSOR_SHADOW)");
        return -1;
    }
    nk::ScanArgs as = *a;
    as.image = shard_image(ix, s, !range, a->k);
    const bool tensor_ok = !range && nk::scan_tensor_supported(s.di, *a);
    const bool filter_ok = ix->dtype == NK_DTYPE_F32 && nk::scan_tensor_filter_supported(s.di, *a);
    const bool shadow_ok = nk::shadow_pass_supported(s.di, as) && nk::scan_tensor_filter_supported(s.di, as);
    int use = NK_PATH_SIMT;
    if (path == NK_PATH_TENSOR || path == NK_PATH_TENSOR_FILTER || path == NK_PATH_TENSOR_SHADOW) {
        if (!(path == NK_PATH_TENSOR ? tensor_ok : path == NK_PATH_TENSOR_FILTER ? filter_ok : shadow_ok)) {
            nk::set_error("tensor path %d does not support this shape (dim=%u dtype=%d metric=%d Q=%u k=%u shadow=%d)", path, ix->dim,
                          ix->dtype, ix->metric, a->Q, a->k, (int)(as.image.kind != nk::RowImage::NONE));
            return -1;
        }
        use = path;
    } else if (path == NK_PATH_AUTO) {
        const bool big_shard = (uint64_t)s.n * ix->dim * 4 >= (64ull << 20);
        if (a->Q >= 5) use = shadow_ok ? NK_PATH_TENSOR_SHADOW : filter_ok ? NK_PATH_TENSOR_FILTER : tensor_ok ? NK_PATH_TENSOR : NK_PATH_SIMT;
        else if (shadow_ok && big_shard && ix->dtype == NK_DTYPE_F32) use = NK_PATH_TENSOR_SHADOW;
    }
    if (use == NK_PATH_TENSOR_SHADOW) *a = as;
    return use;
}

// Times the main kernels of one scan (nk_index_enable_timing): attach() gives the scan an event pair, keep() hands it to the
// shard for nk_index_scan_time_ms if the scan launched a main kernel.  Every pair not kept is destroyed.
class ScanTimer {
  public:
    explicit ScanTimer(NkShard &s) : s_(s) {}
    ~ScanTimer() {
        for (cudaEvent_t e : ev_)
            if (e) cudaEventDestroy(e);
    }
    ScanTimer(const ScanTimer &) = delete;
    ScanTimer &operator=(const ScanTimer &) = delete;
    int attach(const NkIndex *ix, nk::ScanArgs *a) {
        if (!ix->timing_on) return 0;
        for (cudaEvent_t &e : ev_) NK_CUDA_OK(cudaEventCreate(&e));
        a->ev_begin = ev_[0]; a->ev_end = ev_[1]; a->main_launches = &launches_;
        return 0;
    }
    void keep() {  // the scan succeeded
        if (!launches_) return;
        s_.timing.emplace_back(ev_[0], ev_[1]);
        s_.timing_launches.push_back(launches_);
        ev_[0] = ev_[1] = nullptr;
    }

  private:
    NkShard &s_;
    cudaEvent_t ev_[2] = {nullptr, nullptr};
    uint64_t launches_ = 0;
};

// NkStats::bytes_scanned of `passes` scans of a on path `use`: every pass streams the a.n rows once per block of queries
// (8 on CUDA cores, 64 in the exact 3xTF32 scan, 128 in the filters); the 16-bit / int8 pass streams the image's rows.
static uint64_t scan_bytes(const NkIndex *ix, int use, const nk::ScanArgs &a, uint64_t passes) {
    const uint32_t width = use == NK_PATH_SIMT ? 8 : use == NK_PATH_TENSOR ? 64 : 128;
    const uint64_t row_bytes = use == NK_PATH_TENSOR_SHADOW ? a.image.row_bytes() : (uint64_t)ix->dim * ix->esz();
    return (uint64_t)a.n * row_bytes * ((a.Q + width - 1) / width) * passes;
}

// a.k > NK_MAX_K (the reference accepts any k, cuda_bridge.go:327-375): ceil(a.k / NK_MAX_K) fused CUDA-core passes; pass p+1
// only admits keys strictly below the last key pass p returned, so the passes tile the ranking exactly.
static int run_scan_bigk(NkIndex *ix, NkShard &s, nk::ScanArgs a, uint64_t *out_keys) {
    const uint32_t Q = a.Q, k = a.k;
    if (nk::ws_reserve((void **)&s.ws.below, &s.ws.below_bytes, (size_t)Q * 8)) return -1;
    if (nk::ws_reserve((void **)&s.ws.keys2, &s.ws.keys2_bytes, (size_t)Q * NK_MAX_K * 8)) return -1;
    NK_CUDA_OK(cudaMemsetAsync(s.ws.below, 0xff, (size_t)Q * 8, a.stream));
    a.below = s.ws.below;
    for (uint32_t done = 0; done < k;) {
        const uint32_t kp = k - done < NK_MAX_K ? k - done : NK_MAX_K;
        a.k = kp;
        if (nk::scan_simt(s.di, a, s.ws, s.ws.keys2, &ix->stats.kernel_launches)) return -1;
        NK_CUDA_OK(cudaMemcpy2DAsync(out_keys + done, (size_t)k * 8, s.ws.keys2, (size_t)kp * 8, (size_t)kp * 8, Q,
                                     cudaMemcpyDeviceToDevice, a.stream));
        if (nk::update_below(s.ws.keys2, Q, kp, s.ws.below, a.stream)) return -1;
        ix->stats.kernel_launches++;
        ix->stats.bytes_scanned += scan_bytes(ix, NK_PATH_SIMT, a, 1);
        done += kp;
    }
    ix->last_path = NK_PATH_SIMT;
    return 0;
}

// The retry / exact stages a host-synchronous filter search left unqueued, as a value its caller owns: run_scan fills it,
// shard_status queues the stages from it once the host has seen a status word raised.
struct DeferredTail {
    bool pending = false;  // a filter scan ran and its tail has not been looked at yet
    nk::ScanArgs args;     // the scan to re-issue (scan_tensor_filter_tail), without its timing events
    uint64_t *out_keys = nullptr;
};

struct ScanOut {  // what a call asks of run_scan beyond the queries
    explicit ScanOut(int path, nk::ScanMode mode = nk::ScanMode::KNN) : path(path), mode(mode) {}
    int path;                      // the scan path of the call (plan_path)
    nk::ScanMode mode;             // KNN, KNN_TAGS or KNN_WINDOW (set_scan_mode)
    uint32_t *out_idx = nullptr;   // fused decode (single-shard searches)
    float *out_score = nullptr;
    DeferredTail *tail = nullptr;  // host-synchronous caller: retry stages are left to *tail, queued only if a flag was raised
    const NkFilter *qfilter = nullptr;  // the device API's own per-query filters / windows [Q]; nullptr: the workspace's
    const NkWindow *qwindow = nullptr;
};

static int run_scan(NkIndex *ix, NkShard &s, const float *q_dev, uint32_t Q, uint32_t k, uint64_t *out_keys,
                    cudaStream_t stream, const ScanOut &xo) {
    nk::ScanArgs a = shard_scan_args(ix, s, q_dev, Q, k, stream);
    set_scan_mode(s, xo.mode, &a, xo.qfilter, xo.qwindow);
    if (k > NK_MAX_K) {
        if (run_scan_bigk(ix, s, a, out_keys)) return -1;
        if (xo.out_idx) {
            if (nk::decode_keys(out_keys, Q, k, ix->metric, xo.out_idx, xo.out_score, stream)) return -1;
            ix->stats.kernel_launches++;
        }
        return 0;
    }
    a.out_idx = xo.out_idx; a.out_score = xo.out_score; a.defer_tail = xo.tail != nullptr;
    const int use = plan_path(ix, s, xo.path, false, &a);
    if (use < 0) return -1;
    ScanTimer timer(s);
    if (timer.attach(ix, &a)) return -1;
    const bool is_filter = use == NK_PATH_TENSOR_FILTER || use == NK_PATH_TENSOR_SHADOW;
    NK_RANGE_PUSH(use == NK_PATH_TENSOR_SHADOW ? "nk:scan:shadow" : use == NK_PATH_TENSOR_FILTER ? "nk:scan:tf32-filter"
                  : use == NK_PATH_TENSOR ? "nk:scan:3xtf32" : "nk:scan:simt");
    int rc = is_filter ? nk::scan_tensor_filter(s.di, a, s.ws, out_keys, &ix->stats.kernel_launches)
             : use == NK_PATH_TENSOR ? nk::scan_tensor(s.di, a, s.ws, out_keys, &ix->stats.kernel_launches)
                                     : nk::scan_simt(s.di, a, s.ws, out_keys, &ix->stats.kernel_launches);
    NK_RANGE_POP();
    ix->last_path = use;
    if (rc) return rc;
    timer.keep();
    if (is_filter && xo.tail) {  // the timer's events are gone by the time the tail runs
        *xo.tail = DeferredTail{true, a, out_keys};
        xo.tail->args.ev_begin = xo.tail->args.ev_end = nullptr;
        xo.tail->args.main_launches = nullptr;
    }
    ix->stats.bytes_scanned += scan_bytes(ix, use, a, 1);
    if (use == NK_PATH_TENSOR_SHADOW && a.image.kind == nk::RowImage::S8 && shard_s8_watch(s, stream)) return -1;
    return 0;
}

// Host-synchronous searches defer the retry / exact stages of the filter paths.  h is the shard's status words, read after
// the stream has drained: the fatal word set -> clear it and fail (-1); a deferred filter stage overflowed (adversarial
// near-ties, NaN rows) -> queue the tail, and the caller waits and reads again (1); else the results stand (0).  tail: the
// one run_scan filled for this search, nullptr if the call ran no filter scan.  It is queued at most once per search: the
// first look clears it.
static int shard_status(NkIndex *ix, NkShard &s, const int *h, DeferredTail *tail) {
    const bool queue = tail && tail->pending && (h[nk::FLAG_RETRY] || h[nk::FLAG_OVERFLOW]);
    if (tail) tail->pending = false;
    if (h[nk::FLAG_FATAL]) return nk::fatal_overflow(h[nk::FLAG_FATAL], s.ws.flags, s.stream);
    if (!queue) return 0;
    ScopedRange range("nk:retry-tail");
    return nk::scan_tensor_filter_tail(s.di, tail->args, s.ws, tail->out_keys, &ix->stats.kernel_launches) ? -1 : 1;
}

// shard_status on the status words alone, the retry tail included: 0 or -1.
static int finish_deferred(NkIndex *ix, NkShard &s, DeferredTail *tail) {
    for (;;) {
        int h[nk::NK_FLAG_WORDS];
        NK_CUDA_OK(cudaMemcpyAsync(h, s.ws.flags, sizeof(h), cudaMemcpyDeviceToHost, s.stream));
        NK_CUDA_OK(cudaStreamSynchronize(s.stream));
        const int st = shard_status(ix, s, h, tail);
        if (st <= 0) return st;
    }
}

extern "C" {

const char *nk_last_error(void) { return nk::get_error(); }
const char *nk_version(void) { return "nornic-knn-b200 0.1 (sm_90a)"; }

NkIndex *nk_index_create(const int *device_ids, int n_devices, uint32_t dim, int dtype, int metric) {
    nk::DeviceGuard _restore_device;
    if (n_devices <= 0 || !device_ids || dim == 0) {
        nk::set_error("nk_index_create: need >= 1 device and dim > 0");
        return nullptr;
    }
    if (dtype != NK_DTYPE_F32 && dtype != NK_DTYPE_F16 && dtype != NK_DTYPE_BF16) {
        nk::set_error("nk_index_create: unknown dtype %d", dtype);
        return nullptr;
    }
    if (metric < NK_METRIC_COSINE || metric > NK_METRIC_EUCLIDEAN) {
        nk::set_error("nk_index_create: unknown metric %d", metric);
        return nullptr;
    }
    NkIndex *ix = new NkIndex();
    ix->dim = dim; ix->dtype = dtype; ix->metric = metric;
    if (const char *e = getenv("NK_SHADOW")) {  // read once, at creation
        const unsigned native = 1u << nk::RowImage::NATIVE;
        ix->images = strcmp(e, "int8") == 0 ? 1u << nk::RowImage::S8 | native
                     : strcmp(e, "bf16") == 0 ? 1u << nk::RowImage::BF16 | native
                     : atoi(e) != 0 ? ix->images : 0u;
    }
    ix->stats.dim = dim; ix->stats.n_devices = (uint32_t)n_devices;
    ix->shards.resize(n_devices);
    for (int i = 0; i < n_devices; ++i) {
        NkShard &s = ix->shards[i];
        s.device = device_ids[i];
        cudaError_t e = cudaSetDevice(s.device);
        if (e == cudaSuccess && nk::query_device_info(s.device, &s.di) != 0) e = cudaErrorUnknown;
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.last, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaMalloc((void **)&s.ws.flags, sizeof(int) * nk::NK_FLAG_WORDS);
        if (e == cudaSuccess) e = cudaMemset(s.ws.flags, 0, sizeof(int) * nk::NK_FLAG_WORDS);
        if (e != cudaSuccess) {
            if (e != cudaErrorUnknown) nk::set_error("nk_index_create(device %d): %s", s.device, cudaGetErrorString(e));
            cudaGetLastError();
            nk_index_release(ix);
            return nullptr;
        }
    }
    return ix;
}

void nk_index_release(NkIndex *ix) {
    nk::DeviceGuard _restore_device;
    if (!ix) return;
    for (auto &s : ix->shards) {
        cudaSetDevice(s.device);
        if (s.last) {  // work queued on any stream, a device search on the caller's included, may still read the buffers
            cudaEventSynchronize(s.last);
            cudaEventDestroy(s.last);
        }
        if (s.stream) {
            cudaStreamSynchronize(s.stream);
            cudaStreamDestroy(s.stream);
        }
        if (s.rows && s.owns) cudaFree(s.rows);
        s.img.release();
        if (s.img.s8_h) cudaFreeHost(s.img.s8_h);
        if (s.img.s8_ev) cudaEventDestroy(s.img.s8_ev);
        if (s.h_keys) cudaFreeHost(s.h_keys);
        if (s.h_res) cudaFreeHost(s.h_res);
        for (int i = 0; i < 2; ++i) {
            if (s.stage[i]) cudaFreeHost(s.stage[i]);
            if (s.stage_ev[i]) cudaEventDestroy(s.stage_ev[i]);
        }
        if (s.cvt) cudaFree(s.cvt);
        if (s.mask) cudaFree(s.mask);
        if (s.tags) cudaFree(s.tags);
        if (s.values) cudaFree(s.values);
        if (s.group) cudaFree(s.group);
        s.ws.release();
    }
    if (ix->h_qrows) cudaFreeHost(ix->h_qrows);
    delete ix;
}

// Replace the whole corpus by n_rows new rows, shard g taking the contiguous range [g*N/G, (g+1)*N/G): write(s, first, cnt)
// queues the write of rows [first, first+cnt) into the shard's reserved rows on its stream.
using WriteRows = std::function<int(NkShard &, uint64_t first, uint64_t cnt)>;
static int repartition(NkIndex *ix, uint64_t n_rows, const WriteRows &write) {
    std::lock_guard<std::mutex> lk(ix->mu);
    ShardOrder order(ix);
    if (order.failed()) return -1;
    drop_row_mask(ix);
    if (check_row_limit(ix, n_rows)) return -1;
    const uint64_t G = ix->shards.size();
    uint64_t off = 0;
    for (uint64_t g = 0; g < G; ++g) {
        NkShard &s = ix->shards[g];
        const uint64_t cnt = n_rows * (g + 1) / G - n_rows * g / G;
        NK_CUDA_OK(cudaSetDevice(s.device));
        if (!s.owns) { s.rows = nullptr; s.owns = true; s.cap = 0; s.img.attached = false; }
        s.n = 0;
        s.tags_on = false;  // every tag back to 0
        s.values_on = false;  // every value key back to 0
        if (shard_reserve_rows(ix, s, cnt, false)) return -1;
        if (write(s, off, cnt)) return -1;
        s.n = cnt;
        s.img.n = 0;
        if (shard_sync_shadow(ix, s)) return -1;
        off += cnt;
    }
    for (auto &s : ix->shards) {
        NK_CUDA_OK(cudaSetDevice(s.device));
        NK_CUDA_OK(cudaStreamSynchronize(s.stream));
    }
    rebase(ix);
    return 0;
}

static int upload_impl(NkIndex *ix, const void *rows_host, uint64_t n_rows, bool src_is_f32) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    if (n_rows && !rows_host) { nk::set_error("null rows"); return -1; }
    const bool cvt = src_is_f32 && ix->dtype != NK_DTYPE_F32;
    const size_t src_rb = (size_t)ix->dim * (cvt ? 4 : ix->esz());
    return repartition(ix, n_rows, [&](NkShard &s, uint64_t first, uint64_t cnt) {
        if (stream_h2d(s, s.rows, static_cast<const char *>(rows_host) + first * src_rb, cnt * src_rb, cvt, ix->dtype)) return -1;
        ix->stats.bytes_h2d += cnt * src_rb;
        return 0;
    });
}

int nk_index_upload(NkIndex *ix, const void *rows_host, uint64_t n_rows) { return upload_impl(ix, rows_host, n_rows, false); }

int nk_index_upload_from_f32(NkIndex *ix, const float *rows_host_f32, uint64_t n_rows) { return upload_impl(ix, rows_host_f32, n_rows, true); }

// Serialized index (EmbeddingIndex.Serialize, gpu.go:2373-2412): LE [dims u32][count u32][count x (len u32, id bytes)]
// [count x dims fp32].  Walks the id table; the vectors start at *vec_offset (any byte alignment).
int nk_blob_vectors(const void *blob, size_t blob_bytes, uint32_t *dims, uint32_t *count, size_t *vec_offset) {
    if (!blob || !dims || !count || !vec_offset) { nk::set_error("null argument"); return -1; }
    const unsigned char *p = static_cast<const unsigned char *>(blob);
    auto rd32 = [&](size_t at) { return (uint32_t)p[at] | ((uint32_t)p[at + 1] << 8) | ((uint32_t)p[at + 2] << 16) | ((uint32_t)p[at + 3] << 24); };
    if (blob_bytes < 8) { nk::set_error("gpu: invalid serialized data"); return -1; }  // gpu.go:2419-2421
    const uint32_t d = rd32(0), c = rd32(4);
    size_t off = 8;
    for (uint32_t i = 0; i < c; ++i) {
        if (off + 4 > blob_bytes) { nk::set_error("serialized index truncated in the id table (id %u)", i); return -1; }
        const uint32_t len = rd32(off);
        off += 4;
        if (len > blob_bytes - off) { nk::set_error("serialized index truncated in the id table (id %u)", i); return -1; }
        off += len;
    }
    if ((uint64_t)c * d * 4 > blob_bytes - off) { nk::set_error("serialized index truncated: %u x %u vectors do not fit", c, d); return -1; }
    *dims = d; *count = c; *vec_offset = off;
    return 0;
}

int nk_index_append(NkIndex *ix, const void *rows_host, uint64_t n_rows) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    if (n_rows == 0) return 0;
    if (!rows_host) { nk::set_error("null rows"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    NkShard &s = ix->shards.back();
    ShardOrder order(s, s.stream);
    if (order.failed()) return -1;
    drop_row_mask(ix);
    const size_t rb = (size_t)ix->dim * ix->esz();
    if (check_row_limit(ix, ix->rows() + n_rows)) return -1;
    NK_CUDA_OK(cudaSetDevice(s.device));
    if (shard_reserve_rows(ix, s, s.n + n_rows, true)) return -1;
    if (stream_h2d(s, (char *)s.rows + s.n * rb, rows_host, n_rows * rb)) return -1;
    s.n += n_rows;
    if (s.tags_on && shard_tags_grow(s, s.n - n_rows)) return -1;  // appended rows: tag 0
    if (s.values_on && shard_words_grow(s, s.values, s.values_cap, s.n - n_rows)) return -1;  // ... and value key 0
    if (shard_sync_shadow(ix, s)) return -1;  // converts only the appended rows (all of them if the shard was regrown)
    NK_CUDA_OK(cudaStreamSynchronize(s.stream));
    ix->stats.bytes_h2d += n_rows * rb;
    rebase(ix);
    return 0;
}

int nk_index_update_row(NkIndex *ix, uint64_t row, const void *row_host) {
    nk::DeviceGuard _restore_device;
    if (!ix || !row_host) { nk::set_error("null argument"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    uint64_t local;
    NkShard *s = find_shard(ix, row, &local);
    if (!s) { nk::set_error("row %llu out of range", (unsigned long long)row); return -1; }
    ShardOrder order(*s, s->stream);
    if (order.failed()) return -1;
    const size_t rb = (size_t)ix->dim * ix->esz();
    NK_CUDA_OK(cudaSetDevice(s->device));
    NK_CUDA_OK(cudaMemcpyAsync((char *)s->rows + local * rb, row_host, rb, cudaMemcpyHostToDevice, s->stream));
    if (s->img.xnorm2 && local < s->img.n && shard_image_build(ix, *s, local, 1)) return -1;
    NK_CUDA_OK(cudaStreamSynchronize(s->stream));
    ix->stats.bytes_h2d += rb;
    return 0;
}

int nk_index_remove_swap(NkIndex *ix, uint64_t row) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    uint64_t total = ix->rows();
    if (row >= total) { nk::set_error("row %llu out of range", (unsigned long long)row); return -1; }
    ShardOrder order(ix);
    if (order.failed()) return -1;
    drop_row_mask(ix);
    // last non-empty shard holds the last row
    NkShard *last = nullptr;
    for (auto it = ix->shards.rbegin(); it != ix->shards.rend(); ++it)
        if (it->n) { last = &*it; break; }
    uint64_t local;
    NkShard *s = find_shard(ix, row, &local);
    const size_t rb = (size_t)ix->dim * ix->esz();
    if (row != total - 1) {
        const char *src = (const char *)last->rows + (last->n - 1) * rb;
        char *dst = (char *)s->rows + local * rb;
        // The copy must be ordered with the shard's own stream (non-blocking streams do not synchronise with the legacy
        // default stream): drain the source shard first when it is another device, then copy ON s->stream so that the
        // shadow / norm rebuild queued behind reads the new row.
        if (last != s) {
            NK_CUDA_OK(cudaSetDevice(last->device));
            NK_CUDA_OK(cudaStreamSynchronize(last->stream));
        }
        NK_CUDA_OK(cudaSetDevice(s->device));
        if (last->device == s->device) NK_CUDA_OK(cudaMemcpyAsync(dst, src, rb, cudaMemcpyDeviceToDevice, s->stream));
        else NK_CUDA_OK(cudaMemcpyPeerAsync(dst, s->device, src, last->device, rb, s->stream));
        if (s->img.xnorm2 && local < s->img.n && shard_image_build(ix, *s, local, 1)) return -1;
        NK_CUDA_OK(cudaStreamSynchronize(s->stream));
        if (last->tags_on || s->tags_on) {  // the last row's tag moves with its row
            uint64_t tag = 0;
            if (last->tags_on) {
                NK_CUDA_OK(cudaSetDevice(last->device));
                NK_CUDA_OK(cudaMemcpy(&tag, last->tags + (last->n - 1), 8, cudaMemcpyDeviceToHost));
            }
            NK_CUDA_OK(cudaSetDevice(s->device));
            if (shard_tags_on(*s)) return -1;
            NK_CUDA_OK(cudaMemcpy(s->tags + local, &tag, 8, cudaMemcpyHostToDevice));
        }
        if (last->values_on || s->values_on) {  // ... and so does its value key
            uint64_t val = 0;
            if (last->values_on) {
                NK_CUDA_OK(cudaSetDevice(last->device));
                NK_CUDA_OK(cudaMemcpy(&val, last->values + (last->n - 1), 8, cudaMemcpyDeviceToHost));
            }
            NK_CUDA_OK(cudaSetDevice(s->device));
            if (shard_values_on(*s)) return -1;
            NK_CUDA_OK(cudaMemcpy(s->values + local, &val, 8, cudaMemcpyHostToDevice));
        }
    }
    last->n -= 1;
    if (last->img.n > last->n) last->img.n = last->n;
    rebase(ix);
    return 0;
}

static int fill_impl(NkIndex *ix, uint64_t n_rows, uint64_t seed, uint32_t centres, float sigma, int unit) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    return repartition(ix, n_rows, [&](NkShard &s, uint64_t first, uint64_t cnt) {
        const uint64_t row0 = ix->row_base + first;
        if (centres ? nk::fill_clustered(s.rows, ix->dtype, cnt, ix->dim, seed, row0, centres, sigma, unit, s.stream)
                    : nk::fill_uniform(s.rows, ix->dtype, cnt, ix->dim, seed, row0, s.stream))
            return -1;
        ix->stats.kernel_launches++;
        return 0;
    });
}

int nk_index_fill_uniform(NkIndex *ix, uint64_t n_rows, uint64_t seed) { return fill_impl(ix, n_rows, seed, 0, 0.0f, 0); }
int nk_index_fill_clustered(NkIndex *ix, uint64_t n_rows, uint64_t seed, uint32_t n_centres, float sigma, int unit_norm) {
    if (n_centres == 0) { nk::set_error("nk_index_fill_clustered: n_centres must be >= 1"); return -1; }
    return fill_impl(ix, n_rows, seed, n_centres, sigma, unit_norm);
}

int nk_index_set_row_base(NkIndex *ix, uint64_t row_base) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    if (ix->shards.size() != 1) { nk::set_error("row_base applies to single-device indexes"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    ix->row_base = row_base;
    rebase(ix);
    return 0;
}

int nk_index_attach_device_rows(NkIndex *ix, void *rows_dev, uint64_t n_rows) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    if (ix->shards.size() != 1) { nk::set_error("attach applies to single-device indexes"); return -1; }
    if (check_row_limit(ix, n_rows)) return -1;
    std::lock_guard<std::mutex> lk(ix->mu);
    NkShard &s = ix->shards[0];
    ShardOrder order(s, s.stream);
    if (order.failed()) return -1;
    NK_CUDA_OK(cudaSetDevice(s.device));
    if (shard_drain(s)) return -1;
    if (s.rows && s.owns) NK_CUDA_OK(cudaFree(s.rows));
    // caller-owned rows may change behind the library's back (cuda_normalize_vectors runs right after NewBuffer,
    // gpu.go:2100-2106): no shadow until the caller says the rows are final (nk_index_refresh_shadow)
    s.img.release();
    drop_row_mask(ix);
    s.rows = rows_dev; s.owns = false; s.n = n_rows; s.cap = n_rows; s.img.attached = false;
    s.tags_on = false;  // every tag back to 0
    s.values_on = false;  // every value key back to 0
    rebase(ix);
    return 0;
}

// (Re)build the 16-bit image of every shard from the rows as they are now.  For attached (caller-owned) rows this is the
// explicit "rows are final" signal that gives the documented drop-in route the fast filter path; for library-owned shards
// it is a no-op unless rows were changed behind the library's back.
int nk_index_refresh_shadow(NkIndex *ix) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    ShardOrder order(ix);
    if (order.failed()) return -1;
    for (auto &s : ix->shards) {
        NK_CUDA_OK(cudaSetDevice(s.device));
        if (!s.owns) s.img.attached = true;
        s.img.n = 0;
        if (shard_sync_shadow(ix, s)) return -1;
        NK_CUDA_OK(cudaStreamSynchronize(s.stream));
    }
    return 0;
}

int nk_index_set_metric(NkIndex *ix, int metric) {
    if (!ix) { nk::set_error("null index"); return -1; }
    if (metric < NK_METRIC_COSINE || metric > NK_METRIC_EUCLIDEAN) { nk::set_error("unknown metric %d", metric); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    ix->metric = metric;  // rows are stored raw and the shadow's norms are metric-independent: nothing to rebuild
    return 0;
}

int nk_index_set_min_score(NkIndex *ix, float min_score) {
    if (!ix) { nk::set_error("null index"); return -1; }
    if (min_score != min_score) { nk::set_error("min_score is NaN"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    ix->min_score = min_score;
    return 0;
}

// Row filter for subsequent searches (label / type filter of db.index.vector.queryNodes, call_vector.go:177-193; also
// tombstones): bit r of mask_words (LSB first in 32-bit words) set = row r (relative to the index's first row) may be
// returned.  NULL clears the filter.  Row-count changing mutations (upload, append, remove_swap, fill, attach) clear it.
int nk_index_set_row_mask(NkIndex *ix, const uint32_t *mask_words, uint64_t n_bits) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    if (!mask_words) {  // clear the filter only (the row groups stay: the row count did not change)
        ix->mask_on = false;
        for (auto &s : ix->shards) s.mask_on = false;
        return 0;
    }
    if (n_bits != ix->rows()) { nk::set_error("row mask has %llu bits, index has %llu rows", (unsigned long long)n_bits, (unsigned long long)ix->rows()); return -1; }
    ShardOrder order(ix);
    if (order.failed()) return -1;
    uint64_t off = 0, alive = 0;
    std::vector<uint32_t> local;
    for (auto &s : ix->shards) {
        const size_t words = (size_t)((s.n + 31) / 32);
        local.assign(words ? words : 1, 0u);
        for (uint64_t r = 0; r < s.n; ++r) {
            const uint64_t g = off + r;
            if ((mask_words[g >> 5] >> (g & 31)) & 1u) {
                local[r >> 5] |= 1u << (r & 31);
                ++alive;
            }
        }
        NK_CUDA_OK(cudaSetDevice(s.device));
        if (nk::ws_reserve((void **)&s.mask, &s.mask_bytes, local.size() * 4)) return -1;
        NK_CUDA_OK(cudaMemcpyAsync(s.mask, local.data(), local.size() * 4, cudaMemcpyHostToDevice, s.stream));
        NK_CUDA_OK(cudaStreamSynchronize(s.stream));
        s.mask_on = true;
        off += s.n;
    }
    ix->mask_on = true;
    ix->mask_alive = alive;
    return 0;
}

// nk_index_set_row_tags (values = false) / nk_index_set_row_values (values = true): words of rows [first_row, first_row + n_rows).
static int set_row_words(NkIndex *ix, uint64_t first_row, const uint64_t *words_host, uint64_t n_rows, bool values) {
    nk::DeviceGuard _restore_device;
    const char *what = values ? "values" : "tags";
    if (!ix) { nk::set_error("null index"); return -1; }
    if (n_rows == 0) return 0;
    if (!words_host) { nk::set_error("null %s", what); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    const uint64_t total = ix->rows();
    if (first_row > total || n_rows > total - first_row) {
        nk::set_error("row %s [%llu, %llu) out of range (index has %llu rows)", what, (unsigned long long)first_row,
                      (unsigned long long)(first_row + n_rows), (unsigned long long)total);
        return -1;
    }
    ShardOrder order(ix);
    if (order.failed()) return -1;
    for (uint64_t i = 0; i < n_rows;) {
        uint64_t local;
        NkShard *s = find_shard(ix, first_row + i, &local);
        const uint64_t cnt = std::min<uint64_t>(n_rows - i, s->n - local);
        NK_CUDA_OK(cudaSetDevice(s->device));
        if (values ? shard_values_on(*s) : shard_tags_on(*s)) return -1;
        NK_CUDA_OK(cudaMemcpyAsync((values ? s->values : s->tags) + local, words_host + i, cnt * 8, cudaMemcpyHostToDevice, s->stream));
        NK_CUDA_OK(cudaStreamSynchronize(s->stream));
        ix->stats.bytes_h2d += cnt * 8;
        i += cnt;
    }
    return 0;
}

int nk_index_set_row_tags(NkIndex *ix, uint64_t first_row, const uint64_t *tags_host, uint64_t n_rows) {
    return set_row_words(ix, first_row, tags_host, n_rows, false);
}

int nk_index_set_row_values(NkIndex *ix, uint64_t first_row, const uint64_t *keys_host, uint64_t n_rows) {
    return set_row_words(ix, first_row, keys_host, n_rows, true);
}

int nk_index_set_path(NkIndex *ix, int path) {
    if (!ix || path < NK_PATH_AUTO || path > NK_PATH_TENSOR_SHADOW) { nk::set_error("bad path"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    ix->path = path;
    return 0;
}

uint64_t nk_index_rows(const NkIndex *ix) { return ix ? ix->rows() : 0; }

int nk_index_stats(const NkIndex *ix, NkStats *out) {
    if (!ix || !out) { nk::set_error("null argument"); return -1; }
    *out = ix->stats;
    out->rows = ix->rows();
    return 0;
}

// Shard 0's status words once its device has drained (diagnostics); out is the caller's output, checked for null here.
static int shard0_status_words(NkIndex *ix, const void *out, int h[nk::NK_FLAG_WORDS]) {
    if (!ix || !out || ix->shards.empty()) { nk::set_error("null argument"); return -1; }
    NkShard &s = ix->shards[0];
    NK_CUDA_OK(cudaSetDevice(s.device));
    NK_CUDA_OK(cudaDeviceSynchronize());
    NK_CUDA_OK(cudaMemcpy(h, s.ws.flags, sizeof(int) * nk::NK_FLAG_WORDS, cudaMemcpyDeviceToHost));
    return 0;
}

int nk_index_debug_flags(NkIndex *ix, int out[4]) {
    nk::DeviceGuard _restore_device;
    int h[nk::NK_FLAG_WORDS];
    if (shard0_status_words(ix, out, h)) return -1;
    out[0] = h[nk::FLAG_FATAL]; out[1] = h[nk::FLAG_OVERFLOW]; out[2] = h[nk::FLAG_MAXXX]; out[3] = h[nk::FLAG_RETRY];
    return 0;
}

// Cumulative diagnostics of shard 0 since creation: out[0] = filter searches whose first (16-bit) stage overflowed and re-ran
// through the TF32 filter, out[1] = filter searches that fell through to the exact kernels, out[2] = longest per-query
// survivor list of the last filter search.  bench.py reports out[0..1] / searches as the retry rate of a corpus.
int nk_index_debug_counters(NkIndex *ix, uint64_t out[4]) {
    nk::DeviceGuard _restore_device;
    int h[nk::NK_FLAG_WORDS];
    if (shard0_status_words(ix, out, h)) return -1;
    out[0] = (uint64_t)h[nk::FLAG_N_RETRY]; out[1] = (uint64_t)h[nk::FLAG_N_EXACT]; out[2] = (uint64_t)h[nk::FLAG_LONGEST]; out[3] = (uint64_t)h[nk::FLAG_OVF_BITS];
    return 0;
}

// Tests only: the raw score estimate and the error bound the filter kernels work with, for every (row, query) pair of a
// single-device index (rows x Q floats each, row-major [row][query], host buffers).  which = NK_PATH_TENSOR_FILTER (TF32
// pass over fp32 rows) or NK_PATH_TENSOR_SHADOW (16-bit pass).  The filters are sound iff |est - exact score| <= bnd.
int nk_debug_filter_dump(NkIndex *ix, const float *queries_host, uint32_t Q, int which, float *est_host, float *bnd_host) {
    nk::DeviceGuard _restore_device;
    NkShard *s;
    if (!ix || ix->shards.size() != 1) { nk::set_error("single-device index required"); return -1; }
    s = &ix->shards[0];
    std::lock_guard<std::mutex> lk(ix->mu);
    if (!queries_host || !est_host || !bnd_host || Q == 0 || Q > 64 || s->n == 0) { nk::set_error("bad argument (1 <= Q <= 64, non-empty index)"); return -1; }
    ShardOrder order(*s, s->stream);
    if (order.failed()) return -1;
    NK_CUDA_OK(cudaSetDevice(s->device));
    const size_t cells = (size_t)s->n * Q;
    float *d = nullptr;
    NK_CUDA_OK(cudaMalloc((void **)&d, cells * 8));
    int rc = -1;
    do {
        if (nk::ws_reserve((void **)&s->ws.queries, &s->ws.queries_bytes, (size_t)Q * ix->dim * 4)) break;
        if (cudaMemcpyAsync(s->ws.queries, queries_host, (size_t)Q * ix->dim * 4, cudaMemcpyHostToDevice, s->stream) != cudaSuccess) break;
        if (cudaMemsetAsync(d, 0, cells * 8, s->stream) != cudaSuccess) break;
        nk::ScanArgs a = shard_scan_args(ix, *s, s->ws.queries, Q, 1, s->stream);
        a.image = shard_image(ix, *s, true, 1);
        a.row_mask = nullptr;  // every pair (the dump ignores the score floor itself)
        if (nk::scan_filter_dump(s->di, a, s->ws, which, d, d + cells, Q, &ix->stats.kernel_launches)) break;
        if (cudaMemcpyAsync(est_host, d, cells * 4, cudaMemcpyDeviceToHost, s->stream) != cudaSuccess) break;
        if (cudaMemcpyAsync(bnd_host, d + cells, cells * 4, cudaMemcpyDeviceToHost, s->stream) != cudaSuccess) break;
        if (cudaStreamSynchronize(s->stream) != cudaSuccess) break;
        rc = 0;
    } while (0);
    if (rc != 0) {
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) nk::set_error("nk_debug_filter_dump: %s", cudaGetErrorString(e));
        cudaStreamSynchronize(s->stream);
    }
    cudaFree(d);
    return rc;
}

int nk_index_last_path(const NkIndex *ix) { return ix ? ix->last_path : -1; }

int nk_index_enable_timing(NkIndex *ix, int enabled) {
    if (!ix) { nk::set_error("null index"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    ix->timing_on = enabled != 0;
    return 0;
}

int nk_index_scan_time_ms(NkIndex *ix, double *total_ms, uint64_t *scan_launches) {
    nk::DeviceGuard _restore_device;
    if (!ix || !total_ms || !scan_launches) { nk::set_error("null argument"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    double ms = 0.0;
    uint64_t n = 0;
    for (auto &s : ix->shards) {
        NK_CUDA_OK(cudaSetDevice(s.device));
        for (size_t i = 0; i < s.timing.size(); ++i) {
            float t = 0.0f;
            NK_CUDA_OK(cudaEventSynchronize(s.timing[i].second));
            NK_CUDA_OK(cudaEventElapsedTime(&t, s.timing[i].first, s.timing[i].second));
            ms += t;
            n += s.timing_launches[i];
            cudaEventDestroy(s.timing[i].first);
            cudaEventDestroy(s.timing[i].second);
        }
        s.timing.clear();
        s.timing_launches.clear();
    }
    *total_ms = ms;
    *scan_launches = n;
    return 0;
}

int nk_index_read_rows(NkIndex *ix, uint64_t row, uint64_t n_rows, void *rows_host) {
    nk::DeviceGuard _restore_device;
    if (!ix || (!rows_host && n_rows)) { nk::set_error("null argument"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    ShardOrder order(ix);
    if (order.failed()) return -1;
    const size_t rb = (size_t)ix->dim * ix->esz();
    for (uint64_t i = 0; i < n_rows;) {
        uint64_t local;
        NkShard *s = find_shard(ix, row + i, &local);
        if (!s) { nk::set_error("row %llu out of range", (unsigned long long)(row + i)); return -1; }
        uint64_t cnt = std::min<uint64_t>(n_rows - i, s->n - local);
        NK_CUDA_OK(cudaSetDevice(s->device));
        NK_CUDA_OK(cudaMemcpyAsync((char *)rows_host + i * rb, (const char *)s->rows + local * rb, cnt * rb, cudaMemcpyDeviceToHost, s->stream));
        NK_CUDA_OK(cudaStreamSynchronize(s->stream));
        ix->stats.bytes_d2h += cnt * rb;
        i += cnt;
    }
    return 0;
}

// Writes the Q fp32 queries of a search into s.ws.queries (already reserved) on s.stream; the device is s's.
using StageQueries = std::function<int(NkShard &)>;

// n tag filters -> a grow-only device array *dev, on `stream`: filters_host [n], or with filters_host nullptr {0,0,0}, which
// admit every tag (a window scan is also a tag scan, and a windowed graph's row filters are those of a graph without filters).
static int put_filters(NkIndex *ix, NkFilter **dev, size_t *dev_bytes, const NkFilter *filters_host, uint64_t n, cudaStream_t stream) {
    const size_t bytes = n * sizeof(NkFilter);
    if (nk::ws_reserve((void **)dev, dev_bytes, bytes)) return -1;
    if (!filters_host) {
        NK_CUDA_OK(cudaMemsetAsync(*dev, 0, bytes, stream));
        return 0;
    }
    NK_CUDA_OK(cudaMemcpyAsync(*dev, filters_host, bytes, cudaMemcpyHostToDevice, stream));
    ix->stats.bytes_h2d += bytes;
    return 0;
}

// The per-query predicates a scan in mode m reads, for Q queries -> shard s's workspace, on `stream`, next to the queries (the
// deferred retry tail reads them after the call's first synchronisation): under a tag mode the shard's tag array on and the
// filters in s.ws.qfilter (put_filters: filters_host, or {0,0,0}); under a window mode also the shard's value array on and
// windows_host in s.ws.qwindow (nullptr: the windows are written on the device, or the caller passes its own).
static int stage_predicates(NkIndex *ix, NkShard &s, cudaStream_t stream, nk::ScanMode m, uint32_t Q, const NkFilter *filters_host,
                            const NkWindow *windows_host) {
    if (!nk::mode_tags(m)) return 0;
    if (shard_tags_on(s) || put_filters(ix, &s.ws.qfilter, &s.ws.qfilter_bytes, filters_host, Q, stream)) return -1;
    if (!nk::mode_window(m)) return 0;
    if (shard_values_on(s)) return -1;
    if (!windows_host) return 0;
    const size_t wbytes = (size_t)Q * sizeof(NkWindow);
    if (nk::ws_reserve((void **)&s.ws.qwindow, &s.ws.qwindow_bytes, wbytes)) return -1;
    NK_CUDA_OK(cudaMemcpyAsync(s.ws.qwindow, windows_host, wbytes, cudaMemcpyHostToDevice, stream));
    ix->stats.bytes_h2d += wbytes;
    return 0;
}

// What one call asks of every search it runs, passed down by reference: the scan path (the index's setting, or the one a
// graph call chose) and the per-query tag filters and value windows of its queries.
struct SearchOpts {
    int path;
    const NkFilter *filters_host = nullptr;  // [Q], nullptr: none
    const NkWindow *windows_host = nullptr;  // [Q], nullptr: none
};

// One synchronous search of Q staged queries over the live (non-empty) shards, the index lock held: scan, deferred retry
// tail, merge; writes ke results per query into out_idx / out_score [Q x k] (row stride k) and returns ke.
static int search_live(NkIndex *ix, const std::vector<NkShard *> &live, const StageQueries &stage, const SearchOpts &opts, uint32_t Q,
                       uint32_t ke, uint32_t k, uint32_t *out_idx, float *out_score) {
    const size_t qbytes = (size_t)Q * ix->dim * sizeof(float);
    const nk::ScanMode mode = opts.windows_host ? nk::ScanMode::KNN_WINDOW : opts.filters_host ? nk::ScanMode::KNN_TAGS : nk::ScanMode::KNN;
    const bool single = live.size() == 1;
    // one deferred tail per shard; a single shard's lives on the stack, so that search allocates nothing
    DeferredTail tail0;
    std::vector<DeferredTail> tails(single ? 0 : live.size());
    const auto tail_of = [&](size_t i) { return single ? &tail0 : &tails[i]; };

    // Launch every shard asynchronously, then collect.  A single shard writes the decoded (index, score) arrays from
    // the last kernel of its path (no separate decode launch); the retry stages of the filter paths are deferred.
    for (size_t i = 0; i < live.size(); ++i) {
        NkShard *s = live[i];
        NK_CUDA_OK(cudaSetDevice(s->device));
        if (nk::ws_reserve((void **)&s->ws.queries, &s->ws.queries_bytes, qbytes)) return -1;
        if (nk::ws_reserve((void **)&s->ws.keys, &s->ws.keys_bytes, (size_t)Q * ke * 8)) return -1;
        ScanOut xo(opts.path, mode);
        xo.tail = tail_of(i);
        if (single) {
            if (nk::ws_reserve((void **)&s->ws.out_idx, &s->ws.out_idx_bytes, (size_t)Q * ke * 4)) return -1;
            if (nk::ws_reserve((void **)&s->ws.out_score, &s->ws.out_score_bytes, (size_t)Q * ke * 4)) return -1;
            xo.out_idx = s->ws.out_idx; xo.out_score = s->ws.out_score;
        }
        if (stage(*s) || stage_predicates(ix, *s, s->stream, mode, Q, opts.filters_host, opts.windows_host)) return -1;
        if (run_scan(ix, *s, s->ws.queries, Q, ke, s->ws.keys, s->stream, xo)) return -1;
    }

    if (single) {
        // Results and status words come back through ONE pinned staging buffer: three short DMA copies and a single stream
        // synchronisation (pageable cudaMemcpyAsync targets cost a driver-side staging round trip each).
        NkShard *s = live[0];
        NK_CUDA_OK(cudaSetDevice(s->device));
        const size_t rbytes = (size_t)Q * ke * 4;
        if (pinned_reserve((void **)&s->h_res, &s->h_res_bytes, 2 * rbytes + sizeof(int) * nk::NK_FLAG_WORDS)) return -1;
        int *hflags = reinterpret_cast<int *>(s->h_res + 2 * rbytes);
        for (int st = 1; st;) {  // read, and once more after a retry tail
            NK_CUDA_OK(cudaMemcpyAsync(s->h_res, s->ws.out_idx, rbytes, cudaMemcpyDeviceToHost, s->stream));
            NK_CUDA_OK(cudaMemcpyAsync(s->h_res + rbytes, s->ws.out_score, rbytes, cudaMemcpyDeviceToHost, s->stream));
            NK_CUDA_OK(cudaMemcpyAsync(hflags, s->ws.flags, sizeof(int) * nk::NK_FLAG_WORDS, cudaMemcpyDeviceToHost, s->stream));
            NK_CUDA_OK(cudaStreamSynchronize(s->stream));
            ix->stats.bytes_d2h += (uint64_t)Q * ke * 8;
            if ((st = shard_status(ix, *s, hflags, &tail0)) < 0) return -1;
        }
        const uint32_t *hi = reinterpret_cast<const uint32_t *>(s->h_res);
        const float *hs = reinterpret_cast<const float *>(s->h_res + rbytes);
        if (ke == k) {
            memcpy(out_idx, hi, rbytes);
            memcpy(out_score, hs, rbytes);
        } else {
            for (uint32_t q = 0; q < Q; ++q) {
                memcpy(out_idx + (size_t)q * k, hi + (size_t)q * ke, (size_t)ke * 4);
                memcpy(out_score + (size_t)q * k, hs + (size_t)q * ke, (size_t)ke * 4);
            }
        }
        return (int)ke;
    }

    // Multi-shard: gather the per-GPU candidate lists (Q*k*8 B each) and merge on the host with the
    // same (score desc, row asc) order (SURVEY.md §8e "small Q: async D2H + host k-way merge").
    const size_t kbytes = (size_t)Q * ke * 8;
    for (NkShard *s : live) {
        NK_CUDA_OK(cudaSetDevice(s->device));
        if (pinned_reserve((void **)&s->h_keys, &s->h_keys_bytes, kbytes)) return -1;
    }
    for (size_t i = 0; i < live.size(); ++i) {
        NkShard *s = live[i];
        NK_CUDA_OK(cudaSetDevice(s->device));
        if (finish_deferred(ix, *s, tail_of(i)) < 0) return -1;  // runs this shard's retry stages if it needs them
        NK_CUDA_OK(cudaMemcpyAsync(s->h_keys, s->ws.keys, kbytes, cudaMemcpyDeviceToHost, s->stream));
        ix->stats.bytes_d2h += kbytes;
    }
    for (NkShard *s : live) {
        NK_CUDA_OK(cudaSetDevice(s->device));
        NK_CUDA_OK(cudaStreamSynchronize(s->stream));
    }
    std::vector<uint64_t> tmp(live.size() * (size_t)ke);
    for (uint32_t q = 0; q < Q; ++q) {
        size_t m = 0;
        for (NkShard *s : live)
            for (uint32_t i = 0; i < ke; ++i) {
                uint64_t key = s->h_keys[(size_t)q * ke + i];
                if (key) tmp[m++] = key;
            }
        size_t take = std::min<size_t>(ke, m);
        std::partial_sort(tmp.begin(), tmp.begin() + take, tmp.begin() + m, std::greater<uint64_t>());
        for (uint32_t i = 0; i < ke; ++i) {
            if (i < take) {
                decode_key(ix->metric, tmp[i], out_idx + (size_t)q * k + i, out_score + (size_t)q * k + i);
            } else {
                out_idx[(size_t)q * k + i] = 0xffffffffu;
                out_score[(size_t)q * k + i] = 0.0f;
            }
        }
    }
    return (int)ke;
}

// nk_search / nk_search_filtered / nk_search_windowed: filters_host == windows_host == nullptr is plain nk_search.
static int search_host(NkIndex *ix, const float *queries_host, const NkFilter *filters_host, const NkWindow *windows_host, uint32_t Q,
                       uint32_t k, uint32_t *out_idx, float *out_score) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    const uint64_t N = ix->returnable_rows();
    if (k == 0 || N == 0 || Q == 0) return 0;  // cuda_bridge.go:644-646, gpu.go:1540-1542
    if (!queries_host || !out_idx || !out_score) { nk::set_error("null argument"); return -1; }
    const uint32_t ke = k > N ? (uint32_t)N : k;  // cuda_bridge.go:647-649
    if (ke > NK_MAX_K_TOTAL) { nk::set_error("k=%u exceeds NK_MAX_K_TOTAL=%u", ke, NK_MAX_K_TOTAL); return -1; }
    const size_t qbytes = (size_t)Q * ix->dim * sizeof(float);
    ix->stats.searches++;
    ix->stats.queries += Q;
    ScopedRange range("nk_search");
    ShardOrder order(ix);
    if (order.failed()) return -1;

    const std::vector<NkShard *> live = live_shards(ix);
    const StageQueries upload = [&](NkShard &s) {
        NK_CUDA_OK(cudaMemcpyAsync(s.ws.queries, queries_host, qbytes, cudaMemcpyHostToDevice, s.stream));
        ix->stats.bytes_h2d += qbytes;
        return 0;
    };
    return search_live(ix, live, upload, SearchOpts{ix->path, filters_host, windows_host}, Q, ke, k, out_idx, out_score);
}

int nk_search(NkIndex *ix, const float *queries_host, uint32_t Q, uint32_t k, uint32_t *out_idx, float *out_score) {
    return search_host(ix, queries_host, nullptr, nullptr, Q, k, out_idx, out_score);
}

int nk_search_filtered(NkIndex *ix, const float *queries_host, const NkFilter *filters_host, uint32_t Q, uint32_t k,
                       uint32_t *out_idx, float *out_score) {
    return search_host(ix, queries_host, filters_host, nullptr, Q, k, out_idx, out_score);
}

int nk_search_windowed(NkIndex *ix, const float *queries_host, const NkFilter *filters_host, const NkWindow *windows_host,
                       uint32_t Q, uint32_t k, uint32_t *out_idx, float *out_score) {
    return search_host(ix, queries_host, filters_host, windows_host, Q, k, out_idx, out_score);
}

// ---- search by stored row (DESIGN.md §3.5c) ---------------------------------------------------------------------------
// Each query is a stored row, gathered (and widened to fp32) on the device that owns it.  The scan asks for k' = min(k+1, N)
// and the host drops the query's own row from the decoded list, or the last slot if its row is not in it: the k'-list is a
// prefix of the (score desc, row asc) order over the admissible rows, so either way the rest is the top of the other rows.
// Queries run in blocks of SEARCH_ROWS_BLOCK, which bounds the workspace (the 16-bit scan's survivor lists grow with Q)
// whatever Q is, the whole index included; one host synchronisation per block.
constexpr uint32_t SEARCH_ROWS_BLOCK = 1024;

// What stage_row_block writes beside a block of stored-row queries, by the mode of the scan they run in.  Under a tag mode
// (the self-join's and the reverse scan's range modes) each query's filter goes into s.ws.qfilter, with the shard's tag array
// on: f for a row that passes the row mask and f (nk::row_filters), the filter that admits no row otherwise, decided on the
// row's own device.  Under a window mode (a windowed self-join: a window w, a band gap or both) each row's window
// (nk::row_windows) goes into s.ws.qwindow instead, with the shard's value array on, and decides the row's admission alone
// (mask, filter, window and band: a refused row gets the window that admits no row), so every query's filter is f and
// row_filters does not run.  The other modes (KNN, RANGE, REVERSE) write nothing beside the queries.
struct RowAdmit {
    nk::ScanMode mode = nk::ScanMode::KNN;
    NkFilter f{0, 0, 0};
    NkWindow w{0, ~0ull};
    uint64_t gap = NK_NO_GAP;
};

// The admission of a self-join's left rows (nk_search_pairs_windowed, nk_search_pairs_rows_windowed): the call's filter, window and
// band and the index's row mask, and the range mode the join scans in.
static RowAdmit join_admit(const NkIndex *ix, const NkFilter *filter, const NkWindow *window, uint64_t max_gap) {
    RowAdmit adm;
    adm.mode = window || max_gap != NK_NO_GAP ? nk::ScanMode::RANGE_WINDOW
               : filter || ix->mask_on        ? nk::ScanMode::RANGE_TAGS  // some left rows may be inadmissible: per-query filters
                                              : nk::ScanMode::RANGE;
    if (filter) adm.f = *filter;
    if (window) adm.w = *window;
    adm.gap = max_gap;
    return adm;
}

// The admission (RowAdmit, a tag or window mode) of m rows of shard o, their local ids in o.ws.sub_rows: one launch on o's
// stream, into o.ws.qwindow (nk::row_windows) under a window mode, else into o.ws.qfilter (nk::row_filters).
static int admit_rows(NkIndex *ix, NkShard &o, uint32_t m, const RowAdmit &adm) {
    const uint32_t *mask = o.mask_on ? o.mask : nullptr;
    const uint64_t *tags = o.tags_on ? o.tags : nullptr;
    if (nk::mode_window(adm.mode)) {
        if (nk::ws_reserve((void **)&o.ws.qwindow, &o.ws.qwindow_bytes, (size_t)m * sizeof(NkWindow))) return -1;
        if (nk::row_windows(o.ws.sub_rows, m, mask, tags, o.values_on ? o.values : nullptr, adm.f, adm.w, adm.gap, o.ws.qwindow, o.stream))
            return -1;
    } else {
        if (nk::ws_reserve((void **)&o.ws.qfilter, &o.ws.qfilter_bytes, (size_t)m * sizeof(NkFilter))) return -1;
        if (nk::row_filters(o.ws.sub_rows, m, mask, tags, adm.f, o.ws.qfilter, o.stream)) return -1;
    }
    ix->stats.kernel_launches++;
    return 0;
}

// The queries of a block of stored rows ids[nb] (relative to the index's first row), each read and widened to fp32 on the
// device that holds it, and their admission under adm.  *stage then writes the block into s.ws.queries (reserved by the
// caller) of any shard the search runs on, the admission beside it.  With one live shard only the ids cross PCIe, the rows
// are gathered straight into the query block and the admission is written in place; otherwise each owner gathers its rows and
// admits them now, the block is assembled in pinned host memory and *stage sends it.
static int stage_row_block(NkIndex *ix, const std::vector<NkShard *> &live, const uint32_t *ids, uint32_t nb, const RowAdmit &adm,
                           StageQueries *stage) {
    const size_t rb = (size_t)ix->dim * sizeof(float);
    const bool admit = nk::mode_tags(adm.mode), win = nk::mode_window(adm.mode);
    std::vector<uint32_t> local(nb);
    if (live.size() == 1) {
        std::vector<NkFilter> every(win ? nb : 0, adm.f);  // a windowed block's filters: f for every query
        *stage = [ix, ids, nb, local, adm, admit, win, every](NkShard &s) mutable {
            for (uint32_t q = 0; q < nb; ++q) local[q] = ids[q] - (uint32_t)ix->first_row(s);
            if (nk::ws_reserve((void **)&s.ws.sub_rows, &s.ws.sub_rows_bytes, (size_t)nb * 4)) return -1;
            NK_CUDA_OK(cudaMemcpyAsync(s.ws.sub_rows, local.data(), (size_t)nb * 4, cudaMemcpyHostToDevice, s.stream));
            if (nk::gather_rows(s.rows, ix->dtype, ix->dim, s.ws.sub_rows, nb, s.ws.queries, true, s.stream)) return -1;
            ix->stats.bytes_h2d += (uint64_t)nb * 4;
            ix->stats.kernel_launches++;
            if (!admit) return 0;
            if (win ? stage_predicates(ix, s, s.stream, adm.mode, nb, every.data(), nullptr) : shard_tags_on(s)) return -1;
            return admit_rows(ix, s, nb, adm);
        };
        return 0;
    }
    // the block may straddle shards: gather on each owner, assemble in pinned host memory, send to every shard
    if (pinned_reserve((void **)&ix->h_qrows, &ix->h_qrows_bytes, 2 * nb * rb)) return -1;
    float *blk = ix->h_qrows, *part = ix->h_qrows + (size_t)nb * ix->dim;
    std::vector<uint32_t> pos(nb);
    std::vector<NkFilter> filters(admit ? nb : 0, adm.f), part_f(admit && !win ? nb : 0);
    std::vector<NkWindow> windows(win ? nb : 0), part_w(win ? nb : 0);
    for (NkShard *o : live) {
        uint32_t m = 0;
        for (uint32_t q = 0; q < nb; ++q) {
            uint64_t l;
            if (find_shard(ix, ids[q], &l) == o) { pos[m] = q; local[m++] = (uint32_t)l; }
        }
        if (m == 0) continue;
        NK_CUDA_OK(cudaSetDevice(o->device));
        if (nk::ws_reserve((void **)&o->ws.sub_rows, &o->ws.sub_rows_bytes, (size_t)m * 4)) return -1;
        if (nk::ws_reserve(&o->ws.sub_gather, &o->ws.sub_gather_bytes, (size_t)m * rb)) return -1;
        NK_CUDA_OK(cudaMemcpyAsync(o->ws.sub_rows, local.data(), (size_t)m * 4, cudaMemcpyHostToDevice, o->stream));
        if (nk::gather_rows(o->rows, ix->dtype, ix->dim, o->ws.sub_rows, m, o->ws.sub_gather, true, o->stream)) return -1;
        NK_CUDA_OK(cudaMemcpyAsync(part, o->ws.sub_gather, (size_t)m * rb, cudaMemcpyDeviceToHost, o->stream));
        if (admit) {  // the owner's qfilter / qwindow slot is free until the scan stages its own
            if (admit_rows(ix, *o, m, adm)) return -1;
            if (win) NK_CUDA_OK(cudaMemcpyAsync(part_w.data(), o->ws.qwindow, (size_t)m * sizeof(NkWindow), cudaMemcpyDeviceToHost, o->stream));
            else NK_CUDA_OK(cudaMemcpyAsync(part_f.data(), o->ws.qfilter, (size_t)m * sizeof(NkFilter), cudaMemcpyDeviceToHost, o->stream));
            ix->stats.bytes_d2h += (uint64_t)m * (win ? sizeof(NkWindow) : sizeof(NkFilter));
        }
        NK_CUDA_OK(cudaStreamSynchronize(o->stream));
        ix->stats.bytes_h2d += (uint64_t)m * 4;
        ix->stats.bytes_d2h += (uint64_t)m * rb;
        ix->stats.kernel_launches++;
        for (uint32_t i = 0; i < m; ++i) {
            memcpy(blk + (size_t)pos[i] * ix->dim, part + (size_t)i * ix->dim, rb);
            if (win) windows[pos[i]] = part_w[i];
            else if (admit) filters[pos[i]] = part_f[i];
        }
    }
    *stage = [ix, blk, nb, rb, mode = adm.mode, filters, windows](NkShard &s) {
        NK_CUDA_OK(cudaMemcpyAsync(s.ws.queries, blk, (size_t)nb * rb, cudaMemcpyHostToDevice, s.stream));
        ix->stats.bytes_h2d += (uint64_t)nb * rb;
        return stage_predicates(ix, s, s.stream, mode, nb, filters.data(), windows.data());
    };
    return 0;
}

// The body of nk_search_rows, nk_search_rows_filtered and nk_search_rows_windowed (opts.filters_host / opts.windows_host [Q] or
// nullptr), the index lock held and the ids checked: returns ke, the entries written per query (the rest of each k-wide output row is left as it is).
static int search_rows_locked(NkIndex *ix, const std::vector<NkShard *> &live, const uint32_t *rows_host, const SearchOpts &opts,
                              uint32_t Q, uint32_t k, uint32_t *out_idx, float *out_score) {
    const uint64_t N = ix->returnable_rows();
    const uint32_t kk = (uint32_t)std::min<uint64_t>((uint64_t)k + 1, N);  // asked of the scan
    const uint32_t ke = (uint32_t)std::min<uint64_t>(k, N);                // returned
    const uint32_t QB = std::min(Q, SEARCH_ROWS_BLOCK);
    std::vector<uint32_t> bidx((size_t)QB * kk);
    std::vector<float> bsc((size_t)QB * kk);
    for (uint32_t b = 0; b < Q; b += QB) {
        const uint32_t nb = std::min(QB, Q - b);
        const uint32_t *ids = rows_host + b;
        StageQueries stage;
        if (stage_row_block(ix, live, ids, nb, RowAdmit{}, &stage)) return -1;
        const SearchOpts block{opts.path, opts.filters_host ? opts.filters_host + b : nullptr, opts.windows_host ? opts.windows_host + b : nullptr};
        if (search_live(ix, live, stage, block, nb, kk, kk, bidx.data(), bsc.data()) < 0) return -1;
        for (uint32_t q = 0; q < nb; ++q) {
            const uint32_t self = (uint32_t)(ix->row_base + ids[q]);
            const uint32_t *ri = bidx.data() + (size_t)q * kk;
            const float *rs = bsc.data() + (size_t)q * kk;
            uint32_t drop = kk - 1;
            for (uint32_t j = 0; j < kk; ++j)
                if (ri[j] == self) { drop = j; break; }
            uint32_t *oi = out_idx + (size_t)(b + q) * k;
            float *os = out_score + (size_t)(b + q) * k;
            uint32_t w = 0;
            for (uint32_t j = 0; j < kk && w < ke; ++j)
                if (j != drop) { oi[w] = ri[j]; os[w] = rs[j]; ++w; }
            for (; w < ke; ++w) { oi[w] = 0xffffffffu; os[w] = 0.0f; }  // k >= N: one admissible row fewer than k'
        }
    }
    return (int)ke;
}

// nk_search_rows / nk_search_rows_filtered / nk_search_rows_windowed: filters_host == windows_host == nullptr is plain
// nk_search_rows.
static int search_rows_host(NkIndex *ix, const char *what, const uint32_t *rows_host, const NkFilter *filters_host,
                            const NkWindow *windows_host, uint32_t Q, uint32_t k, uint32_t *out_idx, float *out_score) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    if (Q && (!rows_host || !out_idx || !out_score)) { nk::set_error("null argument"); return -1; }
    if (k > NK_MAX_K_TOTAL - 1) { nk::set_error("%s: k=%u exceeds NK_MAX_K_TOTAL - 1 = %u", what, k, NK_MAX_K_TOTAL - 1); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    const uint64_t total = ix->rows();
    const uint64_t N = ix->returnable_rows();
    if (k == 0 || N == 0 || Q == 0) return 0;
    for (uint32_t q = 0; q < Q; ++q)
        if (rows_host[q] >= total) {
            nk::set_error("%s: row %u (query %u) out of range, index has %llu rows", what, rows_host[q], q, (unsigned long long)total);
            return -1;
        }
    ix->stats.searches++;
    ix->stats.queries += Q;
    ScopedRange range(what);
    ShardOrder order(ix);
    if (order.failed()) return -1;
    return search_rows_locked(ix, live_shards(ix), rows_host, SearchOpts{ix->path, filters_host, windows_host}, Q, k, out_idx, out_score);
}

int nk_search_rows(NkIndex *ix, const uint32_t *rows_host, uint32_t Q, uint32_t k, uint32_t *out_idx, float *out_score) {
    return search_rows_host(ix, "nk_search_rows", rows_host, nullptr, nullptr, Q, k, out_idx, out_score);
}

int nk_search_rows_filtered(NkIndex *ix, const uint32_t *rows_host, const NkFilter *filters_host, uint32_t Q, uint32_t k,
                            uint32_t *out_idx, float *out_score) {
    return search_rows_host(ix, "nk_search_rows_filtered", rows_host, filters_host, nullptr, Q, k, out_idx, out_score);
}

int nk_search_rows_windowed(NkIndex *ix, const uint32_t *rows_host, const NkFilter *filters_host, const NkWindow *windows_host,
                            uint32_t Q, uint32_t k, uint32_t *out_idx, float *out_score) {
    return search_rows_host(ix, "nk_search_rows_windowed", rows_host, filters_host, windows_host, Q, k, out_idx, out_score);
}

// ---- range search ---------------------------------------------------------------------------------------------------
// Threshold of the API (cosine / dot: minimum score; euclidean: maximum distance) -> key space (score; -distance^2), the
// index floor folded in: the stricter one wins.  Euclidean: a row qualifies iff the distance it is returned with,
// sqrtf(d), is <= t, i.e. iff d <= the largest float whose sqrtf is <= t (sqrtf is correctly rounded, here as on the device),
// so a threshold taken from a returned distance admits that row.  A negative maximum distance admits no row.
static float range_key_threshold(const NkIndex *ix, float t) {
    float key = t;
    if (ix->metric == NK_METRIC_EUCLIDEAN) {
        if (t < 0.0f) {
            key = INFINITY;
        } else if (t == INFINITY) {
            key = -INFINITY;
        } else {
            float d = t * t;
            while (d < INFINITY && sqrtf(nextafterf(d, INFINITY)) <= t) d = nextafterf(d, INFINITY);
            while (d > 0.0f && sqrtf(d) > t) d = nextafterf(d, 0.0f);
            key = -d;
        }
    }
    return std::max(key, ix->key_floor());
}

// One block of Q range queries as every shard it runs on scans it.  The queries are those the block's StageQueries wrote into
// s.ws.queries; the same step wrote what the block's mode reads beside them (set_scan_mode: stage_predicates, stage_row_block,
// and for the reverse scan of a k-NN graph update graph_reverse_scan, whose per-row thresholds and keep mask select the rows
// whose lists are updated, not the rows that may be returned).
struct RangeBlock {
    int path;                              // the scan path of the call (plan_path)
    nk::ScanMode mode;                     // a range mode
    uint32_t Q;
    const uint32_t *thr;                   // [Q] thresholds in key space, as nk::ord_bits (host)
    const uint64_t *pair_first = nullptr;  // the self-join's triangle: see range_scan_shard
    // The pairs incident to listed rows (nk_search_pairs_rows): s.ws.pair_rows holds one bit per row of the shard for the
    // listed rows, then the block's query rows (global ids); see nk::IncidentRows.
    bool incident = false;
};

// One shard's range scan of a block, rows [from, s.n): path, scan and exact re-scoring -> counts[Q] (host), *list_cap
// (range_scan_shard).  from > 0 (the self-join's triangular window) is a multiple of the 256-row scan tile, so the window's
// row-mask words, TMA base and 16-byte alignment are those of the shard; the window gets its own TMA maps (tc_cached_map keys
// on the base).
static int range_shard(NkIndex *ix, NkShard &s, const RangeBlock &b, uint64_t from, int *counts, uint32_t *list_cap) {
    // Paths: the 16-bit and TF32 filters with fixed thresholds, or the CUDA-core scan.
    nk::ScanArgs a = shard_scan_args(ix, s, s.ws.queries, b.Q, 1, s.stream);
    set_scan_mode(s, b.mode, &a);
    const int use = plan_path(ix, s, b.path, true, &a);
    if (use < 0) return -1;
    if (from) {
        a.rows = static_cast<const char *>(a.rows) + from * ix->dim * ix->esz();
        a.n = (uint32_t)(s.n - from);
        a.row_base = s.base + from;
        if (a.row_mask) a.row_mask += from / 32;
        if (a.row_tags) a.row_tags += from;
        if (a.row_values) a.row_values += from;
        a.image = a.image.window(from);
    }
    ScanTimer timer(s);
    if (timer.attach(ix, &a)) return -1;
    int retried = 0;
    nk::IncidentRows inc{nullptr, nullptr};
    if (b.incident) inc = {s.ws.pair_rows + (s.n + 31) / 32, s.ws.pair_rows};  // reserved by pairs_rows_locked
    if (nk::range_scan_shard(s.di, a, use != NK_PATH_SIMT, b.thr, s.ws, &ix->stats.kernel_launches, counts, list_cap, &retried, b.pair_first,
                             b.incident ? &inc : nullptr))
        return -1;
    timer.keep();
    ix->last_path = use;
    ix->stats.bytes_scanned += scan_bytes(ix, use, a, retried ? 2 : 1);
    return 0;
}

// The shards a block of range queries runs on, and what their scans leave behind for range_collect.
struct RangeShards {
    std::vector<NkShard *> shards;
    std::vector<uint64_t> from;            // per shard: the first row scanned (range_shard); empty: every shard from row 0
    std::vector<std::vector<int>> counts;  // [shard][query] survivors
    std::vector<uint32_t> list_cap;        // per shard (range_scan_shard)
};

// Run one block of range queries over on->shards: on each, reserve the query block, stage it and scan.  *per_query [b.Q]: each
// query's survivors, summed over the shards (all zero if there is no shard to scan; `stage` is not called then).
static int range_scan(NkIndex *ix, RangeShards *on, const StageQueries &stage, const RangeBlock &b, std::vector<uint64_t> *per_query) {
    on->counts.assign(on->shards.size(), std::vector<int>(b.Q, 0));
    on->list_cap.assign(on->shards.size(), 0);
    per_query->assign(b.Q, 0);
    for (size_t i = 0; i < on->shards.size(); ++i) {
        NkShard &s = *on->shards[i];
        NK_CUDA_OK(cudaSetDevice(s.device));
        if (nk::ws_reserve((void **)&s.ws.queries, &s.ws.queries_bytes, (size_t)b.Q * ix->dim * sizeof(float))) return -1;
        if (stage(s)) return -1;
        if (range_shard(ix, s, b, on->from.empty() ? 0 : on->from[i], on->counts[i].data(), &on->list_cap[i])) return -1;
        for (uint32_t q = 0; q < b.Q; ++q) (*per_query)[q] += (uint64_t)on->counts[i][q];
    }
    return 0;
}

// After range_scan: each of the Q queries' survivors, the shards' sorted runs merged into nk_search's order (keys are unique
// across shards), appended to *out query after query.
static int range_collect(NkIndex *ix, const RangeShards &on, uint32_t Q, std::vector<uint64_t> *out) {
    const std::vector<NkShard *> &shards = on.shards;
    std::vector<std::vector<uint64_t>> keys(shards.size());
    std::vector<std::vector<uint64_t>> offs(shards.size(), std::vector<uint64_t>(Q + 1, 0));
    for (size_t i = 0; i < shards.size(); ++i) {
        NK_CUDA_OK(cudaSetDevice(shards[i]->device));
        if (nk::range_sorted_keys(shards[i]->di, shards[i]->ws, shards[i]->stream, Q, on.counts[i].data(), on.list_cap[i], &keys[i],
                                  &ix->stats.kernel_launches))
            return -1;
        ix->stats.bytes_d2h += keys[i].size() * 8;
        for (uint32_t q = 0; q < Q; ++q) offs[i][q + 1] = offs[i][q] + (uint64_t)on.counts[i][q];
    }
    std::vector<uint64_t> merged, tmp;
    for (uint32_t q = 0; q < Q; ++q) {
        merged.clear();
        for (size_t i = 0; i < shards.size(); ++i) {
            tmp.resize(merged.size() + (size_t)on.counts[i][q]);
            std::merge(merged.begin(), merged.end(), keys[i].begin() + offs[i][q], keys[i].begin() + offs[i][q + 1], tmp.begin(),
                       std::greater<uint64_t>());
            merged.swap(tmp);
        }
        out->insert(out->end(), merged.begin(), merged.end());
    }
    return 0;
}

// The end of a call that returns CSR lists, its offsets written: *out_total = total and, if the lists fit capacity (else the
// caller calls again with room) and are not empty, collect(&keys) gives them in order and they are written decoded.
static int write_csr(const NkIndex *ix, uint64_t total, uint64_t capacity, uint32_t *out_idx, float *out_score, uint64_t *out_total,
                     const std::function<int(std::vector<uint64_t> *)> &collect) {
    *out_total = total;
    if (total > capacity || total == 0) return 0;
    if (!out_idx || !out_score) { nk::set_error("null argument"); return -1; }
    std::vector<uint64_t> keys;
    if (collect(&keys)) return -1;
    for (size_t j = 0; j < keys.size(); ++j) decode_key(ix->metric, keys[j], out_idx + j, out_score + j);
    return 0;
}

int nk_search_range(NkIndex *ix, const float *queries_host, const float *thresholds_host, const NkFilter *filters_host, uint32_t Q,
                    uint64_t capacity, uint64_t *out_offsets, uint32_t *out_idx, float *out_score, uint64_t *out_total) {
    return nk_search_range_windowed(ix, queries_host, thresholds_host, filters_host, nullptr, Q, capacity, out_offsets, out_idx, out_score,
                                    out_total);
}

int nk_search_range_windowed(NkIndex *ix, const float *queries_host, const float *thresholds_host, const NkFilter *filters_host,
                             const NkWindow *windows_host, uint32_t Q, uint64_t capacity, uint64_t *out_offsets, uint32_t *out_idx,
                             float *out_score, uint64_t *out_total) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    if (!out_offsets || !out_total) { nk::set_error("null argument"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    out_offsets[0] = 0;
    *out_total = 0;
    if (Q == 0) return 0;
    if (!queries_host || !thresholds_host) { nk::set_error("null argument"); return -1; }
    std::vector<uint32_t> thr(Q);
    for (uint32_t q = 0; q < Q; ++q) {
        if (thresholds_host[q] != thresholds_host[q]) { nk::set_error("nk_search_range: threshold of query %u is NaN", q); return -1; }
        thr[q] = nk::ord_bits(range_key_threshold(ix, thresholds_host[q]));
    }
    ix->stats.searches++;
    ix->stats.queries += Q;
    ScopedRange range("nk_search_range");
    ShardOrder order(ix);
    if (order.failed()) return -1;
    RangeShards on{live_shards(ix)};
    const size_t qbytes = (size_t)Q * ix->dim * sizeof(float);
    const RangeBlock block{ix->path, windows_host   ? nk::ScanMode::RANGE_WINDOW
                                     : filters_host ? nk::ScanMode::RANGE_TAGS
                                                    : nk::ScanMode::RANGE,
                           Q, thr.data()};
    const StageQueries upload = [&](NkShard &s) {
        NK_CUDA_OK(cudaMemcpyAsync(s.ws.queries, queries_host, qbytes, cudaMemcpyHostToDevice, s.stream));
        ix->stats.bytes_h2d += qbytes;
        return stage_predicates(ix, s, s.stream, block.mode, Q, filters_host, windows_host);
    };
    std::vector<uint64_t> per_query;
    if (range_scan(ix, &on, upload, block, &per_query)) return -1;
    // offsets: the shards' survivors of query q are merged into one run
    for (uint32_t q = 0; q < Q; ++q) out_offsets[q + 1] = out_offsets[q] + per_query[q];
    return write_csr(ix, out_offsets[Q], capacity, out_idx, out_score, out_total, [&](std::vector<uint64_t> *keys) {
        keys->reserve(out_offsets[Q]);
        return range_collect(ix, on, Q, keys);
    });
}

// ---- similarity self-join (DESIGN.md §3.5d) ---------------------------------------------------------------------------
// The stripe's rows are range queries, one threshold for all, in blocks of SEARCH_ROWS_BLOCK consecutive rows gathered on the
// device as nk_search_rows gathers them.  For a block starting at row s0 the scan skips every shard whose rows all lie at or
// below s0, and in the shard holding s0 covers only the window from s0 rounded down to the 256-row scan tile; the re-scoring
// kernel keeps row j for the block's query q only if j > s0 + q.  Left rows that fail the row mask or the filter get the filter
// that admits no row, on the device that holds them.  A windowed join (a window, a band or both) also gives each left row its
// own value window on that device (nk::row_windows) and scans in the windowed range mode: the band is symmetric, so the
// triangle still holds each unordered pair once.  Each block's merged survivors are staged in host memory (8 B per pair)
// until the whole stripe is done, so the offsets and the total are exact before anything is written.
constexpr uint64_t SCAN_TILE_ROWS = 256;

int nk_search_pairs(NkIndex *ix, uint64_t first_row, uint64_t n_rows, float threshold, const NkFilter *filter, uint64_t capacity,
                    uint64_t *out_offsets, uint32_t *out_idx, float *out_score, uint64_t *out_total) {
    return nk_search_pairs_windowed(ix, first_row, n_rows, threshold, filter, nullptr, NK_NO_GAP, capacity, out_offsets, out_idx,
                                    out_score, out_total);
}

int nk_search_pairs_windowed(NkIndex *ix, uint64_t first_row, uint64_t n_rows, float threshold, const NkFilter *filter,
                             const NkWindow *window, uint64_t max_gap, uint64_t capacity, uint64_t *out_offsets, uint32_t *out_idx,
                             float *out_score, uint64_t *out_total) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    if (n_rows && (!out_offsets || !out_total)) { nk::set_error("null argument"); return -1; }
    if (threshold != threshold) { nk::set_error("nk_search_pairs: threshold is NaN"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    if (ix->path == NK_PATH_TENSOR) {
        nk::set_error("nk_search_pairs: the exact 3xTF32 path has no range mode (use AUTO, SIMT, TENSOR_FILTER or TENSOR_SHADOW)");
        return -1;
    }
    const uint64_t total_rows = ix->rows();
    if (first_row > total_rows || n_rows > total_rows - first_row) {
        nk::set_error("nk_search_pairs: rows [%llu, %llu) past the end of the index (%llu rows)", (unsigned long long)first_row,
                      (unsigned long long)(first_row + n_rows), (unsigned long long)total_rows);
        return -1;
    }
    if (out_offsets) out_offsets[0] = 0;
    if (out_total) *out_total = 0;
    if (n_rows == 0) return 0;
    ix->stats.searches++;
    ix->stats.queries += n_rows;
    ScopedRange range("nk_search_pairs");
    ShardOrder order(ix);
    if (order.failed()) return -1;

    const std::vector<NkShard *> live = live_shards(ix);
    const RowAdmit adm = join_admit(ix, filter, window, max_gap);
    const uint32_t QB = (uint32_t)std::min<uint64_t>(n_rows, SEARCH_ROWS_BLOCK);
    const std::vector<uint32_t> thr(QB, nk::ord_bits(range_key_threshold(ix, threshold)));
    std::vector<uint32_t> ids(QB);
    std::vector<uint64_t> keys;  // the result so far, [out_offsets[0], out_offsets[b])
    std::vector<uint64_t> per_query;
    for (uint64_t b = 0; b < n_rows; b += QB) {
        const uint32_t nb = (uint32_t)std::min<uint64_t>(QB, n_rows - b);
        const uint64_t s0 = first_row + b;  // the block's first row, relative to the index's first row
        for (uint32_t q = 0; q < nb; ++q) ids[q] = (uint32_t)(s0 + q);
        RangeShards scan;
        for (NkShard *s : live) {
            const uint64_t lo = ix->first_row(*s);
            if (lo + s->n <= s0 + 1) continue;  // every row at or below s0
            scan.shards.push_back(s);
            scan.from.push_back(lo <= s0 ? (s0 - lo) / SCAN_TILE_ROWS * SCAN_TILE_ROWS : 0);
        }
        StageQueries stage;
        if (!scan.shards.empty() && stage_row_block(ix, live, ids.data(), nb, adm, &stage)) return -1;
        const uint64_t pair_first = ix->row_base + s0;
        RangeBlock block{ix->path, adm.mode, nb, thr.data()};
        block.pair_first = &pair_first;
        if (range_scan(ix, &scan, stage, block, &per_query)) return -1;
        for (uint32_t q = 0; q < nb; ++q) out_offsets[b + q + 1] = out_offsets[b + q] + per_query[q];
        if (out_offsets[b + nb] > keys.size() && range_collect(ix, scan, nb, &keys)) return -1;
    }
    return write_csr(ix, out_offsets[n_rows], capacity, out_idx, out_score, out_total, [&](std::vector<uint64_t> *out) {
        out->swap(keys);
        return 0;
    });
}

// ---- k-NN graph update and remap (DESIGN.md §3.5e) ----------------------------------------------------------------------
// Current row f holds the contents old row src[f] had when the graph was built (kept: src[f] == f; moved: src[f] != f), or
// contents the graph never saw (NK_ROW_NEW: appended or rewritten).  Rows whose list may have changed in more than one place
// are searched again, as nk_search_rows searches them: the new and moved rows, and every kept row whose list holds an old row
// that no longer sits at its id (gone, moved or rewritten: a moved row's key changes with its id).  Every other kept row r
// lists only kept rows, so only the rows C that are new or moved can enter its list (a moved row when its new id wins a tie):
// they are scanned as queries over the index with the row's own threshold (the k-th entry's score, or the floor if the list
// is not full) and the rows searched again masked out, re-scored as r's list scores them (K(r, q), warp_pair_score), and
// merged with the old entries, whose keys are recomputed the same way.  The graph path (16-bit pass or TF32 filter) is
// forced for the whole call: every score it makes is warp_exact_score's, whichever block of queries it is computed in.
constexpr uint32_t GRAPH_PAD = 0xffffffffu;

// Whether each current row (relative id) passes the row mask -> ok[rows()].
static int admissible_rows(NkIndex *ix, std::vector<uint8_t> *ok) {
    ok->assign(ix->rows(), 1);
    if (!ix->mask_on) return 0;
    for (auto &s : ix->shards) {
        if (s.n == 0 || !s.mask_on) continue;
        const uint64_t lo = ix->first_row(s);
        std::vector<uint32_t> w((s.n + 31) / 32);
        NK_CUDA_OK(cudaSetDevice(s.device));
        NK_CUDA_OK(cudaMemcpyAsync(w.data(), s.mask, w.size() * 4, cudaMemcpyDeviceToHost, s.stream));
        NK_CUDA_OK(cudaStreamSynchronize(s.stream));
        for (uint64_t i = 0; i < s.n; ++i) (*ok)[lo + i] = (w[i >> 5] >> (i & 31)) & 1u;
    }
    return 0;
}

// The tag word (values = false) or value key (values = true) of each current row (relative id) -> words[rows()]; 0 where a
// shard has none.
static int host_row_words(NkIndex *ix, bool values, std::vector<uint64_t> *words) {
    words->assign(ix->rows(), 0ull);
    for (auto &s : ix->shards) {
        if (s.n == 0 || !(values ? s.values_on : s.tags_on)) continue;
        NK_CUDA_OK(cudaSetDevice(s.device));
        NK_CUDA_OK(cudaMemcpyAsync(words->data() + ix->first_row(s), values ? s.values : s.tags, s.n * 8, cudaMemcpyDeviceToHost, s.stream));
        NK_CUDA_OK(cudaStreamSynchronize(s.stream));
        ix->stats.bytes_d2h += s.n * 8;
    }
    return 0;
}

// Searches that fell through to the exact stage so far, all shards (cumulative status word FLAG_N_EXACT).
static int exact_stage_runs(NkIndex *ix, uint64_t *out) {
    uint64_t c = 0;
    for (auto &s : ix->shards) {
        if (!s.ws.flags) continue;
        int h = 0;
        NK_CUDA_OK(cudaSetDevice(s.device));
        NK_CUDA_OK(cudaMemcpyAsync(&h, s.ws.flags + nk::FLAG_N_EXACT, 4, cudaMemcpyDeviceToHost, s.stream));
        NK_CUDA_OK(cudaStreamSynchronize(s.stream));
        c += (uint64_t)h;
    }
    *out = c;
    return 0;
}

// The keys K(r, j) of pairs (pr[i], pj[i]) (relative ids) -> keys[i], computed on the shard that holds r: each shard's distinct j
// are gathered in blocks of SEARCH_ROWS_BLOCK (stage_row_block) and every block's pairs are scored in one launch.
static int pair_keys(NkIndex *ix, const std::vector<NkShard *> &live, const std::vector<uint32_t> &pr, const std::vector<uint32_t> &pj,
                     std::vector<uint64_t> *keys) {
    keys->assign(pr.size(), 0ull);
    std::vector<std::vector<uint32_t>> of_shard(ix->shards.size());  // the pairs whose r each shard holds, in order
    for (size_t i = 0; i < pr.size(); ++i) {
        uint64_t local;
        of_shard[find_shard(ix, pr[i], &local) - ix->shards.data()].push_back((uint32_t)i);
    }
    for (size_t si = 0; si < of_shard.size(); ++si) {
        if (of_shard[si].empty()) continue;
        NkShard &s = ix->shards[si];
        std::vector<uint32_t> order(of_shard[si]), js(order.size());  // distinct j, staged in blocks of SEARCH_ROWS_BLOCK
        for (size_t i = 0; i < order.size(); ++i) js[i] = pj[order[i]];
        std::sort(js.begin(), js.end());
        js.erase(std::unique(js.begin(), js.end()), js.end());
        std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return pj[a] < pj[b]; });
        size_t at = 0;
        for (size_t b = 0; b < js.size(); b += SEARCH_ROWS_BLOCK) {
            const uint32_t nb = (uint32_t)std::min<size_t>(SEARCH_ROWS_BLOCK, js.size() - b);
            StageQueries stage;
            if (stage_row_block(ix, live, js.data() + b, nb, RowAdmit{}, &stage)) return -1;
            NK_CUDA_OK(cudaSetDevice(s.device));
            if (nk::ws_reserve((void **)&s.ws.queries, &s.ws.queries_bytes, (size_t)nb * ix->dim * sizeof(float))) return -1;
            if (stage(s)) return -1;
            const uint32_t last = js[b + nb - 1];
            std::vector<uint32_t> arg;  // [r local | slot of j | global j]
            std::vector<uint32_t> idx;
            for (; at < order.size() && pj[order[at]] <= last; ++at) idx.push_back(order[at]);
            const size_t n = idx.size();
            if (n == 0) continue;
            arg.resize(3 * n);
            for (size_t i = 0; i < n; ++i) {
                arg[i] = pr[idx[i]] - (uint32_t)ix->first_row(s);
                arg[n + i] = (uint32_t)(std::lower_bound(js.begin() + b, js.begin() + b + nb, pj[idx[i]]) - (js.begin() + b));
                arg[2 * n + i] = (uint32_t)(ix->row_base + pj[idx[i]]);
            }
            if (nk::ws_reserve(&s.ws.scratch, &s.ws.scratch_bytes, n * 12 + n * 8 + 8)) return -1;
            uint32_t *d_arg = static_cast<uint32_t *>(s.ws.scratch);
            uint64_t *d_out = reinterpret_cast<uint64_t *>(static_cast<char *>(s.ws.scratch) + (n * 12 + 7) / 8 * 8);
            std::vector<uint64_t> out(n);
            NK_CUDA_OK(cudaMemcpyAsync(d_arg, arg.data(), n * 12, cudaMemcpyHostToDevice, s.stream));
            if (nk::graph_pair_keys(s.rows, ix->dtype, ix->dim, ix->metric, s.ws.queries, d_arg, d_arg + n, d_arg + 2 * n, (uint32_t)n, d_out,
                                    s.stream))
                return -1;
            NK_CUDA_OK(cudaMemcpyAsync(out.data(), d_out, n * 8, cudaMemcpyDeviceToHost, s.stream));
            NK_CUDA_OK(cudaStreamSynchronize(s.stream));
            ix->stats.kernel_launches++;
            ix->stats.bytes_h2d += n * 12;
            ix->stats.bytes_d2h += n * 8;
            for (size_t i = 0; i < n; ++i) (*keys)[idx[i]] = out[i];
        }
    }
    return 0;
}

// One nk_knn_graph_remap / nk_knn_graph_update call, the index lock held and the caller's own arguments checked (src is
// non-null if the index has rows).  gi_in / gs_in [n_old x k] is the old graph, gi / gs [N x k] the output; they are one
// array only when every old row that is still named keeps its id (nk_knn_graph_update): each row's old list is read before
// that row is written.  by_id: the lists counted as changed are those of every row f < n_old whose list differs from old row
// f's, else only the kept rows'.  filters [N] (nullptr: none): the graph of nk_search_rows_filtered, each row's list bounded by
// its own filter.  A kept row has the tag and the filter it had when the graph was built (the caller reports any other row as
// new), so the rows searched again are the same; they are searched with their own filters, and the reverse scan also holds
// each pair (r, c) to r's filter admitting c's tag.  windows [N] (nullptr: none): the graph of nk_search_rows_windowed, each
// row's list bounded by its own window as well, in the same way: a kept row has the value key and the window it had, the rows
// searched again are searched with their own windows, and the reverse scan holds each pair (r, c) to r's window admitting c's
// value key.
struct GraphCall {
    const char *what;
    uint32_t k;
    uint64_t n_old;
    const uint32_t *src;
    const NkFilter *filters;
    const NkWindow *windows;
    const uint32_t *gi_in; const float *gs_in;
    uint32_t *gi; float *gs;
    bool by_id;
    uint64_t changed = 0;  // lists written that differ from the old graph's (by_id)
    void write_list(uint64_t r, const uint32_t *li, const float *ls) {
        if (r < n_old && (by_id || src[r] == r) && (memcmp(gi_in + r * k, li, (size_t)k * 4) || memcmp(gs_in + r * k, ls, (size_t)k * 4)))
            ++changed;
        memcpy(gi + r * k, li, (size_t)k * 4);
        memcpy(gs + r * k, ls, (size_t)k * 4);
    }
};

// Is row r's old list that of a NaN row (every score -inf, decoded)?
static bool graph_nan_list(const NkIndex *ix, const uint32_t *li, const float *ls) {
    return li[0] != GRAPH_PAD && ls[0] == (ix->metric == NK_METRIC_EUCLIDEAN ? INFINITY : -INFINITY);
}

// Check src [rows()] (the old row each current row holds, or NK_ROW_NEW) -> now_at [n_old]: the current id of old row o,
// NK_ROW_NEW once it is gone.
static int check_src_of_row(const NkIndex *ix, const char *what, const uint32_t *src, uint64_t n_old, std::vector<uint32_t> *now_at) {
    const uint64_t N = ix->rows();
    now_at->assign(n_old, NK_ROW_NEW);
    for (uint64_t f = 0; f < N; ++f) {
        const uint32_t o = src[f];
        if (o == NK_ROW_NEW) continue;
        if (o >= n_old) {
            nk::set_error("%s: src_of_row[%llu] = %u is not an old row (n_old=%llu)", what, (unsigned long long)f, o, (unsigned long long)n_old);
            return -1;
        }
        if ((*now_at)[o] != NK_ROW_NEW) {
            nk::set_error("%s: old row %u is the source of rows %u and %llu", what, o, (*now_at)[o], (unsigned long long)f);
            return -1;
        }
        (*now_at)[o] = (uint32_t)f;
    }
    return 0;
}

// Check src and the old graph's entries -> now_at [n_old] (check_src_of_row).
static int graph_check(const NkIndex *ix, const GraphCall &g, std::vector<uint32_t> *now_at) {
    if (check_src_of_row(ix, g.what, g.src, g.n_old, now_at)) return -1;
    for (uint64_t i = 0; i < g.n_old * g.k; ++i)
        if (g.gi_in[i] != GRAPH_PAD && (g.gi_in[i] < ix->row_base || g.gi_in[i] - ix->row_base >= g.n_old)) {
            nk::set_error("%s: entry %llu of the graph (row %u) is not an old row", g.what, (unsigned long long)i, g.gi_in[i]);
            return -1;
        }
    return 0;
}

// The graph path (the k-NN graph calls and the incident pairs of the self-join): the forced one, or under AUTO the 16-bit pass
// where every live shard has a 16-bit image, else the TF32 filter; -1 if a live shard cannot serve it for a block of
// SEARCH_ROWS_BLOCK queries asking k each (range: range queries) (the error names the path and the shape).
static int graph_path(const NkIndex *ix, const std::vector<NkShard *> &live, uint32_t k, bool range) {
    int path = ix->path;
    if (path == NK_PATH_AUTO) {
        path = NK_PATH_TENSOR_SHADOW;
        for (NkShard *s : live)
            if (!s->img.current(s->n)) path = NK_PATH_TENSOR_FILTER;
    }
    for (NkShard *s : live) {
        nk::ScanArgs a = shard_scan_args(ix, *s, nullptr, SEARCH_ROWS_BLOCK, k, s->stream);
        if (plan_path(ix, *s, path, range, &a) < 0) return -1;
    }
    return path;
}

// The rows to search again, R: in_r [N] comes in with the new and moved rows set and leaves with every row of R set.
static int graph_rows_searched_again(NkIndex *ix, const GraphCall &g, const std::vector<uint32_t> &now_at, std::vector<uint8_t> *in_r) {
    const uint64_t N = ix->rows();
    const uint32_t k = g.k;
    // nk_search_rows treats a row specially while no more than k rows are admissible (its list drops one of them when the row
    // itself is not admissible): then every row is searched again.  Gone rows have no mask bit any more, so whether that held
    // when the graph was built is bounded: then every old list was short, and no more than k of the old rows still present
    // are admissible.  With no row gone this is exactly "no more than k old rows are admissible".
    // Filters leave this rule as it is: the scan still asks for k' = min(k + 1, rows passing the mask), so with more than k
    // such rows the last slot a row drops is the (k+1)-th of its filtered order, and a list shorter than k holds every other
    // row its filter and the floor admit — its threshold is the floor, as for an unfiltered short list.  A list that is
    // full implies more than k rows passing the mask, filtered or not.
    bool all = ix->returnable_rows() <= k;
    if (!all) {
        bool full = false;
        for (uint64_t o = 0; o < g.n_old && !full; ++o) full = g.gi_in[o * k + k - 1] != GRAPH_PAD;
        if (!full) {
            std::vector<uint8_t> ok;
            if (admissible_rows(ix, &ok)) return -1;
            uint64_t still = 0;
            for (uint64_t f = 0; f < N; ++f) still += g.src[f] != NK_ROW_NEW && ok[f];
            all = still <= k;
        }
    }
    for (uint64_t r = 0; r < N; ++r) {
        if ((*in_r)[r]) continue;  // r is kept from here on: r < n_old
        // A NaN row's list (every score -inf, decoded) comes from the exact stage its search block falls through to: its keys
        // are that stage's, not warp_exact_score's, so such a row is searched again rather than merged.
        if (all || graph_nan_list(ix, g.gi_in + r * k, g.gs_in + r * k)) { (*in_r)[r] = 1; continue; }
        for (uint32_t j = 0; j < k; ++j) {
            const uint32_t e = g.gi_in[r * k + j];
            if (e != GRAPH_PAD && now_at[e - ix->row_base] != e - ix->row_base) { (*in_r)[r] = 1; break; }
        }
    }
    return 0;
}

// Before the reverse scan in mode m: every live shard gets its per-row thresholds and, behind them, the mask of the rows outside
// R (s.ws.row_thr), under a row-filter mode each row's own filter for the row side of the scan (s.ws.row_filter: put_filters,
// {0,0,0} for a windowed graph without filters), and under REVERSE_RWINDOW each row's own window (s.ws.row_window).
static int graph_upload_row_thresholds(NkIndex *ix, const GraphCall &g, nk::ScanMode m, const std::vector<NkShard *> &live,
                                       const std::vector<uint8_t> &in_r) {
    const uint32_t k = g.k;
    for (NkShard *s : live) {
        const uint64_t lo = ix->first_row(*s), words = (s->n + 31) / 32;
        std::vector<float> thr(s->n + words);
        uint32_t *keep = reinterpret_cast<uint32_t *>(thr.data() + s->n);
        for (uint64_t w = 0; w < words; ++w) keep[w] = 0u;
        for (uint64_t l = 0; l < s->n; ++l) {
            const uint64_t r = lo + l;
            thr[l] = INFINITY;
            if (in_r[r]) continue;
            keep[l >> 5] |= 1u << (l & 31);
            thr[l] = g.gi_in[r * k + k - 1] != GRAPH_PAD ? range_key_threshold(ix, g.gs_in[r * k + k - 1]) : ix->key_floor();
        }
        NK_CUDA_OK(cudaSetDevice(s->device));
        if (nk::ws_reserve((void **)&s->ws.row_thr, &s->ws.row_thr_bytes, thr.size() * 4)) return -1;
        NK_CUDA_OK(cudaMemcpyAsync(s->ws.row_thr, thr.data(), thr.size() * 4, cudaMemcpyHostToDevice, s->stream));
        if (nk::mode_row_filter(m) &&
            put_filters(ix, &s->ws.row_filter, &s->ws.row_filter_bytes, g.filters ? g.filters + lo : nullptr, s->n, s->stream))
            return -1;
        if (nk::mode_row_window(m)) {
            if (nk::ws_reserve((void **)&s->ws.row_window, &s->ws.row_window_bytes, s->n * sizeof(NkWindow))) return -1;
            NK_CUDA_OK(cudaMemcpyAsync(s->ws.row_window, g.windows + lo, s->n * sizeof(NkWindow), cudaMemcpyHostToDevice, s->stream));
            ix->stats.bytes_h2d += s->n * sizeof(NkWindow);
        }
        NK_CUDA_OK(cudaStreamSynchronize(s->stream));  // thr is pageable and goes out of scope
        ix->stats.bytes_h2d += thr.size() * 4;
    }
    return 0;
}

// The reverse scan for the kept rows outside R: the new and moved rows C, in blocks, are range queries over every live shard
// with each row's own threshold -> *entrants, sorted: (kept row r, key of the new or moved row in r's list).
using GraphEntrants = std::vector<std::pair<uint32_t, uint64_t>>;
static int graph_reverse_scan(NkIndex *ix, const GraphCall &g, const std::vector<NkShard *> &live, int path, const std::vector<uint8_t> &in_r,
                              const std::vector<uint32_t> &C, GraphEntrants *entrants) {
    // a windowed graph's scan holds each pair to the row's window and its filter (those of a graph without filters admit every
    // tag), a filtered graph's to the row's filter; every mode but REVERSE applies per-query filters (masked-out queries get
    // the filter that admits no row, stage_row_block)
    const RowAdmit all_rows{g.windows ? nk::ScanMode::REVERSE_RWINDOW
                            : g.filters ? nk::ScanMode::REVERSE_RFILT
                            : ix->mask_on ? nk::ScanMode::REVERSE_TAGS
                                          : nk::ScanMode::REVERSE};
    if (graph_upload_row_thresholds(ix, g, all_rows.mode, live, in_r)) return -1;
    // a filtered graph's queries also carry their tags, a windowed graph's their value keys (and tag 0 without filters)
    std::vector<uint64_t> tags, values, qtags, qvalues;
    if (g.filters && host_row_words(ix, false, &tags)) return -1;
    if (g.windows && host_row_words(ix, true, &values)) return -1;
    const uint32_t QB = (uint32_t)std::min<size_t>(C.size(), SEARCH_ROWS_BLOCK);
    const std::vector<uint32_t> floor_thr(QB, nk::ord_bits(ix->key_floor()));
    RangeBlock block{path, all_rows.mode, 0, floor_thr.data()};
    RangeShards on{live};
    std::vector<uint64_t> keys, per_query;
    for (size_t b = 0; b < C.size(); b += QB) {
        const uint32_t nb = block.Q = (uint32_t)std::min<size_t>(QB, C.size() - b);
        StageQueries stage_rows;
        if (stage_row_block(ix, live, C.data() + b, nb, all_rows, &stage_rows)) return -1;
        if (nk::mode_row_filter(block.mode)) {
            qtags.assign(nb, 0ull);
            if (g.filters)
                for (uint32_t q = 0; q < nb; ++q) qtags[q] = tags[C[b + q]];
        }
        if (g.windows) {
            qvalues.resize(nb);
            for (uint32_t q = 0; q < nb; ++q) qvalues[q] = values[C[b + q]];
        }
        const StageQueries stage = [&](NkShard &s) {
            if (stage_rows(s)) return -1;
            if (!nk::mode_row_filter(block.mode)) return 0;
            // the queries' tags and value keys: read by the scan before range_shard's first synchronisation
            if (nk::ws_reserve((void **)&s.ws.qtags, &s.ws.qtags_bytes, (size_t)nb * 8)) return -1;
            NK_CUDA_OK(cudaMemcpyAsync(s.ws.qtags, qtags.data(), (size_t)nb * 8, cudaMemcpyHostToDevice, s.stream));
            ix->stats.bytes_h2d += (uint64_t)nb * 8;
            if (!nk::mode_row_window(block.mode)) return 0;
            if (nk::ws_reserve((void **)&s.ws.qvalues, &s.ws.qvalues_bytes, (size_t)nb * 8)) return -1;
            NK_CUDA_OK(cudaMemcpyAsync(s.ws.qvalues, qvalues.data(), (size_t)nb * 8, cudaMemcpyHostToDevice, s.stream));
            ix->stats.bytes_h2d += (uint64_t)nb * 8;
            return 0;
        };
        if (range_scan(ix, &on, stage, block, &per_query)) return -1;
        keys.clear();
        if (range_collect(ix, on, nb, &keys)) return -1;
        size_t at = 0;
        for (uint32_t q = 0; q < nb; ++q) {
            const uint64_t qrow = 0xffffffffull - (ix->row_base + C[b + q]);
            for (uint64_t j = 0; j < per_query[q]; ++j, ++at)
                entrants->emplace_back((uint32_t)(nk::key_row(keys[at]) - ix->row_base), (keys[at] & 0xffffffff00000000ull) | qrow);
        }
    }
    std::sort(entrants->begin(), entrants->end());
    return 0;
}

// Merge the entrants into the lists of the rows they touch: each touched row's old entries, their keys recomputed as the
// row's list scores them (pair_keys), and its entrants in key space, the best k kept.
static int graph_merge_entrants(NkIndex *ix, GraphCall &g, const std::vector<NkShard *> &live, const GraphEntrants &entrants) {
    const uint32_t k = g.k;
    std::vector<uint32_t> touched, opr, opj;
    for (size_t i = 0; i < entrants.size(); ++i)
        if (i == 0 || entrants[i].first != entrants[i - 1].first) touched.push_back(entrants[i].first);
    for (const uint32_t r : touched)
        for (uint32_t j = 0; j < k; ++j) {
            const uint32_t e = g.gi_in[(uint64_t)r * k + j];
            if (e == GRAPH_PAD) break;
            opr.push_back(r);
            opj.push_back((uint32_t)(e - ix->row_base));
        }
    std::vector<uint64_t> okeys;
    if (pair_keys(ix, live, opr, opj, &okeys)) return -1;
    std::vector<uint64_t> cand;
    std::vector<uint32_t> li(k);
    std::vector<float> ls(k);
    size_t o0 = 0, e0 = 0;
    for (const uint32_t r : touched) {
        cand.clear();
        for (; o0 < opr.size() && opr[o0] == r; ++o0) cand.push_back(okeys[o0]);
        for (; e0 < entrants.size() && entrants[e0].first == r; ++e0) cand.push_back(entrants[e0].second);
        const size_t take = std::min<size_t>(k, cand.size());
        std::partial_sort(cand.begin(), cand.begin() + take, cand.end(), std::greater<uint64_t>());
        for (uint32_t j = 0; j < k; ++j) {
            if (j < take) decode_key(ix->metric, cand[j], &li[j], &ls[j]);
            else { li[j] = GRAPH_PAD; ls[j] = 0.0f; }
        }
        g.write_list(r, li.data(), ls.data());
    }
    return 0;
}

// The rows of R, searched again.  A block with a NaN row among its queries overflows the filter and falls through to the
// exact stage, whose arithmetic differs: such a block is searched once more without its NaN rows (lists of -inf scores,
// the same on every path), so the other rows get the lists a rebuild gives them in blocks without a NaN query.
static int graph_search_again(NkIndex *ix, GraphCall &g, const std::vector<NkShard *> &live, int path, const std::vector<uint8_t> &in_r) {
    const uint32_t k = g.k;
    std::vector<uint32_t> rows;
    for (uint64_t r = 0; r < in_r.size(); ++r)
        if (in_r[r]) rows.push_back((uint32_t)r);
    std::vector<uint32_t> ri((size_t)std::min<size_t>(rows.size(), SEARCH_ROWS_BLOCK) * k), sub;
    std::vector<float> rs(ri.size());
    std::vector<NkFilter> rf;  // filters: the block's rows' own
    std::vector<NkWindow> rw;  // windows: the block's rows' own
    auto search = [&](const uint32_t *ids, uint32_t nb) {
        SearchOpts opts{path};
        if (g.filters) {
            rf.resize(nb);
            for (uint32_t q = 0; q < nb; ++q) rf[q] = g.filters[ids[q]];
            opts.filters_host = rf.data();
        }
        if (g.windows) {
            rw.resize(nb);
            for (uint32_t q = 0; q < nb; ++q) rw[q] = g.windows[ids[q]];
            opts.windows_host = rw.data();
        }
        return search_rows_locked(ix, live, ids, opts, nb, k, ri.data(), rs.data());
    };
    for (size_t b = 0; b < rows.size(); b += SEARCH_ROWS_BLOCK) {
        uint32_t nb = (uint32_t)std::min<size_t>(SEARCH_ROWS_BLOCK, rows.size() - b);
        std::fill(ri.begin(), ri.end(), GRAPH_PAD);
        std::fill(rs.begin(), rs.end(), 0.0f);
        uint64_t exact0 = 0, exact1 = 0;
        if (exact_stage_runs(ix, &exact0) || search(rows.data() + b, nb) < 0 || exact_stage_runs(ix, &exact1)) return -1;
        sub.clear();
        for (uint32_t q = 0; q < nb; ++q) {
            const uint32_t *li = ri.data() + (size_t)q * k;
            const float *ls = rs.data() + (size_t)q * k;
            if (exact1 == exact0 || graph_nan_list(ix, li, ls)) g.write_list(rows[b + q], li, ls);
            else sub.push_back(rows[b + q]);
        }
        if (sub.empty()) continue;
        nb = (uint32_t)sub.size();
        if (search(sub.data(), nb) < 0) return -1;
        for (uint32_t q = 0; q < nb; ++q) g.write_list(sub[q], ri.data() + (size_t)q * k, rs.data() + (size_t)q * k);
    }
    return 0;
}

// The body of nk_knn_graph_remap and nk_knn_graph_update.  Returns ke, or -1 with nothing written; *n_lists_changed (nullable):
// g.changed.
static int knn_graph_remap_locked(NkIndex *ix, GraphCall g, uint64_t *n_lists_changed) {
    if (g.k == 0 || g.k > NK_GRAPH_MAX_K) { nk::set_error("%s: k=%u outside [1, %u]", g.what, g.k, NK_GRAPH_MAX_K); return -1; }
    if (ix->path == NK_PATH_SIMT || ix->path == NK_PATH_TENSOR) {
        nk::set_error("%s: the graph is kept on the filter paths (AUTO, TENSOR_FILTER or TENSOR_SHADOW), not path %d", g.what, ix->path);
        return -1;
    }
    const uint64_t N = ix->rows();
    std::vector<uint32_t> now_at;
    if (graph_check(ix, g, &now_at)) return -1;
    const std::vector<NkShard *> live = live_shards(ix);
    const int path = graph_path(ix, live, g.k + 1, false);
    if (path < 0) return -1;
    if (n_lists_changed) *n_lists_changed = 0;
    ix->stats.searches++;
    ScopedRange range(g.what);
    ShardOrder order(ix);
    if (order.failed()) return -1;
    if (g.gi != g.gi_in)  // kept rows start from their old lists
        for (uint64_t f = 0; f < N; ++f)
            if (g.src[f] == f) {
                memcpy(g.gi + f * g.k, g.gi_in + f * g.k, (size_t)g.k * 4);
                memcpy(g.gs + f * g.k, g.gs_in + f * g.k, (size_t)g.k * 4);
            }

    // the rows to search again (R) and the queries of the reverse scan (C: new and moved rows)
    std::vector<uint8_t> in_r(N, 0);
    std::vector<uint32_t> C;
    for (uint64_t f = 0; f < N; ++f)
        if (g.src[f] != f) { in_r[f] = 1; C.push_back((uint32_t)f); }
    const int ke = (int)std::min<uint64_t>(g.k, ix->returnable_rows());
    if (C.empty() && N == g.n_old) return ke;  // every row kept at its id
    if (graph_rows_searched_again(ix, g, now_at, &in_r)) return -1;

    // reverse scan + merge for the kept rows outside R
    bool reverse = false;
    for (uint64_t r = 0; r < N && !reverse; ++r) reverse = !in_r[r];
    if (reverse) {
        GraphEntrants entrants;
        if (graph_reverse_scan(ix, g, live, path, in_r, C, &entrants)) return -1;
        if (graph_merge_entrants(ix, g, live, entrants)) return -1;
    }
    if (graph_search_again(ix, g, live, path, in_r)) return -1;
    if (n_lists_changed) *n_lists_changed = g.changed;
    return ke;
}

// The arguments of nk_knn_graph_remap[_filtered] checked, then the call itself.
static int knn_graph_remap_host(NkIndex *ix, const GraphCall &g, uint64_t *n_lists_changed) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    if (!g.gi || !g.gs || (g.n_old && (!g.gi_in || !g.gs_in))) { nk::set_error("null argument"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    const uint64_t N = ix->rows();
    if (N && !g.src) { nk::set_error("null argument"); return -1; }
    // the output is written while the input is still read: overlapping arrays are refused
    auto overlap = [](const void *a, size_t na, const void *b, size_t nb) {
        const uintptr_t pa = (uintptr_t)a, pb = (uintptr_t)b;
        return na && nb && pa < pb + nb && pb < pa + na;
    };
    const size_t in_bytes = (size_t)(g.n_old * g.k) * 4, out_bytes = (size_t)(N * g.k) * 4;
    for (const void *in : {(const void *)g.gi_in, (const void *)g.gs_in})
        for (const void *out : {(const void *)g.gi, (const void *)g.gs})
            if (overlap(in, in_bytes, out, out_bytes)) {
                nk::set_error("%s: the output arrays overlap the input graph", g.what);
                return -1;
            }
    return knn_graph_remap_locked(ix, g, n_lists_changed);
}

int nk_knn_graph_remap(NkIndex *ix, uint32_t k, uint64_t n_old, const uint32_t *src_of_row, const uint32_t *graph_idx_in,
                       const float *graph_score_in, uint32_t *graph_idx_out, float *graph_score_out, uint64_t *n_lists_changed) {
    return knn_graph_remap_host(ix, GraphCall{"nk_knn_graph_remap", k, n_old, src_of_row, nullptr, nullptr, graph_idx_in, graph_score_in,
                                              graph_idx_out, graph_score_out, false}, n_lists_changed);
}

int nk_knn_graph_remap_filtered(NkIndex *ix, uint32_t k, uint64_t n_old, const uint32_t *src_of_row, const NkFilter *filters_host,
                                const uint32_t *graph_idx_in, const float *graph_score_in, uint32_t *graph_idx_out,
                                float *graph_score_out, uint64_t *n_lists_changed) {
    return knn_graph_remap_host(ix, GraphCall{"nk_knn_graph_remap_filtered", k, n_old, src_of_row, filters_host, nullptr, graph_idx_in,
                                              graph_score_in, graph_idx_out, graph_score_out, false}, n_lists_changed);
}

int nk_knn_graph_remap_windowed(NkIndex *ix, uint32_t k, uint64_t n_old, const uint32_t *src_of_row, const NkFilter *filters_host,
                                const NkWindow *windows_host, const uint32_t *graph_idx_in, const float *graph_score_in,
                                uint32_t *graph_idx_out, float *graph_score_out, uint64_t *n_lists_changed) {
    return knn_graph_remap_host(ix, GraphCall{"nk_knn_graph_remap_windowed", k, n_old, src_of_row, filters_host, windows_host, graph_idx_in,
                                              graph_score_in, graph_idx_out, graph_score_out, false}, n_lists_changed);
}

// An old row keeps its id; a rewritten row and every row from n_old on hold contents the graph never saw.  In place: g.src
// and the input graph are filled in here.
static int knn_graph_update_host(NkIndex *ix, GraphCall g, const uint32_t *changed_rows, uint32_t n_changed, uint64_t *n_lists_changed) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    if (!g.gi || !g.gs || (n_changed && !changed_rows)) { nk::set_error("null argument"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    const uint64_t N = ix->rows();
    if (g.n_old > N) { nk::set_error("%s: n_old=%llu exceeds the index's %llu rows", g.what, (unsigned long long)g.n_old, (unsigned long long)N); return -1; }
    std::vector<uint32_t> src(N, NK_ROW_NEW);
    for (uint64_t f = 0; f < g.n_old; ++f) src[f] = (uint32_t)f;
    for (uint32_t i = 0; i < n_changed; ++i) {
        if (changed_rows[i] >= g.n_old) { nk::set_error("%s: changed row %u is not an old row (n_old=%llu)", g.what, changed_rows[i], (unsigned long long)g.n_old); return -1; }
        src[changed_rows[i]] = NK_ROW_NEW;
    }
    g.src = src.data();
    g.gi_in = g.gi;
    g.gs_in = g.gs;
    return knn_graph_remap_locked(ix, g, n_lists_changed);
}

int nk_knn_graph_update(NkIndex *ix, uint32_t k, uint64_t n_old, const uint32_t *changed_rows, uint32_t n_changed,
                        uint32_t *graph_idx, float *graph_score, uint64_t *n_lists_changed) {
    return knn_graph_update_host(ix, GraphCall{"nk_knn_graph_update", k, n_old, nullptr, nullptr, nullptr, nullptr, nullptr, graph_idx, graph_score,
                                               true},
                                 changed_rows, n_changed, n_lists_changed);
}

int nk_knn_graph_update_filtered(NkIndex *ix, uint32_t k, uint64_t n_old, const uint32_t *changed_rows, uint32_t n_changed,
                                 const NkFilter *filters_host, uint32_t *graph_idx, float *graph_score, uint64_t *n_lists_changed) {
    return knn_graph_update_host(ix, GraphCall{"nk_knn_graph_update_filtered", k, n_old, nullptr, filters_host, nullptr, nullptr, nullptr,
                                               graph_idx, graph_score, true}, changed_rows, n_changed, n_lists_changed);
}

int nk_knn_graph_update_windowed(NkIndex *ix, uint32_t k, uint64_t n_old, const uint32_t *changed_rows, uint32_t n_changed,
                                 const NkFilter *filters_host, const NkWindow *windows_host, uint32_t *graph_idx, float *graph_score,
                                 uint64_t *n_lists_changed) {
    return knn_graph_update_host(ix, GraphCall{"nk_knn_graph_update_windowed", k, n_old, nullptr, filters_host, windows_host, nullptr, nullptr,
                                               graph_idx, graph_score, true}, changed_rows, n_changed, n_lists_changed);
}

// ---- the self-join kept current (DESIGN.md §3.5d, "Pairs incident to rows") ---------------------------------------------
// The listed rows are range queries over every shard whole (no triangle), in blocks of SEARCH_ROWS_BLOCK gathered by
// stage_row_block with the join's admission (a listed row the join would refuse gets the filter, or the window, that admits no
// row), on the graph path.  range_rescore_incident_kernel drops each query's own row and the listed rows below it, and scores
// every other pair with its lower row as the query: each key is the one the whole-index join gives the pair.
struct PairsCall {
    const char *what;
    float threshold;
    const NkFilter *filter;
    const NkWindow *window;
    uint64_t max_gap;
};

// The pairs of the whole-index join incident to rows[n] (relative ids, distinct, checked), the index lock held: row i's are
// keys[off[i], off[i + 1]), in nk_search's order.
static int pairs_rows_locked(NkIndex *ix, const PairsCall &c, int path, const std::vector<NkShard *> &live, const uint32_t *rows,
                             uint32_t n, std::vector<uint64_t> *off, std::vector<uint64_t> *keys) {
    off->assign((size_t)n + 1, 0);
    keys->clear();
    if (n == 0) return 0;
    const RowAdmit adm = join_admit(ix, c.filter, c.window, c.max_gap);
    const uint32_t QB = std::min(n, SEARCH_ROWS_BLOCK);
    // every live shard: the bits of the listed rows it holds, room for a block's query rows behind them
    for (NkShard *s : live) {
        const uint64_t lo = ix->first_row(*s), words = (s->n + 31) / 32;
        std::vector<uint32_t> bits(words, 0u);
        for (uint32_t i = 0; i < n; ++i)
            if (rows[i] >= lo && rows[i] - lo < s->n) bits[(rows[i] - lo) >> 5] |= 1u << ((rows[i] - lo) & 31);
        NK_CUDA_OK(cudaSetDevice(s->device));
        if (nk::ws_reserve((void **)&s->ws.pair_rows, &s->ws.pair_rows_bytes, (size_t)(words + QB) * 4)) return -1;
        NK_CUDA_OK(cudaMemcpyAsync(s->ws.pair_rows, bits.data(), words * 4, cudaMemcpyHostToDevice, s->stream));
        NK_CUDA_OK(cudaStreamSynchronize(s->stream));  // bits is pageable and goes out of scope
        ix->stats.bytes_h2d += words * 4;
    }
    const std::vector<uint32_t> thr(QB, nk::ord_bits(range_key_threshold(ix, c.threshold)));
    std::vector<uint32_t> qrow(QB);
    std::vector<uint64_t> per_query;
    RangeShards on{live};
    for (uint32_t b = 0; b < n; b += QB) {
        const uint32_t nb = std::min(QB, n - b);
        for (uint32_t q = 0; q < nb; ++q) qrow[q] = (uint32_t)(ix->row_base + rows[b + q]);
        StageQueries stage_rows;
        if (stage_row_block(ix, live, rows + b, nb, adm, &stage_rows)) return -1;
        const StageQueries stage = [&](NkShard &s) {
            if (stage_rows(s)) return -1;
            // the block's query rows behind the listed-row bits (range_shard's IncidentRows), read before its first synchronisation
            NK_CUDA_OK(cudaMemcpyAsync(s.ws.pair_rows + (s.n + 31) / 32, qrow.data(), (size_t)nb * 4, cudaMemcpyHostToDevice, s.stream));
            ix->stats.bytes_h2d += (uint64_t)nb * 4;
            return 0;
        };
        RangeBlock block{path, adm.mode, nb, thr.data()};
        block.incident = true;
        if (range_scan(ix, &on, stage, block, &per_query)) return -1;
        for (uint32_t q = 0; q < nb; ++q) (*off)[b + q + 1] = (*off)[b + q] + per_query[q];
        if ((*off)[b + nb] > keys->size() && range_collect(ix, on, nb, keys)) return -1;
    }
    return 0;
}

// The checks every call of this section makes before any work, the index lock held.
static int pairs_check(const NkIndex *ix, const PairsCall &c) {
    if (c.threshold != c.threshold) { nk::set_error("%s: threshold is NaN", c.what); return -1; }
    if (ix->path == NK_PATH_SIMT || ix->path == NK_PATH_TENSOR) {
        nk::set_error("%s: the incident pairs are scanned on the filter paths (AUTO, TENSOR_FILTER or TENSOR_SHADOW), not path %d",
                      c.what, ix->path);
        return -1;
    }
    return 0;
}

static int pairs_rows_host(NkIndex *ix, const PairsCall &c, const uint32_t *rows_host, uint32_t n, uint64_t capacity,
                           uint64_t *out_offsets, uint32_t *out_idx, float *out_score, uint64_t *out_total) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    if (n && (!rows_host || !out_offsets || !out_total)) { nk::set_error("null argument"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    if (pairs_check(ix, c)) return -1;
    const uint64_t total_rows = ix->rows();
    std::vector<uint8_t> seen(n ? total_rows : 0, 0);
    for (uint32_t i = 0; i < n; ++i) {
        if (rows_host[i] >= total_rows) {
            nk::set_error("%s: row %u (entry %u) out of range, index has %llu rows", c.what, rows_host[i], i, (unsigned long long)total_rows);
            return -1;
        }
        if (seen[rows_host[i]]++) { nk::set_error("%s: row %u is listed twice", c.what, rows_host[i]); return -1; }
    }
    if (out_offsets) out_offsets[0] = 0;
    if (out_total) *out_total = 0;
    if (n == 0) return 0;
    const std::vector<NkShard *> live = live_shards(ix);
    const int path = graph_path(ix, live, 1, true);
    if (path < 0) return -1;
    ix->stats.searches++;
    ix->stats.queries += n;
    ScopedRange range(c.what);
    ShardOrder order(ix);
    if (order.failed()) return -1;
    std::vector<uint64_t> off, keys;
    if (pairs_rows_locked(ix, c, path, live, rows_host, n, &off, &keys)) return -1;
    memcpy(out_offsets, off.data(), ((size_t)n + 1) * 8);
    return write_csr(ix, off[n], capacity, out_idx, out_score, out_total, [&](std::vector<uint64_t> *out) {
        out->swap(keys);
        return 0;
    });
}

int nk_search_pairs_rows(NkIndex *ix, const uint32_t *rows_host, uint32_t n, float threshold, const NkFilter *filter, uint64_t capacity,
                         uint64_t *out_offsets, uint32_t *out_idx, float *out_score, uint64_t *out_total) {
    return pairs_rows_host(ix, PairsCall{"nk_search_pairs_rows", threshold, filter, nullptr, NK_NO_GAP}, rows_host, n, capacity, out_offsets,
                           out_idx, out_score, out_total);
}

int nk_search_pairs_rows_windowed(NkIndex *ix, const uint32_t *rows_host, uint32_t n, float threshold, const NkFilter *filter,
                                  const NkWindow *window, uint64_t max_gap, uint64_t capacity, uint64_t *out_offsets, uint32_t *out_idx,
                                  float *out_score, uint64_t *out_total) {
    return pairs_rows_host(ix, PairsCall{"nk_search_pairs_rows_windowed", threshold, filter, window, max_gap}, rows_host, n, capacity,
                           out_offsets, out_idx, out_score, out_total);
}

// The remap: old pairs whose two ends are kept at their id are carried (their ids, orientation and keys cannot have changed),
// every other old pair is dropped, and the pairs incident to the new and moved rows C are found by pairs_rows_locked.  Each
// found pair goes to its lower end's list and is merged there with the carried entries in key space.  Carried keys come back
// from the old scores (cosine / dot: the score is the key's); under euclidean two squared distances one ulp apart decode to one
// distance, so the carried keys of a list that takes in found pairs are computed again on the device (pair_keys).
int nk_pairs_remap(NkIndex *ix, float threshold, const NkFilter *filter, const NkWindow *window, uint64_t max_gap, uint64_t n_old,
                   const uint32_t *src_of_row, const uint64_t *old_offsets, const uint32_t *old_idx, const float *old_score,
                   uint64_t capacity, uint64_t *out_offsets, uint32_t *out_idx, float *out_score, uint64_t *out_total,
                   uint64_t *n_dropped, uint64_t *n_found) {
    const PairsCall c{"nk_pairs_remap", threshold, filter, window, max_gap};
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    if (!old_offsets || !out_offsets || !out_total) { nk::set_error("null argument"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    if (pairs_check(ix, c)) return -1;
    const uint64_t N = ix->rows();
    if (N && !src_of_row) { nk::set_error("null argument"); return -1; }
    if (n_old > 0xffffffffull) { nk::set_error("%s: n_old=%llu is past the 32-bit row ids", c.what, (unsigned long long)n_old); return -1; }
    if (old_offsets[0] != 0) { nk::set_error("%s: old_offsets[0] = %llu, not 0", c.what, (unsigned long long)old_offsets[0]); return -1; }
    for (uint64_t o = 0; o < n_old; ++o)
        if (old_offsets[o + 1] < old_offsets[o]) { nk::set_error("%s: old_offsets decrease at row %llu", c.what, (unsigned long long)o); return -1; }
    const uint64_t n_old_pairs = old_offsets[n_old];
    if (n_old_pairs && (!old_idx || !old_score)) { nk::set_error("null argument"); return -1; }
    std::vector<uint32_t> now_at;
    if (check_src_of_row(ix, c.what, src_of_row, n_old, &now_at)) return -1;
    for (uint64_t o = 0; o < n_old; ++o)
        for (uint64_t e = old_offsets[o]; e < old_offsets[o + 1]; ++e) {
            const uint64_t j = (uint64_t)old_idx[e] - ix->row_base;
            if (old_idx[e] < ix->row_base || j >= n_old || j <= o) {
                nk::set_error("%s: entry %llu of old row %llu (row %u) is not an old row above it", c.what, (unsigned long long)e,
                              (unsigned long long)o, old_idx[e]);
                return -1;
            }
        }
    out_offsets[0] = 0;
    *out_total = 0;
    if (n_dropped) *n_dropped = 0;
    if (n_found) *n_found = 0;
    auto kept = [&](uint64_t o) { return o < N && now_at[o] == o; };  // an old row still at its id
    std::vector<uint32_t> C;  // new and moved rows
    for (uint64_t f = 0; f < N; ++f)
        if (src_of_row[f] != f) C.push_back((uint32_t)f);
    const std::vector<NkShard *> live = live_shards(ix);
    const int path = C.empty() ? 0 : graph_path(ix, live, 1, true);
    if (path < 0) return -1;
    ix->stats.searches++;
    ix->stats.queries += C.size();
    ScopedRange range(c.what);
    ShardOrder order(ix);
    if (order.failed()) return -1;
    std::vector<uint64_t> coff, ckeys;
    if (pairs_rows_locked(ix, c, path, live, C.data(), (uint32_t)C.size(), &coff, &ckeys)) return -1;
    // the found pairs under their lower end: (owner, key), owners ascending, each owner's keys descending
    std::vector<std::pair<uint32_t, uint64_t>> found;
    found.reserve(ckeys.size());
    for (size_t i = 0; i < C.size(); ++i)
        for (uint64_t e = coff[i]; e < coff[i + 1]; ++e) {
            const uint32_t j = (uint32_t)(nk::key_row(ckeys[e]) - ix->row_base);
            if (j > C[i]) found.emplace_back(C[i], ckeys[e]);
            else found.emplace_back(j, (ckeys[e] & 0xffffffff00000000ull) | (0xffffffffull - (ix->row_base + C[i])));
        }
    std::sort(found.begin(), found.end(), [](const std::pair<uint32_t, uint64_t> &a, const std::pair<uint32_t, uint64_t> &b) {
        return a.first != b.first ? a.first < b.first : a.second > b.second;
    });
    // carried entries of every current row -> offsets; the keys of those that meet found pairs
    std::vector<uint8_t> touched(N, 0);
    for (const auto &p : found) touched[p.first] = 1;
    uint64_t carried = 0;
    std::vector<uint64_t> cnt(N, 0);
    for (uint64_t r = 0; r < N && r < n_old; ++r) {
        if (!kept(r)) continue;
        for (uint64_t e = old_offsets[r]; e < old_offsets[r + 1]; ++e) cnt[r] += kept(old_idx[e] - ix->row_base);
        carried += cnt[r];
    }
    for (const auto &p : found) ++cnt[p.first];
    for (uint64_t r = 0; r < N; ++r) out_offsets[r + 1] = out_offsets[r] + cnt[r];
    *out_total = out_offsets[N];
    if (n_dropped) *n_dropped = n_old_pairs - carried;
    if (n_found) *n_found = found.size();
    if (*out_total > capacity || *out_total == 0) return 0;
    if (!out_idx || !out_score) { nk::set_error("null argument"); return -1; }
    std::vector<uint64_t> okey(ix->metric == NK_METRIC_EUCLIDEAN ? n_old_pairs : 0, 0ull);
    if (!okey.empty()) {
        std::vector<uint32_t> pr, pj;
        std::vector<uint64_t> at, keys;
        for (uint64_t r = 0; r < N && r < n_old; ++r) {
            if (!touched[r] || !kept(r)) continue;
            for (uint64_t e = old_offsets[r]; e < old_offsets[r + 1]; ++e)
                if (kept(old_idx[e] - ix->row_base)) {
                    pr.push_back((uint32_t)r);
                    pj.push_back((uint32_t)(old_idx[e] - ix->row_base));
                    at.push_back(e);
                }
        }
        if (pair_keys(ix, live, pr, pj, &keys)) return -1;
        for (size_t t = 0; t < at.size(); ++t) okey[at[t]] = keys[t];
    }
    std::vector<uint64_t> mine, merged;
    size_t f0 = 0;
    for (uint64_t r = 0; r < N; ++r) {
        uint64_t w = out_offsets[r];
        const bool old_list = r < n_old && kept(r);
        if (!touched[r]) {  // the carried entries as they were
            if (old_list)
                for (uint64_t e = old_offsets[r]; e < old_offsets[r + 1]; ++e)
                    if (kept(old_idx[e] - ix->row_base)) { out_idx[w] = old_idx[e]; out_score[w] = old_score[e]; ++w; }
            continue;
        }
        mine.clear();
        if (old_list)
            for (uint64_t e = old_offsets[r]; e < old_offsets[r + 1]; ++e)
                if (kept(old_idx[e] - ix->row_base)) mine.push_back(okey.empty() ? nk::make_key(old_score[e], old_idx[e]) : okey[e]);
        const size_t f1 = f0;
        while (f0 < found.size() && found[f0].first == r) ++f0;
        merged.resize(mine.size() + (f0 - f1));
        std::vector<uint64_t> fk(f0 - f1);
        for (size_t i = f1; i < f0; ++i) fk[i - f1] = found[i].second;
        std::merge(mine.begin(), mine.end(), fk.begin(), fk.end(), merged.begin(), std::greater<uint64_t>());
        for (uint64_t key : merged) { decode_key(ix->metric, key, out_idx + w, out_score + w); ++w; }
    }
    return 0;
}

static int single_shard(NkIndex *ix, NkShard **out) {
    if (!ix) { nk::set_error("null index"); return -1; }
    if (ix->shards.size() != 1) { nk::set_error("device-resident search needs a single-device index"); return -1; }
    *out = &ix->shards[0];
    return 0;
}

// nk_search_keys_device with the index lock and the shard's call order held by the caller (Q, k > 0)
static int search_keys_locked(NkIndex *ix, NkShard *s, const float *queries_dev, uint32_t Q, uint32_t k, uint64_t *out_keys_dev,
                              cudaStream_t st) {
    if (!queries_dev || !out_keys_dev) { nk::set_error("null argument"); return -1; }
    if (k > NK_MAX_K_TOTAL) { nk::set_error("k=%u exceeds NK_MAX_K_TOTAL=%u", k, NK_MAX_K_TOTAL); return -1; }
    NK_CUDA_OK(cudaSetDevice(s->device));
    ix->stats.searches++;
    ix->stats.queries += Q;
    if (s->n == 0) {
        NK_CUDA_OK(cudaMemsetAsync(out_keys_dev, 0, (size_t)Q * k * 8, st));
        return (int)k;
    }
    if (run_scan(ix, *s, queries_dev, Q, k, out_keys_dev, st, ScanOut(ix->path))) return -1;
    return (int)k;
}

int nk_search_keys_device(NkIndex *ix, const float *queries_dev, uint32_t Q, uint32_t k, uint64_t *out_keys_dev,
                          void *stream) {
    nk::DeviceGuard _restore_device;
    NkShard *s;
    if (single_shard(ix, &s)) return -1;
    if (k == 0 || Q == 0) return 0;
    std::lock_guard<std::mutex> lk(ix->mu);
    const cudaStream_t st = stream ? (cudaStream_t)stream : s->stream;
    ShardOrder order(*s, st);
    if (order.failed()) return -1;
    return search_keys_locked(ix, s, queries_dev, Q, k, out_keys_dev, st);
}

// nk_search_device / nk_search_filtered_device / nk_search_windowed_device: filters_dev == windows_dev == nullptr is plain
// nk_search_device.
static int search_device(NkIndex *ix, const float *queries_dev, const NkFilter *filters_dev, const NkWindow *windows_dev, uint32_t Q,
                         uint32_t k, uint32_t *out_idx_dev, float *out_score_dev, void *stream) {
    nk::DeviceGuard _restore_device;
    NkShard *s;
    if (single_shard(ix, &s)) return -1;
    if (k == 0 || Q == 0) return 0;
    if (!queries_dev || !out_idx_dev || !out_score_dev) { nk::set_error("null argument"); return -1; }
    if (k > NK_MAX_K_TOTAL) { nk::set_error("k=%u exceeds NK_MAX_K_TOTAL=%u", k, NK_MAX_K_TOTAL); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);  // the row count is read under the lock (a concurrent append may change it)
    const uint64_t N = s->n;
    if (N == 0) return 0;
    if (k > N) { nk::set_error("nk_search_device: k=%u > rows=%llu (clamp on the host side)", k, (unsigned long long)N); return -1; }
    const cudaStream_t st = stream ? (cudaStream_t)stream : s->stream;
    ShardOrder order(*s, st);
    if (order.failed()) return -1;
    NK_CUDA_OK(cudaSetDevice(s->device));
    if (nk::ws_reserve((void **)&s->ws.keys, &s->ws.keys_bytes, (size_t)Q * k * 8)) return -1;
    ix->stats.searches++;
    ix->stats.queries += Q;
    ScanOut xo(ix->path, windows_dev ? nk::ScanMode::KNN_WINDOW : filters_dev ? nk::ScanMode::KNN_TAGS : nk::ScanMode::KNN);
    xo.out_idx = out_idx_dev; xo.out_score = out_score_dev;  // decoded by the last kernel of the path
    // the caller's filters and windows are read in place: the caller keeps them valid until the stream has run (the blindly
    // queued tail reads them too); a windowed scan without filters gets {0,0,0} staged on the caller's stream
    xo.qfilter = filters_dev; xo.qwindow = windows_dev;
    if (filters_dev ? shard_tags_on(*s) : stage_predicates(ix, *s, st, xo.mode, Q, nullptr, nullptr)) return -1;
    if (windows_dev && shard_values_on(*s)) return -1;
    if (run_scan(ix, *s, queries_dev, Q, k, s->ws.keys, st, xo)) return -1;
    return (int)k;
}

int nk_search_device(NkIndex *ix, const float *queries_dev, uint32_t Q, uint32_t k, uint32_t *out_idx_dev,
                     float *out_score_dev, void *stream) {
    return search_device(ix, queries_dev, nullptr, nullptr, Q, k, out_idx_dev, out_score_dev, stream);
}

int nk_search_filtered_device(NkIndex *ix, const float *queries_dev, const NkFilter *filters_dev, uint32_t Q, uint32_t k,
                              uint32_t *out_idx_dev, float *out_score_dev, void *stream) {
    return search_device(ix, queries_dev, filters_dev, nullptr, Q, k, out_idx_dev, out_score_dev, stream);
}

int nk_search_windowed_device(NkIndex *ix, const float *queries_dev, const NkFilter *filters_dev, const NkWindow *windows_dev,
                              uint32_t Q, uint32_t k, uint32_t *out_idx_dev, float *out_score_dev, void *stream) {
    return search_device(ix, queries_dev, filters_dev, windows_dev, Q, k, out_idx_dev, out_score_dev, stream);
}

// Device-resident searches cannot report a (never expected) candidate-buffer overflow when they return: this call waits
// for `stream` (NULL = the index's own streams), reads and clears the sticky status word of every shard, and returns 0 or -1
// with the message nk_search would have given.  Call it wherever the caller synchronises anyway.
int nk_index_status(NkIndex *ix, void *stream) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    int bad = 0;
    for (auto &s : ix->shards) {
        NK_CUDA_OK(cudaSetDevice(s.device));
        if (stream) NK_CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));
        if (shard_drain(s)) return -1;
        int h = 0;
        NK_CUDA_OK(cudaMemcpy(&h, s.ws.flags, sizeof(int), cudaMemcpyDeviceToHost));
        if (h) {
            // cleared synchronously: this call holds no ShardOrder, so a clear queued on a stream would not be ordered
            // before the index's next call
            NK_CUDA_OK(cudaMemset(s.ws.flags, 0, sizeof(int)));
            bad = h;
        }
    }
    return bad ? nk::fatal_overflow(bad, nullptr, nullptr) : 0;
}

// (No scratch buffer: the merge kernel writes the decoded arrays itself, so concurrent merges on different streams share
// nothing.)
int nk_merge_keys_device(int device_id, const uint64_t *keys_dev, uint32_t n_lists, uint32_t Q, uint32_t k, int metric,
                         uint32_t *out_idx_dev, float *out_score_dev, void *stream) {
    nk::DeviceGuard _restore_device;
    if (k == 0 || Q == 0 || n_lists == 0) return 0;
    if (k > NK_MAX_K) { nk::set_error("nk_merge_keys_device: k=%u exceeds NK_MAX_K=%u (the merge width)", k, NK_MAX_K); return -1; }
    if (!keys_dev || !out_idx_dev || !out_score_dev) { nk::set_error("null argument"); return -1; }
    if (device_id < 0 || device_id >= 64) { nk::set_error("bad device id %d", device_id); return -1; }
    NK_CUDA_OK(cudaSetDevice(device_id));
    cudaStream_t st = (cudaStream_t)stream;
    // No stream given: behave synchronously (the producers may have run on the indexes' own non-blocking streams,
    // which the legacy default stream does not order against).
    if (!st) NK_CUDA_OK(cudaDeviceSynchronize());
    // one fused launch: merge the lists and write the decoded (index, score) arrays; no intermediate key buffer
    int rc = nk::merge_keys(keys_dev, n_lists, (size_t)Q * k, k, Q, k, nullptr, st, nullptr, 0, out_idx_dev, out_score_dev, metric);
    if (rc == 0 && !st) NK_CUDA_OK(cudaStreamSynchronize(st));
    return rc;
}

int nk_score_subset(NkIndex *ix, const float *query_host, const uint32_t *rows_host, uint32_t n_subset, uint32_t k,
                    uint32_t *out_idx, float *out_score) {
    nk::DeviceGuard _restore_device;
    NkShard *s;
    if (single_shard(ix, &s)) return -1;
    if (n_subset == 0 || k == 0) return 0;
    if (!query_host || !rows_host || !out_idx || !out_score) { nk::set_error("null argument"); return -1; }
    const uint32_t ke = std::min(k, n_subset);
    if (ke > NK_MAX_K_TOTAL) { nk::set_error("k=%u exceeds NK_MAX_K_TOTAL=%u", ke, NK_MAX_K_TOTAL); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    for (uint32_t i = 0; i < n_subset; ++i)
        if (rows_host[i] < ix->row_base || rows_host[i] - ix->row_base >= s->n) {
            nk::set_error("subset row %u out of range", rows_host[i]);
            return -1;
        }
    ShardOrder order(*s, s->stream);
    if (order.failed()) return -1;
    NK_CUDA_OK(cudaSetDevice(s->device));
    const size_t rb = (size_t)ix->dim * ix->esz();
    // grow-only workspace of the shard: no allocation per call (cuda.Device.Search allocates two buffers per query,
    // cuda_bridge.go:652-663)
    if (nk::ws_reserve((void **)&s->ws.sub_rows, &s->ws.sub_rows_bytes, (size_t)n_subset * 4)) return -1;
    if (nk::ws_reserve(&s->ws.sub_gather, &s->ws.sub_gather_bytes, (size_t)n_subset * rb)) return -1;
    uint32_t *d_rows = s->ws.sub_rows;
    void *d_gather = s->ws.sub_gather;
    std::vector<uint32_t> local(rows_host, rows_host + n_subset);
    for (auto &r : local) r -= (uint32_t)ix->row_base;
    int rc = 0;
    std::vector<uint32_t> pos((size_t)ke);
    do {
        if (cudaMemcpyAsync(d_rows, local.data(), (size_t)n_subset * 4, cudaMemcpyHostToDevice, s->stream) != cudaSuccess) { rc = -1; break; }
        if (nk::gather_rows(s->rows, ix->dtype, ix->dim, d_rows, n_subset, d_gather, false, s->stream)) { rc = -1; break; }
        if (nk::ws_reserve((void **)&s->ws.queries, &s->ws.queries_bytes, (size_t)ix->dim * 4)) { rc = -1; break; }
        if (nk::ws_reserve((void **)&s->ws.keys, &s->ws.keys_bytes, (size_t)ke * 8)) { rc = -1; break; }
        if (nk::ws_reserve((void **)&s->ws.out_idx, &s->ws.out_idx_bytes, (size_t)ke * 4)) { rc = -1; break; }
        if (nk::ws_reserve((void **)&s->ws.out_score, &s->ws.out_score_bytes, (size_t)ke * 4)) { rc = -1; break; }
        if (cudaMemcpyAsync(s->ws.queries, query_host, (size_t)ix->dim * 4, cudaMemcpyHostToDevice, s->stream) != cudaSuccess) { rc = -1; break; }
        // the gathered rows, positions 0..n_subset-1: no row mask, score floor or tags
        nk::ScanArgs a;
        a.rows = d_gather; a.dtype = ix->dtype; a.n = n_subset; a.dim = ix->dim; a.row_base = 0;
        a.queries = s->ws.queries; a.Q = 1; a.k = ke; a.metric = ix->metric; a.stream = s->stream;
        if (ke > NK_MAX_K) {  // ScoreSubset ranks every candidate (up to MaxCandidates = 5000, vector_pipeline.go:24-31)
            if (run_scan_bigk(ix, *s, a, s->ws.keys)) { rc = -1; break; }
            if (nk::decode_keys(s->ws.keys, 1, ke, ix->metric, s->ws.out_idx, s->ws.out_score, s->stream)) { rc = -1; break; }
        } else {
            a.out_idx = s->ws.out_idx; a.out_score = s->ws.out_score;  // decoded by the merge launch
            if (nk::scan_simt(s->di, a, s->ws, s->ws.keys, &ix->stats.kernel_launches)) { rc = -1; break; }
            ix->stats.bytes_scanned += scan_bytes(ix, NK_PATH_SIMT, a, 1);
        }
        if (cudaMemcpyAsync(pos.data(), s->ws.out_idx, (size_t)ke * 4, cudaMemcpyDeviceToHost, s->stream) != cudaSuccess) { rc = -1; break; }
        if (cudaMemcpyAsync(out_score, s->ws.out_score, (size_t)ke * 4, cudaMemcpyDeviceToHost, s->stream) != cudaSuccess) { rc = -1; break; }
    } while (0);
    if (rc != 0) {
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) nk::set_error("nk_score_subset: %s", cudaGetErrorString(e));
        cudaStreamSynchronize(s->stream);
        return -1;
    }
    if (finish_deferred(ix, *s, nullptr) < 0) return -1;
    // positions within the subset -> global row ids (ties broken by subset position, like the stable
    // order of ScoreSubset's input list)
    for (uint32_t i = 0; i < ke; ++i) out_idx[i] = pos[i] < n_subset ? rows_host[pos[i]] : 0xffffffffu;
    return (int)ke;
}

// ---- k-means routing on device (pkg/gpu/kmeans.go; SURVEY.md §8(f)4) -----------------------------------------------
// Assignment (DESIGN §7 item 3).  With a usable BF16 shadow it is ONE pass of the tensor-core scan with an argmax
// epilogue (assign_tensor.cu); otherwise the fused kNN scan with the roles swapped: the K centroids are the indexed corpus,
// the shard's rows are the queries — read in place from HBM, 8192 at a time — and k = min(2, K).  Either way the rows a
// rigorous bound cannot decide are listed and assign_fixup_kernel decides them with the contract's arithmetic, so both
// paths return the same assignment.  ties_* (tests, single-device index): the near-tie list of that call.
static int assign_nearest(NkIndex *ix, const float *centroids_host, uint32_t K, int metric, int32_t *assign_io, uint64_t *changed,
                          uint32_t *ties_rows, uint32_t *ties_cand, uint32_t ties_cap, uint32_t *ties_count) {
    nk::DeviceGuard _restore_device;
    if (!ix || !centroids_host || !assign_io) { nk::set_error("null argument"); return -1; }
    if (ix->dtype != NK_DTYPE_F32) { nk::set_error("nk_index_assign_nearest: fp32 index required"); return -1; }
    if (K == 0) { nk::set_error("nk_index_assign_nearest: K must be >= 1"); return -1; }
    if (metric < NK_METRIC_COSINE || metric > NK_METRIC_EUCLIDEAN) { nk::set_error("unknown metric %d", metric); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    ShardOrder order(ix);
    if (order.failed()) return -1;
    uint64_t total_changed = 0, off = 0;
    if (ties_count) *ties_count = 0;
    for (auto &s : ix->shards) {
        if (s.n == 0) continue;
        NK_CUDA_OK(cudaSetDevice(s.device));
        const nk::RowImage img = shard_image(ix, s, false, 0);
        const bool tensor = img.kind != nk::RowImage::NONE && nk::assign_tensor_supported(s.di, ix->dim, K, metric);
        const uint32_t k = K < 2 ? K : 2u;
        NkIndex *cx = tensor ? nullptr : nk_index_create(&s.device, 1, ix->dim, NK_DTYPE_F32, metric);
        if (!tensor && !cx) return -1;
        // one grow-only scratch buffer per shard, carved up (no cudaMalloc / cudaFree per call): search results [n x k]
        // (indices, scores), the assignment, the previous one, the changed count, the near-tie list, the centroids
        const size_t n4 = (s.n * 4 + 255) & ~(size_t)255, cen_b = ((size_t)K * ix->dim * 4 + 255) & ~(size_t)255;
        const size_t o_sc = 2 * n4, o_asg = 4 * n4, o_prev = 5 * n4, o_chg = 6 * n4, o_tc = o_chg + 256, o_tr = o_tc + 256, o_tcand = o_tr + n4,
                     o_cen = o_tcand + 4 * n4;
        unsigned long long h_changed = 0;
        int rc = tensor ? 0 : nk_index_upload(cx, centroids_host, K);
        if (rc == 0 && nk::ws_reserve(&s.ws.scratch, &s.ws.scratch_bytes, o_cen + cen_b)) rc = -1;
        unsigned char *base = static_cast<unsigned char *>(s.ws.scratch);
        uint32_t *d_idx = reinterpret_cast<uint32_t *>(base);
        float *d_sc = reinterpret_cast<float *>(base + o_sc);
        uint32_t *d_asg = reinterpret_cast<uint32_t *>(base + o_asg);
        int32_t *d_prev = reinterpret_cast<int32_t *>(base + o_prev);
        unsigned long long *d_changed = reinterpret_cast<unsigned long long *>(base + o_chg);
        nk::AssignTies ties;
        ties.count = reinterpret_cast<uint32_t *>(base + o_tc);
        ties.rows = reinterpret_cast<uint32_t *>(base + o_tr);
        ties.cand = reinterpret_cast<uint32_t *>(base + o_tcand);
        ties.cap = (uint32_t)s.n;
        float *d_cen = reinterpret_cast<float *>(base + o_cen);
        cudaError_t e = cudaSuccess;
        if (rc == 0) {
            e = cudaMemcpyAsync(d_cen, centroids_host, (size_t)K * ix->dim * 4, cudaMemcpyHostToDevice, s.stream);
            if (e == cudaSuccess) e = cudaMemsetAsync(d_changed, 0, 8, s.stream);
            if (e == cudaSuccess) e = cudaMemcpyAsync(d_prev, assign_io + off, s.n * 4, cudaMemcpyHostToDevice, s.stream);
            if (e != cudaSuccess) rc = -1;
        }
        const float *rows = static_cast<const float *>(s.rows);
        if (rc == 0 && tensor)
            rc = nk::assign_tensor(s.di, rows, img, (uint32_t)s.n, ix->dim, d_cen, K, metric, ties, d_asg, s.stream, &ix->stats.kernel_launches,
                                   &s.ws.sub_gather, &s.ws.sub_gather_bytes);
        const uint64_t B = 8192;  // rows per fused search: amortises the ~12 fixed launches of a search over 8 scan launches
        for (uint64_t b = 0; rc == 0 && !tensor && b < s.n; b += B) {
            const uint32_t nb = (uint32_t)std::min<uint64_t>(B, s.n - b);
            if (nk_search_device(cx, rows + b * ix->dim, nb, k, d_idx + b * k, d_sc + b * k, s.stream) < 0) rc = -1;
        }
        if (rc == 0 && !tensor)
            rc = nk::assign_from_search(s.di, rows, (uint32_t)s.n, ix->dim, d_cen, K, metric, d_idx, d_sc, k, ties, d_asg, s.stream,
                                        &ix->stats.kernel_launches);
        if (rc == 0 && nk::count_changed(d_prev, d_asg, s.n, d_changed, s.stream)) rc = -1;
        uint32_t h_ties = 0;
        if (rc == 0) {
            e = cudaMemcpyAsync(assign_io + off, d_asg, s.n * 4, cudaMemcpyDeviceToHost, s.stream);
            if (e == cudaSuccess) e = cudaMemcpyAsync(&h_changed, d_changed, 8, cudaMemcpyDeviceToHost, s.stream);
            if (e == cudaSuccess && ties_count) e = cudaMemcpyAsync(&h_ties, ties.count, 4, cudaMemcpyDeviceToHost, s.stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(s.stream);
            const uint32_t m = std::min(h_ties, ties_cap);
            if (e == cudaSuccess && m) e = cudaMemcpyAsync(ties_rows, ties.rows, (size_t)m * 4, cudaMemcpyDeviceToHost, s.stream);
            if (e == cudaSuccess && m) e = cudaMemcpyAsync(ties_cand, ties.cand, (size_t)m * 16, cudaMemcpyDeviceToHost, s.stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(s.stream);
            if (e != cudaSuccess) rc = -1;
        }
        if (e != cudaSuccess) { nk::set_error("nk_index_assign_nearest: %s", cudaGetErrorString(e)); cudaGetLastError(); }
        cudaStreamSynchronize(s.stream);
        ix->stats.kernel_launches += (cx ? cx->stats.kernel_launches : 0) + 1;
        if (cx) nk_index_release(cx);
        if (rc != 0) return -1;
        if (ties_count) *ties_count = h_ties;
        total_changed += h_changed;
        off += s.n;
    }
    if (changed) *changed = total_changed;
    return 0;
}

int nk_index_assign_nearest(NkIndex *ix, const float *centroids_host, uint32_t K, int metric, int32_t *assign_io, uint64_t *changed) {
    return assign_nearest(ix, centroids_host, K, metric, assign_io, changed, nullptr, nullptr, 0, nullptr);
}

// Tests only: run the assignment of every row (from a zero assignment; the result is discarded) and return the number of
// rows it listed as near-ties; the first min(count, cap) rows and their 4 candidate ids are copied to rows_out / cand_out.
int nk_debug_assign_ties(NkIndex *ix, const float *centroids_host, uint32_t K, int metric, uint32_t *rows_out, uint32_t *cand_out,
                         uint32_t cap) {
    if (!ix || ix->shards.size() != 1) { nk::set_error("single-device index required"); return -1; }
    if (cap && (!rows_out || !cand_out)) { nk::set_error("null argument"); return -1; }
    if (ix->shards[0].n == 0) return 0;
    std::vector<int32_t> assign(ix->shards[0].n, 0);
    uint32_t count = 0;
    if (assign_nearest(ix, centroids_host, K, metric, assign.data(), nullptr, rows_out, cand_out, cap, &count)) return -1;
    return (int)count;
}

// Update step (kmeans.go:585-618): centroid c <- float32(mean in float64 of the rows assigned to c); clusters without
// members keep their previous position.  Rows with an assignment outside [0, K) are ignored.
int nk_index_cluster_means(NkIndex *ix, const int32_t *assign_host, uint32_t K, float *centroids_io, uint32_t *counts_out) {
    nk::DeviceGuard _restore_device;
    if (!ix || !assign_host || !centroids_io) { nk::set_error("null argument"); return -1; }
    if (ix->dtype != NK_DTYPE_F32) { nk::set_error("nk_index_cluster_means: fp32 index required"); return -1; }
    if (K == 0) return 0;
    std::lock_guard<std::mutex> lk(ix->mu);
    ShardOrder order(ix);
    if (order.failed()) return -1;
    const size_t KD = (size_t)K * ix->dim;
    std::vector<double> sums(KD, 0.0), part(KD);
    std::vector<unsigned long long> counts(K, 0ull), cpart(K);
    uint64_t off = 0;
    for (auto &s : ix->shards) {
        if (s.n == 0) continue;
        NK_CUDA_OK(cudaSetDevice(s.device));
        const size_t kd8 = (KD * 8 + 255) & ~(size_t)255, k8 = ((size_t)K * 8 + 255) & ~(size_t)255;
        if (nk::ws_reserve(&s.ws.scratch, &s.ws.scratch_bytes, kd8 + k8 + s.n * 4)) return -1;  // grow-only, reused across calls
        unsigned char *base = static_cast<unsigned char *>(s.ws.scratch);
        double *d_sums = reinterpret_cast<double *>(base);
        unsigned long long *d_counts = reinterpret_cast<unsigned long long *>(base + kd8);
        int32_t *d_assign = reinterpret_cast<int32_t *>(base + kd8 + k8);
        cudaError_t e = cudaMemsetAsync(d_sums, 0, KD * 8, s.stream);
        if (e == cudaSuccess) e = cudaMemsetAsync(d_counts, 0, (size_t)K * 8, s.stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_assign, assign_host + off, s.n * 4, cudaMemcpyHostToDevice, s.stream);
        int rc = e == cudaSuccess ? nk::cluster_sums(static_cast<const float *>(s.rows), s.n, ix->dim, d_assign, K, d_sums, d_counts, s.stream) : -1;
        if (rc == 0) {
            e = cudaMemcpyAsync(part.data(), d_sums, KD * 8, cudaMemcpyDeviceToHost, s.stream);
            if (e == cudaSuccess) e = cudaMemcpyAsync(cpart.data(), d_counts, (size_t)K * 8, cudaMemcpyDeviceToHost, s.stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(s.stream);
        }
        if (e != cudaSuccess) { nk::set_error("nk_index_cluster_means: %s", cudaGetErrorString(e)); cudaGetLastError(); rc = -1; }
        cudaStreamSynchronize(s.stream);
        if (rc != 0) return -1;
        ix->stats.kernel_launches++;
        for (size_t i = 0; i < KD; ++i) sums[i] += part[i];
        for (uint32_t c = 0; c < K; ++c) counts[c] += cpart[c];
        off += s.n;
    }
    for (uint32_t c = 0; c < K; ++c) {
        if (counts[c])
            for (uint32_t d = 0; d < ix->dim; ++d) centroids_io[(size_t)c * ix->dim + d] = (float)(sums[(size_t)c * ix->dim + d] / (double)counts[c]);
        if (counts_out) counts_out[c] = (uint32_t)counts[c];
    }
    return 0;
}

// k-means++ seeding over every row (kmeans.go:364-426; include/nornic_knn.h, DESIGN §7 item 3).  Each shard keeps, in its
// scratch, every row's D² and nearest seed, the sums of its chunks of 256 rows, the δ² of the newest seed to the earlier
// ones and the grow-only list of the seeds so far.  Per seed: one pass per shard (kmeanspp_pass), then the pick on the
// host from the chunk sums and the weights of the one chunk the target falls in, the same code for any number of devices.
struct KmppShard {
    NkShard *s = nullptr;
    uint64_t first = 0, nch = 0;
    double *d2 = nullptr, *sums = nullptr, *delta = nullptr;
    uint32_t *near = nullptr;
    float *seeds = nullptr;
    unsigned long long *read = nullptr;
    std::vector<double> h_sums;
};

int nk_index_kmeanspp(NkIndex *ix, uint32_t K, uint64_t first_row, const double *u_host, uint32_t *seeds_out, float *centroids_out,
                      double *potential_out, double *min_d2_out, uint64_t *rows_read) {
    nk::DeviceGuard _restore_device;
    if (!ix || !seeds_out || (K > 1 && !u_host)) { nk::set_error("null argument"); return -1; }
    if (ix->dtype != NK_DTYPE_F32) { nk::set_error("nk_index_kmeanspp: fp32 index required"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    const uint64_t n = ix->rows();
    if (K == 0 || K > n) { nk::set_error("nk_index_kmeanspp: K=%u outside [1, %llu rows]", K, (unsigned long long)n); return -1; }
    if (first_row >= n) { nk::set_error("nk_index_kmeanspp: first_row %llu >= %llu rows", (unsigned long long)first_row, (unsigned long long)n); return -1; }
    for (uint32_t c = 0; c + 1 < K; ++c)
        if (!(u_host[c] >= 0.0 && u_host[c] < 1.0)) { nk::set_error("nk_index_kmeanspp: u[%u] = %g is not in [0, 1)", c, u_host[c]); return -1; }
    bool prune = true;
    if (const char *e = getenv("NK_KMPP_PRUNE"))
        if (atoi(e) == 0) prune = false;
    ShardOrder order(ix);
    if (order.failed()) return -1;
    const uint32_t dim = ix->dim;
    const size_t rowb = (size_t)dim * 4;
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    std::vector<KmppShard> sh;
    for (NkShard *s : live_shards(ix)) {
        KmppShard k;
        k.s = s; k.first = ix->first_row(*s); k.nch = (s->n + nk::KMPP_CHUNK - 1) / nk::KMPP_CHUNK;
        const size_t o_near = al(s->n * 8), o_sums = o_near + al(s->n * 4), o_delta = o_sums + al(k.nch * 8),
                     o_seeds = o_delta + al((size_t)K * 8), o_read = o_seeds + al((size_t)K * rowb);
        NK_CUDA_OK(cudaSetDevice(s->device));
        if (nk::ws_reserve(&s->ws.scratch, &s->ws.scratch_bytes, o_read + 256)) return -1;  // grow-only, reused across calls
        unsigned char *base = static_cast<unsigned char *>(s->ws.scratch);
        k.d2 = reinterpret_cast<double *>(base);
        k.near = reinterpret_cast<uint32_t *>(base + o_near);
        k.sums = reinterpret_cast<double *>(base + o_sums);
        k.delta = reinterpret_cast<double *>(base + o_delta);
        k.seeds = reinterpret_cast<float *>(base + o_seeds);
        k.read = reinterpret_cast<unsigned long long *>(base + o_read);
        k.h_sums.resize(k.nch);
        NK_CUDA_OK(cudaMemsetAsync(k.read, 0, 8, s->stream));
        sh.push_back(std::move(k));
    }
    auto owner = [&](uint64_t row) -> KmppShard & {
        for (auto &k : sh)
            if (row < k.first + k.s->n) return k;
        return sh.back();
    };
    std::vector<float> crow(dim);
    std::vector<double> prefix;  // P_j over every shard's chunks, in row order
    std::vector<double> w(nk::KMPP_CHUNK);
    uint64_t seed = first_row;
    for (uint32_t c = 0; c < K; ++c) {
        seeds_out[c] = (uint32_t)seed;
        KmppShard &o = owner(seed);
        NK_CUDA_OK(cudaSetDevice(o.s->device));
        NK_CUDA_OK(cudaMemcpyAsync(crow.data(), static_cast<const float *>(o.s->rows) + (seed - o.first) * dim, rowb, cudaMemcpyDeviceToHost, o.s->stream));
        NK_CUDA_OK(cudaStreamSynchronize(o.s->stream));
        if (centroids_out) memcpy(centroids_out + (size_t)c * dim, crow.data(), rowb);
        for (auto &k : sh) {
            NkShard &s = *k.s;
            NK_CUDA_OK(cudaSetDevice(s.device));
            NK_CUDA_OK(cudaMemcpyAsync(k.seeds + (size_t)c * dim, crow.data(), rowb, cudaMemcpyHostToDevice, s.stream));
            cudaEvent_t ev[2] = {nullptr, nullptr};
            if (ix->timing_on) {
                NK_CUDA_OK(cudaEventCreate(&ev[0]));
                NK_CUDA_OK(cudaEventCreate(&ev[1]));
                NK_CUDA_OK(cudaEventRecord(ev[0], s.stream));
            }
            uint64_t launches = 0;
            const int rc = nk::kmeanspp_pass(s.di, static_cast<const float *>(s.rows), s.n, dim, k.seeds, c, k.delta, prune, k.d2, k.near,
                                             k.sums, k.read, s.stream, &launches);
            if (ev[0]) {
                cudaEventRecord(ev[1], s.stream);
                s.timing.emplace_back(ev[0], ev[1]);
                s.timing_launches.push_back(launches);
            }
            if (rc) return -1;
            ix->stats.kernel_launches += launches;
            NK_CUDA_OK(cudaMemcpyAsync(k.h_sums.data(), k.sums, k.nch * 8, cudaMemcpyDeviceToHost, s.stream));
        }
        prefix.clear();
        double T = 0.0;
        for (auto &k : sh) {
            NK_CUDA_OK(cudaSetDevice(k.s->device));
            NK_CUDA_OK(cudaStreamSynchronize(k.s->stream));
            for (double S : k.h_sums) prefix.push_back(T = T + S);
        }
        if (potential_out) potential_out[c] = T;
        if (c + 1 == K) break;
        // the next seed: the first chunk whose inclusive prefix reaches the target, then the first row of it whose running
        // sum does; no chunk (a NaN sum or target): the last row, kmeans.go:397
        const double target = u_host[c] * T;
        const size_t j = std::find_if(prefix.begin(), prefix.end(), [&](double P) { return P >= target; }) - prefix.begin();
        if (j == prefix.size()) { seed = n - 1; continue; }
        size_t jj = j;
        KmppShard *kj = nullptr;
        for (auto &k : sh) {
            if (jj < k.nch) { kj = &k; break; }
            jj -= k.nch;
        }
        const uint64_t r0 = jj * nk::KMPP_CHUNK, cnt = std::min<uint64_t>(nk::KMPP_CHUNK, kj->s->n - r0);
        NK_CUDA_OK(cudaSetDevice(kj->s->device));
        NK_CUDA_OK(cudaMemcpyAsync(w.data(), kj->d2 + r0, cnt * 8, cudaMemcpyDeviceToHost, kj->s->stream));
        NK_CUDA_OK(cudaStreamSynchronize(kj->s->stream));
        const double before = j ? prefix[j - 1] : 0.0;
        uint64_t pick = cnt - 1;  // reached at the latest by the chunk's last row: its running sum is S_j, added in the same order
        double L = 0.0;
        for (uint64_t i = 0; i < cnt; ++i) {
            L = L + w[i];
            if (before + L >= target) { pick = i; break; }
        }
        seed = kj->first + r0 + pick;
    }
    uint64_t total_read = 0;
    for (auto &k : sh) {
        NkShard &s = *k.s;
        unsigned long long r = 0;
        NK_CUDA_OK(cudaSetDevice(s.device));
        if (min_d2_out) NK_CUDA_OK(cudaMemcpyAsync(min_d2_out + k.first, k.d2, s.n * 8, cudaMemcpyDeviceToHost, s.stream));
        NK_CUDA_OK(cudaMemcpyAsync(&r, k.read, 8, cudaMemcpyDeviceToHost, s.stream));
        NK_CUDA_OK(cudaStreamSynchronize(s.stream));
        total_read += r;
    }
    ix->stats.bytes_scanned += total_read * rowb;
    if (rows_read) *rows_read = total_read;
    return 0;
}

// ---- best-of-chunks per node (db.index.vector.queryNodes, call_vector.go:177-256; SURVEY.md §8(f)2) -------------------------
// Rows are chunk embeddings; group_of_row[r] = the node row r belongs to (ids in [0, n_groups)).  Stays set until a
// row-count changing mutation (like the row mask, whose bits are positions).
int nk_index_set_row_groups(NkIndex *ix, const uint32_t *group_of_row, uint64_t n_rows, uint32_t n_groups) {
    nk::DeviceGuard _restore_device;
    if (!ix) { nk::set_error("null index"); return -1; }
    std::lock_guard<std::mutex> lk(ix->mu);
    if (!group_of_row) {
        ix->n_groups = 0;
        for (auto &s : ix->shards) s.group_on = false;
        return 0;
    }
    if (ix->shards.size() != 1) { nk::set_error("row groups apply to single-device indexes"); return -1; }
    if (n_rows != ix->rows()) { nk::set_error("row groups: %llu entries, index has %llu rows", (unsigned long long)n_rows, (unsigned long long)ix->rows()); return -1; }
    if (n_groups == 0) { nk::set_error("row groups: n_groups must be >= 1"); return -1; }
    for (uint64_t r = 0; r < n_rows; ++r)
        if (group_of_row[r] >= n_groups) { nk::set_error("row groups: group id %u of row %llu out of range", group_of_row[r], (unsigned long long)r); return -1; }
    NkShard &s = ix->shards[0];
    ShardOrder order(s, s.stream);
    if (order.failed()) return -1;
    NK_CUDA_OK(cudaSetDevice(s.device));
    if (nk::ws_reserve((void **)&s.group, &s.group_bytes, (size_t)(n_rows ? n_rows : 1) * 4)) return -1;
    NK_CUDA_OK(cudaMemcpyAsync(s.group, group_of_row, n_rows * 4, cudaMemcpyHostToDevice, s.stream));
    NK_CUDA_OK(cudaStreamSynchronize(s.stream));
    s.group_on = true;
    ix->n_groups = n_groups;
    return 0;
}

// One query against the chunk rows; result = the k best NODES, each with the score and row of its best chunk, ordered by
// (score desc, best-chunk row asc).  Honours the row mask (label filter) and the score floor (nk_index_set_min_score: the
// reference keeps a node only if bestScore >= 0, call_vector.go:243).  Exact fp32 scores, no over-select loop: one pass
// with a per-node atomic max (segment-max), one top-k over the node keys.  Returns the number of nodes found (<= k).
int nk_search_groups(NkIndex *ix, const float *query_host, uint32_t k, uint32_t *out_group, uint32_t *out_row, float *out_score) {
    nk::DeviceGuard _restore_device;
    NkShard *s;
    if (single_shard(ix, &s)) return -1;
    std::lock_guard<std::mutex> lk(ix->mu);
    if (k == 0 || s->n == 0) return 0;
    if (!query_host || !out_group || !out_row || !out_score) { nk::set_error("null argument"); return -1; }
    if (!s->group_on || ix->n_groups == 0) { nk::set_error("nk_search_groups: no row groups set (nk_index_set_row_groups)"); return -1; }
    const uint32_t G = ix->n_groups, ke = k < G ? k : G;
    if (ke > NK_MAX_K) { nk::set_error("nk_search_groups: k=%u exceeds NK_MAX_K=%u", ke, NK_MAX_K); return -1; }
    ShardOrder order(*s, s->stream);
    if (order.failed()) return -1;
    NK_CUDA_OK(cudaSetDevice(s->device));
    ScopedRange range("nk_search_groups");
    if (nk::ws_reserve((void **)&s->ws.queries, &s->ws.queries_bytes, (size_t)ix->dim * 4)) return -1;
    if (nk::ws_reserve(&s->ws.scratch, &s->ws.scratch_bytes, (size_t)G * 8)) return -1;
    if (nk::ws_reserve((void **)&s->ws.keys, &s->ws.keys_bytes, (size_t)ke * 8)) return -1;
    if (nk::ws_reserve((void **)&s->ws.out_idx, &s->ws.out_idx_bytes, (size_t)ke * 8)) return -1;
    if (nk::ws_reserve((void **)&s->ws.out_score, &s->ws.out_score_bytes, (size_t)ke * 4)) return -1;
    unsigned long long *best = static_cast<unsigned long long *>(s->ws.scratch);
    NK_CUDA_OK(cudaMemcpyAsync(s->ws.queries, query_host, (size_t)ix->dim * 4, cudaMemcpyHostToDevice, s->stream));
    NK_CUDA_OK(cudaMemsetAsync(best, 0, (size_t)G * 8, s->stream));
    if (nk::group_best(s->di, s->rows, ix->dtype, s->n, ix->dim, s->base, s->ws.queries, ix->metric, s->group, s->mask_on ? s->mask : nullptr,
                       ix->key_floor(), best, s->stream))
        return -1;
    if (nk::topk_keys(s->di, best, G, ke, s->ws, s->ws.keys, s->stream)) return -1;
    if (nk::decode_group_keys(s->ws.keys, ke, ix->metric, s->group, s->base, s->ws.out_idx, s->ws.out_idx + ke, s->ws.out_score, s->stream)) return -1;
    ix->stats.kernel_launches += 4;
    ix->stats.searches++; ix->stats.queries++;
    ix->stats.bytes_scanned += (uint64_t)s->n * ix->dim * ix->esz();
    NK_CUDA_OK(cudaMemcpyAsync(out_group, s->ws.out_idx, (size_t)ke * 4, cudaMemcpyDeviceToHost, s->stream));
    NK_CUDA_OK(cudaMemcpyAsync(out_row, s->ws.out_idx + ke, (size_t)ke * 4, cudaMemcpyDeviceToHost, s->stream));
    NK_CUDA_OK(cudaMemcpyAsync(out_score, s->ws.out_score, (size_t)ke * 4, cudaMemcpyDeviceToHost, s->stream));
    if (finish_deferred(ix, *s, nullptr) < 0) return -1;
    uint32_t found = 0;
    while (found < ke && out_group[found] != 0xffffffffu) ++found;
    return (int)found;
}

// ---- row-sharded search with the exchange behind the ABI (exchange.cu) ----------------------------------------------------
// One rank per GPU (one process each, or several single-device indexes in one process): scan this rank's shard, push the
// Q*k candidate keys into every peer's buffer over NVLink, merge what the peers pushed.  Asynchronous on `stream`; every
// rank must make the same sequence of calls.  out_*_dev: [Q x k] on this rank's device, identical on every rank.
int nk_search_sharded_device(NkIndex *ix, NkComm *comm, const float *queries_dev, uint32_t Q, uint32_t k, uint32_t *out_idx_dev,
                             float *out_score_dev, void *stream) {
    nk::DeviceGuard _restore_device;
    NkShard *s;
    if (single_shard(ix, &s)) return -1;
    if (!comm) { nk::set_error("null communicator"); return -1; }
    if (k == 0 || Q == 0) return 0;
    // refused before the scan: the exchange could not merge the lists
    if (k > NK_MAX_K) { nk::set_error("nk_search_sharded_device: k=%u exceeds NK_MAX_K=%u (the merge width)", k, NK_MAX_K); return -1; }
    const cudaStream_t st = stream ? (cudaStream_t)stream : s->stream;
    // one call in the shard's order: the exchange reads the keys from the shard's workspace, which the next call may reuse
    std::lock_guard<std::mutex> lk(ix->mu);
    ShardOrder order(*s, st);
    if (order.failed()) return -1;
    NK_CUDA_OK(cudaSetDevice(s->device));
    if (nk::ws_reserve((void **)&s->ws.keys, &s->ws.keys_bytes, (size_t)Q * k * 8)) return -1;
    if (search_keys_locked(ix, s, queries_dev, Q, k, s->ws.keys, st) < 0) return -1;
    if (nk_comm_exchange_merge(comm, s->ws.keys, Q, k, ix->metric, out_idx_dev, out_score_dev, st) < 0) return -1;
    ix->stats.kernel_launches += 2;
    return (int)k;
}

int nk_fill_uniform_device(int device_id, float *out_dev, uint64_t n_rows, uint32_t dim, uint64_t seed,
                           uint64_t row_base, void *stream) {
    nk::DeviceGuard _restore_device;
    NK_CUDA_OK(cudaSetDevice(device_id));
    return nk::fill_uniform(out_dev, NK_DTYPE_F32, n_rows, dim, seed, row_base, (cudaStream_t)stream);
}

}  // extern "C"
