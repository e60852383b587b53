// nornic_cuda.hpp — C++ host-side mirror of the reference's Go host layer over the C ABI (include/nornic_knn.h).
//
// The reference's host side is Go (pkg/gpu/cuda/cuda_bridge.go:379-723 and pkg/gpu/gpu.go:1224-2454); no Go toolchain
// exists in the build image, so the compiled-language host mirror is C++ (header-only, links libnornic_knn.so).
// Same type / method names, argument meaning and error behaviour as the Go code, so tests/cpp/host_mirror_test.cpp
// reads like pkg/gpu/cuda/cuda_test.go and pkg/gpu/gpu_test.go.  Go's (value, error) returns become exceptions
// carrying the same sentinel identities (ErrCUDANotAvailable, ErrDeviceCreation, ErrBufferCreation,
// ErrKernelExecution, ErrInvalidBuffer — cuda_bridge.go:387-393; ErrInvalidDimensions — gpu.go).
//
//   namespace nornic::cuda   Device / Buffer / SearchResult / IsAvailable / DeviceCount / NewDevice
//   namespace nornic::gpu    EmbeddingIndex (Add / AddBatch / Remove / Search / SearchBatch / ScoreSubset /
//                            Count / Has / Get / Serialize / Deserialize), device corpus kept in step incrementally
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/nornic_knn.h"

namespace nornic {
namespace cuda {

struct CudaError : std::runtime_error { using std::runtime_error::runtime_error; };
struct ErrCUDANotAvailable : CudaError { ErrCUDANotAvailable() : CudaError("cuda: CUDA is not available on this system") {} };
struct ErrDeviceCreation : CudaError { using CudaError::CudaError; };
struct ErrBufferCreation : CudaError { using CudaError::CudaError; };
struct ErrKernelExecution : CudaError { using CudaError::CudaError; };
struct ErrInvalidBuffer : CudaError { using CudaError::CudaError; };

enum MemoryType { MemoryDevice = 0, MemoryPinned = 1 };  // cuda_bridge.go:396-404
enum class Metric { Cosine = NK_METRIC_COSINE, Dot = NK_METRIC_DOT, Euclidean = NK_METRIC_EUCLIDEAN };  // vectorspace/registry.go:27-31

struct SearchResult {  // cuda_bridge.go:425-428
    uint32_t Index;
    float Score;
};

inline std::string takeError() {  // cuda_bridge.go:452-453: read then clear
    const char *m = cuda_get_last_error();
    std::string s = m ? m : "";
    cuda_clear_error();
    return s;
}

inline bool IsAvailable() { return cuda_is_available() != 0; }                       // cuda_bridge.go:431
inline int DeviceCount() { int c = cuda_get_device_count(); return c < 0 ? 0 : c; }  // cuda_bridge.go:436

class Device;

class Buffer {  // cuda_bridge.go:417-422
public:
    Buffer(CudaBuffer *p, uint64_t size, Device *dev) : ptr_(p), size_(size), device_(dev) {}
    Buffer(const Buffer &) = delete;
    Buffer &operator=(const Buffer &) = delete;
    ~Buffer() { Release(); }
    void Release() {  // cuda_bridge.go:560-565 (idempotent)
        if (index_) { nk_index_release(index_); index_ = nullptr; }
        if (ptr_) { cuda_release_buffer(ptr_); ptr_ = nullptr; }
    }
    uint64_t Size() const { return size_; }
    std::vector<float> ReadFloat32(int count) const {  // cuda_bridge.go:573-585 (empty = Go's nil)
        if (count <= 0 || (uint64_t)count * 4 > size_ || !ptr_) return {};
        std::vector<float> out((size_t)count);
        if (cuda_buffer_copy_to_host(ptr_, out.data(), (size_t)count) != 0) return {};
        return out;
    }
    CudaBuffer *raw() const { return ptr_; }

private:
    friend class Device;
    CudaBuffer *ptr_;
    uint64_t size_;
    Device *device_;
    NkIndex *index_ = nullptr;  // cached fused-search handle over this buffer
    uint64_t index_n_ = 0;
    uint32_t index_dim_ = 0;
    int index_metric_ = -1;
};

class Device {  // cuda_bridge.go:407-415
public:
    explicit Device(int deviceID) : id_(deviceID) {
        if (!IsAvailable()) throw ErrCUDANotAvailable();
        ptr_ = cuda_create_device(deviceID);
        if (!ptr_) throw ErrDeviceCreation("cuda: failed to create CUDA device: " + takeError());
        int cc = cuda_device_compute_capability(deviceID);
        name_ = cuda_device_name(deviceID);
        memory_ = cuda_device_memory(deviceID);
        ccMajor_ = cc / 10;
        ccMinor_ = cc % 10;
    }
    Device(const Device &) = delete;
    Device &operator=(const Device &) = delete;
    ~Device() { Release(); }
    void Release() {  // cuda_bridge.go:470-478
        std::lock_guard<std::mutex> lk(mu_);
        if (ptr_) { cuda_release_device(ptr_); ptr_ = nullptr; }
    }
    int ID() const { return id_; }
    const std::string &Name() const { return name_; }
    uint64_t MemoryBytes() const { return memory_; }
    int MemoryMB() const { return (int)(memory_ / (1024 * 1024)); }
    std::pair<int, int> ComputeCapability() const { return {ccMajor_, ccMinor_}; }

    std::unique_ptr<Buffer> NewBuffer(const std::vector<float> &data, MemoryType memType = MemoryDevice) {  // cuda_bridge.go:506-532
        if (data.empty()) throw CudaError("cuda: cannot create empty buffer");
        std::lock_guard<std::mutex> lk(mu_);
        CudaBuffer *p = cuda_create_buffer(ptr_, const_cast<float *>(data.data()), data.size(), (int)memType);
        if (!p) throw ErrBufferCreation("cuda: failed to create buffer: " + takeError());
        return std::unique_ptr<Buffer>(new Buffer(p, data.size() * 4, this));
    }
    std::unique_ptr<Buffer> NewEmptyBuffer(uint64_t count, MemoryType memType = MemoryDevice) {  // cuda_bridge.go:535-557
        std::lock_guard<std::mutex> lk(mu_);
        CudaBuffer *p = cuda_create_buffer(ptr_, nullptr, (size_t)count, (int)memType);
        if (!p) throw ErrBufferCreation("cuda: failed to create buffer: " + takeError());
        return std::unique_ptr<Buffer>(new Buffer(p, count * 4, this));
    }
    void NormalizeVectors(Buffer &vectors, uint32_t n, uint32_t dimensions) {  // cuda_bridge.go:587-598
        std::lock_guard<std::mutex> lk(mu_);
        if (cuda_normalize_vectors(ptr_, vectors.ptr_, n, dimensions) != 0)
            throw ErrKernelExecution("cuda: kernel execution failed: " + takeError());
        // the buffer was rewritten: the 16-bit image of a cached index must follow
        if (vectors.index_ && nk_index_refresh_shadow(vectors.index_) != 0)
            throw ErrKernelExecution(std::string("cuda: kernel execution failed: ") + nk_last_error());
    }
    void CosineSimilarity(Buffer &embeddings, Buffer &query, Buffer &scores, uint32_t n, uint32_t dimensions, bool normalized) {  // :600-618
        std::lock_guard<std::mutex> lk(mu_);
        if (cuda_cosine_similarity(ptr_, embeddings.ptr_, query.ptr_, scores.ptr_, n, dimensions, normalized ? 1 : 0) != 0)
            throw ErrKernelExecution("cuda: kernel execution failed: " + takeError());
    }
    std::pair<std::vector<uint32_t>, std::vector<float>> TopK(Buffer &scores, uint32_t n, uint32_t k) {  // cuda_bridge.go:620-640
        std::lock_guard<std::mutex> lk(mu_);
        std::vector<uint32_t> idx(k);
        std::vector<float> top(k);
        if (cuda_topk(ptr_, scores.ptr_, idx.data(), top.data(), n, k) != 0)
            throw ErrKernelExecution("cuda: kernel execution failed: " + takeError());
        return {idx, top};
    }
    // cuda_bridge.go:643-686 — ONE fused call instead of NewBuffer + NewEmptyBuffer + CosineSimilarity + TopK.
    // normalized=true keeps the reference's meaning (raw dot of pre-normalised rows); false = true cosine.
    std::vector<SearchResult> Search(Buffer &embeddings, const std::vector<float> &query, uint32_t n, uint32_t dimensions, int k,
                                     bool normalized) {
        auto all = SearchBatch(embeddings, query, 1, n, dimensions, k, normalized ? Metric::Dot : Metric::Cosine);
        return all.empty() ? std::vector<SearchResult>{} : all[0];
    }
    // Q queries (row-major [Q x dimensions]) in one fused launch.
    std::vector<std::vector<SearchResult>> SearchBatch(Buffer &embeddings, const std::vector<float> &queries, uint32_t Q, uint32_t n,
                                                       uint32_t dimensions, int k, Metric metric) {
        if (k <= 0) return {};           // cuda_bridge.go:644-646
        if (k > (int)n) k = (int)n;      // cuda_bridge.go:647-649
        std::lock_guard<std::mutex> lk(mu_);
        if ((uint64_t)n * dimensions * 4 > embeddings.size_) throw ErrInvalidBuffer("cuda: invalid buffer");
        if (!embeddings.index_ || embeddings.index_n_ != n || embeddings.index_dim_ != dimensions || embeddings.index_metric_ != (int)metric) {
            if (embeddings.index_) nk_index_release(embeddings.index_);
            int dev = id_;
            embeddings.index_ = nk_index_create(&dev, 1, dimensions, NK_DTYPE_F32, (int)metric);
            // rows are final by the time they are searched (syncToCUDA = NewBuffer + NormalizeVectors, gpu.go:2073-2118):
            // refresh_shadow gives the attached (caller-owned) rows the fast BF16 filter path
            if (!embeddings.index_ || nk_index_attach_device_rows(embeddings.index_, cuda_buffer_data(embeddings.ptr_), n) != 0 ||
                nk_index_refresh_shadow(embeddings.index_) != 0)
                throw ErrKernelExecution(std::string("cuda: kernel execution failed: ") + nk_last_error());
            embeddings.index_n_ = n; embeddings.index_dim_ = dimensions; embeddings.index_metric_ = (int)metric;
        }
        std::vector<uint32_t> idx((size_t)Q * k);
        std::vector<float> sc((size_t)Q * k);
        int got = nk_search(embeddings.index_, queries.data(), Q, (uint32_t)k, idx.data(), sc.data());
        if (got < 0) throw ErrKernelExecution(std::string("cuda: kernel execution failed: ") + nk_last_error());
        std::vector<std::vector<SearchResult>> out(Q);
        for (uint32_t q = 0; q < Q; ++q)
            for (int i = 0; i < got; ++i) out[q].push_back({idx[(size_t)q * k + i], sc[(size_t)q * k + i]});
        return out;
    }

private:
    CudaDevice *ptr_ = nullptr;
    int id_;
    std::string name_;
    uint64_t memory_ = 0;
    int ccMajor_ = 0, ccMinor_ = 0;
    std::mutex mu_;
};

inline std::unique_ptr<Device> NewDevice(int deviceID) { return std::unique_ptr<Device>(new Device(deviceID)); }  // cuda_bridge.go:445

}  // namespace cuda

namespace gpu {

struct ErrInvalidDimensions : std::invalid_argument { ErrInvalidDimensions() : std::invalid_argument("gpu: invalid dimensions") {} };

struct SearchResult {  // gpu.go SearchResult{ID, Score, Distance}
    std::string ID;
    float Score;
    float Distance;
};

struct SimilarPair {  // one pair of a self-join: A is the node at the lower row
    std::string A, B;
    float Score;
};

// gpu.EmbeddingIndex (gpu.go:1224-2454) with the device corpus kept in step incrementally (no re-upload on Add/Remove,
// rows stay raw, cosine computed in-kernel).  Node-id strings live on the host only (gpu.go:1228-1231).
class EmbeddingIndex {
public:
    EmbeddingIndex(int dimensions, cuda::Metric metric = cuda::Metric::Cosine, std::vector<int> devices = {0}) : dims_(dimensions) {
        ix_ = nk_index_create(devices.data(), (int)devices.size(), (uint32_t)dimensions, NK_DTYPE_F32, (int)metric);
        if (!ix_) throw cuda::ErrDeviceCreation(std::string("gpu: ") + nk_last_error());
    }
    EmbeddingIndex(const EmbeddingIndex &) = delete;
    EmbeddingIndex &operator=(const EmbeddingIndex &) = delete;
    ~EmbeddingIndex() { Release(); }
    void Release() { if (ix_) { nk_index_release(ix_); ix_ = nullptr; } }

    void Add(const std::string &nodeID, const std::vector<float> &embedding) {  // gpu.go:1378-1403
        if ((int)embedding.size() != dims_) throw ErrInvalidDimensions();
        std::lock_guard<std::mutex> lk(mu_);
        gpuSynced_ = false;
        auto it = idToIndex_.find(nodeID);
        if (it != idToIndex_.end()) {
            check(nk_index_update_row(ix_, it->second, embedding.data()));
            if (graphK_) graphSrc_[it->second] = NK_ROW_NEW;  // contents SimilarGraph's graph never saw
            if (pairsOn_) pairsSrc_[it->second] = NK_ROW_NEW;  // ... nor SimilarPairs' join
        } else {
            check(nk_index_append(ix_, embedding.data(), 1));
            if (graphK_) graphSrc_.push_back(NK_ROW_NEW);
            if (pairsOn_) pairsSrc_.push_back(NK_ROW_NEW);
            tags_.push_back(0);    // nk_index_append: tag 0
            values_.push_back(0);  // ... and value key 0
            idToIndex_[nodeID] = nodeIDs_.size();
            nodeIDs_.push_back(nodeID);
        }
    }
    void AddBatch(const std::vector<std::string> &nodeIDs, const std::vector<std::vector<float>> &embeddings) {  // gpu.go:1406-1434
        if (nodeIDs.size() != embeddings.size()) throw std::invalid_argument("gpu: nodeIDs and embeddings length mismatch");
        for (size_t i = 0; i < nodeIDs.size(); ++i) Add(nodeIDs[i], embeddings[i]);
    }
    bool Remove(const std::string &nodeID) {  // gpu.go:1437-1471 (swap with last)
        std::lock_guard<std::mutex> lk(mu_);
        auto it = idToIndex_.find(nodeID);
        if (it == idToIndex_.end()) return false;
        const uint64_t idx = it->second, last = nodeIDs_.size() - 1;
        gpuSynced_ = false;
        check(nk_index_remove_swap(ix_, idx));
        if (graphK_) {  // the last row's contents move to idx, as on the device
            graphSrc_[idx] = graphSrc_[last];
            graphSrc_.pop_back();
        }
        if (pairsOn_) {
            pairsSrc_[idx] = pairsSrc_[last];
            pairsSrc_.pop_back();
        }
        tags_[idx] = tags_[last];  // the tag and the value key move with their row
        tags_.pop_back();
        values_[idx] = values_[last];
        values_.pop_back();
        if (idx != last) {
            nodeIDs_[idx] = nodeIDs_[last];
            idToIndex_[nodeIDs_[idx]] = idx;
        }
        nodeIDs_.pop_back();
        idToIndex_.erase(nodeID);
        return true;
    }
    std::vector<SearchResult> Search(const std::vector<float> &query, int k) {  // gpu.go:1532-1550
        if ((int)query.size() != dims_) throw ErrInvalidDimensions();
        auto r = SearchBatch(query, 1, k);
        return r.empty() ? std::vector<SearchResult>{} : r[0];
    }
    std::vector<std::vector<SearchResult>> SearchBatch(const std::vector<float> &queries, uint32_t Q, int k) {
        if (queries.size() != (size_t)Q * dims_) throw ErrInvalidDimensions();
        std::lock_guard<std::mutex> lk(mu_);
        if (nodeIDs_.empty() || k <= 0) return {};  // gpu.go:1540-1542
        std::vector<uint32_t> idx((size_t)Q * k);
        std::vector<float> sc((size_t)Q * k);
        int got = nk_search(ix_, queries.data(), Q, (uint32_t)k, idx.data(), sc.data());
        if (got < 0) throw cuda::ErrKernelExecution(std::string("gpu: ") + nk_last_error());
        std::vector<std::vector<SearchResult>> out(Q);
        for (uint32_t q = 0; q < Q; ++q)
            for (int i = 0; i < got; ++i) {
                uint32_t r = idx[(size_t)q * k + i];
                float s = sc[(size_t)q * k + i];
                if (r < nodeIDs_.size()) out[q].push_back({nodeIDs_[r], s, 1.0f - s});  // gpu.go:1679-1688
            }
        return out;
    }
    // Per-query tag filters: tag words of rows [firstRow, firstRow + tags.size()) (row order of Add; 0 = untagged), then a
    // batch whose queries each carry an NkFilter (Qdrant must / must_not / should over bit conditions) in one corpus pass.
    // A row whose tag changes is new contents to SimilarGraph's graph.
    void SetRowTags(uint64_t firstRow, const std::vector<uint64_t> &tags) {
        std::lock_guard<std::mutex> lk(mu_);
        check(nk_index_set_row_tags(ix_, firstRow, tags.data(), tags.size()));
        for (size_t i = 0; i < tags.size(); ++i) {
            if (graphK_ && tags_[firstRow + i] != tags[i]) graphSrc_[firstRow + i] = NK_ROW_NEW;
            if (pairsOn_ && tags_[firstRow + i] != tags[i]) pairsSrc_[firstRow + i] = NK_ROW_NEW;
            tags_[firstRow + i] = tags[i];
        }
    }
    std::vector<std::vector<SearchResult>> SearchBatchFiltered(const std::vector<float> &queries, const std::vector<NkFilter> &filters,
                                                               uint32_t Q, int k) {
        if (queries.size() != (size_t)Q * dims_) throw ErrInvalidDimensions();
        if (filters.size() != Q) throw std::invalid_argument("gpu: one filter per query");
        std::lock_guard<std::mutex> lk(mu_);
        if (nodeIDs_.empty() || k <= 0) return std::vector<std::vector<SearchResult>>(Q);
        std::vector<uint32_t> idx((size_t)Q * k);
        std::vector<float> sc((size_t)Q * k);
        int got = nk_search_filtered(ix_, queries.data(), filters.data(), Q, (uint32_t)k, idx.data(), sc.data());
        if (got < 0) throw cuda::ErrKernelExecution(std::string("gpu: ") + nk_last_error());
        std::vector<std::vector<SearchResult>> out(Q);
        for (uint32_t q = 0; q < Q; ++q)
            for (int i = 0; i < got; ++i) {
                uint32_t r = idx[(size_t)q * k + i];
                float s = sc[(size_t)q * k + i];
                if (r < nodeIDs_.size()) out[q].push_back({nodeIDs_[r], s, 1.0f - s});  // 0xffffffff: fewer admissible rows than k
            }
        return out;
    }
    // Per-query value windows: value keys of rows [firstRow, firstRow + keys.size()) (row order of Add; 0 = no value, keys
    // encoded by the caller so that key order is number order), then a batch whose queries each carry an NkWindow {lo, hi}
    // (inclusive, unsigned) on top of an optional tag filter (filters empty = none, else one per query), in one corpus pass.
    // A row whose value key changes is new contents to SimilarGraph's graph.
    void SetRowValues(uint64_t firstRow, const std::vector<uint64_t> &keys) {
        std::lock_guard<std::mutex> lk(mu_);
        check(nk_index_set_row_values(ix_, firstRow, keys.data(), keys.size()));
        for (size_t i = 0; i < keys.size(); ++i) {
            if (graphK_ && values_[firstRow + i] != keys[i]) graphSrc_[firstRow + i] = NK_ROW_NEW;
            if (pairsOn_ && values_[firstRow + i] != keys[i]) pairsSrc_[firstRow + i] = NK_ROW_NEW;
            values_[firstRow + i] = keys[i];
        }
    }
    std::vector<std::vector<SearchResult>> SearchBatchWindowed(const std::vector<float> &queries, const std::vector<NkFilter> &filters,
                                                               const std::vector<NkWindow> &windows, uint32_t Q, int k) {
        if (queries.size() != (size_t)Q * dims_) throw ErrInvalidDimensions();
        if (!filters.empty() && filters.size() != Q) throw std::invalid_argument("gpu: one filter per query");
        if (windows.size() != Q) throw std::invalid_argument("gpu: one window per query");
        std::lock_guard<std::mutex> lk(mu_);
        if (nodeIDs_.empty() || k <= 0) return std::vector<std::vector<SearchResult>>(Q);
        std::vector<uint32_t> idx((size_t)Q * k);
        std::vector<float> sc((size_t)Q * k);
        int got = nk_search_windowed(ix_, queries.data(), filters.empty() ? nullptr : filters.data(), windows.data(), Q, (uint32_t)k,
                                     idx.data(), sc.data());
        if (got < 0) throw cuda::ErrKernelExecution(std::string("gpu: ") + nk_last_error());
        std::vector<std::vector<SearchResult>> out(Q);
        for (uint32_t q = 0; q < Q; ++q)
            for (int i = 0; i < got; ++i) {
                uint32_t r = idx[(size_t)q * k + i];
                float s = sc[(size_t)q * k + i];
                if (r < nodeIDs_.size()) out[q].push_back({nodeIDs_[r], s, 1.0f - s});  // 0xffffffff: fewer admissible rows than k
            }
        return out;
    }
    // Every node whose similarity reaches the query's threshold (cosine / dot: minimum score; euclidean: maximum distance),
    // best first; filters empty = none, else one per query.  Sizes its buffers from the library's exact total.
    std::vector<std::vector<SearchResult>> SearchRange(const std::vector<float> &queries, const std::vector<float> &thresholds,
                                                       const std::vector<NkFilter> &filters, uint32_t Q) {
        return SearchRange(queries, thresholds, filters, {}, Q);
    }
    // ... with one value window per query on top (windows empty = none: the call above).
    std::vector<std::vector<SearchResult>> SearchRange(const std::vector<float> &queries, const std::vector<float> &thresholds,
                                                       const std::vector<NkFilter> &filters, const std::vector<NkWindow> &windows, uint32_t Q) {
        if (queries.size() != (size_t)Q * dims_) throw ErrInvalidDimensions();
        if (thresholds.size() != Q) throw std::invalid_argument("gpu: one threshold per query");
        if (!filters.empty() && filters.size() != Q) throw std::invalid_argument("gpu: one filter per query");
        if (!windows.empty() && windows.size() != Q) throw std::invalid_argument("gpu: one window per query");
        std::lock_guard<std::mutex> lk(mu_);
        std::vector<std::vector<SearchResult>> out(Q);
        if (nodeIDs_.empty() || Q == 0) return out;
        std::vector<uint64_t> off((size_t)Q + 1);
        std::vector<uint32_t> idx;
        std::vector<float> sc;
        uint64_t total = 0;
        for (int pass = 0; pass < 2; ++pass) {
            if (nk_search_range_windowed(ix_, queries.data(), thresholds.data(), filters.empty() ? nullptr : filters.data(),
                                         windows.empty() ? nullptr : windows.data(), Q, idx.size(), off.data(), idx.data(), sc.data(), &total) < 0)
                throw cuda::ErrKernelExecution(std::string("gpu: ") + nk_last_error());
            if (total <= idx.size()) break;
            idx.resize(total);
            sc.resize(total);
        }
        for (uint32_t q = 0; q < Q; ++q)
            for (uint64_t i = off[q]; i < off[q + 1]; ++i)
                if (idx[i] < nodeIDs_.size()) out[q].push_back({nodeIDs_[idx[i]], sc[i], 1.0f - sc[i]});
        return out;
    }
    // Every pair of stored nodes whose similarity reaches the threshold (cosine / dot: minimum score; euclidean: maximum
    // distance), each pair once, grouped by its lower row and best first within a group; filter = nullptr or one tag filter
    // both nodes must pass.  The join runs in stripes of at most stripeRows left rows, so the staging (8 B per pair) and the
    // cost of a call that outgrows its buffer stay bounded.  Sizes its buffers from the library's exact total.
    std::vector<SimilarPair> SearchPairs(float threshold, const NkFilter *filter = nullptr, uint64_t stripeRows = 1u << 16) {
        return SearchPairs(threshold, filter, nullptr, NK_NO_GAP, stripeRows);
    }
    // ... with value conditions on both nodes: window = nullptr or one NkWindow both value keys must lie in; maxGap = a band,
    // |key(A) - key(B)| <= maxGap with both keys set (NK_NO_GAP: none), e.g. near-duplicates within the same hour.
    std::vector<SimilarPair> SearchPairs(float threshold, const NkFilter *filter, const NkWindow *window, uint64_t maxGap,
                                         uint64_t stripeRows = 1u << 16) {
        std::lock_guard<std::mutex> lk(mu_);
        std::vector<SimilarPair> out;
        const uint64_t n = nk_index_rows(ix_);
        if (stripeRows == 0) stripeRows = 1;
        std::vector<uint32_t> idx;
        std::vector<float> sc;
        for (uint64_t first = 0; first < n; first += stripeRows) {
            const uint64_t rows = std::min<uint64_t>(stripeRows, n - first);
            std::vector<uint64_t> off(rows + 1);
            uint64_t total = 0;
            for (int pass = 0; pass < 2; ++pass) {
                if (nk_search_pairs_windowed(ix_, first, rows, threshold, filter, window, maxGap, idx.size(), off.data(), idx.data(), sc.data(),
                                             &total) < 0)
                    throw cuda::ErrKernelExecution(std::string("gpu: ") + nk_last_error());
                if (total <= idx.size()) break;
                idx.resize(total);
                sc.resize(total);
            }
            for (uint64_t r = 0; r < rows; ++r)
                for (uint64_t i = off[r]; i < off[r + 1]; ++i)
                    if (first + r < nodeIDs_.size() && idx[i] < nodeIDs_.size()) out.push_back({nodeIDs_[first + r], nodeIDs_[idx[i]], sc[i]});
        }
        return out;
    }
    // The k most similar OTHER nodes of each stored node (FindSimilar, GraphQL similar, OnStore's related nodes), best first,
    // searched with the node's embedding as stored.  One list per id; an id the index does not hold gets an empty list
    // (missing ids are ignored, as in ScoreSubset).  filters empty = none, else one tag filter per id (e.g. "same collection"):
    // each list then holds only nodes its filter admits.
    std::vector<std::vector<SearchResult>> SearchSimilar(const std::vector<std::string> &ids, int k, const std::vector<NkFilter> &filters = {}) {
        return SearchSimilar(ids, k, filters, {});
    }
    // ... with one value window per id on top (windows empty = none: the call above), e.g. "nodes like this one from the last
    // 7 days": each list then holds only nodes whose value key the id's window admits.
    std::vector<std::vector<SearchResult>> SearchSimilar(const std::vector<std::string> &ids, int k, const std::vector<NkFilter> &filters,
                                                         const std::vector<NkWindow> &windows) {
        if (!filters.empty() && filters.size() != ids.size()) throw std::invalid_argument("gpu: one filter per id");
        if (!windows.empty() && windows.size() != ids.size()) throw std::invalid_argument("gpu: one window per id");
        std::lock_guard<std::mutex> lk(mu_);
        std::vector<std::vector<SearchResult>> out(ids.size());
        std::vector<uint32_t> rows;
        std::vector<NkFilter> f;
        std::vector<NkWindow> w;
        std::vector<size_t> at;
        for (size_t i = 0; i < ids.size(); ++i) {
            auto it = idToIndex_.find(ids[i]);
            if (it != idToIndex_.end()) {
                rows.push_back((uint32_t)it->second);
                at.push_back(i);
                if (!filters.empty()) f.push_back(filters[i]);
                if (!windows.empty()) w.push_back(windows[i]);
            }
        }
        if (rows.empty() || k <= 0) return out;
        std::vector<uint32_t> idx(rows.size() * (size_t)k);
        std::vector<float> sc(rows.size() * (size_t)k);
        int got = nk_search_rows_windowed(ix_, rows.data(), f.empty() ? nullptr : f.data(), w.empty() ? nullptr : w.data(), (uint32_t)rows.size(),
                                          (uint32_t)k, idx.data(), sc.data());
        if (got < 0) throw cuda::ErrKernelExecution(std::string("gpu: ") + nk_last_error());
        for (size_t j = 0; j < rows.size(); ++j)
            for (int i = 0; i < got; ++i) {
                uint32_t r = idx[j * k + i];
                float s = sc[j * k + i];
                if (r < nodeIDs_.size()) out[at[j]].push_back({nodeIDs_[r], s, 1.0f - s});  // 0xffffffff: fewer other nodes than k
            }
        return out;
    }
    // The k-NN graph of every node (SearchSimilar over all ids), kept current across Add / AddBatch / Remove: the index keeps,
    // for each row, which row of the last graph its contents came from (swapped by Remove as the device swaps rows), and the
    // next call hands that map to nk_knn_graph_remap instead of rebuilding.  The first call, a new k, or a Deserialize since
    // the last call rebuild it with nk_search_rows.  Lists in row order (the order of insertion, as swapped by Remove).  The
    // graph is built and updated on the 16-bit filter path (the TF32 filter if the shape has no 16-bit image), which the
    // update requires; other searches keep the automatic choice.  filters empty = none, else one tag filter per row (row
    // order): each node's list holds only nodes its filter admits, e.g. one graph per collection of the shared index.  windows
    // empty = none, else one value window per row (row order): each node's list holds only nodes whose value key (SetRowValues)
    // its window admits, a time-local graph.  A node whose filter, window, tag (SetRowTags) or value key (SetRowValues) changed
    // since the last call is handed to the update as new contents.
    std::vector<std::vector<SearchResult>> SimilarGraph(int k, const std::vector<NkFilter> &filters = {}, const std::vector<NkWindow> &windows = {}) {
        std::lock_guard<std::mutex> lk(mu_);
        const uint64_t n = nodeIDs_.size();
        if (!filters.empty() && filters.size() != n) throw std::invalid_argument("gpu: one filter per node");
        if (!windows.empty() && windows.size() != n) throw std::invalid_argument("gpu: one window per node");
        if (n == 0 || k <= 0) return std::vector<std::vector<SearchResult>>(n);
        auto filter_of = [&](uint64_t r) { return filters.empty() ? NkFilter{0, 0, 0} : filters[r]; };
        auto same_filter = [](const NkFilter &a, const NkFilter &b) { return a.all_of == b.all_of && a.none_of == b.none_of && a.any_of == b.any_of; };
        auto window_of = [&](uint64_t r) { return windows.empty() ? NkWindow{0, ~0ull} : windows[r]; };  // none: every key
        auto same_window = [](const NkWindow &a, const NkWindow &b) { return a.lo == b.lo && a.hi == b.hi; };
        const NkFilter *fp = filters.empty() ? nullptr : filters.data();
        const NkWindow *wp = windows.empty() ? nullptr : windows.data();
        int got = -1;
        std::vector<uint32_t> gi(n * k, 0xffffffffu);
        std::vector<float> gs(n * k, 0.0f);
        std::vector<uint32_t> src;  // graphSrc_ with the rows whose filter or window changed as new contents
        if (graphK_ == (uint32_t)k) {
            src = graphSrc_;
            for (uint64_t f = 0; f < n; ++f)
                if (src[f] != NK_ROW_NEW && (!same_filter(filter_of(f), graphFilter_[src[f]]) || !same_window(window_of(f), graphWindow_[src[f]])))
                    src[f] = NK_ROW_NEW;
        }
        for (int path : {NK_PATH_TENSOR_SHADOW, NK_PATH_TENSOR_FILTER}) {
            check(nk_index_set_path(ix_, path));
            if (graphK_ == (uint32_t)k) {
                got = nk_knn_graph_remap_windowed(ix_, (uint32_t)k, graphRows_, src.data(), fp, wp, graphIdx_.data(), graphScore_.data(), gi.data(),
                                                  gs.data(), nullptr);
            } else {
                std::vector<uint32_t> rows(n);
                for (uint64_t r = 0; r < n; ++r) rows[r] = (uint32_t)r;
                got = nk_search_rows_windowed(ix_, rows.data(), fp, wp, (uint32_t)n, (uint32_t)k, gi.data(), gs.data());
                if (got >= 0) ++graphRebuilds_;
            }
            if (got >= 0) break;
        }
        check(nk_index_set_path(ix_, NK_PATH_AUTO));
        if (got < 0) { graphK_ = 0; throw cuda::ErrKernelExecution(std::string("gpu: ") + nk_last_error()); }
        graphK_ = (uint32_t)k;
        graphRows_ = n;
        graphIdx_.swap(gi);
        graphScore_.swap(gs);
        graphSrc_.resize(n);
        graphFilter_.resize(n);
        graphWindow_.resize(n);
        for (uint64_t r = 0; r < n; ++r) { graphSrc_[r] = (uint32_t)r; graphFilter_[r] = filter_of(r); graphWindow_[r] = window_of(r); }
        std::vector<std::vector<SearchResult>> out(n);
        for (uint64_t r = 0; r < n; ++r)
            for (int i = 0; i < got; ++i) {
                const uint32_t j = graphIdx_[r * k + i];
                const float s = graphScore_[r * k + i];
                if (j < n) out[r].push_back({nodeIDs_[j], s, 1.0f - s});  // 0xffffffff: fewer other nodes than k
            }
        return out;
    }
    // Auto-link on write: every pair of the whole-index join (SearchPairs with the same threshold, filter, window and maxGap)
    // that has an end among `ids`, each as {listed node, other node, score}, grouped by the listed node in the order of `ids`
    // (a pair with both ends listed once, under the node with the lower row), best first within a group.  Missing and repeated
    // ids are ignored.  Scores are the join's (nk_search_pairs_rows_windowed), on the filter path SimilarGraph uses.
    std::vector<SimilarPair> PairsOfNodes(const std::vector<std::string> &ids, float threshold, const NkFilter *filter = nullptr,
                                          const NkWindow *window = nullptr, uint64_t maxGap = NK_NO_GAP) {
        std::lock_guard<std::mutex> lk(mu_);
        std::vector<uint32_t> rows;
        std::unordered_map<uint64_t, bool> seen;
        for (auto &id : ids) {
            auto it = idToIndex_.find(id);
            if (it != idToIndex_.end() && !seen[it->second]) { seen[it->second] = true; rows.push_back((uint32_t)it->second); }
        }
        std::vector<SimilarPair> out;
        if (rows.empty()) return out;
        std::vector<uint64_t> off(rows.size() + 1);
        std::vector<uint32_t> idx;
        std::vector<float> sc;
        on_graph_path([&] {
            uint64_t total = 0;
            for (int pass = 0; pass < 2; ++pass) {
                if (nk_search_pairs_rows_windowed(ix_, rows.data(), (uint32_t)rows.size(), threshold, filter, window, maxGap, idx.size(), off.data(),
                                                  idx.data(), sc.data(), &total) < 0)
                    return -1;
                if (total <= idx.size()) break;
                idx.resize(total);
                sc.resize(total);
            }
            return 0;
        });
        for (size_t r = 0; r < rows.size(); ++r)
            for (uint64_t i = off[r]; i < off[r + 1]; ++i)
                if (idx[i] < nodeIDs_.size()) out.push_back({nodeIDs_[rows[r]], nodeIDs_[idx[i]], sc[i]});
        return out;
    }
    // The whole-index join (SearchPairs with the same arguments, in the same order) kept current across Add / AddBatch /
    // Remove / SetRowTags / SetRowValues, as SimilarGraph keeps its graph: the index follows which row of the last join each
    // row's contents came from (a rewritten, retagged or re-valued row is new contents), and the next call hands that map to
    // nk_pairs_remap instead of joining again.  The first call, a new threshold, filter, window or maxGap, or a Deserialize
    // since the last call rebuild the join in stripes of stripeRows left rows, as SearchPairs does.  Runs on the filter path
    // SimilarGraph uses, which the remap requires.  The join is held in host memory, 8 B per pair.
    std::vector<SimilarPair> SimilarPairs(float threshold, const NkFilter *filter = nullptr, const NkWindow *window = nullptr,
                                          uint64_t maxGap = NK_NO_GAP, uint64_t stripeRows = 1u << 16) {
        std::lock_guard<std::mutex> lk(mu_);
        const uint64_t n = nodeIDs_.size();
        const NkFilter f = filter ? *filter : NkFilter{0, 0, 0};
        const NkWindow w = window ? *window : NkWindow{0, ~0ull};
        const bool same = pairsOn_ && std::memcmp(&pairsT_, &threshold, 4) == 0 && pairsHasF_ == (filter != nullptr) &&
                          pairsF_.all_of == f.all_of && pairsF_.none_of == f.none_of && pairsF_.any_of == f.any_of &&
                          pairsHasW_ == (window != nullptr) && pairsW_.lo == w.lo && pairsW_.hi == w.hi && pairsGap_ == maxGap;
        std::vector<uint64_t> off(n + 1, 0);
        std::vector<uint32_t> idx;
        std::vector<float> sc;
        if (stripeRows == 0) stripeRows = 1;
        on_graph_path([&] {
            uint64_t total = 0;
            if (same) {
                for (int pass = 0; pass < 2; ++pass) {
                    if (nk_pairs_remap(ix_, threshold, filter, window, maxGap, pairsRows_, pairsSrc_.data(), pairsOff_.data(), pairsIdx_.data(),
                                       pairsScore_.data(), idx.size(), off.data(), idx.data(), sc.data(), &total, nullptr, nullptr) < 0)
                        return -1;
                    if (total <= idx.size()) return 0;
                    idx.resize(total);
                    sc.resize(total);
                }
                return 0;
            }
            idx.clear();
            sc.clear();
            std::vector<uint32_t> si;
            std::vector<float> ss;
            for (uint64_t first = 0; first < n; first += stripeRows) {  // stripes of the whole join, concatenated
                const uint64_t rows = std::min<uint64_t>(stripeRows, n - first);
                std::vector<uint64_t> so(rows + 1);
                for (int pass = 0; pass < 2; ++pass) {
                    if (nk_search_pairs_windowed(ix_, first, rows, threshold, filter, window, maxGap, si.size(), so.data(), si.data(), ss.data(),
                                                 &total) < 0)
                        return -1;
                    if (total <= si.size()) break;
                    si.resize(total);
                    ss.resize(total);
                }
                for (uint64_t r = 0; r < rows; ++r) off[first + r + 1] = off[first] + so[r + 1];
                idx.insert(idx.end(), si.begin(), si.begin() + total);
                sc.insert(sc.end(), ss.begin(), ss.begin() + total);
            }
            ++pairsRebuilds_;
            return 0;
        });
        idx.resize(off[n]);
        sc.resize(off[n]);
        pairsOn_ = true;
        pairsT_ = threshold;
        pairsHasF_ = filter != nullptr;
        pairsF_ = f;
        pairsHasW_ = window != nullptr;
        pairsW_ = w;
        pairsGap_ = maxGap;
        pairsRows_ = n;
        pairsOff_.swap(off);
        pairsIdx_.swap(idx);
        pairsScore_.swap(sc);
        pairsSrc_.resize(n);
        for (uint64_t r = 0; r < n; ++r) pairsSrc_[r] = (uint32_t)r;
        std::vector<SimilarPair> out;
        out.reserve(pairsIdx_.size());
        for (uint64_t r = 0; r < n; ++r)
            for (uint64_t i = pairsOff_[r]; i < pairsOff_[r + 1]; ++i)
                if (pairsIdx_[i] < n) out.push_back({nodeIDs_[r], nodeIDs_[pairsIdx_[i]], pairsScore_[i]});
        return out;
    }
    uint64_t PairsRebuilds() const { return pairsRebuilds_; }  // SimilarPairs calls that joined every row
    std::vector<SearchResult> ScoreSubset(const std::vector<float> &query, const std::vector<std::string> &ids) {  // gpu.go:1552-1616
        if ((int)query.size() != dims_) throw ErrInvalidDimensions();
        std::lock_guard<std::mutex> lk(mu_);
        std::vector<uint32_t> rows;
        for (auto &id : ids) {
            auto it = idToIndex_.find(id);
            if (it != idToIndex_.end()) rows.push_back((uint32_t)it->second);  // missing ids are ignored
        }
        if (rows.empty()) return {};
        std::vector<uint32_t> idx(rows.size());
        std::vector<float> sc(rows.size());
        int got = nk_score_subset(ix_, query.data(), rows.data(), (uint32_t)rows.size(), (uint32_t)rows.size(), idx.data(), sc.data());
        if (got < 0) throw cuda::ErrKernelExecution(std::string("gpu: ") + nk_last_error());
        std::vector<SearchResult> out;
        for (int i = 0; i < got; ++i) out.push_back({nodeIDs_[idx[i]], sc[i], 1.0f - sc[i]});
        return out;
    }
    // gpu.go:2025: nothing to copy (the device rows are always current); the observable flag of gpu_test.go:1403-1480 is
    // kept: false after Add / Remove / Deserialize, true after SyncToGPU
    void SyncToGPU() { std::lock_guard<std::mutex> lk(mu_); gpuSynced_ = true; }
    bool IsGPUSynced() const { return gpuSynced_; }
    uint64_t GraphRebuilds() const { return graphRebuilds_; }  // SimilarGraph calls that searched every row
    std::vector<uint64_t> RowTags() { std::lock_guard<std::mutex> lk(mu_); return tags_; }  // the tag of each row, row order
    std::vector<uint64_t> RowValues() { std::lock_guard<std::mutex> lk(mu_); return values_; }  // the value key of each row, row order
    int Count() const { return (int)nodeIDs_.size(); }                                   // gpu.go:2225
    bool Has(const std::string &id) const { return idToIndex_.count(id) != 0; }          // gpu.go:2279
    bool Get(const std::string &id, std::vector<float> *out) {                           // gpu.go:2287
        std::lock_guard<std::mutex> lk(mu_);
        auto it = idToIndex_.find(id);
        if (it == idToIndex_.end()) return false;
        out->resize(dims_);
        check(nk_index_read_rows(ix_, it->second, 1, out->data()));
        return true;
    }
    // gpu.go:2373-2411: LE [dims u32][count u32][len-prefixed ids...][float32 vectors...]
    std::vector<uint8_t> Serialize() {
        std::lock_guard<std::mutex> lk(mu_);
        std::vector<uint8_t> buf;
        auto put32 = [&buf](uint32_t v) { for (int i = 0; i < 4; ++i) buf.push_back((uint8_t)(v >> (8 * i))); };
        put32((uint32_t)dims_);
        put32((uint32_t)nodeIDs_.size());
        for (auto &id : nodeIDs_) { put32((uint32_t)id.size()); buf.insert(buf.end(), id.begin(), id.end()); }
        size_t off = buf.size(), n = nodeIDs_.size();
        buf.resize(off + n * dims_ * 4);
        if (n) check(nk_index_read_rows(ix_, 0, n, buf.data() + off));
        return buf;
    }
    void Deserialize(const std::vector<uint8_t> &data) {  // gpu.go:2414-2454
        if (data.size() < 8) throw std::invalid_argument("gpu: invalid serialized data");
        auto get32 = [&data](size_t o) { return (uint32_t)data[o] | (uint32_t)data[o + 1] << 8 | (uint32_t)data[o + 2] << 16 | (uint32_t)data[o + 3] << 24; };
        uint32_t dims = get32(0), count = get32(4);
        if ((int)dims != dims_) throw ErrInvalidDimensions();
        size_t off = 8;
        std::vector<std::string> ids(count);
        for (uint32_t i = 0; i < count; ++i) {
            uint32_t len = get32(off);
            off += 4;
            ids[i].assign((const char *)&data[off], len);
            off += len;
        }
        std::lock_guard<std::mutex> lk(mu_);
        check(nk_index_upload(ix_, data.data() + off, count));  // the blob streams straight into device memory
        gpuSynced_ = false;
        graphK_ = 0;
        pairsOn_ = false;
        tags_.assign(count, 0);    // nk_index_upload: every tag 0
        values_.assign(count, 0);  // ... and every value key 0
        nodeIDs_ = ids;
        idToIndex_.clear();
        for (uint32_t i = 0; i < count; ++i) idToIndex_[nodeIDs_[i]] = i;
    }

private:
    void check(int rc) { if (rc != 0) throw cuda::ErrKernelExecution(std::string("gpu: ") + nk_last_error()); }
    // Run call() on the 16-bit filter path, or the TF32 filter if the shape has no 16-bit image (SimilarGraph's choice), then
    // go back to AUTO; throw if neither serves it.
    template <class F> void on_graph_path(F call) {
        int rc = -1;
        for (int path : {NK_PATH_TENSOR_SHADOW, NK_PATH_TENSOR_FILTER}) {
            check(nk_index_set_path(ix_, path));
            if ((rc = call()) >= 0) break;
        }
        check(nk_index_set_path(ix_, NK_PATH_AUTO));
        if (rc < 0) throw cuda::ErrKernelExecution(std::string("gpu: ") + nk_last_error());
    }
    int dims_;
    NkIndex *ix_ = nullptr;
    std::vector<std::string> nodeIDs_;
    std::unordered_map<std::string, uint64_t> idToIndex_;
    bool gpuSynced_ = false;
    // SimilarGraph: the graph of rows [0, graphRows_) for k = graphK_ (0: none), and for each current row the graph row its
    // contents came from (NK_ROW_NEW: appended or rewritten since); how many times the graph was built from scratch
    uint32_t graphK_ = 0;
    uint64_t graphRows_ = 0;
    std::vector<uint32_t> graphIdx_;
    std::vector<float> graphScore_;
    std::vector<uint32_t> graphSrc_;
    std::vector<NkFilter> graphFilter_;  // the filter of each graph row's list when it was made ({0,0,0}: none)
    std::vector<NkWindow> graphWindow_;  // ... and its window ({0, ~0}: none)
    std::vector<uint64_t> tags_;         // the tag of each row, as on the device
    std::vector<uint64_t> values_;       // the value key of each row, as on the device
    uint64_t graphRebuilds_ = 0;
    // SimilarPairs: the join of rows [0, pairsRows_) (CSR) with its arguments (pairsOn_ = false: none), and for each current row
    // the join row its contents came from (NK_ROW_NEW: appended, rewritten, retagged or re-valued since)
    bool pairsOn_ = false;
    float pairsT_ = 0.0f;
    bool pairsHasF_ = false, pairsHasW_ = false;
    NkFilter pairsF_{0, 0, 0};
    NkWindow pairsW_{0, ~0ull};
    uint64_t pairsGap_ = NK_NO_GAP;
    uint64_t pairsRows_ = 0;
    std::vector<uint64_t> pairsOff_;
    std::vector<uint32_t> pairsIdx_;
    std::vector<float> pairsScore_;
    std::vector<uint32_t> pairsSrc_;
    uint64_t pairsRebuilds_ = 0;
    std::mutex mu_;
};

}  // namespace gpu
}  // namespace nornic
