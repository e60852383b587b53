// legacy_abi.cu — the C symbols of the cgo preamble of pkg/gpu/cuda/cuda_bridge.go:20-375, re-implemented
// on this library's kernels (no cuBLAS).  Signatures, return conventions and ownership are the
// reference's; the differences are all fixes of defects listed in SURVEY.md §3.1:
//   * every call binds its device (the reference only does so in cuda_create_device);
//   * the error message is thread-local;
//   * cuda_compute_norms / cuda_normalize_vectors are one kernel each instead of 2n cuBLAS calls;
//   * cuda_cosine_similarity honours `normalized`;
//   * cuda_topk selects on the device (k pairs cross PCIe, not n scores).
#include <mutex>
#include <stdlib.h>
#include <string.h>

#include "kernels.cuh"

struct CudaDevice {
    int device_id;
    cudaStream_t stream;
    nk::DeviceInfo info;
    nk::Workspace ws;
    std::mutex mu;
};

extern "C" {

void cuda_set_error(const char *msg) { nk::set_error("%s", msg ? msg : ""); }
const char *cuda_get_last_error(void) { return nk::get_error(); }
void cuda_clear_error(void) { nk::clear_error(); }

int cuda_get_device_count(void) {
    int count = 0;
    cudaError_t err = cudaGetDeviceCount(&count);
    if (err != cudaSuccess) {
        nk::set_error("%s", cudaGetErrorString(err));
        cudaGetLastError();
        return -1;
    }
    return count;
}

int cuda_is_available(void) { return cuda_get_device_count() > 0 ? 1 : 0; }

CudaDevice *cuda_create_device(int device_id) {
    nk::DeviceGuard _restore_device;
    NK_CUDA_OK_PTR(cudaSetDevice(device_id));
    CudaDevice *dev = new (std::nothrow) CudaDevice();
    if (!dev) {
        nk::set_error("Failed to allocate device struct");
        return nullptr;
    }
    dev->device_id = device_id;
    if (nk::query_device_info(device_id, &dev->info) != 0) {
        delete dev;
        return nullptr;
    }
    cudaError_t err = cudaStreamCreateWithFlags(&dev->stream, cudaStreamNonBlocking);
    if (err == cudaSuccess) err = cudaMalloc((void **)&dev->ws.flags, sizeof(int) * 8);
    if (err == cudaSuccess) err = cudaMemset(dev->ws.flags, 0, sizeof(int) * 8);
    if (err != cudaSuccess) {
        nk::set_error("%s", cudaGetErrorString(err));
        delete dev;
        return nullptr;
    }
    return dev;
}

void cuda_release_device(CudaDevice *dev) {
    nk::DeviceGuard _restore_device;
    if (!dev) return;
    cudaSetDevice(dev->device_id);
    if (dev->stream) {
        cudaStreamSynchronize(dev->stream);
        cudaStreamDestroy(dev->stream);
    }
    dev->ws.release();
    delete dev;
}

const char *cuda_device_name(int device_id) {
    static thread_local char name[256];
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device_id) != cudaSuccess) {
        cudaGetLastError();
        return "Unknown";
    }
    strncpy(name, prop.name, sizeof(name) - 1);
    name[sizeof(name) - 1] = 0;
    return name;
}

size_t cuda_device_memory(int device_id) {
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device_id) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return prop.totalGlobalMem;
}

int cuda_device_compute_capability(int device_id) {
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device_id) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return prop.major * 10 + prop.minor;
}

CudaBuffer *cuda_create_buffer(CudaDevice *dev, float *host_data, size_t count, int memory_type) {
    nk::DeviceGuard _restore_device;
    if (dev) NK_CUDA_OK_PTR(cudaSetDevice(dev->device_id));
    CudaBuffer *buf = (CudaBuffer *)malloc(sizeof(CudaBuffer));
    if (!buf) {
        nk::set_error("Failed to allocate buffer struct");
        return nullptr;
    }
    buf->data = nullptr;
    buf->size = count * sizeof(float);
    buf->memory_type = memory_type;
    cudaError_t err;
    if (memory_type == 0) {
        err = cudaMalloc((void **)&buf->data, buf->size ? buf->size : 4);
        if (err == cudaSuccess && host_data && buf->size)
            err = cudaMemcpy(buf->data, host_data, buf->size, cudaMemcpyHostToDevice);
        // a pageable cudaMemcpy may return before its DMA has landed, and the calls below run on the device's non-blocking
        // stream, which does not wait for the legacy stream: finish the copy here, as the header promises
        if (err == cudaSuccess && host_data && buf->size) err = cudaStreamSynchronize(cudaStreamLegacy);
        if (err != cudaSuccess) {
            nk::set_error("%s", cudaGetErrorString(err));
            cudaGetLastError();
            if (buf->data) cudaFree(buf->data);
            free(buf);
            return nullptr;
        }
    } else {
        err = cudaMallocHost((void **)&buf->data, buf->size ? buf->size : 4);
        if (err != cudaSuccess) {
            nk::set_error("%s", cudaGetErrorString(err));
            cudaGetLastError();
            free(buf);
            return nullptr;
        }
        if (host_data && buf->size) memcpy(buf->data, host_data, buf->size);
    }
    return buf;
}

void cuda_release_buffer(CudaBuffer *buf) {
    nk::DeviceGuard _restore_device;
    if (!buf) return;
    if (buf->data) {
        if (buf->memory_type == 0) cudaFree(buf->data);
        else cudaFreeHost(buf->data);
    }
    free(buf);
}

void *cuda_buffer_data(CudaBuffer *buf) { return buf ? buf->data : nullptr; }
size_t cuda_buffer_size(CudaBuffer *buf) { return buf ? buf->size : 0; }

int cuda_buffer_copy_to_host(CudaBuffer *buf, float *host_data, size_t count) {
    nk::DeviceGuard _restore_device;
    if (!buf || !host_data) return -1;
    size_t copy_size = count * sizeof(float);
    if (copy_size > buf->size) copy_size = buf->size;
    if (copy_size == 0) return 0;
    if (buf->memory_type == 0) {
        cudaError_t err = cudaMemcpy(host_data, buf->data, copy_size, cudaMemcpyDeviceToHost);
        if (err != cudaSuccess) {
            nk::set_error("%s", cudaGetErrorString(err));
            cudaGetLastError();
            return -1;
        }
    } else {
        memcpy(host_data, buf->data, copy_size);
    }
    return 0;
}

static int check_buf(const CudaBuffer *b, size_t floats, const char *what) {
    if (!b || !b->data) {
        nk::set_error("invalid %s buffer", what);
        return -1;
    }
    if (b->size < floats * sizeof(float)) {
        nk::set_error("%s buffer too small: %zu bytes < %zu", what, b->size, floats * sizeof(float));
        return -1;
    }
    return 0;
}

int cuda_compute_norms(CudaDevice *dev, CudaBuffer *vectors, CudaBuffer *norms, unsigned int n, unsigned int dims) {
    nk::DeviceGuard _restore_device;
    if (!dev) { nk::set_error("invalid device"); return -1; }
    if (check_buf(vectors, (size_t)n * dims, "vectors") || check_buf(norms, n, "norms")) return -1;
    std::lock_guard<std::mutex> lk(dev->mu);
    NK_CUDA_OK(cudaSetDevice(dev->device_id));
    if (nk::row_norms(vectors->data, norms->data, n, dims, dev->stream)) return -1;
    NK_CUDA_OK(cudaStreamSynchronize(dev->stream));
    return 0;
}

int cuda_normalize_vectors(CudaDevice *dev, CudaBuffer *vectors, unsigned int n, unsigned int dims) {
    nk::DeviceGuard _restore_device;
    if (!dev) { nk::set_error("invalid device"); return -1; }
    if (check_buf(vectors, (size_t)n * dims, "vectors")) return -1;
    std::lock_guard<std::mutex> lk(dev->mu);
    NK_CUDA_OK(cudaSetDevice(dev->device_id));
    if (nk::normalize_rows(vectors->data, n, dims, dev->stream)) return -1;
    NK_CUDA_OK(cudaStreamSynchronize(dev->stream));
    return 0;
}

int cuda_cosine_similarity(CudaDevice *dev, CudaBuffer *embeddings, CudaBuffer *query, CudaBuffer *scores,
                           unsigned int n, unsigned int dims, int normalized) {
    nk::DeviceGuard _restore_device;
    if (!dev) { nk::set_error("invalid device"); return -1; }
    if (check_buf(embeddings, (size_t)n * dims, "embeddings") || check_buf(query, dims, "query") ||
        check_buf(scores, n, "scores"))
        return -1;
    std::lock_guard<std::mutex> lk(dev->mu);
    NK_CUDA_OK(cudaSetDevice(dev->device_id));
    if (nk::row_scores(embeddings->data, query->data, scores->data, n, dims, normalized, dev->stream)) return -1;
    NK_CUDA_OK(cudaStreamSynchronize(dev->stream));
    return 0;
}

int cuda_topk(CudaDevice *dev, CudaBuffer *scores, unsigned int *out_indices, float *out_scores, unsigned int n,
              unsigned int k) {
    nk::DeviceGuard _restore_device;
    if (k == 0 || n == 0) return 0;  // cuda_bridge.go:329-331
    if (k > n) k = n;                // cuda_bridge.go:332-334
    if (!dev) { nk::set_error("invalid device"); return -1; }
    if (check_buf(scores, n, "scores")) return -1;
    if (!out_indices || !out_scores) { nk::set_error("null output"); return -1; }
    std::lock_guard<std::mutex> lk(dev->mu);
    NK_CUDA_OK(cudaSetDevice(dev->device_id));
    nk::Workspace &ws = dev->ws;
    if (k > NK_MAX_K_TOTAL) { nk::set_error("k=%u exceeds NK_MAX_K_TOTAL=%u", k, NK_MAX_K_TOTAL); return -1; }
    if (nk::ws_reserve((void **)&ws.keys, &ws.keys_bytes, (size_t)k * 8)) return -1;
    if (nk::ws_reserve((void **)&ws.out_idx, &ws.out_idx_bytes, (size_t)k * 4)) return -1;
    if (nk::ws_reserve((void **)&ws.out_score, &ws.out_score_bytes, (size_t)k * 4)) return -1;
    if (k <= NK_MAX_K) {
        if (nk::topk_scores(dev->info, scores->data, n, k, ws, ws.keys, dev->stream)) return -1;
    } else {
        // any k (cuda_bridge.go:327-375): passes of NK_MAX_K, each bounded above by the previous pass's last key
        if (nk::ws_reserve((void **)&ws.below, &ws.below_bytes, 8)) return -1;
        NK_CUDA_OK(cudaMemsetAsync(ws.below, 0xff, 8, dev->stream));
        for (unsigned int done = 0; done < k;) {
            const unsigned int kp = k - done < NK_MAX_K ? k - done : NK_MAX_K;
            if (nk::topk_scores(dev->info, scores->data, n, kp, ws, ws.keys + done, dev->stream, ws.below)) return -1;
            if (nk::update_below(ws.keys + done, 1, kp, ws.below, dev->stream)) return -1;
            done += kp;
        }
    }
    if (nk::decode_topk_scores(ws.keys, k, scores->data, ws.out_idx, ws.out_score, dev->stream)) return -1;
    NK_CUDA_OK(cudaMemcpyAsync(out_indices, ws.out_idx, (size_t)k * 4, cudaMemcpyDeviceToHost, dev->stream));
    NK_CUDA_OK(cudaMemcpyAsync(out_scores, ws.out_score, (size_t)k * 4, cudaMemcpyDeviceToHost, dev->stream));
    NK_CUDA_OK(cudaStreamSynchronize(dev->stream));
    return 0;
}

}  // extern "C"
