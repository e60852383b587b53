// exchange.cu — the one exchange step of the row-sharded search (SURVEY.md §8e), behind the C ABI and over NVLink peer
// memory instead of a library collective.
//
// The reference has a single DeviceID (pkg/gpu/gpu.go:218); a multi-GPU host runs one rank (process, or in-process index)
// per GPU, each scanning its row range.  What has to cross GPUs is tiny — Q*k packed 64-bit keys per rank (5 KB at Q=64,
// k=10) — so the cost of the step is latency, not bandwidth: an NCCL all-gather through a framework costs 20-30 us per
// search, about as much as everything else around the scan.  Here every rank owns a small device buffer
//     [2 parities][world slots][slot_bytes]  +  arrival words [2][world]
// exported through CUDA IPC (nk_comm_export / nk_comm_connect; ranks of one process connect with plain pointers).  A search:
//   1. scan + finish produce this shard's sorted key list (the usual kernels);
//   2. exchange_push_kernel: CTA p stores the list into slot[rank] of PEER p's buffer with plain P2P stores over
//      NVLink / NVSwitch, then publishes the search's epoch in p's arrival word (system-scope release);
//   3. merge_keys_kernel (merge.cu) with its fused wait: polls the local arrival words (system-scope acquire, bounded by a
//      wall-clock timeout), merges the world lists with the same (score desc, row asc) rule and writes the decoded result.
// Two launches, no host involvement, no NCCL.  Parity double-buffering makes the slots reusable without a barrier: a rank
// can only push epoch e+2 after it has merged e+1, which needed every peer's push of e+1, which those peers issued after
// their own merge of e — so nobody still reads the parity that is being overwritten.
#include <string.h>

#include "kernels.cuh"

struct NkComm {
    int device = 0, rank = 0, world = 1;
    size_t slot_bytes = 0, flag_bytes = 0, total_bytes = 0;
    unsigned char *local = nullptr;  // this rank's buffer
    unsigned char *peer[64] = {nullptr};
    bool ipc_open[64] = {false};
    uint32_t epoch = 0;
    int *err = nullptr;  // device word: 2 = a peer timed out
    bool connected = false;
};

namespace nk {

struct PushParams {
    const uint64_t *keys;  // this rank's [Q*k] keys
    uint32_t n_keys;
    unsigned char *peer[64];
    size_t data_off;   // byte offset of slot[parity][rank] inside a peer buffer
    size_t flag_off;   // byte offset of arrival word [parity][rank]
    uint32_t epoch;
};

__global__ void exchange_push_kernel(PushParams p) {
    pdl_trigger();
    pdl_wait();  // programmatic dependent of the kernel that produced p.keys (common.cuh)
    unsigned char *dst_base = p.peer[blockIdx.x];
    uint64_t *dst = reinterpret_cast<uint64_t *>(dst_base + p.data_off);
    for (uint32_t i = threadIdx.x; i < p.n_keys; i += blockDim.x) dst[i] = p.keys[i];
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        uint32_t *flag = reinterpret_cast<uint32_t *>(dst_base + p.flag_off);
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flag), "r"(p.epoch) : "memory");
    }
}

}  // namespace nk

extern "C" {

NkComm *nk_comm_create(int device_id, int rank, int world, size_t slot_bytes) {
    nk::DeviceGuard _restore_device;
    if (world < 1 || world > 64 || rank < 0 || rank >= world || slot_bytes == 0) {
        nk::set_error("nk_comm_create: bad arguments (1 <= world <= 64, 0 <= rank < world, slot_bytes > 0)");
        return nullptr;
    }
    NkComm *c = new NkComm();
    c->device = device_id; c->rank = rank; c->world = world;
    c->slot_bytes = (slot_bytes + 255) & ~(size_t)255;
    c->flag_bytes = ((size_t)2 * world * 4 + 255) & ~(size_t)255;
    c->total_bytes = c->flag_bytes + (size_t)2 * world * c->slot_bytes;
    cudaError_t e = cudaSetDevice(device_id);
    if (e == cudaSuccess) e = cudaMalloc((void **)&c->local, c->total_bytes);  // cudaMalloc memory is IPC-exportable
    if (e == cudaSuccess) e = cudaMemset(c->local, 0, c->total_bytes);
    if (e == cudaSuccess) e = cudaMalloc((void **)&c->err, sizeof(int));
    if (e == cudaSuccess) e = cudaMemset(c->err, 0, sizeof(int));
    if (e != cudaSuccess) {
        nk::set_error("nk_comm_create(device %d): %s", device_id, cudaGetErrorString(e));
        cudaGetLastError();
        if (c->local) cudaFree(c->local);
        if (c->err) cudaFree(c->err);
        delete c;
        return nullptr;
    }
    c->peer[rank] = c->local;
    if (world == 1) c->connected = true;
    return c;
}

int nk_comm_export(NkComm *c, void *handle_out) {
    nk::DeviceGuard _restore_device;
    if (!c || !handle_out) { nk::set_error("null argument"); return -1; }
    static_assert(sizeof(cudaIpcMemHandle_t) == NK_COMM_HANDLE_BYTES, "IPC handle size");
    NK_CUDA_OK(cudaSetDevice(c->device));
    cudaIpcMemHandle_t h;
    NK_CUDA_OK(cudaIpcGetMemHandle(&h, c->local));
    memcpy(handle_out, &h, sizeof(h));
    return 0;
}

int nk_comm_connect(NkComm *c, const void *handles) {
    nk::DeviceGuard _restore_device;
    if (!c || !handles) { nk::set_error("null argument"); return -1; }
    NK_CUDA_OK(cudaSetDevice(c->device));
    for (int r = 0; r < c->world; ++r) {
        if (r == c->rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, static_cast<const unsigned char *>(handles) + (size_t)r * NK_COMM_HANDLE_BYTES, sizeof(h));
        void *p = nullptr;
        NK_CUDA_OK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        c->peer[r] = static_cast<unsigned char *>(p);
        c->ipc_open[r] = true;
    }
    c->connected = true;
    return 0;
}

int nk_comm_connect_local(NkComm **comms, int world) {
    nk::DeviceGuard _restore_device;
    if (!comms || world < 1) { nk::set_error("null argument"); return -1; }
    for (int a = 0; a < world; ++a) {
        if (!comms[a] || comms[a]->world != world || comms[a]->rank != a) { nk::set_error("nk_comm_connect_local: comms must be in rank order"); return -1; }
        NK_CUDA_OK(cudaSetDevice(comms[a]->device));
        for (int b = 0; b < world; ++b) {
            if (comms[b]->device != comms[a]->device) {
                cudaError_t e = cudaDeviceEnablePeerAccess(comms[b]->device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
                    nk::set_error("peer access %d -> %d: %s", comms[a]->device, comms[b]->device, cudaGetErrorString(e));
                    cudaGetLastError();
                    return -1;
                }
                cudaGetLastError();
            }
            comms[a]->peer[b] = comms[b]->local;
        }
        comms[a]->connected = true;
    }
    return 0;
}

void nk_comm_release(NkComm *c) {
    nk::DeviceGuard _restore_device;
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    for (int r = 0; r < c->world; ++r)
        if (c->ipc_open[r]) cudaIpcCloseMemHandle(c->peer[r]);
    if (c->local) cudaFree(c->local);
    if (c->err) cudaFree(c->err);
    delete c;
}

// Device-side state of the last exchange: 0 ok, 2 = a peer did not arrive within the timeout.  Synchronises `stream`.
int nk_comm_status(NkComm *c, void *stream) {
    nk::DeviceGuard _restore_device;
    if (!c) { nk::set_error("null argument"); return -1; }
    NK_CUDA_OK(cudaSetDevice(c->device));
    NK_CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));
    int h = 0;
    NK_CUDA_OK(cudaMemcpy(&h, c->err, sizeof(int), cudaMemcpyDeviceToHost));
    if (h) {
        cudaMemset(c->err, 0, sizeof(int));
        nk::set_error("exchange: a peer rank did not deliver its candidate list within the timeout");
        return -1;
    }
    return 0;
}

// keys_dev: this rank's [Q x k] keys (device, produced earlier on `stream`); writes the merged, decoded result.
int nk_comm_exchange_merge(NkComm *c, const uint64_t *keys_dev, uint32_t Q, uint32_t k, int metric, uint32_t *out_idx_dev,
                           float *out_score_dev, void *stream) {
    nk::DeviceGuard _restore_device;
    if (!c || !keys_dev || !out_idx_dev || !out_score_dev) { nk::set_error("null argument"); return -1; }
    if (!c->connected) { nk::set_error("exchange: communicator is not connected"); return -1; }
    if (Q == 0 || k == 0) return 0;
    // refused before the epoch advances and anything reaches a peer: a failed call leaves every rank's buffers untouched
    if (k > NK_MAX_K) { nk::set_error("exchange: k=%u exceeds NK_MAX_K=%u (the merge width)", k, NK_MAX_K); return -1; }
    const size_t bytes = (size_t)Q * k * 8;
    if (bytes > c->slot_bytes) { nk::set_error("exchange: Q*k*8 = %zu bytes exceeds the slot size %zu", bytes, c->slot_bytes); return -1; }
    NK_CUDA_OK(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    const uint32_t epoch = ++c->epoch;
    const uint32_t parity = epoch & 1u;
    nk::PushParams p;
    p.keys = keys_dev; p.n_keys = Q * k; p.epoch = epoch;
    for (int r = 0; r < c->world; ++r) p.peer[r] = c->peer[r];
    p.data_off = c->flag_bytes + ((size_t)parity * c->world + c->rank) * c->slot_bytes;
    p.flag_off = ((size_t)parity * c->world + c->rank) * 4;
    NK_CUDA_OK(nk::launch_pdl(nk::exchange_push_kernel, dim3(c->world), dim3(256), 0, st, true, p));
    const uint64_t *lists = reinterpret_cast<const uint64_t *>(c->local + c->flag_bytes + (size_t)parity * c->world * c->slot_bytes);
    const uint32_t *flags = reinterpret_cast<const uint32_t *>(c->local) + (size_t)parity * c->world;
    return nk::merge_keys(lists, (uint32_t)c->world, c->slot_bytes / 8, k, Q, k, nullptr, st, nullptr, 0, out_idx_dev, out_score_dev, metric,
                          flags, epoch, c->err);
}

}  // extern "C"
