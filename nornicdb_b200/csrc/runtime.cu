// runtime.cu — error state, device info and grow-only workspaces.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>

#include "kernels.cuh"

namespace nk {

// Thread-local message (the reference's buffer is one racy process-global, cuda_bridge.go:21-33) with a process-wide
// fallback: cgo may move a goroutine to another OS thread between the failing call and cuda_get_last_error(), and a thread
// that has no message of its own then reads the most recent one of the process instead of an empty string.
static thread_local char g_err[512] = {0};
static thread_local char g_ret[512] = {0};
static std::mutex g_last_mu;
static char g_last[512] = {0};

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    std::lock_guard<std::mutex> lk(g_last_mu);
    memcpy(g_last, g_err, sizeof(g_last));
}
const char *get_error() {
    if (g_err[0]) return g_err;
    std::lock_guard<std::mutex> lk(g_last_mu);
    memcpy(g_ret, g_last, sizeof(g_ret));  // a stable per-thread copy: the caller reads it after the lock is gone
    return g_ret;
}
bool pdl_enabled() {
    static const bool on = [] {
        const char *e = getenv("NK_PDL");
        return e ? atoi(e) != 0 : true;
    }();
    return on;
}
void clear_error() {
    g_err[0] = 0;
    std::lock_guard<std::mutex> lk(g_last_mu);
    g_last[0] = 0;
}

int fatal_overflow(int flag, int *flags, cudaStream_t stream) {
    if (flags) cudaMemsetAsync(flags, 0, sizeof(int), stream);
    set_error("internal: candidate buffer overflow (flag=%d)", flag);
    return -1;
}

int ScanArgs::check(bool range, bool cuda_cores) const {
    if (!mode_dump(mode) && mode_range(mode) == range && !(cuda_cores && mode_row_thr(mode)) && mode_tags(mode) == (qfilter != nullptr) &&
        mode_row_thr(mode) == (row_thr != nullptr) && mode_row_filter(mode) == (row_filter != nullptr) && mode_row_filter(mode) == (qtags != nullptr) &&
        mode_window(mode) == (qwindow != nullptr) && mode_window(mode) == (row_values != nullptr) &&
        mode_row_window(mode) == (row_window != nullptr) && mode_row_window(mode) == (qvalues != nullptr))
        return 0;
    set_error("internal: scan mode %d does not fit this %s scan (%s) or its pointers", (int)mode, range ? "range" : "kNN", cuda_cores ? "CUDA cores" : "tensor");
    return -1;
}

int query_device_info(int device_id, DeviceInfo *out) {
    cudaDeviceProp prop;
    NK_CUDA_OK(cudaGetDeviceProperties(&prop, device_id));
    out->device_id = device_id;
    out->num_sms = prop.multiProcessorCount;
    out->max_smem_optin = prop.sharedMemPerBlockOptin;
    out->cc = prop.major * 10 + prop.minor;
    return 0;
}

int ws_reserve(void **p, size_t *cur, size_t need) {
    if (need <= *cur && *p) return 0;
    if (*p) {
        // Earlier launches on any stream may still be using the old buffer.
        NK_CUDA_OK(cudaDeviceSynchronize());
        NK_CUDA_OK(cudaFree(*p));
        *p = nullptr;
        *cur = 0;
    }
    size_t sz = need + need / 4;  // slack so slowly growing Q / k do not re-allocate every call
    if (sz < 4096) sz = 4096;
    NK_CUDA_OK(cudaMalloc(p, sz));
    *cur = sz;
    return 0;
}

int Workspace::release() {
    void *ptrs[] = {cand, partial, keys, keys2, below, queries, qfilter, out_idx, out_score, qaux, rownorm, flags, sub_rows, sub_gather, scratch, row_thr, row_filter, qtags, qwindow, row_window, qvalues, pair_rows};
    for (void *q : ptrs)
        if (q) cudaFree(q);
    *this = Workspace();
    return 0;
}

}  // namespace nk
