// common.cuh — shared device/host utilities of libnornic_knn (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include <nvtx3/nvToolsExt.h>  // header-only NVTX v3: ranges show up under nsys / ncu --nvtx, no-ops otherwise

#include "../../include/nornic_knn.h"

#define NK_RANGE_PUSH(name) nvtxRangePushA(name)
#define NK_RANGE_POP() nvtxRangePop()

namespace nk {

// ---------------------------------------------------------------------------------------------
// Error plumbing: thread-local message (the reference's is a racy process-global,
// pkg/gpu/cuda/cuda_bridge.go:21-33).
// ---------------------------------------------------------------------------------------------
void set_error(const char *fmt, ...);
const char *get_error();
void clear_error();

#define NK_CUDA_OK(call)                                                                      \
    do {                                                                                      \
        cudaError_t _e = (call);                                                              \
        if (_e != cudaSuccess) {                                                              \
            nk::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return -1;                                                                        \
        }                                                                                     \
    } while (0)

// Every entry point binds the device it needs (cudaSetDevice per call, so callers may hop OS threads) and puts the caller's
// current device back on return: hosts that track the current device themselves (PyTorch, CuPy) never see it move.
// ---- programmatic dependent launch (sm_90+): a kernel launched through launch_pdl() may be scheduled while the kernel
// before it in the stream is still running; pdl_wait() — the first statement of every such kernel — blocks until that
// kernel has completed and its memory is visible (a no-op for an ordinary launch), pdl_trigger() lets the NEXT kernel's
// launch start early.  Used for the short, dependent launches of one search (finish, the early-exit retry stages, the
// cross-GPU push and merge): their launch latency, ~2 us each, overlaps the predecessor instead of following it.
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
bool pdl_enabled();  // NK_PDL (default 1), read once
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool dependent, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = (dependent && pdl_enabled()) ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
#endif

struct DeviceGuard {
    int prev = -1;
    DeviceGuard() {
        if (cudaGetDevice(&prev) != cudaSuccess) {
            prev = -1;
            cudaGetLastError();
        }
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

#define NK_CUDA_OK_PTR(call)                                                                  \
    do {                                                                                      \
        cudaError_t _e = (call);                                                              \
        if (_e != cudaSuccess) {                                                              \
            nk::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return nullptr;                                                                   \
        }                                                                                     \
    } while (0)

// ---------------------------------------------------------------------------------------------
// Candidate keys.  A (score, row) pair is one u64: order-preserving score bits in the high word,
// ~row in the low word, so that a plain unsigned compare implements the boundary's ordering
// "(score desc, row index asc)" (strict '>' forward scan of cuda_bridge.go:356-371).  Euclidean
// search stores score = -dist^2, giving (distance asc, row asc).  Key 0 is below every real key
// (ord(-inf) = 0x007fffff) and marks an empty slot.
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t ord_bits(float s) {
#ifdef __CUDA_ARCH__
    uint32_t b = __float_as_uint(s);
#else
    union { float f; uint32_t u; } c; c.f = s; uint32_t b = c.u;
#endif
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord_to_float(uint32_t o) {
    uint32_t b = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#ifdef __CUDA_ARCH__
    return __uint_as_float(b);
#else
    union { float f; uint32_t u; } c; c.u = b; return c.f;
#endif
}
__host__ __device__ __forceinline__ uint64_t make_key(float s, uint32_t row) {
    return ((uint64_t)ord_bits(s) << 32) | (uint64_t)(0xffffffffu - row);
}
__host__ __device__ __forceinline__ float key_score(uint64_t k) { return ord_to_float((uint32_t)(k >> 32)); }
__host__ __device__ __forceinline__ uint32_t key_row(uint64_t k) { return 0xffffffffu - (uint32_t)k; }

// Per-query tag filter (nk_search_filtered): may a row with tag word `tag` be returned for a query with filter f?
__host__ __device__ __forceinline__ bool tag_admits(uint64_t tag, uint64_t all_of, uint64_t none_of, uint64_t any_of) {
    return (tag & all_of) == all_of && (tag & none_of) == 0 && (any_of == 0 || (tag & any_of) != 0);
}
#ifdef __CUDACC__
// The same against a device filter array [Q] (read through the read-only cache: 24 B per query, shared by every row).
__device__ __forceinline__ bool tag_admits(uint64_t tag, const NkFilter *f) {
    return tag_admits(tag, __ldg(&f->all_of), __ldg(&f->none_of), __ldg(&f->any_of));
}
#endif
// Per-query value window (nk_search_windowed): may a row with value key v be returned for a query with window [lo, hi]?
__host__ __device__ __forceinline__ bool window_admits(uint64_t v, uint64_t lo, uint64_t hi) { return lo <= v && v <= hi; }
#ifdef __CUDACC__
// The same against a device window array [Q] (16 B per query, shared by every row).
__device__ __forceinline__ bool window_admits(uint64_t v, const NkWindow *w) { return window_admits(v, __ldg(&w->lo), __ldg(&w->hi)); }
#endif

// Counter-based U[-1,1) generator, bit-identical to oracle/knn_oracle.c orc_uniform_at().
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z) {
    z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ULL;
    z ^= z >> 27; z *= 0x94D049BB133111EBULL;
    z ^= z >> 31;
    return z;
}
__host__ __device__ __forceinline__ float uniform_at(uint64_t seed, uint64_t elem) {
    uint64_t z = mix64((seed + 1) * 0x9E3779B97F4A7C15ULL + elem * 0xD1B54A32D192ED03ULL);
    uint32_t m = (uint32_t)(z >> 40);
    return (float)m * (1.0f / 8388608.0f) - 1.0f;
}

static inline uint32_t next_pow2(uint32_t v) {
    uint32_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

#ifdef __CUDACC__
// ---------------------------------------------------------------------------------------------
// Block-wide bitonic sort (descending) of P u64 keys in shared memory.  P is a power of two.
// Every thread of the block must call it.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void block_bitonic_sort_desc(uint64_t *s, int P) {
    for (int size = 2; size <= P; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (int t = threadIdx.x; t < (P >> 1); t += blockDim.x) {
                int lo = 2 * t - (t & (stride - 1));
                int hi = lo + stride;
                bool desc = (lo & size) == 0;
                uint64_t a = s[lo], b = s[hi];
                if ((a < b) == desc) {
                    s[lo] = b;
                    s[hi] = a;
                }
            }
        }
    }
    __syncthreads();
}

// Prune one candidate buffer (global, capacity cap, *cnt live entries) down to its best k entries,
// sorted descending, and refresh the pass threshold.  Block-wide; sbuf has P >= cap slots.
// tau is the score a new candidate must reach (>=) to be worth buffering.
__device__ __forceinline__ void block_prune(uint64_t *cand, int cap, int *cnt, float *tau, uint32_t k,
                                            uint64_t *sbuf, int P) {
    __syncthreads();
    int n = *cnt;
    if (n > cap) n = cap;
    for (int i = threadIdx.x; i < P; i += blockDim.x) sbuf[i] = i < n ? cand[i] : 0ull;
    block_bitonic_sort_desc(sbuf, P);
    int keep = n < (int)k ? n : (int)k;
    for (int i = threadIdx.x; i < keep; i += blockDim.x) cand[i] = sbuf[i];
    if (threadIdx.x == 0) {
        *cnt = keep;
        *tau = (n >= (int)k) ? key_score(sbuf[k - 1]) : -INFINITY;
    }
    __syncthreads();
}
// Barrier of a sub-group of `nthreads` threads (a multiple of 32, all of whole warps) on named barrier `bar_id` instead
// of the whole CTA: used by the consumer warpgroups of the tensor-core scans.
__device__ __forceinline__ void group_sync(int bar_id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(nthreads) : "memory");
}
// ---------------------------------------------------------------------------------------------
// Warp-level prune: select the best k of n <= 32*PER_LANE buffered keys with the keys held in registers
// (PER_LANE per lane) by repeated warp-wide max extraction; writes them back sorted descending.  No block
// barrier, so several warps prune different queries concurrently.  Cost ~ k * 60 instructions.
// Caller guarantees every producer of cand[] has finished (barrier) and that *cnt <= 32*PER_LANE.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t warp_max_u64(uint64_t v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        uint32_t lo = __shfl_xor_sync(0xffffffffu, (uint32_t)v, o);
        uint32_t hi = __shfl_xor_sync(0xffffffffu, (uint32_t)(v >> 32), o);
        uint64_t w = ((uint64_t)hi << 32) | lo;
        v = w > v ? w : v;
    }
    return v;
}
// Warp-level prune by RADIX SELECT (cost independent of k): the buffered keys sit in registers (PER_LANE per lane);
// the k-th largest key is found by a most-significant-bit-first binary search whose population counts are one
// redux.sync each, then the survivors are compacted back (unsorted - merge_keys sorts).
//   exact mode : keeps exactly the k largest keys (64-bit search: score, then lowest row);  tau = k-th score.
//   margin mode (tensor-core filter scan; keys carry UPPER bounds): 32-bit search for the k-th largest bound S_k,
//                then keeps everything with bound >= S_k - margin2 (it may beat the k-th once re-scored exactly), at
//                most max_keep entries;  tau = S_k - margin2.
// Caller guarantees every producer of cand[] has finished (barrier) and that *cnt <= 32*PER_LANE.
//   floor_tau (margin mode): a threshold learnt elsewhere (the cross-CTA shared bound); survivors must also reach it.
//   gcount != nullptr: `out` is a shared per-query list; the survivors are appended at atomicAdd(gcount, keep)
//   (entries past out_len are dropped - the caller sizes the list so that cannot happen).
//   nonfinite (margin mode, nullable): set when the k-th bound or the margin is not finite (k or more NaN / Inf rows, or an
//   Inf norm): no threshold can be derived from it — everything is kept and the caller escalates to the exact stage.
template <int PER_LANE>
__device__ __forceinline__ void warp_prune(uint64_t *cand, int *cnt, float *tau, uint32_t k, int lane, uint64_t *out,
                                           int out_len, bool margin_mode, float margin2, int max_keep,
                                           float floor_tau = -INFINITY, int *gcount = nullptr, int *nonfinite = nullptr) {
    int n = *cnt;
    if (n > 32 * PER_LANE) n = 32 * PER_LANE;
    uint64_t v[PER_LANE];
#pragma unroll
    for (int i = 0; i < PER_LANE; ++i) {
        int idx = lane + 32 * i;
        v[i] = idx < n ? cand[idx] : 0ull;
    }
    __syncwarp();
    uint64_t thr_key = 1ull;  // keep every live key
    float new_tau = -INFINITY;
    // margin mode: keys with bound +inf are rows whose score is undecidable (NaN); they are kept but say nothing about the
    // k-th best score, so the threshold comes from the k-th largest FINITE bound = the (k + n_inf)-th largest key
    int k_eff = (int)k;
    if (margin_mode) {
        int inf_mine = 0;
#pragma unroll
        for (int i = 0; i < PER_LANE; ++i) inf_mine += v[i] >= (0xFF800000ull << 32) ? 1 : 0;
        k_eff += __reduce_add_sync(0xffffffffu, inf_mine);
    }
    if (n >= k_eff) {
        uint64_t prefix = 0ull;
        const int low = margin_mode ? 32 : 0;
#pragma unroll 1
        for (int bit = 63; bit >= low; --bit) {
            const uint64_t c = prefix | (1ull << bit);
            int mine = 0;
#pragma unroll
            for (int i = 0; i < PER_LANE; ++i) mine += v[i] >= c ? 1 : 0;
            if (__reduce_add_sync(0xffffffffu, mine) >= k_eff) prefix = c;
        }
        if (prefix == 0ull) {
            // fewer than k LIVE keys (empty slots are key 0): keep them all, no threshold yet
        } else if (margin_mode) {
            new_tau = ord_to_float((uint32_t)(prefix >> 32)) - margin2;
            if (!(new_tau < INFINITY)) {  // +inf or NaN: k rows with undecidable bounds, or a non-finite margin
                new_tau = -INFINITY;
                if (nonfinite && lane == 0) atomicOr(nonfinite, 8);
            } else {
                thr_key = (uint64_t)ord_bits(new_tau) << 32;  // lowest key with that score
                if (thr_key == 0ull) thr_key = 1ull;
            }
        } else {
            new_tau = key_score(prefix);
            thr_key = prefix;
        }
    }
    if (floor_tau > new_tau) {  // a threshold learnt elsewhere (shared bound, caller's score floor) outranks the local one
        new_tau = floor_tau;
        thr_key = (uint64_t)ord_bits(new_tau) << 32;
        if (thr_key == 0ull) thr_key = 1ull;
    }
    // compaction: exclusive prefix of per-lane survivor counts
    int mine = 0;
#pragma unroll
    for (int i = 0; i < PER_LANE; ++i) mine += v[i] >= thr_key ? 1 : 0;
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    const int total = __shfl_sync(0xffffffffu, incl, 31);
    const int cap = margin_mode ? max_keep : (int)k;
    const int keep = total < cap ? total : cap;
    int goff = 0;
    if (gcount) {
        if (lane == 0 && keep > 0) goff = atomicAdd(gcount, keep);
        goff = __shfl_sync(0xffffffffu, goff, 0);
    }
    int pos = incl - mine;
#pragma unroll
    for (int i = 0; i < PER_LANE; ++i) {
        if (v[i] >= thr_key) {
            if (pos < keep) {
                cand[pos] = v[i];
                if (out && goff + pos < out_len) out[goff + pos] = v[i];
            }
            ++pos;
        }
    }
    if (out && !gcount)
        for (int j = keep + lane; j < out_len; j += 32) out[j] = 0ull;
    if (lane == 0) {
        *cnt = keep;
        *tau = new_tau;
    }
    __syncwarp();
}
// Emission without a selection (filter scans): the buffer holds n <= max_keep live-or-stale keys; append those that still
// reach thr_key to the query's shared list (the finish kernel does the global selection anyway).  One ballot compaction
// per 32 entries instead of warp_prune's 32-step radix search: the tail of a scan launch is 64-128 of these per CTA.
__device__ __forceinline__ void warp_emit_above(const uint64_t *cand, int n, uint64_t thr_key, int lane, uint64_t *out, int out_len,
                                                int *gcount) {
    int total = 0;
    for (int base = 0; base < n; base += 32) {
        const uint64_t v = base + lane < n ? cand[base + lane] : 0ull;
        total += __popc(__ballot_sync(0xffffffffu, v >= thr_key));
    }
    if (total == 0) return;
    int goff = 0;
    if (lane == 0) goff = atomicAdd(gcount, total);
    goff = __shfl_sync(0xffffffffu, goff, 0);
    for (int base = 0; base < n; base += 32) {
        const uint64_t v = base + lane < n ? cand[base + lane] : 0ull;
        const bool keep = v >= thr_key;
        const uint32_t m = __ballot_sync(0xffffffffu, keep);
        const int pos = goff + __popc(m & ((1u << lane) - 1u));
        if (keep && pos < out_len) out[pos] = v;
        goff += __popc(m);
    }
}
#endif  // __CUDACC__

}  // namespace nk
