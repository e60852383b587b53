// range.cu — range search (nk_search_range): every admissible row whose exact fp32 score meets the query's threshold.
//
// The scan (scan_tensor_range: 16-bit or TF32 filter with fixed thresholds; scan_simt_range: CUDA cores) appends its
// survivors to one list per query.  Here, per shard:
//   1. the list fills come back to the host; a pass whose lists were too short is re-run ONCE with lists of the exact size
//      (the fills count past the capacity, and the scan is deterministic);
//   2. range_rescore_kernel re-scores every listed pair exactly in fp32 (warp_exact_score, the arithmetic of every filter
//      path's finish) and keeps those that meet the threshold; the survivor counts come back to the host (size protocol).
//      The self-join (nk_search_pairs) runs its twin range_rescore_pairs_kernel, which also drops every row at or below the
//      query's own row; the pairs incident to listed rows (nk_search_pairs_rows) run range_rescore_incident_kernel, which
//      scores each pair with its lower row as the query; the reverse scan of nk_knn_graph_update runs range_rescore_reverse_kernel, which scores each pair as
//      the listed row's k-NN list ranks the query (warp_pair_score) and also holds it to the row's threshold;
//   3. range_compact_kernel packs the survivors of every query into one CSR array, range_sort_runs_kernel sorts runs of
//      RUN keys per query in shared memory, range_merge_kernel merges sorted runs pairwise until each query's segment is
//      one run: (score desc, row asc), the order of nk_search.
#include <algorithm>
#include <vector>

#include "kernels.cuh"
#include "scan_tensor_shared.cuh"

namespace nk {

constexpr int RS_THREADS = 256;    // re-scoring: one warp per list entry
constexpr int RS_ENTRIES = 512;    // list entries per re-scoring CTA (the query is staged once per CTA)
constexpr int CP_THREADS = 256;    // compaction: one thread per list entry
constexpr int RUN = 4096;          // keys one CTA sorts in shared memory (32 KB)
constexpr int RUN_THREADS = 1024;
constexpr uint32_t MAX_GRID_Y = 65535;

struct RescoreParams {
    const void *rows;
    int dtype;
    uint32_t dim;
    uint64_t row_base;
    int metric;
    const float *queries;  // raw fp32 queries [Q x dim]
    uint64_t *lists;       // [Q][list_cap]
    uint32_t list_cap;
    const int *fill;       // [Q], <= list_cap here
    const uint32_t *thr;   // [Q] order-preserving bits of the key-space thresholds
    int *count;            // [Q] survivors (zeroed by the caller)
    uint32_t q_base;       // first query of this launch (grid.y covers at most MAX_GRID_Y queries)
    int rescore;           // 0: CUDA-core lists (already exact): count only
    const float *row_thr;  // REVERSE: key-space threshold per local row
};

// The body of range_rescore_kernel: one CTA per (RS_ENTRIES-entry chunk, query); each listed key becomes the exact key if
// that meets the threshold, else 0.  A NaN score (-inf after warp_exact_score) or -inf never qualifies.
// PAIRS (nk_search_pairs): query q is stored row pair_first + q (global id), and only rows above it are kept, so each
// unordered pair of a self-join survives once, under its lower row.  Compiled in only for the pairs kernel: range searches
// run the code they always ran.
// REVERSE (nk_knn_graph_update): query q is a new or rewritten stored row and each listed row r an old row whose k-NN list q
// may enter.  The score is K(r, q), q's score in r's list (warp_pair_score: |q|^2 as a stored row's), and it must reach both
// the query's threshold (the score floor) and r's own (the score of r's k-th entry).  Tensor-core lists only.
// INCIDENT (nk_search_pairs_rows): query q is stored row c = qrow[q] (global id) and every listed row j forms the pair {c, j}
// of the self-join, which scores it with the lower row as the query.  j == c is dropped, and so is j < c when j is listed
// too (bit j - row_base of `listed`: the pair belongs to j's list); j > c is scored with c as the query (warp_exact_score),
// j < c with j as the query (warp_pair_score: |c|^2 as a stored row's).  Tensor-core lists only.
template <bool PAIRS, bool REVERSE = false, bool INCIDENT = false>
__device__ __forceinline__ void rescore_lists(const RescoreParams &p, uint64_t pair_first, const uint32_t *qrow = nullptr,
                                              const uint32_t *listed = nullptr) {
    extern __shared__ __align__(16) float qs[];  // the query, [dim]
    __shared__ float s_qq;
    __shared__ int s_cnt;
    __shared__ float s_qx;  // INCIDENT: |q|^2 as a stored row's
    const uint32_t q = p.q_base + blockIdx.y;
    const int len = p.fill[q];
    const int i0 = blockIdx.x * RS_ENTRIES;
    if (i0 >= len) return;  // uniform over the CTA
    const int i1 = min(len, i0 + RS_ENTRIES);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint64_t *list = p.lists + (size_t)q * p.list_cap;
    const float thr = ord_to_float(p.thr[q]);
    const uint64_t self = INCIDENT ? (uint64_t)qrow[q] : pair_first + q;  // PAIRS: keep rows > self
    if (tid == 0) s_cnt = 0;
    int mine = 0;
    if (INCIDENT || p.rescore) {
        for (uint32_t j = tid; j < p.dim; j += RS_THREADS) qs[j] = p.queries[(size_t)q * p.dim + j];
        __syncthreads();
        if (REVERSE) {
            if (warp == 0) {
                const float a = warp_stored_sqnorm(qs, p.dtype, p.dim, lane);
                if (lane == 0) s_qq = a;
            }
        } else if (warp == 0) {  // |q|^2 as filter_finish_kernel computes it
            float a = 0.0f;
            for (uint32_t j = lane; j < p.dim; j += 32) a = fmaf(qs[j], qs[j], a);
#pragma unroll
            for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
            if (lane == 0) s_qq = a;
            if (INCIDENT) {
                const float x = warp_stored_sqnorm(qs, p.dtype, p.dim, lane);
                if (lane == 0) s_qx = x;
            }
        }
        __syncthreads();
        for (int i = i0 + warp; i < i1; i += RS_THREADS / 32) {
            const uint32_t grow = key_row(list[i]);
            if (PAIRS && grow <= self) {  // the pair belongs to the lower row's list: not scored here
                if (lane == 0) list[i] = 0ull;
                continue;
            }
            const size_t local = (size_t)(grow - (uint32_t)p.row_base);
            if (INCIDENT && (grow == self || (grow < self && (__ldg(listed + (local >> 5)) >> (local & 31) & 1u)))) {
                if (lane == 0) list[i] = 0ull;
                continue;
            }
            const float sc = REVERSE || (INCIDENT && grow < self)
                                 ? warp_pair_score(p.rows, p.dtype, local, p.dim, qs, INCIDENT ? s_qx : s_qq, p.metric, lane)
                                 : warp_exact_score(p.rows, p.dtype, local, p.dim, qs, s_qq, p.metric, lane);
            // (the graph keeps -inf scores, as filter_finish_kernel does under no floor)
            const bool keep = REVERSE ? sc >= thr && sc >= __ldg(p.row_thr + local) : sc > -INFINITY && sc >= thr;
            if (lane == 0) {
                list[i] = keep ? make_key(sc, grow) : 0ull;
                mine += keep ? 1 : 0;
            }
        }
    } else {
        __syncthreads();
        for (int i = i0 + tid; i < i1; i += RS_THREADS) {
            uint64_t key = list[i];
            if (PAIRS && key != 0ull && key_row(key) <= self) list[i] = key = 0ull;
            mine += key != 0ull ? 1 : 0;
        }
    }
    mine = __reduce_add_sync(0xffffffffu, mine);
    if (lane == 0 && mine) atomicAdd(&s_cnt, mine);
    __syncthreads();
    if (tid == 0 && s_cnt) atomicAdd(p.count + q, s_cnt);
}

__global__ void __launch_bounds__(RS_THREADS) range_rescore_kernel(RescoreParams p) { rescore_lists<false>(p, 0); }
__global__ void __launch_bounds__(RS_THREADS) range_rescore_pairs_kernel(RescoreParams p, uint64_t pair_first) {
    rescore_lists<true>(p, pair_first);
}
__global__ void __launch_bounds__(RS_THREADS) range_rescore_reverse_kernel(RescoreParams p) { rescore_lists<false, true>(p, 0); }
__global__ void __launch_bounds__(RS_THREADS) range_rescore_incident_kernel(RescoreParams p, const uint32_t *qrow, const uint32_t *listed) {
    rescore_lists<false, false, true>(p, 0, qrow, listed);
}

// The keys K(r, j) of given pairs (nk_knn_graph_update's merge), one warp per pair: r = local row rl[i] of `rows`, j = row
// js_row[i] of the widened block js [.. x dim] (global id jid[i]).
__global__ void __launch_bounds__(RS_THREADS) graph_pair_keys_kernel(const void *rows, int dtype, uint32_t dim, int metric, const float *js,
                                                                     const uint32_t *rl, const uint32_t *js_row, const uint32_t *jid,
                                                                     uint32_t n_pairs, uint64_t *out) {
    const int lane = threadIdx.x & 31;
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n_pairs) return;  // uniform over the warp
    const float *j = js + (size_t)js_row[i] * dim;
    const float jj = warp_stored_sqnorm(j, dtype, dim, lane);
    const float sc = warp_pair_score(rows, dtype, rl[i], dim, j, jj, metric, lane);
    if (lane == 0) out[i] = make_key(sc, jid[i]);
}

// Survivors (non-zero keys) of query q's list -> out[off[q] ..), in list order.
__global__ void __launch_bounds__(CP_THREADS) range_compact_kernel(const uint64_t *lists, uint32_t list_cap, const int *fill,
                                                                 const uint64_t *off, int *cursor, uint64_t *out, uint32_t q_base) {
    const uint32_t q = q_base + blockIdx.y;
    const int len = fill[q];
    if ((int)(blockIdx.x * CP_THREADS) >= len) return;  // uniform over the CTA
    const int i = blockIdx.x * CP_THREADS + threadIdx.x, lane = threadIdx.x & 31;
    const uint64_t key = i < len ? lists[(size_t)q * list_cap + i] : 0ull;
    const uint32_t m = __ballot_sync(0xffffffffu, key != 0ull);
    int base = 0;
    if (lane == 0 && m) base = atomicAdd(cursor + q, __popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (key) out[off[q] + base + __popc(m & ((1u << lane) - 1u))] = key;
}

// Runs of RUN keys of every query's segment [off[q], off[q+1]) sorted descending in place, one CTA per run.
__global__ void __launch_bounds__(RUN_THREADS) range_sort_runs_kernel(uint64_t *keys, const uint64_t *off, uint32_t q_base) {
    __shared__ uint64_t s[RUN];
    const uint32_t q = q_base + blockIdx.y;
    const uint64_t n = off[q + 1] - off[q], r0 = (uint64_t)blockIdx.x * RUN;
    if (r0 >= n) return;
    const int len = n - r0 < (uint64_t)RUN ? (int)(n - r0) : RUN;
    int P2 = 2;
    while (P2 < len) P2 <<= 1;
    uint64_t *seg = keys + off[q] + r0;
    for (int i = threadIdx.x; i < P2; i += RUN_THREADS) s[i] = i < len ? seg[i] : 0ull;  // 0 sorts last
    block_bitonic_sort_desc(s, P2);
    for (int i = threadIdx.x; i < len; i += RUN_THREADS) seg[i] = s[i];
}

// One merge pass over every segment: the sorted runs of w keys of a segment are merged pairwise, src -> dst.  A key's place
// is its index in its own run plus its rank in the partner run (binary search); an equal key counts as before it only when
// it sits in the earlier run, so no two keys share a place.
__global__ void range_merge_kernel(const uint64_t *src, uint64_t *dst, const uint64_t *off, uint32_t Q, uint64_t w) {
    const uint64_t total = off[Q];
    for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t lo = 0, hi = Q;  // the last segment starting at or before g (empty segments start where the next one does)
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (off[mid] <= g) lo = mid;
            else hi = mid;
        }
        const uint64_t base = off[lo], n = off[lo + 1] - base, j = g - base;
        const uint64_t run = j / w, start = run * w, pstart = (run ^ 1ull) * w;
        const uint64_t key = src[g];
        if (pstart >= n) {  // no partner run: already in place
            dst[g] = key;
            continue;
        }
        const uint64_t *pr = src + base + pstart;
        const bool first = (run & 1ull) == 0;
        uint64_t a = 0, b = min(n, pstart + w) - pstart;
        while (a < b) {
            const uint64_t m = (a + b) >> 1;
            if (first ? pr[m] > key : pr[m] >= key) a = m + 1;
            else b = m;
        }
        dst[base + min(start, pstart) + (j - start) + a] = key;
    }
}

// ---- host ---------------------------------------------------------------------------------------------------------------
// Workspace layout (see range_qa): ws.keys2 = thresholds [QA] | fills [QA] | counts [Q] | cursors [Q] | offsets [Q+1] (u64).
static uint32_t *ws_thr(Workspace &ws) { return reinterpret_cast<uint32_t *>(ws.keys2); }
static int *ws_fill(Workspace &ws, uint32_t Q) { return reinterpret_cast<int *>(ws.keys2) + range_qa(Q); }
static int *ws_count(Workspace &ws, uint32_t Q) { return ws_fill(ws, Q) + range_qa(Q); }
static int *ws_cursor(Workspace &ws, uint32_t Q) { return ws_count(ws, Q) + Q; }
static uint64_t *ws_off(Workspace &ws, uint32_t Q) { return reinterpret_cast<uint64_t *>(ws_cursor(ws, Q) + Q); }

constexpr uint32_t LIST0 = 1024;  // first list capacity per query (the workspace only grows: later calls start larger)

// Steps 1 and 2 on one shard: survivors per query -> counts[Q] (host); *list_cap = the list capacity the lists were filled
// with (range_sorted_keys reads them); *retried = 1 if the scan ran twice.
int range_scan_shard(const DeviceInfo &di, const ScanArgs &a, bool tensor, const uint32_t *thr_bits, Workspace &ws, uint64_t *launches,
                     int *counts, uint32_t *list_cap_out, int *retried, const uint64_t *pair_first, const IncidentRows *incident) {
    const uint32_t Q = a.Q, QA = range_qa(Q);
    *retried = 0;
    if (a.check(true, !tensor)) return -1;
    if (incident && !tensor) { set_error("internal: the incident pairs are re-scored from tensor-core lists only"); return -1; }
    if (ws_reserve((void **)&ws.keys2, &ws.keys2_bytes, (size_t)(2 * QA + 2 * Q) * 4 + (size_t)(Q + 1) * 8)) return -1;
    uint32_t list_cap = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(LIST0, ws.partial_bytes / ((size_t)Q * 8)), 0x7fffffffu);
    std::vector<int> fill(Q);
    for (int attempt = 0;; ++attempt) {
        if (ws_reserve((void **)&ws.partial, &ws.partial_bytes, (size_t)Q * list_cap * 8)) {
            set_error("nk_search_range: no device memory for the survivor lists (%u queries x %u rows): %s", Q, list_cap, get_error());
            return -1;
        }
        NK_CUDA_OK(cudaMemcpyAsync(ws_thr(ws), thr_bits, (size_t)Q * 4, cudaMemcpyHostToDevice, a.stream));
        NK_CUDA_OK(cudaMemsetAsync(ws_fill(ws, Q), 0, (size_t)(QA + 2 * Q) * 4, a.stream));  // fills, counts, cursors
        if (tensor ? scan_tensor_range(di, a, ws, list_cap, launches) : scan_simt_range(di, a, ws, list_cap, launches)) return -1;
        int fatal = 0;
        NK_CUDA_OK(cudaMemcpyAsync(fill.data(), ws_fill(ws, Q), (size_t)Q * 4, cudaMemcpyDeviceToHost, a.stream));
        NK_CUDA_OK(cudaMemcpyAsync(&fatal, ws.flags + FLAG_FATAL, 4, cudaMemcpyDeviceToHost, a.stream));
        NK_CUDA_OK(cudaStreamSynchronize(a.stream));
        if (fatal) return fatal_overflow(fatal, ws.flags, a.stream);
        int longest = 0;
        for (int f : fill) {
            if (f < 0) { set_error("nk_search_range: more than 2^31 survivors for one query"); return -1; }
            longest = std::max(longest, f);
        }
        if ((uint32_t)longest <= list_cap) break;
        if (attempt) { set_error("internal: range scan survivors changed between two passes (%d > %u)", longest, list_cap); return -1; }
        list_cap = (uint32_t)longest;  // the exact size: the scan is deterministic
        *retried = 1;
    }
    uint32_t longest = 0;
    for (int f : fill) longest = std::max<uint32_t>(longest, (uint32_t)f);
    RescoreParams rp{};
    rp.rows = a.rows; rp.dtype = a.dtype; rp.dim = a.dim; rp.row_base = a.row_base; rp.metric = a.metric; rp.queries = a.queries;
    rp.lists = ws.partial; rp.list_cap = list_cap; rp.fill = ws_fill(ws, Q); rp.thr = ws_thr(ws); rp.count = ws_count(ws, Q);
    rp.rescore = tensor ? 1 : 0; rp.row_thr = a.row_thr;
    const size_t smem = tensor ? (size_t)a.dim * 4 : 0;
    const void *kern = mode_row_thr(a.mode) ? reinterpret_cast<const void *>(range_rescore_reverse_kernel)
                       : incident ? reinterpret_cast<const void *>(range_rescore_incident_kernel)
                       : pair_first ? reinterpret_cast<const void *>(range_rescore_pairs_kernel) : reinterpret_cast<const void *>(range_rescore_kernel);
    if (ensure_smem(di, kern, smem, "range re-scoring", a.dim)) return -1;
    if (longest > 0)
        for (uint32_t q0 = 0; q0 < Q; q0 += MAX_GRID_Y) {
            rp.q_base = q0;
            const dim3 grid((longest + RS_ENTRIES - 1) / RS_ENTRIES, std::min(MAX_GRID_Y, Q - q0));
            if (mode_row_thr(a.mode)) range_rescore_reverse_kernel<<<grid, RS_THREADS, smem, a.stream>>>(rp);
            else if (incident) range_rescore_incident_kernel<<<grid, RS_THREADS, smem, a.stream>>>(rp, incident->qrow, incident->listed);
            else if (pair_first) range_rescore_pairs_kernel<<<grid, RS_THREADS, smem, a.stream>>>(rp, *pair_first);
            else range_rescore_kernel<<<grid, RS_THREADS, smem, a.stream>>>(rp);
            NK_CUDA_OK(cudaGetLastError());
            if (launches) ++*launches;
        }
    NK_CUDA_OK(cudaMemcpyAsync(counts, ws_count(ws, Q), (size_t)Q * 4, cudaMemcpyDeviceToHost, a.stream));
    NK_CUDA_OK(cudaStreamSynchronize(a.stream));
    *list_cap_out = list_cap;
    return 0;
}

// Step 3 after range_scan_shard: the shard's survivors, CSR by counts[Q], each query's run sorted -> *keys (host).
int range_sorted_keys(const DeviceInfo &di, Workspace &ws, cudaStream_t stream, uint32_t Q, const int *counts, uint32_t list_cap,
                      std::vector<uint64_t> *keys, uint64_t *launches) {
    std::vector<uint64_t> off(Q + 1, 0);
    uint32_t longest = 0;
    for (uint32_t q = 0; q < Q; ++q) {
        off[q + 1] = off[q] + (uint64_t)counts[q];
        longest = std::max<uint32_t>(longest, (uint32_t)counts[q]);
    }
    const uint64_t total = off[Q];
    keys->resize(total);
    if (total == 0) return 0;
    // the re-scored fills, for the compaction's grid
    std::vector<int> fill(Q);
    NK_CUDA_OK(cudaMemcpyAsync(fill.data(), ws_fill(ws, Q), (size_t)Q * 4, cudaMemcpyDeviceToHost, stream));
    NK_CUDA_OK(cudaStreamSynchronize(stream));
    int longest_list = 0;
    for (int f : fill) longest_list = std::max(longest_list, f);
    if (ws_reserve((void **)&ws.keys, &ws.keys_bytes, total * 8) || ws_reserve(&ws.scratch, &ws.scratch_bytes, total * 8)) {
        set_error("nk_search_range: no device memory to sort %llu results: %s", (unsigned long long)total, get_error());
        return -1;
    }
    uint64_t *a = ws.keys, *b = static_cast<uint64_t *>(ws.scratch), *d_off = ws_off(ws, Q);
    NK_CUDA_OK(cudaMemcpyAsync(d_off, off.data(), (size_t)(Q + 1) * 8, cudaMemcpyHostToDevice, stream));
    for (uint32_t q0 = 0; q0 < Q; q0 += MAX_GRID_Y) {
        const uint32_t qn = std::min(MAX_GRID_Y, Q - q0);
        range_compact_kernel<<<dim3((longest_list + CP_THREADS - 1) / CP_THREADS, qn), CP_THREADS, 0, stream>>>(
            ws.partial, list_cap, ws_fill(ws, Q), d_off, ws_cursor(ws, Q), a, q0);
        NK_CUDA_OK(cudaGetLastError());
        range_sort_runs_kernel<<<dim3((longest + RUN - 1) / RUN, qn), RUN_THREADS, 0, stream>>>(a, d_off, q0);
        NK_CUDA_OK(cudaGetLastError());
        if (launches) *launches += 2;
    }
    for (uint64_t w = RUN; w < longest; w *= 2) {
        const uint64_t blocks = std::min<uint64_t>((total + 255) / 256, (uint64_t)di.num_sms * 16);
        range_merge_kernel<<<(unsigned)blocks, 256, 0, stream>>>(a, b, d_off, Q, w);
        NK_CUDA_OK(cudaGetLastError());
        if (launches) ++*launches;
        std::swap(a, b);
    }
    NK_CUDA_OK(cudaMemcpyAsync(keys->data(), a, total * 8, cudaMemcpyDeviceToHost, stream));
    NK_CUDA_OK(cudaStreamSynchronize(stream));
    return 0;
}

int graph_pair_keys(const void *rows, int dtype, uint32_t dim, int metric, const float *js, const uint32_t *rl, const uint32_t *js_row,
                    const uint32_t *jid, uint32_t n_pairs, uint64_t *out, cudaStream_t stream) {
    if (n_pairs == 0) return 0;
    const uint64_t blocks = ((uint64_t)n_pairs * 32 + RS_THREADS - 1) / RS_THREADS;
    graph_pair_keys_kernel<<<(unsigned)blocks, RS_THREADS, 0, stream>>>(rows, dtype, dim, metric, js, rl, js_row, jid, n_pairs, out);
    NK_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace nk
