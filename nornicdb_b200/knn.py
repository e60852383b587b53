"""KnnIndex — thin host wrapper over the fused batched C ABI (nk_* in include/nornic_knn.h).

This is the object gpu.EmbeddingIndex would hold instead of a cuda.Buffer (pkg/gpu/gpu.go:1224-1260): a
row-major corpus resident in HBM, row-sharded across the GPUs of this process, searched Q queries at a
time by one fused distance + top-k kernel per shard."""
from __future__ import annotations

import ctypes as C
import datetime as _dt
import math
from typing import List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

from . import _lib

METRICS = {"cosine": 0, "dot": 1, "euclidean": 2}
DTYPES = {"f32": 0, "fp32": 0, "float32": 0, "f16": 1, "fp16": 1, "float16": 1, "bf16": 2, "bfloat16": 2}
PATHS = {"auto": 0, "simt": 1, "tensor": 2, "filter": 3, "shadow": 4}
NK_MAX_K = 1024


class KnnError(RuntimeError):
    pass


def _check(ret: int, what: str) -> int:
    if ret < 0:
        raise KnnError(f"{what}: {_lib.last_error()}")
    return ret


class KnnIndex:
    def __init__(self, dim: int, metric: str = "cosine", dtype: str = "f32", devices: Sequence[int] = (0,)):
        self.lib = _lib.load()
        self.dim = int(dim)
        self.metric = metric
        self.dtype = DTYPES[dtype]
        # bf16 rows travel as raw uint16 bit patterns (numpy has no bfloat16): see to_bf16_bits / from_bf16_bits
        self.np_dtype = np.float16 if self.dtype == 1 else np.uint16 if self.dtype == 2 else np.float32
        self.devices = list(devices)
        ids = (C.c_int * len(self.devices))(*self.devices)
        self.ptr = self.lib.nk_index_create(ids, len(self.devices), self.dim, self.dtype, METRICS[metric])
        if not self.ptr:
            raise KnnError(f"nk_index_create: {_lib.last_error()}")

    # -- lifecycle ---------------------------------------------------------------------------------
    def release(self) -> None:
        if self.ptr:
            self.lib.nk_index_release(self.ptr)
            self.ptr = None

    close = release

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def __len__(self) -> int:
        return int(self.lib.nk_index_rows(self.ptr))

    # -- corpus ------------------------------------------------------------------------------------
    def _rows(self, rows) -> np.ndarray:
        if self.dtype == 2 and np.asarray(rows).dtype.kind == "f":
            rows = to_bf16_bits(rows)  # float input to a bf16 index: round to nearest even, like the device does
        a = np.ascontiguousarray(np.asarray(rows, dtype=self.np_dtype))
        if a.size % self.dim:
            raise KnnError("rows are not a multiple of dim")
        return a.reshape(-1, self.dim)

    def upload(self, rows) -> None:
        a = self._rows(rows)
        _check(self.lib.nk_index_upload(self.ptr, a.ctypes.data_as(C.c_void_p), a.shape[0]), "nk_index_upload")

    def upload_from_f32(self, rows=None, ptr: Optional[int] = None, n_rows: Optional[int] = None) -> None:
        """Upload fp32 host rows whatever the dtype of the index (fp16 indexes convert on the device while loading).
        Either a [n x dim] array, or a raw host address + row count (e.g. the payload of a serialized index)."""
        if ptr is None:
            a = np.ascontiguousarray(np.asarray(rows, dtype=np.float32)).reshape(-1, self.dim)
            ptr, n_rows = a.ctypes.data, a.shape[0]
        _check(self.lib.nk_index_upload_from_f32(self.ptr, C.c_void_p(ptr), int(n_rows)), "nk_index_upload_from_f32")

    def set_row_mask(self, keep) -> None:
        """Row filter for the following searches: `keep` = boolean array with one entry per row (True = may be returned),
        or None to clear.  (Label filter of queryNodes, call_vector.go:177-193, evaluated inside the scan kernels.)"""
        if keep is None:
            _check(self.lib.nk_index_set_row_mask(self.ptr, None, 0), "nk_index_set_row_mask")
            return
        b = np.asarray(keep, dtype=bool).reshape(-1)
        words = np.packbits(b, bitorder="little")
        words = np.concatenate([words, np.zeros((-len(words)) % 4, dtype=np.uint8)]).view("<u4")
        words = np.ascontiguousarray(words)
        _check(self.lib.nk_index_set_row_mask(self.ptr, words.ctypes.data_as(C.c_void_p), int(b.size)), "nk_index_set_row_mask")

    def append(self, rows) -> None:
        a = self._rows(rows)
        _check(self.lib.nk_index_append(self.ptr, a.ctypes.data_as(C.c_void_p), a.shape[0]), "nk_index_append")

    def update_row(self, row: int, vec) -> None:
        a = self._rows(vec)
        _check(self.lib.nk_index_update_row(self.ptr, int(row), a.ctypes.data_as(C.c_void_p)), "nk_index_update_row")

    def remove_swap(self, row: int) -> None:
        _check(self.lib.nk_index_remove_swap(self.ptr, int(row)), "nk_index_remove_swap")

    def fill_uniform(self, n_rows: int, seed: int) -> None:
        _check(self.lib.nk_index_fill_uniform(self.ptr, int(n_rows), int(seed)), "nk_index_fill_uniform")

    def fill_clustered(self, n_rows: int, seed: int, n_centres: int = 1000, sigma: float = 0.1, unit_norm: bool = False) -> None:
        """SURVEY.md 8(d)'s Gaussian-mixture corpus, generated on the device (near-tie stress case)."""
        _check(self.lib.nk_index_fill_clustered(self.ptr, int(n_rows), int(seed), int(n_centres), float(sigma), 1 if unit_norm else 0),
               "nk_index_fill_clustered")

    def refresh_shadow(self) -> None:
        _check(self.lib.nk_index_refresh_shadow(self.ptr), "nk_index_refresh_shadow")

    def set_metric(self, metric: str) -> None:
        _check(self.lib.nk_index_set_metric(self.ptr, METRICS[metric]), "nk_index_set_metric")
        self.metric = metric

    def set_min_score(self, min_score: Optional[float]) -> None:
        """Score floor evaluated inside the kernels (cosine / dot: minimum similarity; euclidean: maximum distance).
        None clears it."""
        if min_score is None:
            min_score = float("inf") if self.metric == "euclidean" else float("-inf")
        _check(self.lib.nk_index_set_min_score(self.ptr, float(min_score)), "nk_index_set_min_score")

    def set_row_groups(self, group_of_row, n_groups: Optional[int] = None) -> None:
        if group_of_row is None:
            _check(self.lib.nk_index_set_row_groups(self.ptr, None, 0, 0), "nk_index_set_row_groups")
            return
        g = np.ascontiguousarray(np.asarray(group_of_row, dtype=np.uint32).reshape(-1))
        ng = int(g.max()) + 1 if n_groups is None and g.size else int(n_groups or 1)
        _check(self.lib.nk_index_set_row_groups(self.ptr, g.ctypes.data_as(C.c_void_p), int(g.size), ng), "nk_index_set_row_groups")

    def search_groups(self, query, k: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Best-of-chunks per node: (node ids, rows of their best chunks, scores), best first."""
        q = np.ascontiguousarray(np.asarray(query, dtype=np.float32).reshape(-1))
        if q.size != self.dim:
            raise KnnError(f"invalid dimensions: query has {q.size}, index has {self.dim}")
        k = int(k)
        if k <= 0:
            return np.empty(0, np.uint32), np.empty(0, np.uint32), np.empty(0, np.float32)
        grp = np.empty(k, dtype=np.uint32); row = np.empty(k, dtype=np.uint32); sc = np.empty(k, dtype=np.float32)
        n = _check(self.lib.nk_search_groups(self.ptr, q.ctypes.data_as(C.c_void_p), k, grp.ctypes.data_as(C.c_void_p),
                                             row.ctypes.data_as(C.c_void_p), sc.ctypes.data_as(C.c_void_p)), "nk_search_groups")
        return grp[:n], row[:n], sc[:n]

    def debug_counters(self) -> dict:
        out = (C.c_uint64 * 4)()
        _check(self.lib.nk_index_debug_counters(self.ptr, out), "nk_index_debug_counters")
        return {"bf16_stage_retries": int(out[0]), "exact_stage_runs": int(out[1]), "longest_list": int(out[2]), "overflow_bits": int(out[3])}

    def filter_dump(self, queries, which: str = "shadow") -> Tuple[np.ndarray, np.ndarray]:
        """Tests only: (estimate, bound) arrays [rows x Q] of the filter kernel `which` ("shadow" | "filter")."""
        q = np.ascontiguousarray(np.asarray(queries, dtype=np.float32)).reshape(-1, self.dim)
        n = len(self)
        est = np.empty((n, q.shape[0]), dtype=np.float32)
        bnd = np.empty((n, q.shape[0]), dtype=np.float32)
        _check(self.lib.nk_debug_filter_dump(self.ptr, q.ctypes.data_as(C.c_void_p), q.shape[0], PATHS[which],
                                             est.ctypes.data_as(C.c_void_p), bnd.ctypes.data_as(C.c_void_p)), "nk_debug_filter_dump")
        return est, bnd

    def assign_ties(self, centroids, metric: str = "euclidean") -> Tuple[np.ndarray, np.ndarray]:
        """Tests only: (rows, candidates [rows x 4]) that assign_nearest listed as near-ties and decided exactly;
        candidate 0xfffffffe = every centroid, 0xffffffff = none.  Every other row was decided by the error bound."""
        c = np.ascontiguousarray(np.asarray(centroids, dtype=np.float32))
        if c.ndim != 2 or c.shape[1] != self.dim:
            raise KnnError(f"invalid dimensions: centroids {c.shape}, index has {self.dim}")
        n = len(self)
        rows = np.empty(max(n, 1), dtype=np.uint32)
        cand = np.empty((max(n, 1), 4), dtype=np.uint32)
        m = _check(self.lib.nk_debug_assign_ties(self.ptr, c.ctypes.data_as(C.c_void_p), c.shape[0], METRICS[metric],
                                                 rows.ctypes.data_as(C.c_void_p), cand.ctypes.data_as(C.c_void_p), n),
                   "nk_debug_assign_ties")
        return rows[:m].copy(), cand[:m].copy()

    def status(self, stream: int = 0) -> None:
        _check(self.lib.nk_index_status(self.ptr, stream), "nk_index_status")

    def search_sharded_device(self, comm: "Comm", q_ptr: int, Q: int, k: int, out_idx_ptr: int, out_score_ptr: int, stream: int = 0) -> int:
        return _check(self.lib.nk_search_sharded_device(self.ptr, comm.ptr, q_ptr, Q, k, out_idx_ptr, out_score_ptr, stream),
                      "nk_search_sharded_device")

    def set_row_base(self, row_base: int) -> None:
        _check(self.lib.nk_index_set_row_base(self.ptr, int(row_base)), "nk_index_set_row_base")

    def attach_device_rows(self, dev_ptr: int, n_rows: int) -> None:
        _check(self.lib.nk_index_attach_device_rows(self.ptr, int(dev_ptr), int(n_rows)), "nk_index_attach_device_rows")

    def set_path(self, path: str) -> None:
        _check(self.lib.nk_index_set_path(self.ptr, PATHS[path]), "nk_index_set_path")

    def read_rows(self, row: int, n_rows: int) -> np.ndarray:
        out = np.empty((n_rows, self.dim), dtype=self.np_dtype)
        _check(self.lib.nk_index_read_rows(self.ptr, int(row), int(n_rows), out.ctypes.data_as(C.c_void_p)),
               "nk_index_read_rows")
        return out

    def debug_flags(self):
        out = (C.c_int * 4)()
        _check(self.lib.nk_index_debug_flags(self.ptr, out), "nk_index_debug_flags")
        return [int(v) for v in out]

    def last_path(self) -> str:
        return {1: "simt", 2: "tensor", 3: "filter", 4: "shadow"}.get(int(self.lib.nk_index_last_path(self.ptr)), "?")

    def enable_timing(self, on: bool = True) -> None:
        _check(self.lib.nk_index_enable_timing(self.ptr, 1 if on else 0), "nk_index_enable_timing")

    def scan_time_ms(self) -> Tuple[float, int]:
        ms, n = C.c_double(0), C.c_uint64(0)
        _check(self.lib.nk_index_scan_time_ms(self.ptr, C.byref(ms), C.byref(n)), "nk_index_scan_time_ms")
        return float(ms.value), int(n.value)

    def stats(self) -> dict:
        st = _lib.NkStats()
        _check(self.lib.nk_index_stats(self.ptr, C.byref(st)), "nk_index_stats")
        return {name: int(getattr(st, name)) for name, _ in st._fields_}

    # -- search ------------------------------------------------------------------------------------
    def _queries(self, queries) -> np.ndarray:
        """queries [Q x dim] (or one [dim] vector) -> contiguous fp32 [Q x dim]."""
        q = np.ascontiguousarray(np.asarray(queries, dtype=np.float32))
        if q.ndim == 1:
            q = q.reshape(1, -1)
        if q.shape[1] != self.dim:
            raise KnnError(f"invalid dimensions: query has {q.shape[1]}, index has {self.dim}")  # gpu.go:1533-1535
        return q

    def search(self, queries, k: int) -> Tuple[np.ndarray, np.ndarray]:
        """queries [Q x dim] fp32 host -> (idx [Q x k'] uint32, score [Q x k'] fp32), k' = min(k, N).
        Euclidean scores are distances (ascending); cosine / dot are similarities (descending)."""
        q = self._queries(queries)
        Q = q.shape[0]
        k = int(k)
        if k <= 0 or Q == 0:
            return np.empty((Q, 0), np.uint32), np.empty((Q, 0), np.float32)
        idx = np.empty((Q, k), dtype=np.uint32)
        sc = np.empty((Q, k), dtype=np.float32)
        ke = _check(self.lib.nk_search(self.ptr, q.ctypes.data_as(C.c_void_p), Q, k, idx.ctypes.data_as(C.c_void_p),
                                       sc.ctypes.data_as(C.c_void_p)), "nk_search")
        return idx[:, :ke], sc[:, :ke]

    def search_rows(self, rows, k: int, filters=None, windows=None) -> Tuple[np.ndarray, np.ndarray]:
        """The k nearest OTHER rows of stored rows: rows = row ids (< len(self), repeats allowed), each searched as stored now
        -> (idx [Q x k'] uint32, score [Q x k'] fp32), k' = min(k, admissible rows), with search()'s conventions.  A query
        with fewer admissible other rows gets index 0xffffffff and score 0 in its unused slots.  rows = every row id gives
        the k-NN graph of the index in one call (served in blocks of 1024 queries).  filters: None, or one tag filter per
        query ([Q x 3] uint64, as in search_filtered): query q then lists only rows its filter admits (its own row may be
        refused by it) (nk_search_rows_filtered).  windows: None, or one value window per query ([Q x 2] uint64, as in
        search_windowed; one pair applies to every query): query q then lists only rows whose value key its window admits (its
        own row may lie outside it); band_windows(keys[rows], below, above) gives "near this row's value"
        (nk_search_rows_windowed)."""
        r = np.asarray(rows, dtype=np.int64).reshape(-1)
        if r.size and (r.min() < 0 or r.max() > 0xFFFFFFFF):
            raise KnnError("search_rows: row ids must be in [0, 2^32)")
        r = np.ascontiguousarray(r.astype(np.uint32))
        Q = r.size
        f = None if filters is None else as_filters(filters, Q)
        w = None if windows is None else as_windows(windows, Q)
        k = int(k)
        if k <= 0 or Q == 0:
            return np.empty((Q, 0), np.uint32), np.empty((Q, 0), np.float32)
        idx = np.empty((Q, k), dtype=np.uint32)
        sc = np.empty((Q, k), dtype=np.float32)
        if w is not None:
            ke = _check(self.lib.nk_search_rows_windowed(self.ptr, r.ctypes.data_as(C.c_void_p), None if f is None else f.ctypes.data_as(C.c_void_p),
                                                         w.ctypes.data_as(C.c_void_p), Q, k, idx.ctypes.data_as(C.c_void_p),
                                                         sc.ctypes.data_as(C.c_void_p)), "nk_search_rows_windowed")
        elif f is None:
            ke = _check(self.lib.nk_search_rows(self.ptr, r.ctypes.data_as(C.c_void_p), Q, k, idx.ctypes.data_as(C.c_void_p),
                                                sc.ctypes.data_as(C.c_void_p)), "nk_search_rows")
        else:
            ke = _check(self.lib.nk_search_rows_filtered(self.ptr, r.ctypes.data_as(C.c_void_p), f.ctypes.data_as(C.c_void_p), Q, k,
                                                         idx.ctypes.data_as(C.c_void_p), sc.ctypes.data_as(C.c_void_p)),
                        "nk_search_rows_filtered")
        return idx[:, :ke], sc[:, :ke]

    def _graph_filters(self, filters, what: str):
        """filters of a graph call: None, or one [n x 3] uint64 filter per current row"""
        if filters is None:
            return None
        n = len(self)
        f = np.ascontiguousarray(np.asarray(filters, dtype=np.uint64))
        if f.shape != (n, 3):
            raise KnnError(f"{what}: filters must be [{n} x 3] (one per current row), not {list(f.shape)}")
        return f

    def _graph_windows(self, windows, what: str):
        """windows of a graph call: None, or one [n x 2] uint64 (lo, hi) window per current row"""
        if windows is None:
            return None
        n = len(self)
        w = np.ascontiguousarray(np.asarray(windows, dtype=np.uint64))
        if w.shape != (n, 2):
            raise KnnError(f"{what}: windows must be [{n} x 2] (one per current row), not {list(w.shape)}")
        return w

    def update_knn_graph(self, idx, score, n_old: int, changed=None, k: Optional[int] = None,
                         filters=None, windows=None) -> Tuple[np.ndarray, np.ndarray, int]:
        """Bring the k-NN graph search_rows(range(n_old), k) returned up to date after rows were appended (rows n_old ..
        len(self) - 1) and old rows rewritten (`changed`: their ids, repeats allowed) -> (idx, score, lists_changed): what
        search_rows(every row, k) returns now, k' = min(k, admissible rows) columns, and how many old rows' lists changed.
        idx / score: [n_old x w]; k defaults to w, and a narrower graph (search_rows returns fewer than k columns while fewer
        rows are admissible) is padded with 0xffffffff / 0.  Build the graph with the path set (set_path("shadow") or
        "filter"), and keep the metric, the score floor and the old rows' mask bits (set the mask again after append).  After
        remove_swap, use remap_knn_graph (nk_knn_graph_update).
        filters: None, or one tag filter per current row ([len(self) x 3] uint64): the graph of search_rows(every row, k,
        filters), each list bounded by its row's own filter.  An old row whose tag or filter changed since the graph was built
        must be listed in `changed`, like a rewritten row (nk_knn_graph_update_filtered).
        windows: None, or one value window per current row ([len(self) x 2] uint64, as band_windows returns them): the graph
        of search_rows(every row, k, filters, windows), a time-local graph.  An old row whose value key or window changed
        since the graph was built must be listed in `changed`, like a retag; a band window moves with its row's key, so
        re-valuing a row is such a change (nk_knn_graph_update_windowed)."""
        idx = np.asarray(idx, dtype=np.uint32)
        score = np.asarray(score, dtype=np.float32)
        n_old = int(n_old)
        if idx.ndim != 2 or score.shape != idx.shape or idx.shape[0] != n_old:
            raise KnnError("update_knn_graph: idx and score must both be [n_old x w]")
        k = idx.shape[1] if k is None else int(k)
        if k < idx.shape[1]:
            raise KnnError(f"update_knn_graph: k={k} is narrower than the graph ({idx.shape[1]} columns)")
        n = len(self)
        if n_old > n:
            raise KnnError(f"update_knn_graph: n_old={n_old} exceeds the index's {n} rows")
        ch = np.ascontiguousarray(np.asarray([] if changed is None else changed, dtype=np.int64).reshape(-1))
        if ch.size and ch.min() < 0:
            raise KnnError("update_knn_graph: changed row ids must be >= 0")
        ch = np.ascontiguousarray(ch.astype(np.uint32))
        f = self._graph_filters(filters, "update_knn_graph")
        w = self._graph_windows(windows, "update_knn_graph")
        if k <= 0 or n == 0:
            return np.empty((n, 0), np.uint32), np.empty((n, 0), np.float32), 0
        gi = np.full((n, k), 0xFFFFFFFF, dtype=np.uint32)
        gs = np.zeros((n, k), dtype=np.float32)
        gi[:n_old, :idx.shape[1]] = idx
        gs[:n_old, :idx.shape[1]] = score
        changed_lists = C.c_uint64(0)
        chp = ch.ctypes.data_as(C.c_void_p) if ch.size else None
        if w is not None:
            ke = _check(self.lib.nk_knn_graph_update_windowed(self.ptr, k, n_old, chp, int(ch.size), None if f is None else f.ctypes.data_as(C.c_void_p),
                                                              w.ctypes.data_as(C.c_void_p), gi.ctypes.data_as(C.c_void_p),
                                                              gs.ctypes.data_as(C.c_void_p), C.byref(changed_lists)),
                        "nk_knn_graph_update_windowed")
        elif f is None:
            ke = _check(self.lib.nk_knn_graph_update(self.ptr, k, n_old, chp, int(ch.size), gi.ctypes.data_as(C.c_void_p),
                                                     gs.ctypes.data_as(C.c_void_p), C.byref(changed_lists)), "nk_knn_graph_update")
        else:
            ke = _check(self.lib.nk_knn_graph_update_filtered(self.ptr, k, n_old, chp, int(ch.size), f.ctypes.data_as(C.c_void_p),
                                                              gi.ctypes.data_as(C.c_void_p), gs.ctypes.data_as(C.c_void_p),
                                                              C.byref(changed_lists)), "nk_knn_graph_update_filtered")
        return gi[:, :ke], gs[:, :ke], int(changed_lists.value)

    def remap_knn_graph(self, idx, score, n_old: int, src, k: Optional[int] = None,
                        filters=None, windows=None) -> Tuple[np.ndarray, np.ndarray, int]:
        """Bring the k-NN graph search_rows(range(n_old), k) returned up to date after any mix of append, update_row and
        remove_swap -> (idx, score, lists_changed): what search_rows(every row, k) returns now, k' = min(k, admissible rows)
        columns, and how many rows that hold their old contents at their old id got a different list.  src: a GraphRowMap
        that followed the changes, or its src_of_row (one entry per current row: the old row whose contents it holds, or
        ROW_NEW).  idx / score / k and the preconditions are those of update_knn_graph, the mask bit of a moved row included
        (nk_knn_graph_remap).
        filters: None, or one tag filter per current row ([len(self) x 3] uint64, in current row order): the graph of
        search_rows(every row, k, filters).  A row whose tag or filter changed since the graph was built must be ROW_NEW in
        src: record it with GraphRowMap.update_row, like a rewrite (nk_knn_graph_remap_filtered).
        windows: None, or one value window per current row ([len(self) x 2] uint64, in current row order): the graph of
        search_rows(every row, k, filters, windows).  A row whose value key or window changed since the graph was built must
        be ROW_NEW in src, like a retag: record it with GraphRowMap.update_row (nk_knn_graph_remap_windowed)."""
        idx = np.asarray(idx, dtype=np.uint32)
        score = np.asarray(score, dtype=np.float32)
        n_old = int(n_old)
        if idx.ndim != 2 or score.shape != idx.shape or idx.shape[0] != n_old:
            raise KnnError("remap_knn_graph: idx and score must both be [n_old x w]")
        k = idx.shape[1] if k is None else int(k)
        if k < idx.shape[1]:
            raise KnnError(f"remap_knn_graph: k={k} is narrower than the graph ({idx.shape[1]} columns)")
        s = np.asarray(src.src_of_row if isinstance(src, GraphRowMap) else src, dtype=np.int64).reshape(-1)
        n = len(self)
        if s.size != n:
            raise KnnError(f"remap_knn_graph: src_of_row has {s.size} entries, the index {n} rows")
        if s.size and (s.min() < 0 or s.max() > ROW_NEW):
            raise KnnError("remap_knn_graph: src_of_row entries must be old row ids or ROW_NEW")
        s = np.ascontiguousarray(s.astype(np.uint32))
        f = self._graph_filters(filters, "remap_knn_graph")
        w = self._graph_windows(windows, "remap_knn_graph")
        if k <= 0 or n == 0:
            return np.empty((n, 0), np.uint32), np.empty((n, 0), np.float32), 0
        oi = np.full((n_old, k), 0xFFFFFFFF, dtype=np.uint32)
        osc = np.zeros((n_old, k), dtype=np.float32)
        oi[:, :idx.shape[1]] = idx
        osc[:, :idx.shape[1]] = score
        gi = np.full((n, k), 0xFFFFFFFF, dtype=np.uint32)
        gs = np.zeros((n, k), dtype=np.float32)
        changed_lists = C.c_uint64(0)
        graph = (oi.ctypes.data_as(C.c_void_p), osc.ctypes.data_as(C.c_void_p), gi.ctypes.data_as(C.c_void_p),
                 gs.ctypes.data_as(C.c_void_p), C.byref(changed_lists))
        if w is not None:
            ke = _check(self.lib.nk_knn_graph_remap_windowed(self.ptr, k, n_old, s.ctypes.data_as(C.c_void_p),
                                                             None if f is None else f.ctypes.data_as(C.c_void_p),
                                                             w.ctypes.data_as(C.c_void_p), *graph), "nk_knn_graph_remap_windowed")
        elif f is None:
            ke = _check(self.lib.nk_knn_graph_remap(self.ptr, k, n_old, s.ctypes.data_as(C.c_void_p), *graph), "nk_knn_graph_remap")
        else:
            ke = _check(self.lib.nk_knn_graph_remap_filtered(self.ptr, k, n_old, s.ctypes.data_as(C.c_void_p),
                                                             f.ctypes.data_as(C.c_void_p), *graph), "nk_knn_graph_remap_filtered")
        return gi[:, :ke], gs[:, :ke], int(changed_lists.value)

    def search_device(self, q_ptr: int, Q: int, k: int, out_idx_ptr: int, out_score_ptr: int, stream: int = 0) -> int:
        return _check(self.lib.nk_search_device(self.ptr, q_ptr, Q, k, out_idx_ptr, out_score_ptr, stream),
                      "nk_search_device")

    # -- per-query tag filters ---------------------------------------------------------------------
    def set_row_tags(self, tags, first_row: int = 0) -> None:
        """Tag words (uint64, one per row) of rows [first_row, first_row + len(tags)); untagged rows have tag 0.  A filtered
        k-NN graph is not told: the caller reports each row whose tag changed as rewritten (GraphRowMap.update_row, or
        update_knn_graph's `changed`)."""
        t = np.ascontiguousarray(np.asarray(tags, dtype=np.uint64).reshape(-1))
        _check(self.lib.nk_index_set_row_tags(self.ptr, int(first_row), t.ctypes.data_as(C.c_void_p), int(t.size)),
               "nk_index_set_row_tags")

    def search_filtered(self, queries, k: int, filters) -> Tuple[np.ndarray, np.ndarray]:
        """search() with one tag filter per query: filters [Q x 3] uint64 (all_of, none_of, any_of), None = no filter.
        Slots beyond a query's admissible rows hold index 0xffffffff and score 0."""
        q = self._queries(queries)
        Q = q.shape[0]
        f = None if filters is None else as_filters(filters, Q)
        k = int(k)
        if k <= 0 or Q == 0:
            return np.empty((Q, 0), np.uint32), np.empty((Q, 0), np.float32)
        idx = np.empty((Q, k), dtype=np.uint32)
        sc = np.empty((Q, k), dtype=np.float32)
        ke = _check(self.lib.nk_search_filtered(self.ptr, q.ctypes.data_as(C.c_void_p), None if f is None else f.ctypes.data_as(C.c_void_p),
                                                Q, k, idx.ctypes.data_as(C.c_void_p), sc.ctypes.data_as(C.c_void_p)), "nk_search_filtered")
        return idx[:, :ke], sc[:, :ke]

    def search_range(self, queries, thresholds, filters=None, windows=None) -> List[Tuple[np.ndarray, np.ndarray]]:
        """Every admissible row whose score reaches the query's threshold (cosine / dot: minimum score; euclidean: maximum
        distance), one threshold per query (a scalar applies to all).  Returns one (idx uint32, score float32) pair per query,
        in search()'s order.  The result buffer grows to the size the library reports (nk_search_range's size protocol).
        windows: None, or per-query value windows as for search_windowed (nk_search_range_windowed)."""
        q = self._queries(queries)
        Q = q.shape[0]
        t = np.ascontiguousarray(np.broadcast_to(np.asarray(thresholds, dtype=np.float32), (Q,)))
        f = None if filters is None else as_filters(filters, Q)
        w = None if windows is None else as_windows(windows, Q)
        off = np.zeros(Q + 1, dtype=np.uint64)
        total = C.c_uint64(0)
        cap = getattr(self, "_range_cap", 0)
        while True:
            idx = np.empty(max(cap, 1), dtype=np.uint32)
            sc = np.empty(max(cap, 1), dtype=np.float32)
            if w is None:
                _check(self.lib.nk_search_range(self.ptr, q.ctypes.data_as(C.c_void_p), t.ctypes.data_as(C.c_void_p),
                                                None if f is None else f.ctypes.data_as(C.c_void_p), Q, cap,
                                                off.ctypes.data_as(C.c_void_p), idx.ctypes.data_as(C.c_void_p),
                                                sc.ctypes.data_as(C.c_void_p), C.byref(total)), "nk_search_range")
            else:
                _check(self.lib.nk_search_range_windowed(self.ptr, q.ctypes.data_as(C.c_void_p), t.ctypes.data_as(C.c_void_p),
                                                         None if f is None else f.ctypes.data_as(C.c_void_p), w.ctypes.data_as(C.c_void_p),
                                                         Q, cap, off.ctypes.data_as(C.c_void_p), idx.ctypes.data_as(C.c_void_p),
                                                         sc.ctypes.data_as(C.c_void_p), C.byref(total)), "nk_search_range_windowed")
            if total.value <= cap:
                break
            cap = int(total.value)
            self._range_cap = cap
        o = off.astype(np.int64)
        return [(idx[o[i]:o[i + 1]].copy(), sc[o[i]:o[i + 1]].copy()) for i in range(Q)]

    def search_pairs(self, threshold: float, first_row: int = 0, n_rows: Optional[int] = None,
                     filter=None, window=None, max_gap=None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Similarity self-join: for each left row i of the stripe [first_row, first_row + n_rows) (default: to the end of the
        index), every admissible row j > i whose score against row i reaches `threshold` (cosine / dot: minimum score;
        euclidean: maximum distance), so each pair of the stripe appears once, under its lower row.  filter = one
        (all_of, none_of, any_of) tag filter for both sides, None = none.  Returns CSR arrays (offsets uint64 [n_rows + 1],
        idx uint32, score float32): row first_row + r's list is [offsets[r], offsets[r + 1]), in search()'s order.  The result
        buffer grows to the size the library reports (nk_search_pairs' size protocol); a call that outgrows it joins twice.
        window = one (lo, hi) value window for both sides, None = none.  max_gap = a band: a pair also needs both rows to have a
        value and |key[i] - key[j]| <= max_gap, in key units (value units for int and datetime columns); an np.timedelta64 is
        taken in nanoseconds.  None = no band (nk_search_pairs_windowed)."""
        first_row = int(first_row)
        n_rows = max(len(self) - first_row, 0) if n_rows is None else int(n_rows)
        if first_row < 0 or n_rows < 0:
            raise KnnError("search_pairs: first_row and n_rows must be >= 0")
        f = None if filter is None else as_filters(filter, 1)
        w = None if window is None else as_windows(window, 1)
        gap = NO_GAP if max_gap is None else _gap_keys(max_gap)
        windowed = w is not None or gap != NO_GAP
        off = np.zeros(n_rows + 1, dtype=np.uint64)
        total = C.c_uint64(0)
        cap = getattr(self, "_pairs_cap", 0)
        while True:
            idx = np.empty(max(cap, 1), dtype=np.uint32)
            sc = np.empty(max(cap, 1), dtype=np.float32)
            out = (cap, off.ctypes.data_as(C.c_void_p), idx.ctypes.data_as(C.c_void_p), sc.ctypes.data_as(C.c_void_p), C.byref(total))
            fp = None if f is None else f.ctypes.data_as(C.c_void_p)
            if windowed:
                _check(self.lib.nk_search_pairs_windowed(self.ptr, first_row, n_rows, float(threshold), fp,
                                                         None if w is None else w.ctypes.data_as(C.c_void_p), gap, *out),
                       "nk_search_pairs_windowed")
            else:
                _check(self.lib.nk_search_pairs(self.ptr, first_row, n_rows, float(threshold), fp, *out), "nk_search_pairs")
            if total.value <= cap:
                break
            cap = int(total.value)
            self._pairs_cap = cap
        t = int(total.value)
        return off, idx[:t].copy(), sc[:t].copy()

    def _pairs_args(self, filter, window, max_gap):
        f = None if filter is None else as_filters(filter, 1)
        w = None if window is None else as_windows(window, 1)
        gap = NO_GAP if max_gap is None else _gap_keys(max_gap)
        return (None if f is None else f.ctypes.data_as(C.c_void_p), None if w is None else w.ctypes.data_as(C.c_void_p), gap), (f, w)

    def search_pairs_rows(self, rows, threshold: float, filter=None, window=None,
                          max_gap=None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """The pairs of the whole-index self-join (search_pairs over every row, with the same threshold, filter, window and
        max_gap) that have at least one end among `rows` (distinct row ids), grouped by that end; a pair with both ends listed
        goes under the lower one.  Scores are the join's (the lower row of the pair is the query), each list in search()'s
        order.  Returns CSR arrays (offsets uint64 [len(rows) + 1], idx uint32, score float32): rows[r]'s pairs are
        [offsets[r], offsets[r + 1]).  Runs on the graph path (TENSOR_SHADOW or TENSOR_FILTER), so it equals the join with that
        path forced; SIMT or TENSOR forced is refused (nk_search_pairs_rows_windowed)."""
        r = np.ascontiguousarray(np.asarray(rows, dtype=np.int64).reshape(-1))
        if r.size and (r.min() < 0 or r.max() > 0xFFFFFFFF):
            raise KnnError("search_pairs_rows: row ids must lie in [0, 2^32)")
        r = np.ascontiguousarray(r.astype(np.uint32))
        args, keep = self._pairs_args(filter, window, max_gap)
        off = np.zeros(r.size + 1, dtype=np.uint64)
        total = C.c_uint64(0)
        cap = getattr(self, "_pairs_cap", 0)
        while True:
            idx = np.empty(max(cap, 1), dtype=np.uint32)
            sc = np.empty(max(cap, 1), dtype=np.float32)
            _check(self.lib.nk_search_pairs_rows_windowed(self.ptr, r.ctypes.data_as(C.c_void_p), int(r.size), float(threshold), *args,
                                                          cap, off.ctypes.data_as(C.c_void_p), idx.ctypes.data_as(C.c_void_p),
                                                          sc.ctypes.data_as(C.c_void_p), C.byref(total)),
                   "nk_search_pairs_rows_windowed")
            if total.value <= cap:
                break
            cap = int(total.value)
            self._pairs_cap = cap
        t = int(total.value)
        return off, idx[:t].copy(), sc[:t].copy()

    def remap_pairs(self, pairs, n_old: int, src, threshold: float, filter=None, window=None,
                    max_gap=None) -> Tuple[np.ndarray, np.ndarray, np.ndarray, int, int]:
        """Bring a stored self-join up to date after any mix of append, update_row, remove_swap, retags and re-valued rows.
        pairs = (offsets, idx, score): what search_pairs(threshold, filter=, window=, max_gap=) over the whole index of n_old
        rows returned.  src: a GraphRowMap that followed the changes (call update_row for a retagged or re-valued row too), or
        its src_of_row.  Returns (offsets, idx, score, n_dropped, n_found): what that search_pairs call over every row returns
        now on the graph path, bit for bit; the old pairs dropped (an end gone, moved or new) and the pairs found incident to
        the new and moved rows (nk_pairs_remap)."""
        oo, oi, osc = pairs
        n_old = int(n_old)
        oo = np.ascontiguousarray(np.asarray(oo, dtype=np.uint64).reshape(-1))
        oi = np.ascontiguousarray(np.asarray(oi, dtype=np.uint32).reshape(-1))
        osc = np.ascontiguousarray(np.asarray(osc, dtype=np.float32).reshape(-1))
        if oo.size != n_old + 1 or oi.size != osc.size or int(oo[-1]) != oi.size:
            raise KnnError("remap_pairs: pairs must be CSR over n_old rows (n_old + 1 offsets, offsets[-1] entries)")
        s = np.asarray(src.src_of_row if isinstance(src, GraphRowMap) else src, dtype=np.int64).reshape(-1)
        n = len(self)
        if s.size != n:
            raise KnnError(f"remap_pairs: src_of_row has {s.size} entries, the index {n} rows")
        if s.size and (s.min() < 0 or s.max() > ROW_NEW):
            raise KnnError("remap_pairs: src_of_row entries must be old row ids or ROW_NEW")
        s = np.ascontiguousarray(s.astype(np.uint32))
        args, keep = self._pairs_args(filter, window, max_gap)
        off = np.zeros(n + 1, dtype=np.uint64)
        total, dropped, found = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        cap = getattr(self, "_pairs_cap", 0)
        while True:
            idx = np.empty(max(cap, 1), dtype=np.uint32)
            sc = np.empty(max(cap, 1), dtype=np.float32)
            _check(self.lib.nk_pairs_remap(self.ptr, float(threshold), *args, n_old, s.ctypes.data_as(C.c_void_p),
                                           oo.ctypes.data_as(C.c_void_p), oi.ctypes.data_as(C.c_void_p), osc.ctypes.data_as(C.c_void_p),
                                           cap, off.ctypes.data_as(C.c_void_p), idx.ctypes.data_as(C.c_void_p),
                                           sc.ctypes.data_as(C.c_void_p), C.byref(total), C.byref(dropped), C.byref(found)),
                   "nk_pairs_remap")
            if total.value <= cap:
                break
            cap = int(total.value)
            self._pairs_cap = cap
        t = int(total.value)
        return off, idx[:t].copy(), sc[:t].copy(), int(dropped.value), int(found.value)

    def search_filtered_device(self, q_ptr: int, filters_ptr: int, Q: int, k: int, out_idx_ptr: int, out_score_ptr: int,
                               stream: int = 0) -> int:
        """Device-resident filtered search: filters_ptr = device [Q x 3] uint64 (0 = no filter), valid until the stream ran."""
        return _check(self.lib.nk_search_filtered_device(self.ptr, q_ptr, filters_ptr or None, Q, k, out_idx_ptr, out_score_ptr, stream),
                      "nk_search_filtered_device")

    # -- per-query value windows -------------------------------------------------------------------
    def set_row_values(self, values, first_row: int = 0) -> None:
        """Value keys of rows [first_row, first_row + len(values)); rows never given one have key 0 (no value).  `values`:
        keys already encoded (uint64), or numbers (int64, float, datetime64), which are encoded with value_keys()."""
        a = np.asarray(values).reshape(-1)
        v = np.ascontiguousarray(a if a.dtype == np.uint64 else value_keys(a))
        _check(self.lib.nk_index_set_row_values(self.ptr, int(first_row), v.ctypes.data_as(C.c_void_p), int(v.size)),
               "nk_index_set_row_values")

    def search_windowed(self, queries, k: int, windows, filters=None) -> Tuple[np.ndarray, np.ndarray]:
        """search_filtered() with one value window per query on top: windows [Q x 2] uint64 (lo, hi), inclusive key bounds (one
        pair applies to every query; window() turns Qdrant Range bounds into one), None = none.  Row r is admissible iff
        lo <= value[r] <= hi and the query's tag filter (None = none) admits it.  Slots beyond a query's admissible rows hold
        index 0xffffffff and score 0."""
        q = self._queries(queries)
        Q = q.shape[0]
        f = None if filters is None else as_filters(filters, Q)
        w = None if windows is None else as_windows(windows, Q)
        k = int(k)
        if k <= 0 or Q == 0:
            return np.empty((Q, 0), np.uint32), np.empty((Q, 0), np.float32)
        idx = np.empty((Q, k), dtype=np.uint32)
        sc = np.empty((Q, k), dtype=np.float32)
        ke = _check(self.lib.nk_search_windowed(self.ptr, q.ctypes.data_as(C.c_void_p), None if f is None else f.ctypes.data_as(C.c_void_p),
                                                None if w is None else w.ctypes.data_as(C.c_void_p), Q, k,
                                                idx.ctypes.data_as(C.c_void_p), sc.ctypes.data_as(C.c_void_p)), "nk_search_windowed")
        return idx[:, :ke], sc[:, :ke]

    def search_windowed_device(self, q_ptr: int, filters_ptr: int, windows_ptr: int, Q: int, k: int, out_idx_ptr: int,
                               out_score_ptr: int, stream: int = 0) -> int:
        """Device-resident windowed search: filters_ptr = device [Q x 3] uint64 (0 = no filter), windows_ptr = device [Q x 2]
        uint64 (0 = no window), both valid until the stream ran."""
        return _check(self.lib.nk_search_windowed_device(self.ptr, q_ptr, filters_ptr or None, windows_ptr or None, Q, k, out_idx_ptr,
                                                         out_score_ptr, stream), "nk_search_windowed_device")

    def search_keys_device(self, q_ptr: int, Q: int, k: int, out_keys_ptr: int, stream: int = 0) -> int:
        return _check(self.lib.nk_search_keys_device(self.ptr, q_ptr, Q, k, out_keys_ptr, stream),
                      "nk_search_keys_device")

    def score_subset(self, query, rows: Sequence[int], k: Optional[int] = None) -> Tuple[np.ndarray, np.ndarray]:
        q = np.ascontiguousarray(np.asarray(query, dtype=np.float32).reshape(-1))
        if q.size != self.dim:
            raise KnnError(f"invalid dimensions: query has {q.size}, index has {self.dim}")
        r = np.ascontiguousarray(np.asarray(rows, dtype=np.uint32).reshape(-1))
        kk = len(r) if k is None else min(int(k), len(r))
        if kk <= 0:
            return np.empty(0, np.uint32), np.empty(0, np.float32)
        idx = np.empty(kk, dtype=np.uint32)
        sc = np.empty(kk, dtype=np.float32)
        ke = _check(self.lib.nk_score_subset(self.ptr, q.ctypes.data_as(C.c_void_p), r.ctypes.data_as(C.c_void_p),
                                             len(r), kk, idx.ctypes.data_as(C.c_void_p),
                                             sc.ctypes.data_as(C.c_void_p)), "nk_score_subset")
        return idx[:ke], sc[:ke]

    # ---- k-means routing on device (pkg/gpu/kmeans.go) ----------------------------------------------------------
    def assign_nearest(self, centroids, assign: np.ndarray, metric: str = "euclidean") -> int:
        """assignToCentroids (euclidean) / assignToCentroidsGPU (cosine): `assign` (int32 [rows]) is updated in place,
        returns the number of changed assignments."""
        c = np.ascontiguousarray(np.asarray(centroids, dtype=np.float32))
        if c.ndim != 2 or c.shape[1] != self.dim:
            raise KnnError(f"invalid dimensions: centroids {c.shape}, index has {self.dim}")
        if assign.dtype != np.int32 or not assign.flags.c_contiguous or assign.size != len(self):
            raise KnnError("assign must be a contiguous int32 array with one entry per row")
        changed = C.c_uint64(0)
        _check(self.lib.nk_index_assign_nearest(self.ptr, c.ctypes.data_as(C.c_void_p), c.shape[0], METRICS[metric],
                                                assign.ctypes.data_as(C.c_void_p), C.byref(changed)), "nk_index_assign_nearest")
        return int(changed.value)

    def cluster_means(self, assign: np.ndarray, centroids) -> Tuple[np.ndarray, np.ndarray]:
        """updateCentroidsWithBuffer: returns (new centroids float32 [K x dim], member counts uint32 [K])."""
        c = np.array(centroids, dtype=np.float32, order="C", copy=True)
        a = np.ascontiguousarray(assign, dtype=np.int32)
        if a.size != len(self):
            raise KnnError("assign must have one entry per row")
        counts = np.zeros(c.shape[0], dtype=np.uint32)
        _check(self.lib.nk_index_cluster_means(self.ptr, a.ctypes.data_as(C.c_void_p), c.shape[0], c.ctypes.data_as(C.c_void_p),
                                               counts.ctypes.data_as(C.c_void_p)), "nk_index_cluster_means")
        return c, counts

    def kmeanspp(self, K: int, first_row: int, u, min_d2: bool = False) -> "KmeansppSeeds":
        """initCentroidsKMeansPlusPlus (kmeans.go:364-426) over every row, on the device: `first_row` plays rand.Intn(n) and
        `u` (K-1 floats in [0, 1)) rand.Float64() for seeds 1 .. K-1.  Returns (seeds uint32 [K], centroids float32 [K x dim],
        potential float64 [K]: the D² total after seeds 0..c, min_d2 float64 [rows] or None, rows_read)."""
        K = int(K)
        uu = np.ascontiguousarray(np.asarray(u, dtype=np.float64).reshape(-1))
        if K < 1 or uu.size != K - 1:
            raise KnnError(f"kmeanspp: K={K} needs K-1 uniforms, got {uu.size}")
        seeds = np.empty(K, dtype=np.uint32)
        cen = np.empty((K, self.dim), dtype=np.float32)
        pot = np.empty(K, dtype=np.float64)
        d2 = np.empty(len(self), dtype=np.float64) if min_d2 else None
        read = C.c_uint64(0)
        _check(self.lib.nk_index_kmeanspp(self.ptr, K, int(first_row), uu.ctypes.data_as(C.c_void_p) if uu.size else None,
                                          seeds.ctypes.data_as(C.c_void_p), cen.ctypes.data_as(C.c_void_p),
                                          pot.ctypes.data_as(C.c_void_p), d2.ctypes.data_as(C.c_void_p) if d2 is not None else None,
                                          C.byref(read)), "nk_index_kmeanspp")
        return KmeansppSeeds(seeds, cen, pot, d2, int(read.value))


class KmeansppSeeds(NamedTuple):
    seeds: np.ndarray
    centroids: np.ndarray
    potential: np.ndarray
    min_d2: Optional[np.ndarray]
    rows_read: int


ALL_BITS = 0xFFFFFFFFFFFFFFFF
ADMIT_NONE = (ALL_BITS, ALL_BITS, 0)  # all_of = none_of = ~0: no row can meet it
ROW_NEW = 0xFFFFFFFF  # NK_ROW_NEW: a row whose contents a k-NN graph never saw


class GraphRowMap:
    """Where each row of an index came from since a k-NN graph of its first n_old rows was built: follow the index's own
    append / update_row / remove_swap on it, then hand it (or src_of_row) to KnnIndex.remap_knn_graph.  src_of_row[f] is
    the old row whose contents row f holds unchanged, or ROW_NEW for appended or rewritten contents."""

    def __init__(self, n_old: int):
        self.n_old = int(n_old)
        self._src = np.arange(self.n_old, dtype=np.uint32)
        self._n = self.n_old

    def __len__(self) -> int:
        return self._n

    @property
    def src_of_row(self) -> np.ndarray:
        return self._src[:self._n].copy()

    def append(self, n_rows: int = 1) -> None:
        n_rows = int(n_rows)
        if self._n + n_rows > self._src.size:
            grown = np.empty(max(self._n + n_rows, 2 * self._src.size), dtype=np.uint32)
            grown[:self._n] = self._src[:self._n]
            self._src = grown
        self._src[self._n:self._n + n_rows] = ROW_NEW
        self._n += n_rows

    def _row(self, row: int) -> int:
        row = int(row)
        if not 0 <= row < self._n:
            raise KnnError(f"GraphRowMap: row {row} out of range ({self._n} rows)")
        return row

    def update_row(self, row: int) -> None:
        """The row's contents changed (update_row).  For a filtered graph, also call it for a row whose tag or filter
        changed, and for a windowed graph for a row whose value key or window changed: the graph treats such a row as
        rewritten."""
        self._src[self._row(row)] = ROW_NEW

    def remove_swap(self, row: int) -> None:
        """nk_index_remove_swap: the last row moves into `row`, and the index shrinks by one"""
        row = self._row(row)
        self._src[row] = self._src[self._n - 1]
        self._n -= 1


def as_filters(filters, Q: int) -> np.ndarray:
    """[Q x 3] uint64 (all_of, none_of, any_of) rows, C-contiguous: the NkFilter array layout."""
    f = np.ascontiguousarray(np.asarray(filters, dtype=np.uint64)).reshape(-1, 3)
    if f.shape[0] != Q:
        raise KnnError(f"filters: {f.shape[0]} rows for {Q} queries")
    return f


def admits(tags, all_of: int, none_of: int, any_of: int):
    """The admissibility predicate of nk_search_filtered on host tag words (numpy; tests, callers' bookkeeping)."""
    t = np.asarray(tags, dtype=np.uint64)
    a, n, s = np.uint64(all_of), np.uint64(none_of), np.uint64(any_of)
    return ((t & a) == a) & ((t & n) == 0) & ((s == 0) | ((t & s) != 0))


SIGN64 = 1 << 63
ADMIT_ALL_WINDOW = (0, ALL_BITS)  # every row, with or without a value
EMPTY_WINDOW = (ALL_BITS, 0)       # lo > hi: no row


def value_keys(values) -> np.ndarray:
    """Numbers -> the uint64 value keys of nk_index_set_row_values, in the same order as the numbers:
      - integers (int64 range): v ^ 2^63;
      - float64, and float32 widened exactly: -0.0 becomes +0.0, then ~bits if the sign bit is set, else bits | 2^63;
      - datetime64: its int64 nanoseconds since the epoch, as an integer.
    Raises on NaN and on INT64_MIN (NaT for datetimes), so key 0 always means "no value": a window with lo >= 1 never admits a
    row that was not given one (Qdrant's rule for a missing key)."""
    a = np.asarray(values)
    if a.dtype.kind == "M":
        a = a.astype("datetime64[ns]").astype(np.int64)
    if a.dtype.kind == "b":
        a = a.astype(np.int64)
    if a.dtype.kind in "iu":
        if a.dtype.kind == "u" and a.size and int(a.max()) > (1 << 63) - 1:
            raise KnnError("value_keys: unsigned value above INT64_MAX")
        v = a.astype(np.int64)
        if (v == np.iinfo(np.int64).min).any():
            raise KnnError("value_keys: INT64_MIN (or NaT) has no key: key 0 means 'no value'")
        return v.view(np.uint64) ^ np.uint64(SIGN64)
    if a.dtype.kind == "f":
        f = a.astype(np.float64)
        if np.isnan(f).any():
            raise KnnError("value_keys: NaN has no key")
        f = np.where(f == 0.0, 0.0, f)  # -0.0 -> +0.0
        b = np.ascontiguousarray(f).view(np.uint64).reshape(f.shape)
        neg = (b >> np.uint64(63)) != 0
        return np.where(neg, ~b, b | np.uint64(SIGN64)).astype(np.uint64)
    raise KnnError(f"value_keys: unsupported dtype {a.dtype}")


_I64_MIN, _I64_MAX = -(1 << 63), (1 << 63) - 1


def _closed_key(x, kind: Optional[str], op: str) -> int:
    """One Qdrant Range bound (op: gt / gte / lt / lte) as the key of the closed bound it implies: the smallest admitted key
    for gt / gte, the largest for lt / lte.  The result may fall outside [1, ALL_BITS] (ALL_BITS + 1 or 0): nothing admitted.
    kind None infers int / float / datetime from the bound itself."""
    if kind is None:
        kind = ("datetime" if isinstance(x, (np.datetime64, _dt.datetime, _dt.date))
                else "float" if isinstance(x, (float, np.floating)) else "int")
    lower = op in ("gt", "gte")
    if kind == "float":
        k = int(value_keys(np.float64(x))[()])  # NaN refused there
        return k + 1 if op == "gt" else k - 1 if op == "lt" else k
    if kind == "datetime":
        t = np.datetime64(x, "ns").astype(np.int64)
        if t == _I64_MIN:
            raise KnnError("window: NaT bound")
        x = int(t)
    elif kind != "int":
        raise KnnError(f"window: unknown kind {kind!r} (int, float or datetime)")
    # integer column: the closed integer bound t, rounded inward when the bound is fractional (Qdrant bounds are doubles)
    if isinstance(x, (float, np.floating)):
        f = float(x)
        if math.isnan(f):
            raise KnnError("window: NaN bound")
        if math.isinf(f):
            return (ALL_BITS + 1 if f > 0 else 1) if lower else (ALL_BITS if f > 0 else 0)
        t = math.floor(f) + 1 if op == "gt" else math.ceil(f) if op == "gte" else math.ceil(f) - 1 if op == "lt" else math.floor(f)
    else:
        t = int(x) + (1 if op == "gt" else -1 if op == "lt" else 0)
    if lower:
        return ALL_BITS + 1 if t > _I64_MAX else max(t, _I64_MIN + 1) + (1 << 63)
    return 0 if t < _I64_MIN + 1 else min(t, _I64_MAX) + (1 << 63)


def window(gt=None, gte=None, lt=None, lte=None, kind: Optional[str] = None) -> Tuple[int, int]:
    """Qdrant Range bounds (gt / gte / lt / lte, any subset; None = open) as the closed key window (lo, hi) of
    search_windowed, over values encoded with value_keys().  kind: "int", "float" or "datetime" — the encoding of the
    indexed values; None infers it from each bound (pass it when, e.g., integer bounds filter a float column).  A strict bound
    steps one key inward; on an int (or datetime) column a fractional bound is rounded inward (gte=2.5 admits 3, lt=2.5
    admits 2).  A bound past either end of the key space gives EMPTY_WINDOW.  Rows without a value (key 0) never match, as
    a missing key never matches a Qdrant range: lo is at least 1."""
    lo, hi = 1, ALL_BITS
    for op, x in (("gt", gt), ("gte", gte), ("lt", lt), ("lte", lte)):
        if x is None:
            continue
        k = _closed_key(x, kind, op)
        if op in ("gt", "gte"):
            lo = max(lo, k)
        else:
            hi = min(hi, k)
    return (lo, hi) if lo <= hi else EMPTY_WINDOW


def as_windows(windows, Q: int) -> np.ndarray:
    """[Q x 2] uint64 (lo, hi) rows, C-contiguous: the NkWindow array layout.  A single (lo, hi) pair applies to every query."""
    w = np.ascontiguousarray(np.asarray(windows, dtype=np.uint64)).reshape(-1, 2)
    if w.shape[0] == 1 and Q != 1:
        w = np.ascontiguousarray(np.broadcast_to(w, (Q, 2)))
    if w.shape[0] != Q:
        raise KnnError(f"windows: {w.shape[0]} rows for {Q} queries")
    return w


NO_GAP = ALL_BITS  # nk_search_pairs_windowed: no band


def _gap_keys(gap) -> int:
    """A band width in key units: an int >= 0 (< NO_GAP), or an np.timedelta64 / datetime.timedelta, in nanoseconds."""
    if isinstance(gap, (np.timedelta64, _dt.timedelta)):
        g = np.timedelta64(gap).astype("timedelta64[ns]").astype(np.int64)
        if g == _I64_MIN:
            raise KnnError("max_gap: NaT")
        gap = int(g)
    elif isinstance(gap, (bool, np.bool_, float, np.floating)) or not isinstance(gap, (int, np.integer)):
        raise KnnError(f"max_gap: an integer number of key units or a timedelta, not {type(gap).__name__}")
    gap = int(gap)
    if gap < 0 or gap >= NO_GAP:
        raise KnnError(f"max_gap: {gap} outside [0, 2^64 - 1)")
    return gap


def band_windows(keys, below, above=None) -> np.ndarray:
    """Per-row value windows [key - below, key + above] (above defaults to below), saturating at 1 and 2^64 - 1, as [n x 2]
    uint64: the windows of a time-local k-NN graph or of "near this row" search_rows calls.  below / above are in key units
    (ints, or np.timedelta64 in nanoseconds for datetime columns, as for search_pairs' max_gap).  A row without a value (key 0)
    gets EMPTY_WINDOW, and no window admits key 0."""
    k = np.asarray(keys, dtype=np.uint64).reshape(-1)
    b = _gap_keys(below)
    a = b if above is None else _gap_keys(above)
    lo = np.where(k > np.uint64(b), k - np.uint64(b), np.uint64(1))
    hi = np.where(k > np.uint64(ALL_BITS - a), np.uint64(ALL_BITS), k + np.uint64(a))
    w = np.stack([lo, hi], axis=1).astype(np.uint64)
    w[k == 0] = EMPTY_WINDOW
    return np.ascontiguousarray(w)


def window_admits(keys, lo: int, hi: int):
    """The window predicate of nk_search_windowed on host value keys (numpy; tests, callers' bookkeeping)."""
    k = np.asarray(keys, dtype=np.uint64)
    return (k >= np.uint64(lo)) & (k <= np.uint64(hi))


def synthetic_tags(n_rows: int, seed: int, row_base: int = 0) -> np.ndarray:
    """Synthetic tag words (bench.py, tests): splitmix64 of (seed, row), so every bit is set with probability 1/2 and a
    row's tag depends only on (seed, row)."""
    with np.errstate(over="ignore"):
        z = (np.arange(row_base, row_base + n_rows, dtype=np.uint64) + np.uint64(seed) * np.uint64(0x9E3779B97F4A7C15))
        z = z * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


class Labels:
    """Maps up to 64 label names (labels, types, collections, keyword values) to tag bits, in order of first use.

        lab = Labels(); ix.set_row_tags(lab.row_tags([["Person"], ["Person", "Admin"], []]))
        ix.search_filtered(q, 10, [lab.filter(must=["Person"], must_not=["Admin"])])
    """

    def __init__(self, names: Sequence[str] = ()):
        self.bits = {}
        for n in names:
            self.bit(n)

    def bit(self, name: str) -> int:
        """The bit of `name`, assigned on first use; a 65th label raises."""
        if name not in self.bits:
            if len(self.bits) >= 64:
                raise KnnError(f"label {name!r}: a tag word holds at most 64 labels")
            self.bits[name] = 1 << len(self.bits)
        return self.bits[name]

    def row_tags(self, labels_per_row) -> np.ndarray:
        """One uint64 tag word per row from an iterable of label collections."""
        out = np.zeros(len(labels_per_row), dtype=np.uint64)
        for r, names in enumerate(labels_per_row):
            w = 0
            for n in names:
                w |= self.bit(n)
            out[r] = w
        return out

    def filter(self, must=(), must_not=(), should=()) -> Tuple[int, int, int]:
        """(all_of, none_of, any_of) of Qdrant-style conditions.  Names never seen: a `must` one admits no row; `must_not`
        ones are ignored; `should` ones are ignored unless every `should` name is unknown (then no row matches)."""
        if any(n not in self.bits for n in must):
            return ADMIT_NONE
        all_of = none_of = any_of = 0
        for n in must:
            all_of |= self.bits[n]
        for n in must_not:
            none_of |= self.bits.get(n, 0)
        known = [n for n in should if n in self.bits]
        if should and not known:
            return ADMIT_NONE
        for n in known:
            any_of |= self.bits[n]
        return all_of, none_of, any_of


def to_bf16_bits(a) -> np.ndarray:
    """fp32 array -> bf16 bit patterns (uint16), round to nearest even (what the device conversion does)."""
    u = np.ascontiguousarray(np.asarray(a, dtype=np.float32)).view(np.uint32)
    r = ((u >> 16) & 1) + np.uint32(0x7FFF)
    return ((u + r) >> 16).astype(np.uint16)


def from_bf16_bits(b) -> np.ndarray:
    return (np.asarray(b, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


class Comm:
    """One rank's exchange context of a row-sharded search (nk_comm_*): candidate lists cross GPUs by peer stores."""

    def __init__(self, device: int, rank: int, world: int, slot_bytes: int):
        self.lib = _lib.load()
        self.rank, self.world = rank, world
        self.ptr = self.lib.nk_comm_create(int(device), int(rank), int(world), int(slot_bytes))
        if not self.ptr:
            raise KnnError(f"nk_comm_create: {_lib.last_error()}")

    def export(self) -> bytes:
        buf = C.create_string_buffer(64)
        _check(self.lib.nk_comm_export(self.ptr, buf), "nk_comm_export")
        return bytes(buf.raw)

    def connect(self, handles: Sequence[bytes]) -> None:
        blob = b"".join(handles)
        assert len(blob) == 64 * self.world
        _check(self.lib.nk_comm_connect(self.ptr, C.c_char_p(blob)), "nk_comm_connect")

    @staticmethod
    def connect_local(comms: Sequence["Comm"]) -> None:
        arr = (C.c_void_p * len(comms))(*[c.ptr for c in comms])
        _check(_lib.load().nk_comm_connect_local(arr, len(comms)), "nk_comm_connect_local")

    def status(self, stream: int = 0) -> None:
        _check(self.lib.nk_comm_status(self.ptr, stream), "nk_comm_status")

    def release(self) -> None:
        if self.ptr:
            self.lib.nk_comm_release(self.ptr)
            self.ptr = None


def blob_vectors(data: bytes) -> Tuple[int, int, int]:
    """(dims, count, byte offset of the fp32 vectors) of a serialized index (gpu.go:2373-2412)."""
    dims, count, off = C.c_uint32(0), C.c_uint32(0), C.c_size_t(0)
    _check(_lib.load().nk_blob_vectors(C.c_char_p(data), len(data), C.byref(dims), C.byref(count), C.byref(off)), "nk_blob_vectors")
    return int(dims.value), int(count.value), int(off.value)


def merge_keys_device(device_id: int, keys_ptr: int, n_lists: int, Q: int, k: int, metric: str, out_idx_ptr: int,
                      out_score_ptr: int, stream: int = 0) -> None:
    _check(_lib.load().nk_merge_keys_device(device_id, keys_ptr, n_lists, Q, k, METRICS[metric], out_idx_ptr,
                                            out_score_ptr, stream), "nk_merge_keys_device")


def fill_uniform_device(device_id: int, out_ptr: int, n_rows: int, dim: int, seed: int, row_base: int = 0,
                        stream: int = 0) -> None:
    _check(_lib.load().nk_fill_uniform_device(device_id, out_ptr, n_rows, dim, seed, row_base, stream),
           "nk_fill_uniform_device")
