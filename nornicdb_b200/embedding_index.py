"""Host-side mirror of gpu.EmbeddingIndex (pkg/gpu/gpu.go:1224-2454) over the fused C ABI.

Same method names / argument meaning / error behaviour as the Go type, so the tests read like
pkg/gpu/gpu_test.go.  Differences, all on purpose (SURVEY.md §8f row 1):
  * the device corpus is kept in step INCREMENTALLY (nk_index_append / update_row / remove_swap) — the
    reference marks gpuSynced=false on every mutation and re-uploads the whole corpus in syncToCUDA
    (gpu.go:2088-2098); SyncToGPU() has nothing to copy.  The OBSERVABLE state machine is kept (gpu_test.go:1403-1480):
    Stats().GPUSynced / IsGPUSynced() turn false on Add / AddBatch / Remove / Clear / Deserialize and true on SyncToGPU();
  * rows stay raw on the device (cosine is computed in the kernel), so ScoreSubset is a device gather +
    fused scan, not a host gather + normalise + re-upload (gpu.go:1578-1589,1945);
  * there is no CPU fallback: without the CUDA library / a GPU every search raises.
Only node-id strings live on the host ("NEVER transferred to GPU", gpu.go:1228-1231)."""
from __future__ import annotations

import ctypes as C
import struct
import threading
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from .knn import KnnError, KnnIndex, blob_vectors


class ErrInvalidDimensions(ValueError):  # gpu.go ErrInvalidDimensions
    def __init__(self):
        super().__init__("gpu: invalid dimensions")


@dataclass
class SearchResult:  # gpu.go SearchResult{ID, Score, Distance}
    ID: str
    Score: float
    Distance: float


@dataclass
class EmbeddingIndexStats:  # gpu.go:2267-2276
    Count: int
    Dimensions: int
    GPUSynced: bool
    SearchesGPU: int
    SearchesCPU: int
    UploadsCount: int
    UploadBytes: int


class EmbeddingIndex:
    def __init__(self, dimensions: int, metric: str = "cosine", devices: Sequence[int] = (0,), dtype: str = "f32"):
        self.dimensions = int(dimensions)
        self.metric = metric
        self.nodeIDs: List[str] = []
        self.idToIndex: Dict[str, int] = {}
        self._ix = KnnIndex(self.dimensions, metric=metric, dtype=dtype, devices=devices)
        self._np_dtype = self._ix.np_dtype
        self._multi = len(devices) > 1
        self.mu = threading.RLock()
        self.searchesGPU = 0
        self.gpuSynced = False  # gpu.go:1260: a fresh index is not synced

    # -- mutation ------------------------------------------------------------------------------------
    def _vec(self, embedding) -> np.ndarray:
        v = np.ascontiguousarray(np.asarray(embedding, dtype=self._np_dtype).reshape(-1))
        if v.size != self.dimensions:
            raise ErrInvalidDimensions()
        return v

    def Add(self, nodeID: str, embedding) -> None:  # gpu.go:1378-1403
        v = self._vec(embedding)
        with self.mu:
            self.gpuSynced = False
            idx = self.idToIndex.get(nodeID)
            if idx is not None:
                self._ix.update_row(idx, v)
            else:
                self._ix.append(v)
                self.nodeIDs.append(nodeID)
                self.idToIndex[nodeID] = len(self.nodeIDs) - 1

    def AddBatch(self, nodeIDs: Sequence[str], embeddings) -> None:  # gpu.go:1406-1434
        if len(nodeIDs) != len(embeddings):
            raise ValueError("gpu: nodeIDs and embeddings length mismatch")
        vecs = [self._vec(e) for e in embeddings]
        with self.mu:
            self.gpuSynced = False
            fresh_ids, fresh = [], []
            pending: Dict[str, int] = {}
            for nid, v in zip(nodeIDs, vecs):
                idx = self.idToIndex.get(nid)
                if idx is not None:
                    self._ix.update_row(idx, v)
                elif nid in pending:
                    fresh[pending[nid]] = v
                else:
                    pending[nid] = len(fresh)
                    fresh_ids.append(nid)
                    fresh.append(v)
            if fresh:
                self._ix.append(np.stack(fresh))
                for nid in fresh_ids:
                    self.nodeIDs.append(nid)
                    self.idToIndex[nid] = len(self.nodeIDs) - 1

    def Remove(self, nodeID: str) -> bool:  # gpu.go:1437-1471 (swap with last)
        with self.mu:
            idx = self.idToIndex.get(nodeID)
            if idx is None:
                return False
            last = len(self.nodeIDs) - 1
            self.gpuSynced = False
            self._ix.remove_swap(idx)
            if idx != last:
                moved = self.nodeIDs[last]
                self.nodeIDs[idx] = moved
                self.idToIndex[moved] = idx
            self.nodeIDs.pop()
            del self.idToIndex[nodeID]
            return True

    def Clear(self) -> None:  # gpu.go:2303-2327
        with self.mu:
            self._ix.upload(np.empty((0, self.dimensions), dtype=self._np_dtype))
            self.nodeIDs = []
            self.idToIndex = {}
            self.gpuSynced = False

    def Release(self) -> None:
        with self.mu:
            self._ix.release()

    # -- queries -------------------------------------------------------------------------------------
    def _results(self, idx: np.ndarray, sc: np.ndarray) -> List[SearchResult]:
        out = []
        for i, s in zip(idx.tolist(), sc.tolist()):
            if i < len(self.nodeIDs):
                out.append(SearchResult(self.nodeIDs[i], float(s), float(1.0 - s)))  # gpu.go:1679-1688
        return out

    def Search(self, query, k: int) -> Optional[List[SearchResult]]:  # gpu.go:1532-1550
        q = np.asarray(query, dtype=np.float32).reshape(-1)
        if q.size != self.dimensions:
            raise ErrInvalidDimensions()
        with self.mu:
            if not self.nodeIDs or k <= 0:
                return None
            self.searchesGPU += 1
            idx, sc = self._ix.search(q, k)
            return self._results(idx[0], sc[0])

    def SearchBatch(self, queries, k: int) -> List[List[SearchResult]]:
        q = np.asarray(queries, dtype=np.float32)
        if q.ndim != 2 or q.shape[1] != self.dimensions:
            raise ErrInvalidDimensions()
        with self.mu:
            if not self.nodeIDs or k <= 0:
                return [[] for _ in range(q.shape[0])]
            self.searchesGPU += 1
            idx, sc = self._ix.search(q, k)
            return [self._results(idx[i], sc[i]) for i in range(q.shape[0])]

    def ScoreSubset(self, query, ids: Sequence[str]) -> Optional[List[SearchResult]]:  # gpu.go:1552-1616
        q = np.asarray(query, dtype=np.float32).reshape(-1)
        if q.size != self.dimensions:
            raise ErrInvalidDimensions()
        if not ids:
            return None
        with self.mu:
            rows = [self.idToIndex[i] for i in ids if i in self.idToIndex]  # missing ids are ignored
            if not rows:
                return None
            if self._multi:
                raise KnnError("ScoreSubset needs a single-device index")
            self.searchesGPU += 1
            idx, sc = self._ix.score_subset(q, rows)
            return self._results(idx, sc)

    def SearchSimilar(self, ids: Sequence[str], k: int) -> List[List[SearchResult]]:
        """The k most similar OTHER nodes of each stored node (FindSimilar, GraphQL `similar`, OnStore's related nodes), best
        first, searched with the node's embedding as stored.  One list per id; an id the index does not hold gets an empty
        list (missing ids are ignored, as in ScoreSubset)."""
        with self.mu:
            out: List[List[SearchResult]] = [[] for _ in ids]
            at = [(i, self.idToIndex[n]) for i, n in enumerate(ids) if n in self.idToIndex]
            if not at or k <= 0:
                return out
            self.searchesGPU += 1
            idx, sc = self._ix.search_rows([r for _, r in at], k)
            for j, (i, _) in enumerate(at):
                out[i] = self._results(idx[j], sc[j])
            return out

    # -- bookkeeping ---------------------------------------------------------------------------------
    def SyncToGPU(self) -> None:  # gpu.go:2025 — nothing to copy: the device rows are always current
        with self.mu:
            self.gpuSynced = True

    def IsGPUSynced(self) -> bool:
        return self.gpuSynced

    def Count(self) -> int:  # gpu.go:2225
        return len(self.nodeIDs)

    def Has(self, nodeID: str) -> bool:  # gpu.go:2279
        return nodeID in self.idToIndex

    def Get(self, nodeID: str) -> Tuple[Optional[np.ndarray], bool]:  # gpu.go:2287
        with self.mu:
            idx = self.idToIndex.get(nodeID)
            if idx is None:
                return None, False
            return self._ix.read_rows(idx, 1)[0], True

    def MemoryUsageMB(self) -> float:
        return len(self.nodeIDs) * self.dimensions * np.dtype(self._np_dtype).itemsize / (1024 * 1024)

    GPUMemoryUsageMB = MemoryUsageMB

    def Stats(self) -> EmbeddingIndexStats:  # gpu.go:2252-2276
        st = self._ix.stats()
        return EmbeddingIndexStats(len(self.nodeIDs), self.dimensions, self.gpuSynced, self.searchesGPU, 0,
                                   st["searches"], st["bytes_h2d"])

    # -- checkpoint (gpu.go:2373-2454): LE [dims u32][count u32][len-prefixed ids...][float32 vectors...] ------
    def Serialize(self) -> bytes:
        with self.mu:
            n = len(self.nodeIDs)
            parts = [struct.pack("<II", self.dimensions, n)]
            for nid in self.nodeIDs:
                b = nid.encode("utf-8")
                parts.append(struct.pack("<I", len(b)))
                parts.append(b)
            if n:
                parts.append(self._ix.read_rows(0, n).astype("<f4").tobytes())
            return b"".join(parts)

    def Deserialize(self, data: bytes) -> None:
        if len(data) < 8:
            raise ValueError("gpu: invalid serialized data")
        dims, count = struct.unpack_from("<II", data, 0)
        if dims != self.dimensions:
            raise ErrInvalidDimensions()
        off = 8
        ids = []
        for _ in range(count):
            (ln,) = struct.unpack_from("<I", data, off)
            off += 4
            ids.append(data[off:off + ln].decode("utf-8"))
            off += ln
        _, _, voff = blob_vectors(data)  # validates the table and the payload length
        assert voff == off
        with self.mu:
            # the fp32 payload (arbitrarily aligned inside the blob) streams straight to device memory through the
            # library's pinned double buffer; an fp16 index converts on the device while loading
            base = C.cast(C.c_char_p(data), C.c_void_p).value
            self._ix.upload_from_f32(ptr=base + voff, n_rows=count)
            self.gpuSynced = False  # gpu.go:2452
            self.nodeIDs = ids
            self.idToIndex = {nid: i for i, nid in enumerate(ids)}
