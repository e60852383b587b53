"""A long-lived index against an fp64 model: seeded mutation scripts across shard layouts, every search path after each step.

Every per-row array of an index has to follow its row through append, update_row and remove_swap: the rows, the BF16 shadow
or int8 image with their norms (fp32 shards), |x|^2 (16-bit shards), tags and value keys.  Model is a plain numpy index that
follows the documented rules (remove_swap moves the last row, its tag and its key into the slot; append and remove drop the row
mask; upload resets tags and keys; appended rows get tag 0 and key 0) and answers every search by fp64 brute force.  It also
follows the shard layout (repartition: shard g of G holds rows [ng/G, n(g+1)/G) with exactly that capacity after an upload;
append writes to the last shard, remove_swap shrinks the last non-empty one), so build_script can place each edge on purpose:
a regrowth that reallocates the last shard's images, an append that fits, rewrites of the first and last row of every shard,
a removal whose moved row crosses shards (and devices on (0, 1)), removals that empty the trailing shard and an append into
it, tag and value ranges that straddle a boundary, the row mask and the score floor set after mutations, and a metric change.

After every step:
  - images (single shard): the maintained index's filter dumps ("shadow", and "filter" for fp32) equal those of a fresh
    upload of the model's rows bit for bit, and every estimate is within its bound of the fp64 score;
  - results: AUTO and every forced path of search, search_filtered, search_windowed, search_range, search_rows (plain and
    windowed), search_pairs (plain and windowed) and score_subset agree with the fp64 model under the parity rule
    (tests/parity.py) or the fp64 band (test_gpu_range.check_range), and equal a fresh single-shard index of the model's
    rows on the same path bit for bit.  Planted queries are near-copies of each row the step rewrote or moved; the exact
    contents of each removed row are queried too, and must come back under no id;
  - graph: the plain, filtered and windowed k-NN graphs carried forward with remap_knn_graph (GraphRowMap) equal the
    search_rows rebuild bit for bit and the model's graph under the parity rule.

The harness takes the index factory as an argument, so tests/test_index_lifecycle_cpu.py runs it end to end with
ModelIndex (the model answering as the device) where there is no GPU."""
from __future__ import annotations

from typing import Callable, List, NamedTuple, Optional, Sequence

import numpy as np
import pytest

from parity import check_parity
from test_gpu_range import check_range, fp64_keys, key_threshold
from test_gpu_search_pairs import BAND

pytestmark = pytest.mark.gpu

PAD = 0xFFFFFFFF
K = 10
TAG_BITS = 3
GRAPH_FILTER = (0, 4, 0)  # every list of the filtered graph refuses rows with tag bit 2
QUERY_FILTERS = [(0, 0, 0), (1, 0, 0), (0, 2, 0), (0, 0, 6)]  # none, all_of bit 0, none_of bit 1, any_of bits 1 | 2
VALUE_RANGE = 1000       # value keys encode ints in [0, VALUE_RANGE)
BAND_BELOW = 200         # windows of search_rows and the windowed graph: [value - 200, value + 200]
PAIR_GAP = 300           # band of the windowed self-join
METRICS = ("cosine", "dot", "euclidean")


# ---- the fp64 model ----------------------------------------------------------------------------------------------------
def rounded(rows, dtype):
    """rows as the index stores them, widened exactly to fp32"""
    from nornicdb_b200.knn import from_bf16_bits, to_bf16_bits
    a = np.asarray(rows, dtype=np.float32)
    if dtype == "f16":
        return a.astype(np.float16).astype(np.float32)
    if dtype == "bf16":
        return from_bf16_bits(to_bf16_bits(a))
    return a.copy()


def int_values(keys):
    """value keys of ints back to their ints (v ^ 2^63); meaningful where key != 0"""
    from nornicdb_b200.knn import SIGN64
    return (np.asarray(keys, dtype=np.uint64) ^ np.uint64(SIGN64)).view(np.int64)


class Model:
    """The index as documented, in numpy.  x: the rows as stored (fp32 holding f16 / bf16 values exactly); tags, keys: uint64
    per row; mask: bool per row or None; floor: the score floor in the API's domain or None.  shard_n / shard_cap follow the
    layout rules of repartition, nk_index_append and nk_index_remove_swap; edges records which named edges the operations
    reached; moved marks rows whose contents changed since the last clear_marks (rewritten, appended or moved into); intent is
    a mask bit that travels with its row, for setting the mask again after mutations."""

    def __init__(self, dim, dtype, metric, n_devices):
        self.dim, self.dtype, self.metric, self.G = int(dim), dtype, metric, int(n_devices)
        self.x = np.empty((0, self.dim), np.float32)
        self.tags = np.empty(0, np.uint64)
        self.keys = np.empty(0, np.uint64)
        self.intent = np.empty(0, bool)
        self.moved = np.empty(0, bool)
        self.mask: Optional[np.ndarray] = None
        self.floor: Optional[float] = None
        self.shard_n = [0] * self.G
        self.shard_cap = [0] * self.G
        self.edges = set()
        self.removed: List[np.ndarray] = []  # contents removed since clear_marks
        self.mutated = False                 # a row-changing call since the last set_row_mask / set_min_score

    def __len__(self):
        return self.x.shape[0]

    # -- layout
    def shard_of(self, row):
        """(shard, local row) of a global row: rows are ordered shard by shard"""
        b = 0
        for g, n in enumerate(self.shard_n):
            if row < b + n:
                return g, row - b
            b += n
        raise IndexError(row)

    def shard_first_rows(self):
        return np.cumsum([0] + self.shard_n[:-1]).tolist()

    # -- mutations
    def upload(self, rows, intent):
        n = len(rows)
        self.x = rounded(rows, self.dtype)
        self.tags = np.zeros(n, np.uint64)
        self.keys = np.zeros(n, np.uint64)
        self.intent = np.asarray(intent, bool).copy()
        self.moved = np.zeros(n, bool)
        self.mask = None
        self.shard_n = [n * (g + 1) // self.G - n * g // self.G for g in range(self.G)]
        self.shard_cap = [max(c, 16) for c in self.shard_n]  # shard_reserve_rows(keep = false) on an empty shard

    def append(self, rows, intent):
        m = len(rows)
        g = self.G - 1
        need = self.shard_n[g] + m
        if need > self.shard_cap[g]:
            self.shard_cap[g] = max(need, self.shard_cap[g] + self.shard_cap[g] // 2, 16)  # keep = true
            self.edges.add("regrow")
        else:
            self.edges.add("append_fits")
        if self.G > 1 and self.shard_n[g] == 0:
            self.edges.add("append_into_emptied_shard")
        self.shard_n[g] = need
        self.x = np.concatenate([self.x, rounded(rows, self.dtype)])
        self.tags = np.concatenate([self.tags, np.zeros(m, np.uint64)])
        self.keys = np.concatenate([self.keys, np.zeros(m, np.uint64)])
        self.intent = np.concatenate([self.intent, np.asarray(intent, bool)])
        self.moved = np.concatenate([self.moved, np.ones(m, bool)])
        self.mask = None
        self.mutated = True

    def update_row(self, row, vec):
        g, local = self.shard_of(row)
        if local == 0:
            self.edges.add("update_shard_first")
        if local == self.shard_n[g] - 1:
            self.edges.add("update_shard_last")
        if row == len(self) - 1:
            self.edges.add("update_index_last")
        self.x[row] = rounded(np.asarray(vec).reshape(1, -1), self.dtype)[0]
        self.moved[row] = True
        self.mutated = True

    def remove_swap(self, row):
        last = len(self) - 1
        g_last, _ = self.shard_of(last)  # the last non-empty shard holds the last row
        g_row, _ = self.shard_of(row)
        self.removed.append(self.x[row].copy())
        if row != last:
            self.edges.add("cross_shard_move" if g_row != g_last else "same_shard_move")
            for a in (self.x, self.tags, self.keys, self.intent):
                a[row] = a[last]
            self.moved[row] = True
        else:
            self.edges.add("remove_last")
        self.x, self.tags, self.keys = self.x[:-1], self.tags[:-1], self.keys[:-1]
        self.intent, self.moved = self.intent[:-1], self.moved[:-1]
        self.shard_n[g_last] -= 1
        if self.G > 1 and self.shard_n[g_last] == 0 and g_last == self.G - 1:
            self.edges.add("trailing_shard_emptied")
        self.mask = None
        self.mutated = True

    def _straddles(self, first, count, what):
        if count and self.shard_of(first)[0] != self.shard_of(first + count - 1)[0]:
            self.edges.add(f"{what}_straddle_shards")

    def set_row_tags(self, first, tags):
        self._straddles(first, len(tags), "tags")
        self.tags[first:first + len(tags)] = tags

    def set_row_values(self, first, keys):
        self._straddles(first, len(keys), "values")
        self.keys[first:first + len(keys)] = keys

    def set_row_mask(self, keep):
        if self.mutated:
            self.edges.add("mask_after_mutation")
        self.mask = np.asarray(keep, bool).copy()

    def set_min_score(self, floor):
        if self.mutated:
            self.edges.add("floor_after_mutation")
        self.floor = floor

    def set_metric(self, metric):
        self.edges.add("set_metric")
        self.metric = metric

    def clear_marks(self):
        self.moved[:] = False
        self.removed = []
        self.mutated = False

    # -- fp64 answers
    def scores(self, q):
        """[Q, n] fp64 scores in the API's domain (euclidean: distances)"""
        x = self.x.astype(np.float64)
        qq = np.asarray(q, dtype=np.float64).reshape(-1, self.dim)
        dots = qq @ x.T
        if self.metric == "dot":
            return dots
        xn = np.linalg.norm(x, axis=1)[None, :]
        qn = np.linalg.norm(qq, axis=1)[:, None]
        if self.metric == "cosine":
            den = qn * xn
            with np.errstate(invalid="ignore", divide="ignore"):
                return np.where(den > 0, dots / den, 0.0)
        return np.sqrt(np.maximum(qn ** 2 + xn ** 2 - 2.0 * dots, 0.0))

    def floor_ok(self, S):
        if self.floor is None:
            return np.ones(S.shape, bool)
        return S <= self.floor if self.metric == "euclidean" else S >= self.floor

    def row_ok(self):
        return np.ones(len(self), bool) if self.mask is None else self.mask

    def admissible(self, Q, filters=None, windows=None):
        """[Q, n]: the row mask, then per-query tag filters ([Q x 3]) and value windows ([Q x 2])"""
        from nornicdb_b200.knn import admits
        adm = np.tile(self.row_ok(), (Q, 1))
        if filters is not None:
            for qi, (a, b, c) in enumerate(np.asarray(filters, np.uint64).reshape(-1, 3)):
                adm[qi] &= admits(self.tags, int(a), int(b), int(c))
        if windows is not None:
            for qi, (lo, hi) in enumerate(np.asarray(windows, np.uint64).reshape(-1, 2)):
                adm[qi] &= (self.keys >= lo) & (self.keys <= hi)
        return adm

    def topk(self, S, adm, k):
        """the best k admissible rows per query: score desc (distance asc), then row asc -> [(idx, fp64 score)]"""
        ok = adm & np.isfinite(S) & self.floor_ok(S)
        out = []
        for qi in range(S.shape[0]):
            c = np.nonzero(ok[qi])[0]
            s = S[qi, c]
            o = np.lexsort((c, s if self.metric == "euclidean" else -s))[:k]
            out.append((c[o], s[o]))
        return out


# ---- operation scripts -------------------------------------------------------------------------------------------------
class Case(NamedTuple):
    name: str
    dtype: str
    image: Optional[str]       # NK_SHADOW at creation (None: unset)
    devices: Sequence[int]
    dim: int
    n: int
    metric: str
    big: bool = False           # large enough for AUTO to serve k <= 16 from the int8 image: no graph, a stripe of pairs


def has_image(case):
    """does a shard of this case carry a scan image (shard_sync_shadow's shape rule)?"""
    return case.dim >= 32 and (case.dim % 4 == 0 if case.dtype == "f32" else case.dim % 8 == 0)


def knn_paths(case, metric):
    p = ["auto", "simt"]
    if case.dtype == "f32":
        p += ["filter"] + (["tensor"] if metric != "euclidean" else [])
    if has_image(case):
        p.append("shadow")
    return p


def graph_path(case):
    """the path a k-NN graph is kept on; None: the index has no filter path (16-bit rows without an image), so a graph is
    only rebuilt there, never carried forward"""
    return "shadow" if has_image(case) else "filter" if case.dtype == "f32" else None


def build_script(case, seed=0):
    """-> (steps, model): steps[0] sets the index up, each later step is one batch of operations; model is the Model after
    the whole script (its edges name what the script reached).  Each step is a list of (op, *args) tuples."""
    from nornicdb_b200.knn import value_keys
    rng = np.random.default_rng([seed, case.n, case.dim, len(case.devices)])
    m = Model(case.dim, case.dtype, case.metric, len(case.devices))
    d = case.dim
    steps = []

    def rows(cnt):
        return rng.standard_normal((cnt, d)).astype(np.float32)

    def op(step, *a):
        step.append(a)
        getattr(m, {"upload": "upload", "append": "append", "update": "update_row", "remove": "remove_swap",
                    "tags": "set_row_tags", "values": "set_row_values", "mask": "set_row_mask", "floor": "set_min_score",
                    "metric": "set_metric"}[a[0]])(*a[1:])

    def tags(cnt):
        return rng.integers(0, 1 << TAG_BITS, cnt).astype(np.uint64)

    def values(cnt):
        v = value_keys(rng.integers(0, VALUE_RANGE, cnt).astype(np.int64))
        v[rng.random(cnt) < 0.1] = 0  # some rows without a value
        return v

    def intent(cnt):
        return rng.random(cnt) > 0.15

    def floor_for(metric):
        """a floor that cuts the lists of random queries short (rows and queries are standard normal, the random queries a
        row plus unit noise): about 2.5 standard deviations into the tail of their scores"""
        return float({"cosine": 2.5 / np.sqrt(d), "dot": 2.5 * np.sqrt(2.0 * d),
                      "euclidean": np.sqrt(3.0 * d - 2.5 * np.sqrt(18.0 * d))}[metric])

    # 0: upload, tags and values on every row, the mask and a floor
    s = []
    op(s, "upload", rows(case.n), intent(case.n))
    op(s, "tags", 0, tags(case.n))
    op(s, "values", 0, values(case.n))
    op(s, "mask", m.intent.copy())
    op(s, "floor", floor_for(m.metric))
    steps.append(s)

    # 1: the first append regrows the last shard (its capacity is exactly its rows after an upload), a second one fits
    s = []
    op(s, "append", rows(5), intent(5))
    op(s, "append", rows(2), intent(2))
    op(s, "mask", m.intent.copy())
    steps.append(s)

    # 2: rewrite the first and last row of every shard and the last row of the index; retag and revalue ranges that
    # straddle every shard boundary
    s = []
    targets = []
    for f, c in zip(m.shard_first_rows(), m.shard_n):
        if c:
            targets += [f, f + c - 1]
    for r in sorted(set(targets + [len(m) - 1])):
        v = rows(1)[0]
        if r % 3 == 0:  # some rewrites are near-copies of another row: near ties with an unchanged row
            v = m.x[(r + 7) % len(m)] + np.float32(1e-3) * v
        op(s, "update", r, v)
    for b in m.shard_first_rows()[1:] or [len(m) // 2]:
        op(s, "tags", max(b - 3, 0), tags(6))
        op(s, "values", max(b - 4, 0), values(8))
    op(s, "mask", m.intent.copy())
    steps.append(s)

    # 3: remove the last row, then a row of shard 0 (the last row lives in another shard when there are several) and one in
    # the middle of the index
    s = []
    op(s, "remove", len(m) - 1)
    op(s, "remove", 3)
    op(s, "remove", len(m) // 2)
    op(s, "mask", m.intent.copy())
    steps.append(s)

    # 4: several shards: removals empty the trailing shard (rows taken from anywhere, the last row moving into them), two
    # more come from the shard before it, then an append lands in the empty trailing shard.  One shard (or a case that
    # must stay large): a few removals and appends.
    s = []
    if m.G > 1 and not case.big:
        while m.shard_n[-1] > 0:
            op(s, "remove", int(rng.integers(len(m))))
        op(s, "remove", int(rng.integers(len(m))))
        op(s, "remove", len(m) - 1)
        op(s, "append", rows(4), intent(4))
    else:
        for _ in range(12):
            op(s, "remove", int(rng.integers(len(m))))
        op(s, "append", rows(3), intent(3))
    op(s, "tags", len(m) - 4, tags(4))
    op(s, "mask", m.intent.copy())
    steps.append(s)

    # 5: another metric, then interleaved rewrites, removals, appends and retags; the mask and a new floor after them
    s = []
    nxt = METRICS[(METRICS.index(m.metric) + 1) % 3]
    op(s, "metric", nxt)
    for _ in range(24):
        u = rng.random()
        if u < 0.35:
            op(s, "update", int(rng.integers(len(m))), rows(1)[0])
        elif u < 0.7:
            op(s, "remove", int(rng.integers(len(m))))
        elif u < 0.85:
            op(s, "append", rows(2), intent(2))
        else:
            f = int(rng.integers(len(m) - 5))
            op(s, "values" if u < 0.93 else "tags", f, values(5) if u < 0.93 else tags(5))
    op(s, "mask", m.intent.copy())
    op(s, "floor", floor_for(nxt))
    steps.append(s)
    return steps, m


def required_edges(case):
    e = {"regrow", "append_fits", "update_shard_first", "update_shard_last", "update_index_last", "remove_last",
         "same_shard_move", "mask_after_mutation", "floor_after_mutation", "set_metric"}
    if len(case.devices) > 1:
        e |= {"cross_shard_move", "tags_straddle_shards", "values_straddle_shards"}
        if not case.big:
            e |= {"trailing_shard_emptied", "append_into_emptied_shard"}
    return e


# ---- the model answering as the device ---------------------------------------------------------------------------------
class ModelIndex:
    """The KnnIndex calls the harness makes, answered by a Model in fp64 and rounded to fp32 (CPU runs of the harness)."""

    def __init__(self, dim, metric="cosine", dtype="f32", devices=(0,)):
        self.m = Model(dim, dtype, metric, len(devices))
        self.dim, self.metric, self.path = int(dim), metric, "auto"

    def release(self):
        pass

    def __len__(self):
        return len(self.m)

    def upload(self, rows):
        self.m.upload(rows, np.ones(len(rows), bool))

    def append(self, rows):
        self.m.append(rows, np.ones(len(rows), bool))

    def update_row(self, row, vec):
        self.m.update_row(row, vec)

    def remove_swap(self, row):
        self.m.remove_swap(row)

    def set_row_tags(self, tags, first_row=0):
        self.m.set_row_tags(first_row, np.asarray(tags, np.uint64))

    def set_row_values(self, values, first_row=0):
        self.m.set_row_values(first_row, np.asarray(values, np.uint64))

    def set_row_mask(self, keep):
        self.m.mask = None if keep is None else np.asarray(keep, bool).copy()

    def set_min_score(self, v):
        self.m.floor = v

    def set_metric(self, metric):
        self.m.metric = self.metric = metric

    def set_path(self, path):
        self.path = path

    def last_path(self):
        return "shadow" if self.path == "auto" else self.path

    def _lists(self, S, adm, k):
        res = self.m.topk(S, adm, k)
        w = min(k, max([len(i) for i, _ in res] + [0]))
        idx = np.full((len(res), w), PAD, np.uint32)
        sc = np.zeros((len(res), w), np.float32)
        for qi, (i, s) in enumerate(res):
            idx[qi, :len(i)] = i
            sc[qi, :len(i)] = s
        return idx, sc

    def search(self, q, k):
        return self.search_windowed(q, k, None, None)

    def search_filtered(self, q, k, filters):
        return self.search_windowed(q, k, None, filters)

    def search_windowed(self, q, k, windows, filters=None):
        q = np.asarray(q, np.float32).reshape(-1, self.dim)
        return self._lists(self.m.scores(q), self.m.admissible(len(q), filters, windows), k)

    def search_rows(self, rows, k, filters=None, windows=None):
        r = np.asarray(rows, np.int64)
        adm = self.m.admissible(len(r), filters, windows)
        adm[np.arange(len(r)), r] = False
        return self._lists(self.m.scores(self.m.x[r]), adm, k)

    def search_range(self, q, thresholds, filters=None, windows=None):
        q = np.asarray(q, np.float32).reshape(-1, self.dim)
        t = np.broadcast_to(np.asarray(thresholds, np.float64), (len(q),))
        S = self.m.scores(q)
        adm = self.m.admissible(len(q), filters, windows) & self.m.floor_ok(S)
        out = []
        for qi in range(len(q)):
            ok = adm[qi] & ((S[qi] <= t[qi]) if self.metric == "euclidean" else (S[qi] >= t[qi]))
            c = np.nonzero(ok)[0]
            o = np.lexsort((c, S[qi, c] if self.metric == "euclidean" else -S[qi, c]))
            out.append((c[o].astype(np.uint32), S[qi, c[o]].astype(np.float32)))
        return out

    def search_pairs(self, threshold, first_row=0, n_rows=None, filter=None, window=None, max_gap=None):
        from nornicdb_b200.knn import admits
        n = len(self.m)
        n_rows = n - first_row if n_rows is None else n_rows
        ok_row = self.m.row_ok().copy()
        if filter is not None:
            ok_row &= admits(self.m.tags, *[int(v) for v in filter])
        res = self.search_range(self.m.x[first_row:first_row + n_rows], threshold)
        off, idx, sc = [0], [], []
        v = int_values(self.m.keys)
        for r, (i, s) in enumerate(res):
            row = first_row + r
            keep = (i.astype(np.int64) > row) & ok_row[i] & ok_row[row]
            if max_gap is not None:
                keep &= (self.m.keys[i] != 0) & (self.m.keys[row] != 0) & (np.abs(v[i] - v[row]) <= max_gap)
            idx.append(i[keep])
            sc.append(s[keep])
            off.append(off[-1] + int(keep.sum()))
        return (np.asarray(off, np.uint64), np.concatenate(idx).astype(np.uint32) if idx else np.empty(0, np.uint32),
                np.concatenate(sc).astype(np.float32) if sc else np.empty(0, np.float32))

    def score_subset(self, q, rows, k=None):
        r = np.asarray(rows, np.int64)
        S = Model.scores(self.m, q)[0, r]
        o = np.lexsort((np.arange(len(r)), S if self.metric == "euclidean" else -S))[:k]
        return r[o].astype(np.uint32), S[o].astype(np.float32)

    def remap_knn_graph(self, gi, gs, n_old, src, k=None, filters=None, windows=None):
        ui, us = self.search_rows(np.arange(len(self.m)), k or gi.shape[1], filters, windows)
        return ui, us, 0

    def update_knn_graph(self, gi, gs, n_old, changed=None, k=None, filters=None, windows=None):
        return self.remap_knn_graph(gi, gs, n_old, None, k, filters, windows)

    def filter_dump(self, q, which="shadow"):
        keys, _ = fp64_keys(self.m.x, np.asarray(q, np.float32).reshape(-1, self.dim), self.metric)
        return keys.T.astype(np.float32), np.full(keys.T.shape, 1e-3, np.float32)


# ---- checks ------------------------------------------------------------------------------------------------------------
def same_bits(a, b, what):
    """two results of one call (tuples of arrays, or range lists of them) are identical, score bits included"""
    if isinstance(a, list):
        assert len(a) == len(b), what
        for qi, (x, y) in enumerate(zip(a, b)):
            same_bits(x, y, f"{what} query {qi}")
        return
    for x, y in zip(a, b):
        x, y = np.asarray(x), np.asarray(y)
        assert x.shape == y.shape, (what, x.shape, y.shape)
        if x.dtype == np.float32:
            x, y = x.view(np.uint32), y.view(np.uint32)
        bad = np.argwhere(x != y)
        assert bad.size == 0, (what, bad[:4].tolist())


def check_lists(model, queries, got, want, what):
    """kNN lists (idx [Q x w] with PAD after the last real slot, scores) against the model's fp64 top-k, parity rule"""
    gi, gs = got
    for qi, (ei, es) in enumerate(want):
        row = gi[qi]
        real = row != PAD
        nr = int(real.sum())
        assert real[:nr].all(), (what, qi, "a pad before a real slot", row)
        assert nr == len(ei), (what, qi, f"{nr} rows listed, the model has {len(ei)} admissible", row, ei)
        if nr == 0:
            continue
        if (row[:nr] == ei).all() and (np.abs(gs[qi, :nr] - es) <= 1e-4 * np.abs(es) + 1e-6).all():
            continue
        try:
            check_parity(model.x, queries[qi:qi + 1], nr, model.metric, row[None, :nr], gs[qi:qi + 1, :nr], ei[None, :], es[None, :])
        except AssertionError as e:
            raise AssertionError(f"{what}, query {qi}: {e}") from None


def check_pairs(model, res, first, n_rows, t, adm_row, max_gap=None):
    """a self-join stripe against fp64 over every pair j > i of admissible rows, outside the band of check_range"""
    off, idx, _ = res
    x = model.x
    keys, scale = fp64_keys(x, x[first:first + n_rows], model.metric)
    tk = key_threshold(float(t), model.metric)
    n = len(x)
    rows = np.arange(first, first + n_rows)
    ok = (np.arange(n)[None, :] > rows[:, None]) & np.isfinite(keys) & (keys >= tk) & adm_row[rows][:, None] & adm_row[None, :]
    if max_gap is not None:
        v = int_values(model.keys)
        has = model.keys != 0
        ok &= has[rows][:, None] & has[None, :] & (np.abs(v[rows][:, None] - v[None, :]) <= max_gap)
    in_band = np.isfinite(keys) & (np.abs(keys - tk) <= BAND * scale)
    got = np.zeros(ok.shape, bool)
    for r in range(n_rows):
        got[r, idx[int(off[r]):int(off[r + 1])].astype(np.int64)] = True
    assert not (got & ~ok & ~in_band).any(), ("pairs that should not be listed", np.argwhere(got & ~ok & ~in_band)[:4])
    assert not (ok & ~got & ~in_band).any(), ("pairs missing", np.argwhere(ok & ~got & ~in_band)[:4])


class Lifecycle:
    """One case: the index under test, the model, the k-NN graphs carried forward, and the checks after each step."""

    def __init__(self, case, make: Callable, seed=0, images=True):
        self.case, self.make, self.images = case, make, images
        self.steps, _ = build_script(case, seed)
        self.rng = np.random.default_rng([seed, 99, case.n])
        self.model = Model(case.dim, case.dtype, case.metric, len(case.devices))
        self.ix = make(case.devices, case.metric)
        self.graph = None  # (gi, gs per kind, GraphRowMap, (metric, floor) it was built under)

    def close(self):
        self.ix.release()

    def apply(self, a):
        ix, m = self.ix, self.model
        kind = a[0]
        g = self.graph
        if kind == "upload":
            ix.upload(a[1]); m.upload(a[1], a[2])
        elif kind == "append":
            ix.append(a[1]); m.append(a[1], a[2])
            if g: g[1].append(len(a[1]))
        elif kind == "update":
            ix.update_row(a[1], a[2]); m.update_row(a[1], a[2])
            if g: g[1].update_row(a[1])
        elif kind == "remove":
            ix.remove_swap(a[1]); m.remove_swap(a[1])
            if g: g[1].remove_swap(a[1])
        elif kind in ("tags", "values"):
            first, w = a[1], a[2]
            old = (m.tags if kind == "tags" else m.keys)[first:first + len(w)].copy()
            (ix.set_row_tags if kind == "tags" else ix.set_row_values)(w, first)
            (m.set_row_tags if kind == "tags" else m.set_row_values)(first, w)
            if g:  # a retag or a revalue is a rewrite to the filtered and windowed graphs
                for r in np.nonzero(old != w)[0]:
                    g[1].update_row(first + int(r))
        elif kind == "mask":
            ix.set_row_mask(a[1]); m.set_row_mask(a[1])
        elif kind == "floor":
            ix.set_min_score(a[1]); m.set_min_score(a[1])
        elif kind == "metric":
            ix.set_metric(a[1]); m.set_metric(a[1])
        else:
            raise ValueError(kind)

    def run(self, n_steps=None):
        for si, step in enumerate(self.steps[:n_steps]):
            for a in step:
                self.apply(a)
            self.check(si)
            self.model.clear_marks()

    # -- one step's checks
    def fresh(self):
        """a single-shard index of the model's rows, tags, keys, mask, floor and metric"""
        m = self.model
        f = self.make((0,), m.metric)
        f.upload(m.x)
        f.set_row_tags(m.tags)
        f.set_row_values(m.keys)
        if m.mask is not None:
            f.set_row_mask(m.mask)
        f.set_min_score(m.floor)
        return f

    def queries(self):
        """planted near-copies of every row the step rewrote or moved, each removed row's exact contents, random rows"""
        m = self.model
        moved = np.nonzero(m.moved)[0]
        if len(moved) > 24:
            moved = self.rng.choice(moved, 24, replace=False)
        near = m.x[moved] * np.float32(1.0) + np.float32(1e-2) * self.rng.standard_normal((len(moved), m.dim)).astype(np.float32) * \
            np.linalg.norm(m.x[moved], axis=1, keepdims=True).astype(np.float32) / np.float32(np.sqrt(m.dim))
        gone = np.asarray(m.removed[:8], np.float32).reshape(-1, m.dim)
        rnd = m.x[self.rng.integers(0, len(m), 6)] + self.rng.standard_normal((6, m.dim)).astype(np.float32)
        q = np.concatenate([near, gone, rnd]).astype(np.float32)[:60]
        return q, moved, len(near), len(gone)

    def check(self, si):
        case, m, ix = self.case, self.model, self.ix
        q, moved, n_near, n_gone = self.queries()
        Q = len(q)
        filters = np.asarray([QUERY_FILTERS[i % len(QUERY_FILTERS)] for i in range(Q)], np.uint64)
        from nornicdb_b200.knn import band_windows, value_keys
        lo = self.rng.integers(0, VALUE_RANGE // 2, Q)
        windows = np.stack([value_keys(lo.astype(np.int64)), value_keys((lo + VALUE_RANGE // 3).astype(np.int64))], 1)
        S = m.scores(q)
        want_plain = m.topk(S, m.admissible(Q), K)
        want_filt = m.topk(S, m.admissible(Q, filters), K)
        want_win = m.topk(S, m.admissible(Q, filters, windows), K)
        keys, scale = fp64_keys(m.x, q, m.metric)
        ranks = [1, 5, 40]
        thr = np.empty(Q, np.float32)
        for qi in range(Q):
            v = np.sort(keys[qi][np.isfinite(keys[qi])])[::-1]
            kk = v[min(ranks[qi % 3], len(v)) - 1]
            thr[qi] = np.sqrt(-kk) if m.metric == "euclidean" else kk
        adm_range = m.admissible(Q, filters) & m.floor_ok(S)
        # search by stored row: the rows the step touched, the first and last row of each shard, a few others
        firsts = [f for f, c in zip(m.shard_first_rows(), m.shard_n) if c]
        lasts = [f + c - 1 for f, c in zip(m.shard_first_rows(), m.shard_n) if c]
        rq = np.unique(np.concatenate([moved, firsts, lasts, self.rng.integers(0, len(m), 6)]).astype(np.int64))
        rwin = band_windows(m.keys[rq], BAND_BELOW)
        Sr = m.scores(m.x[rq])
        adm_r = m.admissible(len(rq))
        adm_r[np.arange(len(rq)), rq] = False
        adm_rw = m.admissible(len(rq), None, rwin)
        adm_rw[np.arange(len(rq)), rq] = False
        want_rows, want_rows_w = m.topk(Sr, adm_r, K), m.topk(Sr, adm_rw, K)
        # the self-join: the whole index, or a stripe over the touched region of a large one
        first, n_rows = (0, len(m)) if not case.big else (max(int(moved.min()) - 8, 0) if len(moved) else 0, 48)
        n_rows = min(n_rows, len(m) - first)
        pk, _ = fp64_keys(m.x, m.x[first:first + n_rows], m.metric)
        off_diag = pk[np.arange(len(m))[None, :] > np.arange(first, first + n_rows)[:, None]]
        pt_key = np.quantile(off_diag[np.isfinite(off_diag)], 1.0 - 4.0 / len(m))
        pt = np.float32(np.sqrt(-pt_key) if m.metric == "euclidean" else pt_key)
        if m.floor is not None:  # the join keeps to the stricter of its threshold and the floor
            pt = np.float32(min(pt, m.floor) if m.metric == "euclidean" else max(pt, m.floor))
        from nornicdb_b200.knn import admits
        pair_filter = (0, 1, 0)
        adm_pairs = m.row_ok() & admits(m.tags, *pair_filter)

        fresh = self.fresh()
        try:
            for path in knn_paths(case, m.metric):
                ix.set_path(path); fresh.set_path(path)

                def both(fn, what):
                    a = fn(ix)
                    if path != "auto":
                        assert ix.last_path() == path, (what, path, ix.last_path())
                    same_bits(a, fn(fresh), f"step {si} {path} {what}: sharded / maintained vs fresh")
                    return a

                tag = f"step {si} {path} {m.metric}"
                check_lists(m, q, both(lambda i: i.search(q, K), "search"), want_plain, f"{tag} search")
                if path == "auto":
                    check_lists(m, q[:3], both(lambda i: i.search(q[:3], K), "search Q=3"), want_plain[:3], f"{tag} search Q=3")
                check_lists(m, q, both(lambda i: i.search_filtered(q, K, filters), "filtered"), want_filt, f"{tag} filtered")
                check_lists(m, q, both(lambda i: i.search_windowed(q, K, windows, filters), "windowed"), want_win, f"{tag} windowed")
                rows_q = m.x[rq]
                check_lists(m, rows_q, both(lambda i: i.search_rows(rq, K), "rows"), want_rows, f"{tag} search_rows")
                check_lists(m, rows_q, both(lambda i: i.search_rows(rq, K, None, rwin), "rows windowed"), want_rows_w,
                            f"{tag} search_rows windowed")
                if path != "tensor":  # no range mode on the exact 3xTF32 path
                    res = both(lambda i: i.search_range(q, thr, filters), "range")
                    check_range(res, keys, scale, thr, m.metric, adm_range)
                    pr = both(lambda i: i.search_pairs(pt, first, n_rows, filter=pair_filter), "pairs")
                    check_pairs(m, pr, first, n_rows, pt, adm_pairs)
                    pw = both(lambda i: i.search_pairs(pt, first, n_rows, max_gap=PAIR_GAP), "pairs windowed")
                    check_pairs(m, pw, first, n_rows, pt, m.row_ok(), PAIR_GAP)
                # a removed row's exact contents come back under no id
                for g in range(n_near, n_near + n_gone):
                    top = ix.search(q[g:g + 1], 1)[0][0]
                    if len(top) and top[0] != PAD and not (m.x == q[g]).all(axis=1).any():
                        assert not (m.x[int(top[0])] == q[g]).all(), (tag, "a removed row is still listed")
            if len(case.devices) == 1:
                sub = np.unique(np.concatenate([moved, self.rng.integers(0, len(m), 40)]).astype(np.int64))
                for qi in range(min(Q, 4)):
                    a = ix.score_subset(q[qi], sub, K)
                    same_bits(a, fresh.score_subset(q[qi], sub, K), f"step {si} score_subset")
                    Ss = m.scores(q[qi:qi + 1])[0, sub]
                    o = np.lexsort((np.arange(len(sub)), Ss if m.metric == "euclidean" else -Ss))[:K]
                    check_parity(m.x, q[qi:qi + 1], K, m.metric, a[0][None, :], a[1][None, :], sub[o][None, :], Ss[o][None, :])
                if self.images and has_image(case):
                    self.check_images(si, q[:64], fresh)
        finally:
            fresh.release()
        if not case.big:
            self.check_graph(si)

    def check_images(self, si, q, fresh):
        m = self.model
        for which in ("shadow", "filter") if m.dtype == "f32" else ("shadow",):
            est, bnd = self.ix.filter_dump(q, which)
            fe, fb = fresh.filter_dump(q, which)
            same_bits((est, bnd), (fe, fb), f"step {si} filter_dump({which}): maintained vs fresh image")
            s64, _ = fp64_keys(m.x, q, m.metric)
            err = np.abs(est.astype(np.float64) - s64.T)
            bad = np.argwhere(~(err <= bnd.astype(np.float64)))
            assert bad.size == 0, (f"step {si} filter_dump({which}): |est - s| > bnd", bad[:4].tolist())

    def check_graph(self, si):
        """carry the graphs forward (or build them when the metric or the floor changed) and check them"""
        from nornicdb_b200.knn import ROW_NEW, GraphRowMap, band_windows
        m, ix = self.model, self.ix
        n = len(m)
        path = graph_path(self.case)
        ix.set_path(path or "auto")
        filt = np.tile(np.asarray(GRAPH_FILTER, np.uint64), (n, 1))
        win = band_windows(m.keys, BAND_BELOW)
        args = {"plain": {}, "filtered": {"filters": filt}, "windowed": {"windows": win}}
        rebuild = {kind: ix.search_rows(np.arange(n), K, **a) for kind, a in args.items()}
        state = (m.metric, m.floor)
        if path is not None and self.graph is not None and self.graph[2] == state:
            lists, gmap = self.graph[0], self.graph[1]
            src = gmap.src_of_row
            kept = src[:gmap.n_old] == np.arange(min(gmap.n_old, len(src)))
            no_removal = len(src) >= gmap.n_old and ((src[:gmap.n_old] == ROW_NEW) | kept).all()
            for kind, a in args.items():
                gi, gs = lists[kind]
                ui, us, _ = ix.remap_knn_graph(gi, gs, gmap.n_old, gmap, k=K, **a)
                same_bits((ui, us), rebuild[kind], f"step {si} {kind} graph: remapped vs rebuilt")
                if no_removal:  # appends and rewrites only: the update call serves it too
                    changed = np.nonzero(~kept)[0]
                    ui, us, _ = ix.update_knn_graph(gi, gs, gmap.n_old, changed, k=K, **a)
                    same_bits((ui, us), rebuild[kind], f"step {si} {kind} graph: updated vs rebuilt")
        S = m.scores(m.x)
        np.fill_diagonal(S, np.nan)
        from nornicdb_b200.knn import admits
        adm = {"plain": m.admissible(n),
               "filtered": m.admissible(n) & admits(m.tags, *GRAPH_FILTER)[None, :],
               "windowed": m.admissible(n, None, win)}
        for kind in args:
            check_lists(m, m.x, rebuild[kind], m.topk(S, adm[kind], K), f"step {si} {kind} graph vs fp64")
        self.graph = ({kind: rebuild[kind] for kind in args}, GraphRowMap(n), state)


# ---- the GPU cases -----------------------------------------------------------------------------------------------------
CASES = [
    Case("f32-int8-1shard-d100", "f32", "int8", (0,), 100, 1200, "cosine"),
    Case("f32-bf16-1shard-d36", "f32", "bf16", (0,), 36, 1000, "euclidean"),
    Case("f32-int8-3shards-d100", "f32", "int8", (0, 0, 0), 100, 1500, "dot"),
    Case("f32-bf16-3shards-d1024", "f32", "bf16", (0, 0, 0), 1024, 900, "cosine"),
    Case("f16-1shard-d1024", "f16", None, (0,), 1024, 800, "euclidean"),
    Case("f16-3shards-d36", "f16", None, (0, 0, 0), 36, 900, "cosine"),
    Case("bf16-1shard-d1024", "bf16", None, (0,), 1024, 700, "dot"),
    Case("bf16-3shards-d100", "bf16", None, (0, 0, 0), 100, 900, "euclidean"),
    Case("f32-int8-2gpus-d100", "f32", "int8", (0, 1), 100, 1200, "cosine"),
    # 16 500 x 1024 fp32 rows (> 64 MB, and still >= 16 384 rows after the removals): AUTO's k <= 16 searches scan the int8 image
    Case("f32-auto-1shard-d1024-large", "f32", None, (0,), 1024, 16_500, "cosine", big=True),
]


def device_factory(case, monkeypatch):
    from nornicdb_b200.knn import KnnIndex
    if case.image is None:
        monkeypatch.delenv("NK_SHADOW", raising=False)
    else:
        monkeypatch.setenv("NK_SHADOW", case.image)  # read at creation, by every index of the case
    return lambda devices, metric: KnnIndex(case.dim, metric=metric, dtype=case.dtype, devices=devices)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_index_lifecycle_against_fp64_model(knn_lib, monkeypatch, case):
    if max(case.devices) > 0:
        from nornicdb_b200 import cuda
        if cuda.DeviceCount() < 2:
            pytest.skip("needs two GPUs")
    run = Lifecycle(case, device_factory(case, monkeypatch))
    try:
        run.run()
        if case.big:
            assert min(c for c in run.model.shard_n) * case.dim * 4 >= 64 << 20
            run.ix.set_path("auto")
            run.ix.search(np.zeros((3, case.dim), np.float32) + 1, K)
            assert run.ix.last_path() == "shadow"
    finally:
        run.close()
