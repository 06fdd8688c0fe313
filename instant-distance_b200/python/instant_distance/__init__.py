"""Drop-in for the reference's Python module `instant_distance` (instant-distance-py/src/lib.rs:18-357), GPU backed.

Same classes, method names and argument meaning as the PyO3 module: `Config, Heuristic, Hnsw, HnswMap, Search, Neighbor`.
Everything numeric happens in libinstant_distance_b200.so through the C ABI (no CPU fallback).  Differences, all additive:
  * points may have any dimension (the reference fixes DIMENSIONS = 300, py:448, and zero-pads shorter inputs, py:367-374;
    here every point of an index is zero-padded to the longest point given at build time, and a longer query raises the
    same `TypeError("point array too long")`, py:369-370);
  * `Hnsw.search_many / HnswMap.search_many` expose the batched search the GPU is built for;
  * `Hnsw.search_exact / HnswMap.search_exact` return the exact k nearest points (a scan of every point, ties by lower PointId),
    the ground truth to tune `ef_search` against;
  * `Hnsw.search_range / HnswMap.search_range` return every point within a radius of each query (exact, however many there are;
    DESIGN.md §9b), nearest first, as CSR;
  * `Hnsw.search_range_graph / HnswMap.search_range_graph` return the points within a radius that the graph reaches from each
    query's approximate nearest neighbours (a subset of search_range's result at a cost that follows the hits; DESIGN.md §9c);
  * `Hnsw.insert / HnswMap.insert` append points to a built or loaded index (layer 0 only, PointIds continue from the current
    count; DESIGN.md §6);
  * `Config.metric = "cosine"` builds an index that reports 1 - cos (points and queries normalised in the canonical order,
    DESIGN.md §3a; default "l2sq"); the file does not record it, so `Hnsw.load / HnswMap.load(..., metric=)` take it;
  * `Config.storage = "bf16"` or `"f16"` keeps the points in GPU memory rounded to 2 bytes per element (default "f32"; DESIGN.md
    §3b: results are those of the f32 index on the rounded points; "f16" refuses values that round to infinity, |x| >= 65520).
  * `Config.storage = "q8"` keeps them as one byte per element on a grid of each point's own (DESIGN.md §3c: results are those of
    the f32 index on the dequantised points; points with a NaN or infinite value, or whose grid would overflow f32, are refused).
  * `Config.storage = "bin"` keeps 0/1 points at one byte per four elements (DESIGN.md §3d): every point value must be 0.0, -0.0
    or 1.0 (others are refused), and the metric must be "l2sq".  Queries are any floats; the reported distance is the squared L2 to
    the 0/1 point, which for 0/1 queries is exactly the Hamming distance.  Packed codes (8 bits per byte) unpack with
    `np.unpackbits(codes, axis=1).astype(np.float32)`.
    The file holds the points widened to f32, so `Hnsw.load / HnswMap.load(..., storage=)` take the storage too.
"""
import ctypes as C
import random

import numpy as np

from instant_distance_b200 import _abi

__all__ = ["Config", "Heuristic", "Hnsw", "HnswMap", "Search", "Neighbor"]


class Heuristic:
    """py:276-303.  Defaults: extend_candidates=False, keep_pruned=True (lib.rs:121-128)."""

    def __init__(self):
        self.extend_candidates = False
        self.keep_pruned = True


class Config:
    """py:216-256: Builder defaults (lib.rs:101-113); `seed` is drawn from entropy like `rand::random()`."""

    def __init__(self):
        p = _abi.default_params()
        self.ef_search = int(p.ef_search)
        self.ef_construction = int(p.ef_construction)
        self.ml = float(p.ml)
        self.seed = random.getrandbits(64)
        self.heuristic = Heuristic()
        self.metric = "l2sq"  # or "cosine"
        self.storage = "f32"  # or "bf16", "f16", "q8", "bin"

    def _params(self):
        kw = dict(ef_search=self.ef_search, ef_construction=self.ef_construction, ml=self.ml, seed=self.seed, metric=self.metric,
                  storage=_abi._storage(self.storage))
        if self.heuristic is None:
            kw["heuristic"] = 0
        else:
            kw.update(heuristic=1, extend_candidates=int(bool(self.heuristic.extend_candidates)),
                      keep_pruned=int(bool(self.heuristic.keep_pruned)))
        return kw


class Neighbor:
    """py:327-357."""

    def __init__(self, distance, pid, value=None):
        self.distance, self.pid, self.value = float(distance), int(pid), value

    def __repr__(self):
        if self.value is not None:
            return f"instant_distance.Neighbor(distance={self.distance}, pid={self.pid}, value={self.value!r})"
        return f"instant_distance.Item(distance={self.distance}, pid={self.pid})"


class Search:
    """py:159-209: search buffer and result set; iterate it after `index.search(point, search)`."""

    def __init__(self):
        self._ids = self._dist = None
        self._len = 0
        self._values = None
        self._cur = None

    def __iter__(self):
        return self

    def __next__(self):
        if self._cur is None or self._cur >= self._len:
            self._cur = None
            raise StopIteration
        i = self._cur
        self._cur += 1
        pid = int(self._ids[i])
        return Neighbor(self._dist[i], pid, None if self._values is None else self._values[pid])


def _to_matrix(points, dim=None):
    rows = [np.asarray(list(p), dtype=np.float32) for p in points]
    width = max([len(r) for r in rows], default=1) if dim is None else dim
    m = np.zeros((len(rows), max(width, 1)), dtype=np.float32)
    for i, r in enumerate(rows):
        if len(r) > m.shape[1]:
            raise TypeError("point array too long")
        m[i, :len(r)] = r
    return m


class Hnsw:
    """py:97-157."""

    def __init__(self, index, values=None):
        self._ix = index
        self._values = values
        info = index.info()
        self._dim, self._ef = int(info.dim), int(info.ef_search)

    @staticmethod
    def build(points, config):
        m = _to_matrix(points)
        ix, ids = _abi.Index.build(m, **config._params())
        return Hnsw(ix), [int(i) for i in ids]

    def search(self, point, search):
        q = _to_matrix([point], self._dim)
        k = max(self._ef, 1)
        ids, dist, lens = self._ix.search(q, ef_search=self._ef, k=k) if self._ef else (np.zeros((1, 1), np.uint32), np.zeros((1, 1), np.float32), [0])
        search._ids, search._dist, search._len, search._values, search._cur = ids[0], dist[0], int(lens[0]), self._values, 0

    def search_many(self, points, k=10, ef_search=None):
        """Batched Hnsw::search: returns (ids [nq, k], distances [nq, k], lens [nq])."""
        q = _to_matrix(points, self._dim) if not isinstance(points, np.ndarray) else points
        return self._ix.search(q, ef_search=ef_search or self._ef, k=k)

    def search_exact(self, points, k=10):
        """Exact k-NN over every point of the index: returns (ids [nq, k], distances [nq, k], lens [nq]) like search_many."""
        q = _to_matrix(points, self._dim) if not isinstance(points, np.ndarray) else points
        return self._ix.exact_search(q, k=k)

    def search_range(self, points, radius):
        """Every point within `radius` of each query (distance <= radius, in the index's metric), exact: returns (offsets [nq + 1],
        ids [total], distances [total]); query i's neighbours are ids[offsets[i]:offsets[i + 1]], nearest first, ties by PointId."""
        q = _to_matrix(points, self._dim) if not isinstance(points, np.ndarray) else points
        return self._ix.range_search(q, radius)

    def search_range_graph(self, points, radius, ef_search=None):
        """The points within `radius` of each query that layer 0 reaches from the query's ef_search nearest neighbours (default: the
        index's ef_search) through points within `radius` (DESIGN.md §9c): a subset of search_range's result with the same
        distances, laid out the same way, at a cost that follows the hits rather than the number of points."""
        q = _to_matrix(points, self._dim) if not isinstance(points, np.ndarray) else points
        return self._ix.graph_range_search(q, radius, ef_search=ef_search or 0)

    @staticmethod
    def _link_kw(config):
        """The idb_params fields an insert or a removal reads from config: ef_construction and the heuristic."""
        kw = dict(ef_construction=config.ef_construction)
        if config.heuristic is None:
            kw["heuristic"] = 0
        else:
            kw.update(heuristic=1, extend_candidates=int(bool(config.heuristic.extend_candidates)),
                      keep_pruned=int(bool(config.heuristic.keep_pruned)))
        return kw

    def _insert(self, points, config, on_partial=None):
        """on_partial(k): called before an IdbError propagates, with how many of the points the index kept (an insert that fails
        with ERR_CAPACITY keeps the batches before the failing one)."""
        m = _to_matrix(points, self._dim)
        config = Config() if config is None else config
        kw = self._link_kw(config)
        n0 = int(self._ix.info().n)
        try:
            return [int(i) for i in self._ix.insert(m, **kw)]
        except _abi.IdbError:
            if on_partial is not None:
                on_partial(int(self._ix.info().n) - n0)
            raise

    def insert(self, points, config=None):
        """Not in the reference module: adds points to the index and returns their PointIds (the current count onwards, in order).
        Construction::insert on layer 0 (the upper layers keep sampling the points the index was built with).  config supplies
        ef_construction and the heuristic (None: Config() defaults); points are zero-padded to the index's dimension."""
        return self._insert(points, config)

    def remove(self, pids, config=None):
        """Not in the reference module: removes the points `pids` (distinct PointIds) and returns new_ids, one entry per point the
        index had: the point's PointId afterwards, or INVALID (0xFFFFFFFF) for a removed one.  The surviving points keep their order
        and are renumbered without gaps.  The rows that listed a removed point are re-selected from their own entries and the
        removed point's neighbours; config supplies ef_construction and the heuristic (None: Config() defaults)."""
        config = Config() if config is None else config
        return [int(i) for i in self._ix.remove(pids, **self._link_kw(config))]

    def dump(self, fname):
        """py:131-137: bincode layout of `Hnsw` (ef_search, points, zero, layers)."""
        self._ix.save(fname)

    @staticmethod
    def load(fname, dim=300, M=32, metric="l2sq", storage="f32"):
        """py:121-129.  The file does not store dim / M (fixed arrays in the reference: 300 / 32), nor the metric or storage."""
        try:
            ix, _ = _abi.Index.load(fname, dim, M, metric=metric, storage=storage)
        except _abi.IdbError as e:
            if e.status == _abi.ERR_IO:
                raise OSError(str(e)) from e
            raise ValueError(f"deserialization error: {e}") from e
        return Hnsw(ix)


class HnswMap(Hnsw):
    """py:30-95: values are kept on the host, permuted to PointId order as HnswMap::new does (lib.rs:144-149)."""

    @staticmethod
    def build(points, values, config):
        m = _to_matrix(points)
        vals = [str(v) if not isinstance(v, str) else v for v in values]
        ix, ids = _abi.Index.build(m, **config._params())
        by_pid = [None] * len(ids)
        for orig, pid in enumerate(ids):
            by_pid[int(pid)] = vals[orig]
        return HnswMap(ix, by_pid)

    def insert(self, points, values, config=None):
        """Hnsw.insert, with one value per point; values follow the new PointIds (and `dump` writes them).  If the insert fails
        with ERR_CAPACITY, the values of the points the index kept are appended before the error propagates."""
        vals = [str(v) if not isinstance(v, str) else v for v in values]
        if len(vals) != len(points):
            raise ValueError("one value per point")
        # values follow PointIds, also for the points a failed insert kept
        ids = self._insert(points, config, on_partial=lambda kept: self._values.extend(vals[:kept]))
        self._values.extend(vals)
        return ids

    def remove(self, pids, config=None):
        """Hnsw.remove; the values of the removed points are dropped and the others follow their points' new PointIds (so `dump`
        writes them in PointId order)."""
        new_ids = Hnsw.remove(self, pids, config)
        self._values = [v for v, y in zip(self._values, new_ids) if y != _abi.INVALID]
        return new_ids

    @property
    def values(self):
        return self._values

    def dump(self, fname):
        """py:69-75: `HnswMap { hnsw, values }` — the Hnsw body, then Vec<MapValue::String> (u32 variant 0, u64 len, utf-8)."""
        import struct

        self._ix.save(fname)
        with open(fname, "ab") as f:
            f.write(struct.pack("<Q", len(self._values)))
            for v in self._values:
                b = v.encode("utf-8")
                f.write(struct.pack("<IQ", 0, len(b)) + b)

    @staticmethod
    def load(fname, dim=300, M=32, metric="l2sq", storage="f32"):
        """py:58-67."""
        import struct

        try:
            ix, off = _abi.Index.load(fname, dim, M, metric=metric, storage=storage)
        except _abi.IdbError as e:
            if e.status == _abi.ERR_IO:
                raise OSError(str(e)) from e
            raise ValueError(f"deserialization error: {e}") from e
        values = []
        with open(fname, "rb") as f:
            f.seek(off)
            head = f.read(8)
            if len(head) != 8:
                raise ValueError("deserialization error: no values section (an Hnsw file, not an HnswMap?)")
            (count,) = struct.unpack("<Q", head)
            for _ in range(count):
                variant, ln = struct.unpack("<IQ", f.read(12))
                if variant != 0:
                    raise ValueError(f"deserialization error: unknown MapValue variant {variant}")
                values.append(f.read(ln).decode("utf-8"))
        if len(values) != int(ix.info().n):
            raise ValueError("deserialization error: values length does not match the point count")
        return HnswMap(ix, values)
