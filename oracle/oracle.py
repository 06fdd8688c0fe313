"""ctypes loader for the CPU oracle (oracle/hnsw_oracle.cpp).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs.  The product package never imports this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "liboracle.so")


class Params(C.Structure):
    _fields_ = [
        ("M", C.c_uint32),
        ("ef_construction", C.c_uint32),
        ("ef_search", C.c_uint32),
        ("ml", C.c_float),
        ("seed", C.c_uint64),
        ("heuristic", C.c_int32),
        ("extend_candidates", C.c_int32),
        ("keep_pruned", C.c_int32),
        ("threads", C.c_int32),
        ("metric", C.c_int32),
    ]


class BatchStats(C.Structure):
    _fields_ = [(name, C.c_uint64) for name in (
        "batches", "max_batch", "link_requests", "targets", "max_target_requests", "multi_new_rounds", "multi_round_targets",
        "admission_limited_rounds", "simple_multi_targets", "max_insert_dist")]


def build_lib(force=False):
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(os.path.join(_HERE, "hnsw_oracle.cpp")):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_SO):
        build_lib()
    L = C.CDLL(_SO)
    u32p, f32p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_uint64)
    L.orc_params_default.argtypes = [C.POINTER(Params)]
    L.orc_default_ml.restype = C.c_float
    L.orc_default_ml.argtypes = [C.c_uint32]
    L.orc_l2sq.restype = C.c_float
    L.orc_l2sq.argtypes = [f32p, f32p, C.c_uint32]
    L.orc_l2sq_scalar.restype = C.c_float
    L.orc_l2sq_scalar.argtypes = [f32p, f32p, C.c_uint32]
    L.orc_l2sq_reference_order.restype = C.c_float
    L.orc_l2sq_reference_order.argtypes = [f32p, f32p, C.c_uint32]
    L.orc_simd_level.restype = C.c_int
    L.orc_layer_schedule.restype = C.c_uint32
    L.orc_layer_schedule.argtypes = [C.c_uint64, C.c_uint32, C.c_float, u64p, C.c_uint32]
    L.orc_shuffle.argtypes = [C.c_uint64, C.c_uint64, u32p]
    L.orc_rng_kat.argtypes = [u64p, C.c_uint64, u64p, C.c_uint32]
    L.orc_rng_kat.restype = None
    L.orc_build.restype = C.c_void_p
    L.orc_build.argtypes = [f32p, C.c_uint64, C.c_uint32, C.POINTER(Params), u32p]
    L.orc_build_batched.restype = C.c_void_p
    L.orc_build_batched.argtypes = [f32p, C.c_uint64, C.c_uint32, C.POINTER(Params), C.c_uint32, C.c_uint32, C.POINTER(BatchStats),
                                    u64p, C.c_uint64, u32p, u32p]
    L.orc_from_graph.restype = C.c_void_p
    L.orc_from_graph.argtypes = [f32p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, u32p, C.c_uint32,
                                 C.POINTER(u32p), u64p, C.c_int32]
    L.orc_free.argtypes = [C.c_void_p]
    for name, rt in [("orc_n", C.c_uint64), ("orc_dim", C.c_uint32), ("orc_M", C.c_uint32), ("orc_num_layers", C.c_uint32)]:
        getattr(L, name).restype = rt
        getattr(L, name).argtypes = [C.c_void_p]
    L.orc_layer_count.restype = C.c_uint64
    L.orc_layer_count.argtypes = [C.c_void_p, C.c_uint32]
    L.orc_export_points.argtypes = [C.c_void_p, f32p]
    L.orc_export_zero.argtypes = [C.c_void_p, u32p]
    L.orc_export_upper.argtypes = [C.c_void_p, C.c_uint32, u32p]
    L.orc_search.restype = C.c_int
    L.orc_search.argtypes = [C.c_void_p, f32p, C.c_uint64, C.c_uint32, C.c_uint32, u32p, f32p, u32p, u64p, C.c_int32]
    L.orc_bruteforce.restype = C.c_int
    L.orc_bruteforce.argtypes = [f32p, C.c_uint64, C.c_uint32, f32p, C.c_uint64, C.c_uint32, u32p, f32p, C.c_int32, C.c_int32]
    L.orc_select_heuristic.restype = C.c_uint32
    L.orc_select_heuristic.argtypes = [C.c_void_p, f32p, u32p, C.c_uint32, C.c_int32, u32p, f32p]
    _lib = L
    return L


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def default_params(**kw):
    p = Params()
    lib().orc_params_default(C.byref(p))
    if "M" in kw and "ml" not in kw:
        kw["ml"] = float(lib().orc_default_ml(kw["M"]))
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def l2sq(a, b, scalar=False):
    a, b = _f32(a), _f32(b)
    fn = lib().orc_l2sq_scalar if scalar else lib().orc_l2sq
    return np.float32(fn(_p(a, C.c_float), _p(b, C.c_float), a.shape[0]))


METRIC_CANONICAL, METRIC_SQRT_SEQ, METRIC_REFERENCE_AVX2 = 0, 1, 2


def l2sq_reference_order(a, b):
    """FloatArray::distance in the reference's own AVX2 summation order (py:378-421); needs dim % 8 == 4 (the reference: 300)."""
    a, b = _f32(a), _f32(b)
    assert a.shape[0] % 8 == 4 and a.shape == b.shape
    return np.float32(lib().orc_l2sq_reference_order(_p(a, C.c_float), _p(b, C.c_float), a.shape[0]))


def layer_schedule(n, M=32, ml=None):
    ml = float(lib().orc_default_ml(M)) if ml is None else ml
    counts = np.zeros(64, dtype=np.uint64)
    L = lib().orc_layer_schedule(n, M, ml, _p(counts, C.c_uint64), 64)
    return [int(c) for c in counts[:L]]


def shuffle(n, seed):
    out = np.empty(n, dtype=np.uint32)
    lib().orc_shuffle(n, seed, _p(out, C.c_uint32))
    return out


def rng_kat(count=10, state=None, seed=0):
    """First `count` u64 outputs of the rand restatement, from a raw xoshiro256++ state or from seed_from_u64(seed)."""
    out = np.empty(count, dtype=np.uint64)
    st = None if state is None else np.ascontiguousarray(state, dtype=np.uint64)
    lib().orc_rng_kat(None if st is None else _p(st, C.c_uint64), seed, _p(out, C.c_uint64), count)
    return out


class Graph:
    """Plain-numpy view of an index: what crosses into the product's `idb_index_from_graph`."""

    def __init__(self, points, zero, upper, M, ef_search):
        self.points, self.zero, self.upper, self.M, self.ef_search = points, zero, upper, M, ef_search


class Index:
    def __init__(self, handle, keepalive=None):
        self._h = handle
        self._keep = keepalive

    def __del__(self):
        try:
            if getattr(self, "_h", None) and _lib is not None:
                _lib.orc_free(self._h)
            self._h = None
        except Exception:  # noqa: BLE001  (interpreter shutdown)
            pass

    @property
    def n(self):
        return int(lib().orc_n(self._h))

    @property
    def dim(self):
        return int(lib().orc_dim(self._h))

    @property
    def M(self):
        return int(lib().orc_M(self._h))

    @property
    def num_layers(self):
        return int(lib().orc_num_layers(self._h))

    def layer_counts(self):
        return [int(lib().orc_layer_count(self._h, l)) for l in range(self.num_layers)]

    def export(self, ef_search=100):
        n, dim, M = self.n, self.dim, self.M
        pts = np.empty((n, dim), dtype=np.float32)
        zero = np.empty((n, 2 * M), dtype=np.uint32)
        if n:
            lib().orc_export_points(self._h, _p(pts, C.c_float))
            lib().orc_export_zero(self._h, _p(zero, C.c_uint32))
        upper = []
        for l in range(1, self.num_layers):
            u = np.empty((int(lib().orc_layer_count(self._h, l)), M), dtype=np.uint32)
            lib().orc_export_upper(self._h, l, _p(u, C.c_uint32))
            upper.append(u)
        return Graph(pts, zero, upper, M, ef_search)

    def search(self, queries, ef_search=100, k=None, threads=1, counters=False):
        q = _f32(queries)
        if q.ndim == 1:
            q = q[None, :]
        nq = q.shape[0]
        k = ef_search if k is None else k
        ids = np.empty((nq, k), dtype=np.uint32)
        dist = np.empty((nq, k), dtype=np.float32)
        lens = np.empty(nq, dtype=np.uint32)
        cnt = np.zeros((nq, 4), dtype=np.uint64) if counters else None
        lib().orc_search(self._h, _p(q, C.c_float), nq, ef_search, k, _p(ids, C.c_uint32), _p(dist, C.c_float),
                         _p(lens, C.c_uint32), _p(cnt, C.c_uint64) if counters else None, threads)
        return (ids, dist, lens, cnt) if counters else (ids, dist, lens)

    def select_heuristic(self, point, cand_ids, keep_pruned=True):
        point = _f32(point)
        cand = np.ascontiguousarray(cand_ids, dtype=np.uint32)
        out = np.empty(2 * self.M, dtype=np.uint32)
        outd = np.empty(2 * self.M, dtype=np.float32)
        c = lib().orc_select_heuristic(self._h, _p(point, C.c_float), _p(cand, C.c_uint32), cand.shape[0],
                                       1 if keep_pruned else 0, _p(out, C.c_uint32), _p(outd, C.c_float))
        return out[:c].copy(), outd[:c].copy()


def build(rows, **kw):
    """Builder::build_hnsw (core:83-85).  Returns (Index, ids) with ids[orig] = PointId."""
    rows = _f32(rows)
    n, dim = rows.shape
    p = default_params(**kw)
    ids = np.empty(n, dtype=np.uint32)
    h = lib().orc_build(_p(rows, C.c_float), n, dim, C.byref(p), _p(ids, C.c_uint32))
    if not h:
        raise ValueError("orc_build failed (N >= u32::MAX?)")
    return Index(h), ids


def build_batched(rows, max_batch, growth, threads=1, **kw):
    """The library's batched build schedule (DESIGN.md §6), stated on the CPU.  Returns (Index, ids, stats).

    max_batch / growth: the schedule's cap and divisor (the library takes them from insert_batch, or from IDB_BUILD_MAXBATCH /
    IDB_BUILD_GROWTH when insert_batch is 0; its defaults are 16384 and 8).  stats: the BatchStats counters as a dict, plus
    "bounds" (batches x 2: first PointId, inserts, in build order) and "row_batch" (per zero row, the last batch that wrote it).
    """
    rows = _f32(rows)
    n, dim = rows.shape
    p = default_params(threads=threads, **kw)
    ids = np.empty(n, dtype=np.uint32)
    st = BatchStats()
    cap = n + 1  # a batch holds at least one insert
    bounds = np.zeros((cap, 2), dtype=np.uint64)
    row_batch = np.empty(n, dtype=np.uint32)
    h = lib().orc_build_batched(_p(rows, C.c_float), n, dim, C.byref(p), max_batch, growth, C.byref(st), _p(bounds, C.c_uint64), cap,
                                _p(row_batch, C.c_uint32), _p(ids, C.c_uint32))
    if not h:
        raise ValueError("orc_build_batched failed (max_batch or growth 0, extend_candidates, or N >= u32::MAX)")
    stats = {name: int(getattr(st, name)) for name, _ in BatchStats._fields_}
    stats["bounds"] = bounds[:stats["batches"]].copy()
    stats["row_batch"] = row_batch
    return Index(h), ids, stats


def from_graph(g, metric=0):
    pts, zero = _f32(g.points), np.ascontiguousarray(g.zero, dtype=np.uint32)
    n, dim = pts.shape
    ups = [np.ascontiguousarray(u, dtype=np.uint32) for u in g.upper]
    arr = (C.POINTER(C.c_uint32) * max(1, len(ups)))(*[_p(u, C.c_uint32) for u in ups])
    un = np.array([u.shape[0] for u in ups], dtype=np.uint64)
    h = lib().orc_from_graph(_p(pts, C.c_float), n, dim, g.M, g.ef_search, _p(zero, C.c_uint32), len(ups), arr,
                             _p(un, C.c_uint64), metric)
    return Index(h, keepalive=(pts, zero, ups))


def bruteforce(points, queries, k, metric=0, threads=1):
    pts, q = _f32(points), _f32(queries)
    if q.ndim == 1:
        q = q[None, :]
    ids = np.empty((q.shape[0], k), dtype=np.uint32)
    dist = np.empty((q.shape[0], k), dtype=np.float32)
    lib().orc_bruteforce(_p(pts, C.c_float), pts.shape[0], pts.shape[1], _p(q, C.c_float), q.shape[0], k,
                         _p(ids, C.c_uint32), _p(dist, C.c_float), metric, threads)
    return ids, dist
