"""ctypes binding of the C ABI declared in include/instant_distance_b200.h.

This is the exact stub a Python-side maintainer of the reference binding would write (INTEGRATION.md); nothing here
computes anything — every call goes to libinstant_distance_b200.so, which fails loudly when no CUDA device exists.
"""
import ctypes as C
import os

import numpy as np

_PKG = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
LIB_PATH = os.environ.get("IDB_LIB_PATH") or os.path.join(_PKG, "lib", "libinstant_distance_b200.so")  # (IDB_LIB_PATH: A/B builds)

INVALID = 0xFFFFFFFF
RANGE_MAX_CAPACITY = 0x7FFFFFFF  # the range search's largest capacity (and nq)

OK, ERR_INVALID_ARG, ERR_OOM, ERR_CUDA, ERR_NCCL, ERR_IO, ERR_FORMAT, ERR_CAPACITY, ERR_UNSUPPORTED = range(9)

SYMBOLS = [
    "idb_params_default", "idb_build_f32", "idb_index_from_graph_f32", "idb_index_from_graph_bf16", "idb_search_batch_f32",
    "idb_search_batch_device", "idb_search_batch_device_lane", "idb_last_search_counters", "idb_last_search_failures", "idb_last_search_retried",
    "idb_index_num_lanes", "idb_index_lane_stream", "idb_device_set_persisting_l2", "idb_index_info", "idb_index_export_points",
    "idb_index_export_zero", "idb_index_export_upper", "idb_index_save", "idb_index_load", "idb_index_set_profiling", "idb_index_last_kernel_ms", "idb_debug_gather_bench", "idb_debug_gather_mix_bench",
    "idb_index_stream", "idb_index_sync", "idb_index_free",
    "idb_comm_unique_id", "idb_comm_create", "idb_comm_free", "idb_index_set_id_map", "idb_sharded_search_batch_f32",
    "idb_sharded_search_batch_device", "idb_sharded_search_batch_f32_multi", "idb_sharded_search_batch_device_multi", "idb_distance_f32", "idb_host_alloc", "idb_host_free", "idb_last_error", "idb_version", "idb_device_count",
    "idb_build_ex", "idb_index_from_graph_ex", "idb_index_load_ex", "idb_normalize_f32", "idb_index_metric",
    "idb_last_search_full_fetches", "idb_debug_screen_bound", "idb_last_search_kernel", "idb_debug_merge_topk",
    "idb_exact_search_batch_f32", "idb_exact_search_batch_device_lane", "idb_index_insert_f32", "idb_index_load_storage",
    "idb_range_search_batch_f32", "idb_range_search_batch_device_lane", "idb_index_remove",
    "idb_graph_range_search_batch_f32", "idb_graph_range_search_batch_device_lane",
]


class Params(C.Structure):
    _fields_ = [
        ("M", C.c_uint32), ("ef_construction", C.c_uint32), ("ef_search", C.c_uint32), ("ml", C.c_float),
        ("seed", C.c_uint64), ("heuristic", C.c_int32), ("extend_candidates", C.c_int32), ("keep_pruned", C.c_int32),
        ("insert_batch", C.c_uint32), ("device", C.c_int32), ("storage", C.c_uint32),
        ("progress", C.c_void_p), ("progress_user", C.c_void_p),
    ]


class Info(C.Structure):
    _fields_ = [
        ("n", C.c_uint64), ("dim", C.c_uint32), ("M", C.c_uint32), ("ef_search", C.c_uint32), ("n_layers", C.c_uint32),
        ("layer_n", C.c_uint64 * 32), ("device", C.c_int32), ("storage", C.c_uint32),
    ]


class IdbError(RuntimeError):
    def __init__(self, status, message):
        super().__init__(f"idb status {status}: {message}")
        self.status = status


_lib = None


def lib():
    """Load the shared library.  Raises if it has not been built: there is no fallback implementation."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise IdbError(ERR_CUDA, f"{LIB_PATH} is missing — run `python -c 'import __graft_entry__ as g; g.build()'` "
                                 "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    u32p, f32p, u64p, vp = C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_uint64), C.c_void_p
    L.idb_params_default.argtypes = [C.POINTER(Params)]
    L.idb_build_f32.argtypes = [f32p, C.c_uint64, C.c_uint32, C.POINTER(Params), C.POINTER(vp), u32p]
    L.idb_index_from_graph_f32.argtypes = [f32p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, u32p, C.c_uint32,
                                           C.POINTER(u32p), u64p, C.c_int32, C.POINTER(vp)]
    L.idb_index_from_graph_bf16.argtypes = L.idb_index_from_graph_f32.argtypes
    L.idb_build_ex.argtypes = [f32p, C.c_uint64, C.c_uint32, C.POINTER(Params), C.c_uint32, C.POINTER(vp), u32p]
    L.idb_index_from_graph_ex.argtypes = [f32p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, u32p, C.c_uint32,
                                          C.POINTER(u32p), u64p, C.c_uint32, C.c_uint32, C.c_int32, C.POINTER(vp)]
    L.idb_index_load_ex.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int32, C.POINTER(vp), u64p]
    L.idb_index_load_storage.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int32, C.POINTER(vp), u64p]
    L.idb_index_insert_f32.argtypes = [vp, f32p, C.c_uint64, C.c_uint32, C.POINTER(Params), u32p, u32p]
    L.idb_index_remove.argtypes = [vp, u32p, C.c_uint64, C.POINTER(Params), u32p]
    L.idb_normalize_f32.argtypes = [f32p, C.c_uint64, C.c_uint32, C.c_int32, f32p]
    L.idb_index_metric.argtypes = [vp, u32p]
    L.idb_search_batch_f32.argtypes = [vp, f32p, C.c_uint64, C.c_uint32, C.c_uint32, u32p, f32p, u32p]
    L.idb_search_batch_device.argtypes = [vp, vp, C.c_uint64, C.c_uint32, C.c_uint32, vp, vp, vp]
    L.idb_search_batch_device_lane.argtypes = [vp, C.c_uint32, vp, C.c_uint64, C.c_uint32, C.c_uint32, vp, vp, vp]
    L.idb_exact_search_batch_f32.argtypes = [vp, f32p, C.c_uint64, C.c_uint32, u32p, f32p, u32p]
    L.idb_exact_search_batch_device_lane.argtypes = [vp, C.c_uint32, vp, C.c_uint64, C.c_uint32, vp, vp, vp]
    L.idb_range_search_batch_f32.argtypes = [vp, f32p, C.c_uint64, C.c_float, C.c_uint64, u64p, u32p, f32p]
    L.idb_range_search_batch_device_lane.argtypes = [vp, C.c_uint32, vp, C.c_uint64, C.c_float, C.c_uint64, vp, vp, vp, u64p]
    L.idb_graph_range_search_batch_f32.argtypes = [vp, f32p, C.c_uint64, C.c_uint32, C.c_float, C.c_uint64, u64p, u32p, f32p]
    L.idb_graph_range_search_batch_device_lane.argtypes = [vp, C.c_uint32, vp, C.c_uint64, C.c_uint32, C.c_float, C.c_uint64, vp, vp, vp,
                                                           u64p]
    L.idb_last_search_counters.argtypes = [vp, C.c_uint64, u64p]
    L.idb_last_search_failures.argtypes = [vp, C.c_uint32, u32p]
    L.idb_last_search_retried.argtypes = [vp, C.c_uint32, u32p]
    L.idb_last_search_full_fetches.argtypes = [vp, C.c_uint32, u64p]
    L.idb_debug_screen_bound.argtypes = [vp, f32p, C.c_uint64, u32p, C.c_uint64, f32p, f32p]
    L.idb_last_search_kernel.argtypes = [vp, C.c_uint32, u32p]
    L.idb_debug_merge_topk.argtypes = [vp, u64p, C.c_uint32, C.c_uint64, C.c_uint32, u32p, f32p, u32p, u64p]
    L.idb_index_num_lanes.restype = C.c_uint32
    L.idb_index_lane_stream.argtypes = [vp, C.c_uint32]
    L.idb_index_lane_stream.restype = vp
    L.idb_device_set_persisting_l2.argtypes = [C.c_int32, C.c_int32]
    L.idb_index_info.argtypes = [vp, C.POINTER(Info)]
    L.idb_index_export_points.argtypes = [vp, f32p]
    L.idb_index_export_zero.argtypes = [vp, u32p]
    L.idb_index_export_upper.argtypes = [vp, C.c_uint32, u32p]
    L.idb_index_save.argtypes = [vp, C.c_char_p]
    L.idb_index_load.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32, C.c_int32, C.POINTER(vp), u64p]
    L.idb_debug_gather_bench.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, f32p, C.POINTER(C.c_double)]
    L.idb_debug_gather_mix_bench.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, f32p, C.POINTER(C.c_double)]
    L.idb_index_set_profiling.argtypes = [vp, C.c_int32]
    L.idb_index_last_kernel_ms.argtypes = [vp, f32p, u32p]
    L.idb_index_stream.argtypes = [vp]
    L.idb_index_stream.restype = vp
    L.idb_index_sync.argtypes = [vp]
    L.idb_index_free.argtypes = [vp]
    L.idb_index_free.restype = None
    L.idb_comm_unique_id.argtypes = [vp]
    L.idb_comm_create.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, C.POINTER(vp)]
    L.idb_comm_free.argtypes = [vp]
    L.idb_comm_free.restype = None
    L.idb_index_set_id_map.argtypes = [vp, u32p]
    L.idb_sharded_search_batch_f32.argtypes = [vp, vp, f32p, C.c_uint64, C.c_uint32, C.c_uint32, u32p, f32p, u32p]
    L.idb_sharded_search_batch_device.argtypes = [vp, vp, vp, C.c_uint64, C.c_uint32, C.c_uint32, vp, vp, vp]
    L.idb_sharded_search_batch_f32_multi.argtypes = [C.POINTER(vp), C.c_uint32, vp, f32p, C.c_uint64, C.c_uint32, C.c_uint32, u32p, f32p, u32p]
    L.idb_sharded_search_batch_device_multi.argtypes = [C.POINTER(vp), C.c_uint32, vp, vp, C.c_uint64, C.c_uint32, C.c_uint32, vp, vp, vp]
    L.idb_distance_f32.argtypes = [f32p, f32p, C.c_uint32, C.c_int32, f32p]
    L.idb_host_alloc.argtypes = [C.c_size_t, C.POINTER(vp)]
    L.idb_host_free.argtypes = [vp]
    L.idb_host_free.restype = None
    L.idb_last_error.restype = C.c_char_p
    L.idb_version.restype = C.c_char_p
    L.idb_device_count.restype = C.c_int32
    for name in SYMBOLS:
        fn = getattr(L, name)
        if name not in ("idb_index_stream", "idb_index_lane_stream", "idb_index_num_lanes", "idb_index_free", "idb_host_free", "idb_last_error", "idb_version", "idb_device_count",
                        "idb_comm_free"):
            fn.restype = C.c_int
    _lib = L
    return L


def check(status):
    if status != OK:
        raise IdbError(status, lib().idb_last_error().decode("utf-8", "replace"))


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def ptr(a, t):
    return a.ctypes.data_as(C.POINTER(t))


# IDB_STORAGE_*: how an index keeps its rows (2-byte rows are widened exactly to f32; q8 rows are dequantised exactly, DESIGN.md §3c;
# bin rows are 0/1, one byte per four elements, DESIGN.md §3d)
STORAGE = {"f32": 0, "bf16": 1, "f16": 2, "q8": 4, "bin": 8}
METRIC = {"l2sq": 0, "cosine": 1}  # IDB_METRIC_*: squared L2, or 1 - cos through canonically normalised rows (DESIGN.md §3a)


def _metric(metric):
    if metric not in METRIC:
        raise ValueError(f"metric must be one of {sorted(METRIC)}, not {metric!r}")
    return METRIC[metric]


def _storage(storage):
    if storage not in STORAGE:
        raise ValueError(f"storage must be one of {sorted(STORAGE)}, not {storage!r}")
    return STORAGE[storage]


def _ef(ef_search):
    """A search width as the C ABI's uint32_t: a value ctypes would wrap (negative, or 2^32 and up) is refused here."""
    ef = int(ef_search)
    if not 0 <= ef <= 0xFFFFFFFF:
        raise ValueError(f"ef_search must be 0 (the index's) or 1..1024, not {ef_search!r}")
    return ef


PROGRESS_FN = C.CFUNCTYPE(None, C.c_uint64, C.c_uint64, C.c_void_p)


def default_params(**kw):
    p = Params()
    check(lib().idb_params_default(C.byref(p)))
    if isinstance(kw.get("storage"), str):
        kw["storage"] = STORAGE[kw["storage"]]
    if "M" in kw and "ml" not in kw:
        kw["ml"] = float(np.float32(1.0) / np.log(np.float32(kw["M"])))
    for k, v in kw.items():
        setattr(p, k, v)
    return p


class Index:
    """Owns one idb_index handle."""

    def __init__(self, handle):
        self._h = handle

    def close(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.idb_index_free(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001  (interpreter shutdown)
            pass

    @classmethod
    def from_graph(cls, points, zero, upper, M, ef_search=100, device=0, storage="f32", metric="l2sq"):
        """metric="cosine": the points are taken as given and must be unit rows (or all zeros) — see normalize()."""
        points, zero = f32(points), np.ascontiguousarray(zero, dtype=np.uint32)
        n, dim = points.shape
        ups = [np.ascontiguousarray(u, dtype=np.uint32) for u in upper]
        arr = (C.POINTER(C.c_uint32) * max(1, len(ups)))(*[ptr(u, C.c_uint32) for u in ups])
        un = np.array([u.shape[0] for u in ups] or [0], dtype=np.uint64)
        h = C.c_void_p()
        check(lib().idb_index_from_graph_ex(ptr(points, C.c_float), n, dim, M, ef_search, ptr(zero, C.c_uint32), len(ups), arr,
                                            ptr(un, C.c_uint64), STORAGE[storage], _metric(metric), device, C.byref(h)))
        return cls(h)

    @classmethod
    def build(cls, rows, progress=None, metric="l2sq", **kw):
        """progress: optional callable(done, total) — Builder::progress (lib.rs:70-75).  metric: "l2sq" or "cosine"."""
        rows = f32(rows)
        n, dim = rows.shape
        p = default_params(**kw)
        cb = None
        if progress is not None:
            cb = PROGRESS_FN(lambda done, total, _user: progress(int(done), int(total)))
            p.progress = C.cast(cb, C.c_void_p)
        ids = np.empty(n, dtype=np.uint32)
        h = C.c_void_p()
        check(lib().idb_build_ex(ptr(rows, C.c_float), n, dim, C.byref(p), _metric(metric), C.byref(h), ptr(ids, C.c_uint32)))
        return cls(h), ids

    def insert(self, rows, global_ids=None, progress=None, **kw):
        """Appends rows (m x dim) to the index on layer 0 (idb_index_insert_f32); returns their PointIds, n0 .. n0+m-1.
        kw: idb_params fields (ef_construction, heuristic, keep_pruned, insert_batch; M defaults to the index's).  global_ids: the
        rows' entries for the id map, required when the index has one."""
        rows = f32(rows)
        if rows.ndim == 1:
            rows = rows[None, :]
        m, dim = rows.shape
        kw.setdefault("M", int(self.info().M))
        p = default_params(**kw)
        cb = None
        if progress is not None:
            cb = PROGRESS_FN(lambda done, total, _user: progress(int(done), int(total)))
            p.progress = C.cast(cb, C.c_void_p)
        g = None
        if global_ids is not None:
            g = np.ascontiguousarray(global_ids, dtype=np.uint32)
            if g.shape != (m,):
                raise ValueError("global_ids must have one entry per row")
        ids = np.empty(m, dtype=np.uint32)
        check(lib().idb_index_insert_f32(self._h, ptr(rows, C.c_float), m, dim, C.byref(p), None if g is None else ptr(g, C.c_uint32),
                                         ptr(ids, C.c_uint32)))
        return ids

    def remove(self, pids, **kw):
        """Removes the points `pids` (distinct PointIds) from the index (idb_index_remove); returns new_ids (n entries): the PointId
        each point has afterwards, or INVALID for a removed one.  kw: idb_params fields (ef_construction, heuristic, keep_pruned;
        M defaults to the index's)."""
        pids = np.ascontiguousarray(pids, dtype=np.uint32).reshape(-1)
        kw.setdefault("M", int(self.info().M))
        p = default_params(**kw)
        n = int(self.info().n)
        new_ids = np.empty(max(n, 1), dtype=np.uint32)
        check(lib().idb_index_remove(self._h, ptr(pids, C.c_uint32), pids.shape[0], C.byref(p), ptr(new_ids, C.c_uint32)))
        return new_ids[:n]

    def save(self, path):
        check(lib().idb_index_save(self._h, os.fsencode(path)))

    @classmethod
    def load(cls, path, dim=300, M=32, device=0, metric="l2sq", storage="f32"):
        """Returns (Index, offset of the HnswMap values in the file).  The file records neither the metric nor the storage: it
        holds f32 rows, stored again as `storage` ("f32", "bf16", "f16", "q8" or "bin")."""
        h, off = C.c_void_p(), C.c_uint64()
        check(lib().idb_index_load_storage(os.fsencode(path), dim, M, _metric(metric), _storage(storage), device, C.byref(h),
                                           C.byref(off)))
        return cls(h), int(off.value)

    def info(self):
        i = Info()
        check(lib().idb_index_info(self._h, C.byref(i)))
        return i

    @property
    def metric(self):
        m = C.c_uint32()
        check(lib().idb_index_metric(self._h, C.byref(m)))
        return {v: k for k, v in METRIC.items()}[int(m.value)]

    def _queries(self, queries):
        """n x dim f32 matrix; narrower rows are zero-padded like the reference pads short points (py:363-375), wider ones rejected."""
        q = f32(queries)
        if q.ndim == 1:
            q = q[None, :]
        dim = int(self.info().dim)
        if q.shape[1] > dim:
            raise ValueError(f"query has {q.shape[1]} elements, the index holds {dim}-d points (py:369-370: 'point array too long')")
        if q.shape[1] < dim:
            q = np.ascontiguousarray(np.pad(q, ((0, 0), (0, dim - q.shape[1]))))
        return q

    def search(self, queries, ef_search=0, k=None):
        q = self._queries(queries)
        nq = q.shape[0]
        if k is None:
            k = ef_search or self.info().ef_search
        ids = np.empty((nq, k), dtype=np.uint32)
        dist = np.empty((nq, k), dtype=np.float32)
        lens = np.empty(nq, dtype=np.uint32)
        check(lib().idb_search_batch_f32(self._h, ptr(q, C.c_float), nq, ef_search, k, ptr(ids, C.c_uint32),
                                         ptr(dist, C.c_float), ptr(lens, C.c_uint32)))
        return ids, dist, lens

    def search_device(self, d_queries, nq, ef_search, k, d_ids, d_dist, d_len, lane=0):
        """Asynchronous: enqueues on submission lane `lane` (own stream; lanes overlap on the device)."""
        check(lib().idb_search_batch_device_lane(self._h, lane, d_queries, nq, ef_search, k, d_ids, d_dist, d_len))

    def exact_search(self, queries, k=10):
        """Exact k-NN over every stored row (idb_exact_search_batch_f32): (ids, dist, lens) laid out like search()."""
        q = self._queries(queries)
        nq = q.shape[0]
        ids = np.empty((nq, k), dtype=np.uint32)
        dist = np.empty((nq, k), dtype=np.float32)
        lens = np.empty(nq, dtype=np.uint32)
        check(lib().idb_exact_search_batch_f32(self._h, ptr(q, C.c_float), nq, k, ptr(ids, C.c_uint32), ptr(dist, C.c_float),
                                               ptr(lens, C.c_uint32)))
        return ids, dist, lens

    def exact_search_device(self, d_queries, nq, k, d_ids, d_dist, d_len, lane=0):
        """Asynchronous exact k-NN on device buffers, enqueued on submission lane `lane`."""
        check(lib().idb_exact_search_batch_device_lane(self._h, lane, d_queries, nq, k, d_ids, d_dist, d_len))

    def range_search(self, queries, radius, capacity=None):
        """Exact range search (idb_range_search_batch_f32): every point within `radius` of each query, as CSR (offsets u64 [nq + 1],
        ids u32 [total], dist f32 [total]); query i's hits are ids[offsets[i]:offsets[i + 1]], nearest first.  capacity=None: a first
        guess, and once more with the exact total when the hits did not fit."""
        return self._csr(lambda q, nq, cap, o, i, d: lib().idb_range_search_batch_f32(self._h, q, nq, float(radius), cap, o, i, d),
                         queries, capacity)

    def graph_range_search(self, queries, radius, ef_search=0, capacity=None):
        """Graph range search (idb_graph_range_search_batch_f32): the points within `radius` that layer 0 reaches from each query's
        approximate nearest neighbours (ef_search: 0 = the index's) — a subset of range_search()'s result, laid out the same way."""
        ef_search = _ef(ef_search)
        return self._csr(lambda q, nq, cap, o, i, d: lib().idb_graph_range_search_batch_f32(self._h, q, nq, ef_search, float(radius),
                                                                                            cap, o, i, d), queries, capacity)

    def _csr(self, call, queries, capacity):
        """A range entry call(queries, nq, capacity, offsets, ids, dist) as CSR; capacity=None: a first guess, and once more with the
        exact total when the hits did not fit."""
        q = self._queries(queries)
        nq = q.shape[0]
        guess = capacity is None
        cap = min(max(64 * nq, 1 << 16), RANGE_MAX_CAPACITY) if guess else int(capacity)
        offsets = np.empty(nq + 1, dtype=np.uint64)
        while True:
            ids = np.empty(cap, dtype=np.uint32)
            dist = np.empty(cap, dtype=np.float32)
            st = call(ptr(q, C.c_float), nq, cap, ptr(offsets, C.c_uint64), ptr(ids, C.c_uint32), ptr(dist, C.c_float))
            if st == ERR_CAPACITY and guess and int(offsets[-1]) > cap:  # (a graph range search's seed overflow is not a size)
                guess, cap = False, int(offsets[-1])
                continue
            check(st)
            total = int(offsets[-1])
            return offsets, ids[:total].copy(), dist[:total].copy()

    def range_search_device(self, d_queries, nq, radius, capacity, d_offsets, d_ids, d_dist, lane=0):
        """Exact range search on device buffers on submission lane `lane`; returns the total (raises IdbError with status
        ERR_CAPACITY, the offsets written, when it exceeds `capacity`).  Returns once the lane has run the call."""
        total = C.c_uint64()
        st = lib().idb_range_search_batch_device_lane(self._h, lane, d_queries, nq, float(radius), capacity, d_offsets, d_ids, d_dist,
                                                       C.byref(total))
        if st == ERR_CAPACITY:
            raise IdbError(st, lib().idb_last_error().decode("utf-8", "replace") + f" (total {int(total.value)})")
        check(st)
        return int(total.value)

    def graph_range_search_device(self, d_queries, nq, radius, capacity, d_offsets, d_ids, d_dist, ef_search=0, lane=0):
        """Graph range search on device buffers on submission lane `lane`; returns the total (raises IdbError with status
        ERR_CAPACITY, the offsets written, when it exceeds `capacity`).  Returns once the lane has run the call."""
        ef_search = _ef(ef_search)
        total = C.c_uint64()
        st = lib().idb_graph_range_search_batch_device_lane(self._h, lane, d_queries, nq, ef_search, float(radius), capacity, d_offsets,
                                                             d_ids, d_dist, C.byref(total))
        if st == ERR_CAPACITY:
            raise IdbError(st, lib().idb_last_error().decode("utf-8", "replace") + f" (total {int(total.value)})")
        check(st)
        return int(total.value)

    def lane_stream(self, lane):
        return lib().idb_index_lane_stream(self._h, lane)

    def last_retried(self, lane=0):
        out = C.c_uint32()
        check(lib().idb_last_search_retried(self._h, lane, C.byref(out)))
        return int(out.value)

    def last_full_fetches(self, lane=0xFFFFFFFF):
        """Candidate rows the last call fetched in full (all queries; equal to the summed distance counters when unscreened)."""
        out = C.c_uint64()
        check(lib().idb_last_search_full_fetches(self._h, lane, C.byref(out)))
        return int(out.value)

    KERNEL_FIELDS = ("ch", "row_t", "ef_t", "b", "bf16", "full", "tma", "variant")

    def last_kernel(self, lane=0xFFFFFFFF):
        """The search-kernel instantiation the last call launched, as a dict over KERNEL_FIELDS (all zeros: none launched).
        The "bf16" field carries the row type, a STORAGE value: 0 f32, 1 bf16, 2 f16, 4 q8, 8 bin."""
        out = (C.c_uint32 * 8)()
        check(lib().idb_last_search_kernel(self._h, lane, out))
        return dict(zip(self.KERNEL_FIELDS, (int(v) for v in out)))

    def screen_bound(self, queries, pairs):
        """(bound, canonical distance) per (query index, PointId) pair: the screening bound K1 compares with the furthest distance."""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        p = np.ascontiguousarray(pairs, dtype=np.uint32).reshape(-1, 2)
        bound = np.empty(p.shape[0], dtype=np.float32)
        dist = np.empty(p.shape[0], dtype=np.float32)
        check(lib().idb_debug_screen_bound(self._h, ptr(q, C.c_float), q.shape[0], ptr(p, C.c_uint32), p.shape[0],
                                           ptr(bound, C.c_float), ptr(dist, C.c_float)))
        return bound, dist

    def merge_topk(self, keys, k, premerge=False):
        """The sharded search's merge kernel on keys (G x nq x k u64): the merged keys (nq x k) when `premerge`, else
        (ids, dist, lens) with distances reported in this index's metric."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        G, nq, kk = keys.shape
        if kk != k:
            raise ValueError("keys must be G x nq x k")
        if premerge:
            out = np.empty((nq, k), dtype=np.uint64)
            check(lib().idb_debug_merge_topk(self._h, ptr(keys, C.c_uint64), G, nq, k, None, None, None, ptr(out, C.c_uint64)))
            return out
        ids = np.empty((nq, k), dtype=np.uint32)
        dist = np.empty((nq, k), dtype=np.float32)
        lens = np.empty(nq, dtype=np.uint32)
        check(lib().idb_debug_merge_topk(self._h, ptr(keys, C.c_uint64), G, nq, k, ptr(ids, C.c_uint32), ptr(dist, C.c_float),
                                         ptr(lens, C.c_uint32), None))
        return ids, dist, lens

    def last_failures(self, lane=0):
        out = C.c_uint32()
        check(lib().idb_last_search_failures(self._h, lane, C.byref(out)))
        return int(out.value)

    def set_id_map(self, global_ids):
        """global_ids[pid] = caller's id of the row that became PointId pid; None clears the map."""
        if global_ids is None:
            check(lib().idb_index_set_id_map(self._h, None))
            return
        g = np.ascontiguousarray(global_ids, dtype=np.uint32)
        if g.shape[0] != int(self.info().n):
            raise ValueError("id map must have one entry per point")
        check(lib().idb_index_set_id_map(self._h, ptr(g, C.c_uint32)))

    def sharded_search(self, comm, queries, ef_search=0, k=10):
        q = self._queries(queries)
        nq = q.shape[0]
        ids = np.empty((nq, k), dtype=np.uint32)
        dist = np.empty((nq, k), dtype=np.float32)
        lens = np.empty(nq, dtype=np.uint32)
        check(lib().idb_sharded_search_batch_f32(self._h, comm._h, ptr(q, C.c_float), nq, ef_search, k, ptr(ids, C.c_uint32),
                                                 ptr(dist, C.c_float), ptr(lens, C.c_uint32)))
        return ids, dist, lens

    def sharded_search_device(self, comm, d_queries, nq, ef_search, k, d_ids, d_dist, d_len):
        check(lib().idb_sharded_search_batch_device(self._h, comm._h, d_queries, nq, ef_search, k, d_ids, d_dist, d_len))

    def last_counters(self, nq):
        out = np.zeros((nq, 4), dtype=np.uint64)
        check(lib().idb_last_search_counters(self._h, nq, ptr(out, C.c_uint64)))
        return out

    def export_graph(self):
        i = self.info()
        n, dim, M = int(i.n), int(i.dim), int(i.M)
        pts = np.empty((n, dim), dtype=np.float32)
        zero = np.empty((n, 2 * M), dtype=np.uint32)
        if n:
            check(lib().idb_index_export_points(self._h, ptr(pts, C.c_float)))
            check(lib().idb_index_export_zero(self._h, ptr(zero, C.c_uint32)))
        upper = []
        for l in range(1, int(i.n_layers)):
            u = np.empty((int(i.layer_n[l]), M), dtype=np.uint32)
            check(lib().idb_index_export_upper(self._h, l, ptr(u, C.c_uint32)))
            upper.append(u)
        return pts, zero, upper

    def gather_bench(self, n_items=10000, batches=288, chain=0, reps=3):
        ms, by = C.c_float(), C.c_double()
        check(lib().idb_debug_gather_bench(self._h, n_items, batches, chain, reps, C.byref(ms), C.byref(by)))
        return float(ms.value), float(by.value)

    def gather_mix_bench(self, n_items=10000, batches=288, chain=0, reps=3, atomics=21, mode=1):
        ms, by = C.c_float(), C.c_double()
        check(lib().idb_debug_gather_mix_bench(self._h, n_items, batches, chain, reps, atomics, mode, C.byref(ms), C.byref(by)))
        return float(ms.value), float(by.value)

    def set_profiling(self, on=True):
        check(lib().idb_index_set_profiling(self._h, 1 if on else 0))

    def last_kernel_ms(self):
        ms, n = C.c_float(), C.c_uint32()
        check(lib().idb_index_last_kernel_ms(self._h, C.byref(ms), C.byref(n)))
        return float(ms.value), int(n.value)

    @property
    def stream(self):
        return lib().idb_index_stream(self._h)

    def sync(self):
        check(lib().idb_index_sync(self._h))


UNIQUE_ID_BYTES = 128


def comm_unique_id():
    buf = C.create_string_buffer(UNIQUE_ID_BYTES)
    check(lib().idb_comm_unique_id(buf))
    return bytes(buf.raw)


class Comm:
    """One NCCL communicator (idb_comm): rank `rank` of `world`, bound to CUDA device `device`."""

    def __init__(self, unique_id, rank, world, device):
        h = C.c_void_p()
        buf = C.create_string_buffer(unique_id, UNIQUE_ID_BYTES)
        check(lib().idb_comm_create(buf, rank, world, device, C.byref(h)))
        self._h, self.rank, self.world = h, rank, world

    def close(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.idb_comm_free(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001  (interpreter shutdown)
            pass


def _handles(shards):
    return (C.c_void_p * len(shards))(*[s._h for s in shards])


def sharded_search_multi(shards, comm, queries, ef_search=0, k=10):
    """Collective: this rank's shards (all on one device) + ONE all-gather over `comm`.  Host buffers."""
    q = shards[0]._queries(queries)
    nq = q.shape[0]
    ids = np.empty((nq, k), dtype=np.uint32)
    dist = np.empty((nq, k), dtype=np.float32)
    lens = np.empty(nq, dtype=np.uint32)
    check(lib().idb_sharded_search_batch_f32_multi(_handles(shards), len(shards), comm._h, ptr(q, C.c_float), nq, ef_search, k,
                                                   ptr(ids, C.c_uint32), ptr(dist, C.c_float), ptr(lens, C.c_uint32)))
    return ids, dist, lens


def sharded_search_multi_device(shards, comm, d_queries, nq, ef_search, k, d_ids, d_dist, d_len):
    """Device pointers; enqueues on lane 0 of shards[0] (every shard's stream is joined into it) and returns."""
    check(lib().idb_sharded_search_batch_device_multi(_handles(shards), len(shards), comm._h, d_queries, nq, ef_search, k, d_ids, d_dist, d_len))


def normalize(rows, device=0):
    """The canonical normalisation of every row on the device (idb_normalize_f32): what a cosine index stores for them."""
    rows = f32(rows)
    if rows.ndim == 1:
        rows = rows[None, :]
    out = np.empty_like(rows)
    check(lib().idb_normalize_f32(ptr(rows, C.c_float), rows.shape[0], rows.shape[1], device, ptr(out, C.c_float)))
    return out


def distance(a, b, device=0):
    a, b = f32(a), f32(b)
    out = C.c_float()
    check(lib().idb_distance_f32(ptr(a, C.c_float), ptr(b, C.c_float), a.shape[0], device, C.byref(out)))
    return np.float32(out.value)
