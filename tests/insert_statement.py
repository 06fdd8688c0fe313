"""ctypes loader of the CPU statement of the index insert (statements/insert_statement.cpp), which the GPU insert is checked against.

build_batched(rows, max_batch, growth, stop_at=None, **kw) -> (Graph, ids): the library's batched build, optionally stopped at the
first layer-0 batch boundary >= stop_at.  insert_batched(graph, rows, max_batch, growth, **kw) -> Graph: Construction::insert on
layer 0 of each row appended to `graph`, in the insert's batch schedule.  kw: oracle params (M, ef_construction, heuristic,
keep_pruned, ml, seed, metric, threads).  schedule(insert_batch) gives the (max_batch, growth) the library uses.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle as O

_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "statements")
_SO = os.path.join(_DIR, "_build", "libinsert_statement.so")
_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_SO):
        subprocess.check_call(["make", "-C", _DIR, "-s"])
    L = C.CDLL(_SO)
    u32p, f32p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_uint64)
    L.ins_build_batched.restype = C.c_void_p
    L.ins_build_batched.argtypes = [f32p, C.c_uint64, C.c_uint32, C.POINTER(O.Params), C.c_uint32, C.c_uint32, C.c_uint64, u32p]
    L.ins_insert_batched.restype = C.c_int
    L.ins_insert_batched.argtypes = [C.c_void_p, f32p, C.c_uint64, C.POINTER(O.Params), C.c_uint32, C.c_uint32]
    L.orc_from_graph.restype = C.c_void_p
    L.orc_from_graph.argtypes = [f32p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, u32p, C.c_uint32, C.POINTER(u32p), u64p,
                                 C.c_int32]
    L.orc_free.argtypes = [C.c_void_p]
    for name, rt in [("orc_n", C.c_uint64), ("orc_dim", C.c_uint32), ("orc_M", C.c_uint32), ("orc_num_layers", C.c_uint32)]:
        getattr(L, name).restype = rt
        getattr(L, name).argtypes = [C.c_void_p]
    L.orc_layer_count.restype = C.c_uint64
    L.orc_layer_count.argtypes = [C.c_void_p, C.c_uint32]
    L.orc_export_points.argtypes = [C.c_void_p, f32p]
    L.orc_export_zero.argtypes = [C.c_void_p, u32p]
    L.orc_export_upper.argtypes = [C.c_void_p, C.c_uint32, u32p]
    _lib = L
    return L


def schedule(insert_batch=0):
    """(max_batch, growth) of the build's and the insert's batch schedule for params.insert_batch (0: the defaults)."""
    return (insert_batch, 8) if insert_batch else (16384, 8)


def _export(h, ef_search):
    L = lib()
    n, dim, M = int(L.orc_n(h)), int(L.orc_dim(h)), int(L.orc_M(h))
    pts = np.empty((n, dim), dtype=np.float32)
    zero = np.empty((n, 2 * M), dtype=np.uint32)
    if n:
        L.orc_export_points(h, O._p(pts, C.c_float))
        L.orc_export_zero(h, O._p(zero, C.c_uint32))
    upper = []
    for l in range(1, int(L.orc_num_layers(h))):
        u = np.empty((int(L.orc_layer_count(h, l)), M), dtype=np.uint32)
        L.orc_export_upper(h, l, O._p(u, C.c_uint32))
        upper.append(u)
    return O.Graph(pts, zero, upper, M, ef_search)


def build_batched(rows, max_batch, growth, stop_at=None, threads=1, **kw):
    rows = O._f32(rows)
    n, dim = rows.shape
    p = O.default_params(threads=threads, **kw)
    ids = np.empty(n, dtype=np.uint32)
    h = lib().ins_build_batched(O._p(rows, C.c_float), n, dim, C.byref(p), max_batch, growth, n if stop_at is None else stop_at,
                                O._p(ids, C.c_uint32))
    if not h:
        raise ValueError("ins_build_batched failed")
    try:
        return _export(h, p.ef_search), ids
    finally:
        lib().orc_free(h)


def insert_batched(graph, rows, max_batch, growth, threads=1, **kw):
    """graph: an oracle Graph (points as stored, zero, upper); rows: m x dim, as the index stores them (normalised / bf16-rounded)."""
    pts, zero = O._f32(graph.points), np.ascontiguousarray(graph.zero, dtype=np.uint32)
    rows = O._f32(rows)
    if rows.ndim == 1:
        rows = rows[None, :]
    n, dim = pts.shape[0], rows.shape[1]
    pts = pts.reshape(n, dim)
    ups = [np.ascontiguousarray(u, dtype=np.uint32) for u in graph.upper]
    arr = (C.POINTER(C.c_uint32) * max(1, len(ups)))(*[O._p(u, C.c_uint32) for u in ups])
    un = np.array([u.shape[0] for u in ups] or [0], dtype=np.uint64)
    kw.setdefault("M", graph.M)
    p = O.default_params(threads=threads, **kw)
    h = lib().orc_from_graph(O._p(pts, C.c_float), n, dim, graph.M, graph.ef_search, O._p(zero, C.c_uint32), len(ups), arr,
                             O._p(un, C.c_uint64), p.metric)
    try:
        if lib().ins_insert_batched(h, O._p(rows, C.c_float), rows.shape[0], C.byref(p), max_batch, growth) != 0:
            raise ValueError("ins_insert_batched failed (M mismatch, extend_candidates, or N >= u32::MAX)")
        return _export(h, graph.ef_search)
    finally:
        lib().orc_free(h)
