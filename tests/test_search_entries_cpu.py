"""CPU-side checks of the nine search entry points: the status each one returns for every argument error, with and without queries,
and that a valid call without a device fails loudly (no CPU fallback) before it touches the index handle.

The three families order their checks differently, and those differences are pinned here as they are:
- an approximate or sharded call with nq = 0 accepts k = 0; an exact call refuses it, and refuses k > 1024;
- a lane out of range is refused even when nq = 0;
- a sharded call checks its comm before anything else and its shard list only when nq > 0."""
import ctypes as C

import numpy as np
import pytest

from tests.conftest import _has_gpu

APPROX = ("idb_search_batch_f32", "idb_search_batch_device", "idb_search_batch_device_lane")
EXACT = ("idb_exact_search_batch_f32", "idb_exact_search_batch_device_lane")
SHARDED = ("idb_sharded_search_batch_f32", "idb_sharded_search_batch_device", "idb_sharded_search_batch_f32_multi",
           "idb_sharded_search_batch_device_multi")
ENTRIES = APPROX + EXACT + SHARDED
HAS_LANE = {"idb_search_batch_device_lane", "idb_exact_search_batch_device_lane"}

# Argument checks come before the handles are used, so any non-null pointer stands in for an index or a comm in these rows.
_FAKE_INDEX = C.create_string_buffer(64)
_FAKE_COMM = C.create_string_buffer(64)
FAKE = C.addressof(_FAKE_INDEX)
FAKE_COMM = C.addressof(_FAKE_COMM)


def _abi():
    from instant_distance_b200 import _abi

    return _abi


def _call(name, index, comm, queries, nq, k, out_ids, lane):
    """Calls one entry; the arguments an entry does not take are dropped."""
    L = _abi().lib()
    fn = getattr(L, name)
    queries = None if queries is None else C.cast(C.c_void_p(queries), C.POINTER(C.c_float))
    out_ids = None if out_ids is None else C.cast(C.c_void_p(out_ids), C.POINTER(C.c_uint32))
    if name in ("idb_search_batch_f32", "idb_search_batch_device"):
        return fn(index, queries, nq, 0, k, out_ids, None, None)
    if name == "idb_search_batch_device_lane":
        return fn(index, lane, queries, nq, 0, k, out_ids, None, None)
    if name == "idb_exact_search_batch_f32":
        return fn(index, queries, nq, k, out_ids, None, None)
    if name == "idb_exact_search_batch_device_lane":
        return fn(index, lane, queries, nq, k, out_ids, None, None)
    if name.endswith("_multi"):
        shards = (C.c_void_p * 1)(index)
        return fn(shards, 1, comm, queries, nq, 0, k, out_ids, None, None)
    return fn(index, comm, queries, nq, 0, k, out_ids, None, None)


def _family(name):
    return "approx" if name in APPROX else "exact" if name in EXACT else "sharded"


# (row, family) -> expected status name for nq = 2 and for nq = 0.  None: the call would go on to use the fake handle, so the row is
# not run with it.  Rows about a lane apply to the lane entries only, rows about a comm to the sharded ones only.
ROWS = {
    "null_index": {"approx": ("ERR_INVALID_ARG", "ERR_INVALID_ARG"), "exact": ("ERR_INVALID_ARG", "ERR_INVALID_ARG"),
                   "sharded": ("ERR_INVALID_ARG", "OK")},
    "null_queries": {"approx": ("ERR_INVALID_ARG", "OK"), "exact": ("ERR_INVALID_ARG", "OK"), "sharded": ("ERR_INVALID_ARG", "OK")},
    "null_out_ids": {"approx": ("ERR_INVALID_ARG", "OK"), "exact": ("ERR_INVALID_ARG", "OK"), "sharded": ("ERR_INVALID_ARG", "OK")},
    "null_comm": {"sharded": ("ERR_INVALID_ARG", "ERR_INVALID_ARG")},
    "k_0": {"approx": ("ERR_INVALID_ARG", "OK"), "exact": ("ERR_INVALID_ARG", "ERR_INVALID_ARG"), "sharded": ("ERR_INVALID_ARG", "OK")},
    "k_1025": {"approx": (None, "OK"), "exact": ("ERR_UNSUPPORTED", "ERR_UNSUPPORTED"), "sharded": (None, "OK")},
    "lane_out_of_range": {"approx": ("ERR_INVALID_ARG", "ERR_INVALID_ARG"), "exact": ("ERR_INVALID_ARG", "ERR_INVALID_ARG")},
    "valid": {"approx": (None, "OK"), "exact": (None, "OK"), "sharded": (None, "OK")},
}


def _cases():
    for name in ENTRIES:
        for row, fam in ROWS.items():
            if _family(name) not in fam:
                continue
            if row == "lane_out_of_range" and name not in HAS_LANE:
                continue
            for nq, want in zip((2, 0), fam[_family(name)]):
                if want is not None:
                    yield pytest.param(name, row, nq, want, id=f"{name}-{row}-nq{nq}")


@pytest.mark.parametrize("name,row,nq,want", list(_cases()))
def test_argument_status(name, row, nq, want):
    abi = _abi()
    q = np.zeros((2, 4), dtype=np.float32)
    ids = np.zeros((2, 1025), dtype=np.uint32)
    args = dict(index=FAKE, comm=FAKE_COMM, queries=q.ctypes.data, nq=nq, k=8, out_ids=ids.ctypes.data, lane=0)
    if row == "null_index":
        args["index"] = None
    elif row == "null_queries":
        args["queries"] = None
    elif row == "null_out_ids":
        args["out_ids"] = None
    elif row == "null_comm":
        args["comm"] = None
    elif row == "k_0":
        args["k"] = 0
    elif row == "k_1025":
        args["k"] = 1025
    elif row == "lane_out_of_range":
        args["lane"] = abi.lib().idb_index_num_lanes()
    st = _call(name, **args)
    assert st == getattr(abi, want), (st, abi.lib().idb_last_error())
    assert ids.max() == 0 and q.max() == 0  # nothing was written


@pytest.mark.skipif(_has_gpu(), reason="checks the no-device behaviour")
@pytest.mark.parametrize("name", ENTRIES)
def test_valid_call_fails_loudly_without_a_device(name):
    abi = _abi()
    q = np.zeros((2, 4), dtype=np.float32)
    ids = np.zeros((2, 8), dtype=np.uint32)
    st = _call(name, FAKE, FAKE_COMM, q.ctypes.data, 2, 8, ids.ctypes.data, 0)
    assert st == abi.ERR_CUDA
    assert b"no CPU fallback" in abi.lib().idb_last_error()
