"""CPU-side checks of the exact search's entry points: both are exported, every argument error is reported without a device, and a
valid call without a device fails loudly (no CPU fallback)."""
import ctypes as C

import numpy as np
import pytest

from tests.conftest import _has_gpu

ENTRIES = ("idb_exact_search_batch_f32", "idb_exact_search_batch_device_lane")


def _abi():
    from instant_distance_b200 import _abi

    return _abi


def _calls(index, queries, nq, k, out_ids, lane=0):
    """Both entries with the same arguments (the host one has no lane)."""
    L = _abi().lib()
    return (L.idb_exact_search_batch_f32(index, queries, nq, k, out_ids, None, None),
            L.idb_exact_search_batch_device_lane(index, lane, queries, nq, k, out_ids, None, None))


def test_both_entries_are_exported():
    abi = _abi()
    L = abi.lib()
    for name in ENTRIES:
        assert hasattr(L, name) and name in abi.SYMBOLS


def test_argument_errors_need_no_device():
    abi = _abi()
    # argument checks come before the handle is used, so any non-null pointer stands in for an index here
    fake = C.c_void_p(C.addressof(C.create_string_buffer(64)))
    q = np.zeros((2, 4), dtype=np.float32)
    qp = q.ctypes.data_as(C.POINTER(C.c_float))
    ids = np.zeros((2, 8), dtype=np.uint32)
    ip = ids.ctypes.data_as(C.POINTER(C.c_uint32))
    assert _calls(None, qp, 2, 8, ip) == (abi.ERR_INVALID_ARG,) * 2  # null index
    assert _calls(fake, None, 2, 8, ip) == (abi.ERR_INVALID_ARG,) * 2  # null queries with nq > 0
    assert _calls(fake, qp, 2, 8, None) == (abi.ERR_INVALID_ARG,) * 2  # null out_ids
    assert _calls(fake, qp, 2, 0, ip) == (abi.ERR_INVALID_ARG,) * 2  # k == 0
    assert _calls(fake, qp, 2, 1025, ip) == (abi.ERR_UNSUPPORTED,) * 2  # k > 1024
    n_lanes = abi.lib().idb_index_num_lanes()
    assert abi.lib().idb_exact_search_batch_device_lane(fake, n_lanes, qp, 2, 8, ip, None, None) == abi.ERR_INVALID_ARG
    assert _calls(fake, None, 0, 8, None) == (abi.OK,) * 2  # nq == 0: nothing to do, nothing written
    assert ids.max() == 0


@pytest.mark.skipif(_has_gpu(), reason="checks the no-device behaviour")
def test_valid_call_fails_loudly_without_a_device():
    abi = _abi()
    fake = C.c_void_p(C.addressof(C.create_string_buffer(64)))
    q = np.zeros((2, 4), dtype=np.float32)
    ids = np.zeros((2, 8), dtype=np.uint32)
    st = _calls(fake, q.ctypes.data_as(C.POINTER(C.c_float)), 2, 8, ids.ctypes.data_as(C.POINTER(C.c_uint32)))
    assert st == (abi.ERR_CUDA,) * 2
    assert b"no CPU fallback" in abi.lib().idb_last_error()
