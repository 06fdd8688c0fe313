"""CPU-side checks of the graph range search's entry points: both are exported, every argument error is reported without a device (also
at nq = 0), nq = 0 succeeds with an empty result, and a valid call without a device fails loudly (no CPU fallback)."""
import ctypes as C

import numpy as np
import pytest

from tests.conftest import _has_gpu

ENTRIES = ("idb_graph_range_search_batch_f32", "idb_graph_range_search_batch_device_lane")
NAN = float("nan")


def _abi():
    from instant_distance_b200 import _abi

    return _abi


def _fake():
    """Argument checks come before the handle is used, so any non-null pointer stands in for an index here."""
    return C.c_void_p(C.addressof(C.create_string_buffer(64)))


class _Bufs:
    def __init__(self, nq=2):
        self.q = np.zeros((nq, 4), dtype=np.float32)
        self.offsets = np.full(nq + 1, 7, dtype=np.uint64)
        self.ids = np.zeros(8, dtype=np.uint32)
        self.total = C.c_uint64(7)
        self.qp = self.q.ctypes.data_as(C.POINTER(C.c_float))
        self.op = self.offsets.ctypes.data_as(C.POINTER(C.c_uint64))
        self.ip = self.ids.ctypes.data_as(C.POINTER(C.c_uint32))


def _calls(index, queries, nq, radius, capacity, offsets, ids, ef=0, lane=0, b=None):
    """Both entries with the same arguments (the host one has no lane and no out_total)."""
    L = _abi().lib()
    return (L.idb_graph_range_search_batch_f32(index, queries, nq, ef, radius, capacity, offsets, ids, None),
            L.idb_graph_range_search_batch_device_lane(index, lane, queries, nq, ef, radius, capacity, offsets, ids, None,
                                                       C.byref(b.total)))


def test_both_entries_are_exported():
    abi = _abi()
    L = abi.lib()
    for name in ENTRIES:
        assert hasattr(L, name) and name in abi.SYMBOLS


@pytest.mark.parametrize("nq", [0, 2])
def test_argument_errors_need_no_device(nq):
    abi = _abi()
    fake, b = _fake(), _Bufs()
    bad = (abi.ERR_INVALID_ARG,) * 2
    assert _calls(None, b.qp, nq, 1.0, 8, b.op, b.ip, b=b) == bad  # null index
    assert _calls(fake, b.qp, nq, 1.0, 8, b.op, None, b=b) == bad  # capacity > 0 with null ids
    assert _calls(fake, b.qp, nq, NAN, 8, b.op, b.ip, b=b) == bad  # NaN radius
    assert _calls(fake, b.qp, nq, 1.0, 8, b.op, b.ip, ef=1025, b=b) == bad  # ef_search above 1024
    assert _calls(fake, b.qp, nq, 1.0, 8, b.op, b.ip, ef=0xFFFFFFFF, b=b) == bad
    assert _calls(fake, b.qp, nq, 1.0, 1 << 31, b.op, b.ip, b=b) == (abi.ERR_UNSUPPORTED,) * 2  # capacity above 2^31 - 1
    L = abi.lib()
    n_lanes = L.idb_index_num_lanes()
    assert L.idb_graph_range_search_batch_device_lane(fake, n_lanes, b.qp, nq, 0, 1.0, 8, b.op, b.ip, None,
                                                      C.byref(b.total)) == abi.ERR_INVALID_ARG
    assert L.idb_graph_range_search_batch_device_lane(fake, 0, b.qp, nq, 0, 1.0, 8, b.op, b.ip, None, None) == abi.ERR_INVALID_ARG
    if nq:
        assert _calls(fake, None, nq, 1.0, 8, b.op, b.ip, b=b) == bad  # null queries
        assert _calls(fake, b.qp, nq, 1.0, 8, None, b.ip, b=b) == bad  # null offsets
    assert (b.offsets == 7).all() and b.total.value == 7 and b.ids.max() == 0  # nothing written


def test_query_count_over_the_int_limit_needs_no_device():
    abi = _abi()
    fake, b = _fake(), _Bufs()
    assert _calls(fake, b.qp, abi.RANGE_MAX_CAPACITY, 1.0, 8, b.op, b.ip, b=b) == (abi.ERR_UNSUPPORTED,) * 2
    assert (b.offsets == 7).all() and b.total.value == 7


def test_no_queries_is_an_empty_result():
    abi = _abi()
    fake, b = _fake(), _Bufs()
    assert _calls(fake, None, 0, 1.0, 0, b.op, None, ef=1024, b=b) == (abi.OK,) * 2
    assert b.offsets[0] == 0 and (b.offsets[1:] == 7).all()  # the host entry writes offsets[0]
    assert b.total.value == 0  # the device entry reports a total of 0 (and writes nothing on the device)
    assert _calls(fake, None, 0, -5.0, 0, None, None, b=b) == (abi.OK,) * 2  # no offsets to write


@pytest.mark.skipif(_has_gpu(), reason="checks the no-device behaviour")
def test_valid_call_fails_loudly_without_a_device():
    abi = _abi()
    fake, b = _fake(), _Bufs()
    for cap, ids in ((8, b.ip), (0, None)):
        assert _calls(fake, b.qp, 2, 1.0, cap, b.op, ids, ef=16, b=b) == (abi.ERR_CUDA,) * 2
        assert b"no CPU fallback" in abi.lib().idb_last_error()


@pytest.mark.parametrize("ef", [-1, 1 << 32, (1 << 32) + 100])
def test_the_binding_refuses_a_width_ctypes_would_wrap(ef):
    abi = _abi()
    ix = abi.Index(_fake())
    try:
        with pytest.raises(ValueError):
            ix.graph_range_search(np.zeros((1, 4), np.float32), 1.0, ef_search=ef)
        with pytest.raises(ValueError):
            ix.graph_range_search_device(0, 1, 1.0, 0, 0, 0, 0, ef_search=ef)
    finally:
        ix._h = None  # not a real handle: nothing to free
