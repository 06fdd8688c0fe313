"""CPU-side checks of idb_index_insert_f32: the argument errors it reports before it touches the index handle, and that a valid call
without a device fails loudly (no CPU fallback).  The checks that need the index (dim, M, the id map, n0 + m) are in
tests/test_gpu_insert.py."""
import ctypes as C

import numpy as np
import pytest

from tests.conftest import _has_gpu

_FAKE_INDEX = C.create_string_buffer(64)
FAKE = C.addressof(_FAKE_INDEX)


def _abi():
    from instant_distance_b200 import _abi

    return _abi


def _insert(index, rows, m, params):
    a = _abi()
    ids = np.empty(max(m, 1), np.uint32)
    rp = None if rows is None else a.ptr(rows, C.c_float)
    return a.lib().idb_index_insert_f32(index, rp, m, 4, None if params is None else C.byref(params), None, a.ptr(ids, C.c_uint32))


ROWS = np.zeros((3, 4), np.float32)


@pytest.mark.parametrize("case,status", [
    ("null index", "ERR_INVALID_ARG"),
    ("null params", "ERR_INVALID_ARG"),
    ("null rows", "ERR_INVALID_ARG"),
    ("ef_construction 0", "ERR_UNSUPPORTED"),
    ("ef_construction 1025", "ERR_UNSUPPORTED"),
    ("extend_candidates", "ERR_UNSUPPORTED"),
])
def test_argument_errors_come_before_the_handle(case, status):
    a = _abi()
    p = a.default_params()
    index, rows = FAKE, ROWS
    if case == "null index":
        index = None
    if case == "null rows":
        rows = None
    if case == "ef_construction 0":
        p.ef_construction = 0
    if case == "ef_construction 1025":
        p.ef_construction = 1025
    if case == "extend_candidates":
        p.extend_candidates = 1
    st = _insert(index, rows, 3, None if case == "null params" else p)
    assert st == getattr(a, status), a.lib().idb_last_error()


def test_null_rows_are_fine_when_there_are_none():
    if _has_gpu():
        pytest.skip("without a device only: a valid call would use the fake handle")
    a = _abi()
    assert _insert(FAKE, None, 0, a.default_params()) == a.ERR_CUDA


def test_valid_call_without_a_device_fails_loudly():
    if _has_gpu():
        pytest.skip("without a device only")
    a = _abi()
    assert _insert(FAKE, ROWS, 3, a.default_params()) == a.ERR_CUDA
    assert "no CPU fallback" in a.lib().idb_last_error().decode()
