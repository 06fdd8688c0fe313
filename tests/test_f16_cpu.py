"""fp16 row storage, the parts that need no device: the storage value passes every argument check (and stops at the device check),
the argument refusals of idb_index_load_storage, `Config.storage`, the K1 dispatch statement's fp16 cells, and numpy's fp16
rounding pinned against an integer statement of round-to-nearest-even (the GPU tests use numpy as the rounding reference)."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import f16_ref, k1_dispatch
from tests.conftest import _has_gpu
from tests.k1_dispatch import all_cells
from tests.k1_dispatch_f16 import f16_cells, k1_cell


def _abi():
    from instant_distance_b200 import _abi

    return _abi


ROWS = np.zeros((3, 4), np.float32)


def _build(storage):
    a = _abi()
    p = a.default_params(storage=storage)
    h = C.c_void_p()
    return a.lib().idb_build_ex(a.ptr(ROWS, C.c_float), 3, 4, C.byref(p), 0, C.byref(h), None)


def _adopt(storage):
    a = _abi()
    zero = np.full((3, 4), a.INVALID, np.uint32)
    h = C.c_void_p()
    return a.lib().idb_index_from_graph_ex(a.ptr(ROWS, C.c_float), 3, 4, 2, 10, a.ptr(zero, C.c_uint32), 0, None, None, storage, 0, 0,
                                           C.byref(h))


def _load(path, dim=4, M=2, metric=0, storage=2, out=True):
    a = _abi()
    h, off = C.c_void_p(), C.c_uint64()
    return a.lib().idb_index_load_storage(None if path is None else os.fsencode(path), dim, M, metric, storage, 0,
                                          C.byref(h) if out else None, C.byref(off))


@pytest.mark.parametrize("call", [_build, _adopt])
def test_storage_3_is_refused(call):
    a = _abi()
    assert call(3) == a.ERR_INVALID_ARG
    assert "unknown storage 3" in a.lib().idb_last_error().decode()


@pytest.mark.parametrize("call", [_build, _adopt])
def test_storage_f16_passes_the_argument_checks(call):
    if _has_gpu():
        pytest.skip("without a device only: with one, the call builds an index")
    a = _abi()
    assert call(a.STORAGE["f16"]) == a.ERR_CUDA


@pytest.mark.parametrize("case", ["null path", "null out", "dim 0", "M 1", "M 65", "metric 2", "storage 3"])
def test_load_storage_argument_refusals(tmp_path, case):
    a = _abi()
    kw = dict(path=str(tmp_path / "missing.idx"))
    if case == "null path":
        kw["path"] = None
    if case == "null out":
        kw["out"] = False
    if case == "dim 0":
        kw["dim"] = 0
    if case == "M 1":
        kw["M"] = 1
    if case == "M 65":
        kw["M"] = 65
    if case == "metric 2":
        kw["metric"] = 2
    if case == "storage 3":
        kw["storage"] = 3
    assert _load(**kw) == a.ERR_INVALID_ARG, a.lib().idb_last_error()


def test_load_storage_f16_passes_the_argument_checks(tmp_path):
    a = _abi()
    for storage in (0, 1, 2):
        assert _load(str(tmp_path / "missing.idx"), storage=storage) == a.ERR_IO


def test_config_storage_maps_to_the_abi_values():
    from instant_distance import Config

    c = Config()
    assert c.storage == "f32" and c._params()["storage"] == 0
    for name, value in (("bf16", 1), ("f16", 2)):
        c.storage = name
        assert c._params()["storage"] == value
        assert _abi().default_params(**c._params()).storage == value
    c.storage = "fp8"
    with pytest.raises(ValueError):
        c._params()


def test_f16_dispatch_equals_bf16_but_for_the_row_type():
    """tests/k1_dispatch_f16.py agrees with tests/k1_dispatch.py on f32 and bf16 rows (IDB_VARIANT cases included), and its fp16
    cell is the bf16 cell of tests/k1_dispatch.py with the row type 2."""
    for dim in (3, 100, 128, 129, 256, 300, 384, 512, 700, 768, 1024, 1025, 2049):
        for M in (2, 16, 32, 33, 64):
            for ef in (1, 10, 100, 128, 129, 257, 513, 1024):
                for v in range(0, 9):
                    for storage in ("f32", "bf16"):
                        assert k1_cell(dim, M, ef, 5000, storage, v) == k1_dispatch.k1_cell(dim, M, ef, 5000, storage, v)
                    bf = k1_dispatch.k1_cell(dim, M, ef, 5000, "bf16")
                    assert k1_cell(dim, M, ef, 5000, "f16", v) == bf._replace(bf16=2)  # the variants are f32 instantiations


def test_f16_cells_are_91_and_all_reachable():
    from tests.test_gpu_k1_f16_instantiations import planned_cells

    cells = f16_cells()
    assert len(cells) == 91 and not (cells & all_cells()) and len(all_cells()) == 190
    assert {c._replace(bf16=1) for c in cells} == {c for c in all_cells() if c.bf16 == 1}
    assert planned_cells() == cells


def test_numpy_f16_rounding_is_round_to_nearest_even():
    x = f16_ref.boundary_values()
    assert (x.astype(np.float16).view(np.uint16) == f16_ref.rne_bits(x)).all()
    # ties: a midpoint goes to the neighbour with an even mantissa
    v = np.arange(0x7C00, dtype=np.uint16).view(np.float16).astype(np.float32)
    mid = ((v[:-1].astype(np.float64) + v[1:]) / 2).astype(np.float32)
    got = f16_ref.rne_bits(mid)
    lo = np.arange(0x7C00 - 1, dtype=np.uint16)
    assert (got == np.where(lo % 2 == 0, lo, lo + 1)).all()
    assert f16_ref.rne_bits(np.float32([65519.996, 65520, -70000, np.inf, -np.inf, 0.0, -0.0])).tolist() == [
        0x7BFF, 0x7C00, 0xFC00, 0x7C00, 0xFC00, 0, 0x8000]
    nan = np.float32([np.nan, -np.nan]).astype(np.float16)
    assert np.isnan(nan).all() and nan.view(np.uint16).tolist() == [0x7E00, 0xFE00]
