"""bin row storage, the parts that need no device: the ABI constant in every binding, the storage value passing every argument check
(and stopping at the device check), cosine with bin refused before the device, `Config.storage`, the byte layout and the refusal rule
of tests/bin_ref.py, and K1's bin dispatch cells."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tests import bin_ref, k1_dispatch
from tests.conftest import ROOT, _has_gpu
from tests.k1_dispatch_bin import bin_cells, k1_cell
from tests.k1_dispatch_f16 import f16_cells
from tests.k1_dispatch_q8 import q8_cells


def _abi():
    from instant_distance_b200 import _abi

    return _abi


# ---- the constant ------------------------------------------------------------------------------------------------------------

def test_storage_bin_is_8_in_every_binding():
    header = open(os.path.join(ROOT, "include", "instant_distance_b200.h")).read()
    rust = open(os.path.join(ROOT, "instant-distance_b200", "rust", "src", "lib.rs")).read()
    assert re.search(r"#define IDB_STORAGE_BIN 8u\b", header)
    assert re.search(r"pub const STORAGE_BIN: u32 = 8;", rust)
    assert _abi().STORAGE["bin"] == 8


def test_config_storage_bin_maps_to_8():
    from instant_distance import Config

    c = Config()
    c.storage = "bin"
    assert c._params()["storage"] == 8
    assert _abi().default_params(**c._params()).storage == 8


# ---- argument checks before the device ---------------------------------------------------------------------------------------

ROWS = np.zeros((3, 4), np.float32)


def _build(storage, metric=0):
    a = _abi()
    p = a.default_params(storage=storage)
    h = C.c_void_p()
    return a.lib().idb_build_ex(a.ptr(ROWS, C.c_float), 3, 4, C.byref(p), metric, C.byref(h), None)


def _adopt(storage, metric=0):
    a = _abi()
    zero = np.full((3, 4), a.INVALID, np.uint32)
    h = C.c_void_p()
    return a.lib().idb_index_from_graph_ex(a.ptr(ROWS, C.c_float), 3, 4, 2, 10, a.ptr(zero, C.c_uint32), 0, None, None, storage,
                                           metric, 0, C.byref(h))


def _load(path, storage, metric=0):
    a = _abi()
    h, off = C.c_void_p(), C.c_uint64()
    return a.lib().idb_index_load_storage(os.fsencode(path), 4, 2, metric, storage, 0, C.byref(h), C.byref(off))


@pytest.mark.parametrize("call", [_build, _adopt])
def test_storage_bin_passes_the_argument_checks(call):
    if _has_gpu():
        pytest.skip("without a device only: with one, the call builds an index")
    assert call(8) == _abi().ERR_CUDA


@pytest.mark.parametrize("call", [_build, _adopt])
@pytest.mark.parametrize("storage", [5, 6, 7, 9])
def test_storages_5_to_7_and_above_8_are_refused(call, storage):
    a = _abi()
    assert call(storage) == a.ERR_INVALID_ARG
    assert f"unknown storage {storage}" in a.lib().idb_last_error().decode()


@pytest.mark.parametrize("call", [_build, _adopt])
def test_cosine_with_bin_is_unsupported(call):
    a = _abi()
    assert call(8, metric=1) == a.ERR_UNSUPPORTED
    assert "bin storage takes the squared L2 only" in a.lib().idb_last_error().decode()


def test_load_storage_bin_checks(tmp_path):
    a = _abi()
    missing = str(tmp_path / "missing.idx")
    assert _load(missing, 8) == a.ERR_IO
    assert _load(missing, 8, metric=1) == a.ERR_UNSUPPORTED  # refused before the file is read
    assert _load(missing, 7) == a.ERR_INVALID_ARG


# ---- the byte layout and the refusal rule ------------------------------------------------------------------------------------

def test_element_4c_plus_k_is_bit_k_of_byte_c():
    for dim in (1, 4, 5, 37, 128):
        for e in range(dim):
            x = np.zeros((1, dim), np.float32)
            x[0, e] = 1.0
            codes = bin_ref.pack(x)
            assert codes.shape == (1, (dim + 3) // 4)
            want = np.zeros_like(codes)
            want[0, e // 4] = 1 << (e % 4)
            assert (codes == want).all(), (dim, e)


@pytest.mark.parametrize("dim", [1, 3, 4, 16, 37, 300, 1025])
def test_pack_unpack_round_trip_and_zero_high_nibble(dim):
    r = np.random.default_rng(dim)
    x = (r.random((200, dim)) < 0.5).astype(np.float32)
    x[0] = 1.0  # every bit set: the ragged last chunk still leaves its padding bits and the high nibble clear
    x[1] = -0.0  # stored as 0
    codes = bin_ref.pack(x)
    assert (codes >> 4 == 0).all()
    assert bin_ref.unpack(codes, dim).tobytes() == np.where(x == 1.0, np.float32(1), np.float32(0)).tobytes()
    if dim % 4:
        assert (codes[0, -1] >> (dim % 4) == 0) and codes[0, -1] == (1 << (dim % 4)) - 1


def test_refusal_table():
    f = np.float32
    accepted = np.array([0.0, -0.0, 1.0], f)
    refused = np.array([0.5, 2.0, -1.0, np.nan, -np.nan, np.inf, -np.inf, np.finfo(f).smallest_subnormal,
                        -np.finfo(f).smallest_subnormal, np.nextafter(f(1), f(2)), np.nextafter(f(1), f(0)), f(1e-30)], f)
    assert not bin_ref.refused(accepted).any()
    assert bin_ref.refused(refused).all()
    payload_nan = np.array([0x7FC00001, 0xFF800001], np.uint32).view(np.float32)
    assert bin_ref.refused(payload_nan).all()


def test_hamming_equals_the_canonical_chain_on_0_1_rows():
    """For 0/1 rows every (q_i - x_i)^2 is 0 or 1, so the f32 sums of any order are exact integers: the Hamming distance."""
    r = np.random.default_rng(5)
    q = (r.random((20, 333)) < 0.5).astype(np.float32)
    x = (r.random((50, 333)) < 0.5).astype(np.float32)
    h = bin_ref.hamming(q, x)
    d = ((q[:, None, :] - x[None, :, :]) ** 2).astype(np.float32).sum(axis=2, dtype=np.float32)
    assert (d == h).all() and (h == (q[:, None, :] != x[None, :, :]).sum(axis=2)).all()


# ---- K1's bin cells ----------------------------------------------------------------------------------------------------------

def test_bin_dispatch_is_the_q8_dispatch_with_row_type_8():
    for dim in (3, 16, 37, 100, 128, 129, 256, 300, 384, 512, 700, 768, 1024, 1025, 2049):
        for M in (2, 16, 32, 33, 64):
            for ef in (1, 10, 100, 128, 129, 257, 513, 1024):
                for v in range(0, 9):
                    want = k1_dispatch.k1_cell(dim, M, ef, 5000, "bf16")._replace(bf16=8)
                    assert k1_cell(dim, M, ef, 5000, "bin", v) == want
                    assert k1_cell(dim, M, ef, 5000, "f32", v) == k1_dispatch.k1_cell(dim, M, ef, 5000, "f32", v)


def test_bin_cells_are_91_and_all_planned():
    from tests.test_gpu_k1_bin_instantiations import planned_cells

    cells = bin_cells()
    assert len(cells) == 91 and not (cells & (k1_dispatch.all_cells() | f16_cells() | q8_cells()))
    assert {c._replace(bf16=4) for c in cells} == q8_cells()
    assert planned_cells() == cells
