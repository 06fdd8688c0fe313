"""q8 row storage, the parts that need no device: tests/q8_ref.py (the quantiser the GPU tests compare against) pinned against an
integer-only statement of it and checked for its properties, the storage value passing every argument check (and stopping at the
device check), `Config.storage`, and K1's q8 dispatch cells."""
import ctypes as C
import os
import struct

import numpy as np
import pytest

from tests import k1_dispatch, q8_ref
from tests.conftest import _has_gpu
from tests.k1_dispatch import all_cells
from tests.k1_dispatch_f16 import f16_cells
from tests.k1_dispatch_q8 import k1_cell, q8_cells

SHIFT = 149  # x * 2^149 is an integer for every finite f32


def _int_of(x):
    """x * 2^149 as a Python int, from the f32 bits alone."""
    u = struct.unpack("<I", struct.pack("<f", float(x)))[0]
    sign, ex, man = u >> 31, (u >> 23) & 0xFF, u & 0x7FFFFF
    assert ex != 0xFF
    m, k = (man, -149) if ex == 0 else (man | 0x800000, ex - 150)
    v = m << (k + SHIFT)
    return -v if sign else v


def _floor_div(v, e):  # floor(v / 2^(e + 149)) for an int v
    s = e + SHIFT
    return v >> s if s >= 0 else v << -s


def _ceil_div(v, e):
    return -_floor_div(-v, e)


def _rint_div(v, e):  # round to nearest, ties to even, of v / 2^(e + 149)
    s = e + SHIFT
    if s <= 0:
        return v << -s
    q, r = v >> s, v & ((1 << s) - 1)
    half = 1 << (s - 1)
    return q + 1 if r > half or (r == half and q & 1) else q


def int_grid(row):
    """(e, b, c) of one row by brute force over e, in integers only."""
    X = [_int_of(x) for x in row]
    A = max(abs(v) for v in X)
    if A == 0:
        return -149, 0, [0] * len(X)
    e_lo = max(-149, A.bit_length() - 1 - SHIFT - 23)
    lo, hi = min(X), max(X)
    e = next(e for e in range(-149, 200) if e >= e_lo and _ceil_div(hi, e) - _floor_div(lo, e) <= 255)
    b = _floor_div(lo, e)
    return e, b, [_rint_div(v, e) - b for v in X]


def int_refused(row):
    e, b, c = int_grid(row)
    return max(abs(b), max(abs(b + ci) for ci in c)) * 2 ** (e + SHIFT) >= 2 ** (128 + SHIFT)


def _random_rows(n, dim, seed):
    r = np.random.default_rng(seed)
    out = []
    for i in range(n):
        kind = i % 6
        scale = np.float32(2.0) ** r.integers(-120, 100)
        if kind == 0:
            x = r.standard_normal(dim) * scale
        elif kind == 1:
            x = np.abs(r.standard_normal(dim)) * scale
        elif kind == 2:
            x = 1000 + r.standard_normal(dim) * 1e-3
        elif kind == 3:
            x = r.integers(-300, 300, dim) * scale
        elif kind == 4:
            x = np.full(dim, r.standard_normal() * scale)
        else:
            x = r.standard_normal(dim) * np.float32(2.0) ** r.integers(-149, -125, dim)  # subnormal and tiny
        out.append(np.asarray(x, np.float32))
    return out


def _rows():
    rows = list(q8_ref.boundary_rows(8)) + list(q8_ref.boundary_rows(3))
    for dim in (1, 2, 7, 37, 128, 300):
        rows += _random_rows(40, dim, dim)
    return rows


def test_q8_ref_equals_the_integer_statement():
    for row in _rows():
        e, b, c = q8_ref.grid(row[None, :])
        ie, ib, ic = int_grid(row)
        assert (int(e[0]), int(b[0]), c[0].tolist()) == (ie, ib, ic), row


def test_rint_ties_go_to_even():
    s = np.ldexp(1.0, -3)
    for k in range(20):
        row = np.float32([0.0, (k + 0.5) * s, 255 * s])
        e, b, c = q8_ref.grid(row[None, :])
        assert e[0] == -3 and c[0, 1] == (k if k % 2 == 0 else k + 1)


def test_span_of_exactly_255_steps_and_one_ulp_either_side():
    for e in (-140, -20, 0, 60, 100):
        s = np.ldexp(1.0, e)
        for lo in (0.0, -7.0, 3.0):
            top = np.float32((lo + 255) * s)
            assert q8_ref.grid(np.float32([[lo * s, top]]))[0][0] == e
            above = np.nextafter(top, np.float32(np.inf))
            assert q8_ref.grid(np.float32([[lo * s, above]]))[0][0] == e + 1
            below = np.nextafter(top, np.float32(-np.inf))
            assert q8_ref.grid(np.float32([[lo * s, below]]))[0][0] <= e


def test_e_lo_clamp_on_constant_rows_and_dim_1():
    for v in (1.0, 3.0, -1000.0, 1e-45, -2.5e-40, 3.3e38, np.ldexp(1.0, 24)):
        for dim in (1, 5):
            row = np.full((1, dim), v, np.float32)
            e, b, c = q8_ref.grid(row)
            A = abs(float(np.float32(v)))
            assert e[0] == max(-149, int(np.frexp(A)[1]) - 1 - 23) and (c == 0).all()
            assert q8_ref.dequantize(e, b, c).tobytes() == row.tobytes()


def test_tiny_negative_minimum_floors_below_zero():
    """floor(-tiny / 2^e) is -1, not the floor of an underflowed -0 (the trap of an f32 statement)."""
    for lo in (-1e-45, -2e-45, -1e-40):
        row = np.float32([[lo, 0.0, 1e-44]])
        e, b, c = q8_ref.grid(row)
        assert b[0] < 0 and (int(e[0]), int(b[0])) == int_grid(row[0])[:2]
        assert q8_ref.dequantize(e, b, c)[0, 0] == row[0, 0] or lo == -1e-40  # (-1e-40 and 1e-44 need a coarser grid than 2^-149)


def test_zeros_of_either_sign_are_stored_as_plus_zero():
    row = np.float32([[-0.0, 0.0, -0.0, 5.0]])
    d = q8_ref.roundtrip(row)
    assert d.view(np.uint32)[0, :3].tolist() == [0, 0, 0]
    z = q8_ref.roundtrip(np.float32([[-0.0, -0.0]]))
    assert z.view(np.uint32).tolist() == [[0, 0]]


def test_overflow_refusal_threshold():
    refused, accepted = q8_ref.overflow_rows()
    assert q8_ref.refused(refused).all() and not q8_ref.refused(accepted).any()
    for row in refused:
        assert int_refused(row)
    for row in accepted:
        assert not int_refused(row)
    assert q8_ref.refused(np.float32([[np.nan, 1.0], [1.0, np.inf], [-np.inf, 0.0]])).all()
    fmax = np.finfo(np.float32).max
    assert not q8_ref.refused(np.float32([[fmax]])) and not int_refused([fmax])  # alone, fmax is on its own grid


@pytest.mark.parametrize("dim", [1, 3, 8, 37, 128, 300])
def test_properties_on_random_and_adversarial_rows(dim):
    rows = np.stack(_random_rows(300, dim, 7 * dim) + list(q8_ref.boundary_rows(dim)))
    assert not q8_ref.refused(rows).any()
    e, b, c, d = q8_ref.quantize(rows)
    bc = b[:, None] + c.astype(np.int64)
    assert (np.abs(bc) < 2**24).all()
    # e is minimal: one step finer spans more than 255 steps (or is below the clamp)
    x = rows.astype(np.float64)
    E = np.frexp(np.abs(x).max(axis=1))[1] - 1
    finer = e - 1
    clamp = (np.abs(x).max(axis=1) == 0) | (finer < np.maximum(-149, E - 23))
    wide = np.ceil(np.ldexp(x.max(axis=1), -finer)) - np.floor(np.ldexp(x.min(axis=1), -finer)) > 255
    assert (clamp | wide).all()
    # fmaf(c, s, o) == (b + c) 2^e: the f32 header widens exactly (evaluated in f64, where c s + o is exact, then rounded once)
    o, s = q8_ref.header(e, b)
    fma = (c.astype(np.float64) * s[:, None].astype(np.float64) + o[:, None].astype(np.float64)).astype(np.float32) + np.float32(0)
    assert fma.tobytes() == d.tobytes()
    assert (np.ldexp(bc.astype(np.float64), e[:, None]).astype(np.float32) + np.float32(0)).tobytes() == d.tobytes()
    # idempotence: quantising the dequantised rows gives back the same rows
    assert q8_ref.roundtrip(d).tobytes() == d.tobytes()


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


def _load(path, storage):
    a = _abi()
    h, off = C.c_void_p(), C.c_uint64()
    return a.lib().idb_index_load_storage(os.fsencode(path), 4, 2, 0, storage, 0, C.byref(h), C.byref(off))


@pytest.mark.parametrize("call", [_build, _adopt])
def test_storage_q8_passes_the_argument_checks(call):
    if _has_gpu():
        pytest.skip("without a device only: with one, the call builds an index")
    a = _abi()
    assert a.STORAGE["q8"] == 4
    assert call(4) == a.ERR_CUDA


@pytest.mark.parametrize("call", [_build, _adopt])
@pytest.mark.parametrize("storage", [3, 5, 6, 0xFFFFFFFF])
def test_storages_3_and_above_4_are_refused(call, storage):
    a = _abi()
    assert call(storage) == a.ERR_INVALID_ARG
    assert f"unknown storage {storage}" in a.lib().idb_last_error().decode()


def test_load_storage_q8_passes_the_argument_checks(tmp_path):
    a = _abi()
    assert _load(str(tmp_path / "missing.idx"), 4) == a.ERR_IO
    for storage in (3, 5):
        assert _load(str(tmp_path / "missing.idx"), storage) == a.ERR_INVALID_ARG
        assert f"unknown storage {storage}" in a.lib().idb_last_error().decode()


def test_config_storage_q8_maps_to_4():
    from instant_distance import Config

    c = Config()
    c.storage = "q8"
    assert c._params()["storage"] == 4
    assert _abi().default_params(**c._params()).storage == 4


def test_q8_dispatch_is_the_f16_dispatch_with_row_type_4():
    for dim in (3, 100, 128, 129, 256, 300, 384, 512, 700, 768, 1024, 1025, 2049):
        for M in (2, 16, 32, 33, 64):
            for ef in (1, 10, 100, 128, 129, 257, 513, 1024):
                for v in range(0, 9):
                    f16 = k1_dispatch.k1_cell(dim, M, ef, 5000, "bf16")._replace(bf16=2)
                    assert k1_cell(dim, M, ef, 5000, "q8", v) == f16._replace(bf16=4)
                    assert k1_cell(dim, M, ef, 5000, "f32", v) == k1_dispatch.k1_cell(dim, M, ef, 5000, "f32", v)


def test_q8_cells_are_91_and_all_planned():
    from tests.test_gpu_k1_q8_instantiations import planned_cells

    cells = q8_cells()
    assert len(cells) == 91 and not (cells & all_cells()) and not (cells & f16_cells())
    assert {c._replace(bf16=2) for c in cells} == f16_cells()
    assert planned_cells() == cells
