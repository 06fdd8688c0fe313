"""Every compiled K1 instantiation for q8 rows (`search_kernel<..., RowQ8, ...>`) against the oracle on the dequantised rows, bit for
bit: ids, distance bytes, lengths and per-layer counters, and the cell `Index.last_kernel()` reports must be the one
tests/k1_dispatch_q8.py states.  At the end, the cells reached must be all 91 of `k1_dispatch_q8.q8_cells()`.

The graphs and the case tables are those of tests/test_gpu_k1_instantiations.py (f32 and bf16 rows), so every q8 cell runs on the
same shapes as its bf16 and fp16 twins.  A q8 index has no screening table, so every candidate is fetched in full.  Beyond every
cell: exact ties at every (ROW_T, EF_T), the retry pass and the hash / bitmap / b16 visited flavours per CH, IDB_VARIANT (f32
instantiations: a q8 index must take its default cell), and cosine at every CH.
"""
import numpy as np
import pytest

from tests.q8_ref import roundtrip
from tests.k1_dispatch import Cell
from tests.k1_dispatch_q8 import k1_cell, q8_cells
from tests.test_gpu_k1_instantiations import (CASES, CH_DIMS, N, TIE_CASES, VARIANTS, _graph, _run, _same, _want)

pytestmark = pytest.mark.gpu


def planned_cells():
    """The cells the case table is meant to reach, by the CPU statement."""
    return {k1_cell(dim, M, ef, N, "q8") for dim, M, efs in CASES for ef in efs}


REACHED = set()
DONE = set()


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    assert _abi.lib().idb_device_count() >= 1
    return _abi


def _indexes(abi, oracle, g, M, metric="l2sq"):
    """A q8 GPU index of the graph, and the oracle on the rows it holds (the dequantised rows)."""
    p, zero, upper, _ = g
    ix = abi.Index.from_graph(p, zero, upper, M, storage="q8", metric=metric)
    rows = ix.export_graph()[0]
    assert rows.tobytes() == roundtrip(p).tobytes() and (rows != p).any()
    return ix, oracle.from_graph(oracle.Graph(rows, zero, upper, M, 100))


def _check(oracle, ix, ox, q, ef, cell, what, metric="l2sq"):
    got = _run(ix, q, ef)
    assert got[4] == cell, f"{what}: launched {got[4]}, the dispatch statement says {cell}"
    want = _want(oracle, ox, q, ef, metric)
    _same(got, want, what)
    REACHED.add(got[4])
    return got, want


@pytest.mark.parametrize("dim,M,efs", CASES, ids=[f"dim{d}-M{m}" for d, m, _ in CASES])
def test_every_q8_cell(abi, oracle, dim, M, efs):
    g = _graph("sift", dim, M)
    ix, ox = _indexes(abi, oracle, g, M)
    for ef in efs:
        cell = k1_cell(dim, M, ef, N, "q8")
        assert cell.bf16 == 4
        got, want = _check(oracle, ix, ox, g[3], ef, cell, f"q8 dim {dim} M {M} ef {ef}")
        assert ix.last_full_fetches() == int(got[3][:, 1].sum() + got[3][:, 3].sum())  # no screening table: every row in full
    ix.close()
    DONE.add((dim, M))


@pytest.mark.parametrize("dim,side,M,efs", TIE_CASES, ids=[f"dim{d}-side{s}-M{m}" for d, s, m, _ in TIE_CASES])
def test_exact_ties_at_every_row_and_ef_tile(abi, oracle, dim, side, M, efs):
    g = _graph("grid", dim, M, side=side)
    p, zero, upper, q = g
    ix = abi.Index.from_graph(p, zero, upper, M, storage="q8")  # small integers: fp16 holds them exactly
    assert ix.export_graph()[0].tobytes() == p.tobytes()
    ox = oracle.from_graph(oracle.Graph(p, zero, upper, M, 100))
    for ef in efs:
        _, want = _check(oracle, ix, ox, q, ef, k1_cell(dim, M, ef, N, "q8"), f"q8 grid dim {dim} M {M} ef {ef}")
        d = want[1]
        assert ((np.diff(d, axis=1) == 0) & np.isfinite(d[:, 1:])).any(axis=1).mean() > 0.75
    ix.close()


def _sift(dim):
    return _graph("sift", dim, 32, n=4000)


@pytest.mark.parametrize("dim", CH_DIMS)
def test_retry_pass_at_every_ch(abi, oracle, monkeypatch, dim):
    g = _sift(dim)
    monkeypatch.setenv("IDB_VIS_TIER", "0")
    monkeypatch.setenv("IDB_VIS_SLOTS", "1024")
    ix, ox = _indexes(abi, oracle, g, 32)
    _check(oracle, ix, ox, g[3], 100, k1_cell(dim, 32, 100, 4000, "q8"), f"q8 retry dim {dim}")
    assert ix.last_retried(0xFFFFFFFF) > 0
    ix.close()


@pytest.mark.parametrize("tier", [0, 1, 2], ids=["hash", "bitmap", "b16"])
@pytest.mark.parametrize("dim", CH_DIMS)
def test_visited_flavours_at_every_ch(abi, oracle, monkeypatch, dim, tier):
    g = _sift(dim)
    monkeypatch.setenv("IDB_VIS_TIER", str(tier))
    ix, ox = _indexes(abi, oracle, g, 32)
    _check(oracle, ix, ox, g[3], 200, k1_cell(dim, 32, 200, 4000, "q8"), f"q8 IDB_VIS_TIER={tier} dim {dim}")
    ix.close()


def test_variants_leave_q8_rows_to_the_default_dispatch(abi, oracle, monkeypatch):
    """The variants are f32 instantiations: a q8 index must launch its default cell (variant 0) and match the oracle."""
    g = _graph("sift", 100, 32)
    for v in VARIANTS:
        monkeypatch.setenv("IDB_VARIANT", str(v))
        ix, ox = _indexes(abi, oracle, g, 32)
        for ef in (10, 128):
            cell = k1_cell(100, 32, ef, N, "q8", v)
            assert cell == k1_cell(100, 32, ef, N, "q8") and cell.variant == 0
            _check(oracle, ix, ox, g[3], ef, cell, f"q8 IDB_VARIANT={v} ef {ef}")
        ix.close()


@pytest.mark.parametrize("dim", CH_DIMS)
def test_cosine_at_every_ch(abi, oracle, dim):
    g = _graph("sift", dim, 24, metric="cosine")
    ix, ox = _indexes(abi, oracle, g, 24, metric="cosine")
    _check(oracle, ix, ox, g[3], 64, k1_cell(dim, 24, 64, N, "q8"), f"q8 cosine dim {dim}", metric="cosine")
    ix.close()


def test_every_q8_cell_was_reached():
    if not {(d, m) for d, m, _ in CASES} <= DONE:
        pytest.skip("needs every case of test_every_q8_cell in this session")
    missing, extra = q8_cells() - REACHED, REACHED - q8_cells()
    assert not missing and not extra, f"{len(missing)} cells never ran: {sorted(missing)[:8]}; unknown cells: {sorted(extra)[:8]}"
    assert len(REACHED) == 91 and all(isinstance(c, Cell) and c.bf16 == 4 for c in REACHED)
