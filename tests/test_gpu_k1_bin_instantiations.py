"""Every compiled K1 instantiation for bin rows (`search_kernel<..., RowBin, ...>`) against the f32 oracle on the same 0/1 rows, bit
for bit: ids, distance bytes, lengths and per-layer counters, and the cell `Index.last_kernel()` reports must be the one
tests/k1_dispatch_bin.py states.  At the end, the cells reached must be all 91 of `k1_dispatch_bin.bin_cells()`.

The case table is that of tests/test_gpu_k1_instantiations.py, so every bin cell runs on the dims, M and ef of its f32, bf16, fp16 and
q8 twins.  The points are sift-shaped rows binarised at their column medians, and the graphs are built on the GPU as bin indexes.
Queries are 0/1 (distances are then Hamming distances, many of them tied) and, at every CH, arbitrary f32.  A bin index has no
screening table, so every candidate is fetched in full.  Beyond every cell: the retry pass and the hash / bitmap / b16 visited
flavours per CH, and IDB_VARIANT (f32 instantiations: a bin index must take its default cell).
"""
import functools

import numpy as np
import pytest

from tests import bin_ref, datagen
from tests.k1_dispatch import Cell
from tests.k1_dispatch_bin import bin_cells, k1_cell
from tests.test_gpu_k1_instantiations import CASES, CH_DIMS, N, NQ, VARIANTS, _run, _same, _want

pytestmark = pytest.mark.gpu


def planned_cells():
    """The cells the case table is meant to reach, by the CPU statement."""
    return {k1_cell(dim, M, ef, N, "bin") for dim, M, efs in CASES for ef in efs}


REACHED = set()
DONE = set()


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    assert _abi.lib().idb_device_count() >= 1
    return _abi


@functools.lru_cache(maxsize=None)
def _graph(dim, M, n=N):
    """(0/1 points, zero, upper, 0/1 queries, f32 queries) of a graph the GPU built as a bin index."""
    from instant_distance_b200 import _abi

    raw = datagen.sift_shaped(n, dim, 1000 + dim)
    pts = bin_ref.binarise(raw)
    fq = datagen.sift_shaped(NQ, dim, 2000 + dim)
    q = bin_ref.binarise(fq, raw)
    fq = fq / np.float32(np.abs(fq).max() or 1)  # f32 queries on the rows' scale
    kw = {"ml": 0.5} if M == 2 else {}
    ix, ids = _abi.Index.build(pts, M=M, seed=dim + M, storage="bin", **kw)
    p, zero, upper = ix.export_graph()
    assert p.tobytes() == pts[np.argsort(ids)].tobytes()  # (export is in PointId order)
    ix.close()
    return p, zero, upper, q, fq.astype(np.float32)


def _indexes(abi, oracle, g, M):
    p, zero, upper = g[:3]
    ix = abi.Index.from_graph(p, zero, upper, M, storage="bin")
    assert ix.export_graph()[0].tobytes() == p.tobytes()
    return ix, oracle.from_graph(oracle.Graph(p, zero, upper, M, 100))


def _check(oracle, ix, ox, q, ef, cell, what):
    got = _run(ix, q, ef)
    assert got[4] == cell, f"{what}: launched {got[4]}, the dispatch statement says {cell}"
    want = _want(oracle, ox, q, ef)
    _same(got, want, what)
    REACHED.add(got[4])
    return got, want


@pytest.mark.parametrize("dim,M,efs", CASES, ids=[f"dim{d}-M{m}" for d, m, _ in CASES])
def test_every_bin_cell(abi, oracle, dim, M, efs):
    g = _graph(dim, M)
    ix, ox = _indexes(abi, oracle, g, M)
    for ef in efs:
        cell = k1_cell(dim, M, ef, N, "bin")
        assert cell.bf16 == 8
        got, _ = _check(oracle, ix, ox, g[3], ef, cell, f"bin dim {dim} M {M} ef {ef}")
        if ix.last_retried(0xFFFFFFFF) == 0:  # (a retried query's rows are fetched by K1 and again by the retry pass)
            assert ix.last_full_fetches() == int(got[3][:, 1].sum() + got[3][:, 3].sum())  # no screening table: every row in full
        # 0/1 queries: the reported distances are the Hamming distances to the reported points, as integers
        ids, dist, lens = got[:3]
        for i in range(0, NQ, 8):
            h = bin_ref.hamming(g[3][i:i + 1], g[0][ids[i, :lens[i]]])[0]
            assert (dist[i, :lens[i]] == h).all(), f"dim {dim} ef {ef}: query {i} is not at its Hamming distances"
    ix.close()
    DONE.add((dim, M))


@pytest.mark.parametrize("dim", CH_DIMS)
def test_f32_queries_at_every_ch(abi, oracle, dim):
    """The asymmetric case: arbitrary f32 queries against 0/1 rows are the f32 engine on those rows."""
    g = _graph(dim, 32)
    ix, ox = _indexes(abi, oracle, g, 32)
    for ef in (10, 100):
        _check(oracle, ix, ox, g[4], ef, k1_cell(dim, 32, ef, N, "bin"), f"bin f32 queries dim {dim} ef {ef}")
    ix.close()


@pytest.mark.parametrize("dim", CH_DIMS)
def test_retry_pass_at_every_ch(abi, oracle, monkeypatch, dim):
    g = _graph(dim, 32, n=4000)
    monkeypatch.setenv("IDB_VIS_TIER", "0")
    monkeypatch.setenv("IDB_VIS_SLOTS", "1024")
    ix, ox = _indexes(abi, oracle, g, 32)
    _check(oracle, ix, ox, g[3], 100, k1_cell(dim, 32, 100, 4000, "bin"), f"bin retry dim {dim}")
    assert ix.last_retried(0xFFFFFFFF) > 0
    ix.close()


@pytest.mark.parametrize("tier", [0, 1, 2], ids=["hash", "bitmap", "b16"])
@pytest.mark.parametrize("dim", CH_DIMS)
def test_visited_flavours_at_every_ch(abi, oracle, monkeypatch, dim, tier):
    g = _graph(dim, 32, n=4000)
    monkeypatch.setenv("IDB_VIS_TIER", str(tier))
    ix, ox = _indexes(abi, oracle, g, 32)
    _check(oracle, ix, ox, g[3], 200, k1_cell(dim, 32, 200, 4000, "bin"), f"bin IDB_VIS_TIER={tier} dim {dim}")
    ix.close()


def test_variants_leave_bin_rows_to_the_default_dispatch(abi, oracle, monkeypatch):
    g = _graph(100, 32)
    for v in VARIANTS:
        monkeypatch.setenv("IDB_VARIANT", str(v))
        ix, ox = _indexes(abi, oracle, g, 32)
        for ef in (10, 128):
            cell = k1_cell(100, 32, ef, N, "bin", v)
            assert cell == k1_cell(100, 32, ef, N, "bin") and cell.variant == 0
            _check(oracle, ix, ox, g[3], ef, cell, f"bin IDB_VARIANT={v} ef {ef}")
        ix.close()


def test_every_bin_cell_was_reached():
    if not {(d, m) for d, m, _ in CASES} <= DONE:
        pytest.skip("needs every case of test_every_bin_cell in this session")
    missing, extra = bin_cells() - REACHED, REACHED - bin_cells()
    assert not missing and not extra, f"{len(missing)} cells never ran: {sorted(missing)[:8]}; unknown cells: {sorted(extra)[:8]}"
    assert len(REACHED) == 91 and all(isinstance(c, Cell) and c.bf16 == 8 for c in REACHED)
