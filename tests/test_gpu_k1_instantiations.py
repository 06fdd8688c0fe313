"""Every compiled instantiation of K1 (`search_kernel<CH, ROW_T, EF_T, B, OCC, RT, FULL, TMA>`) against the oracle, bit for bit.

K1 is a template; the search dispatch picks CH from the row length, ROW_T from M, EF_T from ef, the row type from the storage and
FULL from whether the row fills every chunk slot, and IDB_VARIANT swaps the headline shape for a tuning variant.  Screening
(`screen_candidates<CH, FULL>`) and tie collection (`collect_ties<ROW_T, EF_T>`) are compiled into each cell separately, so a bug can
live in one cell and nowhere else.  Here every cell runs on a graph built on the GPU and adopted by the oracle: ids, distance bytes,
lengths and per-layer counters must equal the oracle's, and the cell the library reports (`Index.last_kernel()`) must be the one
tests/k1_dispatch.py states.  At the end, the cells reached must be all of `k1_dispatch.all_cells()`.

Beyond every cell: exact ties at every (ROW_T, EF_T), screening off and on, the retry pass and the hash / bitmap visited flavours
per CH, the IDB_VARIANT cases (and where they do not apply), and cosine at every CH.
"""
import functools
import os

import numpy as np
import pytest

from tests import cosine_ref, datagen
from tests.k1_dispatch import Cell, all_cells, k1_cell

pytestmark = pytest.mark.gpu

THREADS = min(32, os.cpu_count() or 8)
NQ = 64
N = 1500  # > 1024: ef 1024 is not clipped to n

# ---- the case tables (tests/test_k1_dispatch_model.py checks on the CPU that they reach every cell) ----------------------------

# Every (CH, FULL): 383 and 1021 are FULL with padding inside the last chunk; 300, 600, 700 and 900 are not FULL.
DIMS = (3, 100, 128, 129, 256, 300, 383, 384, 385, 512, 600, 700, 768, 900, 1021, 1024, 1025, 1152, 2049)
# ef per ROW_T: every EF_T of that ROW_T, each set on both sides of the EF_T boundaries
EF_SETS = {2: ((10, 129, 257, 513), (128, 256, 512, 1024)), 4: ((10, 129, 1024), (128, 257, 513))}
M_SETS = {2: (2, 17, 32), 4: (33, 64)}
CASES = [(dim, M_SETS[rt][i % len(M_SETS[rt])], EF_SETS[rt][i % 2]) for i, dim in enumerate(DIMS) for rt in (2, 4)]
STORAGES = ("f32", "bf16")

# Ties at every (ROW_T, EF_T).  With M > 32 and a small ef, the first expansion on layer 0 evicts tied candidates from beyond the
# first 64 entries of its row, where collect_ties counts the admitted entries of all four 32-entry groups.
TIE_CASES = [(8, 2, 32, (10, 129, 257, 513)), (8, 2, 64, (10, 40, 129, 513)), (300, 3, 17, (128, 256, 512, 1024)),
             (300, 3, 48, (10, 64, 257, 1024))]
REGISTER_DIMS = (100, 256, 300, 512, 700, 1024)  # one per register CH
CH_DIMS = REGISTER_DIMS + (1152,)                # ... and the long-row kernel
VARIANT_DIMS = (100, 128)
VARIANT_EFS = (10, 128)
VARIANTS = tuple(range(1, 9))


def planned_cells():
    """The cells the case tables above are meant to reach, by the CPU statement."""
    cells = {k1_cell(dim, M, ef, N, s) for dim, M, efs in CASES for ef in efs for s in STORAGES}
    cells |= {k1_cell(dim, 32, ef, N, "f32", v) for dim in VARIANT_DIMS for ef in VARIANT_EFS for v in VARIANTS}
    return cells


REACHED = set()
DONE = set()


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    assert _abi.lib().idb_device_count() >= 1
    return _abi


# ---- graphs: built on the GPU once per shape, exported, adopted by the oracle ------------------------------------------------

@functools.lru_cache(maxsize=None)
def _graph(kind, dim, M, n=N, metric="l2sq", side=0):
    """(points, zero, upper, queries) of a GPU-built graph; points as the GPU index stores them (cosine: normalised)."""
    from instant_distance_b200 import _abi

    if kind == "sift":
        pts, q = datagen.sift_shaped(n, dim, 1000 + dim), datagen.sift_shaped(NQ, dim, 2000 + dim)
    else:
        pts, q = datagen.grid_ties(n, dim, 3000 + dim, side=side), datagen.grid_ties(NQ, dim, 4000 + dim, side=side)
    kw = {"ml": 0.5} if M == 2 else {}  # 1 / ln 2 > 1 is not a valid ml
    ix, _ = _abi.Index.build(pts, M=M, seed=dim + M, metric=metric, **kw)
    p, zero, upper = ix.export_graph()
    ix.close()
    return p, zero, upper, q


def _indexes(abi, oracle, g, M, storage="f32", metric="l2sq"):
    """A GPU index of the graph with this row storage, and the oracle on the rows the GPU index holds (bf16: already rounded)."""
    p, zero, upper, _ = g
    ix = abi.Index.from_graph(p, zero, upper, M, storage=storage, metric=metric)
    rows = ix.export_graph()[0] if storage == "bf16" else p
    assert storage == "f32" or (rows != p).any()
    return ix, oracle.from_graph(oracle.Graph(rows, zero, upper, M, 100))


def _run(ix, q, ef):
    ids, dist, lens = ix.search(q, ef_search=ef, k=ef)
    return ids, dist, lens, ix.last_counters(len(q)), Cell(**ix.last_kernel())


def _want(oracle, ox, q, ef, metric="l2sq"):
    if metric == "cosine":
        return cosine_ref.search(oracle, ox, q, ef_search=ef, k=ef, counters=True, threads=THREADS)
    return ox.search(q, ef_search=ef, k=ef, counters=True, threads=THREADS)


def _same(got, want, what):
    ids, dist, lens, cnt = got[:4]
    assert (lens == want[2]).all(), f"{what}: lengths differ"
    bad = (ids != want[0]).any(axis=1)
    assert not bad.any(), f"{what}: ids differ in {bad.sum()} of {len(ids)} queries (first: query {np.argmax(bad)})"
    assert dist.tobytes() == want[1].tobytes(), f"{what}: distance bytes differ"
    assert (cnt == want[3]).all(), f"{what}: per-layer counters differ"


def _check(oracle, ix, ox, q, ef, cell, what, metric="l2sq"):
    """Search ix at ef; assert the oracle's results and the reported cell.  Returns (GPU results, the oracle's)."""
    got = _run(ix, q, ef)
    assert got[4] == cell, f"{what}: launched {got[4]}, the dispatch statement says {cell}"
    want = _want(oracle, ox, q, ef, metric)
    _same(got, want, what)
    REACHED.add(got[4])
    return got, want


# ---- every cell -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dim,M,efs", CASES, ids=[f"dim{d}-M{m}" for d, m, _ in CASES])
def test_every_cell(abi, oracle, dim, M, efs):
    g = _graph("sift", dim, M)
    q = g[3]
    for storage in STORAGES:
        ix, ox = _indexes(abi, oracle, g, M, storage)
        for ef in efs:
            cell = k1_cell(dim, M, ef, N, storage)
            got, want = _check(oracle, ix, ox, q, ef, cell, f"{storage} dim {dim} M {M} ef {ef}")
            n_dist, full = int(got[3][:, 1].sum() + got[3][:, 3].sum()), ix.last_full_fetches()
            if cell.ch == 0:
                assert full == n_dist  # the long-row kernel does not screen
            elif ef >= 128 and M > 2:  # (M = 2: rows of 4 neighbours, a traversal reaches fewer than 1024 points)
                assert (want[2] == min(ef, N)).mean() > 0.9  # `nearest` fills, so the screen has a furthest distance ...
                assert full < n_dist  # ... and drops rows with it
        ix.close()
    DONE.add(("cell", dim, M))


# ---- ties at every (ROW_T, EF_T) ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("dim,side,M,efs", TIE_CASES, ids=[f"dim{d}-side{s}-M{m}" for d, s, m, _ in TIE_CASES])
def test_exact_ties_at_every_row_and_ef_tile(abi, oracle, dim, side, M, efs):
    """Integer-grid rows: many exact distance ties and duplicate rows at the ef boundary, where collect_ties decides."""
    g = _graph("grid", dim, M, side=side)
    ix, ox = _indexes(abi, oracle, g, M)
    for ef in efs:
        cell = k1_cell(dim, M, ef, N)
        _, want = _check(oracle, ix, ox, g[3], ef, cell, f"grid dim {dim} M {M} ef {ef}")
        d = want[1]
        tied = (np.diff(d, axis=1) == 0) & np.isfinite(d[:, 1:])
        assert tied.any(axis=1).mean() > 0.75, "the grid should give most queries tied distances"
    ix.close()


# ---- screening, the retry pass and the visited flavours per CH ------------------------------------------------------------

def _sift(dim):
    return _graph("sift", dim, 32, n=4000)


@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("dim", REGISTER_DIMS)
def test_screen_off_and_on_match_the_oracle(abi, oracle, monkeypatch, dim, storage):
    g = _sift(dim)
    res = {}
    for screen in (0, 1):
        monkeypatch.setenv("IDB_SCREEN", str(screen))
        ix, ox = _indexes(abi, oracle, g, 32, storage)
        res[screen] = _check(oracle, ix, ox, g[3], 100, k1_cell(dim, 32, 100, 4000, storage), f"IDB_SCREEN={screen}")
        res[screen] += (ix.last_full_fetches(),)
        ix.close()
    off, on = res[0], res[1]
    assert on[0][1].tobytes() == off[0][1].tobytes() and (on[0][3] == off[0][3]).all()
    n_dist = int(off[0][3][:, 1].sum() + off[0][3][:, 3].sum())
    assert off[2] == n_dist  # unscreened: every candidate is fetched in full
    assert on[2] < n_dist, f"screening dropped no row ({on[2]} of {n_dist} fetched in full)"


@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("dim", CH_DIMS)
def test_retry_pass_at_every_ch(abi, oracle, monkeypatch, dim, storage):
    """A 1024-slot hash set overflows in every query here (each evaluates over 1700 distances): the retry pass (same cell, 2^18-slot
    hash sets) must give the oracle's results."""
    g = _sift(dim)
    monkeypatch.setenv("IDB_VIS_TIER", "0")
    monkeypatch.setenv("IDB_VIS_SLOTS", "1024")
    ix, ox = _indexes(abi, oracle, g, 32, storage)
    _check(oracle, ix, ox, g[3], 100, k1_cell(dim, 32, 100, 4000, storage), f"retry {storage} dim {dim}")
    assert ix.last_retried(0xFFFFFFFF) > 0
    ix.close()


@pytest.mark.parametrize("tier", [0, 1], ids=["hash", "bitmap"])
@pytest.mark.parametrize("dim", CH_DIMS)
def test_visited_flavours_at_every_ch(abi, oracle, monkeypatch, dim, tier):
    g = _sift(dim)
    monkeypatch.setenv("IDB_VIS_TIER", str(tier))
    ix, ox = _indexes(abi, oracle, g, 32)
    _check(oracle, ix, ox, g[3], 200, k1_cell(dim, 32, 200, 4000), f"IDB_VIS_TIER={tier} dim {dim}")
    assert ix.last_retried(0xFFFFFFFF) == 0
    ix.close()


# ---- IDB_VARIANT --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dim", VARIANT_DIMS)
def test_variants_on_f32_rows(abi, oracle, monkeypatch, dim):
    g = _graph("sift", dim, 32)
    for v in VARIANTS:
        monkeypatch.setenv("IDB_VARIANT", str(v))
        ix, ox = _indexes(abi, oracle, g, 32)
        for ef in VARIANT_EFS:
            cell = k1_cell(dim, 32, ef, N, "f32", v)
            assert cell.variant == v
            _check(oracle, ix, ox, g[3], ef, cell, f"IDB_VARIANT={v} dim {dim} ef {ef}")
        ix.close()
    DONE.add(("variant", dim))


def test_variants_leave_bf16_rows_to_the_default_dispatch(abi, oracle, monkeypatch):
    """The variants are f32 instantiations: a bf16 index must launch its default cell (bf16 rows, doubled B) and match the oracle."""
    g = _graph("sift", 100, 32)
    for v in VARIANTS:
        monkeypatch.setenv("IDB_VARIANT", str(v))
        ix, ox = _indexes(abi, oracle, g, 32, "bf16")
        cell = k1_cell(100, 32, 100, N, "bf16", v)
        assert cell == k1_cell(100, 32, 100, N, "bf16") and cell.bf16 == 1 and cell.variant == 0
        _check(oracle, ix, ox, g[3], 100, cell, f"bf16 IDB_VARIANT={v}")
        ix.close()


@pytest.mark.parametrize("M,ef", [(33, 100), (32, 129)])
def test_variants_apply_to_the_headline_shape_only(abi, oracle, monkeypatch, M, ef):
    g = _graph("sift", 100, M)
    monkeypatch.setenv("IDB_VARIANT", "1")
    ix, ox = _indexes(abi, oracle, g, M)
    cell = k1_cell(100, M, ef, N, "f32", 1)
    assert cell.variant == 0
    _check(oracle, ix, ox, g[3], ef, cell, f"IDB_VARIANT=1 M {M} ef {ef}")
    ix.close()


# ---- cosine ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dim", CH_DIMS)
def test_cosine_at_every_ch(abi, oracle, dim):
    """The metric changes K1's epilogue only: one cell per CH."""
    g = _graph("sift", dim, 24, metric="cosine")
    ix, ox = _indexes(abi, oracle, g, 24, metric="cosine")
    _check(oracle, ix, ox, g[3], 64, k1_cell(dim, 24, 64, N), f"cosine dim {dim}", metric="cosine")
    ix.close()


# ---- the session reached every cell -------------------------------------------------------------------------------------

def test_every_cell_was_reached():
    wanted = {("cell", d, m) for d, m, _ in CASES} | {("variant", d) for d in VARIANT_DIMS}
    if not wanted <= DONE:
        pytest.skip("needs every case of test_every_cell and test_variants_on_f32_rows in this session")
    missing, extra = all_cells() - REACHED, REACHED - all_cells()
    assert not missing and not extra, f"{len(missing)} cells never ran: {sorted(missing)[:8]}; unknown cells: {sorted(extra)[:8]}"
    assert len(REACHED) == 190
