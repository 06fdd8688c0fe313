"""The CPU statement of K1's dispatch (tests/k1_dispatch.py): its boundaries, its cells, and the GPU case table's coverage of them."""
import pytest

from tests import test_gpu_k1_instantiations as gpu_cases
from tests.k1_dispatch import VARIANTS, Cell, all_cells, k1_cell


@pytest.mark.parametrize("dim,ch,full", [
    (1, 1, 0), (124, 1, 0), (125, 1, 1), (128, 1, 1), (129, 2, 0), (256, 2, 1), (257, 3, 0), (384, 3, 1), (385, 4, 0), (512, 4, 1),
    (513, 6, 0), (640, 6, 0), (641, 6, 0), (765, 6, 1), (768, 6, 1), (769, 8, 0), (1021, 8, 1), (1024, 8, 1), (1025, 0, 0), (10240, 0, 0),
])
def test_dim_picks_ch_and_full(dim, ch, full):
    c = k1_cell(dim, 32, 100, 5000)
    assert (c.ch, c.full) == (ch, full)


@pytest.mark.parametrize("M,ef,row_t,ef_t", [
    (2, 1, 2, 4), (16, 128, 2, 4), (32, 128, 2, 4), (33, 128, 4, 4), (64, 128, 4, 4),
    (32, 129, 2, 8), (33, 129, 4, 16), (32, 256, 2, 8), (33, 256, 4, 16), (32, 257, 2, 16), (33, 257, 4, 16),
    (32, 512, 2, 16), (64, 512, 4, 16), (32, 513, 2, 32), (33, 513, 4, 32), (2, 1024, 2, 32), (64, 1024, 4, 32),
])
def test_m_and_ef_pick_the_tiles(M, ef, row_t, ef_t):
    c = k1_cell(128, M, ef, 5000)
    assert (c.row_t, c.ef_t) == (row_t, ef_t)


def test_ef_is_clipped_to_n():
    assert k1_cell(128, 32, 1024, 100).ef_t == 4
    assert k1_cell(128, 32, 1024, 129).ef_t == 8
    assert k1_cell(128, 32, 5000, 1000).ef_t == 32
    with pytest.raises(ValueError):
        k1_cell(128, 32, 1025, 2000)


@pytest.mark.parametrize("dim,b_f32,b_bf16", [(128, 16, 16), (200, 8, 16), (300, 4, 8), (400, 4, 8), (700, 2, 4), (1000, 2, 4),
                                              (2000, 8, 16)])
def test_bf16_doubles_rows_in_flight_up_to_16(dim, b_f32, b_bf16):
    f, h = k1_cell(dim, 32, 100, 5000, "f32"), k1_cell(dim, 32, 100, 5000, "bf16")
    assert (f.b, f.bf16, h.b, h.bf16) == (b_f32, 0, b_bf16, 1)
    assert f._replace(b=0, bf16=0) == h._replace(b=0, bf16=0)


def test_variants_replace_the_headline_shape_of_f32_rows_only():
    for v, (b, tma) in VARIANTS.items():
        assert k1_cell(128, 32, 100, 5000, "f32", v) == Cell(1, 2, 4, b, 0, 0, tma, v)  # never FULL, even at dim 128
        assert k1_cell(3, 2, 1, 5000, "f32", v).variant == v
        default = k1_cell(128, 32, 100, 5000, "f32")
        for shape in [(129, 32, 100), (128, 33, 100), (128, 32, 129)]:  # CH 2, ROW_T 4, EF_T 8: the default dispatch
            assert k1_cell(*shape, 5000, "f32", v) == k1_cell(*shape, 5000, "f32")
        assert k1_cell(128, 32, 1000, 100, "f32", v).variant == v  # ef clipped to n = 100 first
        bf = k1_cell(128, 32, 100, 5000, "bf16", v)
        assert bf == k1_cell(128, 32, 100, 5000, "bf16") and bf.bf16 == 1 and bf.b == 16 and bf.variant == 0
        assert default.variant == 0
    for v in (-1, 9, 100):
        assert k1_cell(128, 32, 100, 5000, "f32", v) == k1_cell(128, 32, 100, 5000, "f32")


def test_all_cells_are_the_reachable_cells():
    cells = all_cells()
    assert len(cells) == 190
    assert len({c for c in cells if c.ch and not c.variant}) == 168 and len({c for c in cells if c.ch == 0}) == 14
    reached = set()
    for dim in (1, 100, 128, 129, 256, 300, 384, 385, 512, 600, 768, 900, 1024, 1025, 4000):
        for M in (2, 32, 33, 64):
            for ef in (1, 128, 129, 256, 257, 512, 513, 1024):
                for storage in ("f32", "bf16"):
                    for v in range(0, 10):
                        reached.add(k1_cell(dim, M, ef, 2000, storage, v))
    assert reached == cells


def test_the_gpu_case_table_reaches_every_cell():
    planned = gpu_cases.planned_cells()
    assert planned == all_cells(), f"missing: {sorted(all_cells() - planned)[:8]}"
    for dim, M, efs in gpu_cases.CASES:
        if any(k1_cell(dim, M, ef, gpu_cases.N).ef_t == 32 for ef in efs):
            assert gpu_cases.N >= 1100
    # ties at every (ROW_T, EF_T)
    tiles = {(k1_cell(d, M, ef, gpu_cases.N).row_t, k1_cell(d, M, ef, gpu_cases.N).ef_t) for d, _, M, efs in gpu_cases.TIE_CASES for ef in efs}
    assert tiles == {(2, 4), (2, 8), (2, 16), (2, 32), (4, 4), (4, 16), (4, 32)}
    # screening, the retry pass, the visited flavours and cosine: every register CH (and the long-row kernel where they apply)
    assert sorted(k1_cell(d, 32, 100, 4000).ch for d in gpu_cases.REGISTER_DIMS) == [1, 2, 3, 4, 6, 8]
    assert sorted(k1_cell(d, 32, 100, 4000).ch for d in gpu_cases.CH_DIMS) == [0, 1, 2, 3, 4, 6, 8]
