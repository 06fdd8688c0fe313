"""CPU statement of K1's dispatch with q8 rows: which instantiation of `search_kernel<CH, ROW_T, EF_T, B, OCC, RT, FULL, TMA>` a
search on a q8 index launches.  q8 rows take the packed rows' rule (twice the rows in flight, up to 16) and the default dispatch
(the IDB_VARIANT cases are f32 only), so a q8 cell is the bf16 / fp16 cell with the row type 4.  Other row types are stated by
tests/k1_dispatch_f16.py, whose constants and cell type (tests/k1_dispatch.py) this reuses.
"""
from tests import k1_dispatch_f16
from tests.k1_dispatch import EF_TILES, REGISTER_CH, ROWS_IN_FLIGHT, Cell

ROW_TYPE_Q8 = 4  # IDB_STORAGE_Q8


def k1_cell(dim, M, ef, n, storage="q8", variant=0):
    """The cell a search with ef_search `ef` on an index of n >= 1 points of this dim, M and row storage launches."""
    if storage != "q8":
        return k1_dispatch_f16.k1_cell(dim, M, ef, n, storage, variant)
    return k1_dispatch_f16.k1_cell(dim, M, ef, n, "f16", 0)._replace(bf16=ROW_TYPE_Q8)


def q8_cells():
    """Every K1 kernel a q8 index can run: 6 CH x 7 (ROW_T, EF_T) x 2 FULL and the long-row kernel's 7."""
    cells = set()
    for row_t, efs in EF_TILES.items():
        for ef_t in efs:
            for ch in REGISTER_CH + (0,):
                b = ROWS_IN_FLIGHT[ch] * 2 if ROWS_IN_FLIGHT[ch] * 2 <= 16 else ROWS_IN_FLIGHT[ch]
                for full in ((0, 1) if ch else (0,)):
                    cells.add(Cell(ch, row_t, ef_t, b, ROW_TYPE_Q8, full, 0, 0))
    return frozenset(cells)
