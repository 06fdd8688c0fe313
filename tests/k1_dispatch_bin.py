"""CPU statement of K1's dispatch with bin rows: which instantiation of `search_kernel<CH, ROW_T, EF_T, B, OCC, RT, FULL, TMA>` a
search on a bin index launches.  bin rows take the packed rows' rule (twice the rows in flight, up to 16) and the default dispatch
(the IDB_VARIANT cases are f32 only), so a bin cell is the q8 cell with the row type 8.  Other row types are stated by
tests/k1_dispatch_q8.py, whose cells this reuses.
"""
from tests import k1_dispatch_q8

ROW_TYPE_BIN = 8  # IDB_STORAGE_BIN


def k1_cell(dim, M, ef, n, storage="bin", variant=0):
    """The cell a search with ef_search `ef` on an index of n >= 1 points of this dim, M and row storage launches."""
    if storage != "bin":
        return k1_dispatch_q8.k1_cell(dim, M, ef, n, storage, variant)
    return k1_dispatch_q8.k1_cell(dim, M, ef, n, "q8", 0)._replace(bf16=ROW_TYPE_BIN)


def bin_cells():
    """Every K1 kernel a bin index can run: 6 CH x 7 (ROW_T, EF_T) x 2 FULL and the long-row kernel's 7."""
    return frozenset(c._replace(bf16=ROW_TYPE_BIN) for c in k1_dispatch_q8.q8_cells())
