"""CPU statement of K1's dispatch for every row type, fp16 included: which instantiation of
`search_kernel<CH, ROW_T, EF_T, B, OCC, RT, FULL, TMA>` a search launches (`Index::enqueue_search`, `dispatch_search`,
`with_cell`, `search_cells`, `dispatch_row_ef_rt`).

tests/k1_dispatch.py states the f32 and bf16 dispatch; this restates it with the row type as an IDB_STORAGE_* value, so that the
fp16 GPU tests can check the cell `idb_last_search_kernel` reports, and tests/test_f16_cpu.py checks that it agrees with
tests/k1_dispatch.py on f32 and bf16 rows.  A cell is tests/k1_dispatch.py's `Cell`; its `bf16` field carries the row type.
"""
from tests.k1_dispatch import EF_TILES, REGISTER_CH, ROWS_IN_FLIGHT, VARIANTS, Cell

ROW_TYPE = {"f32": 0, "bf16": 1, "f16": 2}  # IDB_STORAGE_*


def _cdiv(a, b):
    return (a + b - 1) // b


def k1_cell(dim, M, ef, n, storage="f32", variant=0):
    """The cell a search with ef_search `ef` (>= 1) on an index of n >= 1 points of this dim, M and row storage launches."""
    if storage not in ROW_TYPE:
        raise ValueError(storage)
    rt = ROW_TYPE[storage]
    ef = min(ef, n)  # the library clips ef to n before it dispatches
    if ef > 1024:
        raise ValueError("ef_search > 1024 on an index of more than 1024 points is not supported")
    nchunks = _cdiv(dim, 4)
    ch = _cdiv(nchunks, 32)
    if ch > 8 and ch * 512 > 40 * 1024:
        raise ValueError("dim > 10240 is not supported")
    CH = ch if ch <= 4 else 6 if ch <= 6 else 8 if ch <= 8 else 0
    row_t, ef_t = _cdiv(2 * M, 32), _cdiv(ef, 32)
    # the IDB_VARIANT cases replace the default instantiation of the headline shape, for f32 rows only
    if variant in VARIANTS and rt == 0 and CH == 1 and row_t <= 2 and ef_t <= 4:
        b, tma = VARIANTS[variant]
        return Cell(1, 2, 4, b, 0, 0, tma, variant)
    ROW_T = 2 if row_t <= 2 else 4
    EF_T = next((t for t in EF_TILES[ROW_T] if ef_t <= t), 32)
    b = ROWS_IN_FLIGHT[CH]
    if rt and 2 * b <= 16:  # packed bf16 / fp16 rows take half the registers: twice the rows in flight, up to 16
        b *= 2
    full = CH > 0 and nchunks == 32 * CH
    return Cell(CH, ROW_T, EF_T, b, rt, int(full), 0, 0)


def f16_cells():
    """Every K1 kernel an fp16 index can run: 6 CH x 7 (ROW_T, EF_T) x 2 FULL and the long-row kernel's 7.  fp16 rows are packed
    like bf16 rows (twice the rows in flight, up to 16), and the IDB_VARIANT cases are f32 only."""
    cells = set()
    for row_t, efs in EF_TILES.items():
        for ef_t in efs:
            for ch in REGISTER_CH + (0,):
                b = ROWS_IN_FLIGHT[ch] * 2 if ROWS_IN_FLIGHT[ch] * 2 <= 16 else ROWS_IN_FLIGHT[ch]
                for full in ((0, 1) if ch else (0,)):
                    cells.add(Cell(ch, row_t, ef_t, b, ROW_TYPE["f16"], full, 0, 0))
    return frozenset(cells)
