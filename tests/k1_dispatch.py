"""CPU statement of K1's dispatch: which instantiation of `search_kernel<CH, ROW_T, EF_T, B, OCC, RT, FULL, TMA>` a search launches.

It restates, in plain Python, what `Index::enqueue_search` and `dispatch_search` (api.cu), `with_cell` and `Cell` (internal.cuh),
`search_cells` (search_cells.cu, with the IDB_VARIANT cases) and `dispatch_row_ef_rt` (search_kernel.cuh) decide, so that the GPU
tests can check the cell `idb_last_search_kernel` reports against it and can prove that every compiled cell was run.

A cell is (ch, row_t, ef_t, b, bf16, full, tma, variant): the fields of `Index.last_kernel()`.
"""
from collections import namedtuple

Cell = namedtuple("Cell", "ch row_t ef_t b bf16 full tma variant")

REGISTER_CH = (1, 2, 3, 4, 6, 8)  # float4 chunks per lane held in registers; 0 is the long-row kernel (query in shared memory)
ROWS_IN_FLIGHT = {1: 16, 2: 8, 3: 4, 4: 4, 6: 2, 8: 2, 0: 8}  # B of f32 rows per CH (internal.cuh Cell)
EF_TILES = {2: (4, 8, 16, 32), 4: (4, 16, 32)}  # EF_T instantiated per ROW_T: ROW_T 4 has no EF_T 8
# IDB_VARIANT cases of the CH-1 headline shape (ROW_T 2, EF_T 4, f32 rows, never FULL): variant -> (B, TMA)
VARIANTS = {1: (8, 0), 2: (8, 0), 3: (4, 0), 4: (16, 0), 5: (16, 1), 6: (8, 1), 7: (8, 1), 8: (32, 1)}


def _cdiv(a, b):
    return (a + b - 1) // b


def k1_cell(dim, M, ef, n, storage="f32", variant=0):
    """The cell a search with ef_search `ef` (>= 1) on an index of n >= 1 points of this dim and M launches."""
    if storage not in ("f32", "bf16"):
        raise ValueError(storage)
    ef = min(ef, n)  # admission is rank < ef and there are only n ids: the library clips ef before it dispatches
    if ef > 1024:
        raise ValueError("ef_search > 1024 on an index of more than 1024 points is not supported")
    nchunks = _cdiv(dim, 4)
    ch = _cdiv(nchunks, 32)
    if ch > 8 and ch * 512 > 40 * 1024:
        raise ValueError("dim > 10240 is not supported")
    CH = ch if ch <= 4 else 6 if ch <= 6 else 8 if ch <= 8 else 0
    row_t, ef_t = _cdiv(2 * M, 32), _cdiv(ef, 32)
    bf16 = storage == "bf16"
    # the variants replace the default instantiation of the headline shape only, and only for f32 rows
    if variant in VARIANTS and not bf16 and CH == 1 and row_t <= 2 and ef_t <= 4:
        b, tma = VARIANTS[variant]
        return Cell(1, 2, 4, b, 0, 0, tma, variant)
    ROW_T = 2 if row_t <= 2 else 4
    EF_T = next((t for t in EF_TILES[ROW_T] if ef_t <= t), 32)
    b = ROWS_IN_FLIGHT[CH]
    if bf16 and 2 * b <= 16:  # packed bf16 rows take half the registers: twice the rows in flight, up to 16
        b *= 2
    full = CH > 0 and nchunks == 32 * CH
    return Cell(CH, ROW_T, EF_T, b, int(bf16), int(full), 0, 0)


def all_cells():
    """Every K1 kernel that can run: 6 CH x 7 (ROW_T, EF_T) x 2 row types x 2 FULL, the long-row kernel's 7 x 2, and 8 variants."""
    cells = set()
    for bf16 in (0, 1):
        for row_t, efs in EF_TILES.items():
            for ef_t in efs:
                for ch in REGISTER_CH + (0,):
                    b = ROWS_IN_FLIGHT[ch] * 2 if bf16 and ROWS_IN_FLIGHT[ch] * 2 <= 16 else ROWS_IN_FLIGHT[ch]
                    for full in ((0, 1) if ch else (0,)):
                        cells.add(Cell(ch, row_t, ef_t, b, bf16, full, 0, 0))
    for v, (b, tma) in VARIANTS.items():
        cells.add(Cell(1, 2, 4, b, 0, 0, tma, v))
    return frozenset(cells)
