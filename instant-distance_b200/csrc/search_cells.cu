// K1's cells of one CH and row family: the Makefile compiles this unit once per (IDB_CELL_CH, IDB_CELL_BIN), so each object holds the
// cells api.cu's with_cell reaches for rows of that CH (0: more than 1024 elements, the query in shared memory) and for bin rows
// (IDB_CELL_BIN = 1) or for f32, bf16, fp16 and q8 rows (0).
#include "search_kernel.cuh"
namespace idb {
template <int CH, bool BIN>
cudaError_t search_cells(const SearchArgs& a, int row_t, int ef_t, int grid, cudaStream_t st, const LaunchWindow& win) {
#if IDB_CELL_CH == 1 && !IDB_CELL_BIN
    // tuning variants of the headline shape (ROW_T=2, EF_T=4): rows in flight per lane x resident CTAs per SM.  They are
    // instantiated for f32 rows only: a bf16 or fp16 index takes the default dispatch below.
    if (a.variant && a.g.row_type == kRowF32 && row_t <= 2 && ef_t <= 4) {
        switch (a.variant) {
            case 1: return launch_search<1, 2, 4, 8, occ_for_warps(20)>(a, grid, st, win, 1);
            case 2: return launch_search<1, 2, 4, 8, occ_for_warps(24)>(a, grid, st, win, 2);
            case 3: return launch_search<1, 2, 4, 4, occ_for_warps(32)>(a, grid, st, win, 3);
            case 4: return launch_search<1, 2, 4, 16, occ_for_warps(12)>(a, grid, st, win, 4);
            // EXPERIMENT: rows via cp.async.bulk into a shared-memory ring, no register staging
            case 5: return launch_search<1, 2, 4, 16, occ_for_warps(16), RowF32, false, true>(a, grid, st, win, 5);
            case 6: return launch_search<1, 2, 4, 8, occ_for_warps(20), RowF32, false, true>(a, grid, st, win, 6);
            case 7: return launch_search<1, 2, 4, 8, occ_for_warps(24), RowF32, false, true>(a, grid, st, win, 7);
            case 8: return launch_search<1, 2, 4, 32, occ_for_warps(8), RowF32, false, true>(a, grid, st, win, 8);
            default: break;
        }
    }
#endif
    constexpr int B = Cell<CH>::B;
    if constexpr (BIN) return dispatch_row_ef_rt<CH, rows_in_flight<B, RowBin>(), RowBin>(a, row_t, ef_t, grid, st, win);
    else return with_row_type(a.g.row_type, [&](auto rt) {
        using RT = decltype(rt);
        if constexpr (RT::kType == kRowBin) return cudaErrorInvalidValue;  // search_cells<CH, true>'s rows
        else return dispatch_row_ef_rt<CH, rows_in_flight<B, RT>(), RT>(a, row_t, ef_t, grid, st, win);
    });
}
template cudaError_t search_cells<IDB_CELL_CH, IDB_CELL_BIN>(const SearchArgs&, int, int, int, cudaStream_t, const LaunchWindow&);
}  // namespace idb

#if defined(IDB_K1_PHASES) && IDB_CELL_CH == 1 && !IDB_CELL_BIN
// The phase tallies of this translation unit's K1 kernels (hnsw_device.cuh, "K1 phase clock"): copies kPhSlots u64 to out, then zeroes
// them when reset != 0.  Only in a library built with -DIDB_K1_PHASES (scripts/k1_phases.py).
extern "C" __attribute__((visibility("default"))) int idb_debug_k1_phases(unsigned long long* out, int reset) {
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    if (cudaMemcpyFromSymbol(out, idb::g_k1_phases, sizeof(idb::g_k1_phases)) != cudaSuccess) return -1;
    if (reset) {
        static const unsigned long long zero[idb::kPhSlots] = {};
        if (cudaMemcpyToSymbol(idb::g_k1_phases, zero, sizeof(zero)) != cudaSuccess) return -1;
    }
    return idb::kPhSlots;
}
#endif
