// K1 instantiation for rows of up to 128 floats (1 float4 chunk(s) per lane, 16 row loads in flight per lane).
#include "search_kernel.cuh"
namespace idb {
cudaError_t dispatch_search_ch1(const SearchArgs& a, int row_t, int ef_t, int grid, cudaStream_t st, const LaunchWindow& win) {
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
    return dispatch_row_ef<1, 16>(a, row_t, ef_t, grid, st, win);
}
}  // namespace idb

#ifdef IDB_K1_PHASES
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
