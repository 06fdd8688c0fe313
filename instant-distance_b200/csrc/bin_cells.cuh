// bin_cells.cuh — the definitions behind dispatch_row_ef_bin (search_kernel.cuh) and build_dispatch_bin (build_dispatch.cuh): K1's and
// the construction's cells for bin rows (DESIGN §3d).  Included only by search_bin_chN.cu and build_bin_chN.cu, each of which
// instantiates one CH, so the bin cells compile in translation units of their own.
#pragma once
#include "build_dispatch.cuh"

namespace idb {

template <int CH, int B>
cudaError_t dispatch_row_ef_bin(const SearchArgs& a, int row_t, int ef_t, int grid, cudaStream_t st, const LaunchWindow& win) {
    return dispatch_row_ef_rt<CH, rows_in_flight<B, RowBin>(), RowBin>(a, row_t, ef_t, grid, st, win);
}

template <int CH, int B, int NB>
cudaError_t build_dispatch_bin(const BuildArgs& a, const BuildLaunch& l, cudaStream_t st) {
    return build_dispatch_rt<CH, B, NB, RowBin>(a, l, st);
}

}  // namespace idb
