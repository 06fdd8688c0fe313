// Construction kernels (KA insert search, K2 select / relink) of one CH and row family: the Makefile compiles this unit once per
// (IDB_CELL_CH, IDB_CELL_BIN), so each object holds the cells build.cu's with_cell reaches for rows of that CH (0: more than 1024
// elements) and for bin rows (IDB_CELL_BIN = 1) or for f32, bf16, fp16 and q8 rows (0).
#include "build_dispatch.cuh"
namespace idb {
template <int CH, bool BIN>
cudaError_t build_cells(const BuildArgs& a, const BuildLaunch& l, cudaStream_t st) {
    if constexpr (BIN) return build_dispatch_rt<CH, RowBin>(a, l, st);
    else return with_row_type(a.g.row_type, [&](auto rt) {
        using RT = decltype(rt);
        if constexpr (RT::kType == kRowBin) return cudaErrorInvalidValue;  // build_cells<CH, true>'s rows
        else return build_dispatch_rt<CH, RT>(a, l, st);
    });
}
template cudaError_t build_cells<IDB_CELL_CH, IDB_CELL_BIN>(const BuildArgs&, const BuildLaunch&, cudaStream_t);
}  // namespace idb
