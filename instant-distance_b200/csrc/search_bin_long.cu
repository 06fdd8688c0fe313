// K1's bin-row cells for rows of more than 1024 elements (the search_long.cu shape).
#include "bin_cells.cuh"
namespace idb {
template cudaError_t dispatch_row_ef_bin<0, kLongRowsInFlight>(const SearchArgs&, int, int, int, cudaStream_t, const LaunchWindow&);
}  // namespace idb
