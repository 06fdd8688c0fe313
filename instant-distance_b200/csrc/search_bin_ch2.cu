// K1's bin-row cells for rows of up to 256 elements (the search_ch2.cu shape).
#include "bin_cells.cuh"
namespace idb {
template cudaError_t dispatch_row_ef_bin<2, 8>(const SearchArgs&, int, int, int, cudaStream_t, const LaunchWindow&);
}  // namespace idb
