// K1's bin-row cells for rows of up to 512 elements (the search_ch4.cu shape).
#include "bin_cells.cuh"
namespace idb {
template cudaError_t dispatch_row_ef_bin<4, 4>(const SearchArgs&, int, int, int, cudaStream_t, const LaunchWindow&);
}  // namespace idb
