// K1's bin-row cells for rows of up to 128 elements (the search_ch1.cu shape).
#include "bin_cells.cuh"
namespace idb {
template cudaError_t dispatch_row_ef_bin<1, 16>(const SearchArgs&, int, int, int, cudaStream_t, const LaunchWindow&);
}  // namespace idb
