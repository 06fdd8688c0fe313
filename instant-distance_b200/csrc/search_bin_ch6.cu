// K1's bin-row cells for rows of up to 768 elements (the search_ch6.cu shape).
#include "bin_cells.cuh"
namespace idb {
template cudaError_t dispatch_row_ef_bin<6, 2>(const SearchArgs&, int, int, int, cudaStream_t, const LaunchWindow&);
}  // namespace idb
