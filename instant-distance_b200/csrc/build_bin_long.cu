// Construction kernels (KA insert search, K2 select/relink) of bin rows for rows of more than 1024 elements (the build_long.cu shape).
#include "bin_cells.cuh"
namespace idb {
template cudaError_t build_dispatch_bin<0, kLongRowsInFlight, kLongRowsInFlight>(const BuildArgs&, const BuildLaunch&, cudaStream_t);
}  // namespace idb
