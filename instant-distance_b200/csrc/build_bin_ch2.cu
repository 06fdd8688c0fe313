// Construction kernels (KA insert search, K2 select/relink) of bin rows for rows of up to 256 elements (the build_ch2.cu shape).
#include "bin_cells.cuh"
namespace idb {
template cudaError_t build_dispatch_bin<2, 8, 8>(const BuildArgs&, const BuildLaunch&, cudaStream_t);
}  // namespace idb
