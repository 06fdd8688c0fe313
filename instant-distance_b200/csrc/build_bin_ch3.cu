// Construction kernels (KA insert search, K2 select/relink) of bin rows for rows of up to 384 elements (the build_ch3.cu shape).
#include "bin_cells.cuh"
namespace idb {
template cudaError_t build_dispatch_bin<3, 4, 4>(const BuildArgs&, const BuildLaunch&, cudaStream_t);
}  // namespace idb
