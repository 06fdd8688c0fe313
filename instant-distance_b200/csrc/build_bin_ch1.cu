// Construction kernels (KA insert search, K2 select/relink) of bin rows for rows of up to 128 elements (the build_ch1.cu shape).
#include "bin_cells.cuh"
namespace idb {
template cudaError_t build_dispatch_bin<1, 16, 16>(const BuildArgs&, const BuildLaunch&, cudaStream_t);
}  // namespace idb
