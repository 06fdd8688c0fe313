// The graph range search's expansion cells for bin rows (DESIGN §3d, §9c), in a translation unit of their own (as K1's, search_cells.cu).
#include "graph_range.cuh"
namespace idb {
GraphRangeKernel graph_range_bin_cell(uint32_t nchunks) { return graph_range_cell<RowBin>(nchunks); }
}  // namespace idb
