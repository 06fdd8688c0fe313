// build_dispatch.cuh — launch helpers for the construction kernels, instantiated once per CH and row family in build_cells.cu.
#pragma once
#include "build_kernels.cuh"

namespace idb {

enum BuildOp : int { kOpInsertSearch = 0, kOpSelectNew = 1, kOpRelink = 2, kOpRelinkSimple = 3 };

struct BuildLaunch {
    BuildOp op;
    int row_t, ef_t;        // KA template selectors
    bool stage;             // K2: kept rows staged in shared memory
    int grid;
    uint32_t smem_per_warp; // K2
    LaunchWindow win;       // KA: persisting-L2 window on the b16 visited tables
};

template <int CH, int NB, bool kStage, class RT>
cudaError_t launch_k2(const BuildArgs& a, const BuildLaunch& l, cudaStream_t st) {
    const int smem = (int)l.smem_per_warp * kBuildWarps;
    if (l.op == kOpSelectNew) {
        auto kern = select_new_kernel<CH, NB, kStage, RT>;
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return e;
        kern<<<l.grid, kBuildWarps * 32, smem, st>>>(a, l.smem_per_warp);
    } else {
        auto kern = relink_kernel<CH, NB, kStage, RT>;
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return e;
        kern<<<l.grid, kBuildWarps * 32, smem, st>>>(a, l.smem_per_warp);
    }
    return cudaGetLastError();
}

// The construction kernels of Cell<CH> for row type RT: B rows in flight per lane, as is, in KA and in K2 / K2'.
template <int CH, class RT>
cudaError_t build_dispatch_rt(const BuildArgs& a, const BuildLaunch& l, cudaStream_t st) {
    constexpr int B = Cell<CH>::B;
    switch (l.op) {
        case kOpInsertSearch:
            return with_tile(l.row_t, l.ef_t, [&](auto row, auto ef) {
                constexpr int ROW_T = decltype(row)::value, EF_T = decltype(ef)::value;
                return launch_traversal<CH, EF_T>(insert_search_kernel<CH, ROW_T, EF_T, B, RT>, a, 0, l.grid, st, l.win);
            });
        case kOpSelectNew:
        case kOpRelink:
            if constexpr (CH > 0) {
                if (l.stage) return launch_k2<CH, B, true, RT>(a, l, st);
            }
            return launch_k2<CH, B, false, RT>(a, l, st);
        case kOpRelinkSimple: {
            const int smem = CH == 0 ? (int)long_q_bytes(a.g.nchunks) * kBuildWarps : 0;
            auto kern = relink_simple_kernel<CH, RT>;
            if (smem > 48 * 1024) {
                cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
                if (e != cudaSuccess) return e;
            }
            kern<<<l.grid, kBuildWarps * 32, smem, st>>>(a);
            return cudaGetLastError();
        }
    }
    return cudaErrorInvalidValue;
}
// The construction cells of Cell<CH> for bin rows (BIN) or for f32, bf16, fp16 and q8 rows: defined in build_cells.cu, which is
// compiled once per (CH, BIN) so that the cells build in parallel (DESIGN §3d).
template <int CH, bool BIN>
cudaError_t build_cells(const BuildArgs& a, const BuildLaunch& l, cudaStream_t st);

}  // namespace idb
