// build_dispatch.cuh — launch helpers for the construction kernels, instantiated once per CH in build_chN.cu.
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

template <int CH, int B, int NB, class RT>
cudaError_t build_dispatch_rt(const BuildArgs& a, const BuildLaunch& l, cudaStream_t st) {
    switch (l.op) {
        case kOpInsertSearch:
            return with_tile(l.row_t, l.ef_t, [&](auto row, auto ef) {
                constexpr int ROW_T = decltype(row)::value, EF_T = decltype(ef)::value;
                return launch_traversal<CH, EF_T>(insert_search_kernel<CH, ROW_T, EF_T, B, RT>, a, 0, l.grid, st, l.win);
            });
        case kOpSelectNew:
        case kOpRelink:
            if constexpr (CH > 0) {
                if (l.stage) return launch_k2<CH, NB, true, RT>(a, l, st);
            }
            return launch_k2<CH, NB, false, RT>(a, l, st);
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
// The construction cells of bin rows (DESIGN §3d): declared here and defined in bin_cells.cuh, which only build_bin_chN.cu includes,
// so that they compile in translation units of their own, in parallel with build_chN.cu's cells of the other row types.
template <int CH, int B, int NB>
cudaError_t build_dispatch_bin(const BuildArgs& a, const BuildLaunch& l, cudaStream_t st);
template <int CH, int B, int NB>
cudaError_t build_dispatch(const BuildArgs& a, const BuildLaunch& l, cudaStream_t st) {
    return with_row_type(a.g.row_type, [&](auto rt) {
        using RT = decltype(rt);
        if constexpr (RT::kType == kRowBin) return build_dispatch_bin<CH, B, NB>(a, l, st);
        else return build_dispatch_rt<CH, B, NB, RT>(a, l, st);
    });
}

// K2's ladder, for other kernels built on select_heuristic_warp (remove.cu): f(CH, NB) as integral constants, with the (CH, NB) that
// build_chN.cu instantiates for rows of `nchunks` chunks.
template <int CH_, int NB_>
struct K2Cell {
    static constexpr int CH = CH_, NB = NB_;
};
template <class F>
cudaError_t with_k2_cell(uint32_t nchunks, F&& f) {
    switch (kernel_ch(nchunks)) {
        case 1: return f(K2Cell<1, 16>());
        case 2: return f(K2Cell<2, 8>());
        case 3: return f(K2Cell<3, 4>());
        case 4: return f(K2Cell<4, 4>());
        case 6: return f(K2Cell<6, 2>());
        case 8: return f(K2Cell<8, 2>());
        default: return f(K2Cell<0, kLongRowsInFlight>());
    }
}

}  // namespace idb
