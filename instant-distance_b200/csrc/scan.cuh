// scan.cuh — the exact scan (DESIGN.md §9a, §9b): every stored row of one slice against a warp's queries, with K1's own distance
// bits, shared by the exact k-NN search (exact.cu) and the range search (range.cu).  What happens to a distance once it is computed
// is the caller's: the top-k list insert, or the range collector.
#pragma once
#include <algorithm>

#include "internal.cuh"

namespace idb {

constexpr int kScanWarps = 8;                  // warps per CTA: they walk the same rows in the same order (L1 serves the others)
constexpr uint64_t kScanMinSliceRows = 1024;   // rows per slice at least

// Queries per warp (QW) and rows per step (NB) of each CH: about 32 registers of query and 32-64 of rows per lane.
template <int CH>
struct ScanShape {
    static constexpr int QW = CH == 1 ? 8 : CH == 2 ? 4 : (CH == 3 || CH == 4 || CH == 6) ? 2 : 1;
    static constexpr int NB = CH == 0 ? kLongRowsInFlight : CH == 1 ? 8 : CH <= 3 ? 4 : 2;
};

// One step of the scan: the distances of rows [b0, b0 + nb) (nb <= NB) to the warp's QW queries q, lane_base = g.points + lane *
// RT::kChunkBytes.  Every distance comes from lane_partial + batch_butterfly, the helpers K1 computes its distances with, so the two
// agree bit for bit.  Lane l gets d[qj] = the distance of query slot qj to row b0 + (l & (NB - 1)).  Warp-uniform call.
//
// The caller keeps the loop over the steps and what it does with d: with the loop here and the collector a template parameter, the
// exact cells' registers moved (DESIGN §9b).
template <int CH, class RT>
__device__ __forceinline__ void scan_step(const GraphView& g, uint32_t nchunks, QVec<CH> (&q)[ScanShape<CH>::QW], const char* lane_base,
                                          uint32_t row_bytes, uint64_t b0, uint32_t nb, int lane, float (&d)[ScanShape<CH>::QW]) {
    constexpr int QW = ScanShape<CH>::QW, NB = ScanShape<CH>::NB;
    if constexpr (CH == 0) {  // batch_distances_long's order: four chains per row carried across groups of 32 chunks
        const char* row[NB];
        typename RT::Hdr h[NB];
        float4 acc[NB];
#pragma unroll
        for (int i = 0; i < NB; ++i) {
            row[i] = lane_base + (size_t)(b0 + ((uint32_t)i < nb ? i : 0)) * row_bytes;
            h[i] = RT::hdr(g, (uint32_t)(b0 + ((uint32_t)i < nb ? i : 0)));
            acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll 1
        for (uint32_t j = 0; j < q[0].ngroups; ++j) {
            const bool ok = lane + 32u * j < nchunks;
            const float4 qq = q[0].s[lane + 32u * j];
            typename RT::Raw v[NB];
#pragma unroll
            for (int i = 0; i < NB; ++i) v[i] = (ok && (uint32_t)i < nb) ? RT::ld_raw(row[i] + (size_t)j * 32 * RT::kChunkBytes) : RT::zero();
#pragma unroll
            for (int i = 0; i < NB; ++i) l2_step(acc[i], qq, widen_chunk<RT>(g, v[i], h[i], lane + 32u * j));
        }
        float p[NB];
#pragma unroll
        for (int i = 0; i < NB; ++i) p[i] = lane_sum(acc[i]);
        d[0] = batch_butterfly<NB>(p, lane);
    } else {  // batch_distances_impl's order, the rows shared by the warp's QW queries
        typename RT::Raw v[NB][CH];
        typename RT::Hdr h[NB];
#pragma unroll
        for (int i = 0; i < NB; ++i) {
            const bool ok = (uint32_t)i < nb;
            const char* row = lane_base + (size_t)(b0 + (ok ? i : 0)) * row_bytes;
            h[i] = RT::hdr(g, (uint32_t)(b0 + (ok ? i : 0)));
#pragma unroll
            for (int j = 0; j < CH; ++j)
                v[i][j] = (ok && (uint32_t)(lane + 32 * j) < nchunks) ? RT::ld_raw(row + j * 32 * RT::kChunkBytes) : RT::zero();
        }
#pragma unroll
        for (int qj = 0; qj < QW; ++qj) {
            float p[NB];
#pragma unroll
            for (int i = 0; i < NB; ++i) p[i] = lane_partial_raw<CH, RT>(g, q[qj].r, v[i], h[i], lane);
            d[qj] = batch_butterfly<NB>(p, lane);  // lane l: row b0 + (l & (NB - 1))
        }
    }
}

// How a scan kernel is launched for rows of `nchunks` chunks: warps per CTA (wpc), dynamic shared memory (the long-row kernels keep
// one query per warp there, so very long rows get fewer warps per CTA) and resident CTAs per SM (occ).
struct ScanLaunch {
    int wpc;
    size_t smem;
    int occ;
};
template <class Kernel>
idb_status scan_launch(const Index* ix, Kernel* fn, ScanLaunch* out) {
    out->wpc = kScanWarps;
    out->smem = 0;
    const uint32_t nchunks = ix->nchunks;
    if (kernel_ch(nchunks) == 0) {
        int max_smem = 0;
        CUDA_TRY(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, ix->device));
        const size_t per_warp = (size_t)(nchunks + 31) / 32 * 32 * 16;
        out->wpc = (int)std::min<size_t>(kScanWarps, (size_t)max_smem / per_warp);
        if (out->wpc < 1) return fail(IDB_ERR_UNSUPPORTED, "dim %u: one query does not fit the device's shared memory", ix->dim);
        out->smem = per_warp * out->wpc;
        if (out->smem > 48 * 1024) CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)out->smem));
    }
    out->occ = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&out->occ, fn, out->wpc * 32, out->smem));
    return IDB_OK;
}

}  // namespace idb
