// graph_range.cu — graph range search (DESIGN.md §9c): for every query, the points within the radius that layer 0 reaches from the
// hits among the query's approximate nearest neighbours, in key order (canonical distance bits << 32 | PointId), returned as CSR.
//
// The result is a closure, a set fixed by a rule rather than by a visit order, so the expansion may run in any order.  Three steps
// on the lane's stream: the seed search (K1 with k = ef, keys written with PointIds), the expansion (graph_range.cuh: a main pass
// with bounded per-warp scratch, then a retry pass for the queries that overflowed it), and the exact range search's ordering
// (range_on_lane, range.cu).  This unit holds the expansion cells of f32, bf16, fp16 and q8 rows; graph_range_bin.cu those of bin rows.
#include <algorithm>
#include <cstring>

#include "graph_range.cuh"

namespace idb {

namespace {

// Main pass, per warp: a frontier of kGrFrontier hits (64 KB) and a visited set of at most kGrVisWords u32 (128 KB): a bitmap of n
// bits while it fits (n <= 2^20: it never fills), else a hash set of that many slots held at most half full.  A query that needs more
// goes to the retry pass.  kGrCtasPerSm * kGrWarps warps per SM: 203 MB of lane scratch on 132 SMs.
constexpr uint32_t kGrFrontier = 8192;
constexpr uint32_t kGrVisWords = 32768;
constexpr int kGrCtasPerSm = 2;
// Retry pass, per warp: a frontier of n hits and a bitmap of n bits (8.1 MB at n = 1M), as many warps as kGrRetryBytes holds (at least
// one, at most one per query handed over and kGrCtasPerSm * kGrWarps per SM).
constexpr size_t kGrRetryBytes = 2ull << 30;

uint32_t pow2_at_least(uint64_t v) {
    uint32_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

GraphRangeKernel pick_graph_range(const Index* ix) {
    return with_row_type(ix->row_type, [&](auto rt) -> GraphRangeKernel {
        using RT = decltype(rt);
        if constexpr (RT::kType == kRowBin) return graph_range_bin_cell(ix->nchunks);
        else return graph_range_cell<RT>(ix->nchunks);
    });
}

idb_status launch_graph_range(const Index* ix, GraphRangeKernel fn, const GraphRangeArgs& a, uint64_t ctas, int wpc, cudaStream_t st) {
    const size_t smem = (size_t)wpc * (kGrWarpSmem + (kernel_ch(ix->nchunks) == 0 ? long_q_bytes(ix->nchunks) : 0));
    if (smem > 48 * 1024) CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    fn<<<(unsigned)ctas, wpc * 32, smem, st>>>(a);
    CUDA_TRY(cudaGetLastError());
    return IDB_OK;
}

}  // namespace

// The graph range search of nq queries (dim floats per row, any alignment, in host memory when `host`, else on the index's device) on
// the lane (the caller holds ln.mu); the outputs as range_on_lane's.  IDB_ERR_CAPACITY also when a seed search overflowed even K1's
// retry pass (idb_last_search_failures then counts those queries).
static idb_status run_graph_range(Index* ix, Lane& ln, const float* queries, bool host, uint64_t nq, uint32_t ef_search, float radius,
                                  uint64_t capacity, uint64_t* offsets, uint32_t* ids, float* dist, uint64_t* out_total) {
    const uint32_t ef = ef_search ? ef_search : ix->ef_search;
    bool seeded = false;
    const idb_status st = range_on_lane(ix, ln, host, nq, capacity, offsets, ids, dist, out_total, [&](const RangeSink& sink) -> idb_status {
        const uint64_t n = ix->n;
        if (n == 0 || ef == 0) return IDB_OK;  // no seeds: every closure is empty
        const float* qp = nullptr;
        idb_status s = ix->stage_queries(ln, queries, host, nq, &qp);
        if (s != IDB_OK) return s;
        CUDA_TRY(ensure_u32(ln.ids, ln.ids_cap, nq * ef));
        CUDA_TRY(ensure_u64(ln.gr_seeds, ln.gr_seeds_cap, nq * ef));
        s = search_on_lane(ix, ln, qp, true, nq, ef, ef, ln.ids, nullptr, nullptr, ln.gr_seeds, /*map_ids=*/false);
        if (s != IDB_OK) return s;
        seeded = true;

        GraphRangeArgs a;
        std::memset(&a, 0, sizeof(a));
        a.g = ix->view();
        // the seed search normalised a cosine index's queries into ln.qn (once per call); the expansion reads those rows
        a.queries = reinterpret_cast<const float4*>(ix->metric == kMetricCosine ? ln.qn : qp);
        a.nq = nq;
        a.seeds = ln.gr_seeds;
        a.ef = ef;
        a.radius = radius;
        a.metric = ix->metric;
        a.out = sink;
        // Main pass.  A frontier of n hits and a bitmap never overflow, so indexes of up to kGrFrontier points need no retry pass.
        // IDB_GRAPH_RANGE_SCRATCH (tests): that many hits and a hash set of 8x as many slots.
        const uint32_t F = (uint32_t)std::min<uint64_t>(ix->graph_range_scratch ? ix->graph_range_scratch : kGrFrontier, n);
        a.bitmap = !ix->graph_range_scratch && (n + 31) / 32 <= kGrVisWords;
        const uint32_t V = a.bitmap ? (uint32_t)((n + 31) / 32) : ix->graph_range_scratch ? pow2_at_least(8ull * F) : kGrVisWords;
        const uint64_t ctas = std::min<uint64_t>((nq + kGrWarps - 1) / kGrWarps, (uint64_t)ix->num_sms * kGrCtasPerSm);
        CUDA_TRY(ensure_u64(ln.gr_front, ln.gr_front_cap, ctas * kGrWarps * F));
        CUDA_TRY(ensure_u32(ln.gr_vis, ln.gr_vis_cap, ctas * kGrWarps * V));
        CUDA_TRY(ensure_u32(ln.gr_ctl, ln.gr_ctl_cap, nq + 4));
        CUDA_TRY(cudaMemsetAsync(ln.gr_ctl, 0, 16, ln.stream));
        a.ctl = ln.gr_ctl;
        a.front = ln.gr_front;
        a.fcap = F;
        a.fstride = F;
        a.vis = ln.gr_vis;
        a.vwords = V;
        a.vshift = a.bitmap ? 0 : 32 - (uint32_t)__builtin_ctz(V);
        a.vstride = V;
        const GraphRangeKernel fn = pick_graph_range(ix);
        s = launch_graph_range(ix, fn, a, ctas, kGrWarps, ln.stream);
        if (s != IDB_OK) return s;

        // Retry pass, for the queries the main pass handed over.
        uint32_t handed = 0;
        const HostCopy hc{&handed, ln.gr_ctl + 1, 4};
        s = copy_to_host(ln, &hc, 1);
        if (s != IDB_OK || handed == 0) return s;
        const uint64_t per_warp = n + (n + 63) / 64;  // u64 words: the frontier, then the bitmap
        uint64_t warps = std::max<uint64_t>(1, kGrRetryBytes / (per_warp * 8));
        warps = std::min<uint64_t>({warps, handed, (uint64_t)ix->num_sms * kGrCtasPerSm * kGrWarps});
        CUDA_TRY(ensure_u64(ln.gr_retry, ln.gr_retry_cap, warps * per_warp));
        GraphRangeArgs r = a;
        r.retry = true;
        r.bitmap = true;
        r.front = ln.gr_retry;
        r.fcap = (uint32_t)n;
        r.fstride = per_warp;
        r.vis = reinterpret_cast<uint32_t*>(ln.gr_retry + n);
        r.vwords = (uint32_t)((n + 31) / 32);
        r.vstride = per_warp * 2;
        return launch_graph_range(ix, fn, r, warps, 1, ln.stream);
    });
    if (!seeded || (st != IDB_OK && st != IDB_ERR_CAPACITY)) return st;
    // The seed search's control block (range_on_lane has synchronised the stream): the host search's overflow bookkeeping, and the
    // queries whose seed search overflowed even K1's retry pass.
    CUDA_TRY(cudaMemcpyAsync(ln.h_ctrl + 1, ln.ctrl, sizeof(SearchCtrl), cudaMemcpyDeviceToHost, ln.stream));
    CUDA_TRY(cudaStreamSynchronize(ln.stream));
    ix->note_overflows(ef, nq, ln.h_ctrl[1].main.fail_count, ln.last_b16);
    if (const uint32_t failed = ln.h_ctrl[1].retry.fail_count)
        return fail(IDB_ERR_CAPACITY, "%u seed searches of %llu queries overflowed an internal per-query structure (visited table / tie list)",
                    failed, (unsigned long long)nq);
    return st;
}

}  // namespace idb

using namespace idb;

extern "C" {

idb_status idb_graph_range_search_batch_f32(idb_index* index, const float* queries, uint64_t nq, uint32_t ef_search, float radius,
                                            uint64_t capacity, uint64_t* out_offsets, uint32_t* out_ids, float* out_dist) {
    const RangeCheck rc{radius, capacity, out_ids, false, nullptr, ef_search};
    idb_status st = check_search_args(Family::range, &index, 1, nullptr, nullptr, queries, nq, out_offsets, 0, &rc);
    if (st != IDB_OK) return st;
    if (nq == 0) {
        if (out_offsets) out_offsets[0] = 0;
        return IDB_OK;
    }
    Index* ix = reinterpret_cast<Index*>(index);
    Lane& ln = ix->pick_lane();
    std::lock_guard<std::mutex> lk(ln.mu, std::adopt_lock);
    ix->last_lane.store((int)(&ln - ix->lanes));
    return run_graph_range(ix, ln, queries, true, nq, ef_search, radius, capacity, out_offsets, out_ids, out_dist, nullptr);
}

idb_status idb_graph_range_search_batch_device_lane(idb_index* index, uint32_t lane, const float* d_queries, uint64_t nq,
                                                    uint32_t ef_search, float radius, uint64_t capacity, uint64_t* d_out_offsets,
                                                    uint32_t* d_out_ids, float* d_out_dist, uint64_t* out_total) {
    const RangeCheck rc{radius, capacity, d_out_ids, true, out_total, ef_search};
    idb_status st = check_search_args(Family::range, &index, 1, nullptr, &lane, d_queries, nq, d_out_offsets, 0, &rc);
    if (st != IDB_OK) return st;
    if (nq == 0) {
        *out_total = 0;
        return IDB_OK;
    }
    Index* ix = reinterpret_cast<Index*>(index);
    Lane& ln = ix->lanes[lane];
    std::lock_guard<std::mutex> lk(ln.mu);
    ix->last_lane.store((int)lane);
    return run_graph_range(ix, ln, d_queries, false, nq, ef_search, radius, capacity, d_out_offsets, d_out_ids, d_out_dist, out_total);
}

}  // extern "C"
