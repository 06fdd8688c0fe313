// graph_range.cuh — the graph range search's expansion kernel (DESIGN.md §9c): one warp per query walks layer 0 outward from the
// query's seeds (the approximate search's `nearest` list) through the points within the radius, and appends the closure's hits as
// (key, query) pairs for the range search's ordering (range.cu).  Included by graph_range.cu (f32, bf16, fp16 and q8 rows) and
// graph_range_bin.cu (bin rows), so that the bin cells compile in a translation unit of their own.
#pragma once
#include "search_kernel.cuh"

namespace idb {

constexpr int kGrWarps = 4;                 // warps per CTA of the main pass (the retry pass: one)
constexpr int kGrRowsPerStep = 128;         // adjacency entries a warp probes per step: the rows of max(1, 128 / 2M) hits
constexpr int kGrWarpSmem = kGrRowsPerStep * 4 + kGrRowsPerStep * 8 + 32 * 4;  // cpid, ckey, the rows' first INVALID slot

struct GraphRangeArgs {
    GraphView g;
    const float4* queries;      // nq x nchunks (zero padded, 16-byte aligned; a cosine index's normalised queries)
    uint64_t nq;
    const uint64_t* seeds;      // nq x ef keys of the seed search (PointIds, not mapped); kKeyNone past a query's list
    uint32_t ef;
    float radius;
    uint32_t metric;
    bool retry;                 // the retry pass: items from the overflow list, bitmap visited sets, frontiers of n hits
    bool bitmap;                // visited sets of n bits (never full), else hash sets
    uint32_t* ctl;              // [0] main pass work counter, [1] queries the main pass handed over, [2] retry work counter, [3] unused,
                                // then the overflow list
    uint64_t* front;            // per warp: fcap hit keys, in the order found
    uint32_t fcap;
    uint32_t* vis;              // per warp: vwords u32 (bitmap: bit set = not visited; hash: slots, a power of two)
    uint32_t vwords;
    uint32_t vshift;            // hash: 32 - log2(vwords)
    uint64_t vstride;           // u32 words between two warps' visited sets
    uint64_t fstride;           // u64 words between two warps' frontiers
    RangeSink out;
};

// Marks pid visited; true when it was not (exact in both flavours).
__device__ __forceinline__ bool gr_visit(const GraphRangeArgs& a, uint32_t* vis, uint32_t pid) {
    if (a.bitmap) return (vis_bitmap_fetch_clear(vis, pid) >> (pid & 31)) & 1u;
    return vis_insert_big(vis, a.vshift, a.vwords - 1u, pid);
}

// Appends the lanes' hits (key valid where hit) to the frontier; false when it would not fit.  Warp-uniform call.
__device__ __forceinline__ bool gr_append(const GraphRangeArgs& a, uint64_t* front, uint32_t& len, bool hit, uint64_t key, int lane) {
    const uint32_t m = __ballot_sync(kFullMask, hit);
    if (len + __popc(m) > a.fcap) return false;
    if (hit) front[len + __popc(m & ((1u << lane) - 1u))] = key;
    len += __popc(m);
    return true;
}

template <int CH, int NB, class RT>
__global__ void __launch_bounds__(kGrWarps * 32) graph_range_kernel(GraphRangeArgs a) {
    extern __shared__ __align__(16) unsigned char sm_gr[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpc = blockDim.x >> 5;  // wpc: kGrWarps, or 1 in the retry pass
    const uint64_t gw = (uint64_t)blockIdx.x * wpc + warp;
    uint32_t* cpid = reinterpret_cast<uint32_t*>(sm_gr + warp * kGrWarpSmem);
    uint64_t* ckey = reinterpret_cast<uint64_t*>(cpid + kGrRowsPerStep);
    uint32_t* first = reinterpret_cast<uint32_t*>(ckey + kGrRowsPerStep);
    uint64_t* front = a.front + gw * a.fstride;
    uint32_t* vis = a.vis + gw * a.vstride;
    const uint32_t nchunks = a.g.nchunks, M2 = 2 * a.g.M;
    const uint32_t rows_per_step = M2 >= (uint32_t)kGrRowsPerStep ? 1u : kGrRowsPerStep / M2;
    const uint32_t vmax = a.bitmap ? 0xFFFFFFFFu : a.vwords / 2;  // a hash set's load stays <= 1/2; a bitmap holds every PointId
    const uint32_t n_work = a.retry ? a.ctl[1] : (uint32_t)a.nq;
    for (;;) {
        uint32_t wi = 0;
        if (lane == 0) wi = atomicAdd(a.ctl + (a.retry ? 2 : 0), 1u);
        wi = __shfl_sync(kFullMask, wi, 0);
        if (wi >= n_work) break;
        const uint64_t qi = a.retry ? a.ctl[4 + wi] : wi;

        QVec<CH> q;
        if constexpr (CH == 0) {
            q.ngroups = (nchunks + 31) / 32;
            q.s = reinterpret_cast<float4*>(sm_gr + wpc * kGrWarpSmem + (size_t)warp * long_q_bytes(nchunks));
        }
        q_from_f32<CH>(q, a.queries + qi * nchunks, nchunks, lane);
        for (uint32_t i = lane; i < a.vwords; i += 32) vis[i] = kInvalid;  // a clean set: no id visited
        __syncwarp();

        // The seeds: every member of nearest(q) is visited (a non-hit cannot be in the closure); the hits start the frontier.
        uint32_t len = 0, nvis = 0;
        bool ok = true;
        for (uint32_t j0 = 0; j0 < a.ef && ok; j0 += 32) {
            const uint64_t key = j0 + lane < a.ef ? a.seeds[qi * a.ef + j0 + lane] : kKeyNone;
            ok = (uint64_t)nvis + 32 <= vmax;
            if (!ok) break;
            const bool fresh = key != kKeyNone && gr_visit(a, vis, key_pid(key));
            nvis += __popc(__ballot_sync(kFullMask, fresh));
            ok = gr_append(a, front, len, fresh && reported_distance(key_dbits(key), a.metric) <= a.radius, key, lane);  // NaN: never
        }
        __syncwarp();

        // The closure: the hits' zero rows up to their first INVALID, rows_per_step hits at a time; fresh entries get their canonical
        // distance, and those within the radius join the frontier.
        for (uint32_t head = 0; ok && head < len;) {
            const uint32_t nr = min(rows_per_step, len - head), ne = nr * M2;
            if ((uint32_t)lane < nr) first[lane] = M2;
            __syncwarp();
            uint32_t pid[kGrRowsPerStep / 32];
#pragma unroll
            for (int k = 0; k < kGrRowsPerStep / 32; ++k) {
                const uint32_t e = lane + 32 * k, r = e / M2;
                pid[k] = e < ne ? a.g.zero[(uint64_t)key_pid(front[head + r]) * M2 + (e - r * M2)] : kInvalid;
                if (e < ne && pid[k] == kInvalid) atomicMin(first + r, e - r * M2);
            }
            __syncwarp();
            ok = (uint64_t)nvis + ne <= vmax;
            if (!ok) break;
            uint32_t n_new = 0;
#pragma unroll
            for (int k = 0; k < kGrRowsPerStep / 32; ++k) {
                const uint32_t e = lane + 32 * k, r = e / M2;
                const bool fresh = e < ne && e - r * M2 < first[r] && gr_visit(a, vis, pid[k]);
                const uint32_t m = __ballot_sync(kFullMask, fresh);
                if (fresh) cpid[n_new + __popc(m & ((1u << lane) - 1u))] = pid[k];
                n_new += __popc(m);
            }
            __syncwarp();
            nvis += n_new;
            head += nr;
            if (n_new) batch_distances<CH, NB, RT>(a.g, q, cpid, ckey, n_new, lane);
            for (uint32_t i0 = 0; i0 < n_new && ok; i0 += 32) {
                const uint32_t i = i0 + lane;
                const uint64_t key = i < n_new ? ckey[i] : kKeyNone;
                ok = gr_append(a, front, len, i < n_new && reported_distance(key_dbits(key), a.metric) <= a.radius, key, lane);
            }
            __syncwarp();
        }

        if (!ok) {  // main pass only: the retry pass's sets hold every PointId
            if (lane == 0) a.ctl[4 + atomicAdd(a.ctl + 1, 1u)] = (uint32_t)qi;
        } else {  // the range collector: one claim for the query's hits
            unsigned long long base = 0;
            if (lane == 0) {
                a.out.counts[qi] = len;
                if (len) base = atomicAdd(a.out.total, (unsigned long long)len);
            }
            base = shfl64(base, 0);
            for (uint32_t i = lane; i < len; i += 32)
                if (base + i < a.out.capacity) {
                    a.out.keys[base + i] = front[i];
                    a.out.qids[base + i] = (uint32_t)qi;
                }
        }
        __syncwarp();
    }
}

using GraphRangeKernel = void (*)(GraphRangeArgs);

// The cell for rows of nchunks chunks and row type RT: K1's rows in flight per lane, rows_in_flight<B, RT>() of with_cell's Cell (the
// long rows, CH 0, take B as is).
template <class RT>
GraphRangeKernel graph_range_cell(uint32_t nchunks) {
    return with_cell(nchunks, [](auto cell) -> GraphRangeKernel {
        using C = decltype(cell);
        return graph_range_kernel<C::CH, C::CH == 0 ? C::B : rows_in_flight<C::B, RT>(), RT>;
    });
}
// graph_range_bin.cu
GraphRangeKernel graph_range_bin_cell(uint32_t nchunks);

}  // namespace idb
