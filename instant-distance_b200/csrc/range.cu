// range.cu — exact range search: for every query, every stored row whose reported distance is <= radius, in key order (canonical
// distance bits << 32 | PointId), returned as CSR (DESIGN.md §9b).
//
// The distances are the exact scan's (scan_step, scan.cuh), so a query's hits are a prefix of its exact ordering.  The scan appends
// each hit as a (key, query) pair at a position claimed with one 64-bit atomic per warp ballot and counts the query's hits; an
// exclusive scan of the counts gives the offsets.  Once the total is known on the host, the pairs are gathered into their queries'
// segments, each segment is sorted by key (CUB's segmented sort), and the ids (through the id map) and reported distances are
// written.  Keys are unique within a query, so the output does not depend on the order of the appends.
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include <algorithm>
#include <cstring>

#include "scan.cuh"

namespace idb {

namespace {

constexpr size_t kRangeScratchBytes = 256ull << 20;  // pair scratch kept by a lane between calls (the exact search's list scratch)

struct RangeArgs {
    GraphView g;
    const float4* queries;      // nq x nchunks (zero padded, 16-byte aligned)
    uint64_t nq;
    uint64_t slice_rows;        // rows per slice (the last one may be shorter or empty)
    float radius;
    uint32_t metric;
    uint32_t* counts;           // nq: hits per query
    unsigned long long* total;  // hits appended so far
    uint64_t capacity;          // pairs the append buffer holds; later hits are counted only
    uint64_t* keys;             // capacity appended keys ...
    uint32_t* qids;             // ... and their queries
};

template <int CH, class RT>
__global__ void __launch_bounds__(kScanWarps * 32) range_scan_kernel(RangeArgs a) {
    constexpr int QW = ScanShape<CH>::QW;
    static_assert(CH > 0 || QW == 1, "long rows: one query per warp (it lives in shared memory)");
    extern __shared__ float4 sm_range_q[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpc = blockDim.x >> 5;
    const uint64_t q0 = ((uint64_t)blockIdx.x * wpc + warp) * QW;
    if (q0 >= a.nq) return;
    const uint32_t nchunks = a.g.nchunks;
    const uint64_t r0 = min(a.g.n, (uint64_t)blockIdx.y * a.slice_rows), r1 = min(a.g.n, r0 + a.slice_rows);

    QVec<CH> q[QW];
#pragma unroll
    for (int j = 0; j < QW; ++j) {
        const uint64_t qi = q0 + j < a.nq ? q0 + j : q0;
        if constexpr (CH == 0) {
            q[j].ngroups = (nchunks + 31) / 32;
            q[j].s = sm_range_q + (size_t)warp * q[j].ngroups * 32;
        }
        q_from_f32<CH>(q[j], a.queries + qi * nchunks, nchunks, lane);
    }

    constexpr int NB = ScanShape<CH>::NB;
    const uint32_t row_bytes = nchunks * RT::kChunkBytes;
    const char* lane_base = a.g.points + lane * RT::kChunkBytes;
#pragma unroll 1
    for (uint64_t b0 = r0; b0 < r1; b0 += NB) {
        const uint32_t nb = r1 - b0 < (uint64_t)NB ? (uint32_t)(r1 - b0) : (uint32_t)NB;
        float d[QW];
        scan_step<CH, RT>(a.g, nchunks, q, lane_base, row_bytes, b0, nb, lane, d);
        const uint32_t pid = (uint32_t)(b0 + (lane & (NB - 1)));
        const bool mine = lane < NB && (uint32_t)lane < nb;
        // the range collector: a ballot per query slot, one lane claims the hits' positions
#pragma unroll
        for (int qj = 0; qj < QW; ++qj) {
            const uint64_t qi = q0 + qj;
            const uint32_t dbits = canon_bits(d[qj]);
            const bool hit = mine && qi < a.nq && reported_distance(dbits, a.metric) <= a.radius;  // NaN is <= no radius
            const uint32_t m = __ballot_sync(kFullMask, hit);
            if (!m) continue;
            unsigned long long base = 0;
            if (lane == 0) {
                atomicAdd(a.counts + qi, (uint32_t)__popc(m));
                base = atomicAdd(a.total, (unsigned long long)__popc(m));
            }
            const uint64_t pos = shfl64(base, 0) + (uint32_t)__popc(m & ((1u << lane) - 1u));
            if (hit && pos < a.capacity) {
                a.keys[pos] = ((uint64_t)dbits << 32) | pid;
                a.qids[pos] = (uint32_t)qi;
            }
        }
    }
}

// Pair i into its query's segment, at offsets[q] + the next free slot of the query (cursor: nq zeros).
__global__ void range_gather_kernel(const uint64_t* keys, const uint32_t* qids, uint64_t total, const uint64_t* offsets, uint32_t* cursor,
                                    uint64_t* seg) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t q = qids[i];
        seg[offsets[q] + atomicAdd(cursor + q, 1u)] = keys[i];
    }
}

// The sorted keys as the caller sees them: ids through the id map, distances as the metric reports them (dist optional).
__global__ void range_finish_kernel(const uint64_t* sorted, uint64_t total, const uint32_t* id_map, uint32_t metric, uint32_t* ids,
                                    float* dist) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t key = sorted[i];
        const uint32_t pid = key_pid(key);
        ids[i] = id_map ? id_map[pid] : pid;
        if (dist) dist[i] = reported_distance(key_dbits(key), metric);
    }
}

using RangeKernel = void (*)(RangeArgs);
struct RangeChoice {
    RangeKernel fn;
    int qw;
};
RangeChoice pick_range(uint32_t nchunks, uint32_t row_type) {
    return with_cell(nchunks, [&](auto cell) {
        constexpr int CH = decltype(cell)::CH;
        return with_row_type(row_type, [](auto rt) { return RangeChoice{range_scan_kernel<CH, decltype(rt)>, ScanShape<CH>::QW}; });
    });
}

unsigned grid_for(const Index* ix, uint64_t items) {
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((items + 255) / 256, (uint64_t)ix->num_sms * 8));
}

// CUB's scratch for `bytes` bytes in the lane's buffer.
cudaError_t ensure_tmp(Lane& ln, size_t bytes) { return ensure_u64(ln.range_tmp, ln.range_tmp_cap, (bytes + 7) / 8); }

// Frees the lane's pair scratch (and the graph range search's expansion scratch) at the end of a call when one large call grew it past
// kRangeScratchBytes.
struct TrimScratch {
    Lane& ln;
    ~TrimScratch() {
        if (ln.range_keys_cap * 8 + ln.range_qids_cap * 4 + ln.range_seg_cap * 8 + ln.range_tmp_cap * 8 + ln.gr_front_cap * 8 +
                ln.gr_vis_cap * 4 + ln.gr_retry_cap * 8 <=
            kRangeScratchBytes)
            return;
        cudaStreamSynchronize(ln.stream);
        cudaFree(ln.range_keys); cudaFree(ln.range_qids); cudaFree(ln.range_seg); cudaFree(ln.range_tmp);
        cudaFree(ln.gr_front); cudaFree(ln.gr_vis); cudaFree(ln.gr_retry);
        ln.range_keys = ln.range_seg = ln.range_tmp = ln.gr_front = ln.gr_retry = nullptr;
        ln.range_qids = ln.gr_vis = nullptr;
        ln.range_keys_cap = ln.range_qids_cap = ln.range_seg_cap = ln.range_tmp_cap = ln.gr_front_cap = ln.gr_vis_cap = ln.gr_retry_cap = 0;
    }
};

}  // namespace

idb_status range_on_lane(Index* ix, Lane& ln, bool host, uint64_t nq, uint64_t capacity, uint64_t* offsets, uint32_t* ids, float* dist,
                         uint64_t* out_total, const std::function<idb_status(const RangeSink&)>& collect) {
    CUDA_TRY(cudaSetDevice(ix->device));
    TrimScratch trim{ln};
    cudaStream_t st = ln.stream;
    CUDA_TRY(ensure_u64(ln.range_off, ln.range_off_cap, nq + 2));
    uint64_t* d_off = host ? ln.range_off : offsets;                                   // nq + 1
    unsigned long long* d_total = reinterpret_cast<unsigned long long*>(ln.range_off + nq + 1);
    CUDA_TRY(ensure_u32(ln.len, ln.len_cap, nq + 1));
    uint32_t* counts = ln.len;                                                         // nq + 1, the last one stays 0
    CUDA_TRY(cudaMemsetAsync(counts, 0, (nq + 1) * 4, st));
    CUDA_TRY(cudaMemsetAsync(d_total, 0, 8, st));
    if (capacity) {
        CUDA_TRY(ensure_u64(ln.range_keys, ln.range_keys_cap, capacity));
        CUDA_TRY(ensure_u32(ln.range_qids, ln.range_qids_cap, capacity));
    }
    idb_status s = collect(RangeSink{counts, d_total, capacity, ln.range_keys, ln.range_qids});
    if (s != IDB_OK) return s;

    // offsets = the exclusive scan of the counts; offsets[nq] = the total
    size_t scan_bytes = 0;
    CUDA_TRY(cub::DeviceScan::ExclusiveScan(nullptr, scan_bytes, counts, d_off, ::cuda::std::plus<>{}, (uint64_t)0, (int)(nq + 1), st));
    CUDA_TRY(ensure_tmp(ln, scan_bytes));
    CUDA_TRY(cub::DeviceScan::ExclusiveScan(ln.range_tmp, scan_bytes, counts, d_off, ::cuda::std::plus<>{}, (uint64_t)0, (int)(nq + 1), st));
    uint64_t total = 0;
    const HostCopy hc = host ? HostCopy{offsets, d_off, (nq + 1) * 8} : HostCopy{out_total, d_off + nq, 8};
    s = copy_to_host(ln, &hc, 1);
    if (s != IDB_OK) return s;
    total = host ? offsets[nq] : *out_total;
    if (total > capacity)
        return fail(IDB_ERR_CAPACITY, "the range search found %llu hits, capacity is %llu", (unsigned long long)total,
                    (unsigned long long)capacity);
    if (total == 0) return IDB_OK;

    CUDA_TRY(ensure_u64(ln.range_seg, ln.range_seg_cap, total));
    CUDA_TRY(cudaMemsetAsync(counts, 0, nq * 4, st));  // the gather's cursors
    range_gather_kernel<<<grid_for(ix, total), 256, 0, st>>>(ln.range_keys, ln.range_qids, total, d_off, counts, ln.range_seg);
    CUDA_TRY(cudaGetLastError());
    cub::DoubleBuffer<uint64_t> keys(ln.range_seg, ln.range_keys);
    size_t sort_bytes = 0;
    CUDA_TRY(cub::DeviceSegmentedSort::SortKeys(nullptr, sort_bytes, keys, (int)total, (int)nq, d_off, d_off + 1, st));
    CUDA_TRY(ensure_tmp(ln, sort_bytes));
    CUDA_TRY(cub::DeviceSegmentedSort::SortKeys(ln.range_tmp, sort_bytes, keys, (int)total, (int)nq, d_off, d_off + 1, st));
    // the host call's ids and distances go to the free half of the double buffer (total u64 = total ids + total distances)
    uint32_t* d_ids = host ? reinterpret_cast<uint32_t*>(keys.Alternate()) : ids;
    float* d_dist = host ? (dist ? reinterpret_cast<float*>(d_ids + total) : nullptr) : dist;
    range_finish_kernel<<<grid_for(ix, total), 256, 0, st>>>(keys.Current(), total, ix->d_id_map, ix->metric, d_ids, d_dist);
    CUDA_TRY(cudaGetLastError());
    if (!host) {
        CUDA_TRY(cudaStreamSynchronize(st));
        return IDB_OK;
    }
    const HostCopy out[2] = {{ids, d_ids, total * 4}, {dist, d_dist, total * 4}};
    return copy_to_host(ln, out, 2);
}

// The exact range search of nq queries (dim floats per row, any alignment, in host memory when `host`, else on the index's device) on
// the lane (the caller holds ln.mu): range_scan_kernel over every stored row collects the hits.
static idb_status run_range(Index* ix, Lane& ln, const float* queries, bool host, uint64_t nq, float radius, uint64_t capacity,
                            uint64_t* offsets, uint32_t* ids, float* dist, uint64_t* out_total) {
    return range_on_lane(ix, ln, host, nq, capacity, offsets, ids, dist, out_total, [&](const RangeSink& sink) -> idb_status {
        if (ix->n == 0) return IDB_OK;
        const float* qp = nullptr;
        idb_status s = ix->stage_queries(ln, queries, host, nq, &qp);
        if (s == IDB_OK) s = ix->normalize_queries(ln, &qp, nq);
        if (s != IDB_OK) return s;
        const RangeChoice rc = pick_range(ix->nchunks, ix->row_type);
        ScanLaunch sl;
        s = scan_launch(ix, rc.fn, &sl);
        if (s != IDB_OK) return s;
        // Slices: enough CTAs for about four waves of the device, at least kScanMinSliceRows rows each.
        const uint64_t q_per_cta = (uint64_t)sl.wpc * rc.qw;
        const uint64_t want_ctas = 4ull * std::max(1, sl.occ) * ix->num_sms;
        const uint64_t q_ctas = (nq + q_per_cta - 1) / q_per_cta;
        uint64_t S = (want_ctas + q_ctas - 1) / q_ctas;
        S = std::min<uint64_t>(S, (ix->n + kScanMinSliceRows - 1) / kScanMinSliceRows);
        S = std::max<uint64_t>(S, 1);
        RangeArgs a;
        std::memset(&a, 0, sizeof(a));
        a.g = ix->view();
        a.queries = reinterpret_cast<const float4*>(qp);
        a.nq = nq;
        a.slice_rows = (ix->n + S - 1) / S;
        a.radius = radius;
        a.metric = ix->metric;
        a.counts = sink.counts;
        a.total = sink.total;
        a.capacity = sink.capacity;
        a.keys = sink.keys;
        a.qids = sink.qids;
        rc.fn<<<dim3((unsigned)q_ctas, (unsigned)S), sl.wpc * 32, sl.smem, ln.stream>>>(a);
        CUDA_TRY(cudaGetLastError());
        return IDB_OK;
    });
}

}  // namespace idb

using namespace idb;

extern "C" {

idb_status idb_range_search_batch_f32(idb_index* index, const float* queries, uint64_t nq, float radius, uint64_t capacity,
                                      uint64_t* out_offsets, uint32_t* out_ids, float* out_dist) {
    const RangeCheck rc{radius, capacity, out_ids, false, nullptr};
    idb_status st = check_search_args(Family::range, &index, 1, nullptr, nullptr, queries, nq, out_offsets, 0, &rc);
    if (st != IDB_OK) return st;
    if (nq == 0) {
        if (out_offsets) out_offsets[0] = 0;
        return IDB_OK;
    }
    Index* ix = reinterpret_cast<Index*>(index);
    Lane& ln = ix->pick_lane();
    std::lock_guard<std::mutex> lk(ln.mu, std::adopt_lock);
    return run_range(ix, ln, queries, true, nq, radius, capacity, out_offsets, out_ids, out_dist, nullptr);
}

idb_status idb_range_search_batch_device_lane(idb_index* index, uint32_t lane, const float* d_queries, uint64_t nq, float radius,
                                              uint64_t capacity, uint64_t* d_out_offsets, uint32_t* d_out_ids, float* d_out_dist,
                                              uint64_t* out_total) {
    const RangeCheck rc{radius, capacity, d_out_ids, true, out_total};
    idb_status st = check_search_args(Family::range, &index, 1, nullptr, &lane, d_queries, nq, d_out_offsets, 0, &rc);
    if (st != IDB_OK) return st;
    if (nq == 0) {
        *out_total = 0;
        return IDB_OK;
    }
    Index* ix = reinterpret_cast<Index*>(index);
    Lane& ln = ix->lanes[lane];
    std::lock_guard<std::mutex> lk(ln.mu);
    return run_range(ix, ln, d_queries, false, nq, radius, capacity, d_out_offsets, d_out_ids, d_out_dist, out_total);
}

}  // extern "C"
