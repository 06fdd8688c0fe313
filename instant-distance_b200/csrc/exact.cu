// exact.cu — exact k-nearest-neighbour search: for every query, the k smallest keys (canonical distance bits << 32 | PointId) over ALL
// stored rows (DESIGN.md §9a).
//
// A warp holds QW queries in registers (lane l owns chunks l, l+32, ... of each, as in K1) and streams the rows of one slice of the
// index NB at a time (scan_step, scan.cuh), with K1's own distance bits.  Each (query, slice) keeps a sorted list of its k smallest
// keys in global scratch; a new key is compared with the list's k-th key and almost always rejected there.  Slices split the rows when the queries alone do not fill the device; their
// lists are merged by K4 (merge.cu).
#include <algorithm>
#include <cstring>

#include "scan.cuh"

namespace idb {

namespace {

constexpr uint64_t kExactScratchKeys = 1ull << 25;  // keys of per-call list scratch (256 MB): larger batches run in query chunks
constexpr uint32_t kExactMaxSliceKeys = 2048;  // slices x k: K4's cost grows with its square

struct ExactArgs {
    GraphView g;
    const float4* queries;      // nq x nchunks (zero padded, 16-byte aligned)
    uint64_t nq;                // queries of this chunk
    uint32_t k;
    uint32_t S;                 // slices
    uint64_t slice_rows;        // rows per slice (the last one may be shorter or empty)
    uint64_t* lists;            // S x nq x k keys
    // S == 1: the scan kernel writes the results itself
    uint32_t* out_ids;
    float* out_dist;
    uint32_t* out_len;
    const uint32_t* id_map;
    uint32_t metric;
};

// Adds the keys of the lanes in m (distinct, each below the list's k-th key) to the sorted list L of cnt <= k keys.  New position of
// an old entry: its index + #{new keys below it}; of a new key: lower_bound in L + #{new keys below it} (K1's rank rule).  Entries
// only move up, so the old ones are moved top down, 32 at a time, each chunk read before it is written.  Returns the new k-th key
// (kKeyNone while the list holds fewer than k).  Warp-uniform call.
__device__ __forceinline__ uint64_t list_insert(uint64_t* L, uint32_t& cnt, uint32_t k, uint64_t key, uint32_t m, int lane) {
    const bool in = (m >> lane) & 1u;
    uint32_t r = 0;
    uint64_t kmin = kKeyNone;
    for (uint32_t mm = m; mm; mm &= mm - 1) {
        const uint64_t o = shfl64(key, __ffs(mm) - 1);
        r += o < key ? 1u : 0u;
        kmin = o < kmin ? o : kmin;
    }
    const uint32_t lo = lower_bound_keys(L, cnt, kmin);
    const uint32_t pos = in ? lower_bound_keys(L, cnt, key) + r : k;
    if (cnt > lo) {
        for (int32_t base = (int32_t)((cnt - 1) & ~31u); base >= (int32_t)(lo & ~31u); base -= 32) {
            const uint32_t idx = (uint32_t)base + lane;
            const bool have = idx >= lo && idx < cnt;
            const uint64_t x = have ? L[idx] : kKeyNone;
            uint32_t s = 0;
            for (uint32_t mm = m; mm; mm &= mm - 1) s += shfl64(key, __ffs(mm) - 1) < x ? 1u : 0u;
            __syncwarp();
            if (have && idx + s < k) L[idx + s] = x;
            __syncwarp();
        }
    }
    if (in && pos < k) L[pos] = key;
    __syncwarp();
    cnt = min(k, cnt + (uint32_t)__popc(m));
    return cnt == k ? L[k - 1] : kKeyNone;
}

template <int CH, class RT>
__global__ void __launch_bounds__(kScanWarps * 32) exact_scan_kernel(ExactArgs a) {
    constexpr int QW = ScanShape<CH>::QW;
    static_assert(CH > 0 || QW == 1, "long rows: one query per warp (it lives in shared memory)");
    extern __shared__ float4 sm_exact_q[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpc = blockDim.x >> 5;
    const uint64_t q0 = ((uint64_t)blockIdx.x * wpc + warp) * QW;
    if (q0 >= a.nq) return;
    const uint32_t nchunks = a.g.nchunks;
    const uint64_t r0 = min(a.g.n, (uint64_t)blockIdx.y * a.slice_rows), r1 = min(a.g.n, r0 + a.slice_rows);

    QVec<CH> q[QW];
    uint64_t* L[QW];
    uint32_t cnt[QW];
    uint64_t thr[QW];  // the list's k-th key; 0 for a slot past the batch (no key is below it)
#pragma unroll
    for (int j = 0; j < QW; ++j) {
        const uint64_t qi = q0 + j < a.nq ? q0 + j : q0;
        L[j] = a.lists + ((size_t)blockIdx.y * a.nq + qi) * a.k;
        cnt[j] = 0;
        thr[j] = q0 + j < a.nq ? kKeyNone : 0ull;
        if constexpr (CH == 0) {
            q[j].ngroups = (nchunks + 31) / 32;
            q[j].s = sm_exact_q + (size_t)warp * q[j].ngroups * 32;
        }
        q_from_f32<CH>(q[j], a.queries + qi * nchunks, nchunks, lane);
    }

    constexpr int NB = ScanShape<CH>::NB;
    const uint32_t row_bytes = nchunks * RT::kChunkBytes;
    const char* lane_base = a.g.points + lane * RT::kChunkBytes;
    const bool mine_lane = lane < NB;
#pragma unroll 1
    for (uint64_t b0 = r0; b0 < r1; b0 += NB) {
        const uint32_t nb = r1 - b0 < (uint64_t)NB ? (uint32_t)(r1 - b0) : (uint32_t)NB;
        float d[QW];
        scan_step<CH, RT>(a.g, nchunks, q, lane_base, row_bytes, b0, nb, lane, d);
        const uint32_t pid = (uint32_t)(b0 + (lane & (NB - 1)));
        const bool mine = mine_lane && (uint32_t)lane < nb;
#pragma unroll
        for (int qj = 0; qj < QW; ++qj) {
            const uint64_t key = mk_key(d[qj], pid);
            const uint32_t m = __ballot_sync(kFullMask, mine && key < thr[qj]);
            if (m) thr[qj] = list_insert(L[qj], cnt[qj], a.k, key, m, lane);
        }
    }

#pragma unroll
    for (int j = 0; j < QW; ++j) {
        const uint64_t qi = q0 + j;
        if (qi >= a.nq) break;
        if (a.S == 1) {  // K1's epilogue: ids through the id map, distances as the metric reports them, padding
            for (uint32_t t = lane; t < a.k; t += 32) {
                const bool real = t < cnt[j];
                const uint64_t key = real ? L[j][t] : kKeyNone;
                const uint32_t pid = key_pid(key);
                a.out_ids[qi * a.k + t] = real ? (a.id_map ? a.id_map[pid] : pid) : kInvalid;
                if (a.out_dist) a.out_dist[qi * a.k + t] = real ? reported_distance(key_dbits(key), a.metric) : __int_as_float(0x7f800000);
            }
            if (a.out_len && lane == 0) a.out_len[qi] = cnt[j];
        } else {  // K4 reads k keys per list
            for (uint32_t t = cnt[j] + lane; t < a.k; t += 32) L[j][t] = kKeyNone;
        }
    }
}

__global__ void apply_id_map_kernel(uint32_t* ids, uint64_t n, const uint32_t* id_map) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        if (ids[i] != kInvalid) ids[i] = id_map[ids[i]];
}

using ScanKernel = void (*)(ExactArgs);
struct ScanChoice {
    ScanKernel fn;
    int qw;
};
ScanChoice pick_scan(uint32_t nchunks, uint32_t row_type) {
    return with_cell(nchunks, [&](auto cell) {
        constexpr int CH = decltype(cell)::CH;
        return with_row_type(row_type, [](auto rt) { return ScanChoice{exact_scan_kernel<CH, decltype(rt)>, ScanShape<CH>::QW}; });
    });
}

}  // namespace

// The exact search of nq queries (dim floats per row, any alignment, in host memory when `host`, else on the index's device)
// enqueued on the lane's stream.  The caller holds ln.mu.  The lane's diagnostics of approximate searches are left as they are.
static idb_status enqueue_exact(Index* ix, Lane& ln, const float* queries, bool host, uint64_t nq, uint32_t k, uint32_t* d_ids,
                                float* d_dist, uint32_t* d_len) {
    CUDA_TRY(cudaSetDevice(ix->device));
    cudaStream_t st = ln.stream;
    if (ix->n == 0) {
        CUDA_TRY(write_empty(st, nq, k, d_ids, d_dist, d_len, nullptr));
        return IDB_OK;
    }
    const uint32_t nchunks = ix->nchunks;
    const size_t stride = (size_t)nchunks * 4;
    const float* qp = nullptr;
    idb_status s = ix->stage_queries(ln, queries, host, nq, &qp);
    if (s == IDB_OK) s = ix->normalize_queries(ln, &qp, nq);
    if (s != IDB_OK) return s;

    const ScanChoice sc = pick_scan(nchunks, ix->row_type);
    ScanLaunch sl;
    s = scan_launch(ix, sc.fn, &sl);
    if (s != IDB_OK) return s;
    const int wpc = sl.wpc, occ = sl.occ;
    const size_t smem = sl.smem;
    const uint64_t q_per_cta = (uint64_t)wpc * sc.qw;

    // Slices: enough CTAs for about four waves of the device; K4 merges S lists of k keys per query, so S x k stays small, and a
    // slice keeps at least kScanMinSliceRows rows.  S = 1 (no merge) when the queries alone fill the device.
    const uint64_t cap_keys = ix->exact_scratch_keys ? ix->exact_scratch_keys : kExactScratchKeys;
    const uint64_t nq_eff = std::max<uint64_t>(1, std::min<uint64_t>(nq, cap_keys / k));
    const uint64_t want_ctas = 4ull * std::max(1, occ) * ix->num_sms;
    const uint64_t q_ctas = (nq_eff + q_per_cta - 1) / q_per_cta;
    uint64_t S = (want_ctas + q_ctas - 1) / q_ctas;
    S = std::min<uint64_t>(S, std::max<uint64_t>(1, kExactMaxSliceKeys / k));
    S = std::min<uint64_t>(S, (ix->n + kScanMinSliceRows - 1) / kScanMinSliceRows);
    S = std::max<uint64_t>(S, 1);
    int max_smem = 0;
    if (S > 1) {
        s = merge_fits(ix, S, k, &max_smem);
        if (s != IDB_OK) return s;
    }
    const uint64_t chunk = std::max<uint64_t>(1, cap_keys / (S * k));
    CUDA_TRY(ensure_u64(ln.exact_keys, ln.exact_keys_cap, S * std::min(nq, chunk) * k));

    ExactArgs a;
    std::memset(&a, 0, sizeof(a));
    a.g = ix->view();
    a.k = k;
    a.S = (uint32_t)S;
    a.slice_rows = (ix->n + S - 1) / S;
    a.lists = ln.exact_keys;
    a.id_map = ix->d_id_map;
    a.metric = ix->metric;
    for (uint64_t c0 = 0; c0 < nq; c0 += chunk) {
        const uint64_t m = std::min(chunk, nq - c0);
        a.queries = reinterpret_cast<const float4*>(qp + c0 * stride);
        a.nq = m;
        a.out_ids = d_ids + c0 * k;
        a.out_dist = d_dist ? d_dist + c0 * k : nullptr;
        a.out_len = d_len ? d_len + c0 : nullptr;
        const dim3 grid((unsigned)((m + q_per_cta - 1) / q_per_cta), (unsigned)S);
        sc.fn<<<grid, wpc * 32, smem, st>>>(a);
        CUDA_TRY(cudaGetLastError());
        if (S > 1) {
            s = launch_merge(ix, st, a.lists, (uint32_t)S, m, k, a.out_ids, a.out_dist, a.out_len, nullptr, max_smem);
            if (s != IDB_OK) return s;
            if (a.id_map) {  // after the merge: ties are broken by PointId, not by the mapped id
                const uint64_t cnt = m * k;
                const unsigned g = (unsigned)std::min<uint64_t>((cnt + 255) / 256, (uint64_t)ix->num_sms * 8);
                apply_id_map_kernel<<<g, 256, 0, st>>>(a.out_ids, cnt, a.id_map);
                CUDA_TRY(cudaGetLastError());
            }
        }
    }
    return IDB_OK;
}

}  // namespace idb

using namespace idb;

extern "C" {

idb_status idb_exact_search_batch_f32(idb_index* index, const float* queries, uint64_t nq, uint32_t k, uint32_t* out_ids, float* out_dist,
                                      uint32_t* out_len) {
    idb_status st = check_search_args(Family::exact, &index, 1, nullptr, nullptr, queries, nq, out_ids, k);
    if (st != IDB_OK || nq == 0) return st;
    Index* ix = reinterpret_cast<Index*>(index);
    Lane& ln = ix->pick_lane();
    std::lock_guard<std::mutex> lk(ln.mu, std::adopt_lock);
    CUDA_TRY(cudaSetDevice(ix->device));
    CUDA_TRY(ensure_u32(ln.ids, ln.ids_cap, nq * k));
    CUDA_TRY(ensure_f32(ln.dist, ln.dist_cap, nq * k));
    CUDA_TRY(ensure_u32(ln.len, ln.len_cap, nq));
    st = enqueue_exact(ix, ln, queries, true, nq, k, ln.ids, ln.dist, ln.len);
    if (st != IDB_OK) return st;
    return read_back(ln, nq, k, out_ids, out_dist, out_len, nullptr, 0);
}

idb_status idb_exact_search_batch_device_lane(idb_index* index, uint32_t lane, const float* d_queries, uint64_t nq, uint32_t k,
                                              uint32_t* d_out_ids, float* d_out_dist, uint32_t* d_out_len) {
    idb_status st = check_search_args(Family::exact, &index, 1, nullptr, &lane, d_queries, nq, d_out_ids, k);
    if (st != IDB_OK || nq == 0) return st;
    Index* ix = reinterpret_cast<Index*>(index);
    Lane& ln = ix->lanes[lane];
    std::lock_guard<std::mutex> lk(ln.mu);
    return enqueue_exact(ix, ln, d_queries, false, nq, k, d_out_ids, d_out_dist, d_out_len);
}

}  // extern "C"
