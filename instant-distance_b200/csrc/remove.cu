// remove.cu — idb_index_remove (DESIGN.md §6b): take points out of an index, repair the rows that listed them, compact the PointIds.
//
//   repair    one warp per row of a layer (persistent grid): a row that lists a removed id gathers its candidates — its own entries
//             and the entries of each removed point's row on that layer, one hop, without the point itself and without removed ids —
//             in rounds of one source row, keeps the ef_construction smallest keys (distance to the row's point, PointId) in a sorted
//             list, and rewrites the row with select_heuristic_warp (or the list's prefix in simple mode).  A repair reads only its own
//             row and removed points' rows, and removed rows are never written, so every row is repaired in place.
//   compact   new(x) = x - |{r in R : r < x}| from an exclusive scan of the keep flags; one kernel moves the stored rows (any storage),
//             the q8 headers and the id map, one relabels the zero and upper rows into the new buffers, which are then swapped in.
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cstdlib>
#include <vector>

#include "build_dispatch.cuh"

namespace idb {

namespace {

struct RepairArgs {
    GraphView g;                 // the index before the removal (rows, n, M)
    uint32_t* rows;              // the layer's rows, n_rows x width, repaired in place
    uint64_t n_rows;             // n_l
    uint32_t width;              // 2M on layer 0, M above
    const uint32_t* removed;     // bitmap of R: (n + 31) / 32 words
    uint32_t efc;                // ef_construction: keys kept per row
    uint32_t list_cap;           // keys per list buffer (efc rounded up to 32)
    uint32_t heuristic, keep_pruned;
    unsigned long long* work;    // rows handed out so far
};

// A round holds one source row (<= 2M ids) plus room for the rows batch_distances reads ahead (NB <= 16).
__host__ __device__ inline uint32_t round_cap(uint32_t M) { return 2 * M + 32; }

// Shared-memory carve-up of one repair warp.
struct RepairSmem {
    uint64_t* list[2];   // list_cap each: the row's candidate keys so far, ascending and distinct (the two merge buffers)
    uint64_t* rkey;      // round_cap: this round's keys
    uint64_t* rsort;     // round_cap: this round's keys that are new, ascending
    uint32_t* rpid;      // round_cap: this round's ids
    uint32_t* rflag;     // round_cap: 1 = the key is in the list already, or earlier in the round
    uint32_t* own;       // 2M: the row as it was
    uint32_t* out;       // 2M: the selection
    uint32_t* kept_pid;  // 2M
    uint32_t* disc;      // list_cap
    float4* vecs;        // 2M x nchunks kept rows (kStage) — or, for long rows (CH == 0), the warp's query buffer (long_q_bytes)
    __host__ __device__ static size_t bytes(uint32_t list_cap, uint32_t M, uint32_t nchunks, bool stage) {
        const size_t rc = round_cap(M);
        size_t b = 2 * (size_t)list_cap * 8 + 2 * rc * 8 + 2 * rc * 4 + 3 * (size_t)2 * M * 4 + (size_t)list_cap * 4;
        b = (b + 15) / 16 * 16;
        if (stage) b += (size_t)2 * M * nchunks * 16;
        else if (nchunks > 256) b += long_q_bytes(nchunks);
        return b;
    }
    __device__ void carve(unsigned char* base, uint32_t list_cap, uint32_t M) {
        const size_t rc = round_cap(M);
        unsigned char* p = base;
        list[0] = reinterpret_cast<uint64_t*>(p); p += (size_t)list_cap * 8;
        list[1] = reinterpret_cast<uint64_t*>(p); p += (size_t)list_cap * 8;
        rkey = reinterpret_cast<uint64_t*>(p); p += rc * 8;
        rsort = reinterpret_cast<uint64_t*>(p); p += rc * 8;
        rpid = reinterpret_cast<uint32_t*>(p); p += rc * 4;
        rflag = reinterpret_cast<uint32_t*>(p); p += rc * 4;
        own = reinterpret_cast<uint32_t*>(p); p += 2 * M * 4;
        out = reinterpret_cast<uint32_t*>(p); p += 2 * M * 4;
        kept_pid = reinterpret_cast<uint32_t*>(p); p += 2 * M * 4;
        disc = reinterpret_cast<uint32_t*>(p); p += (size_t)list_cap * 4;
        size_t off = (size_t)(p - base);
        off = (off + 15) / 16 * 16;
        vecs = reinterpret_cast<float4*>(base + off);
    }
};

__device__ __forceinline__ bool is_removed(const uint32_t* bits, uint32_t x) { return (bits[x >> 5] >> (x & 31)) & 1u; }

// Position of the first key >= k in a[0, n) (ascending).
__device__ __forceinline__ uint32_t lower_bound_u64(const uint64_t* a, uint32_t n, uint64_t k) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (a[mid] < k) lo = mid + 1; else hi = mid;
    }
    return lo;
}

template <int CH, int NB, bool kStage, class RT>
__global__ void __launch_bounds__(kBuildWarps * 32) repair_kernel(RepairArgs a, uint32_t smem_per_warp) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const uint32_t lt = (1u << lane) - 1u;
    RepairSmem sm;
    sm.carve(smem_raw + (size_t)warp * smem_per_warp, a.list_cap, a.g.M);
    const uint32_t width = a.width;
    for (;;) {
        unsigned long long w = 0;
        if (lane == 0) w = atomicAdd(a.work, 1ull);
        w = __shfl_sync(kFullMask, w, 0);
        if (w >= a.n_rows) break;
        const uint32_t p = (uint32_t)w;
        if (is_removed(a.removed, p)) continue;  // (warp-uniform) removed rows are dropped, never written
        uint32_t* row = a.rows + (size_t)p * width;
        bool hit = false;
        for (uint32_t t = lane; t < width; t += 32) {
            const uint32_t e = row[t];
            sm.own[t] = e;
            hit = hit || (e != kInvalid && is_removed(a.removed, e));
        }
        if (!__any_sync(kFullMask, hit)) continue;  // a row that lists no removed id is not touched
        __syncwarp();
        QVec<CH> q;
        if constexpr (CH == 0) { q.s = sm.vecs; q.ngroups = (a.g.nchunks + 31) / 32; }
        q_from_point<CH, RT>(q, a.g, p, lane);
        uint32_t nl = 0, cur = 0;  // keys in sm.list[cur]
        // rounds: the row itself (s = 0), then the row of each removed id it lists (s = its position + 1)
        for (uint32_t s = 0; s <= width; ++s) {
            if (s > 0) {
                const uint32_t r = sm.own[s - 1];
                if (r == kInvalid || !is_removed(a.removed, r)) continue;
            }
            const uint32_t* src = s == 0 ? sm.own : a.rows + (size_t)sm.own[s - 1] * width;
            uint32_t b = 0;  // gather: valid entries, not p, not removed
            for (uint32_t t0 = 0; t0 < width; t0 += 32) {
                const uint32_t t = t0 + lane;
                const uint32_t x = t < width ? src[t] : kInvalid;
                const bool ok = x != kInvalid && x != p && !is_removed(a.removed, x);
                const uint32_t m = __ballot_sync(kFullMask, ok);
                if (ok) sm.rpid[b + __popc(m & lt)] = x;
                b += __popc(m);
            }
            __syncwarp();
            if (b == 0) continue;
            batch_distances<CH, NB, RT>(a.g, q, sm.rpid, sm.rkey, b, lane);
            // merge: drop keys already listed (in the list or earlier in the round), order the new ones, then interleave both into
            // the other buffer by rank, keeping the efc smallest.  Keys are distinct within and between the two, so ranks are unique.
            const uint64_t* L = sm.list[cur];
            uint64_t* Lo = sm.list[cur ^ 1u];
            for (uint32_t j = lane; j < b; j += 32) {
                const uint64_t k = sm.rkey[j];
                const uint32_t at = lower_bound_u64(L, nl, k);
                bool dup = at < nl && L[at] == k;
                for (uint32_t i = 0; i < j && !dup; ++i) dup = sm.rkey[i] == k;
                sm.rflag[j] = dup ? 1u : 0u;
            }
            __syncwarp();
            uint32_t nb = 0;
            for (uint32_t j0 = 0; j0 < b; j0 += 32) {
                const uint32_t j = j0 + lane;
                const bool fresh = j < b && !sm.rflag[j];
                if (fresh) {
                    const uint64_t k = sm.rkey[j];
                    uint32_t r = 0;
                    for (uint32_t i = 0; i < b; ++i) r += (!sm.rflag[i] && sm.rkey[i] < k) ? 1u : 0u;
                    sm.rsort[r] = k;
                }
                nb += __popc(__ballot_sync(kFullMask, fresh));
            }
            __syncwarp();
            for (uint32_t i = lane; i < nl; i += 32) {
                const uint32_t r = i + lower_bound_u64(sm.rsort, nb, L[i]);
                if (r < a.efc) Lo[r] = L[i];
            }
            for (uint32_t j = lane; j < nb; j += 32) {
                const uint32_t r = j + lower_bound_u64(L, nl, sm.rsort[j]);
                if (r < a.efc) Lo[r] = sm.rsort[j];
            }
            nl = min(a.efc, nl + nb);
            cur ^= 1u;
            __syncwarp();
        }
        // selection (select_heuristic, or the first 2M keys in simple mode), cut to the layer's width
        uint32_t total;
        if (a.heuristic) {
            total = select_heuristic_warp<CH, NB, kStage, RT>(a.g, sm.list[cur], nl, sm.out, sm.disc, sm.vecs, sm.kept_pid,
                                                              a.keep_pruned != 0, lane, q, sm.rkey);
        } else {
            total = min(nl, 2 * a.g.M);
            for (uint32_t t = lane; t < total; t += 32) sm.out[t] = key_pid(sm.list[cur][t]);
            __syncwarp();
        }
        total = min(total, width);
        for (uint32_t t = lane; t < width; t += 32) row[t] = t < total ? sm.out[t] : kInvalid;
        __syncwarp();
    }
}

template <int CH, int NB, bool kStage, class RT>
cudaError_t launch_repair(const RepairArgs& a, int grid, uint32_t smem_per_warp, cudaStream_t st) {
    auto kern = repair_kernel<CH, NB, kStage, RT>;
    const int smem = (int)smem_per_warp * kBuildWarps;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    kern<<<grid, kBuildWarps * 32, smem, st>>>(a, smem_per_warp);
    return cudaGetLastError();
}

cudaError_t repair_dispatch(const RepairArgs& a, bool stage, int grid, uint32_t smem_per_warp, cudaStream_t st) {
    return with_cell(a.g.nchunks, [&](auto cell) {
        constexpr int CH = decltype(cell)::CH, NB = decltype(cell)::B;
        return with_row_type(a.g.row_type, [&](auto rt) {
            using RT = decltype(rt);
            if constexpr (CH > 0) {
                if (stage) return launch_repair<CH, NB, true, RT>(a, grid, smem_per_warp, st);
            }
            return launch_repair<CH, NB, false, RT>(a, grid, smem_per_warp, st);
        });
    });
}

__global__ void keep_flags_kernel(const uint32_t* removed, uint64_t n, uint32_t* keep) {
    for (uint64_t x = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; x < n; x += (uint64_t)gridDim.x * blockDim.x)
        keep[x] = is_removed(removed, (uint32_t)x) ? 0u : 1u;
}
// new_ids: the exclusive scan of the keep flags; a removed id maps to INVALID
__global__ void drop_removed_kernel(const uint32_t* removed, uint64_t n, uint32_t* new_ids) {
    for (uint64_t x = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; x < n; x += (uint64_t)gridDim.x * blockDim.x)
        if (is_removed(removed, (uint32_t)x)) new_ids[x] = kInvalid;
}

// Row x of the store (wpr words W: the raw stored row, any storage), its q8 header and its id-map entry -> position new_ids[x].
template <class W>
__device__ __forceinline__ void compact_rows(const uint32_t* new_ids, uint64_t n, uint32_t wpr, const W* rows, W* rows_out,
                                             const float2* hdr, float2* hdr_out, const uint32_t* id_map, uint32_t* id_map_out) {
    const uint64_t total = n * wpr;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t x = i / wpr;
        const uint32_t c = (uint32_t)(i - x * wpr);
        const uint32_t y = new_ids[x];
        if (y == kInvalid) continue;
        rows_out[(uint64_t)y * wpr + c] = rows[i];
        if (c == 0) {
            if (hdr) hdr_out[y] = hdr[x];
            if (id_map) id_map_out[y] = id_map[x];
        }
    }
}
// Rows that are a whole number of u32 words move as words; bin rows (nchunks bytes, DESIGN §3d) in general are not, and move as bytes.
__global__ void compact_rows_kernel(const uint32_t* new_ids, uint64_t n, uint32_t wpr, const uint32_t* rows, uint32_t* rows_out,
                                    const float2* hdr, float2* hdr_out, const uint32_t* id_map, uint32_t* id_map_out) {
    compact_rows(new_ids, n, wpr, rows, rows_out, hdr, hdr_out, id_map, id_map_out);
}
__global__ void compact_rows_kernel(const uint32_t* new_ids, uint64_t n, uint32_t bpr, const uint8_t* rows, uint8_t* rows_out,
                                    const float2* hdr, float2* hdr_out, const uint32_t* id_map, uint32_t* id_map_out) {
    compact_rows(new_ids, n, bpr, rows, rows_out, hdr, hdr_out, id_map, id_map_out);
}

// Adjacency rows [0, n_rows) of `width` entries -> position new_ids[x], every entry relabelled (INVALID stays INVALID).
__global__ void relabel_rows_kernel(const uint32_t* new_ids, uint64_t n_rows, uint32_t width, const uint32_t* src, uint32_t* dst) {
    const uint64_t total = n_rows * width;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t x = i / width;
        const uint32_t y = new_ids[x];
        if (y == kInvalid) continue;
        const uint32_t e = src[i];
        dst[(uint64_t)y * width + (i - x * width)] = e == kInvalid ? kInvalid : new_ids[e];
    }
}

// The device buffers of one removal other than its compacted graph (a Graph of its own), allocated before anything is written; what
// is not handed to the index is freed.
struct RemoveBuffers {
    uint32_t* removed = nullptr;
    uint32_t* keep = nullptr;
    uint32_t* new_ids = nullptr;
    unsigned long long* work = nullptr;
    void* cub_tmp = nullptr;
    void* rows = nullptr;
    float2* hdr = nullptr;
    uint32_t* id_map = nullptr;
    ~RemoveBuffers() {
        cudaFree(removed); cudaFree(keep); cudaFree(new_ids); cudaFree(work); cudaFree(cub_tmp);
        cudaFree(rows); cudaFree(hdr); cudaFree(id_map);
    }
};

// The removal of the (checked, distinct) PointIds pids[0, m) from ix, which the caller holds exclusively.
idb_status remove_index(Index* ix, const uint32_t* pids, uint64_t m, const idb_params& p, uint32_t* out_new_ids) {
    const uint64_t n = ix->n;
    if (m == 0) {
        if (out_new_ids)
            for (uint64_t x = 0; x < n; ++x) out_new_ids[x] = (uint32_t)x;
        return IDB_OK;
    }
    cudaStream_t st = ix->stream;
    const uint32_t M = ix->M, n_layers = (uint32_t)ix->graph.upper.size() + 1;
    const uint64_t n1 = n - m, cap1 = std::max<uint64_t>(n1, 1);
    // ---- host: the bitmap of R and the surviving layer sizes (per removed id, never per row) ---------------------------------------
    const uint64_t words = (n + 31) / 32;
    std::vector<uint32_t> bits(words, 0u);
    for (uint64_t i = 0; i < m; ++i) bits[pids[i] >> 5] |= 1u << (pids[i] & 31);
    std::vector<uint64_t> upper_n1(n_layers - 1);
    for (uint32_t l = 1; l < n_layers; ++l) {
        uint64_t below = 0;
        for (uint64_t i = 0; i < m; ++i) below += pids[i] < ix->graph.upper_n[l - 1] ? 1u : 0u;
        upper_n1[l - 1] = ix->graph.upper_n[l - 1] - below;
    }
    uint32_t layers1 = 1;  // layers left: the upper layers that keep a point
    while (layers1 < n_layers && upper_n1[layers1 - 1] > 0) ++layers1;
    upper_n1.resize(layers1 - 1);

    // ---- every buffer first: a failed allocation leaves the index as it was ----------------------------------------------------------
    RemoveBuffers b;
    const uint32_t efc = p.ef_construction, list_cap = (efc + 31) / 32 * 32;
    size_t cub_bytes = 0;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, b.keep, b.new_ids, (int64_t)n, st));
    CUDA_TRY(cudaMalloc(&b.cub_tmp, std::max<size_t>(cub_bytes, 16)));
    CUDA_TRY(cudaMalloc(&b.removed, words * 4));
    CUDA_TRY(cudaMalloc(&b.keep, n * 4));
    CUDA_TRY(cudaMalloc(&b.new_ids, n * 4));
    CUDA_TRY(cudaMalloc(&b.work, n_layers * sizeof(unsigned long long)));
    CUDA_TRY(ix->alloc_rows(cap1, &b.rows, &b.hdr));
    Graph next;  // the compacted graph; once swapped in, it frees the old layers, the dropped ones included
    CUDA_TRY(next.alloc(cap1, M, std::move(upper_n1), st));
    next.rows_distinct = ix->graph.rows_distinct;  // repaired rows come from distinct keys, and the relabelling is injective
    if (ix->d_id_map) CUDA_TRY(cudaMalloc(&b.id_map, cap1 * 4));

    // ---- repair every layer in place ------------------------------------------------------------------------------------------------
    CUDA_TRY(cudaMemcpyAsync(b.removed, bits.data(), words * 4, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemsetAsync(b.work, 0, n_layers * sizeof(unsigned long long), st));
    bool stage = false;  // the build's choice (BatchRunner::init): kept rows staged in shared memory only when asked for
    if (const char* e = std::getenv("IDB_BUILD_STAGE")) stage = std::atoi(e) != 0 && RepairSmem::bytes(list_cap, M, ix->nchunks, true) <= 56 * 1024;
    stage = stage && kernel_ch(ix->nchunks) > 0;
    const uint32_t smem = (uint32_t)RepairSmem::bytes(list_cap, M, ix->nchunks, stage);
    const int ctas_per_sm = (int)std::min<uint64_t>(16, std::max<uint64_t>(1, (200 * 1024) / std::max<uint32_t>(1, smem * kBuildWarps)));
    RepairArgs a;
    a.g = ix->view();
    a.removed = b.removed;
    a.efc = efc;
    a.list_cap = list_cap;
    a.heuristic = p.heuristic ? 1u : 0u;
    a.keep_pruned = p.keep_pruned ? 1u : 0u;
    for (uint32_t l = 0; l < n_layers; ++l) {
        a.rows = l == 0 ? ix->graph.zero : ix->graph.upper[l - 1];
        a.n_rows = l == 0 ? n : ix->graph.upper_n[l - 1];
        a.width = l == 0 ? 2 * M : M;
        a.work = b.work + l;
        const int grid = (int)std::max<uint64_t>(1, std::min<uint64_t>((a.n_rows + kBuildWarps - 1) / kBuildWarps, (uint64_t)ix->num_sms * ctas_per_sm));
        CUDA_TRY(repair_dispatch(a, stage, grid, smem, st));
    }

    // ---- compact ----------------------------------------------------------------------------------------------------------------------
    const int blocks = ix->num_sms * 8;
    keep_flags_kernel<<<blocks, 256, 0, st>>>(b.removed, n, b.keep);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(b.cub_tmp, cub_bytes, b.keep, b.new_ids, (int64_t)n, st));
    drop_removed_kernel<<<blocks, 256, 0, st>>>(b.removed, n, b.new_ids);
    CUDA_TRY(cudaGetLastError());
    if (n1 == 0) CUDA_TRY(fill_u32(next.zero, 2 * (size_t)M, kInvalid, st));  // the one row of an empty store
    if (ix->row_bytes() % 4 == 0)
        compact_rows_kernel<<<blocks, 256, 0, st>>>(b.new_ids, n, (uint32_t)(ix->row_bytes() / 4), static_cast<const uint32_t*>(ix->d_rows),
                                                    static_cast<uint32_t*>(b.rows), ix->d_hdr, b.hdr, ix->d_id_map, b.id_map);
    else
        compact_rows_kernel<<<blocks, 256, 0, st>>>(b.new_ids, n, (uint32_t)ix->row_bytes(), static_cast<const uint8_t*>(ix->d_rows),
                                                    static_cast<uint8_t*>(b.rows), ix->d_hdr, b.hdr, ix->d_id_map, b.id_map);
    CUDA_TRY(cudaGetLastError());
    relabel_rows_kernel<<<blocks, 256, 0, st>>>(b.new_ids, n, 2 * M, ix->graph.zero, next.zero);
    CUDA_TRY(cudaGetLastError());
    for (uint32_t l = 1; l < layers1; ++l) {
        relabel_rows_kernel<<<blocks, 256, 0, st>>>(b.new_ids, ix->graph.upper_n[l - 1], M, ix->graph.upper[l - 1], next.upper[l - 1]);
        CUDA_TRY(cudaGetLastError());
    }
    if (out_new_ids) CUDA_TRY(cudaMemcpyAsync(out_new_ids, b.new_ids, n * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));

    // ---- swap in ------------------------------------------------------------------------------------------------------------------------
    std::swap(ix->d_rows, b.rows);
    std::swap(ix->d_hdr, b.hdr);
    std::swap(ix->d_id_map, b.id_map);
    std::swap(ix->graph, next);
    ix->cap = cap1;
    ix->n = n1;
    return ix->build_codes();  // from the stored rows that remain
}

}  // namespace

}  // namespace idb

using namespace idb;

extern "C" idb_status idb_index_remove(idb_index* index, const uint32_t* pids, uint64_t m, const idb_params* params,
                                       uint32_t* out_new_ids) {
    // checks that need neither the handle nor a device first, as the insert does
    if (!index) return fail(IDB_ERR_INVALID_ARG, "index is null");
    if (!params) return fail(IDB_ERR_INVALID_ARG, "params is null");
    if (m && !pids) return fail(IDB_ERR_INVALID_ARG, "pids is null");
    idb_status st = check_link_params(params);
    if (st == IDB_OK) st = require_device();
    if (st != IDB_OK) return st;
    Index* ix = reinterpret_cast<Index*>(index);
    ExclusiveIndex ex(ix);  // &mut self, as the insert: each search on another thread sees the index before or after
    if (params->M != ix->M) return fail(IDB_ERR_INVALID_ARG, "M = %u differs from the index's %u", params->M, ix->M);
    const uint64_t n = ix->n;
    std::vector<uint32_t> seen((n + 31) / 32, 0u);
    for (uint64_t i = 0; i < m; ++i) {
        const uint32_t x = pids[i];
        if (x >= n)
            return fail(IDB_ERR_INVALID_ARG, "pids[%llu] = %u is not a PointId of this index (n = %llu)", (unsigned long long)i, x,
                        (unsigned long long)n);
        if ((seen[x >> 5] >> (x & 31)) & 1u) {
            uint64_t first = 0;
            while (pids[first] != x) ++first;
            return fail(IDB_ERR_INVALID_ARG, "pids[%llu] = %u repeats pids[%llu]", (unsigned long long)i, x, (unsigned long long)first);
        }
        seen[x >> 5] |= 1u << (x & 31);
    }
    CUDA_TRY(ex.drained);
    return remove_index(ix, pids, m, *params, out_new_ids);
}
