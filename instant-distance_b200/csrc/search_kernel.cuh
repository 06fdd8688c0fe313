// search_kernel.cuh — the traversal driver K1 and the build's KA share, K1: batched Hnsw::search kernel (lib.rs:352-383 per query),
// and the traversal kernels' launch helpers.
// Instantiated once per CH (float4 chunks per lane) and row family in search_cells.cu so the translation units build in parallel.
#pragma once
#include <cstring>
#include <type_traits>

#include "internal.cuh"

namespace idb {

// ---------------------------------------------------------------------------------------------------------
// K1: batched Hnsw::search — persistent grid, one warp per live query, queries claimed from an atomic counter.
// ---------------------------------------------------------------------------------------------------------
// FULL: dim is a multiple of 128, i.e. every lane owns a real chunk in each of its CH slots: no chunk predicates, and
// full batches of row loads carry no predicates at all (hnsw_device.cuh batch_distances_impl).
// Shared-memory carve-up of one traversal warp (K1 and the build's KA).
template <int EF_T>
struct WarpSmem {
    static constexpr int kNearBytes = 2 * 32 * EF_T * 8;
    static constexpr int kBytes = kNearBytes + kSmallVisSlots * 4 + 128 * 4 + 128 * 8;
    static __device__ __forceinline__ void carve(WarpState& s, unsigned char* base) {
        s.near_base = reinterpret_cast<uint64_t*>(base);
        s.near_len = 32 * EF_T;
        s.vis.small = reinterpret_cast<uint32_t*>(base + kNearBytes);
        s.cpid = s.vis.small + kSmallVisSlots;
        s.ckey = reinterpret_cast<uint64_t*>(s.cpid + 128);
        s.vis.hist = s.vis.small;  // the b16 tally borrows the small tier's 2 KB while the big tier is live (hnsw_device.cuh)
    }
};
// Long rows (CH == 0): the warps' query buffers follow the per-warp traversal state in dynamic shared memory.
__host__ __device__ inline uint32_t long_q_bytes(uint32_t nchunks) { return (nchunks + 31) / 32 * 32 * 16; }
template <int EF_T, int CH>
__device__ __forceinline__ void long_q_bind(QVec<CH>& q, unsigned char* smem_raw, uint32_t nchunks, int warp, int warps_per_cta) {
    if constexpr (CH == 0) {
        q.ngroups = (nchunks + 31) / 32;
        q.s = reinterpret_cast<float4*>(smem_raw + (size_t)warps_per_cta * WarpSmem<EF_T>::kBytes + (size_t)warp * long_q_bytes(nchunks));
    }
}
// Point the warp at its claimed scratch tables.
// b16 flavour: gslots = words of the first segment in use (8 * nb_lo + stash), b16_nb = buckets over both segments.
__device__ __forceinline__ void bind_tables(WarpState& s, const VisTier& t, uint32_t table) {
    const TablePool& tp = t.pool;
    s.vis.big = tp.vis_tables + (size_t)table * tp.vis_stride;
    s.vis.gslots = t.gslots;
    s.vis.gshift = t.gshift;
    s.vis.mode = t.mode;
    s.vis.nb_lo = t.mode == kVisB16 ? (t.gslots - kB16Stash) >> 3 : 1u;
    s.vis.nb = t.mode == kVisB16 ? t.b16_nb : 1u;
    s.vis.big_hi = t.mode == kVisB16 && tp.vis_ext ? tp.vis_ext + (size_t)table * tp.ext_stride - (size_t)s.vis.nb_lo * 8 : s.vis.big;
    s.vis.nb_inv = 1.0f / (float)s.vis.nb;
    s.vis.cap_ids = t.b16_cap_ids;
    s.vis.stash_cnt = 0;
    s.vis.count = 0;
    s.vis.use_big = false;
    s.ties = tp.tie_tables + (size_t)table * tp.tie_cap;
    s.tie_cap = tp.tie_cap;
}

// The body of both traversal kernels, K1 (a query per warp) and KA (an insert per warp).  The CTA claims its warps' scratch tables;
// each warp then claims work items until none is left: load(item, q) fills the query, `descend` runs it down to `target_layer`, and
// epi(item, nearest, len, s) writes the result (len = 0 when the traversal overflowed).  The item's status is recorded and an
// overflowed item is listed for the retry pass; the warp leaves its tables clean for the next item and the next holder.
// Item: the type of an item's index — u64 for K1's query batches, u32 for the inserts of a build batch.
template <int CH, int ROW_T, int EF_T, int B, class RT, bool FULL, bool TMA, bool SCREEN, class Item, class Load, class Epi>
__device__ __forceinline__ void traverse(const GraphView& g, const TraversalWork& w, const VisTier& tier, uint32_t target_layer,
                                         uint32_t ef, uint32_t* counters, Load load, Epi epi) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ uint32_t s_claim[2];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const Item n_work = w.n_work_dev ? (Item)*w.n_work_dev : (Item)w.n_work;
    if (n_work == 0) return;  // the retry pass, normally: nothing to do, no tables claimed

    WarpState s;
    WarpSmem<EF_T>::carve(s, smem_raw + (size_t)warp * WarpSmem<EF_T>::kBytes);
    const uint32_t table0 = cta_tables_acquire(tier.pool, s_claim, kSearchWarps);
    bind_tables(s, tier, table0 + warp);
    vis_clear_small(s.vis, lane);  // the big tables are handed over clean by their previous holder
    if constexpr (TMA) {  // EXPERIMENT: per-warp ring of B rows + its mbarrier behind the traversal state
        unsigned char* rb = smem_raw + (size_t)kSearchWarps * WarpSmem<EF_T>::kBytes;
        s.mbar = reinterpret_cast<uint64_t*>(rb) + warp;
        s.ring = reinterpret_cast<char*>(rb + 64 + (size_t)warp * B * g.nchunks * 16);
        s.mbar_phase = 0;
        if (lane == 0) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(s.mbar)) : "memory");
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        }
        __syncwarp();
    }

    for (;;) {
        unsigned long long wi = 0;
        if (lane == 0) wi = atomicAdd(w.work_counter, 1ull);
        wi = __shfl_sync(kFullMask, wi, 0);
        if (wi >= n_work) break;
        const Item item = w.work_list ? (Item)w.work_list[wi] : (Item)wi;

        QVec<CH> q;
        long_q_bind<EF_T>(q, smem_raw, g.nchunks, warp, kSearchWarps);
        load(item, q, lane);
        descend<CH, ROW_T, EF_T, B, false, RT, FULL, TMA, SCREEN>(g, s, q, target_layer, ef, lane, counters ? counters + item * 4 : nullptr);

        const uint32_t len = s.status == kQueryOk ? s.cnt : 0u;
        epi(item, s.near_base + s.cur * s.near_len, len, s, lane);
        if (lane == 0) {
            w.status[item] = s.status;
            if (s.status != kQueryOk) {
                const uint32_t slot = atomicAdd(w.fail_count, 1u);
                if (w.fail_list) w.fail_list[slot] = (uint32_t)item;
            }
        }
        finish_query(s, lane);
    }
    cta_tables_release(tier.pool, s_claim);
}

template <int CH, int ROW_T, int EF_T, int B, int OCC, class RT = RowF32, bool FULL = false, bool TMA = false>
__global__ void __launch_bounds__(kSearchWarps * 32, OCC) search_kernel(SearchArgs a) {
    traverse<CH, ROW_T, EF_T, B, RT, FULL, TMA, /*SCREEN=*/!TMA, uint64_t>(
        a.g, a.work, a.tier, 0u, a.ef, a.counters,
        [&](uint64_t qi, QVec<CH>& q, int lane) { q_from_f32<CH>(q, a.queries + qi * a.g.nchunks, a.g.nchunks, lane); },
        [&](uint64_t qi, const uint64_t* near, uint32_t len, const WarpState& s, int lane) {
            for (uint32_t j = lane; j < a.k; j += 32) {
                uint64_t key = j < len ? near[j] : 0ull;
                const uint32_t gid = j < len ? (a.id_map ? a.id_map[key_pid(key)] : key_pid(key)) : kInvalid;
                a.out_ids[qi * a.k + j] = gid;
                if (a.out_keys) a.out_keys[qi * a.k + j] = j < len ? (((uint64_t)key_dbits(key) << 32) | gid) : kKeyNone;
                if (a.out_dist) a.out_dist[qi * a.k + j] = j < len ? reported_distance(key_dbits(key), a.metric) : __int_as_float(0x7f800000);
            }
            if (lane == 0) {
                if (a.full_tally) atomicAdd(a.full_tally, (unsigned long long)s.n_full);
                if (a.out_len) a.out_len[qi] = len;
            }
        });
}

// Launch a traversal kernel (K1 or KA): kSearchWarps warps per CTA, the dynamic shared memory its warps carve up plus `extra` bytes,
// and (optionally) a persisting-L2 access-policy window on the b16 visited tables as a LAUNCH attribute: no stream state.
template <int CH, int EF_T, class Kern, class Args>
static cudaError_t launch_traversal(Kern kern, const Args& a, int extra, int grid, cudaStream_t stream, const LaunchWindow& win) {
    const int smem = (WarpSmem<EF_T>::kBytes + (CH == 0 ? (int)long_q_bytes(a.g.nchunks) : 0)) * kSearchWarps + extra;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3((unsigned)(kSearchWarps * 32));
    cfg.dynamicSmemBytes = (size_t)smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    if (win.base && win.bytes) {
        attr[0].id = cudaLaunchAttributeAccessPolicyWindow;
        attr[0].val.accessPolicyWindow.base_ptr = win.base;
        attr[0].val.accessPolicyWindow.num_bytes = win.bytes;
        attr[0].val.accessPolicyWindow.hitRatio = win.hit_ratio;
        attr[0].val.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
        attr[0].val.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
    }
    return cudaLaunchKernelEx(&cfg, kern, a);
}

// The (ROW_T, EF_T) tiles the traversal kernels are compiled for: f(ROW_T, EF_T) with both as std::integral_constant.
template <class F>
cudaError_t with_tile(int row_t, int ef_t, F&& f) {
    using R2 = std::integral_constant<int, 2>;
    using R4 = std::integral_constant<int, 4>;
    if (row_t <= 2) {
        if (ef_t <= 4) return f(R2(), std::integral_constant<int, 4>());
        if (ef_t <= 8) return f(R2(), std::integral_constant<int, 8>());
        if (ef_t <= 16) return f(R2(), std::integral_constant<int, 16>());
        return f(R2(), std::integral_constant<int, 32>());
    }
    if (ef_t <= 4) return f(R4(), std::integral_constant<int, 4>());
    if (ef_t <= 16) return f(R4(), std::integral_constant<int, 16>());
    return f(R4(), std::integral_constant<int, 32>());
}

// variant: the IDB_VARIANT case that chose this instantiation (0 = the default dispatch); recorded with the template arguments.
template <int CH, int ROW_T, int EF_T, int B, int OCC = kSearchCtasPerSm, class RT = RowF32, bool FULL = false, bool TMA = false>
static cudaError_t launch_search(const SearchArgs& a, int grid, cudaStream_t stream, const LaunchWindow& win, int variant = 0) {
    const int ring = TMA ? 64 + kSearchWarps * B * (int)a.g.nchunks * 16 : 0;
    cudaError_t e = launch_traversal<CH, EF_T>(search_kernel<CH, ROW_T, EF_T, B, OCC, RT, FULL, TMA>, a, ring, grid, stream, win);
    if (e == cudaSuccess && a.launched) {
        const uint32_t cell[8] = {CH, ROW_T, EF_T, B, RT::kType, FULL ? 1u : 0u, TMA ? 1u : 0u,
                                  (uint32_t)variant};
        std::memcpy(a.launched, cell, sizeof(cell));
    }
    return e;
}

template <int CH, int B, class RT>
cudaError_t dispatch_row_ef_rt(const SearchArgs& a, int row_t, int ef_t, int grid, cudaStream_t st, const LaunchWindow& win) {
    return with_tile(row_t, ef_t, [&](auto row, auto ef) {
        constexpr int ROW_T = decltype(row)::value, EF_T = decltype(ef)::value;
        if constexpr (CH > 0) {
            if (a.g.nchunks == 32u * CH) return launch_search<CH, ROW_T, EF_T, B, kSearchCtasPerSm, RT, true>(a, grid, st, win);
        }
        return launch_search<CH, ROW_T, EF_T, B, kSearchCtasPerSm, RT, false>(a, grid, st, win);
    });
}
// Rows in flight per lane for row type RT, given B for f32 rows: bf16 / fp16 / q8 / bin rows stay packed while in flight (a half or a
// quarter of the registers per row), so twice the rows, up to 16 (q8 takes the 2-byte rule: it also carries a header per row; bin
// takes it too, one register per chunk as q8).
template <int B, class RT>
constexpr int rows_in_flight() { return RT::kChunkBytes <= 8 && 2 * B <= 16 ? 2 * B : B; }
// K1's cells of Cell<CH> for bin rows (BIN) or for f32, bf16, fp16 and q8 rows: defined in search_cells.cu, which is compiled once
// per (CH, BIN) so that the cells build in parallel (DESIGN §3d).
template <int CH, bool BIN>
cudaError_t search_cells(const SearchArgs& a, int row_t, int ef_t, int grid, cudaStream_t st, const LaunchWindow& win);

}  // namespace idb
