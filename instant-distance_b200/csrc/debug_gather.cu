// debug_gather.cu — measurement-only: how fast can this GPU gather random point rows in K1's access pattern?
//
// One warp per work item, K1's launch shape (kSearchWarps warps per CTA, kSearchCtasPerSm CTAs per SM, persistent, items
// claimed from an atomic counter).  Each item performs `batches` batches of NB row loads (NB rows in flight per lane, the
// canonical lane_partial + batch_butterfly on them, exactly K1's batch_distances arithmetic) at pseudo-random PointIds.
// `chain` batches are independent of each other, then the next group's ids depend on the previous group's result — that is
// the dependency K1 has between expansions (chain = 3 at the headline config; chain = 0 means fully independent: the pure
// gather ceiling).  No visited set, no adjacency rows, no merge: the gap between this and K1 is what those cost.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "internal.cuh"

namespace idb {

// MIX (idb_debug_gather_mix_bench): K1's OTHER memory stream rides along — per batch `atomics` lanes do one atomicAnd on a random
// word of a per-warp 125 KB bitmap (K1: 64 visited test-and-sets per ~3 batches), and the bitmap is wiped after every item
// (K1: once per query).  mode 1: the atomics overlap the batch's row loads (pure traffic-mix ceiling); mode 2: the row loads
// are issued only after the atomics have returned (K1's dependency: a row is fetched only if it was not visited).
// modes 3 / 4 / 5 replace the returning atomic by  plain load + RED  /  plain load + plain store  /  plain load only.
template <int NB, int MIX>
__global__ void __launch_bounds__(kSearchWarps * 32, kSearchCtasPerSm)
gather_bench_kernel(GraphView g, uint32_t n_items, uint32_t batches, uint32_t chain, unsigned long long* counter, float* sink,
                    uint32_t* bitmaps, uint32_t bm_words, uint32_t atomics) {
    const int lane = threadIdx.x & 31;
    uint32_t* bm = MIX ? bitmaps + (size_t)(blockIdx.x * kSearchWarps + (threadIdx.x >> 5)) * bm_words : nullptr;
    const uint32_t row_bytes = g.nchunks * 16u;
    const char* lane_base = g.points + lane * 16;
    const bool cok = (uint32_t)lane < g.nchunks;
    float acc = 0.f;
    for (;;) {
        unsigned long long w = 0;
        if (lane == 0) w = atomicAdd(counter, 1ull);
        w = __shfl_sync(kFullMask, w, 0);
        if (w >= n_items) break;
        float4 q[1];
        q[0] = cok ? __ldg(reinterpret_cast<const float4*>(lane_base + (size_t)((uint32_t)w % (uint32_t)g.n) * row_bytes)) : make_float4(0, 0, 0, 0);
        uint32_t state = (uint32_t)w * 0x9E3779B1u + 12345u;
        for (uint32_t b = 0; b < batches; ++b) {
            uint32_t old = 0;
            if (MIX && (uint32_t)lane < atomics) {
                uint32_t h = (state ^ 0x5bd1e995u) + (b * 32 + lane) * 0x27D4EB2Fu;
                h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12;
                uint32_t* wp = bm + h % bm_words;
                const uint32_t bit = 1u << (h >> 27);
                if (MIX <= 2) old = atomicAnd(wp, ~bit);                       // ATOM with return value
                else if (MIX == 3) { old = __ldcg(wp); atomicAnd(wp, ~bit); }  // plain load + RED (no return value)
                else if (MIX == 4) { old = __ldcg(wp); __stcg(wp, old & ~bit); }  // plain load + plain store (warp-private table)
                else old = __ldcg(wp);                                         // MIX 5: load only
            }
            uint32_t dep = 0;  // MIX 2 = K1's order: which rows to fetch is known only once the test-and-sets are back
            if (MIX == 2) dep = __any_sync(kFullMask, old == 0x12345u) ? 1u : 0u;  // (never true; a real data dependency)
            float4 v[NB][1];
#pragma unroll
            for (int i = 0; i < NB; ++i) {
                uint32_t h = (state + dep + (b * NB + i) * 0x85EBCA6Bu);
                h ^= h >> 15; h *= 0xC2B2AE35u; h ^= h >> 13;
                const uint32_t pid = h % (uint32_t)g.n;
                v[i][0] = cok ? __ldg(reinterpret_cast<const float4*>(lane_base + (size_t)pid * row_bytes)) : make_float4(0, 0, 0, 0);
            }
            float p[NB];
#pragma unroll
            for (int i = 0; i < NB; ++i) p[i] = lane_partial<1>(q, v[i]);
            const float total = batch_butterfly<NB>(p, lane);
            acc += total;
            if (MIX != 2 && MIX != 0 && old == 0x12345u) acc += 1.f;
            if (chain && (b + 1) % chain == 0) state = state * 1664525u + __float_as_uint(__shfl_sync(kFullMask, total, 0));  // dependency
        }
        if (MIX) {  // Visited::clear once per item, as finish_query does
            uint4* p4 = reinterpret_cast<uint4*>(bm);
            const uint4 e = make_uint4(kInvalid, kInvalid, kInvalid, kInvalid);
            for (uint32_t i = lane; i < bm_words / 4; i += 32) __stcg(p4 + i, e);
            __threadfence();
            __syncwarp();
        }
    }
    if (acc == 123456.789f) sink[0] = acc;  // keep the work alive
}

}  // namespace idb

using namespace idb;

static idb_status gather_bench_impl(idb_index* index, uint32_t n_items, uint32_t batches, uint32_t chain, uint32_t reps,
                                    uint32_t atomics, uint32_t mode, float* out_ms, double* out_bytes) {
    if (!index || !out_ms) return fail(IDB_ERR_INVALID_ARG, "null argument");
    if (mode > 5 || atomics > 32) return fail(IDB_ERR_INVALID_ARG, "gather bench: mode 0..5, atomics <= 32");
    Index* ix = reinterpret_cast<Index*>(index);
    if (ix->row_type != kRowF32 || ix->nchunks > 32 || ix->n == 0) return fail(IDB_ERR_UNSUPPORTED, "gather bench: f32 rows of <= 128 floats only");
    std::lock_guard<std::mutex> lk(ix->mu);
    CUDA_TRY(cudaSetDevice(ix->device));
    unsigned long long* d_counter = nullptr;
    float* d_sink = nullptr;
    CUDA_TRY(cudaMalloc(&d_counter, 8));
    CUDA_TRY(cudaMalloc(&d_sink, 4));
    uint32_t* d_bm = nullptr;
    uint32_t bm_words = (uint32_t)(((ix->n + 31) / 32 + 127) / 128 * 128);
    if (const char* e = std::getenv("IDB_DEBUG_BM_WORDS")) bm_words = (uint32_t)std::max(128, std::atoi(e)) / 128 * 128;  // table-size study
    if (mode) {
        const size_t words = (size_t)ix->search_grid() * kSearchWarps * bm_words;
        CUDA_TRY(cudaMalloc(&d_bm, words * 4));
        CUDA_TRY(fill_u32(d_bm, words, kInvalid, ix->stream));
        if (const char* e = std::getenv("IDB_DEBUG_BM_PERSIST")) {  // keep the tables in L2 with a persisting access-policy window
            if (std::atoi(e)) {
                int max_persist = 0, max_window = 0;
                cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, ix->device);
                cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, ix->device);
                const size_t bytes = words * 4, carve = std::min<size_t>(bytes, (size_t)max_persist);
                std::fprintf(stderr, "[gather bench] tables %zu MB, max persisting L2 %d MB, max window %d MB\n", bytes >> 20, max_persist >> 20, max_window >> 20);
                CUDA_TRY(cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, carve));
                cudaStreamAttrValue av;
                std::memset(&av, 0, sizeof(av));
                av.accessPolicyWindow.base_ptr = d_bm;
                av.accessPolicyWindow.num_bytes = std::min<size_t>(bytes, (size_t)max_window);
                av.accessPolicyWindow.hitRatio = (float)std::min(1.0, (double)carve / (double)av.accessPolicyWindow.num_bytes);
                av.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
                av.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
                CUDA_TRY(cudaStreamSetAttribute(ix->stream, cudaStreamAttributeAccessPolicyWindow, &av));
            }
        }
    }
    cudaEvent_t e0, e1;
    CUDA_TRY(cudaEventCreate(&e0));
    CUDA_TRY(cudaEventCreate(&e1));
    float best = 1e30f;
    for (uint32_t r = 0; r < reps + 1; ++r) {
        CUDA_TRY(cudaMemsetAsync(d_counter, 0, 8, ix->stream));
        CUDA_TRY(cudaEventRecord(e0, ix->stream));
        const int grid = ix->search_grid();
        if (mode == 0) gather_bench_kernel<16, 0><<<grid, kSearchWarps * 32, 0, ix->stream>>>(ix->view(), n_items, batches, chain, d_counter, d_sink, nullptr, 0, 0);
        else if (mode == 1) gather_bench_kernel<16, 1><<<grid, kSearchWarps * 32, 0, ix->stream>>>(ix->view(), n_items, batches, chain, d_counter, d_sink, d_bm, bm_words, atomics);
        else if (mode == 2) gather_bench_kernel<16, 2><<<grid, kSearchWarps * 32, 0, ix->stream>>>(ix->view(), n_items, batches, chain, d_counter, d_sink, d_bm, bm_words, atomics);
        else if (mode == 3) gather_bench_kernel<16, 3><<<grid, kSearchWarps * 32, 0, ix->stream>>>(ix->view(), n_items, batches, chain, d_counter, d_sink, d_bm, bm_words, atomics);
        else if (mode == 4) gather_bench_kernel<16, 4><<<grid, kSearchWarps * 32, 0, ix->stream>>>(ix->view(), n_items, batches, chain, d_counter, d_sink, d_bm, bm_words, atomics);
        else gather_bench_kernel<16, 5><<<grid, kSearchWarps * 32, 0, ix->stream>>>(ix->view(), n_items, batches, chain, d_counter, d_sink, d_bm, bm_words, atomics);
        CUDA_TRY(cudaEventRecord(e1, ix->stream));
        CUDA_TRY(cudaEventSynchronize(e1));
        float ms = 0;
        CUDA_TRY(cudaEventElapsedTime(&ms, e0, e1));
        if (r > 0) best = std::min(best, ms);
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaFree(d_counter);
    cudaFree(d_sink);
    if (d_bm && std::getenv("IDB_DEBUG_BM_PERSIST")) {
        cudaStreamAttrValue av;
        std::memset(&av, 0, sizeof(av));
        cudaStreamSetAttribute(ix->stream, cudaStreamAttributeAccessPolicyWindow, &av);
        cudaCtxResetPersistingL2Cache();
    }
    cudaFree(d_bm);
    *out_ms = best;
    if (out_bytes) *out_bytes = (double)n_items * batches * 16.0 * ix->nchunks * 16.0;
    return IDB_OK;
}

extern "C" idb_status idb_debug_gather_bench(idb_index* index, uint32_t n_items, uint32_t batches, uint32_t chain, uint32_t reps,
                                             float* out_ms, double* out_bytes) {
    return gather_bench_impl(index, n_items, batches, chain, reps, 0, 0, out_ms, out_bytes);
}
extern "C" idb_status idb_debug_gather_mix_bench(idb_index* index, uint32_t n_items, uint32_t batches, uint32_t chain, uint32_t reps,
                                                 uint32_t atomics_per_batch, uint32_t mode, float* out_ms, double* out_bytes) {
    return gather_bench_impl(index, n_items, batches, chain, reps, atomics_per_batch, mode, out_ms, out_bytes);
}
