// build.cu — host driver of Builder::build_hnsw (instant-distance/src/lib.rs:83-85 -> Hnsw::new, lib.rs:209-345) on the GPU.
//
//   1. layer schedule            lib.rs:238-250  (f32 multiply, truncating cast)
//   2. seeded shuffle            lib.rs:257-270  (xoshiro256++ seeded through SplitMix64; widening-multiply range sampling —
//                                                 the rand crate is not vendored in the reference tree: parity unpinned)
//   3. per layer, top first      lib.rs:304-329  batches of concurrent inserts (KA -> K2 -> sort -> K2'), then the
//                                                 UpperNode snapshot (K5)
// The batch schedule replaces rayon: batch = min(16384, max(1, inserted / 8)); the top layer is sequential like the
// reference's (lib.rs:313-314).  insert_batch = 1 reproduces the sequential reference order exactly.
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "build_dispatch.cuh"

namespace idb {

static cudaError_t build_dispatch_any(const BuildArgs& a, const BuildLaunch& l, cudaStream_t st) {
    return with_cell(a.g.nchunks, [&](auto cell) {
        constexpr int CH = decltype(cell)::CH;
        if (a.g.row_type == kRowBin) return build_cells<CH, true>(a, l, st);
        return build_cells<CH, false>(a, l, st);
    });
}

namespace {

// No heuristic (Builder::select_heuristic(None), lib.rs:466-469): found = first min(len, 2M) of `nearest`.
__global__ void select_simple_kernel(BuildArgs a) {
    const uint32_t cap = 2 * a.g.M;
    for (uint32_t w = blockIdx.x; w < a.count; w += gridDim.x) {
        const uint32_t neu = a.base + w;
        const uint32_t total = min(a.cand_cnt[w], cap);
        uint32_t* row = a.zero + (size_t)neu * cap;
        for (uint32_t t = threadIdx.x; t < cap; t += blockDim.x) {
            const uint32_t pid = t < total ? key_pid(a.cand_keys[(size_t)w * a.cand_cap + t]) : kInvalid;
            row[t] = pid;
            a.pairs[(size_t)w * cap + t] = t < total ? (((uint64_t)pid << 32) | neu) : kKeyNone;
        }
    }
}

// Segment heads of the sorted link requests: one work item per distinct target row.
__global__ void segment_heads_kernel(const uint64_t* sorted_pairs, uint32_t n, uint32_t* seg_start, uint32_t* n_seg) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t tgt = (uint32_t)(sorted_pairs[i] >> 32);
    if (tgt == kInvalid) return;
    if (i == 0 || (uint32_t)(sorted_pairs[i - 1] >> 32) != tgt) seg_start[atomicAdd(n_seg, 1u)] = i;
}

// K5: UpperNode::from_zero (types.rs:65-71) for nodes [0, n_l).
__global__ void snapshot_kernel(const uint32_t* zero, uint32_t* upper, uint64_t n_l, uint32_t M) {
    const uint64_t total = n_l * M;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t v = i / M, e = i - v * M;
        upper[i] = zero[v * 2 * M + e];
    }
}

// K6: points[rank] = rows[order[rank]]  (lib.rs:263-270), zero-padding each row to a multiple of 4 floats.
__global__ void gather_rows_kernel(const float* rows, const uint32_t* order, float* points, uint64_t n, uint32_t dim, uint32_t stride) {
    const uint64_t total = n * stride;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = i / stride;
        const uint32_t c = (uint32_t)(i - r * stride);
        points[i] = c < dim ? rows[(uint64_t)order[r] * dim + c] : 0.f;
    }
}

struct Xoshiro256pp {  // rand's SmallRng on 64-bit targets
    uint64_t s[4];
    explicit Xoshiro256pp(uint64_t seed) {  // SeedableRng::seed_from_u64: SplitMix64 stream
        uint64_t state = seed;
        for (int i = 0; i < 4; ++i) {
            state += 0x9e3779b97f4a7c15ull;
            uint64_t z = state;
            z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
            z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
            s[i] = z ^ (z >> 31);
        }
    }
    static uint64_t rotl(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
    uint64_t next_u64() {
        const uint64_t res = rotl(s[0] + s[3], 23) + s[0];
        const uint64_t t = s[1] << 17;
        s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3];
        s[2] ^= t;
        s[3] = rotl(s[3], 45);
        return res;
    }
    uint32_t next_u32() { return (uint32_t)(next_u64() >> 32); }
    uint32_t below(uint32_t range) {  // random_range(0..range)
        const uint64_t m = (uint64_t)next_u32() * range;
        uint32_t result = (uint32_t)(m >> 32);
        const uint32_t lo = (uint32_t)m;
        if (lo > (uint32_t)(0u - range)) {
            const uint32_t hi2 = (uint32_t)(((uint64_t)next_u32() * range) >> 32);
            result += (uint32_t)(lo + hi2 < lo);
        }
        return result;
    }
};

// (size, cumulative) per layer, top layer first (lib.rs:238-249)
std::vector<std::pair<uint64_t, uint64_t>> layer_sizes(uint64_t n, uint32_t M, float ml) {
    std::vector<std::pair<uint64_t, uint64_t>> sizes;
    uint64_t num = n;
    for (;;) {
        const float f = (float)num * ml;
        const uint64_t next = f >= 1.8446744e19f ? UINT64_MAX : (f > 0.0f ? (uint64_t)f : 0);
        if (next < M || next >= num) break;
        sizes.push_back({num - next, num});
        num = next;
    }
    sizes.push_back({num, num});
    std::reverse(sizes.begin(), sizes.end());
    return sizes;
}

// The build's control block, zeroed before every batch.
struct BuildCtrl {
    PassCtrl insert, retry;             // KA and its retry pass
    unsigned long long relink_work;     // K2' work counter
    uint32_t n_seg;                     // K2' work items: distinct target rows of the batch's link requests
};

struct BuildScratch {
    uint64_t* cand_keys = nullptr;
    uint32_t* cand_cnt = nullptr;
    uint64_t* pairs = nullptr;
    uint64_t* sorted = nullptr;
    uint32_t* seg_start = nullptr;
    uint32_t* status = nullptr;
    uint32_t* fail_list = nullptr;
    void* cub_tmp = nullptr;
    size_t cub_bytes = 0;
    BuildCtrl* ctrl = nullptr;
    BuildCtrl* h_ctrl = nullptr;    // pinned: the last batch's control block
    ~BuildScratch() {
        cudaFree(cand_keys); cudaFree(cand_cnt); cudaFree(pairs); cudaFree(sorted); cudaFree(seg_start); cudaFree(status);
        cudaFree(fail_list); cudaFree(cub_tmp); cudaFree(ctrl);
        if (h_ctrl) cudaFreeHost(h_ctrl);
    }
};

// The batch schedule's cap and divisor: a batch at g0 inserts min(max_batch, max(1, g0 / growth)) points.
void batch_schedule(const idb_params& p, uint32_t* max_batch, uint32_t* growth) {
    // Defaults: batch <= 16384 and <= 1/8 of the graph keeps recall@10 of the built graph close to the reference algorithm's own
    // graph (tests/test_gpu_build.py checks it) while giving each batch enough inserts to fill the device.
    *max_batch = p.insert_batch ? p.insert_batch : 16384u;
    *growth = 8;  // a batch never exceeds 1/8 of the graph it is inserted into
    if (!p.insert_batch) {  // tuning knobs for experiments (results stay valid HNSW graphs; determinism per setting)
        if (const char* e = std::getenv("IDB_BUILD_MAXBATCH")) *max_batch = (uint32_t)std::max(1, std::atoi(e));
        if (const char* e = std::getenv("IDB_BUILD_GROWTH")) *growth = (uint32_t)std::max(1, std::atoi(e));
    }
}

// One batch of concurrent inserts — KA (+ its retry pass) -> K2 -> sort -> segment heads -> K2' — and the scratch it runs in.
// The build and the insert (idb_index_insert_f32) both drive their batches through run().
struct BatchRunner {
    Index* ix = nullptr;
    BuildScratch bs;
    BuildArgs a;
    bool heuristic = true;
    bool stage = false;
    uint32_t k2_smem = 0;
    int k2_ctas_per_sm = 1;
    // ka_first: read KA's control block back before K2 and stop there when an insert overflowed even the retry pass, so a failing
    // batch changes no row (the insert's failure semantics).  Otherwise the block is read once, after K2' (the build's flow).
    bool ka_first = false;

    // Scratch for batches of up to max_b inserts into ix as it stands (ix->view(): rows, n, layers).
    idb_status init(Index* index, const idb_params& p, uint64_t max_b, bool ka_first_) {
        ix = index;
        ka_first = ka_first_;
        heuristic = p.heuristic != 0;
        const uint32_t M = ix->M, cap = 2 * M, efc = p.ef_construction;
        cudaStream_t st = ix->stream;
        const uint32_t cand_cap = std::max<uint32_t>((efc + 31) / 32 * 32, cap + kNewCap);
        CUDA_TRY(cudaMalloc(&bs.cand_keys, (size_t)max_b * cand_cap * 8));
        CUDA_TRY(cudaMalloc(&bs.cand_cnt, (size_t)max_b * 4));
        CUDA_TRY(cudaMalloc(&bs.pairs, (size_t)max_b * cap * 8));
        CUDA_TRY(cudaMalloc(&bs.sorted, (size_t)max_b * cap * 8));
        CUDA_TRY(cudaMalloc(&bs.seg_start, (size_t)max_b * cap * 4));
        CUDA_TRY(cudaMalloc(&bs.status, (size_t)max_b * 4));
        CUDA_TRY(cudaMalloc(&bs.fail_list, (size_t)max_b * 4));
        CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(&bs.h_ctrl), sizeof(BuildCtrl), cudaHostAllocDefault));
        CUDA_TRY(cudaMalloc(&bs.ctrl, sizeof(BuildCtrl)));
        CUDA_TRY(cub::DeviceRadixSort::SortKeys(nullptr, bs.cub_bytes, bs.pairs, bs.sorted, (int)(max_b * cap), 0, 64, st));
        CUDA_TRY(cudaMalloc(&bs.cub_tmp, std::max<size_t>(bs.cub_bytes, 16)));

        // Staging the kept rows in shared memory (72 KB per 2-warp CTA -> 6 warps per SM) trades 32 resident warps for 6 to save
        // reads that L1/L2 serve anyway, so it is off unless asked for.
        if (const char* e = std::getenv("IDB_BUILD_STAGE")) stage = std::atoi(e) != 0 && SelectSmem::bytes(cand_cap, M, ix->nchunks, true) <= 56 * 1024;
        k2_smem = (uint32_t)SelectSmem::bytes(cand_cap, M, ix->nchunks, stage);
        // K2 / K2' are persistent grids of 2-warp CTAs.  They are issue-bound (pairwise distances on L1/L2-resident rows), so the
        // grid asks for as many CTAs per SM as shared memory (228 KB per SM on an H100) and registers allow, up to 16 (32 warps per SM).
        k2_ctas_per_sm = (int)std::min<uint64_t>(16, std::max<uint64_t>(1, (200 * 1024) / std::max<uint32_t>(1, k2_smem * kBuildWarps)));
        if (const char* e = std::getenv("IDB_BUILD_CTAS")) k2_ctas_per_sm = std::max(1, std::atoi(e));

        std::memset(&a, 0, sizeof(a));
        a.g = ix->view();
        a.zero = ix->graph.zero;
        a.efc = efc;
        a.cand_cap = cand_cap;
        a.keep_pruned = p.keep_pruned ? 1u : 0u;
        a.cand_keys = bs.cand_keys;
        a.cand_cnt = bs.cand_cnt;
        a.pairs = bs.pairs;
        a.work.status = bs.status;
        a.work.fail_count = &bs.ctrl->insert.fail_count;
        a.work.fail_list = bs.fail_list;
        a.sorted_pairs = bs.sorted;
        a.seg_start = bs.seg_start;
        a.n_seg = &bs.ctrl->n_seg;
        return IDB_OK;
    }

    // Inserts PointIds [g0, g0 + b) on `layer`.  IDB_ERR_CAPACITY: an insert overflowed even the retry pass (with ka_first, before
    // any row of this batch was written).
    idb_status run(uint64_t g0, uint64_t b, uint32_t layer) {
        cudaStream_t st = ix->stream;
        const uint32_t cap = 2 * ix->M, efc = a.efc;
        a.base = (uint32_t)g0;
        a.count = (uint32_t)b;
        a.work.n_work = b;
        a.layer = layer;
        a.n_pairs_cap = (uint32_t)(b * cap);
        CUDA_TRY(cudaMemsetAsync(bs.ctrl, 0, sizeof(BuildCtrl), st));
        // KA: descent of every insert, then (device-side, normally a no-op) a retry pass with 2^18-slot hash sets and 64k-entry
        // tie lists for the inserts whose per-warp structures overflowed (e.g. inside a cluster of thousands of duplicate vectors)
        BuildLaunch l;
        l.op = kOpInsertSearch;
        l.row_t = (int)((cap + 31) / 32);
        l.ef_t = (int)((efc + 31) / 32);
        l.stage = stage;
        l.smem_per_warp = k2_smem;
        l.grid = (int)std::max<uint64_t>(1, std::min<uint64_t>((b + kSearchWarps - 1) / kSearchWarps, (uint64_t)ix->search_grid()));
        {
            std::lock_guard<std::mutex> lk(ix->ctx->mu);  // the pool's tables must not be regrown under these launches
            idb_status ts = ix->select_visited_tier(efc, a.tier, l.win);
            if (ts == IDB_OK) ts = ix->attach_window(ix->lanes[0], l.win);
            if (ts != IDB_OK) return ts;
            a.work.work_counter = &bs.ctrl->insert.work_counter;
            CUDA_TRY(build_dispatch_any(a, l, st));
            BuildLaunch lr = l;
            lr.grid = kRetryCtas;
            lr.win = LaunchWindow();
            BuildArgs r = retry_pass(a, *ix->ctx, &bs.ctrl->retry);
            if (ix->retry_slots_override) {  // tests: a retry pass that can fail (with IDB_VIS_SLOTS, on ordinary data)
                r.tier.gslots = ix->retry_slots_override;
                r.tier.gshift = 32 - (uint32_t)std::log2((double)ix->retry_slots_override);
            }
            CUDA_TRY(build_dispatch_any(r, lr, st));
        }
        const int ka_b16 = a.tier.mode == kVisB16 ? ix->b16_level : 0;
        if (ka_first) {
            CUDA_TRY(cudaMemcpyAsync(bs.h_ctrl, bs.ctrl, sizeof(BuildCtrl), cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaStreamSynchronize(st));
            if (bs.h_ctrl->retry.fail_count)
                return fail(IDB_ERR_CAPACITY, "%u inserts overflowed an internal per-insert structure (visited table / tie list) in the batch starting at %llu",
                            bs.h_ctrl->retry.fail_count, (unsigned long long)g0);
        }
        // K2: neighbour selection for the new nodes, own rows, link requests
        if (heuristic) {
            l.op = kOpSelectNew;
            l.grid = (int)std::max<uint64_t>(1, std::min<uint64_t>((b + kBuildWarps - 1) / kBuildWarps, (uint64_t)ix->num_sms * k2_ctas_per_sm));
            CUDA_TRY(build_dispatch_any(a, l, st));
        } else {
            select_simple_kernel<<<(unsigned)std::min<uint64_t>(b, 1024), 64, 0, st>>>(a);
            CUDA_TRY(cudaGetLastError());
        }
        // group the link requests by target row
        size_t tmp = bs.cub_bytes;
        CUDA_TRY(cub::DeviceRadixSort::SortKeys(bs.cub_tmp, tmp, bs.pairs, bs.sorted, (int)(b * cap), 0, 64, st));
        segment_heads_kernel<<<(unsigned)((b * cap + 255) / 256), 256, 0, st>>>(bs.sorted, (uint32_t)(b * cap), bs.seg_start,
                                                                              &bs.ctrl->n_seg);
        CUDA_TRY(cudaGetLastError());
        // K2': re-prune every target row once
        l.op = heuristic ? kOpRelink : kOpRelinkSimple;
        l.grid = (int)std::max<uint64_t>(1, std::min<uint64_t>((b * cap + kBuildWarps - 1) / kBuildWarps, (uint64_t)ix->num_sms * k2_ctas_per_sm));
        a.work.work_counter = &bs.ctrl->relink_work;
        CUDA_TRY(build_dispatch_any(a, l, st));
        if (!ka_first) {
            CUDA_TRY(cudaMemcpyAsync(bs.h_ctrl, bs.ctrl, sizeof(BuildCtrl), cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaStreamSynchronize(st));  // fail fast: an insert that overflowed even the retry pass ends the build here
            if (bs.h_ctrl->retry.fail_count)
                return fail(IDB_ERR_CAPACITY, "%u inserts overflowed an internal per-insert structure (visited table / tie list) in the batch ending at %llu",
                            bs.h_ctrl->retry.fail_count, (unsigned long long)(g0 + b));
        }
        ix->note_overflows(efc, b, bs.h_ctrl->insert.fail_count, ka_b16);  // too many b16 overflows: later batches use a larger flavour
        return IDB_OK;
    }
};

}  // namespace

idb_status build_index(Index* ix, const float* rows, uint64_t n, uint32_t dim, const idb_params& p, uint32_t* out_ids) {
    const uint32_t M = p.M;
    ix->n = n;
    ix->dim = dim;
    ix->M = M;
    ix->ef_search = p.ef_search;
    ix->nchunks = (dim + 3) / 4;
    if (n == 0) return IDB_OK;  // lib.rs:224-234
    cudaStream_t st = ix->stream;
    const uint32_t cap = 2 * M;
    const size_t stride = (size_t)ix->nchunks * 4;

    // ---- 1. layers, 2. shuffle ------------------------------------------------------------------------------
    const auto sizes = layer_sizes(n, M, p.ml);
    const uint32_t num_layers = (uint32_t)sizes.size(), top = num_layers - 1;
    if (top > 31) return fail(IDB_ERR_INVALID_ARG, "ml = %g produces %u layers (max 32)", (double)p.ml, num_layers);
    std::vector<uint32_t> order(n);
    {
        Xoshiro256pp rng(p.seed);
        std::vector<std::pair<uint32_t, uint64_t>> sh(n);
        for (uint64_t i = 0; i < n; ++i) sh[i] = {rng.below((uint32_t)n), i};
        std::sort(sh.begin(), sh.end());
        for (uint64_t r = 0; r < n; ++r) {
            order[r] = (uint32_t)sh[r].second;
            if (out_ids) out_ids[sh[r].second] = (uint32_t)r;
        }
    }

    // ---- device arrays ----------------------------------------------------------------------------------------
    ix->cap = n;
    idb_status s = ix->put_rows(0, n, order.data(), [&](float* dst) {  // refusals name the caller's row, order[PointId]
        float* d_rows = nullptr;
        uint32_t* d_order = nullptr;
        cudaError_t e = cudaMalloc(&d_rows, n * (size_t)dim * sizeof(float));
        if (e == cudaSuccess) e = cudaMalloc(&d_order, n * sizeof(uint32_t));
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_rows, rows, n * (size_t)dim * sizeof(float), cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_order, order.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) {
            gather_rows_kernel<<<ix->num_sms * 8, 256, 0, st>>>(d_rows, d_order, dst, n, dim, (uint32_t)stride);
            e = cudaGetLastError();
        }
        if (e == cudaSuccess && ix->metric == kMetricCosine)  // DESIGN §3a: a cosine index stores the normalised rows
            e = normalize_rows(dst, stride, dst, n, dim, ix->nchunks, ix->num_sms, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        cudaFree(d_rows);
        cudaFree(d_order);
        return e;
    });
    if (s != IDB_OK) return s;
    std::vector<uint64_t> upper_n;
    for (uint32_t l = 1; l <= top; ++l) upper_n.push_back(sizes[num_layers - 1 - l].second);
    CUDA_TRY(ix->graph.alloc(n, M, std::move(upper_n), st));
    CUDA_TRY(fill_u32(ix->graph.zero, n * (size_t)cap, kInvalid, st));

    // ---- batch schedule + scratch -------------------------------------------------------------------------------
    uint32_t max_batch = 0, growth = 0;
    batch_schedule(p, &max_batch, &growth);
    BatchRunner run;
    idb_status rs = run.init(ix, p, max_batch, false);
    if (rs != IDB_OK) return rs;

    for (uint32_t li = 0; li < num_layers; ++li) {  // lib.rs:304-329
        const uint32_t layer = num_layers - li - 1;
        const uint64_t size = sizes[li].first, cumulative = sizes[li].second;
        const uint64_t start = std::max<uint64_t>(cumulative - size, 1), end = cumulative;
        uint64_t g0 = start;
        while (g0 < end) {
            uint64_t b = 1;
            if (layer != top && max_batch > 1) b = std::min<uint64_t>(max_batch, std::max<uint64_t>(1, g0 / growth));
            b = std::min<uint64_t>(b, end - g0);
            rs = run.run(g0, b, layer);
            if (rs != IDB_OK) return rs;
            g0 += b;
            if (p.progress) p.progress(g0, n, p.progress_user);  // set_position (core:519-525)
        }
        if (layer != 0) {  // lib.rs:323-328
            snapshot_kernel<<<ix->num_sms * 4, 256, 0, st>>>(ix->graph.zero, ix->graph.upper[layer - 1], end, M);
            CUDA_TRY(cudaGetLastError());
        }
    }
    CUDA_TRY(cudaStreamSynchronize(st));
    if (p.progress) p.progress(n, n, p.progress_user);  // finish (core:331-334)
    return IDB_OK;
}

// Construction::insert(new, 0, layers) (core:437-528) for PointIds [n0, n0 + m), in the build's layer-0 batch schedule from g0 = n0
// (also when the index has no upper layer, where the build inserts sequentially).  The caller holds the index exclusively and has
// checked the arguments.  Rows: m x dim host floats, stored as the build stores them (zero padded, normalised for a cosine index,
// then narrowed for a bf16 or fp16 one, quantised for a q8 one or packed for a bin one; fp16 / q8 / bin rows beyond the storage's
// range are refused before the index's rows or graph change).  global_ids: appended to the id map when the index has one.
idb_status insert_index(Index* ix, const float* rows, uint64_t m, const idb_params& p, const uint32_t* global_ids, uint32_t* out_ids) {
    const uint64_t n0 = ix->n, n1 = n0 + m;
    if (out_ids)
        for (uint64_t i = 0; i < m; ++i) out_ids[i] = (uint32_t)(n0 + i);
    if (m == 0) return IDB_OK;
    // ---- storage: grow (copying the first n0 rows), then stage the new rows behind them; nothing below n0 changes -------------
    idb_status s = ix->reserve_rows(n1);
    if (s == IDB_OK)
        s = ix->put_rows(n0, m, nullptr, [&](float* dst) {  // refusals name the row within the call
            cudaError_t e = ix->copy_rows_in(dst, rows, m);
            if (e == cudaSuccess && ix->metric == kMetricCosine)
                e = normalize_rows(dst, (size_t)ix->nchunks * 4, dst, m, ix->dim, ix->nchunks, ix->num_sms, ix->stream);
            return e;
        });
    if (s == IDB_OK) s = ix->stage_rows(n0, m, global_ids);
    if (s != IDB_OK) return s;
    uint32_t max_batch = 0, growth = 0;
    batch_schedule(p, &max_batch, &growth);
    const uint64_t start = std::max<uint64_t>(n0, 1);  // an empty index: PointId 0 is the entry point (lib.rs:304-308)
    BatchRunner run;
    ix->n = n1;  // the traversals' view: every row the insert can reach
    s = run.init(ix, p, std::min<uint64_t>(max_batch, n1 - start + 1), true);
    if (s != IDB_OK) {
        ix->n = n0;
        return s;
    }
    // ---- layer 0, batched from n0 ---------------------------------------------------------------------------------------------
    uint64_t reported = 0;  // the last progress value: the callback sees m exactly once
    for (uint64_t g0 = start; g0 < n1;) {
        const uint64_t b = std::min<uint64_t>(std::min<uint64_t>(max_batch, std::max<uint64_t>(1, g0 / growth)), n1 - g0);
        s = run.run(g0, b, 0);
        if (s == IDB_ERR_CAPACITY) {  // the batches before it stand; its rows were never written
            ix->n = g0;
            idb_status c = ix->build_codes();
            return c == IDB_OK ? s : c;
        }
        if (s != IDB_OK) return s;
        g0 += b;
        reported = g0 - n0;
        if (p.progress) p.progress(reported, m, p.progress_user);
    }
    CUDA_TRY(cudaStreamSynchronize(ix->stream));
    if (p.progress && reported != m) p.progress(m, m, p.progress_user);  // no batch ran: an empty index given one row
    return ix->build_codes();  // from all stored rows: the table's step, offsets and error bound follow the new rows
}

const char kNoExtendCandidates[] =
    "Heuristic::extend_candidates = true is not supported: in the reference it re-locks the row being inserted "
    "(lib.rs:438 write lock vs lib.rs:649 read lock through types.rs:146) and never returns";

idb_status check_link_params(const idb_params* p) {
    if (p->ef_construction == 0 || p->ef_construction > 1024)
        return fail(IDB_ERR_UNSUPPORTED, "ef_construction = %u unsupported (1..1024)", p->ef_construction);
    if (p->heuristic && p->extend_candidates) return fail(IDB_ERR_UNSUPPORTED, "%s", kNoExtendCandidates);
    return IDB_OK;
}

}  // namespace idb

using namespace idb;

extern "C" idb_status idb_build_f32(const float* rows, uint64_t n, uint32_t dim, const idb_params* params, idb_index** out_index,
                                    uint32_t* out_ids) {
    return idb_build_ex(rows, n, dim, params, IDB_METRIC_L2SQ, out_index, out_ids);
}

extern "C" idb_status idb_build_ex(const float* rows, uint64_t n, uint32_t dim, const idb_params* params, uint32_t metric,
                                   idb_index** out_index, uint32_t* out_ids) {
    if (!out_index) return fail(IDB_ERR_INVALID_ARG, "out_index is null");
    if (metric != IDB_METRIC_L2SQ && metric != IDB_METRIC_COSINE) return fail(IDB_ERR_INVALID_ARG, "unknown metric %u", metric);
    *out_index = nullptr;
    if (!params) return fail(IDB_ERR_INVALID_ARG, "params is null");
    if (dim == 0) return fail(IDB_ERR_INVALID_ARG, "dim must be >= 1");
    if (n && !rows) return fail(IDB_ERR_INVALID_ARG, "rows is null");
    if (params->M < 2 || params->M > 64) return fail(IDB_ERR_INVALID_ARG, "M = %u unsupported (2..64)", params->M);
    if (n >= 0xFFFFFFFFull) return fail(IDB_ERR_INVALID_ARG, "N = %llu >= u32::MAX (lib.rs:256)", (unsigned long long)n);
    if (params->ef_construction == 0 || params->ef_construction > 1024)
        return fail(IDB_ERR_UNSUPPORTED, "ef_construction = %u unsupported (1..1024)", params->ef_construction);
    if (dim > 10240) return fail(IDB_ERR_UNSUPPORTED, "dim %u > 10240 is not supported (the owner row of a long-row traversal lives in shared memory)", dim);
    if (!(params->ml > 0.0f) || params->ml >= 1.0f) return fail(IDB_ERR_INVALID_ARG, "ml must be in (0, 1)");
    if (!storage_known(params->storage)) return fail(IDB_ERR_INVALID_ARG, "unknown storage %u", params->storage);
    if (idb_status s = check_storage_metric(params->storage, metric); s != IDB_OK) return s;
    if (params->heuristic && params->extend_candidates) return fail(IDB_ERR_UNSUPPORTED, "%s", kNoExtendCandidates);
    auto* ix = new (std::nothrow) Index();
    if (!ix) return fail(IDB_ERR_OOM, "host allocation failed");
    ix->metric = metric;
    ix->row_type = params->storage;
    idb_status st = ix->init_device(params->device);
    if (st == IDB_OK) {
        std::lock_guard<std::mutex> lk(ix->mu);
        st = build_index(ix, rows, n, dim, *params, out_ids);
        if (st == IDB_OK) st = ix->build_codes();  // from the final stored rows (normalised, narrowed); the build itself does not screen
    }
    if (st != IDB_OK) { delete ix; return st; }
    *out_index = reinterpret_cast<idb_index*>(ix);
    return IDB_OK;
}

extern "C" idb_status idb_index_insert_f32(idb_index* index, const float* rows, uint64_t m, uint32_t dim, const idb_params* params,
                                           const uint32_t* global_ids, uint32_t* out_ids) {
    // checks that need neither the handle nor a device first, as the search entries do
    if (!index) return fail(IDB_ERR_INVALID_ARG, "index is null");
    if (!params) return fail(IDB_ERR_INVALID_ARG, "params is null");
    if (m && !rows) return fail(IDB_ERR_INVALID_ARG, "rows is null");
    idb_status st = check_link_params(params);
    if (st == IDB_OK) st = require_device();
    if (st != IDB_OK) return st;
    Index* ix = reinterpret_cast<Index*>(index);
    // &mut self: no search, export or other insert runs while the index changes, and each search sees it before or after this call
    ExclusiveIndex ex(ix);
    if (dim != ix->dim) return fail(IDB_ERR_INVALID_ARG, "dim %u differs from the index's %u", dim, ix->dim);
    if (params->M != ix->M) return fail(IDB_ERR_INVALID_ARG, "M = %u differs from the index's %u", params->M, ix->M);
    if (m && ix->d_id_map && !global_ids) return fail(IDB_ERR_INVALID_ARG, "the index has an id map: global_ids is required");
    if (!ix->d_id_map && global_ids) return fail(IDB_ERR_INVALID_ARG, "global_ids given, but the index has no id map");
    if (ix->n + m >= 0xFFFFFFFFull)
        return fail(IDB_ERR_INVALID_ARG, "N = %llu + %llu >= u32::MAX (lib.rs:256)", (unsigned long long)ix->n, (unsigned long long)m);
    CUDA_TRY(ex.drained);
    return insert_index(ix, rows, m, *params, global_ids, out_ids);
}
