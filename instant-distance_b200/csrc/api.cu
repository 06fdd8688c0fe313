// api.cu — C ABI (include/instant_distance_b200.h) + the batched search kernel.
//
// Host side of the drop-in boundary: the index object, whose row-major point matrix (rows.cu) and per-layer fixed-stride adjacency
// ("CSR with implicit row_ptr = pid * stride", rows INVALID-terminated; graph.cu) live in HBM, and the sm_90a kernels' launches.
// No PyTorch, no CPU fallback: if the CUDA runtime reports no device every compute entry point fails loudly.
#include "search_kernel.cuh"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace idb {

thread_local char g_err[512] = "";

idb_status fail(idb_status st, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return st;
}

static cudaError_t dispatch_search(const SearchArgs& a, int row_t, int ef_t, int grid, cudaStream_t st, const LaunchWindow& win) {
    return with_cell(a.g.nchunks, [&](auto cell) {
        constexpr int CH = decltype(cell)::CH;
        if (a.g.row_type == kRowBin) return search_cells<CH, true>(a, row_t, ef_t, grid, st, win);
        return search_cells<CH, false>(a, row_t, ef_t, grid, st, win);
    });
}

__global__ void distance_kernel(const float4* a, const float4* b, uint32_t nchunks, float* out) {
    const int lane = threadIdx.x;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (uint32_t c = lane; c < nchunks; c += 32) {
        float4 x = a[c], y = b[c];
        float d0 = __fsub_rn(x.x, y.x), d1 = __fsub_rn(x.y, y.y), d2 = __fsub_rn(x.z, y.z), d3 = __fsub_rn(x.w, y.w);
        acc.x = __fmaf_rn(d0, d0, acc.x);
        acc.y = __fmaf_rn(d1, d1, acc.y);
        acc.z = __fmaf_rn(d2, d2, acc.z);
        acc.w = __fmaf_rn(d3, d3, acc.w);
    }
    float s = butterfly_sum(__fadd_rn(__fadd_rn(acc.x, acc.y), __fadd_rn(acc.z, acc.w)));
    if (lane == 0) *out = s;
}

// One warp per row: the canonical normalisation (hnsw_device.cuh normalize_row).  No __restrict__ / __ldg: dst may alias src.
__global__ void normalize_rows_kernel(const float* src, uint64_t src_stride, float4* dst, uint64_t n, uint32_t dim, uint32_t nchunks) {
    const int lane = threadIdx.x & 31;
    const uint64_t wpb = blockDim.x >> 5;
    for (uint64_t r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += (uint64_t)gridDim.x * wpb)
        normalize_row(src + r * src_stride, dim, dst + r * nchunks, nchunks, lane);
}

cudaError_t normalize_rows(const float* src, uint64_t src_stride, float* dst, uint64_t n, uint32_t dim, uint32_t nchunks, int num_sms,
                           cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const uint64_t blocks = std::min<uint64_t>((n + 7) / 8, (uint64_t)num_sms * 16);
    normalize_rows_kernel<<<(unsigned)blocks, 256, 0, st>>>(src, src_stride, reinterpret_cast<float4*>(dst), n, dim, nchunks);
    return cudaGetLastError();
}

__global__ void nsmid_kernel(uint32_t* out) { asm volatile("mov.u32 %0, %%nsmid;" : "=r"(*out)); }

__global__ void fill_u32_kernel(uint32_t* p, size_t n, uint32_t v) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}

cudaError_t fill_u32(uint32_t* p, size_t n, uint32_t v, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    fill_u32_kernel<<<1184, 256, 0, st>>>(p, n, v);
    return cudaGetLastError();
}

static uint32_t next_pow2(uint64_t v) {
    uint32_t p = 1;
    while (p < v && p < (1u << 30)) p <<= 1;
    return p;
}

// ---------------------------------------------------------------------------------------------------------
// Scratch management
// ---------------------------------------------------------------------------------------------------------
template <class T>
static cudaError_t ensure(T*& p, size_t& cap, size_t need) {
    if (need <= cap && p) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = need + need / 4 + 64;
    cudaError_t e = cudaMalloc(&p, want * sizeof(T));
    if (e == cudaSuccess) cap = want;
    return e;
}

cudaError_t ensure_u32(uint32_t*& p, size_t& cap, size_t need) { return ensure(p, cap, need); }
cudaError_t ensure_u64(uint64_t*& p, size_t& cap, size_t need) { return ensure(p, cap, need); }
cudaError_t ensure_f32(float*& p, size_t& cap, size_t need) { return ensure(p, cap, need); }


// ---------------------------------------------------------------------------------------------------------
// DeviceCtx: the per-device pool of per-warp scratch tables
// ---------------------------------------------------------------------------------------------------------
namespace {
std::mutex g_ctx_mu;
DeviceCtx* g_ctx[64] = {};
int g_l2_pref[64] = {};  // idb_device_set_persisting_l2: 0 default (IDB_L2_PERSIST, else off), 1 enabled, -1 disabled
}  // namespace

TablePool DeviceCtx::main_pool(bool b16) const {
    TablePool tp;
    tp.slot_masks = slot_masks;
    tp.fixed_word = -1;
    tp.word_base = 0;
    tp.slots_per_word = (uint32_t)slots_per_sm;
    tp.vis_tables = b16 ? b16_tables : big_tables;
    tp.vis_stride = b16 ? b16_stride : big_stride;
    tp.vis_ext = b16 ? b16_ext : nullptr;
    tp.ext_stride = b16 ? b16_stride : 0;
    tp.tie_tables = tie_tables;
    tp.tie_cap = kTieCap;
    return tp;
}
VisTier DeviceCtx::retry_tier() const {
    VisTier t = {};
    t.pool.slot_masks = slot_masks;
    t.pool.fixed_word = sm_ids;
    t.pool.word_base = (uint32_t)sm_ids;
    t.pool.slots_per_word = kRetryCtas;
    t.pool.vis_tables = retry_tables;
    t.pool.vis_stride = kRetrySlots;
    t.pool.vis_ext = nullptr;
    t.pool.ext_stride = 0;
    t.pool.tie_tables = retry_ties;
    t.pool.tie_cap = kRetryTieCap;
    t.gslots = kRetrySlots;
    t.gshift = 32 - 18;
    static_assert(kRetrySlots == 1u << 18, "gshift above");
    t.mode = kVisHash;
    return t;
}

idb_status DeviceCtx::acquire(int device, DeviceCtx** out) {
    std::lock_guard<std::mutex> lk(g_ctx_mu);
    if (device < 0 || device >= 64) return fail(IDB_ERR_INVALID_ARG, "device %d out of range", device);
    if (g_ctx[device]) {
        g_ctx[device]->refs++;
        *out = g_ctx[device];
        return IDB_OK;
    }
    auto* c = new (std::nothrow) DeviceCtx();
    if (!c) return fail(IDB_ERR_OOM, "host allocation failed");
    c->device = device;
    cudaDeviceProp prop;
    auto bail = [&](cudaError_t e, int line) {
        delete c;
        return fail(e == cudaErrorMemoryAllocation ? IDB_ERR_OOM : IDB_ERR_CUDA, "CUDA error %s at %s:%d (%s)", cudaGetErrorName(e), __FILE__,
                    line, cudaGetErrorString(e));
    };
#define CTX_TRY(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) return bail(e_, __LINE__); } while (0)
    CTX_TRY(cudaGetDeviceProperties(&prop, device));
    c->num_sms = prop.multiProcessorCount;
    if (const char* e = std::getenv("IDB_CTAS_PER_SM")) c->slots_per_sm = std::min(kMaxCtasPerSm, std::max(1, std::atoi(e)));
    {   // SM ids run up to %nsmid, which counts disabled SMs too
        uint32_t* d = nullptr;
        uint32_t h = 0;
        CTX_TRY(cudaMalloc(&d, 4));
        nsmid_kernel<<<1, 1>>>(d);
        cudaError_t e1 = cudaMemcpy(&h, d, 4, cudaMemcpyDeviceToHost);
        cudaFree(d);
        CTX_TRY(e1);
        c->sm_ids = std::max<int>((int)h, c->num_sms);
    }
    c->n_tables = (uint32_t)c->sm_ids * (uint32_t)c->slots_per_sm * kSearchWarps;
    c->n_tables_live = (uint32_t)c->num_sms * (uint32_t)c->slots_per_sm * kSearchWarps;
    cudaDeviceGetAttribute(&c->max_persist, cudaDevAttrMaxPersistingL2CacheSize, device);
    cudaDeviceGetAttribute(&c->max_window, cudaDevAttrMaxAccessPolicyWindowSize, device);
    // The persisting-L2 set-aside is off unless asked for: on an H100 it takes most of the 50 MB L2 away from the graph's rows and
    // adjacency, and K1 at the headline config ran 2.4x slower with it than with the tables cached like any other data.
    c->l2_allowed = g_l2_pref[device] > 0;
    if (const char* e = std::getenv("IDB_L2_PERSIST"); e && g_l2_pref[device] == 0) c->l2_allowed = std::atoi(e) != 0;
    // b16 tables: two segments of `b16_l2_bytes` per warp.  The first — as many bytes per warp as keep ALL live tables inside the
    // persisting part of L2 (the device's maximum persisting size over 132 SMs x 16 warps on an H100) and the pool inside one
    // access-policy window — is what normal
    // traversals use; the second serves large ef (up to 2040 buckets over both: the per-row tally has 2048 one-byte entries).
    size_t per = c->max_persist > 0 ? (size_t)c->max_persist / c->n_tables_live : (size_t)32 * 1024;
    per = std::min<size_t>(std::max<size_t>(per / 512 * 512, 8 * 1024), 32 * 1024);
    c->b16_l2_bytes = (uint32_t)per;
    c->b16_stride = (uint32_t)(per / 4);
    CTX_TRY(cudaMalloc(&c->slot_masks, ((size_t)c->sm_ids + 1) * 4));
    CTX_TRY(cudaMemset(c->slot_masks, 0, ((size_t)c->sm_ids + 1) * 4));
    CTX_TRY(cudaMalloc(&c->b16_tables, (size_t)c->n_tables * per));
    CTX_TRY(cudaMemset(c->b16_tables, 0xFF, (size_t)c->n_tables * per));
    CTX_TRY(cudaMalloc(&c->b16_ext, (size_t)c->n_tables * per));
    CTX_TRY(cudaMemset(c->b16_ext, 0xFF, (size_t)c->n_tables * per));
    const size_t retry_words = (size_t)kRetryCtas * kSearchWarps * kRetrySlots;
    CTX_TRY(cudaMalloc(&c->retry_tables, retry_words * 4));
    CTX_TRY(cudaMemset(c->retry_tables, 0xFF, retry_words * 4));
    CTX_TRY(cudaMalloc(&c->tie_tables, (size_t)c->n_tables * kTieCap * 8));
    CTX_TRY(cudaMalloc(&c->retry_ties, (size_t)kRetryCtas * kSearchWarps * kRetryTieCap * 8));
    CTX_TRY(cudaDeviceSynchronize());
#undef CTX_TRY
    c->refs = 1;
    g_ctx[device] = c;
    *out = c;
    return IDB_OK;
}

void DeviceCtx::release(DeviceCtx* c) {
    if (!c) return;
    std::lock_guard<std::mutex> lk(g_ctx_mu);
    if (--c->refs > 0) return;
    g_ctx[c->device] = nullptr;
    delete c;
}

DeviceCtx::~DeviceCtx() {
    cudaSetDevice(device);
    cudaDeviceSynchronize();
    if (l2_reserved) {  // hand the persisting lines and the device's L2 set-aside back
        cudaCtxResetPersistingL2Cache();
        cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, 0);
    }
    cudaFree(slot_masks);
    cudaFree(b16_tables);
    cudaFree(b16_ext);
    cudaFree(big_tables);
    cudaFree(retry_tables);
    cudaFree(tie_tables);
    cudaFree(retry_ties);
}

idb_status DeviceCtx::ensure_big(uint32_t stride_words) {
    if (big_tables && stride_words <= big_stride) return IDB_OK;
    CUDA_TRY(cudaDeviceSynchronize());  // nobody may be using the old tables (enqueues are serialised by mu)
    cudaFree(big_tables);
    big_tables = nullptr;
    big_stride = 0;
    const size_t words = (size_t)n_tables * stride_words;
    CUDA_TRY(cudaMalloc(&big_tables, words * 4));
    CUDA_TRY(cudaMemset(big_tables, 0xFF, words * 4));
    CUDA_TRY(cudaDeviceSynchronize());
    big_stride = stride_words;
    return IDB_OK;
}

idb_status DeviceCtx::reserve_l2(size_t bytes) {
    if (!l2_allowed || max_persist <= 0 || max_window <= 0) return IDB_OK;
    bytes = std::min<size_t>(bytes, (size_t)max_persist);
    if (bytes <= l2_reserved) return IDB_OK;
    CUDA_TRY(cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, bytes));
    l2_reserved = bytes;
    return IDB_OK;
}

static bool host_ptr_is_pinned(const void* p) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return at.type == cudaMemoryTypeHost || at.type == cudaMemoryTypeManaged;
}

// Output buffers in pinned (or registered) host memory receive the copies directly.  Pageable buffers do NOT, and neither do the
// control blocks: a device-to-pageable cudaMemcpyAsync blocks inside the driver until the copy has run (i.e. until this call's K1 has
// finished) and stalls the launches of other caller threads meanwhile — concurrent callers would never have a second batch queued
// behind the running one.  Those results are staged in the lane's pinned buffer and copied out after the stream has been synchronised.
idb_status copy_to_host(Lane& ln, const HostCopy* parts, int n_parts, const std::function<cudaError_t()>& also) {
    bool staged = false;
    size_t total = 0;
    size_t off[4] = {};
    for (int i = 0; i < n_parts; ++i) {
        if (!parts[i].user) continue;
        staged = staged || !host_ptr_is_pinned(parts[i].user);
        off[i] = total;
        total += (parts[i].bytes + 63) / 64 * 64;
    }
    if (staged && total > ln.h_out_cap) {
        if (ln.h_out) cudaFreeHost(ln.h_out);
        ln.h_out = nullptr;
        ln.h_out_cap = 0;
        CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(&ln.h_out), total + total / 4, cudaHostAllocDefault));
        ln.h_out_cap = total + total / 4;
    }
    for (int i = 0; i < n_parts; ++i)
        if (parts[i].user)
            CUDA_TRY(cudaMemcpyAsync(staged ? static_cast<void*>(ln.h_out + off[i]) : parts[i].user, parts[i].dev, parts[i].bytes,
                                     cudaMemcpyDeviceToHost, ln.stream));
    if (also) CUDA_TRY(also());
    CUDA_TRY(cudaStreamSynchronize(ln.stream));
    for (int i = 0; i < n_parts; ++i)
        if (staged && parts[i].user) std::memcpy(parts[i].user, ln.h_out + off[i], parts[i].bytes);
    return IDB_OK;
}

idb_status read_back(Lane& ln, uint64_t nq, uint32_t k, uint32_t* out_ids, float* out_dist, uint32_t* out_len, Lane* const* ctrl_lanes,
                     uint32_t n_ctrl) {
    const HostCopy parts[3] = {{out_ids, ln.ids, nq * k * 4}, {out_dist, ln.dist, nq * k * 4}, {out_len, ln.len, nq * 4}};
    const idb_status st = copy_to_host(ln, parts, 3, [&]() {
        for (uint32_t i = 0; i < n_ctrl; ++i)
            if (ctrl_lanes[i]->last_nq) {
                const cudaError_t e = cudaMemcpyAsync(ctrl_lanes[i]->h_ctrl + 1, ctrl_lanes[i]->ctrl, sizeof(SearchCtrl),
                                                      cudaMemcpyDeviceToHost, ln.stream);
                if (e != cudaSuccess) return e;
            }
        return cudaSuccess;
    });
    if (st != IDB_OK) return st;
    uint64_t failed = 0;  // failures that survived the retry pass
    for (uint32_t i = 0; i < n_ctrl; ++i)
        if (ctrl_lanes[i]->last_nq) failed += ctrl_lanes[i]->h_ctrl[1].retry.fail_count;
    if (failed)
        return fail(IDB_ERR_CAPACITY, "%llu traversals of %llu queries overflowed an internal per-query structure (visited table / tie list)",
                    (unsigned long long)failed, (unsigned long long)nq);
    return IDB_OK;
}

idb_status require_device(int* count) {
    int c = 0;
    cudaError_t e = cudaGetDeviceCount(&c);
    if (e != cudaSuccess || c == 0)
        return fail(IDB_ERR_CUDA, "no CUDA device available (%s); this library has no CPU fallback",
                    e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    if (count) *count = c;
    return IDB_OK;
}

idb_status check_search_args(Family f, idb_index* const* shards, uint32_t n_shards, const void* comm, const uint32_t* lane,
                             const void* queries, uint64_t nq, const void* out_ids, uint32_t k, const RangeCheck* rc) {
    if (f == Family::sharded && !comm) return fail(IDB_ERR_INVALID_ARG, "comm is null");
    if (f != Family::sharded && !shards[0]) return fail(IDB_ERR_INVALID_ARG, "index is null");
    if (f == Family::range) {
        if (nq > 0 && (!queries || !out_ids)) return fail(IDB_ERR_INVALID_ARG, "queries/out_offsets is null");
        if (rc->capacity > 0 && !rc->ids)
            return fail(IDB_ERR_INVALID_ARG, "out_ids is null with capacity %llu", (unsigned long long)rc->capacity);
        if (std::isnan(rc->radius)) return fail(IDB_ERR_INVALID_ARG, "radius is NaN");
        if (rc->ef_search > kMaxEf) return fail(IDB_ERR_INVALID_ARG, "ef_search %u is not 0 or 1..%u", rc->ef_search, kMaxEf);
        if (rc->device && !rc->out_total) return fail(IDB_ERR_INVALID_ARG, "out_total is null");
        if (rc->capacity > kRangeMaxCapacity || nq >= kRangeMaxCapacity)
            return fail(IDB_ERR_UNSUPPORTED, "the range search takes a capacity of at most %llu and fewer queries (capacity %llu, nq %llu)",
                        (unsigned long long)kRangeMaxCapacity, (unsigned long long)rc->capacity, (unsigned long long)nq);
    } else {
        if (nq > 0 && (!queries || !out_ids)) return fail(IDB_ERR_INVALID_ARG, "queries/out_ids is null");
        if ((nq > 0 || f == Family::exact) && k == 0) return fail(IDB_ERR_INVALID_ARG, "k must be >= 1");
    }
    if (f == Family::exact && k > kExactMaxK)
        return fail(IDB_ERR_UNSUPPORTED, "k = %u > %u is not supported by the exact search", k, kExactMaxK);
    if (lane && *lane >= (uint32_t)kLanes) return fail(IDB_ERR_INVALID_ARG, "lane %u out of range (0..%d)", *lane, kLanes - 1);
    if (nq == 0) return IDB_OK;
    if (f == Family::sharded) {
        if (!shards || n_shards == 0 || n_shards > 64) return fail(IDB_ERR_INVALID_ARG, "shards: need 1..64 index handles");
        for (uint32_t i = 0; i < n_shards; ++i)
            if (!shards[i]) return fail(IDB_ERR_INVALID_ARG, "shard %u is null", i);
    }
    return require_device();
}

void Lane::free_all() {
    cudaFree(ctrl); cudaFree(status); cudaFree(fail_list); cudaFree(counters);
    cudaFree(q); cudaFree(qn); cudaFree(ids); cudaFree(dist); cudaFree(len);
    cudaFree(keys_local); cudaFree(keys_all); cudaFree(shard_ids); cudaFree(exact_keys);
    cudaFree(range_keys); cudaFree(range_qids); cudaFree(range_seg); cudaFree(range_off); cudaFree(range_tmp);
    cudaFree(gr_seeds); cudaFree(gr_front); cudaFree(gr_vis); cudaFree(gr_ctl); cudaFree(gr_retry);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (ev_ctrl) cudaEventDestroy(ev_ctrl);
    if (h_ctrl) cudaFreeHost(h_ctrl);
    if (h_out) cudaFreeHost(h_out);
    if (stream) cudaStreamDestroy(stream);
}

void Index::note_overflows(uint32_t ef, uint64_t n_work, uint32_t overflowed, int level) {
    if (level < 1 || level > 2) return;
    if ((uint64_t)overflowed * 1000 > n_work) {
        std::atomic<uint32_t>& d = b16_demote_ef[level - 1];
        uint32_t cur = d.load();
        while (ef < cur && !d.compare_exchange_weak(cur, ef)) {}
    }
}

Lane& Index::pick_lane() {
    // prefer an idle lane; otherwise queue behind the next one in rotation
    for (int i = 0; i < kLanes; ++i) {
        Lane& ln = lanes[(next_lane.load() + i) % kLanes];
        if (ln.mu.try_lock()) {
            next_lane.fetch_add(i + 1);
            return ln;
        }
    }
    Lane& ln = lanes[next_lane.fetch_add(1) % kLanes];
    ln.mu.lock();
    return ln;
}

ExclusiveIndex::ExclusiveIndex(Index* index) : ix(index) {
    ix->mu.lock();
    for (auto& ln : ix->lanes) ln.mu.lock();
    drained = cudaSetDevice(ix->device);
    for (auto& ln : ix->lanes)
        if (drained == cudaSuccess) drained = cudaStreamSynchronize(ln.stream);
}

ExclusiveIndex::~ExclusiveIndex() {
    for (auto& ln : ix->lanes) ln.mu.unlock();
    ix->mu.unlock();
}

idb_status Index::last_search(uint32_t lane, bool latest, SearchCtrl* ctrl, uint32_t* kernel) {
    if (latest && lane == 0xFFFFFFFFu) lane = (uint32_t)last_lane.load();
    if (lane >= (uint32_t)kLanes) return fail(IDB_ERR_INVALID_ARG, "lane %u out of range", lane);
    Lane& ln = lanes[lane];
    std::lock_guard<std::mutex> lk(ln.mu);
    if (ctrl) *ctrl = SearchCtrl();
    if (kernel) std::memset(kernel, 0, sizeof(ln.last_kernel));
    if (ln.last_nq == 0) return IDB_OK;
    if (kernel) std::memcpy(kernel, ln.last_kernel, sizeof(ln.last_kernel));
    if (ctrl) {
        CUDA_TRY(cudaSetDevice(device));
        CUDA_TRY(cudaMemcpyAsync(ctrl, ln.ctrl, sizeof(SearchCtrl), cudaMemcpyDeviceToHost, ln.stream));
        CUDA_TRY(cudaStreamSynchronize(ln.stream));
    }
    return IDB_OK;
}

idb_status Index::attach_window(Lane& ln, const LaunchWindow& win) {
    if (ln.win_base == win.base && ln.win_bytes == win.bytes) return IDB_OK;
    cudaStreamAttrValue av;
    std::memset(&av, 0, sizeof(av));
    if (win.base && win.bytes) {
        av.accessPolicyWindow.base_ptr = win.base;
        av.accessPolicyWindow.num_bytes = win.bytes;
        av.accessPolicyWindow.hitRatio = win.hit_ratio;
        av.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
        av.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    }
    CUDA_TRY(cudaStreamSetAttribute(ln.stream, cudaStreamAttributeAccessPolicyWindow, &av));
    ln.win_base = win.base;
    ln.win_bytes = win.bytes;
    return IDB_OK;
}

idb_status Index::ensure_lane_scratch(Lane& ln, uint64_t nq) {
    if (!ln.ctrl) {
        CUDA_TRY(cudaMalloc(&ln.ctrl, sizeof(SearchCtrl)));
        CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(&ln.h_ctrl), 2 * sizeof(SearchCtrl), cudaHostAllocDefault));
        CUDA_TRY(cudaEventCreateWithFlags(&ln.ev_ctrl, cudaEventDisableTiming));
    }
    if (ln.ctrl_pending && cudaEventQuery(ln.ev_ctrl) == cudaSuccess) {  // the previous call's tally has arrived
        note_overflows(ln.ctrl_ef, ln.ctrl_nq, ln.h_ctrl[0].main.fail_count, ln.ctrl_b16);
        ln.ctrl_pending = false;
    }
    CUDA_TRY(ensure(ln.status, ln.status_cap, nq));
    CUDA_TRY(ensure(ln.fail_list, ln.fail_cap, nq));
    CUDA_TRY(ensure(ln.counters, ln.counters_cap, nq * 4));
    if (profiling && !ln.ev0) {
        CUDA_TRY(cudaEventCreate(&ln.ev0));
        CUDA_TRY(cudaEventCreate(&ln.ev1));
    }
    return IDB_OK;
}

// Which flavour of the big visited tier serves a traversal with this ef, and where its tables are.
//   b16 (default): exact while ceil(n / 32768) <= buckets and no adjacency row repeats an id; ~2 u16 slots per id the traversal can
//     possibly visit (2M per expansion, ~ef expansions), clamped to the per-warp stride (= what fits the persisting part of L2);
//   else bitmap (n bits per warp) when that is no bigger than 2x the hash table, else the hash set.
idb_status Index::select_visited_tier(uint32_t ef, VisTier& t, LaunchWindow& win) {
    DeviceCtx& c = *ctx;
    const uint32_t efx = std::max<uint32_t>(ef, 16u);
    // 2.5 u16 slots per id the traversal can possibly insert (2M per expansion, ~ef expansions): typical load 1/3, queries handed to the
    // retry pass beyond 11/16.
    // Tables stay within the L2-resident 32 KB while 0.9 * 2M * ef ids fit below the hand-over point; larger ef uses up to 64 KB.
    const uint64_t want_bytes = ((uint64_t)2 * M * efx * 5 + 511) / 512 * 512;
    const uint32_t seg = c.b16_l2_bytes;                           // bytes per segment
    const uint32_t nb_lo_max = (seg - kB16Stash * 4) / 32;         // the first segment also holds the stash
    // Which flavour:
    //   1. b16 inside the L2-resident first segment while a typical traversal (~0.8 * 2M * ef ids) stays below its hand-over point
    //      (M = 32: up to ef ~ 200) and this index has not been seen to overflow it at this ef;
    //   2. b16 over both segments for BIG indexes only (n > 4M, where the bitmap would be > 512 KB per warp), same conditions;
    //      at 1M points the half-DRAM-resident large table is no faster than the bitmap;
    //   3. bitmap (n bits per warp) when that is no bigger than 2x the hash table, else the hash set.
    auto cap_of = [&](uint32_t buckets) { return (uint64_t)buckets * b16_cap_16ths; };
    const uint64_t typical = (uint64_t)2 * M * efx * 4 / 5;
    int level = 0;
    if (typical <= cap_of(nb_lo_max) && ef < b16_demote_ef[0].load()) level = 1;
    else if (n > 4000000ull && typical <= cap_of(2040u) && ef < b16_demote_ef[1].load()) level = 2;
    uint32_t b16_bytes = (uint32_t)std::min<uint64_t>(want_bytes, level == 2 ? 2ull * seg : seg);
    if (b16_bytes_override) {
        b16_bytes = std::min<uint32_t>(std::max<uint32_t>(b16_bytes_override / 32 * 32, 512u), 2 * seg);
        if (ef < b16_demote_ef[0].load()) level = 1;
    }
    const uint32_t nb = std::min<uint32_t>((b16_bytes - kB16Stash * 4) / 32, 2040u);  // buckets over both segments
    const uint32_t nb_lo = std::min(nb, nb_lo_max);
    const bool b16_exact = graph.rows_distinct && (n + 32767) / 32768 <= nb;
    int tier = vis_tier;
    if (tier == 2 && !b16_exact) tier = -1;
    if (tier < 0) tier = (b16_exact && level > 0) ? 2 : -1;
    b16_level = tier == 2 ? (level > 0 ? level : 1) : 0;
    win = LaunchWindow();
    t = VisTier();
    if (tier == 2) {
        t.pool = c.main_pool(true);
        t.gslots = nb_lo * 8 + kB16Stash;
        t.b16_nb = nb;
        t.mode = kVisB16;
        t.b16_cap_ids = nb * b16_cap_16ths;  // <= 11 of 16 slots on average; fuller tables hand the query to the retry pass
        idb_status st = c.reserve_l2((size_t)c.n_tables_live * std::min(b16_bytes, seg));
        if (st != IDB_OK) return st;
        if (c.l2_reserved) {
            win.base = c.b16_tables;
            win.bytes = std::min<size_t>((size_t)c.n_tables * c.b16_stride * 4, (size_t)c.max_window);
            win.hit_ratio = 1.0f;  // the window covers the first segments only; of those only the bytes in use are ever touched
        }
        return IDB_OK;
    }
    uint32_t want_slots = std::max<uint32_t>(1024u, next_pow2((uint64_t)vis_mult * 2 * M * efx));
    if (vis_slots_override) want_slots = vis_slots_override;  // tests: force the overflow -> retry path
    const uint32_t bm_words = (uint32_t)std::min<uint64_t>(((n + 31) / 32 + 127) / 128 * 128, 0xFFFFFF80u);
    const bool bitmap = tier == 1 || (tier < 0 && !vis_slots_override && (n + 31) / 32 <= 2ull * want_slots);
    idb_status st = c.ensure_big(std::max(want_slots, bitmap ? bm_words : 0u));
    if (st != IDB_OK) return st;
    t.pool = c.main_pool(false);
    t.gslots = bitmap ? bm_words : want_slots;
    t.gshift = 32 - (uint32_t)std::log2((double)want_slots);
    t.mode = bitmap ? kVisBitmap : kVisHash;
    return IDB_OK;
}

int Index::search_grid() const { return num_sms * ctx->slots_per_sm; }

cudaError_t write_empty(cudaStream_t st, uint64_t nq, uint32_t k, uint32_t* ids, float* dist, uint32_t* len, uint64_t* keys) {
    cudaError_t e = fill_u32(ids, nq * k, kInvalid, st);
    if (e == cudaSuccess && dist) e = fill_u32(reinterpret_cast<uint32_t*>(dist), nq * k, 0x7f800000u, st);
    if (e == cudaSuccess && len) e = cudaMemsetAsync(len, 0, nq * 4, st);
    if (e == cudaSuccess && keys) e = cudaMemsetAsync(keys, 0xFF, nq * k * 8, st);  // kKeyNone everywhere
    return e;
}

idb_status Index::stage_queries(Lane& ln, const float* queries, bool host, uint64_t nq, const float** out) {
    const size_t stride = (size_t)nchunks * 4;
    *out = queries;
    if (!host && stride == dim && !(reinterpret_cast<uintptr_t>(queries) & 15)) return IDB_OK;
    CUDA_TRY(ensure(ln.q, ln.q_cap, nq * stride));
    const cudaMemcpyKind kind = host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
    if (stride == dim) {
        CUDA_TRY(cudaMemcpyAsync(ln.q, queries, nq * stride * 4, kind, ln.stream));
    } else {
        CUDA_TRY(cudaMemsetAsync(ln.q, 0, nq * stride * 4, ln.stream));
        CUDA_TRY(cudaMemcpy2DAsync(ln.q, stride * 4, queries, dim * 4, dim * 4, nq, kind, ln.stream));
    }
    *out = ln.q;
    return IDB_OK;
}

idb_status Index::normalize_queries(Lane& ln, const float** q, uint64_t nq) {
    if (metric != kMetricCosine) return IDB_OK;
    CUDA_TRY(ensure(ln.qn, ln.qn_cap, nq * nchunks * 4));
    CUDA_TRY(normalize_rows(*q, (uint64_t)nchunks * 4, ln.qn, nq, dim, nchunks, num_sms, ln.stream));
    *q = ln.qn;
    return IDB_OK;
}

idb_status search_on_lane(Index* ix, Lane& ln, const float* queries, bool staged, uint64_t nq, uint32_t ef_search, uint32_t k,
                          uint32_t* d_ids, float* d_dist, uint32_t* d_len, uint64_t* d_keys, bool map_ids) {
    CUDA_TRY(cudaSetDevice(ix->device));
    const uint32_t ef = ef_search ? ef_search : ix->ef_search;
    if (ix->n == 0 || ef == 0) {  // empty index (core:359-361) / ef_search = 0: empty result lists
        CUDA_TRY(write_empty(ln.stream, nq, k, d_ids, d_dist, d_len, d_keys));
        ln.last_nq = 0;
        return IDB_OK;
    }
    if (!staged) {
        idb_status st = ix->stage_queries(ln, queries, false, nq, &queries);
        if (st != IDB_OK) return st;
    }
    return ix->enqueue_search(ln, queries, nq, ef, k, d_ids, d_dist, d_len, d_keys, map_ids);
}

// Enqueue one batched search on a lane; all pointers are device pointers (d_queries: see internal.cuh).  The caller holds ln.mu.
idb_status Index::enqueue_search(Lane& ln, const float* d_queries, uint64_t nq, uint32_t ef, uint32_t k, uint32_t* d_ids, float* d_dist,
                                 uint32_t* d_len, uint64_t* out_keys, bool map_ids) {
    if (n) ef = (uint32_t)std::min<uint64_t>(ef, n);  // admission is rank < ef and there are only n distinct ids: same results
    if (ef > 1024) return fail(IDB_ERR_UNSUPPORTED, "ef_search %u > 1024 (on an index of more than 1024 points) is not supported", ef);
    idb_status st = ensure_lane_scratch(ln, nq);
    if (st != IDB_OK) return st;
    CUDA_TRY(cudaMemsetAsync(ln.ctrl, 0, sizeof(SearchCtrl), ln.stream));

    SearchArgs a;
    std::memset(&a, 0, sizeof(a));
    a.g = view();
    a.metric = metric;
    a.work.n_work = nq;
    a.work.work_counter = &ln.ctrl->main.work_counter;
    a.work.status = ln.status;
    a.work.fail_count = &ln.ctrl->main.fail_count;
    a.work.fail_list = ln.fail_list;
    a.ef = ef;
    a.k = k;
    a.out_ids = d_ids;
    a.out_dist = d_dist;
    a.out_len = d_len;
    a.counters = ln.counters;
    a.variant = variant;
    a.out_keys = out_keys;
    a.id_map = map_ids ? d_id_map : nullptr;
    a.full_tally = &ln.ctrl->full_fetches;  // K1 and the retry pass both add to it
    std::memset(ln.last_kernel, 0, sizeof(ln.last_kernel));
    a.launched = ln.last_kernel;

    if ((nchunks + 31) / 32 * 512 > 40 * 1024)
        return fail(IDB_ERR_UNSUPPORTED, "dim %u > 10240 is not supported (the query of a long-row traversal lives in shared memory)", dim);
    const int row_t = (int)((2 * M + 31) / 32);
    const int ef_t = (int)((ef + 31) / 32);
    const int grid = std::max(1, (int)std::min<uint64_t>((nq + kSearchWarps - 1) / kSearchWarps, (uint64_t)search_grid()));
    st = normalize_queries(ln, &d_queries, nq);  // once per call: K1 and the retry pass read the same rows
    if (st != IDB_OK) return st;
    a.queries = reinterpret_cast<const float4*>(d_queries);

    std::lock_guard<std::mutex> lk(ctx->mu);  // the tables this launch uses must not be regrown under it
    LaunchWindow win;
    st = select_visited_tier(ef, a.tier, win);
    if (st == IDB_OK) st = attach_window(ln, win);
    if (st != IDB_OK) return st;
    if (profiling) CUDA_TRY(cudaEventRecord(ln.ev0, ln.stream));
    CUDA_TRY(dispatch_search(a, row_t, ef_t, grid, ln.stream, win));
    if (profiling) CUDA_TRY(cudaEventRecord(ln.ev1, ln.stream));
    ln.last_launches = metric == kMetricCosine ? 3 : 2;  // (the query normalisation) + K1 + the (normally idle) retry pass

    SearchArgs r = retry_pass(a, *ctx, &ln.ctrl->retry);
    r.launched = nullptr;  // same instantiation as K1; last_kernel describes the main launch
    CUDA_TRY(dispatch_search(r, row_t, ef_t, kRetryCtas, ln.stream, LaunchWindow()));
    ln.last_b16 = a.tier.mode == kVisB16 ? b16_level : 0;
    if (!ln.ctrl_pending) {  // sample this call's overflow tally (one read-back in flight per lane; evaluated by a later call)
        CUDA_TRY(cudaMemcpyAsync(ln.h_ctrl, ln.ctrl, sizeof(SearchCtrl), cudaMemcpyDeviceToHost, ln.stream));
        CUDA_TRY(cudaEventRecord(ln.ev_ctrl, ln.stream));
        ln.ctrl_pending = true;
        ln.ctrl_b16 = ln.last_b16;
        ln.ctrl_ef = ef;
        ln.ctrl_nq = nq;
    }
    ln.last_nq = nq;
    return IDB_OK;
}

GraphView Index::view() const {
    GraphView g;
    g.points = static_cast<const char*>(d_rows);
    g.row_type = row_type;
    g.nchunks = nchunks;
    g.zero = graph.zero;
    g.upper = graph.upper_ptrs;
    g.n_upper = (uint32_t)graph.upper.size();
    g.M = M;
    g.n = n;
    g.flags = opt_flags;
    g.codes = d_codes;
    g.cwords = code_words(nchunks);
    g.cparams = d_cparams;
    g.cstep = code_step;
    g.cerr = code_err;
    g.hdr = d_hdr;
    g.tail = dim - (nchunks - 1) * 4;
    return g;
}

Index::~Index() {
    cudaSetDevice(device);
    for (auto& ln : lanes)
        if (ln.stream) cudaStreamSynchronize(ln.stream);
    cudaFree(d_rows);
    cudaFree(d_hdr);
    cudaFree(d_codes);
    cudaFree(d_cparams);
    cudaFree(d_id_map);
    for (auto& ln : lanes) ln.free_all();
    DeviceCtx::release(ctx);
}

idb_status Index::init_device(int dev) {
    int count = 0;
    idb_status st = require_device(&count);
    if (st != IDB_OK) return st;
    if (dev < 0 || dev >= count) return fail(IDB_ERR_INVALID_ARG, "device %d out of range (0..%d)", dev, count - 1);
    device = dev;
    CUDA_TRY(cudaSetDevice(dev));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9 || prop.minor != 0)
        return fail(IDB_ERR_CUDA, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", dev, prop.major, prop.minor);
    num_sms = prop.multiProcessorCount;
    st = DeviceCtx::acquire(dev, &ctx);
    if (st != IDB_OK) return st;
    for (auto& ln : lanes) CUDA_TRY(cudaStreamCreateWithFlags(&ln.stream, cudaStreamNonBlocking));
    stream = lanes[0].stream;
    if (const char* e = std::getenv("IDB_OPT")) opt_flags = (uint32_t)std::atoi(e);
    if (const char* e = std::getenv("IDB_VIS_MULT")) vis_mult = std::max(1, std::atoi(e));
    if (const char* e = std::getenv("IDB_VARIANT")) variant = std::atoi(e);
    if (const char* e = std::getenv("IDB_VIS_TIER")) vis_tier = std::atoi(e);
    if (const char* e = std::getenv("IDB_RETRY_SLOTS")) retry_slots_override = std::min(kRetrySlots, next_pow2((uint64_t)std::max(64, std::atoi(e))));
    if (const char* e = std::getenv("IDB_B16_CAP")) b16_cap_16ths = (uint32_t)std::min(14, std::max(1, std::atoi(e)));
    if (const char* e = std::getenv("IDB_B16_BYTES")) b16_bytes_override = (uint32_t)std::max(64, std::atoi(e));
    if (const char* e = std::getenv("IDB_VIS_SLOTS")) vis_slots_override = next_pow2((uint64_t)std::max(64, std::atoi(e)));
    if (const char* e = std::getenv("IDB_SCREEN")) screen = std::atoi(e) != 0;
    if (const char* e = std::getenv("IDB_EXACT_SCRATCH_KEYS")) exact_scratch_keys = (uint64_t)std::max(1LL, std::atoll(e));
    if (const char* e = std::getenv("IDB_GRAPH_RANGE_SCRATCH")) graph_range_scratch = (uint32_t)std::min(1 << 20, std::max(1, std::atoi(e)));
    return IDB_OK;
}

// idb_index_from_graph_ex.  from_file (idb_index_load_storage): a graph or row the checks refuse makes the file malformed
// (IDB_ERR_FORMAT); rows beyond the range of the storage asked for stay IDB_ERR_INVALID_ARG, as for an adopted graph.
idb_status adopt_graph(const float* points, uint64_t n, uint32_t dim, uint32_t M, uint32_t ef_search, const uint32_t* zero,
                       uint32_t n_upper, const uint32_t* const* upper, const uint64_t* upper_n, uint32_t storage, uint32_t metric,
                       int32_t device, idb_index** out_index, bool from_file) {
    if (!out_index) return fail(IDB_ERR_INVALID_ARG, "out_index is null");
    *out_index = nullptr;
    Index* ix = nullptr;
    idb_status st = [&]() -> idb_status {
        if (dim == 0) return fail(IDB_ERR_INVALID_ARG, "dim must be >= 1");
        if (M < 2 || M > 64) return fail(IDB_ERR_INVALID_ARG, "M = %u unsupported (2..64)", M);
        if (n >= 0xFFFFFFFFull) return fail(IDB_ERR_INVALID_ARG, "N = %llu >= u32::MAX (lib.rs:256)", (unsigned long long)n);
        if (n && (!points || !zero)) return fail(IDB_ERR_INVALID_ARG, "points/zero is null");
        if (n_upper > 31) return fail(IDB_ERR_INVALID_ARG, "too many layers");
        if (n_upper && (!upper || !upper_n)) return fail(IDB_ERR_INVALID_ARG, "upper/upper_n is null");
        if (!storage_known(storage)) return fail(IDB_ERR_INVALID_ARG, "unknown storage %u", storage);
        if (metric != IDB_METRIC_L2SQ && metric != IDB_METRIC_COSINE) return fail(IDB_ERR_INVALID_ARG, "unknown metric %u", metric);
        if (idb_status s = check_storage_metric(storage, metric); s != IDB_OK) return s;
        if (metric == IDB_METRIC_COSINE) {
            // Adopted rows are stored as given (normalising is not idempotent bit for bit), so they must already be unit rows; the
            // tolerance lets bf16- and fp16-rounded and q8-quantised unit rows through.
            for (uint64_t r = 0; r < n; ++r) {
                const float* x = points + r * dim;
                double s = 0.0;
                bool all_zero = true;
                for (uint32_t i = 0; i < dim; ++i) {
                    s += (double)x[i] * x[i];
                    all_zero = all_zero && x[i] == 0.f;
                }
                if (!all_zero && !(std::fabs(s - 1.0) <= 1e-2))
                    return fail(IDB_ERR_INVALID_ARG, "cosine index: row %llu has squared norm %g; rows must be unit length or all zeros "
                                "(idb_normalize_f32 gives the canonical normalisation)", (unsigned long long)r, s);
            }
        }
        ix = new (std::nothrow) Index();
        if (!ix) return fail(IDB_ERR_OOM, "host allocation failed");
        ix->metric = metric;
        ix->row_type = storage;
        idb_status s = ix->init_device(device);
        if (s == IDB_OK) s = ix->upload(n, dim, M, ef_search, zero, n_upper, upper, upper_n);
        return s;
    }();
    if (st == IDB_ERR_INVALID_ARG && from_file) st = IDB_ERR_FORMAT;
    if (st == IDB_OK)  // the rows as given; fp16 / q8 / bin rows beyond the storage's range are refused, named by their row in the call
        st = ix->put_rows(0, n, nullptr, [&](float* dst) { return ix->copy_rows_in(dst, points, n); });
    if (st == IDB_OK) st = ix->build_codes();
    if (st != IDB_OK) {
        delete ix;
        return st;
    }
    *out_index = reinterpret_cast<idb_index*>(ix);
    return IDB_OK;
}

}  // namespace idb

using namespace idb;

// =========================================================================================================
// extern "C"
// =========================================================================================================
extern "C" {

const char* idb_last_error(void) { return g_err; }
const char* idb_version(void) { return "instant-distance-b200 0.1.0 (sm_90a)"; }

int32_t idb_device_count(void) {
    int c = 0;
    if (cudaGetDeviceCount(&c) != cudaSuccess) return 0;
    return c;
}

idb_status idb_params_default(idb_params* p) {
    if (!p) return fail(IDB_ERR_INVALID_ARG, "params is null");
    p->M = 32;                               // core:787
    p->ef_construction = 100;                // core:105
    p->ef_search = 100;                      // core:104
    p->ml = 1.0f / std::log((float)32);      // core:107
    p->seed = 0;                             // core:108 draws from entropy; the C ABI makes it explicit
    p->heuristic = 1;                        // core:106
    p->extend_candidates = 0;                // core:124
    p->keep_pruned = 1;                      // core:125
    p->insert_batch = 0;
    p->device = 0;
    p->storage = IDB_STORAGE_F32;
    p->progress = nullptr;
    p->progress_user = nullptr;
    return IDB_OK;
}

idb_status idb_index_from_graph_ex(const float* points, uint64_t n, uint32_t dim, uint32_t M, uint32_t ef_search, const uint32_t* zero,
                                   uint32_t n_upper, const uint32_t* const* upper, const uint64_t* upper_n, uint32_t storage,
                                   uint32_t metric, int32_t device, idb_index** out_index) {
    return adopt_graph(points, n, dim, M, ef_search, zero, n_upper, upper, upper_n, storage, metric, device, out_index, false);
}

idb_status idb_index_from_graph_f32(const float* points, uint64_t n, uint32_t dim, uint32_t M, uint32_t ef_search,
                                    const uint32_t* zero, uint32_t n_upper, const uint32_t* const* upper,
                                    const uint64_t* upper_n, int32_t device, idb_index** out_index) {
    return idb_index_from_graph_ex(points, n, dim, M, ef_search, zero, n_upper, upper, upper_n, IDB_STORAGE_F32, IDB_METRIC_L2SQ, device,
                                   out_index);
}

idb_status idb_index_from_graph_bf16(const float* points, uint64_t n, uint32_t dim, uint32_t M, uint32_t ef_search,
                                     const uint32_t* zero, uint32_t n_upper, const uint32_t* const* upper,
                                     const uint64_t* upper_n, int32_t device, idb_index** out_index) {
    return idb_index_from_graph_ex(points, n, dim, M, ef_search, zero, n_upper, upper, upper_n, IDB_STORAGE_BF16, IDB_METRIC_L2SQ, device,
                                   out_index);
}

}  // extern "C"

extern "C" {

idb_status idb_search_batch_device_lane(idb_index* index, uint32_t lane, const float* d_queries, uint64_t nq, uint32_t ef_search,
                                        uint32_t k, uint32_t* d_out_ids, float* d_out_dist, uint32_t* d_out_len) {
    idb_status st = check_search_args(Family::approx, &index, 1, nullptr, &lane, d_queries, nq, d_out_ids, k);
    if (st != IDB_OK || nq == 0) return st;
    Index* ix = reinterpret_cast<Index*>(index);
    Lane& ln = ix->lanes[lane];
    std::lock_guard<std::mutex> lk(ln.mu);
    ix->last_lane.store((int)lane);
    return search_on_lane(ix, ln, d_queries, false, nq, ef_search, k, d_out_ids, d_out_dist, d_out_len, nullptr);
}

idb_status idb_search_batch_device(idb_index* index, const float* d_queries, uint64_t nq, uint32_t ef_search, uint32_t k,
                                   uint32_t* d_out_ids, float* d_out_dist, uint32_t* d_out_len) {
    return idb_search_batch_device_lane(index, 0, d_queries, nq, ef_search, k, d_out_ids, d_out_dist, d_out_len);
}

idb_status idb_search_batch_f32(idb_index* index, const float* queries, uint64_t nq, uint32_t ef_search, uint32_t k,
                                uint32_t* out_ids, float* out_dist, uint32_t* out_len) {
    idb_status st = check_search_args(Family::approx, &index, 1, nullptr, nullptr, queries, nq, out_ids, k);
    if (st != IDB_OK || nq == 0) return st;
    Index* ix = reinterpret_cast<Index*>(index);
    const uint32_t ef = ef_search ? ef_search : ix->ef_search;
    if (ix->n == 0 || ef == 0) {
        for (uint64_t i = 0; i < nq * k; ++i) out_ids[i] = IDB_INVALID;
        if (out_dist) for (uint64_t i = 0; i < nq * k; ++i) out_dist[i] = INFINITY;
        if (out_len) std::memset(out_len, 0, nq * 4);
        return IDB_OK;
    }
    // Hnsw<P>: Sync (core:352-356): any number of host threads may search at once; each call takes an idle lane (own stream and
    // control state), so concurrent callers overlap on the device instead of serialising.
    Lane& ln = ix->pick_lane();
    std::lock_guard<std::mutex> lk(ln.mu, std::adopt_lock);
    ix->last_lane.store((int)(&ln - ix->lanes));
    CUDA_TRY(cudaSetDevice(ix->device));
    CUDA_TRY(ensure(ln.ids, ln.ids_cap, nq * k));
    CUDA_TRY(ensure(ln.dist, ln.dist_cap, nq * k));
    CUDA_TRY(ensure(ln.len, ln.len_cap, nq));
    const float* qp = nullptr;
    st = ix->stage_queries(ln, queries, true, nq, &qp);
    if (st == IDB_OK) st = ix->enqueue_search(ln, qp, nq, ef, k, ln.ids, ln.dist, ln.len, nullptr);
    if (st != IDB_OK) return st;
    Lane* lp = &ln;
    st = read_back(ln, nq, k, out_ids, out_dist, out_len, &lp, 1);
    if (st == IDB_OK || st == IDB_ERR_CAPACITY) ix->note_overflows(ef, nq, ln.h_ctrl[1].main.fail_count, ln.last_b16);
    return st;
}

idb_status idb_last_search_failures(idb_index* index, uint32_t lane, uint32_t* out_failed) {
    if (!index || !out_failed) return fail(IDB_ERR_INVALID_ARG, "null argument");
    SearchCtrl c;
    idb_status st = reinterpret_cast<Index*>(index)->last_search(lane, false, &c, nullptr);
    if (st == IDB_OK) *out_failed = c.retry.fail_count;
    return st;
}

idb_status idb_last_search_retried(idb_index* index, uint32_t lane, uint32_t* out_retried) {
    if (!index || !out_retried) return fail(IDB_ERR_INVALID_ARG, "null argument");
    SearchCtrl c;
    idb_status st = reinterpret_cast<Index*>(index)->last_search(lane, true, &c, nullptr);
    if (st == IDB_OK) *out_retried = c.main.fail_count;
    return st;
}

idb_status idb_last_search_kernel(idb_index* index, uint32_t lane, uint32_t* out) {
    if (!index || !out) return fail(IDB_ERR_INVALID_ARG, "null argument");
    return reinterpret_cast<Index*>(index)->last_search(lane, true, nullptr, out);
}

idb_status idb_last_search_counters(idb_index* index, uint64_t nq, uint64_t* out) {
    if (!index || !out) return fail(IDB_ERR_INVALID_ARG, "null argument");
    Index* ix = reinterpret_cast<Index*>(index);
    Lane& ln = ix->lanes[ix->last_lane.load()];
    std::lock_guard<std::mutex> lk(ln.mu);
    if (nq > ln.last_nq) return fail(IDB_ERR_INVALID_ARG, "nq exceeds the last search batch (%llu)", (unsigned long long)ln.last_nq);
    CUDA_TRY(cudaSetDevice(ix->device));
    std::vector<uint32_t> tmp(nq * 4);
    CUDA_TRY(cudaMemcpyAsync(tmp.data(), ln.counters, nq * 16, cudaMemcpyDeviceToHost, ln.stream));
    CUDA_TRY(cudaStreamSynchronize(ln.stream));
    for (uint64_t i = 0; i < nq * 4; ++i) out[i] = tmp[i];
    return IDB_OK;
}

idb_status idb_index_info(const idb_index* index, idb_info* out) {
    if (!index || !out) return fail(IDB_ERR_INVALID_ARG, "null argument");
    const Index* ix = reinterpret_cast<const Index*>(index);
    std::memset(out, 0, sizeof(*out));
    const uint64_t n = ix->n;  // one read: an insert on another thread may change it
    out->n = n;
    out->dim = ix->dim;
    out->M = ix->M;
    out->ef_search = ix->ef_search;
    out->device = ix->device;
    out->storage = ix->row_type;
    out->n_layers = n == 0 ? 0 : (uint32_t)ix->graph.upper.size() + 1;
    if (n) out->layer_n[0] = n;
    for (size_t l = 0; l < ix->graph.upper_n.size() && l + 1 < 32; ++l) out->layer_n[l + 1] = ix->graph.upper_n[l];
    return IDB_OK;
}

idb_status idb_index_export_points(const idb_index* index, float* out) {
    if (!index || !out) return fail(IDB_ERR_INVALID_ARG, "null argument");
    Index* ix = const_cast<Index*>(reinterpret_cast<const Index*>(index));
    if (ix->n == 0) return IDB_OK;
    std::lock_guard<std::mutex> lk(ix->mu);
    CUDA_TRY(cudaSetDevice(ix->device));
    idb_status st = ix->copy_points_f32(out, 0, ix->n);
    if (st != IDB_OK) return st;
    return IDB_OK;
}

idb_status idb_index_export_zero(const idb_index* index, uint32_t* out) {
    if (!index || !out) return fail(IDB_ERR_INVALID_ARG, "null argument");
    Index* ix = const_cast<Index*>(reinterpret_cast<const Index*>(index));
    if (ix->n == 0) return IDB_OK;
    std::lock_guard<std::mutex> lk(ix->mu);
    CUDA_TRY(cudaSetDevice(ix->device));
    CUDA_TRY(ix->graph.copy_out(0, 0, ix->n, ix->M, out, ix->stream));
    return IDB_OK;
}

idb_status idb_index_export_upper(const idb_index* index, uint32_t layer, uint32_t* out) {
    if (!index || !out) return fail(IDB_ERR_INVALID_ARG, "null argument");
    Index* ix = const_cast<Index*>(reinterpret_cast<const Index*>(index));
    std::lock_guard<std::mutex> lk(ix->mu);  // before the layer count: a removal can drop layers
    if (layer == 0 || layer > ix->graph.upper.size()) return fail(IDB_ERR_INVALID_ARG, "layer %u out of range", layer);
    CUDA_TRY(cudaSetDevice(ix->device));
    CUDA_TRY(ix->graph.copy_out(layer, 0, ix->graph.upper_n[layer - 1], ix->M, out, ix->stream));
    return IDB_OK;
}

idb_status idb_index_set_profiling(idb_index* index, int32_t enabled) {
    if (!index) return fail(IDB_ERR_INVALID_ARG, "index is null");
    Index* ix = reinterpret_cast<Index*>(index);
    ix->profiling = enabled != 0;  // the events are created by the next call on each lane
    return IDB_OK;
}

idb_status idb_index_last_kernel_ms(idb_index* index, float* out_ms, uint32_t* out_launches) {
    if (!index || !out_ms) return fail(IDB_ERR_INVALID_ARG, "null argument");
    Index* ix = reinterpret_cast<Index*>(index);
    Lane& ln = ix->lanes[ix->last_lane.load()];
    std::lock_guard<std::mutex> lk(ln.mu);
    if (!ix->profiling || !ln.ev0) return fail(IDB_ERR_INVALID_ARG, "profiling is not enabled on this index");
    CUDA_TRY(cudaSetDevice(ix->device));
    CUDA_TRY(cudaEventSynchronize(ln.ev1));
    CUDA_TRY(cudaEventElapsedTime(out_ms, ln.ev0, ln.ev1));
    if (out_launches) *out_launches = ln.last_launches;
    return IDB_OK;
}

void* idb_index_stream(idb_index* index) { return index ? reinterpret_cast<Index*>(index)->stream : nullptr; }
uint32_t idb_index_num_lanes(void) { return (uint32_t)kLanes; }
void* idb_index_lane_stream(idb_index* index, uint32_t lane) {
    return index && lane < (uint32_t)kLanes ? reinterpret_cast<Index*>(index)->lanes[lane].stream : nullptr;
}

idb_status idb_index_sync(idb_index* index) {
    if (!index) return fail(IDB_ERR_INVALID_ARG, "index is null");
    Index* ix = reinterpret_cast<Index*>(index);
    CUDA_TRY(cudaSetDevice(ix->device));
    for (auto& ln : ix->lanes) CUDA_TRY(cudaStreamSynchronize(ln.stream));
    return IDB_OK;
}

idb_status idb_device_set_persisting_l2(int32_t device, int32_t enabled) {
    if (device < 0 || device >= 64) return fail(IDB_ERR_INVALID_ARG, "device %d out of range", device);
    std::lock_guard<std::mutex> lk(g_ctx_mu);
    g_l2_pref[device] = enabled ? 1 : -1;
    if (g_ctx[device]) {
        std::lock_guard<std::mutex> lk2(g_ctx[device]->mu);
        g_ctx[device]->l2_allowed = enabled != 0;
        if (!enabled && g_ctx[device]->l2_reserved) {
            CUDA_TRY(cudaSetDevice(device));
            CUDA_TRY(cudaDeviceSynchronize());
            cudaCtxResetPersistingL2Cache();
            CUDA_TRY(cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, 0));
            g_ctx[device]->l2_reserved = 0;
        }
    }
    return IDB_OK;
}

void idb_index_free(idb_index* index) { delete reinterpret_cast<Index*>(index); }

idb_status idb_distance_f32(const float* a, const float* b, uint32_t dim, int32_t device, float* out) {
    if (!a || !b || !out || dim == 0) return fail(IDB_ERR_INVALID_ARG, "null argument or dim == 0");
    idb_status st = require_device();
    if (st != IDB_OK) return st;
    CUDA_TRY(cudaSetDevice(device));
    const uint32_t nchunks = (dim + 3) / 4;
    float* d = nullptr;
    CUDA_TRY(cudaMalloc(&d, (2 * (size_t)nchunks * 4 + 4) * sizeof(float)));
    cudaMemset(d, 0, (2 * (size_t)nchunks * 4 + 4) * sizeof(float));
    cudaMemcpy(d, a, dim * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(d + nchunks * 4, b, dim * 4, cudaMemcpyHostToDevice);
    distance_kernel<<<1, 32>>>(reinterpret_cast<const float4*>(d), reinterpret_cast<const float4*>(d + nchunks * 4), nchunks,
                               d + 2 * (size_t)nchunks * 4);
    cudaError_t e = cudaMemcpy(out, d + 2 * (size_t)nchunks * 4, 4, cudaMemcpyDeviceToHost);
    cudaFree(d);
    if (e != cudaSuccess) return fail(IDB_ERR_CUDA, "CUDA error: %s", cudaGetErrorString(e));
    return IDB_OK;
}

idb_status idb_normalize_f32(const float* rows, uint64_t n, uint32_t dim, int32_t device, float* out) {
    if (dim == 0 || (n && (!rows || !out))) return fail(IDB_ERR_INVALID_ARG, "null argument or dim == 0");
    int count = 0;
    idb_status st = require_device(&count);
    if (st != IDB_OK) return st;
    if (device < 0 || device >= count) return fail(IDB_ERR_INVALID_ARG, "device %d out of range (0..%d)", device, count - 1);
    if (n == 0) return IDB_OK;
    CUDA_TRY(cudaSetDevice(device));
    int num_sms = 0;
    CUDA_TRY(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
    const uint32_t nchunks = (dim + 3) / 4;
    const size_t in_floats = n * (size_t)dim, in_padded = (in_floats + 3) / 4 * 4, out_floats = n * (size_t)nchunks * 4;
    float* d = nullptr;
    CUDA_TRY(cudaMalloc(&d, (in_padded + out_floats) * sizeof(float)));
    float* d_out = d + in_padded;  // 16-byte aligned
    cudaError_t e = cudaMemcpy(d, rows, in_floats * sizeof(float), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = normalize_rows(d, dim, d_out, n, dim, nchunks, num_sms, 0);
    if (e == cudaSuccess) e = cudaMemcpy2D(out, dim * sizeof(float), d_out, nchunks * 4 * sizeof(float), dim * sizeof(float), n, cudaMemcpyDeviceToHost);
    cudaFree(d);
    if (e != cudaSuccess) return fail(IDB_ERR_CUDA, "CUDA error: %s", cudaGetErrorString(e));
    return IDB_OK;
}

idb_status idb_index_metric(const idb_index* index, uint32_t* out) {
    if (!index || !out) return fail(IDB_ERR_INVALID_ARG, "null argument");
    *out = reinterpret_cast<const Index*>(index)->metric;
    return IDB_OK;
}

idb_status idb_host_alloc(size_t bytes, void** out) {
    if (!out) return fail(IDB_ERR_INVALID_ARG, "out is null");
    cudaError_t e = cudaHostAlloc(out, bytes, cudaHostAllocDefault);
    if (e != cudaSuccess) return fail(IDB_ERR_OOM, "cudaHostAlloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
    return IDB_OK;
}
void idb_host_free(void* p) { if (p) cudaFreeHost(p); }

}  // extern "C"
