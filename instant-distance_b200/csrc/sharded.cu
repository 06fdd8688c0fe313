// sharded.cu — the index sharded by PointId range across the GPUs of one box (SURVEY §8e, BASELINE config 5).
//
// One process per GPU.  Every rank owns an independent HNSW over its contiguous range of the input rows (own shuffle, own
// PointId space, own entry point); every query is searched on every shard with the same ef; then ONE ncclAllGather of the
// per-shard top-k — packed as u64 keys (canonical distance bits << 32 | global row id) by K1's epilogue — and a merge
// kernel that keeps the k smallest keys of the union, ties broken by the lower global id.  No other collective anywhere.
// NCCL is bound at run time (dlopen of libnccl.so.2: the system 2.27 or whichever copy the host application already loaded).
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstring>
#include <vector>

#include "internal.cuh"

namespace idb {

namespace {

struct NcclApi {
    void* handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
};

NcclApi& nccl() {
    static NcclApi api = [] {
        NcclApi a;
        const char* names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char* n : names) {
            a.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (a.handle) break;
        }
        if (!a.handle) return a;
        a.GetUniqueId = reinterpret_cast<decltype(a.GetUniqueId)>(dlsym(a.handle, "ncclGetUniqueId"));
        a.CommInitRank = reinterpret_cast<decltype(a.CommInitRank)>(dlsym(a.handle, "ncclCommInitRank"));
        a.CommDestroy = reinterpret_cast<decltype(a.CommDestroy)>(dlsym(a.handle, "ncclCommDestroy"));
        a.AllGather = reinterpret_cast<decltype(a.AllGather)>(dlsym(a.handle, "ncclAllGather"));
        a.GetErrorString = reinterpret_cast<decltype(a.GetErrorString)>(dlsym(a.handle, "ncclGetErrorString"));
        a.ok = a.GetUniqueId && a.CommInitRank && a.CommDestroy && a.AllGather && a.GetErrorString;
        return a;
    }();
    return api;
}

#define NCCL_TRY(expr)                                                                                                   \
    do {                                                                                                                 \
        ncclResult_t r__ = (expr);                                                                                       \
        if (r__ != ncclSuccess) return ::idb::fail(IDB_ERR_NCCL, "NCCL error at %s:%d: %s", __FILE__, __LINE__, nccl().GetErrorString(r__)); \
    } while (0)

}  // namespace

struct Comm {
    ncclComm_t comm = nullptr;
    int rank = 0, world = 1, device = 0;
};

}  // namespace idb

using namespace idb;

extern "C" {

idb_status idb_comm_unique_id(void* out) {
    if (!out) return fail(IDB_ERR_INVALID_ARG, "out is null");
    if (!nccl().ok) return fail(IDB_ERR_NCCL, "libnccl.so.2 could not be loaded (%s)", dlerror() ? dlerror() : "symbols missing");
    static_assert(IDB_UNIQUE_ID_BYTES == NCCL_UNIQUE_ID_BYTES, "unique id size");
    ncclUniqueId id;
    NCCL_TRY(nccl().GetUniqueId(&id));
    std::memcpy(out, &id, sizeof(id));
    return IDB_OK;
}

idb_status idb_comm_create(const void* unique_id, int32_t rank, int32_t world, int32_t device, idb_comm** out) {
    if (!unique_id || !out) return fail(IDB_ERR_INVALID_ARG, "null argument");
    *out = nullptr;
    if (world < 1 || rank < 0 || rank >= world) return fail(IDB_ERR_INVALID_ARG, "rank %d / world %d invalid", rank, world);
    if (!nccl().ok) return fail(IDB_ERR_NCCL, "libnccl.so.2 could not be loaded");
    CUDA_TRY(cudaSetDevice(device));
    auto* c = new (std::nothrow) Comm();
    if (!c) return fail(IDB_ERR_OOM, "host allocation failed");
    c->rank = rank;
    c->world = world;
    c->device = device;
    ncclUniqueId id;
    std::memcpy(&id, unique_id, sizeof(id));
    ncclResult_t r = nccl().CommInitRank(&c->comm, world, id, rank);
    if (r != ncclSuccess) {
        delete c;
        return fail(IDB_ERR_NCCL, "ncclCommInitRank failed: %s", nccl().GetErrorString(r));
    }
    *out = reinterpret_cast<idb_comm*>(c);
    return IDB_OK;
}

void idb_comm_free(idb_comm* comm) {
    Comm* c = reinterpret_cast<Comm*>(comm);
    if (!c) return;
    if (c->comm && nccl().ok) nccl().CommDestroy(c->comm);
    delete c;
}

idb_status idb_index_set_id_map(idb_index* index, const uint32_t* global_ids) {
    if (!index) return fail(IDB_ERR_INVALID_ARG, "index is null");
    Index* ix = reinterpret_cast<Index*>(index);
    ExclusiveIndex ex(ix);  // searches read the map on the device: none may run on any lane while it changes
    CUDA_TRY(ex.drained);
    if (!global_ids) {
        cudaFree(ix->d_id_map);
        ix->d_id_map = nullptr;
        return IDB_OK;
    }
    if (ix->n == 0) return IDB_OK;
    if (!ix->d_id_map) CUDA_TRY(cudaMalloc(&ix->d_id_map, ix->cap * 4));
    CUDA_TRY(cudaMemcpyAsync(ix->d_id_map, global_ids, ix->n * 4, cudaMemcpyHostToDevice, ix->stream));
    CUDA_TRY(cudaStreamSynchronize(ix->stream));
    return IDB_OK;
}

}  // extern "C" (reopened below)

namespace idb {
// The rank's shards each run K1 on their own lane-0 stream (K1's epilogue packs (distance bits, global id) keys; the launches overlap
// on the device: one table pool, the next shard's thread blocks move in as the previous shard's drain) -> local pre-merge when the
// rank holds more than one shard -> ONE ncclAllGather -> merge kernel.  Main stream = lane 0 of the first shard, which stages the
// queries (in host memory when `host`, else on the device) once for every shard.  The caller holds lanes[0].mu of every shard.
static idb_status sharded_search_locked(Index* const* shards, uint32_t n_local, Comm* c, const float* queries, bool host, uint64_t nq,
                                        uint32_t ef_search, uint32_t k, uint32_t* d_out_ids, float* d_out_dist, uint32_t* d_out_len) {
    Index* ix = shards[0];
    Lane& ln = ix->lanes[0];
    CUDA_TRY(cudaSetDevice(ix->device));
    // merge kernels: world * k (and n_local * k) keys per query in shared memory; check the launches BEFORE anything is enqueued
    int max_smem = 0;
    idb_status st = merge_fits(ix, std::max<uint64_t>((uint64_t)c->world, n_local), k, &max_smem);
    if (st != IDB_OK) return st;
    const size_t per = (size_t)nq * k;
    CUDA_TRY(ensure_u64(ln.keys_local, ln.keys_local_cap, per * (n_local > 1 ? n_local + 1 : 1)));
    CUDA_TRY(ensure_u64(ln.keys_all, ln.keys_all_cap, per * c->world));
    uint64_t* shard_keys = n_local > 1 ? ln.keys_local + per : ln.keys_local;  // [n_local][nq][k]; the pre-merge writes keys_local[0..per)
    const float* qp = nullptr;
    st = ix->stage_queries(ln, queries, host, nq, &qp);
    if (st != IDB_OK) return st;
    cudaEvent_t fork = nullptr;
    if (n_local > 1) {
        CUDA_TRY(cudaEventCreateWithFlags(&fork, cudaEventDisableTiming));
        CUDA_TRY(cudaEventRecord(fork, ln.stream));  // the staged queries (and anything else the caller enqueued) are ready
    }
    for (uint32_t i = 0; i < n_local && st == IDB_OK; ++i) {
        Index* sx = shards[i];
        Lane& sl = sx->lanes[0];
        if (i > 0 && cudaStreamWaitEvent(sl.stream, fork, 0) != cudaSuccess) st = fail(IDB_ERR_CUDA, "cudaStreamWaitEvent failed");
        if (st == IDB_OK && ensure_u32(sl.shard_ids, sl.shard_ids_cap, per) != cudaSuccess) st = fail(IDB_ERR_OOM, "scratch allocation failed");
        if (st == IDB_OK) st = search_on_lane(sx, sl, qp, true, nq, ef_search, k, sl.shard_ids, nullptr, nullptr, shard_keys + (size_t)i * per);
        if (st == IDB_OK && i > 0) {  // join: the main stream continues after this shard's K1
            cudaEvent_t done = nullptr;
            if (cudaEventCreateWithFlags(&done, cudaEventDisableTiming) != cudaSuccess || cudaEventRecord(done, sl.stream) != cudaSuccess ||
                cudaStreamWaitEvent(ln.stream, done, 0) != cudaSuccess)
                st = fail(IDB_ERR_CUDA, "stream join failed");
            if (done) cudaEventDestroy(done);  // (released once the recorded work has completed)
        }
    }
    if (fork) cudaEventDestroy(fork);
    if (st != IDB_OK) return st;
    if (n_local > 1) {
        st = launch_merge(ix, ln.stream, shard_keys, n_local, nq, k, nullptr, nullptr, nullptr, ln.keys_local, max_smem);
        if (st != IDB_OK) return st;
    }
    NCCL_TRY(nccl().AllGather(ln.keys_local, ln.keys_all, per, ncclUint64, c->comm, ln.stream));
    st = launch_merge(ix, ln.stream, ln.keys_all, (uint32_t)c->world, nq, k, d_out_ids, d_out_dist, d_out_len, nullptr, max_smem);
    if (st != IDB_OK) return st;
    // (query normalisation) + K1 + retry per shard, pre-merge, all-gather, merge
    ln.last_launches = (ix->metric == kMetricCosine ? 3 : 2) * n_local + (n_local > 1 ? 1 : 0) + 2;
    return IDB_OK;
}

// Checks that the shards (non-null: check_search_args) fit together and locks lane 0 of every shard (in address order: two callers
// with the same shards cannot deadlock).
struct ShardLocks {
    std::vector<Index*> order;
    ~ShardLocks() { for (auto it = order.rbegin(); it != order.rend(); ++it) (*it)->lanes[0].mu.unlock(); }
    idb_status lock(idb_index* const* shards, uint32_t n) {
        std::vector<Index*> v;
        for (uint32_t i = 0; i < n; ++i) {
            Index* ix = reinterpret_cast<Index*>(shards[i]);
            const Index* first = reinterpret_cast<Index*>(shards[0]);
            if (ix->device != first->device || ix->dim != first->dim)
                return fail(IDB_ERR_INVALID_ARG, "shard %u: all shards of a rank must live on one device and have one dim", i);
            if (ix->metric != first->metric)  // their keys would not be comparable
                return fail(IDB_ERR_INVALID_ARG, "shard %u: all shards of a call must have one metric", i);
            v.push_back(ix);
        }
        std::sort(v.begin(), v.end());
        if (std::adjacent_find(v.begin(), v.end()) != v.end()) return fail(IDB_ERR_INVALID_ARG, "the same index is listed twice");
        for (Index* ix : v) { ix->lanes[0].mu.lock(); order.push_back(ix); ix->last_lane.store(0); }
        return IDB_OK;
    }
};
}  // namespace idb

extern "C" {

// All device pointers; d_queries is nq x dim.  Collective: every rank of `comm` calls it with the same queries.
idb_status idb_sharded_search_batch_device_multi(idb_index* const* shards, uint32_t n_shards, idb_comm* comm, const float* d_queries,
                                                 uint64_t nq, uint32_t ef_search, uint32_t k, uint32_t* d_out_ids, float* d_out_dist,
                                                 uint32_t* d_out_len) {
    idb_status st = check_search_args(Family::sharded, shards, n_shards, comm, nullptr, d_queries, nq, d_out_ids, k);
    if (st != IDB_OK || nq == 0) return st;
    ShardLocks locks;
    if ((st = locks.lock(shards, n_shards)) != IDB_OK) return st;
    return sharded_search_locked(reinterpret_cast<Index* const*>(shards), n_shards, reinterpret_cast<Comm*>(comm), d_queries, false, nq,
                                 ef_search, k, d_out_ids, d_out_dist, d_out_len);
}

idb_status idb_sharded_search_batch_device(idb_index* index, idb_comm* comm, const float* d_queries, uint64_t nq, uint32_t ef_search,
                                           uint32_t k, uint32_t* d_out_ids, float* d_out_dist, uint32_t* d_out_len) {
    return idb_sharded_search_batch_device_multi(&index, 1, comm, d_queries, nq, ef_search, k, d_out_ids, d_out_dist, d_out_len);
}

idb_status idb_sharded_search_batch_f32_multi(idb_index* const* shards, uint32_t n_shards, idb_comm* comm, const float* queries, uint64_t nq,
                                              uint32_t ef_search, uint32_t k, uint32_t* out_ids, float* out_dist, uint32_t* out_len) {
    idb_status st = check_search_args(Family::sharded, shards, n_shards, comm, nullptr, queries, nq, out_ids, k);
    if (st != IDB_OK || nq == 0) return st;
    ShardLocks locks;  // held across staging, search and copy-back: the staging buffers belong to this call
    if ((st = locks.lock(shards, n_shards)) != IDB_OK) return st;
    Index* ix = reinterpret_cast<Index*>(shards[0]);
    Lane& ln = ix->lanes[0];
    CUDA_TRY(cudaSetDevice(ix->device));
    CUDA_TRY(ensure_u32(ln.ids, ln.ids_cap, nq * k));
    CUDA_TRY(ensure_f32(ln.dist, ln.dist_cap, nq * k));
    CUDA_TRY(ensure_u32(ln.len, ln.len_cap, nq));
    st = sharded_search_locked(reinterpret_cast<Index* const*>(shards), n_shards, reinterpret_cast<Comm*>(comm), queries, true, nq,
                               ef_search, k, ln.ids, ln.dist, ln.len);
    if (st != IDB_OK) return st;
    std::vector<Lane*> lanes;  // every shard's stream was joined into ln's
    for (Index* sx : locks.order) lanes.push_back(&sx->lanes[0]);
    return read_back(ln, nq, k, out_ids, out_dist, out_len, lanes.data(), (uint32_t)lanes.size());
}

idb_status idb_sharded_search_batch_f32(idb_index* index, idb_comm* comm, const float* queries, uint64_t nq, uint32_t ef_search, uint32_t k,
                                        uint32_t* out_ids, float* out_dist, uint32_t* out_len) {
    return idb_sharded_search_batch_f32_multi(&index, 1, comm, queries, nq, ef_search, k, out_ids, out_dist, out_len);
}

// The sharded search's merge (launch_merge: the same launch geometry and shared-memory limit) on keys the caller supplies.
idb_status idb_debug_merge_topk(idb_index* index, const uint64_t* keys, uint32_t G, uint64_t nq, uint32_t k, uint32_t* out_ids,
                                float* out_dist, uint32_t* out_len, uint64_t* out_keys) {
    if (!index) return fail(IDB_ERR_INVALID_ARG, "index is null");
    if (G == 0 || k == 0) return fail(IDB_ERR_INVALID_ARG, "G and k must be >= 1");
    Index* ix = reinterpret_cast<Index*>(index);
    std::lock_guard<std::mutex> lk(ix->lanes[0].mu);  // the merge runs on lane 0's stream
    CUDA_TRY(cudaSetDevice(ix->device));
    int max_smem = 0;
    idb_status st = merge_fits(ix, G, k, &max_smem);
    if (st != IDB_OK || nq == 0) return st;
    if (!keys || (!out_keys && !out_ids)) return fail(IDB_ERR_INVALID_ARG, "null argument");
    const size_t per = (size_t)nq * k, in_bytes = per * G * 8, out_bytes = out_keys ? per * 8 : per * 8 + nq * 4;
    char* d = nullptr;
    CUDA_TRY(cudaMalloc(&d, in_bytes + out_bytes));
    uint64_t* d_in = reinterpret_cast<uint64_t*>(d);
    uint64_t* d_keys = out_keys ? reinterpret_cast<uint64_t*>(d + in_bytes) : nullptr;
    uint32_t* d_ids = out_keys ? nullptr : reinterpret_cast<uint32_t*>(d + in_bytes);
    float* d_dist = out_keys || !out_dist ? nullptr : reinterpret_cast<float*>(d + in_bytes + per * 4);
    uint32_t* d_len = out_keys || !out_len ? nullptr : reinterpret_cast<uint32_t*>(d + in_bytes + per * 8);
    cudaStream_t s = ix->lanes[0].stream;
    cudaError_t e = cudaMemcpyAsync(d_in, keys, in_bytes, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) st = launch_merge(ix, s, d_in, G, nq, k, d_ids, d_dist, d_len, d_keys, max_smem);
    if (e == cudaSuccess && st == IDB_OK) {
        if (out_keys) e = cudaMemcpyAsync(out_keys, d_keys, per * 8, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess && d_ids) e = cudaMemcpyAsync(out_ids, d_ids, per * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess && d_dist) e = cudaMemcpyAsync(out_dist, d_dist, per * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess && d_len) e = cudaMemcpyAsync(out_len, d_len, nq * 4, cudaMemcpyDeviceToHost, s);
    }
    const cudaError_t sync = cudaStreamSynchronize(s);  // before the buffer is freed, whatever happened above
    cudaFree(d);
    CUDA_TRY(e);
    if (st != IDB_OK) return st;
    CUDA_TRY(sync);
    return IDB_OK;
}

}  // extern "C"
