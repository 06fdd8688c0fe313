// merge.cu — K4: per query, the k smallest keys of several k-lists (the sharded search's all-gather, a rank's pre-merge of its shards,
// and the slices of an exact search).
#include <algorithm>

#include "internal.cuh"

namespace idb {

// One warp per query: keep the k smallest keys of the union of its G lists.
// Keys are unique (global ids / PointIds are), so rank(key) = #{keys smaller} is a permutation.  The lists are NOT assumed sorted by
// the full key: a shard orders exact-distance ties by its local PointId, the merged order is by global id.
// out_keys != null: write the merged keys (the local pre-merge of a rank that holds several shards) instead of ids / distances.
// The keys carry the traversal's own distance bits; out_dist reports them through reported_distance (the lists' metric).
__global__ void merge_topk_kernel(const uint64_t* all_keys /* G x nq x k */, uint32_t G, uint64_t nq, uint32_t k,
                                  uint32_t* out_ids, float* out_dist, uint32_t* out_len, uint64_t* out_keys, uint32_t metric) {
    extern __shared__ uint64_t sm_keys[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    uint64_t* keys = sm_keys + (size_t)warp * G * k;
    const uint32_t total = G * k;
    for (uint64_t q = (uint64_t)blockIdx.x * wpb + warp; q < nq; q += (uint64_t)gridDim.x * wpb) {
        for (uint32_t t = lane; t < total; t += 32) {
            const uint32_t g = t / k, j = t - g * k;
            keys[t] = all_keys[((size_t)g * nq + q) * k + j];
        }
        __syncwarp();
        uint32_t found = 0;
        for (uint32_t t = lane; t < total; t += 32) {
            const uint64_t key = keys[t];
            if (key == kKeyNone) continue;
            uint32_t rank = 0;
            for (uint32_t i = 0; i < total; ++i) rank += keys[i] < key ? 1u : 0u;
            if (rank < k) {
                if (out_keys) out_keys[q * k + rank] = key;
                else {
                    out_ids[q * k + rank] = (uint32_t)key;
                    if (out_dist) out_dist[q * k + rank] = reported_distance((uint32_t)(key >> 32), metric);
                }
            }
        }
        // number of real results = min(k, total non-empty keys); pad the tail
        uint32_t real = 0;
        for (uint32_t t = lane; t < total; t += 32) real += keys[t] != kKeyNone ? 1u : 0u;
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) real += __shfl_xor_sync(kFullMask, real, off);
        found = min(real, k);
        for (uint32_t j = found + lane; j < k; j += 32) {
            if (out_keys) out_keys[q * k + j] = kKeyNone;
            else {
                out_ids[q * k + j] = kInvalid;
                if (out_dist) out_dist[q * k + j] = __int_as_float(0x7f800000);
            }
        }
        if (out_len && lane == 0) out_len[q] = found;
        __syncwarp();
    }
}

idb_status merge_fits(const Index* ix, uint64_t lists, uint32_t k, int* max_smem) {
    CUDA_TRY(cudaDeviceGetAttribute(max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, ix->device));
    if (lists * k * 8 > (uint64_t)*max_smem)
        return fail(IDB_ERR_UNSUPPORTED, "%llu keys per query do not fit the merge kernel's shared memory (%d bytes)",
                    (unsigned long long)(lists * k), *max_smem);
    return IDB_OK;
}

idb_status launch_merge(Index* ix, cudaStream_t st, const uint64_t* keys, uint32_t G, uint64_t nq, uint32_t k, uint32_t* d_ids,
                        float* d_dist, uint32_t* d_len, uint64_t* d_keys, int max_smem) {
    const size_t per_warp = (size_t)G * k * 8;
    int wpb = 4;
    while (wpb > 1 && per_warp * wpb > (size_t)max_smem) wpb >>= 1;
    const size_t smem = (size_t)wpb * per_warp;
    if (smem > 48 * 1024) CUDA_TRY(cudaFuncSetAttribute(merge_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const unsigned grid = (unsigned)std::min<uint64_t>((nq + wpb - 1) / wpb, (uint64_t)ix->num_sms * 8);
    merge_topk_kernel<<<grid, wpb * 32, smem, st>>>(keys, G, nq, k, d_ids, d_dist, d_len, d_keys, ix->metric);
    CUDA_TRY(cudaGetLastError());
    return IDB_OK;
}

}  // namespace idb
