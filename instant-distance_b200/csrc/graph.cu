// graph.cu — an index's adjacency (DESIGN §2): the zero rows, the upper layers and their device pointer table, allocated, copied
// out and freed in one place, and the checks of a graph adopted from outside.  The one other place that allocates an adjacency
// layer is Index::reserve_rows (rows.cu), which grows zero together with the rows.
#include <algorithm>

#include "internal.cuh"

namespace idb {

// Adjacency sanity check for graphs adopted from outside (idb_index_from_graph_*, idb_index_load): every entry must be
// INVALID or a PointId below `limit`; otherwise the traversal would read out of bounds.
__global__ void validate_rows_kernel(const uint32_t* rows, size_t count, uint32_t limit, uint32_t* bad) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t v = rows[i];
        if (v != kInvalid && v >= limit) atomicAdd(bad, 1u);
    }
}

// Does any adjacency row list a PointId twice?  (The b16 visited flavour assumes it does not; graphs built by this library or by the
// reference never do.)  One warp per row of `width` <= 128 entries.
__global__ void repeated_ids_kernel(const uint32_t* rows, size_t n_rows, uint32_t width, uint32_t* repeats) {
    const int lane = threadIdx.x & 31;
    const size_t wpb = blockDim.x >> 5;
    for (size_t r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n_rows; r += (size_t)gridDim.x * wpb) {
        uint32_t e[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) e[t] = (uint32_t)(lane + 32 * t) < width ? rows[r * width + lane + 32 * t] : kInvalid;
        bool rep = false;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const uint32_t peers = __match_any_sync(kFullMask, e[t] == kInvalid ? (0x80000000u | (uint32_t)lane) + 0u : e[t]);
            rep |= e[t] != kInvalid && (peers & ((1u << lane) - 1u));
#pragma unroll
            for (int t2 = 0; t2 < 4; ++t2)
                if (t2 > t)
                    for (int src = 0; src < 32; ++src) {
                        const uint32_t o = __shfl_sync(kFullMask, e[t], src);
                        rep |= o != kInvalid && o == e[t2];
                    }
        }
        if (__any_sync(kFullMask, rep) && lane == 0) atomicAdd(repeats, 1u);
    }
}

Graph& Graph::operator=(Graph&& o) noexcept {
    std::swap(zero, o.zero);
    std::swap(upper, o.upper);
    std::swap(upper_n, o.upper_n);
    std::swap(upper_ptrs, o.upper_ptrs);
    std::swap(rows_distinct, o.rows_distinct);
    return *this;
}

Graph::~Graph() {
    cudaFree(zero);
    for (auto* p : upper) cudaFree(p);
    cudaFree(upper_ptrs);
}

cudaError_t Graph::alloc(uint64_t cap, uint32_t M, std::vector<uint64_t> layer_n, cudaStream_t st) {
    upper_n = std::move(layer_n);
    cudaError_t e = cudaMalloc(&zero, cap * 2 * (size_t)M * 4);
    for (size_t l = 0; e == cudaSuccess && l < upper_n.size(); ++l) {
        uint32_t* p = nullptr;
        e = cudaMalloc(&p, std::max<size_t>(4, upper_n[l] * (size_t)M * 4));
        if (e == cudaSuccess) upper.push_back(p);
    }
    if (e == cudaSuccess) e = cudaMalloc(&upper_ptrs, std::max<size_t>(1, upper.size()) * sizeof(uint32_t*));
    if (e == cudaSuccess && !upper.empty())
        e = cudaMemcpyAsync(upper_ptrs, upper.data(), upper.size() * sizeof(uint32_t*), cudaMemcpyHostToDevice, st);
    return e;
}

cudaError_t Graph::copy_out(uint32_t l, uint64_t r0, uint64_t m, uint32_t M, uint32_t* host, cudaStream_t st) const {
    if (m == 0) return cudaSuccess;
    const size_t width = l == 0 ? 2 * (size_t)M : M;
    const uint32_t* src = l == 0 ? zero : upper[l - 1];
    cudaError_t e = cudaMemcpyAsync(host, src + r0 * width, m * width * 4, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    return e;
}

idb_status Graph::check(uint64_t n, uint32_t M, int num_sms, cudaStream_t st) {
    uint32_t* d_bad = nullptr;
    CUDA_TRY(cudaMalloc(&d_bad, 4));
    CUDA_TRY(cudaMemsetAsync(d_bad, 0, 4, st));
    validate_rows_kernel<<<num_sms * 4, 256, 0, st>>>(zero, n * 2 * (size_t)M, (uint32_t)n, d_bad);
    for (size_t l = 0; l < upper.size(); ++l)
        validate_rows_kernel<<<num_sms * 4, 256, 0, st>>>(upper[l], upper_n[l] * (size_t)M, (uint32_t)upper_n[l], d_bad);
    uint32_t bad = 0;
    cudaError_t e = cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e == cudaSuccess && bad == 0) {  // rows that list a PointId twice are legal input but rule out the b16 visited flavour
        repeated_ids_kernel<<<num_sms * 8, 128, 0, st>>>(zero, n, 2 * M, d_bad);
        for (size_t l = 0; l < upper.size(); ++l) repeated_ids_kernel<<<num_sms * 8, 128, 0, st>>>(upper[l], upper_n[l], M, d_bad);
        uint32_t rep = 0;
        e = cudaMemcpyAsync(&rep, d_bad, 4, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        rows_distinct = rep == 0;
    }
    cudaFree(d_bad);
    CUDA_TRY(e);
    if (bad) return fail(IDB_ERR_INVALID_ARG, "%u adjacency entries refer to PointIds outside their layer", bad);
    return IDB_OK;
}

idb_status Index::upload(uint64_t n_, uint32_t dim_, uint32_t M_, uint32_t ef, const uint32_t* zero, uint32_t n_upper,
                         const uint32_t* const* upper, const uint64_t* upper_n) {
    // Layer l holds PointIds [0, n_l) (lib.rs:275-281): n >= n_1 >= n_2 >= ... >= 1.  The descent carries ids found on layer l
    // into layer l-1 and seeds PointId 0 on the top layer, so anything else would read adjacency rows out of bounds.
    for (uint32_t l = 0; l < n_upper; ++l) {
        const uint64_t below = l == 0 ? n_ : upper_n[l - 1];
        if (upper_n[l] == 0 || upper_n[l] > below)
            return fail(IDB_ERR_INVALID_ARG, "layer %u has %llu nodes but the layer below has %llu (need n >= n_1 >= ... >= 1)", l + 1,
                        (unsigned long long)upper_n[l], (unsigned long long)below);
    }
    n = n_;
    cap = n_;
    dim = dim_;
    M = M_;
    ef_search = ef;
    nchunks = (dim + 3) / 4;
    if (n == 0) return IDB_OK;
    const size_t stride = (size_t)nchunks * 4;
    if (n > SIZE_MAX / (stride * sizeof(float)) || n > SIZE_MAX / (2 * (size_t)M * 4)) return fail(IDB_ERR_INVALID_ARG, "n * dim overflows size_t");
    CUDA_TRY(graph.alloc(n, M, std::vector<uint64_t>(upper_n, upper_n + n_upper), stream));
    CUDA_TRY(cudaMemcpyAsync(graph.zero, zero, n * 2 * (size_t)M * 4, cudaMemcpyHostToDevice, stream));
    for (uint32_t l = 0; l < n_upper; ++l)
        if (upper[l]) CUDA_TRY(cudaMemcpyAsync(graph.upper[l], upper[l], upper_n[l] * (size_t)M * 4, cudaMemcpyHostToDevice, stream));
    return graph.check(n, M, num_sms, stream);  // reject graphs whose adjacency points outside the layer it belongs to
}

idb_status Index::stage_rows(uint64_t r0, uint64_t m, const uint32_t* global_ids) {
    CUDA_TRY(fill_u32(graph.zero + r0 * 2 * M, m * 2 * M, kInvalid, stream));
    if (d_id_map) CUDA_TRY(cudaMemcpyAsync(d_id_map + r0, global_ids, m * 4, cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    return IDB_OK;
}

}  // namespace idb
