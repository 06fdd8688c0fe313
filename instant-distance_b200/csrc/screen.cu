// screen.cu — the per-index screening table K1 uses to skip candidate rows it would reject (DESIGN §2, §4), and a diagnostic entry
// point that evaluates the screening bound next to the canonical distance for given (query, row) pairs.
//
// Table: per element i of a row (dim rounded up to 4, as the stored rows), an affine 8-bit code  x~ = fmaf(code, scale_i, offset_i)
// (round to nearest) with scale_i = max_i / 255 - min_i / 255 and offset_i = min_i over the stored rows, and E_i = max over the rows
// of |x - x~| rounded up, measured on the device with the same fmaf the screen uses — so |x - x~| <= E_i holds for every stored
// value by construction, whatever the rounding of the codes.
#include <algorithm>
#include <cmath>
#include <vector>

#include "internal.cuh"

namespace idb {

namespace {

__device__ __forceinline__ float stored_at(const void* pts, uint32_t bf16, size_t i) {
    return bf16 ? __uint_as_float((uint32_t)reinterpret_cast<const uint16_t*>(pts)[i] << 16) : reinterpret_cast<const float*>(pts)[i];
}
// order-preserving u32 image of a float (for atomicMin / atomicMax)
__device__ __forceinline__ uint32_t ord_of(float f) {
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float float_of_ord(uint32_t u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u); }

// Blocks own ranges of rows, threads own elements: every step of a thread's loop is one coalesced slice of a row.
__global__ void code_range_kernel(const void* pts, uint32_t bf16, uint64_t n, uint32_t stride, uint64_t rows_per_block, uint32_t* mn,
                                  uint32_t* mx, uint32_t* bad) {
    const uint64_t r0 = (uint64_t)blockIdx.x * rows_per_block, r1 = min(n, r0 + rows_per_block);
    if (r0 >= r1) return;
    for (uint32_t e = threadIdx.x; e < stride; e += blockDim.x) {
        float lo = INFINITY, hi = -INFINITY;
        bool nonfinite = false;
        for (uint64_t r = r0; r < r1; ++r) {
            const float x = stored_at(pts, bf16, r * stride + e);
            nonfinite |= !isfinite(x);
            lo = fminf(lo, x);
            hi = fmaxf(hi, x);
        }
        atomicMin(mn + e, ord_of(lo));
        atomicMax(mx + e, ord_of(hi));
        if (nonfinite) atomicOr(bad, 1u);
    }
}

// prm: [0, stride) scale, [stride, 2 stride) offset; [2 stride, 3 stride) E is zeroed here and filled by code_encode_kernel.
__global__ void code_params_kernel(const uint32_t* mn, const uint32_t* mx, uint32_t stride, float* prm) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= stride) return;
    const float lo = float_of_ord(mn[e]), hi = float_of_ord(mx[e]);
    float scale = __fsub_rn(__fdiv_rn(hi, 255.f), __fdiv_rn(lo, 255.f));  // (hi - lo) / 255 without overflow for finite hi, lo
    if (!(scale > 0.f)) scale = 0.f;                                       // a constant element: every code decodes to offset
    prm[e] = scale;
    prm[stride + e] = lo;
    prm[2 * stride + e] = 0.f;
}

__global__ void code_encode_kernel(const void* pts, uint32_t bf16, uint64_t n, uint32_t stride, uint64_t rows_per_block, float* prm,
                                   unsigned char* codes) {
    const uint64_t r0 = (uint64_t)blockIdx.x * rows_per_block, r1 = min(n, r0 + rows_per_block);
    if (r0 >= r1) return;
    for (uint32_t e = threadIdx.x; e < stride; e += blockDim.x) {
        const float scale = prm[e], offset = prm[stride + e];
        float err = 0.f;
        for (uint64_t r = r0; r < r1; ++r) {
            const float x = stored_at(pts, bf16, r * stride + e);
            const float c = scale > 0.f ? fminf(fmaxf(rintf(__fdiv_rn(__fsub_rn(x, offset), scale)), 0.f), 255.f) : 0.f;
            codes[r * stride + e] = (unsigned char)c;
            const float xt = __fmaf_rn(c, scale, offset);  // the screen's x~ (hnsw_device.cuh screen_term)
            err = fmaxf(err, __fsub_ru(fmaxf(x, xt), fminf(x, xt)));
        }
        atomicMax(reinterpret_cast<uint32_t*>(prm + 2 * stride + e), __float_as_uint(err));  // non-negative: same order as the floats
    }
}

// One warp per (query, row) pair: the screen's bound (what K1 compares with the furthest distance) and the canonical distance.
template <int CH, class RT>
__global__ void screen_bound_kernel(GraphView g, const float4* queries, const uint32_t* pairs, uint64_t npairs, float* out_bound,
                                    float* out_dist) {
    const uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
    const int lane = threadIdx.x & 31;
    if (w >= npairs) return;  // warp-uniform
    const uint32_t qi = pairs[2 * w], pid = pairs[2 * w + 1];
    QVec<CH> q;
    q_from_f32<CH>(q, queries + (size_t)qi * g.nchunks, g.nchunks, lane);
    float4 x[CH];
    load_row<CH, RT>(g, pid, lane, x);
    const float dist = butterfly_sum(lane_partial<CH>(q.r, x));
    float p[1] = {0.f};
#pragma unroll
    for (int j = 0; j < CH; ++j) {
        const uint32_t c = lane + 32 * j;
        const uint32_t cw = c < g.nchunks ? g.codes[(size_t)pid * g.nchunks + c] : 0u;
        p[0] = screen_chunk(q.r[j], cw, screen_chunk_params(g, c, c < g.nchunks), p[0]);
    }
    const float bound = screen_finish(batch_butterfly<1, true>(p, lane));
    if (lane == 0) {
        out_bound[w] = bound;
        out_dist[w] = dist;
    }
}

template <int CH>
cudaError_t launch_screen_bound(const GraphView& g, const float4* q, const uint32_t* pairs, uint64_t npairs, float* ob, float* od,
                                cudaStream_t st) {
    const unsigned grid = (unsigned)((npairs + 7) / 8);
    if (g.bf16) screen_bound_kernel<CH, RowBF16><<<grid, 256, 0, st>>>(g, q, pairs, npairs, ob, od);
    else screen_bound_kernel<CH, RowF32><<<grid, 256, 0, st>>>(g, q, pairs, npairs, ob, od);
    return cudaGetLastError();
}

}  // namespace

idb_status Index::build_codes() {
    cudaFree(d_codes);
    cudaFree(d_cparams);
    d_codes = nullptr;
    d_cparams = nullptr;
    if (!screen || n == 0) return IDB_OK;
    const uint32_t stride = nchunks * 4;
    const void* pts = bf16 ? static_cast<const void*>(d_points_bf16) : static_cast<const void*>(d_points);
    const unsigned grid = (unsigned)std::min<uint64_t>((n + 63) / 64, (uint64_t)num_sms * 8);
    const uint64_t rows_per_block = (n + grid - 1) / grid;
    uint32_t* tmp = nullptr;  // [0, stride) min, [stride, 2 stride) max, [2 stride] non-finite flag
    CUDA_TRY(cudaMalloc(&tmp, (2 * (size_t)stride + 1) * 4));
    cudaError_t e = cudaMalloc(&d_cparams, 3 * (size_t)stride * 4);
    if (e == cudaSuccess) e = cudaMalloc(&d_codes, n * (size_t)stride);
    if (e == cudaSuccess) e = fill_u32(tmp, stride, 0xFFFFFFFFu, stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(tmp + stride, 0, ((size_t)stride + 1) * 4, stream);
    if (e == cudaSuccess) {
        code_range_kernel<<<grid, 128, 0, stream>>>(pts, bf16 ? 1u : 0u, n, stride, rows_per_block, tmp, tmp + stride, tmp + 2 * stride);
        e = cudaGetLastError();
    }
    uint32_t bad = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&bad, tmp + 2 * stride, 4, cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e == cudaSuccess && !bad) {
        float* prm = reinterpret_cast<float*>(d_cparams);
        code_params_kernel<<<(stride + 127) / 128, 128, 0, stream>>>(tmp, tmp + stride, stride, prm);
        code_encode_kernel<<<grid, 128, 0, stream>>>(pts, bf16 ? 1u : 0u, n, stride, rows_per_block, prm,
                                                     reinterpret_cast<unsigned char*>(d_codes));
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    }
    cudaFree(tmp);
    if (e != cudaSuccess || bad) {  // a non-finite stored value: no table, K1 fetches every row in full
        cudaFree(d_codes);
        cudaFree(d_cparams);
        d_codes = nullptr;
        d_cparams = nullptr;
    }
    CUDA_TRY(e);
    return IDB_OK;
}

}  // namespace idb

using namespace idb;

extern "C" idb_status idb_last_search_full_fetches(idb_index* index, uint32_t lane, uint64_t* out_rows) {
    if (!index || !out_rows) return fail(IDB_ERR_INVALID_ARG, "null argument");
    SearchCtrl c;
    idb_status st = reinterpret_cast<Index*>(index)->last_search(lane, true, &c, nullptr);
    if (st == IDB_OK) *out_rows = c.full_fetches;
    return st;
}

extern "C" idb_status idb_debug_screen_bound(idb_index* index, const float* queries, uint64_t nq, const uint32_t* pairs, uint64_t npairs,
                                             float* out_bound, float* out_dist) {
    if (!index || (npairs && (!queries || !pairs || !out_bound || !out_dist))) return fail(IDB_ERR_INVALID_ARG, "null argument");
    Index* ix = reinterpret_cast<Index*>(index);
    if (!ix->d_codes) return fail(IDB_ERR_UNSUPPORTED, "this index has no screening table (IDB_SCREEN=0, empty, or a non-finite value)");
    const int ch = kernel_ch(ix->nchunks);
    if (ch == 0) return fail(IDB_ERR_UNSUPPORTED, "dim %u: rows of more than 1024 elements are not screened", ix->dim);
    for (uint64_t i = 0; i < npairs; ++i)
        if (pairs[2 * i] >= nq || pairs[2 * i + 1] >= ix->n) return fail(IDB_ERR_INVALID_ARG, "pair %llu out of range", (unsigned long long)i);
    if (npairs == 0) return IDB_OK;
    std::lock_guard<std::mutex> lk(ix->mu);
    CUDA_TRY(cudaSetDevice(ix->device));
    const size_t stride = (size_t)ix->nchunks * 4;
    char* d = nullptr;
    const size_t qb = nq * stride * 4, pb = npairs * 8, ob = npairs * 4;
    CUDA_TRY(cudaMalloc(&d, qb + pb + 2 * ob));
    float* dq = reinterpret_cast<float*>(d);
    uint32_t* dp = reinterpret_cast<uint32_t*>(d + qb);
    float* dbound = reinterpret_cast<float*>(d + qb + pb);
    float* ddist = dbound + npairs;
    cudaStream_t st = ix->stream;
    cudaError_t e = cudaMemsetAsync(dq, 0, qb, st);
    if (e == cudaSuccess) e = cudaMemcpy2DAsync(dq, stride * 4, queries, ix->dim * 4, ix->dim * 4, nq, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(dp, pairs, pb, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        const GraphView g = ix->view();
        const float4* q4 = reinterpret_cast<const float4*>(dq);
        switch (ch) {
            case 1: e = launch_screen_bound<1>(g, q4, dp, npairs, dbound, ddist, st); break;
            case 2: e = launch_screen_bound<2>(g, q4, dp, npairs, dbound, ddist, st); break;
            case 3: e = launch_screen_bound<3>(g, q4, dp, npairs, dbound, ddist, st); break;
            case 4: e = launch_screen_bound<4>(g, q4, dp, npairs, dbound, ddist, st); break;
            case 6: e = launch_screen_bound<6>(g, q4, dp, npairs, dbound, ddist, st); break;
            default: e = launch_screen_bound<8>(g, q4, dp, npairs, dbound, ddist, st); break;
        }
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(out_bound, dbound, ob, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out_dist, ddist, ob, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(d);
    CUDA_TRY(e);
    return IDB_OK;
}
