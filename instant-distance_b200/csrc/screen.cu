// screen.cu — the per-index screening table K1 uses to skip candidate rows it would reject (DESIGN §2, §4), and a diagnostic entry
// point that evaluates the screening bound next to the canonical distance for given (query, row) pairs.
//
// Table: one code step S for every element and a per-element offset_i = min_i over the stored rows, codes
// c_i = clamp(rint((x_i - offset_i) / S), 0, 255) with S >= max_i (max_i - min_i) / 255 (rounded up), so that code differences
// measure distance in the same unit everywhere: ||q^ - x~|| = S * sqrt(sum (qc_i - c_i)^2) exactly, where x~_i = offset_i + c_i * S
// in real arithmetic (K1's integer bound, hnsw_device.cuh screen_candidates).  Beside the codes:
//   R   >= ||x - x~|| over every stored row, measured on the device with upward rounding (x~ bracketed by fmaf_rd / fmaf_ru);
//   E_i  = max over the rows of |x - fmaf_rn(c, S, offset_i)| rounded up, and S in every scale slot, so the per-element float bound
//          |q_i - x~_i| - E_i <= |q_i - x_i| holds on the same codes.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "internal.cuh"

namespace idb {

namespace {

// order-preserving u32 image of a float (for atomicMin / atomicMax)
__device__ __forceinline__ uint32_t ord_of(float f) {
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float float_of_ord(uint32_t u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u); }

// Blocks own ranges of rows, threads own elements: every step of a thread's loop is one coalesced slice of a row.
__global__ void code_range_kernel(const StoredRows s, uint64_t n, uint64_t rows_per_block, uint32_t* mn, uint32_t* mx, uint32_t* bad) {
    const uint64_t r0 = (uint64_t)blockIdx.x * rows_per_block, r1 = min(n, r0 + rows_per_block);
    if (r0 >= r1) return;
    for (uint32_t e = threadIdx.x; e < s.stride; e += blockDim.x) {
        float lo = INFINITY, hi = -INFINITY;
        bool nonfinite = false;
        for (uint64_t r = r0; r < r1; ++r) {
            const float x = stored_elem(s, r, e);
            nonfinite |= !isfinite(x);
            lo = fminf(lo, x);
            hi = fmaxf(hi, x);
        }
        atomicMin(mn + e, ord_of(lo));
        atomicMax(mx + e, ord_of(hi));
        if (nonfinite) atomicOr(bad, 1u);
    }
}

// prm: [0, stride) scale (filled with S by code_encode_kernel), [stride, 2 stride) offset; [2 stride, 3 stride) E is zeroed here and
// filled by code_encode_kernel.  step: S, the largest per-element step (hi - lo) / 255 rounded up (atomicMax of non-negative floats).
__global__ void code_params_kernel(const uint32_t* mn, const uint32_t* mx, uint32_t stride, float* prm, uint32_t* step) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= stride) return;
    const float lo = float_of_ord(mn[e]), hi = float_of_ord(mx[e]);
    float scale = __fsub_ru(__fdiv_ru(hi, 255.f), __fdiv_rd(lo, 255.f));  // >= (hi - lo) / 255 without overflow for finite hi, lo
    if (!(scale > 0.f)) scale = 0.f;                                       // a constant element
    atomicMax(step, __float_as_uint(scale));
    prm[stride + e] = lo;
    prm[2 * stride + e] = 0.f;
}

__device__ __forceinline__ float code_of_value(float x, float offset, float step) {
    return step > 0.f ? fminf(fmaxf(rintf(__fdiv_rn(__fsub_rn(x, offset), step)), 0.f), 255.f) : 0.f;
}

// codes: rows of cstride bytes (4 code_words(nchunks)); the bytes past stride are zeroed beforehand.
__global__ void code_encode_kernel(const StoredRows s, uint64_t n, uint32_t cstride, uint64_t rows_per_block, float* prm, const uint32_t* step,
                                   unsigned char* codes) {
    const uint32_t stride = s.stride;
    const float S = __uint_as_float(*step);
    if (blockIdx.x == 0)
        for (uint32_t e = threadIdx.x; e < stride; e += blockDim.x) prm[e] = S;
    const uint64_t r0 = (uint64_t)blockIdx.x * rows_per_block, r1 = min(n, r0 + rows_per_block);
    if (r0 >= r1) return;
    for (uint32_t e = threadIdx.x; e < stride; e += blockDim.x) {
        const float offset = prm[stride + e];
        float err = 0.f;
        for (uint64_t r = r0; r < r1; ++r) {
            const float x = stored_elem(s, r, e);
            const float c = code_of_value(x, offset, S);
            codes[r * cstride + e] = (unsigned char)c;
            const float xt = __fmaf_rn(c, S, offset);  // x~ of the per-element float bound
            err = fmaxf(err, __fsub_ru(fmaxf(x, xt), fminf(x, xt)));
        }
        atomicMax(reinterpret_cast<uint32_t*>(prm + 2 * stride + e), __float_as_uint(err));  // non-negative: same order as the floats
    }
}

// One warp per row (grid-stride): r_x = ||x - x~||, rounded up, with x~_i = offset_i + c_i * S in real arithmetic, which lies in
// [fmaf_rd(c, S, offset), fmaf_ru(c, S, offset)], so |x_i - x~_i| <= max(x_i - lo, hi - x_i).  err_max = max over the rows.
__global__ void code_row_err_kernel(const StoredRows s, uint64_t n, const float* prm, const uint32_t* step, const uint32_t* codes,
                                    uint32_t* err_max) {
    const float S = __uint_as_float(*step);
    const uint32_t stride = s.stride, nchunks = stride / 4, cwords = code_words(nchunks);
    const int lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
    float worst = 0.f;
    for (uint64_t r = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; r < n; r += warps) {
        float acc = 0.f;
        for (uint32_t c = lane; c < nchunks; c += 32) {
            const uint32_t w = codes[r * cwords + c];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t e = 4 * c + k;
                const float x = stored_elem(s, r, e), off = prm[stride + e], code = (float)((w >> (8 * k)) & 0xFFu);
                const float d = fmaxf(__fsub_ru(x, __fmaf_rd(code, S, off)), __fsub_ru(__fmaf_ru(code, S, off), x));
                acc = __fmaf_ru(d, d, acc);
            }
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) acc = __fadd_ru(acc, __shfl_xor_sync(kFullMask, acc, o));
        worst = fmaxf(worst, __fsqrt_ru(acc));
    }
    if (lane == 0) atomicMax(err_max, __float_as_uint(worst));
}

// One warp per (query, row) pair: the screen's bound (what K1 compares with the furthest distance) and the canonical distance.
// The same helpers and layout as K1's screen_candidates (screen_query, screen_slice, ScreenLane, screen_words, batch_butterfly over eight lanes,
// screen_bound_of): each group of eight lanes reduces the row on its own, as one K1 slot does.
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
    ScreenQuery<CH> sq;
    screen_query<CH>(sq, g, q.r, lane);
    uint4 qc[CH], cw[CH];
    screen_slice<CH>(qc, sq, lane);
    ScreenLane<CH, false>(g, lane).load(cw, pid, true);
    uint32_t p[1] = {0u};
#pragma unroll
    for (int j = 0; j < CH; ++j) p[0] = screen_words(qc[j], cw[j], p[0]);
    const float bound = screen_bound_of(g, batch_butterfly<1, false, uint32_t, 8>(p, lane), sq.slack);
    if (lane == 0) {
        out_bound[w] = bound;
        out_dist[w] = dist;
    }
}

template <int CH>
cudaError_t launch_screen_bound(const GraphView& g, const float4* q, const uint32_t* pairs, uint64_t npairs, float* ob, float* od,
                                cudaStream_t st) {
    const unsigned grid = (unsigned)((npairs + 7) / 8);
    with_row_type(g.row_type, [&](auto rt) {
        using RT = decltype(rt);
        if constexpr (RT::kType != kRowQ8 && RT::kType != kRowBin) screen_bound_kernel<CH, RT><<<grid, 256, 0, st>>>(g, q, pairs, npairs, ob, od);  // (no table)
    });
    return cudaGetLastError();
}

}  // namespace

idb_status Index::build_codes() {
    cudaFree(d_codes);
    cudaFree(d_cparams);
    d_codes = nullptr;
    d_cparams = nullptr;
    // DESIGN §3c, §3d: q8 rows are one byte per element already, bin rows a quarter byte
    if (!screen || n == 0 || row_type == kRowQ8 || row_type == kRowBin) return IDB_OK;
    const uint32_t stride = nchunks * 4, cstride = code_words(nchunks) * 4;
    const StoredRows s = stored();
    const unsigned grid = (unsigned)std::min<uint64_t>((n + 63) / 64, (uint64_t)num_sms * 8);
    const uint64_t rows_per_block = (n + grid - 1) / grid;
    uint32_t* tmp = nullptr;  // [0, stride) min, [stride, 2 stride) max, [2 stride] non-finite flag, [2 stride + 1] S, [2 stride + 2] R
    CUDA_TRY(cudaMalloc(&tmp, (2 * (size_t)stride + 3) * 4));
    cudaError_t e = cudaMalloc(&d_cparams, 3 * (size_t)stride * 4);
    if (e == cudaSuccess) e = cudaMalloc(&d_codes, n * (size_t)cstride);
    if (e == cudaSuccess && cstride != stride) e = cudaMemsetAsync(d_codes, 0, n * (size_t)cstride, stream);  // the padding words
    if (e == cudaSuccess) e = fill_u32(tmp, stride, 0xFFFFFFFFu, stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(tmp + stride, 0, ((size_t)stride + 3) * 4, stream);
    if (e == cudaSuccess) {
        code_range_kernel<<<grid, 128, 0, stream>>>(s, n, rows_per_block, tmp, tmp + stride, tmp + 2 * stride);
        e = cudaGetLastError();
    }
    uint32_t bad = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&bad, tmp + 2 * stride, 4, cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    uint32_t step_err[2] = {0u, 0u};
    if (e == cudaSuccess && !bad) {
        float* prm = reinterpret_cast<float*>(d_cparams);
        uint32_t* step = tmp + 2 * stride + 1;
        code_params_kernel<<<(stride + 127) / 128, 128, 0, stream>>>(tmp, tmp + stride, stride, prm, step);
        code_encode_kernel<<<grid, 128, 0, stream>>>(s, n, cstride, rows_per_block, prm, step, reinterpret_cast<unsigned char*>(d_codes));
        code_row_err_kernel<<<num_sms * 8, 256, 0, stream>>>(s, n, prm, step, d_codes, step + 1);
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpyAsync(step_err, step, 8, cudaMemcpyDeviceToHost, stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    }
    std::memcpy(&code_step, &step_err[0], 4);
    std::memcpy(&code_err, &step_err[1], 4);
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
    if (!ix->d_codes) return fail(IDB_ERR_UNSUPPORTED, "this index has no screening table (IDB_SCREEN=0, empty, q8 or bin rows, or a non-finite value)");
    if (kernel_ch(ix->nchunks) == 0) return fail(IDB_ERR_UNSUPPORTED, "dim %u: rows of more than 1024 elements are not screened", ix->dim);
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
        e = with_cell(ix->nchunks, [&](auto cell) {
            constexpr int CH = decltype(cell)::CH;
            if constexpr (CH == 0) return cudaErrorInvalidValue;  // refused above
            else return launch_screen_bound<CH>(g, q4, dp, npairs, dbound, ddist, st);
        });
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(out_bound, dbound, ob, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out_dist, ddist, ob, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(d);
    CUDA_TRY(e);
    return IDB_OK;
}
