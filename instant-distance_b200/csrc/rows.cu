// rows.cu — an index's row storage (DESIGN §2, §3b, §3c, §3d): the one buffer of stored rows, the one way rows go in (staged as
// padded f32, checked against the storage's range, then narrowed, quantised or packed into the store) and the one way they come out (widened
// exactly).  The only host code that branches on the storage type; the kernels read the rows through the row traits of
// hnsw_device.cuh.
#include <algorithm>
#include <cmath>

#include "internal.cuh"

namespace idb {

namespace {

// Bytes per stored 4-element chunk (RT::kChunkBytes of the row trait): a bin chunk is a quarter of a q8 one, so there is no per-element size.
size_t chunk_bytes(uint32_t row_type) {
    return row_type == kRowF32 ? 16 : row_type == kRowQ8 ? 4 : row_type == kRowBin ? 1 : 8;
}

// The store of `rows` rows of the index's storage, and q8's headers beside it.
cudaError_t alloc_store(const Index& ix, uint64_t rows, void** pts, float2** hdr) {
    cudaError_t e = cudaMalloc(pts, rows * ix.row_bytes());
    if (e == cudaSuccess && ix.row_type == kRowQ8) e = cudaMalloc(hdr, rows * sizeof(float2));
    return e;
}

// f32 -> bf16 / fp16 (round to nearest even), element-wise over the padded row matrix
__global__ void narrow_bf16_kernel(const float* src, uint16_t* dst, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t b = __float_as_uint(src[i]);
        uint32_t r;
        if ((b & 0x7fffffffu) > 0x7f800000u) r = (b >> 16) | 0x40u;           // NaN stays NaN
        else r = (b + 0x7fffu + ((b >> 16) & 1u)) >> 16;                       // RNE
        dst[i] = (uint16_t)r;
    }
}
// cvt.rn.f16.f32 is RNE with subnormal results kept and overflow to +-inf (refused beforehand by check_rows); a NaN keeps its sign
// and top payload bits, quieted (what the x86 F16C conversion and numpy give for a quiet NaN).
__global__ void narrow_f16_kernel(const float* src, uint16_t* dst, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float x = src[i];
        const uint32_t b = __float_as_uint(x);
        unsigned short h;
        if ((b & 0x7fffffffu) > 0x7f800000u) h = (unsigned short)(((b >> 16) & 0x8000u) | 0x7e00u | ((b >> 13) & 0x3ffu));
        else asm("cvt.rn.f16.f32 %0, %1;" : "=h"(h) : "f"(x));
        dst[i] = h;
    }
}
// The smallest flat index of a finite element that rounds to +-inf in fp16 (|x| >= 65520, halfway to the next binade past 65504).
__global__ void f16_overflow_kernel(const float* src, size_t n, unsigned long long* first) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float x = fabsf(src[i]);
        if (x >= 65520.f && x <= 3.402823466e38f) atomicMin(first, (unsigned long long)i);
    }
}

// q8 rows (DESIGN §3c).  The grid of a row x of `dim` finite f32 values, in f64, where every step below is exact (x * 2^-e is a
// power-of-two scaling of an f32):
//   A = max |x_i|;  A == 0: e = -149, b = 0.  Else e_lo = max(-149, ilogb(A) - 23) and e = the smallest e >= e_lo with
//   ceil(max x / 2^e) - floor(min x / 2^e) <= 255;  b = floor(min x / 2^e);  c_i = rint(x_i / 2^e) - b in [0, 255].
// Element i is (b + c_i) 2^e, |b + c_i| < 2^24, so it and the header {o, s} = {b 2^e, 2^e} are exact f32 unless they overflow.
struct Q8Grid {
    int e;
    double b, scale;  // scale = 2^-e
};
__device__ __forceinline__ double pow2(int k) { return __hiloint2double((1023 + k) << 20, 0); }  // 2^k, -1022 <= k <= 1023
__device__ __forceinline__ Q8Grid q8_grid(float mn, float mx) {
    Q8Grid g;
    const float A = fmaxf(fabsf(mn), fabsf(mx));
    if (A == 0.f) {
        g.e = -149;
        g.b = 0.0;
        g.scale = pow2(149);
        return g;
    }
    int e = max(-149, ilogbf(A) - 23);
    while (ceil((double)mx * pow2(-e)) - floor((double)mn * pow2(-e)) > 255.0) ++e;  // at most ~25 steps
    g.e = e;
    g.scale = pow2(-e);
    g.b = floor((double)mn * g.scale);
    return g;
}
// The row's min and max over its first dim elements (one warp per row; every lane ends with both) and whether all are finite.
__device__ __forceinline__ bool q8_row_range(const float* x, uint32_t dim, int lane, float* mn, float* mx) {
    float lo = INFINITY, hi = -INFINITY;
    bool fin = true;
    for (uint32_t i = lane; i < dim; i += 32) {
        const float v = x[i];
        fin = fin && isfinite(v);
        lo = fminf(lo, v);
        hi = fmaxf(hi, v);
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        lo = fminf(lo, __shfl_xor_sync(kFullMask, lo, o));
        hi = fmaxf(hi, __shfl_xor_sync(kFullMask, hi, o));
    }
    *mn = lo;
    *mx = hi;
    return __all_sync(kFullMask, fin);
}
// v 2^e is an f32 (not infinite), for an integer |v| < 2^24
__device__ __forceinline__ bool q8_fits(double v, int e) { return fabs(v) * pow2(e) < 0x1p128; }
// The smallest flat index (row * stride + element) of an element that refuses its row: a NaN or +-inf, else (a finite row whose
// header or a dequantised element overflows f32) the first element that overflows, or the row's first minimum when only o does.
__global__ void check_q8_kernel(const float* rows, uint64_t m, uint32_t stride, uint32_t dim, unsigned long long* first) {
    const int lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
    for (uint64_t r = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; r < m; r += warps) {
        const float* x = rows + r * stride;
        float mn, mx;
        if (!q8_row_range(x, dim, lane, &mn, &mx)) {
            for (uint32_t i = lane; i < dim; i += 32)
                if (!isfinite(x[i])) atomicMin(first, (unsigned long long)(r * stride + i));
            continue;
        }
        const Q8Grid g = q8_grid(mn, mx);
        const bool o_ok = q8_fits(g.b, g.e);
        for (uint32_t i = lane; i < dim; i += 32)
            if (!q8_fits(rint((double)x[i] * g.scale), g.e) || (!o_ok && x[i] == mn)) atomicMin(first, (unsigned long long)(r * stride + i));
    }
}
// bin rows (DESIGN §3d): the smallest flat index of an element other than +0.0, -0.0 or 1.0 (NaN, +-inf and subnormals included).
__global__ void check_bin_kernel(const float* src, size_t n, unsigned long long* first) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t b = __float_as_uint(src[i]);
        if ((b & 0x7fffffffu) != 0u && b != 0x3f800000u) atomicMin(first, (unsigned long long)i);
    }
}
// Checked 0/1 rows (nchunks * 4 f32 each, so chunk i of the matrix is src[4i, 4i + 4)) -> one byte per chunk: bit k = element 4i+k.
__global__ void pack_bin_kernel(const float* src, uint8_t* dst, size_t nbytes) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nbytes; i += (size_t)gridDim.x * blockDim.x) {
        const float4 x = reinterpret_cast<const float4*>(src)[i];
        dst[i] = (uint8_t)((x.x == 1.f ? 1u : 0u) | (x.y == 1.f ? 2u : 0u) | (x.z == 1.f ? 4u : 0u) | (x.w == 1.f ? 8u : 0u));
    }
}

// Codes (stride bytes per row, padding codes 0) and headers of m checked rows.  One warp per row.
__global__ void quantize_q8_kernel(const float* rows, uint64_t m, uint32_t stride, uint32_t dim, uint8_t* codes, float2* hdr) {
    const int lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
    for (uint64_t r = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; r < m; r += warps) {
        const float* x = rows + r * stride;
        float mn, mx;
        q8_row_range(x, dim, lane, &mn, &mx);
        const Q8Grid g = q8_grid(mn, mx);
        for (uint32_t i = lane; i < stride; i += 32)
            codes[r * stride + i] = i < dim ? (uint8_t)(rint((double)x[i] * g.scale) - g.b) : (uint8_t)0;
        if (lane == 0) hdr[r] = make_float2((float)(g.b * pow2(g.e)), (float)pow2(g.e));
    }
}

// Stored rows [r0, r0 + m), widened exactly (stored_elem), stride floats per row.
__global__ void widen_rows_kernel(const StoredRows s, uint64_t r0, uint64_t m, float* dst) {
    const size_t total = m * s.stride;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = stored_elem(s, r0 + i / s.stride, (uint32_t)(i % s.stride));
}

// The storage's refusal of m staged rows (nchunks * 4 f32 each, on the device): fp16 refuses a finite element that rounds to +-infinity
// (|x| >= 65520); q8 a NaN or infinite element, or a row whose header or a dequantised element would overflow f32; bin an element other
// than +-0 or 1.  IDB_ERR_INVALID_ARG
// names the first such element and its row, input_row[r] when given, else r.  IDB_OK for the other storages.
idb_status check_rows(const Index& ix, const float* staged, uint64_t m, const uint32_t* input_row) {
    if (ix.row_type != kRowF16 && ix.row_type != kRowQ8 && ix.row_type != kRowBin) return IDB_OK;
    const size_t stride = (size_t)ix.nchunks * 4;
    unsigned long long* d_first = nullptr;
    unsigned long long first = ~0ull;
    CUDA_TRY(cudaMalloc(&d_first, 8));
    cudaError_t e = cudaMemcpyAsync(d_first, &first, 8, cudaMemcpyHostToDevice, ix.stream);
    if (e == cudaSuccess) {
        if (ix.row_type == kRowF16) f16_overflow_kernel<<<ix.num_sms * 8, 256, 0, ix.stream>>>(staged, m * stride, d_first);
        else if (ix.row_type == kRowBin) check_bin_kernel<<<ix.num_sms * 8, 256, 0, ix.stream>>>(staged, m * stride, d_first);
        else check_q8_kernel<<<ix.num_sms * 8, 256, 0, ix.stream>>>(staged, m, (uint32_t)stride, ix.dim, d_first);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(&first, d_first, 8, cudaMemcpyDeviceToHost, ix.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ix.stream);
    float x = 0.f;
    if (e == cudaSuccess && first != ~0ull) e = cudaMemcpy(&x, staged + first, 4, cudaMemcpyDeviceToHost);
    cudaFree(d_first);
    CUDA_TRY(e);
    if (first == ~0ull) return IDB_OK;
    const unsigned long long r = input_row ? input_row[first / stride] : first / stride, i = first % stride;
    if (ix.row_type == kRowF16)
        return fail(IDB_ERR_INVALID_ARG, "fp16 storage: row %llu, element %llu is %g, which rounds to infinity in fp16 (|x| >= 65520)", r,
                    i, (double)x);
    if (ix.row_type == kRowBin)
        return fail(IDB_ERR_INVALID_ARG, "bin storage: row %llu, element %llu is %g; bin rows must be 0 or 1", r, i, (double)x);
    if (!std::isfinite(x))
        return fail(IDB_ERR_INVALID_ARG, "q8 storage: row %llu, element %llu is %g; q8 rows must be finite", r, i, (double)x);
    return fail(IDB_ERR_INVALID_ARG, "q8 storage: row %llu, element %llu (%g): the row's dequantised values would overflow f32", r, i,
                (double)x);
}

}  // namespace

idb_status check_storage_metric(uint32_t storage, uint32_t metric) {
    if (storage == IDB_STORAGE_BIN && metric == IDB_METRIC_COSINE)
        return fail(IDB_ERR_UNSUPPORTED, "bin storage takes the squared L2 only: normalised rows are not 0/1");
    return IDB_OK;
}

StoredRows Index::stored() const { return StoredRows{d_rows, d_hdr, row_type, nchunks * 4, dim}; }

idb_status Index::put_rows(uint64_t r0, uint64_t m, const uint32_t* input_row, const std::function<cudaError_t(float*)>& fill) {
    if (m == 0) return IDB_OK;
    const size_t stride = (size_t)nchunks * 4;
    if (row_type == kRowF32) {  // staged in place: nothing to check or convert
        if (!d_rows) CUDA_TRY(alloc_store(*this, cap, &d_rows, &d_hdr));
        CUDA_TRY(fill(static_cast<float*>(d_rows) + r0 * stride));
        CUDA_TRY(cudaStreamSynchronize(stream));
        return IDB_OK;
    }
    float* staged = nullptr;
    CUDA_TRY(cudaMalloc(&staged, m * stride * 4));
    cudaError_t e = fill(staged);
    const idb_status s = e == cudaSuccess ? check_rows(*this, staged, m, input_row) : IDB_OK;
    if (s == IDB_OK && e == cudaSuccess && !d_rows) e = alloc_store(*this, cap, &d_rows, &d_hdr);
    if (s == IDB_OK && e == cudaSuccess) {
        char* dst = static_cast<char*>(d_rows) + r0 * row_bytes();
        if (row_type == kRowBin)
            pack_bin_kernel<<<num_sms * 8, 256, 0, stream>>>(staged, reinterpret_cast<uint8_t*>(dst), m * nchunks);
        else if (row_type == kRowQ8)  // normalised first (a cosine index), then quantised
            quantize_q8_kernel<<<num_sms * 8, 256, 0, stream>>>(staged, m, (uint32_t)stride, dim, reinterpret_cast<uint8_t*>(dst), d_hdr + r0);
        else if (row_type == kRowF16)  // normalised first, then rounded
            narrow_f16_kernel<<<num_sms * 8, 256, 0, stream>>>(staged, reinterpret_cast<uint16_t*>(dst), m * stride);
        else
            narrow_bf16_kernel<<<num_sms * 8, 256, 0, stream>>>(staged, reinterpret_cast<uint16_t*>(dst), m * stride);
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    }
    cudaFree(staged);
    CUDA_TRY(e);
    return s;
}

size_t Index::row_bytes() const { return (size_t)nchunks * chunk_bytes(row_type); }

cudaError_t Index::alloc_rows(uint64_t rows, void** pts, float2** hdr) const { return alloc_store(*this, rows, pts, hdr); }

cudaError_t Index::copy_rows_in(float* dst, const float* src, uint64_t m) const {
    const size_t stride = (size_t)nchunks * 4;
    if (stride == dim) return cudaMemcpyAsync(dst, src, m * stride * 4, cudaMemcpyHostToDevice, stream);
    cudaError_t e = cudaMemsetAsync(dst, 0, m * stride * 4, stream);
    if (e == cudaSuccess) e = cudaMemcpy2DAsync(dst, stride * 4, src, dim * 4, dim * 4, m, cudaMemcpyHostToDevice, stream);
    return e;
}

idb_status Index::reserve_rows(uint64_t rows) {
    if (rows <= cap) return IDB_OK;
    const uint64_t want = std::max<uint64_t>(rows, 2 * cap);
    const size_t bytes = row_bytes(), width = 2 * (size_t)M;
    void* pts = nullptr;
    float2* hdr = nullptr;
    uint32_t* zero = nullptr;  // the one adjacency layer allocated outside graph.cu: it grows with the rows, all or nothing
    uint32_t* id_map = nullptr;
    cudaError_t e = alloc_store(*this, want, &pts, &hdr);
    if (e == cudaSuccess) e = cudaMalloc(&zero, want * width * 4);
    if (e == cudaSuccess && d_id_map) e = cudaMalloc(&id_map, want * 4);
    if (e == cudaSuccess && n) {
        e = cudaMemcpyAsync(pts, d_rows, n * bytes, cudaMemcpyDeviceToDevice, stream);
        if (e == cudaSuccess && hdr) e = cudaMemcpyAsync(hdr, d_hdr, n * sizeof(float2), cudaMemcpyDeviceToDevice, stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(zero, graph.zero, n * width * 4, cudaMemcpyDeviceToDevice, stream);
        if (e == cudaSuccess && d_id_map) e = cudaMemcpyAsync(id_map, d_id_map, n * 4, cudaMemcpyDeviceToDevice, stream);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) {
        cudaFree(pts);
        cudaFree(hdr);
        cudaFree(zero);
        cudaFree(id_map);
        CUDA_TRY(e);
    }
    cudaFree(d_rows);
    cudaFree(d_hdr);
    cudaFree(graph.zero);
    cudaFree(d_id_map);
    d_rows = pts;
    d_hdr = hdr;
    graph.zero = zero;
    d_id_map = id_map;
    cap = want;
    return IDB_OK;
}

idb_status Index::copy_points_f32(float* host_out, uint64_t r0, uint64_t m) {
    if (m == 0) return IDB_OK;
    const size_t stride = (size_t)nchunks * 4;
    if (row_type == kRowF32) {
        CUDA_TRY(cudaMemcpy2DAsync(host_out, dim * 4, static_cast<const float*>(d_rows) + r0 * stride, stride * 4, dim * 4, m,
                                   cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        return IDB_OK;
    }
    float* tmp = nullptr;
    CUDA_TRY(cudaMalloc(&tmp, m * stride * 4));
    widen_rows_kernel<<<num_sms * 8, 256, 0, stream>>>(stored(), r0, m, tmp);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpy2DAsync(host_out, dim * 4, tmp, stride * 4, dim * 4, m, cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    cudaFree(tmp);
    CUDA_TRY(e);
    return IDB_OK;
}

}  // namespace idb
