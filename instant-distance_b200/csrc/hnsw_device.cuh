// hnsw_device.cuh — warp-level HNSW traversal for sm_90a (one warp per live query / insert).
//
// Restates, as a warp-synchronous data-parallel program, the reference's
//   Search::search  (search_layer, Alg. 2)   instant-distance/src/lib.rs:598-614
//   Search::push                              lib.rs:704-720
//   Search::cull / reset                      lib.rs:729-755
//   Hnsw::search driver                       lib.rs:352-383   (and Construction::insert's descent, lib.rs:443-463)
//   Visited                                   types.rs:13-59
//   NearestIter + take(links)                 types.rs:172-192, lib.rs:606
//   Candidate ordering                        types.rs:228-234
// The traversal is BIT-IDENTICAL to the sequential reference (same expansions, same distance evaluations,
// same result list), see DESIGN.md "exactness under parallel execution":
//   * `nearest` is a sorted array of u64 keys  (canonical distance bits << 32 | pid)  in shared memory;
//     bit 63 (the sign bit of the non-negative distance) flags "already expanded".
//   * `candidates` is never materialised: it equals {unexpanded entries of nearest} U {tie list}, where the
//     tie list holds evicted, unexpanded, ADMITTED candidates whose distance equals the current furthest
//     distance (the reference's stop test is strict `>` and distance-only, lib.rs:601).
//   * a whole row (<= 2M ids) is processed at once: visited test-and-set per lane, distances 32 at a time,
//     admission resolved by the row-order rank rule  rank_S(x) + #{earlier admitted < x} < ef  (lib.rs:712-714).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace idb {

constexpr uint32_t kInvalid = 0xFFFFFFFFu;
constexpr uint64_t kFlagExpanded = 1ull << 63;
constexpr uint64_t kKeyMask = ~kFlagExpanded;
constexpr uint64_t kKeyNone = ~0ull;          // sorts after every real key (real dist bits <= 0x7fc00000)
constexpr int kSmallVisSlots = 512;           // shared-memory visited set used on the ef=1 layers
constexpr int kTieCap = 1024;                 // per-warp tie list capacity (global memory); the retry pool has kRetryTieCap
constexpr int kRetryTieCap = 1 << 16;
constexpr uint32_t kFullMask = 0xFFFFFFFFu;

enum OptFlags : uint32_t { kOptPrefetchVectors = 1u, kOptPrefetchRows = 2u, kOptPrefetchNextRow = 8u };

// How an index stores its rows; the values are the ABI's IDB_STORAGE_* (internal.cuh checks that).
enum RowType : uint32_t { kRowF32 = 0, kRowBF16 = 1, kRowF16 = 2, kRowQ8 = 4, kRowBin = 8 };

enum QueryStatus : uint32_t { kQueryOk = 0, kQueryVisitedOverflow = 1, kQueryTieOverflow = 2 };

struct GraphView {
    const char* points;          // n rows of nchunks 4-element chunks (dim rounded up to 4, zero padded); f32 (16 B/chunk), bf16 or fp16
                                 // (8 B/chunk), q8 (4 B/chunk: one code byte per element), bin (1 B/chunk: one bit per element)
    uint32_t nchunks;            // 4-element chunks per row
    const uint32_t* zero;        // n x 2M
    const uint32_t* const* upper;  // device array: upper[l-1] = n_l x M
    uint32_t n_upper;
    uint32_t M;
    uint64_t n;
    uint32_t flags;              // kOpt* tuning switches (never change results)
    uint32_t row_type;           // RowType (= IDB_STORAGE_*): how the rows are stored; arithmetic stays fp32
    // Screening table (DESIGN §2, §4), or null: K1 then fetches every candidate row in full.
    const uint32_t* codes;       // n rows of cwords u32: word c < nchunks holds the 8-bit codes of elements 4c..4c+3 (byte k = element
                                 // 4c+k); words [nchunks, cwords) are zero
    uint32_t cwords;             // code_words(nchunks): every code row starts 16-byte aligned
    const float4* cparams;       // 3 x nchunks float4: per element scale, offset, E (x~ = fmaf(code, scale, offset), |x - x~| <= E)
    float cstep;                 // S: the one code step of every element (the scale slots of cparams all hold it)
    float cerr;                  // R >= ||x - x~|| over every stored row, x~_i = offset_i + code_i * S in real arithmetic
    // q8 rows (DESIGN §3c), else unused: row r's header {o, s} (element i = fmaf(code_i, s, o)), and how many elements of the last
    // chunk belong to the row (1..4; the codes of the padding do not widen to zero, so the loaders zero them)
    const float2* hdr;
    uint32_t tail;
};
// u32 words per screening-table row: nchunks rounded up to 4, so the screen reads a row in 16-byte words (DESIGN §2)
__host__ __device__ constexpr uint32_t code_words(uint32_t nchunks) { return (nchunks + 3u) & ~3u; }

// ---------------------------------------------------------------------------------------------------------
// Canonical squared-L2 (DESIGN.md "canonical distance"; the CPU checker restates the same order):
//   lane l owns float4 chunks l, l+32, l+64, ...; four fmaf chains (one per float4 component);
//   lane sum (a0+a1)+(a2+a3); xor butterfly over lanes with offsets 1, 2, 4, 8, 16.
// ---------------------------------------------------------------------------------------------------------
// One step of the four fmaf chains: acc.c = fma(q.c - v.c, q.c - v.c, acc.c) per component, every operation IEEE round-to-nearest
// (explicit intrinsics, so the compiler cannot contract or reorder them).
__device__ __forceinline__ void l2_step(float4& acc, const float4& q, const float4& v) {
    const float dx = __fsub_rn(q.x, v.x), dy = __fsub_rn(q.y, v.y), dz = __fsub_rn(q.z, v.z), dw = __fsub_rn(q.w, v.w);
    acc.x = __fmaf_rn(dx, dx, acc.x);
    acc.y = __fmaf_rn(dy, dy, acc.y);
    acc.z = __fmaf_rn(dz, dz, acc.z);
    acc.w = __fmaf_rn(dw, dw, acc.w);
}
__device__ __forceinline__ float lane_sum(const float4& a) { return __fadd_rn(__fadd_rn(a.x, a.y), __fadd_rn(a.z, a.w)); }
template <int CH>
__device__ __forceinline__ float lane_partial(const float4 (&q)[CH], const float4 (&v)[CH]) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);  // the four fmaf chains a0..a3 of the canonical order
#pragma unroll
    for (int j = 0; j < CH; ++j) l2_step(acc, q[j], v[j]);
    return lane_sum(acc);
}

// Row storage types.  A lane always owns the same 4 ELEMENTS per 128-element block (chunk l, l+32, ...), so the canonical
// fp32 summation order is the same for all of them; bf16 and fp16 rows are widened exactly (bf16 -> f32 is a 16-bit shift, fp16 -> f32
// is cvt.f32.f16, exact for every fp16 value, subnormals included), and so are q8 rows (DESIGN §3c: (b + c) 2^e is an f32, so
// fmaf(c, 2^e, b 2^e) is exact however it is evaluated).
// `Raw` is what a lane keeps in registers while a batch of row loads is in flight (bf16 / fp16 / q8 rows stay packed: a half or a
// quarter of the registers per row, so more rows in flight); widen() runs at the point of use.  `Hdr` is what a row carries besides its
// chunks, fetched once per row with hdr(): empty except for q8, whose rows have a grid of their own.
struct NoHdr {};
struct RowF32 {
    static constexpr uint32_t kType = kRowF32;
    static constexpr uint32_t kChunkBytes = 16;
    using Raw = float4;
    using Hdr = NoHdr;
    static __device__ __forceinline__ Hdr hdr(const GraphView&, uint32_t) { return Hdr(); }
    static __device__ __forceinline__ Raw ld_raw(const char* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
    static __device__ __forceinline__ Raw zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
    static __device__ __forceinline__ float4 widen(Raw r, Hdr) { return r; }
    static __device__ __forceinline__ float4 ld(const char* p, Hdr h) { return widen(ld_raw(p), h); }
};
struct RowBF16 {
    static constexpr uint32_t kType = kRowBF16;
    static constexpr uint32_t kChunkBytes = 8;
    using Raw = uint2;
    using Hdr = NoHdr;
    static __device__ __forceinline__ Hdr hdr(const GraphView&, uint32_t) { return Hdr(); }
    static __device__ __forceinline__ Raw ld_raw(const char* p) { return __ldg(reinterpret_cast<const uint2*>(p)); }
    static __device__ __forceinline__ Raw zero() { return make_uint2(0u, 0u); }
    static __device__ __forceinline__ float4 widen(Raw u, Hdr) {
        return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xFFFF0000u), __uint_as_float(u.y << 16),
                           __uint_as_float(u.y & 0xFFFF0000u));
    }
    static __device__ __forceinline__ float4 ld(const char* p, Hdr h) { return widen(ld_raw(p), h); }
};
// The two fp16 values packed in u (element 2i in the low half), widened exactly.
__device__ __forceinline__ float2 widen_f16x2(uint32_t u) {
    float2 f;
    asm("{\n\t.reg .b16 lo, hi;\n\tmov.b32 {lo, hi}, %2;\n\tcvt.f32.f16 %0, lo;\n\tcvt.f32.f16 %1, hi;\n\t}"
        : "=f"(f.x), "=f"(f.y)
        : "r"(u));
    return f;
}
struct RowF16 {
    static constexpr uint32_t kType = kRowF16;
    static constexpr uint32_t kChunkBytes = 8;
    using Raw = uint2;
    using Hdr = NoHdr;
    static __device__ __forceinline__ Hdr hdr(const GraphView&, uint32_t) { return Hdr(); }
    static __device__ __forceinline__ Raw ld_raw(const char* p) { return __ldg(reinterpret_cast<const uint2*>(p)); }
    static __device__ __forceinline__ Raw zero() { return make_uint2(0u, 0u); }
    static __device__ __forceinline__ float4 widen(Raw u, Hdr) {
        const float2 a = widen_f16x2(u.x), b = widen_f16x2(u.y);
        return make_float4(a.x, a.y, b.x, b.y);
    }
    static __device__ __forceinline__ float4 ld(const char* p, Hdr h) { return widen(ld_raw(p), h); }
};
// q8 (DESIGN §3c): one code byte per element (byte k of a chunk's word = element 4c+k, the screening codes' layout) and a per-row
// header {o, s} = {b 2^e, 2^e}; element i = fmaf(c_i, s, o), exact.  A zero Hdr widens every code to 0 (rows past the batch).
struct RowQ8 {
    static constexpr uint32_t kType = kRowQ8;
    static constexpr uint32_t kChunkBytes = 4;
    using Raw = uint32_t;
    using Hdr = float2;
    static __device__ __forceinline__ Hdr hdr(const GraphView& g, uint32_t pid) { return __ldg(g.hdr + pid); }
    static __device__ __forceinline__ Raw ld_raw(const char* p) { return __ldg(reinterpret_cast<const uint32_t*>(p)); }
    static __device__ __forceinline__ Raw zero() { return 0u; }
    static __device__ __forceinline__ float4 widen(Raw u, Hdr h) {
        return make_float4(__fmaf_rn((float)(u & 0xFFu), h.y, h.x), __fmaf_rn((float)((u >> 8) & 0xFFu), h.y, h.x),
                           __fmaf_rn((float)((u >> 16) & 0xFFu), h.y, h.x), __fmaf_rn((float)(u >> 24), h.y, h.x));
    }
    static __device__ __forceinline__ float4 ld(const char* p, Hdr h) { return widen(ld_raw(p), h); }
};
// bin (DESIGN §3d): 0/1 elements, one byte per chunk (bit k of byte c = element 4c+k, high nibble zero), so a warp's 32 chunks are
// 32 contiguous bytes.  Each bit widens to exactly 0.f or 1.f, and the zero padding to 0.f.
struct RowBin {
    static constexpr uint32_t kType = kRowBin;
    static constexpr uint32_t kChunkBytes = 1;
    using Raw = uint32_t;
    using Hdr = NoHdr;
    static __device__ __forceinline__ Hdr hdr(const GraphView&, uint32_t) { return Hdr(); }
    static __device__ __forceinline__ Raw ld_raw(const char* p) { return __ldg(reinterpret_cast<const unsigned char*>(p)); }
    static __device__ __forceinline__ Raw zero() { return 0u; }
    static __device__ __forceinline__ float4 widen(Raw u, Hdr) {
        return make_float4((float)(u & 1u), (float)((u >> 1) & 1u), (float)((u >> 2) & 1u), (float)((u >> 3) & 1u));
    }
    static __device__ __forceinline__ float4 ld(const char* p, Hdr h) { return widen(ld_raw(p), h); }
};
// f(RT()) for the row type `row_type` of an index: the one place a run-time row type becomes a template argument.
template <class F>
auto with_row_type(uint32_t row_type, F&& f) {
    if (row_type == kRowBF16) return f(RowBF16());
    if (row_type == kRowF16) return f(RowF16());
    if (row_type == kRowQ8) return f(RowQ8());
    if (row_type == kRowBin) return f(RowBin());
    return f(RowF32());
}
// Chunk c of a row, widened.  The zero padding of f32 / bf16 / fp16 rows, and the zero Raw loaders put in place of chunks past the
// row, widen to zeros.  q8 codes widen to o instead, so for q8 the elements past the row (in its last chunk, and every chunk c >=
// nchunks) are zeroed here.  (FULL cells too: every chunk is real there, but the last one may still end past dim.)
template <class RT>
__device__ __forceinline__ float4 widen_chunk(const GraphView& g, typename RT::Raw r, typename RT::Hdr h, uint32_t c) {
    float4 v = RT::widen(r, h);
    if constexpr (RT::kType == kRowQ8) {
        if (c + 1u >= g.nchunks) {
            const uint32_t t = c + 1u == g.nchunks ? g.tail : 0u;
            if (t < 1u) v.x = 0.f;
            if (t < 2u) v.y = 0.f;
            if (t < 3u) v.z = 0.f;
            if (t < 4u) v.w = 0.f;
        }
    }
    return v;
}
// This lane's CH chunks of row `pid` (zeros beyond the row's last chunk).
template <int CH, class RT>
__device__ __forceinline__ void load_row(const GraphView& g, uint32_t pid, int lane, float4 (&q)[CH]) {
    const char* row = g.points + (size_t)pid * (g.nchunks * RT::kChunkBytes) + lane * RT::kChunkBytes;
    const typename RT::Hdr h = RT::hdr(g, pid);
#pragma unroll
    for (int j = 0; j < CH; ++j)
        q[j] = (uint32_t)(lane + 32 * j) < g.nchunks ? widen_chunk<RT>(g, RT::ld_raw(row + j * 32 * RT::kChunkBytes), h, lane + 32 * j)
                                                     : make_float4(0.f, 0.f, 0.f, 0.f);
}

template <int CH, class RT>
__device__ __forceinline__ float lane_partial_raw(const GraphView& g, const float4 (&q)[CH], const typename RT::Raw (&r)[CH],
                                                  typename RT::Hdr h, int lane) {
    float4 v[CH];
#pragma unroll
    for (int j = 0; j < CH; ++j) v[j] = widen_chunk<RT>(g, r[j], h, lane + 32 * j);
    return lane_partial<CH>(q, v);
}

// The query / owner row of a traversal as one lane sees it.  CH >= 1: the lane's CH chunks in registers (rows of up to
// 128 * CH elements, one kernel instantiation per CH).  CH == 0 ("long rows", any dim): the whole row, widened to f32 and zero
// padded to a multiple of 32 chunks, in this warp's shared memory; distances then run over groups of 32 chunks in ascending
// order — the same fmaf chains in the same order as the register flavour (DESIGN.md "canonical distance").
template <int CH>
struct QVec {
    float4 r[CH];
};
template <>
struct QVec<0> {
    float4* s;         // shared: ngroups * 32 chunks
    uint32_t ngroups;  // ceil(nchunks / 32)
};
constexpr int kLongRowsInFlight = 8;
// q <- an f32 row of nchunks chunks (a query of the batch)
template <int CH>
__device__ __forceinline__ void q_from_f32(QVec<CH>& q, const float4* row, uint32_t nchunks, int lane) {
    if constexpr (CH == 0) {
        for (uint32_t c = lane; c < q.ngroups * 32u; c += 32) q.s[c] = c < nchunks ? __ldg(row + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        __syncwarp();
    } else {
#pragma unroll
        for (int j = 0; j < CH; ++j) {
            const uint32_t c = lane + 32 * j;
            q.r[j] = c < nchunks ? __ldg(row + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
}
// q <- point row `pid` (any row type, widened)
template <int CH, class RT>
__device__ __forceinline__ void q_from_point(QVec<CH>& q, const GraphView& g, uint32_t pid, int lane) {
    if constexpr (CH == 0) {
        const char* row = g.points + (size_t)pid * (g.nchunks * RT::kChunkBytes);
        const typename RT::Hdr h = RT::hdr(g, pid);
        __syncwarp();  // earlier readers of the buffer are done
        for (uint32_t c = lane; c < q.ngroups * 32u; c += 32)
            q.s[c] = c < g.nchunks ? widen_chunk<RT>(g, RT::ld_raw(row + (size_t)c * RT::kChunkBytes), h, c) : make_float4(0.f, 0.f, 0.f, 0.f);
        __syncwarp();
    } else {
        load_row<CH, RT>(g, pid, lane, q.r);
    }
}

// Butterfly for ONE vector (offsets 1, 2, 4, 8, 16 — the canonical order): every lane ends with the total.
__device__ __forceinline__ float butterfly_sum(float s) {
#pragma unroll
    for (int off = 1; off <= 16; off <<= 1) s = __fadd_rn(s, __shfl_xor_sync(kFullMask, s, off));
    return s;
}

// Butterfly for NB (power of two <= 32) vectors at once: p[i] is this lane's partial for vector i.  The first
// log2(NB) stages are "transposing" (each lane hands half of its values to its partner and keeps the other half,
// split by even/odd index), so NB vectors cost NB-1 shuffles instead of 5*NB; the remaining stages are plain.
// Same add tree as butterfly_sum for every vector.  On return lane l holds the total of vector (l & (NB-1)).
// kDown: every add rounds toward -inf instead.  u32 partials (the screen's squared code distances) add exactly, in any order.
// W < 32 (u32 partials only): the sums run over each aligned group of W lanes on its own (offsets below W).
template <bool kDown>
__device__ __forceinline__ float fadd_dir(float a, float b) { return kDown ? __fadd_rd(a, b) : __fadd_rn(a, b); }
template <bool kDown>
__device__ __forceinline__ uint32_t fadd_dir(uint32_t a, uint32_t b) { return a + b; }
// c ? a : b as one SELP on the two values: a C++ `up ? p[2i] : p[2i+1]` may be folded into one load from a selected address, which
// indexes p at run time and puts it on the stack.
__device__ __forceinline__ float sel(bool c, float a, float b) {
    float r;
    asm("{ .reg .pred p; setp.ne.u32 p, %3, 0; selp.f32 %0, %1, %2, p; }" : "=f"(r) : "f"(a), "f"(b), "r"((uint32_t)c));
    return r;
}
__device__ __forceinline__ uint32_t sel(bool c, uint32_t a, uint32_t b) {
    uint32_t r;
    asm("{ .reg .pred p; setp.ne.u32 p, %3, 0; selp.b32 %0, %1, %2, p; }" : "=r"(r) : "r"(a), "r"(b), "r"((uint32_t)c));
    return r;
}
// The transposing stage at offset OFF, M vectors left, and the stages after it.  One template per stage, so that every loop below
// has a constant trip count: as one loop nest over m, the inner loop (trip count m / 2) was unrolled by four before m was known,
// which indexed p at run time and put it on the stack (64 bytes at NB = 16).
template <int M, int OFF, bool kDown, class T, int NB>
__device__ __forceinline__ void butterfly_stages(T (&p)[NB], int lane) {
    if constexpr (M > 1) {
        const bool up = (lane & OFF) != 0;
#pragma unroll
        for (int i = 0; i < M / 2; ++i) {
            const T send = sel(up, p[2 * i], p[2 * i + 1]);
            const T keep = sel(up, p[2 * i + 1], p[2 * i]);
            p[i] = fadd_dir<kDown>(keep, __shfl_xor_sync(kFullMask, send, OFF));
        }
        butterfly_stages<M / 2, 2 * OFF, kDown>(p, lane);
    }
}
template <int NB, bool kDown = false, class T = float, int W = 32>
__device__ __forceinline__ T batch_butterfly(T (&p)[NB], int lane) {
    static_assert(NB <= W, "one vector per lane of a group at most");
    butterfly_stages<NB, 1, kDown>(p, lane);
#pragma unroll
    for (int o = NB; o < W; o <<= 1) p[0] = fadd_dir<kDown>(p[0], __shfl_xor_sync(kFullMask, p[0], o));
    return p[0];
}

// ---------------------------------------------------------------------------------------------------------
// Cosine distance (DESIGN.md §3a): the canonical squared L2 between canonically normalised rows; the caller is told half of it.
// ---------------------------------------------------------------------------------------------------------
enum Metric : uint32_t { kMetricL2Sq = 0, kMetricCosine = 1 };  // = IDB_METRIC_*

// Chunk c of a row of `dim` elements at any alignment (zeros beyond the row).
__device__ __forceinline__ float4 load_chunk_any(const float* row, uint32_t dim, uint32_t c) {
    const uint32_t e = 4 * c;
    return make_float4(e < dim ? row[e] : 0.f, e + 1 < dim ? row[e + 1] : 0.f, e + 2 < dim ? row[e + 2] : 0.f, e + 3 < dim ? row[e + 3] : 0.f);
}

// The ONE statement of the canonical normalisation, x^ = x / sqrt_rn(s): s = the canonical sum of squares, i.e. the §3 order
// against a zero row (x - 0 == x for every float) in its long-row form — groups of 32 chunks in ascending order carrying the four
// chains, lane_sum, butterfly_sum — then __fsqrt_rn and __fdiv_rn, both correctly rounded.  s == 0: the row stays all zeros;
// s == inf: zeros and NaN (the IEEE result).  A NaN result is written as 0x7fc00000 (the GPU's and the CPU's divide return different
// NaN encodings).  The whole warp calls it.  src: `dim` elements, any alignment; dst: `nchunks` chunks, zero padded.  dst may
// alias src: every lane reads its own chunks before it writes them.
__device__ __forceinline__ float canon_nan(float v) { return isnan(v) ? __int_as_float(0x7fc00000) : v; }
__device__ __forceinline__ void normalize_row(const float* src, uint32_t dim, float4* dst, uint32_t nchunks, int lane) {
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 acc = zero;
    for (uint32_t c = lane; c < nchunks; c += 32) l2_step(acc, load_chunk_any(src, dim, c), zero);
    const float s = butterfly_sum(lane_sum(acc));
    const float r = __fsqrt_rn(s);
    for (uint32_t c = lane; c < nchunks; c += 32) {
        const float4 x = load_chunk_any(src, dim, c);
        const uint32_t e = 4 * c;
        float4 y = zero;
        if (s != 0.f) {
            y.x = canon_nan(__fdiv_rn(x.x, r));  // (element e < dim always: c < nchunks)
            y.y = e + 1 < dim ? canon_nan(__fdiv_rn(x.y, r)) : 0.f;
            y.z = e + 2 < dim ? canon_nan(__fdiv_rn(x.z, r)) : 0.f;
            y.w = e + 3 < dim ? canon_nan(__fdiv_rn(x.w, r)) : 0.f;
        }
        dst[c] = y;
    }
}

// What the caller is told for a key's canonical distance bits.  Squared L2: the distance itself.  Cosine: 0.5 * ‖x^ - y^‖² =
// 1 - cos (exact for normal floats), NaN written as the canonical 0x7fc00000 (a multiply would return 0x7fffffff), +inf stays +inf.
__device__ __forceinline__ float reported_distance(uint32_t dbits, uint32_t metric) {
    const float d = __uint_as_float(dbits);
    if (metric == kMetricL2Sq) return d;
    return dbits == 0x7fc00000u ? d : __fmul_rn(0.5f, d);
}

__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

__device__ __forceinline__ uint32_t canon_bits(float d) {
    uint32_t b = __float_as_uint(d);
    if ((b & 0x7fffffffu) > 0x7f800000u) b = 0x7fc00000u;  // NaN: greatest, equal to itself (ordered-float)
    if (b == 0x80000000u) b = 0u;
    return b;
}
__device__ __forceinline__ uint64_t mk_key(float d, uint32_t pid) { return ((uint64_t)canon_bits(d) << 32) | pid; }
__device__ __forceinline__ uint32_t key_pid(uint64_t k) { return (uint32_t)k; }
__device__ __forceinline__ uint32_t key_dbits(uint64_t k) { return (uint32_t)((k & kKeyMask) >> 32); }
__device__ __forceinline__ uint64_t shfl64(uint64_t v, int src) {
    uint32_t lo = __shfl_sync(kFullMask, (uint32_t)v, src), hi = __shfl_sync(kFullMask, (uint32_t)(v >> 32), src);
    return ((uint64_t)hi << 32) | lo;
}

// ---------------------------------------------------------------------------------------------------------
// Visited (types.rs:13-59): exact set of PointIds.  Two tiers, both open addressing with linear probing:
//   small: kSmallVisSlots u32 in shared memory (the ef=1 layers touch ~30 ids per layer);
//   big:   `gslots` u32 in global memory, private to this warp, L2 resident (layer 0 / ef_construction).
// `clear()` (lib.rs:735, 750) wipes whichever tier is live.  Empty slot = kInvalid (never a valid PointId).
// ---------------------------------------------------------------------------------------------------------
struct VisitedSet {
    uint32_t* small;   // shared
    uint32_t* big;     // global
    uint32_t gslots;   // words in use: hash slots (power of two) / bitmap words / 8 * buckets + kB16Stash (b16)
    uint32_t gshift;   // hash flavour: 32 - log2(gslots)
    uint32_t count;
    bool use_big;
    uint32_t mode;     // flavour of the big tier (VisMode).  A clean table is all ones (kInvalid) in every flavour
    uint32_t nb;       // b16 flavour: buckets in use: [0, nb_lo) in `big` (followed by the stash), [nb_lo, nb) in `big_hi`
    uint32_t nb_lo;
    uint32_t* big_hi;  // b16 flavour: second segment (outside the persisting-L2 window), pre-offset so that bucket b is at big_hi + 8 * b
    float nb_inv;      // 1 / nb
    uint32_t cap_ids;  // b16 flavour: ids the table may hold before the query is handed to the retry pass
    uint32_t stash_cnt;  // b16 flavour: ids in the stash (warp-uniform)
    uint32_t* hist;    // shared, 512 words = 2048 one-byte tallies, one per bucket: slots handed out since the snapshots of the current row
                       // were taken (b16 flavour).  Aliases `small`, which is idle (and clean) whenever the big tier is live and is
                       // wiped again when the warp goes back to it — hence at most 2048 buckets (64 KB) per table
};
// Big-tier flavours, all exact:
//   kVisHash    open addressing, one u32 slot per id, atomicCAS + linear probing (any n; the retry pass and the fallback)
//   kVisBitmap  n bits, bit SET = not visited, one atomicAnd per id (n / 8 bytes per warp: DRAM resident)
//   kVisB16     32-byte buckets of 16 u16 slots, filled in order, NO atomics (the table is private to the warp and the warp
//               arbitrates its own lanes with match/ballot).  slot = 15-bit tag | bit 15 "displaced by one bucket";
//               (home bucket, tag) is an injective function of the PointId, so the set is exact for n <= buckets * 32768.
//               ~2 slots per id a query can possibly visit: the tables of all resident warps together fit the persisting part
//               of L2 (K1's and KA's default): a probe is ONE 32-byte read of an L2-resident sector, an insert one 2-byte
//               store nobody waits for.
enum VisMode : uint32_t { kVisHash = 0, kVisBitmap = 1, kVisB16 = 2 };

__device__ __forceinline__ uint32_t vis_hash(uint32_t pid) { return pid * 0x9E3779B1u; }

__device__ __forceinline__ bool vis_insert_small(uint32_t* tab, uint32_t pid) {
    uint32_t h = vis_hash(pid) >> (32 - 9);
    static_assert(kSmallVisSlots == 512, "shift above assumes 512 slots");
    for (;;) {
        uint32_t old = atomicCAS(&tab[h], kInvalid, pid);
        if (old == kInvalid) return true;
        if (old == pid) return false;
        h = (h + 1) & (kSmallVisSlots - 1);
    }
}
__device__ __forceinline__ bool vis_insert_big(uint32_t* tab, uint32_t gshift, uint32_t gmask, uint32_t pid) {
    uint32_t h = vis_hash(pid) >> gshift;
    for (;;) {
        uint32_t old = atomicCAS(&tab[h], kInvalid, pid);
        if (old == kInvalid) return true;
        if (old == pid) return false;
        h = (h + 1) & gmask;
    }
}

// Bitmap flavour of the big tier: one atomic per id, no probe chains, never overflows.
__device__ __forceinline__ uint32_t vis_bitmap_fetch_clear(uint32_t* tab, uint32_t pid) {
    return atomicAnd(tab + (pid >> 5), ~(1u << (pid & 31)));
}

// ---- b16 bucket set --------------------------------------------------------------------------------------
// Invariants (no deletions, slots of a bucket are filled in order 0..15):
//   * an id lives in its home bucket if that bucket had a free slot when the id was inserted; else, flagged "displaced", in its
//     alternate bucket (home + a step derived from the tag: double hashing, still invertible); else, as a full PointId, in a
//     64-entry stash behind the buckets.  So "not in the home bucket, and the home bucket still has a free slot" proves absence
//     with ONE 32-byte read, and only ids whose home bucket is full ever look further;
//   * the warp owns the table: concurrent inserts only ever come from lanes of this warp handling the same adjacency row, and
//     those are arbitrated in registers (match_any on the home bucket) plus an exact per-bucket tally in shared memory (one byte
//     per bucket) for row entries that live in different registers, so inserts are plain stores and nobody waits for them.
//   * PointIds within one adjacency row are distinct (true for every graph this library or the reference builds; adopted graphs
//     are checked at upload and fall back to the atomic flavours if a row repeats an id).
constexpr uint32_t kB16Stash = 64;  // u32 words behind the buckets: ids whose home and alternate buckets were both full
struct Bucket8 { uint4 lo, hi; };
struct B16 { uint32_t home, tag; };
__device__ __forceinline__ uint32_t* bucket_ptr(const VisitedSet& v, uint32_t b) { return (b < v.nb_lo ? v.big : v.big_hi) + (size_t)b * 8; }
__device__ __forceinline__ Bucket8 bucket_load(const VisitedSet& v, uint32_t b) {
    const uint4* p = reinterpret_cast<const uint4*>(bucket_ptr(v, b));
    Bucket8 r;
    r.lo = __ldcg(p);      // L2 (never L1: other lanes of this warp write these sectors)
    r.hi = __ldcg(p + 1);
    return r;
}
__device__ __forceinline__ void b16_store(const VisitedSet& v, uint32_t b, uint32_t pos, uint32_t val16) {
    unsigned short* p = reinterpret_cast<unsigned short*>(bucket_ptr(v, b)) + pos;
    asm volatile("st.global.cg.u16 [%0], %1;" ::"l"(p), "h"((unsigned short)val16) : "memory");
}
// (home bucket, 15-bit tag) of a PointId: tag = low 15 bits, home = (pid >> 15) + scramble(tag) mod nb.  Injective while
// ceil(n / 32768) <= nb (checked on the host): given (home, tag) the group pid >> 15 is (home - scramble(tag)) mod nb.
__device__ __forceinline__ B16 b16_of(const VisitedSet& v, uint32_t pid) {
    B16 r;
    r.tag = pid & 0x7FFFu;
    const uint32_t x = (pid >> 15) + ((r.tag * 0x9E3779B1u) >> 10);  // < 2^17 + 2^22: exact in fp32
    uint32_t q = (uint32_t)((float)x * v.nb_inv);
    int32_t rem = (int32_t)(x - q * v.nb);
    if (rem < 0) rem += (int32_t)v.nb;
    if (rem >= (int32_t)v.nb) rem -= (int32_t)v.nb;
    r.home = (uint32_t)rem;
    return r;
}
// does any of the 16 halfwords equal val16?  (x - 0x00010001) & ~x & 0x80008000 is non-zero iff x has a zero halfword.
__device__ __forceinline__ bool b16_has(const Bucket8& k, uint32_t val16) {
    const uint32_t p = val16 | (val16 << 16);
    const uint32_t w[8] = {k.lo.x, k.lo.y, k.lo.z, k.lo.w, k.hi.x, k.hi.y, k.hi.z, k.hi.w};
    uint32_t any = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const uint32_t x = w[i] ^ p;
        any |= (x - 0x00010001u) & ~x & 0x80008000u;
    }
    return any != 0;
}
// number of filled slots (slots fill in order, so the empty ones — 0xFFFF — are a suffix; with that invariant the halfword
// zero test is exact for every halfword, not only the lowest)
__device__ __forceinline__ uint32_t b16_count(const Bucket8& k) {
    const uint32_t w[8] = {k.lo.x, k.lo.y, k.lo.z, k.lo.w, k.hi.x, k.hi.y, k.hi.z, k.hi.w};
    uint32_t m = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const uint32_t x = ~w[i];
        m |= ((x - 0x00010001u) & ~x & 0x80008000u) >> i;  // bits 15-i and 31-i
    }
    return 16u - __popc(m);
}
// Per-bucket tally (one byte per bucket, <= 2048 buckets): how many slots of bucket b were handed out since the current row's
// snapshots were taken.  <= 128 per row (4 registers x 32 lanes), so a byte never carries into its neighbour.
__device__ __forceinline__ uint32_t b16_tally_add(VisitedSet& v, uint32_t b, uint32_t n) {
    const uint32_t sh = 8u * (b & 3u);
    return (atomicAdd(&v.hist[b >> 2], n << sh) >> sh) & 0xFFu;
}
// Exact insert by ONE lane on fresh data (the others wait): 1 inserted, 0 already there, 2 no room (home, alternate and stash full).
// *stashed is set when the id went to the stash (the caller bumps the warp-uniform stash count).
template <bool kTally>
__device__ __forceinline__ uint32_t b16_insert_slow(VisitedSet& v, B16 t, uint32_t pid, bool* stashed) {
    {
        const Bucket8 k = bucket_load(v, t.home);
        if (b16_has(k, t.tag)) return 0u;
        const uint32_t cnt = b16_count(k);
        if (cnt < 16u) {
            b16_store(v, t.home, cnt, t.tag);
            if (kTally) b16_tally_add(v, t.home, 1u);  // row entries in other registers hold an older snapshot of this bucket
            return 1u;
        }
    }
    if (t.tag != 0x7FFFu) {  // (0x8000 | 0x7FFF is the EMPTY pattern: such an id cannot be stored displaced)
        uint32_t b = t.home + 1u + ((t.tag * 0x85EBCA6Bu) >> 12) % (v.nb - 1u);  // step in [1, nb): a function of the tag alone
        if (b >= v.nb) b -= v.nb;
        const uint32_t val = 0x8000u | t.tag;
        const Bucket8 k = bucket_load(v, b);
        if (b16_has(k, val)) return 0u;
        const uint32_t cnt = b16_count(k);
        if (cnt < 16u) {
            b16_store(v, b, cnt, val);
            if (kTally) b16_tally_add(v, b, 1u);
            return 1u;
        }
    }
    uint32_t* stash = v.big + (size_t)v.nb_lo * 8;
    for (uint32_t i = 0; i < v.stash_cnt; ++i)
        if (__ldcg(stash + i) == pid) return 0u;
    if (v.stash_cnt >= kB16Stash) return 2u;
    __stcg(stash + v.stash_cnt, pid);
    *stashed = true;
    return 1u;
}
// Visited::insert (types.rs:32-40) for one id per lane, given the snapshot `bk` of its home bucket (loaded by the caller so that
// the snapshots of a whole row are in flight together).  Warp-uniform call.  kTally: other registers of the same row hold snapshots
// taken before this call's stores — the per-bucket tally (entries zeroed since the snapshots were taken, b16_tally_reset) keeps them
// consistent; a caller whose snapshot is fresh and who inserts one register of ids at a time passes false and never touches the tally.
// Returns true iff the id was not in the set; *ovf on overflow.
template <bool kTally>
__device__ __forceinline__ bool b16_commit(VisitedSet& v, B16 tg, uint32_t pid, const Bucket8& bk, bool want, int lane, bool* ovf) {
    bool isnew = false, slow = false;
    uint32_t cnt = 0;
    if (want && !b16_has(bk, tg.tag)) {
        cnt = b16_count(bk);
        if (cnt >= 16u) slow = true;  // full: the id may live displaced in the next bucket
        else isnew = true;
    }
    const uint32_t peers = __match_any_sync(kFullMask, isnew ? tg.home : (0x80000000u | (uint32_t)lane));
    const int leader = __ffs(peers) - 1;
    uint32_t base = 0;
    if (kTally) {
        if (isnew && lane == leader) base = b16_tally_add(v, tg.home, (uint32_t)__popc(peers));
        base = __shfl_sync(kFullMask, base, leader);
    }
    if (isnew) {
        const uint32_t pos = cnt + base + __popc(peers & ((1u << lane) - 1u));
        if (pos < 16u) b16_store(v, tg.home, pos, tg.tag);
        else { isnew = false; slow = true; }
    }
    uint32_t sm = __ballot_sync(kFullMask, slow);
    while (sm) {  // rare: one lane at a time, on fresh data
        __syncwarp();  // orders the stores above / of the previous turn before this turn's loads
        const int src = __ffs(sm) - 1;
        sm &= sm - 1;
        bool stashed = false;
        if (lane == src) {
            const uint32_t r = b16_insert_slow<kTally>(v, tg, pid, &stashed);
            isnew = r == 1u;
            if (r == 2u) *ovf = true;
        }
        v.stash_cnt += __shfl_sync(kFullMask, stashed ? 1u : 0u, src);
    }
    __syncwarp();
    return isnew;
}
__device__ __forceinline__ void b16_tally_reset(VisitedSet& v, B16 tg) { reinterpret_cast<unsigned char*>(v.hist)[tg.home] = 0; }

// One id per lane into the big tier, any flavour.  Warp-uniform call (the b16 flavour is cooperative).
__device__ __forceinline__ bool vis_insert_big_any(VisitedSet& v, uint32_t pid, bool want, int lane, bool* ovf) {
    if (v.mode == kVisB16) {
        const B16 tg = b16_of(v, pid);
        Bucket8 bk;
        bk.lo = bk.hi = make_uint4(0u, 0u, 0u, 0u);
        if (want) bk = bucket_load(v, tg.home);  // a fresh snapshot, one register of ids: no tally needed
        return b16_commit<false>(v, tg, pid, bk, want, lane, ovf);
    }
    if (!want) return false;
    if (v.mode == kVisBitmap) return (vis_bitmap_fetch_clear(v.big, pid) >> (pid & 31)) & 1u;
    return vis_insert_big(v.big, v.gshift, v.gslots - 1, pid);
}

__device__ __forceinline__ void vis_clear_small(VisitedSet& v, int lane) {
#pragma unroll
    for (int i = 0; i < kSmallVisSlots / 32; ++i) v.small[lane + 32 * i] = kInvalid;
    __syncwarp();
}
__device__ __forceinline__ void vis_clear_big(VisitedSet& v, int lane) {
    uint4* p = reinterpret_cast<uint4*>(v.big);
    const uint4 e = make_uint4(kInvalid, kInvalid, kInvalid, kInvalid);
    for (uint32_t i = lane; i < v.gslots / 4; i += 32) __stcg(p + i, e);
    if (v.mode == kVisB16 && v.nb > v.nb_lo) {  // second segment of a large table
        uint4* ph = reinterpret_cast<uint4*>(v.big_hi + (size_t)v.nb_lo * 8);
        for (uint32_t i = lane; i < (v.nb - v.nb_lo) * 2; i += 32) __stcg(ph + i, e);
    }
    __threadfence();  // plain stores must be ordered before later atomics from other lanes
    __syncwarp();
}
// Visited::clear (types.rs:48-58); `next_big` selects the tier for the layer about to be searched.
__device__ __forceinline__ void vis_clear(VisitedSet& v, int lane, bool next_big) {
    if (v.use_big) {
        vis_clear_big(v, lane);
        if (v.mode == kVisB16) vis_clear_small(v, lane);  // the b16 tally lives in the small tier's shared memory
    } else {
        vis_clear_small(v, lane);
    }
    v.count = 0;
    v.stash_cnt = 0;
    v.use_big = next_big;
}
__device__ __forceinline__ void vis_migrate_to_big(VisitedSet& v, int lane) {
    bool ovf = false;  // (a few hundred ids into a table sized for thousands: cannot overflow)
#pragma unroll 1  // (cold path; these single-register inserts never touch the b16 tally, which shares this memory)
    for (int i = 0; i < kSmallVisSlots / 32; ++i) {
        const uint32_t x = v.small[lane + 32 * i];
        vis_insert_big_any(v, x, x != kInvalid, lane, &ovf);
    }
    __syncwarp();
    vis_clear_small(v, lane);
    v.use_big = true;
}
// Visited::insert (types.rs:32-40) for one id per lane, split in two so a lane can have the first probes of all its
// row entries in flight before it waits for any of them (atomic flavours; the b16 flavour has its own row path):
//   vis_probe  issues the first CAS and returns (old value, slot);  vis_settle follows the probe chain if needed.
// Returns false for lanes with !want.  Caller guarantees capacity via vis_reserve.  Warp-uniform calls.
struct VisProbe { uint32_t old, h; };
__device__ __forceinline__ VisProbe vis_probe(VisitedSet& v, uint32_t pid, bool want, int lane) {
    VisProbe r;
    r.old = 0u;
    if (v.use_big && v.mode == kVisBitmap) {
        r.h = pid >> 5;
        if (want) r.old = vis_bitmap_fetch_clear(v.big, pid);
        return r;
    }
    if (v.use_big && v.mode == kVisB16) {  // (rows take their own path in search_layer; this serves cull / the seed)
        bool ovf = false;                  // a handful of ids into an empty table: cannot overflow
        r.h = 0u;
        r.old = vis_insert_big_any(v, pid, want, lane, &ovf) ? 1u : 0u;
        return r;
    }
    r.h = v.use_big ? (vis_hash(pid) >> v.gshift) : (vis_hash(pid) >> (32 - 9));
    if (want) r.old = atomicCAS((v.use_big ? v.big : v.small) + r.h, kInvalid, pid);
    return r;
}
__device__ __forceinline__ bool vis_settle(VisitedSet& v, uint32_t pid, bool want, VisProbe r) {
    if (!want) return false;
    if (v.use_big && v.mode == kVisBitmap) return (r.old >> (pid & 31)) & 1u;
    if (v.use_big && v.mode == kVisB16) return r.old != 0u;
    uint32_t* tab = v.use_big ? v.big : v.small;
    const uint32_t mask = v.use_big ? v.gslots - 1 : (uint32_t)(kSmallVisSlots - 1);
    uint32_t old = r.old, h = r.h;
    for (;;) {
        if (old == kInvalid) return true;
        if (old == pid) return false;
        h = (h + 1) & mask;
        old = atomicCAS(tab + h, kInvalid, pid);
    }
}
__device__ __forceinline__ bool vis_insert(VisitedSet& v, uint32_t pid, bool want, int lane) {
    return vis_settle(v, pid, want, vis_probe(v, pid, want, lane));
}
// Make room for `incoming` more ids.  Returns false if the big table would get too full (the query is aborted with
// kQueryVisitedOverflow and re-run by the retry pass with a 2^18-slot hash set).
__device__ __forceinline__ bool vis_reserve(VisitedSet& v, uint32_t incoming, int lane) {
    if (!v.use_big && v.count + incoming > kSmallVisSlots / 2) vis_migrate_to_big(v, lane);
    if (v.use_big && v.mode == kVisHash && v.count + incoming > (v.gslots / 4) * 3) return false;
    if (v.use_big && v.mode == kVisB16 && v.count + incoming > v.cap_ids) return false;
    return true;
}

// ---------------------------------------------------------------------------------------------------------
// K1 phase clock (compile-time switch IDB_K1_PHASES, off in the product build; scripts/k1_phases.py builds a copy with it on).
// search_layer adds clock64() deltas per warp to one tally per phase of an expansion; a phase ends where its loads have been
// consumed, so a tally holds the phase's issue AND the wait for its own loads.  Each search_layer call of K1 adds its tallies to
// g_k1_phases (one copy per translation unit: search_cells.cu's CH 1 f32 object's is read by idb_debug_k1_phases).
// ---------------------------------------------------------------------------------------------------------
#ifdef IDB_K1_PHASES
enum K1Phase : int {
    kPhPop, kPhAdj, kPhVisit, kPhScreenLoad, kPhScreenMath, kPhGather, kPhMerge, kPhTies, kPhCount,
    // event counts behind the cycle tallies; dist_*: batch_distances_impl's batches, the row slots they load, the rows they hold
    kPhExpansions = kPhCount, kPhScreenBatches, kPhDistBatches, kPhDistSlots, kPhDistRows, kPhSlots
};
static __device__ unsigned long long g_k1_phases[kPhSlots];
#define IDB_PHASE(s, k) k1_phase_mark(s, k)
#define IDB_PHASE_COUNT(s, k, n) ((s).ph[k] += (n))
#else
#define IDB_PHASE(s, k) ((void)0)
#define IDB_PHASE_COUNT(s, k, n) ((void)0)
#endif

// ---------------------------------------------------------------------------------------------------------
// Per-warp traversal state.
// ---------------------------------------------------------------------------------------------------------
struct WarpState {
#ifdef IDB_K1_PHASES
    uint32_t ph[kPhSlots];       // this search_layer call's tallies (warp-uniform)
    long long ph_t;              // clock64() at the end of the last phase
    uint32_t ph_sink;            // keeps the loads a phase waits for from being optimised away
#endif
    uint64_t* near_base;     // shared: two buffers of near_len keys each (ping-pong for the merge)
    uint32_t near_len;       // 32*EF_T
    uint32_t* cpid;          // shared: 128 compacted new ids of the current row
    uint64_t* ckey;          // shared: their 128 keys (canonical distance bits << 32 | pid)
    uint64_t* ties;          // global: tie_cap keys
    uint32_t tie_cap;
    // EXPERIMENT (IDB_VARIANT 5..8): point rows staged in a per-warp shared-memory ring by cp.async.bulk
    char* ring;              // shared: B rows of nchunks * 16 bytes
    uint64_t* mbar;          // shared: the ring's mbarrier
    uint32_t mbar_phase;
    int cur;                 // live near buffer
    uint32_t cnt;            // len(nearest)
    uint32_t ntie;
    uint32_t status;
    uint32_t n_expand, n_dist;   // per-layer instrumentation (SURVEY §8d counters)
    uint32_t n_full;             // rows fetched in full over the whole descent (n_dist minus what the screen dropped)
    VisitedSet vis;
};

#ifdef IDB_K1_PHASES
__device__ __forceinline__ void k1_phase_mark(WarpState& s, int k) {
    const long long t = clock64();
    s.ph[k] += (uint32_t)(t - s.ph_t);
    s.ph_t = t;
}
// Wait for x (a value a phase loaded) before the phase is closed: a vote consumes it.
__device__ __forceinline__ void k1_phase_wait(WarpState& s, uint32_t x) { s.ph_sink ^= __ballot_sync(kFullMask, x == 0x9E3779B9u); }
__device__ __forceinline__ void k1_phase_begin(WarpState& s) {
#pragma unroll
    for (int k = 0; k < kPhSlots; ++k) s.ph[k] = 0;
    s.ph_sink = 0;
    s.ph_t = clock64();
}
__device__ __forceinline__ void k1_phase_flush(WarpState& s, int lane) {
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < kPhSlots; ++k) atomicAdd(&g_k1_phases[k], (unsigned long long)s.ph[k]);
        if (s.ph_sink == 0xFFFFFFFFu) atomicAdd(&g_k1_phases[kPhTies], 0ull);  // (never: a use of the sink)
    }
}
#endif

__device__ __forceinline__ uint32_t lower_bound_keys(const uint64_t* a, uint32_t n, uint64_t key) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        uint32_t mid = (lo + hi) >> 1;
        if ((a[mid] & kKeyMask) < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// The width ladder of batch_distances_impl.  Since the screen, an expansion fetches a handful of rows (DESIGN §5), so most batches
// are the last, part-filled one; a batch costs instructions for every slot, used or not.  So a batch is NB rows wide while NB rows
// are left, and the last one takes the narrowest of NB, NB/2, ..., FLOOR that holds every row left.  FLOOR (batch_floor) is the
// narrowest batch that still keeps four chunk loads and two rows in flight per lane.  A row's sum does not depend on the width
// (batch_butterfly), so neither does any key.
template <int CH>
__host__ __device__ constexpr int batch_floor() { return (4 + CH - 1) / CH > 2 ? (4 + CH - 1) / CH : 2; }
// The width of the next batch when rest >= 1 rows are left.
template <int NB, int FLOOR>
__host__ __device__ constexpr int batch_width(uint32_t rest) {
    int w = NB;
    while (w > FLOOR && rest <= (uint32_t)(w / 2)) w /= 2;
    return w;
}

// One batch of batch_distances_impl: rows b0 .. b0 + min(nb, NB) - 1 of cpid, NB rows in flight per lane.
template <int CH, int NB, bool kFull, class RT>
__device__ __forceinline__ void distance_batch(const GraphView& g, const float4 (&q)[CH], const uint32_t* cpid, uint64_t* ckey,
                                               uint32_t b0, uint32_t nb, const char* lane_base, uint32_t row_bytes,
                                               const bool (&cok)[CH], int lane) {
    typename RT::Raw v[NB][CH];
    typename RT::Hdr h[NB];
    if (kFull && nb >= (uint32_t)NB) {  // uniform; plain loads, no predicates, no zero fill
#pragma unroll
        for (int i = 0; i < NB; ++i) {
            const char* row = lane_base + (size_t)cpid[b0 + i] * row_bytes;  // shared-memory broadcast of the id
            h[i] = RT::hdr(g, cpid[b0 + i]);
#pragma unroll
            for (int j = 0; j < CH; ++j) v[i][j] = RT::ld_raw(row + j * 32 * RT::kChunkBytes);
        }
    } else {
#pragma unroll
        for (int i = 0; i < NB; ++i) {
            // branch-free on purpose: `if (i < nb) {load; use}` makes ptxas emit two branches per row
            const bool ok = (uint32_t)i < nb;
            const char* row = lane_base + (size_t)cpid[b0 + i] * row_bytes;  // shared-memory broadcast of the id
            h[i] = ok ? RT::hdr(g, cpid[b0 + i]) : typename RT::Hdr();
#pragma unroll
            for (int j = 0; j < CH; ++j)
                v[i][j] = (ok && cok[j]) ? RT::ld_raw(row + j * 32 * RT::kChunkBytes) : RT::zero();
        }
    }
    float p[NB];
#pragma unroll
    for (int i = 0; i < NB; ++i) p[i] = lane_partial_raw<CH, RT>(g, q, v[i], h[i], lane);
    const float total = batch_butterfly<NB>(p, lane);
    if ((uint32_t)lane < nb && lane < NB) ckey[b0 + lane] = mk_key(total, cpid[b0 + lane]);
}
// distance_batch at width w, one of NB, NB/2, ..., FLOOR (warp-uniform).
template <int CH, int NB, int FLOOR, bool kFull, class RT>
__device__ __forceinline__ void distance_batch_at(int w, const GraphView& g, const float4 (&q)[CH], const uint32_t* cpid,
                                                  uint64_t* ckey, uint32_t b0, uint32_t nb, const char* lane_base, uint32_t row_bytes,
                                                  const bool (&cok)[CH], int lane) {
    if constexpr (NB > FLOOR) {
        if (w < NB) {
            distance_batch_at<CH, NB / 2, FLOOR, kFull, RT>(w, g, q, cpid, ckey, b0, nb, lane_base, row_bytes, cok, lane);
            return;
        }
    }
    distance_batch<CH, NB, kFull, RT>(g, q, cpid, ckey, b0, nb, lane_base, row_bytes, cok, lane);
}

// Distances from q to the n_new points listed in cpid (shared, 16-byte aligned), up to NB rows in flight per lane; writes the
// keys (canonical distance bits << 32 | pid) to ckey.  The only place in the traversal that touches point rows.
// kFull: every lane owns a real chunk in every one of its CH slots (dim is a multiple of 128) -> no chunk predicates.
template <int CH, int NB, bool kFull, class RT>
__device__ __forceinline__ void batch_distances_impl(const GraphView& g, const float4 (&q)[CH], const uint32_t* cpid,
                                                     uint64_t* ckey, uint32_t n_new, int lane) {
    const uint32_t row_bytes = g.nchunks * RT::kChunkBytes;
    const char* lane_base = g.points + lane * RT::kChunkBytes;
    // keep the lane's base address in a register pair: each row address is then ONE IMAD.WIDE (pid * row_bytes + base)
    // instead of IMAD.WIDE + a 64-bit add of the kernel-parameter base
    asm volatile("" : "+l"(lane_base));
    if (g.flags & kOptPrefetchVectors) {  // pull every row of this expansion into L2 now; the batches below then hit L2
        const uint32_t lines = (row_bytes + 127) / 128;  // 128-byte lines per row
        for (uint32_t ln = 0; ln < lines; ++ln)
            for (uint32_t c = lane; c < n_new; c += 32)
                prefetch_l2(g.points + (size_t)cpid[c] * row_bytes + ln * 128u);
    }
    bool cok[CH];
#pragma unroll
    for (int j = 0; j < CH; ++j) cok[j] = kFull || (uint32_t)(lane + 32 * j) < g.nchunks;
    constexpr int FLOOR = batch_floor<CH>();
#pragma unroll 1
    for (uint32_t b0 = 0, w; b0 < n_new; b0 += w) {
        w = (uint32_t)batch_width<NB, FLOOR>(n_new - b0);  // uniform; rows i >= n_new - b0 of the batch are predicated off
        distance_batch_at<CH, NB, FLOOR, kFull, RT>((int)w, g, q, cpid, ckey, b0, n_new - b0, lane_base, row_bytes, cok, lane);
    }
    __syncwarp();
}
// Long rows (QVec<0>): NB rows in flight per lane and per group of 32 chunks; the accumulators are carried across the groups.
template <int NB, class RT>
__device__ __forceinline__ void batch_distances_long(const GraphView& g, const QVec<0>& q, const uint32_t* cpid, uint64_t* ckey,
                                                     uint32_t n_new, int lane) {
    const uint32_t row_bytes = g.nchunks * RT::kChunkBytes;
    const char* lane_base = g.points + lane * RT::kChunkBytes;
#pragma unroll 1
    for (uint32_t b0 = 0; b0 < n_new; b0 += NB) {
        const uint32_t nb = n_new - b0;
        const char* row[NB];
        typename RT::Hdr h[NB];
        float4 acc[NB];
#pragma unroll
        for (int i = 0; i < NB; ++i) {
            row[i] = lane_base + (size_t)cpid[b0 + ((uint32_t)i < nb ? i : 0)] * row_bytes;
            h[i] = RT::hdr(g, cpid[b0 + ((uint32_t)i < nb ? i : 0)]);
            acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll 1
        for (uint32_t j = 0; j < q.ngroups; ++j) {
            const bool ok = lane + 32u * j < g.nchunks;
            const float4 qq = q.s[lane + 32u * j];  // zero beyond the row
            typename RT::Raw v[NB];
#pragma unroll
            for (int i = 0; i < NB; ++i) v[i] = (ok && (uint32_t)i < nb) ? RT::ld_raw(row[i] + (size_t)j * 32 * RT::kChunkBytes) : RT::zero();
#pragma unroll
            for (int i = 0; i < NB; ++i) l2_step(acc[i], qq, widen_chunk<RT>(g, v[i], h[i], lane + 32u * j));
        }
        float p[NB];
#pragma unroll
        for (int i = 0; i < NB; ++i) p[i] = lane_sum(acc[i]);
        const float total = batch_butterfly<NB>(p, lane);
        if ((uint32_t)lane < nb && lane < NB) ckey[b0 + lane] = mk_key(total, cpid[b0 + lane]);
    }
    __syncwarp();
}
template <int CH, int NB, class RT = RowF32, bool FULL = false>
__device__ __forceinline__ void batch_distances(const GraphView& g, const QVec<CH>& q, const uint32_t* cpid, uint64_t* ckey,
                                                uint32_t n_new, int lane) {
    if constexpr (CH == 0) batch_distances_long<kLongRowsInFlight, RT>(g, q, cpid, ckey, n_new, lane);
    else batch_distances_impl<CH, NB, FULL, RT>(g, q.r, cpid, ckey, n_new, lane);
}

// ---------------------------------------------------------------------------------------------------------
// Screening (DESIGN §4 "screen"): a lower bound of a candidate's canonical distance from its 8-bit codes (128 B per row at dim 128
// instead of 512 B), so that rows the admission test would reject anyway are never fetched in full.  Every element shares one code
// step S (GraphView::cstep), so the bound is a triangle inequality in code space, in integer SIMD:
//   x~_i = offset_i + c_i S, q^_i = offset_i + qc_i S (real arithmetic), R >= ||x - x~|| for every stored row (GraphView::cerr),
//   r_q >= ||q - q^|| (ScreenQuery, once per layer), D = sum (qc_i - c_i)^2 (VABSDIFF4 + IDP.4A, exact in u32), so
//   ||q - x|| >= ||q^ - x~|| - r_q - R = S sqrt(D) - r_q - R,  bound = ((S sqrt(D))_rd - (r_q + R)_ru)_+^2 rounded down,
//   then * (1 - 2^-16)_rd and 0 below 2^-100.  bound > dist(furthest)  =>  canonical distance > dist(furthest).
// The factor covers the canonical order's roundings (at most CH + 9 per term, CH <= 8), the floor its underflow; a NaN or infinite
// query element makes r_q NaN / inf and the bound 0.
// ---------------------------------------------------------------------------------------------------------
constexpr float kScreenKeep = 0.9999847412109375f;  // 1 - 2^-16, exact
constexpr float kScreenFloor = 0x1p-100f;
__device__ __forceinline__ float screen_finish(float lb) {
    const float b = __fmul_rd(lb, kScreenKeep);
    return b > kScreenFloor ? b : 0.f;
}
// The query side of the bound: this lane's codes qc (word j = elements 4c..4c+3 of chunk c = lane + 32 j, packed as the table's
// words; 0 past nchunks) and slack = (r_q + R) rounded up.  Computed once per layer; the retry pass re-runs the layers, so it
// recomputes it.  screen_slice hands a lane the words the screen's layout (below) reads: kept one word per lane here, the codes
// hold CH registers across K1's layer instead of 4 CH, for 4 CH shuffles per screen call.
template <int CH>
struct ScreenQuery {
    uint32_t qc[CH];
    float slack;
};
template <int CH>
__device__ __forceinline__ void screen_query(ScreenQuery<CH>& sq, const GraphView& g, const float4 (&q)[CH], int lane) {
    const float S = g.cstep;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < CH; ++j) {
        const uint32_t c = lane + 32 * j;
        const float4 of = c < g.nchunks ? __ldg(g.cparams + g.nchunks + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float qv[4] = {q[j].x, q[j].y, q[j].z, q[j].w}, ov[4] = {of.x, of.y, of.z, of.w};
        uint32_t w = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            // any code in [0, 255] is valid (r_q measures the one chosen); a NaN element gets 0
            const float code = S > 0.f ? fminf(fmaxf(rintf(__fdiv_rn(__fsub_rn(qv[k], ov[k]), S)), 0.f), 255.f) : 0.f;
            // q^ lies in [fmaf_rd, fmaf_ru]: |q - q^| <= max(q - lo, hi - q), both rounded up (NaN / inf propagate)
            const float d = fmaxf(__fsub_ru(qv[k], __fmaf_rd(code, S, ov[k])), __fsub_ru(__fmaf_ru(code, S, ov[k]), qv[k]));
            acc = __fmaf_ru(d, d, acc);
            w |= (uint32_t)code << (8 * k);
        }
        sq.qc[j] = w;
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) acc = __fadd_ru(acc, __shfl_xor_sync(kFullMask, acc, o));
    sq.slack = __fadd_ru(__fsqrt_ru(acc), g.cerr);
}
// The bound from a row's squared code distance D (all lanes of the warp agree on slack).
__device__ __forceinline__ float screen_bound_of(const GraphView& g, uint32_t D, float slack) {
    const float t = fmaxf(__fsub_rd(__fmul_rd(g.cstep, __fsqrt_rd(__uint2float_rd(D))), slack), 0.f);  // NaN slack: 0
    return screen_finish(__fmul_rd(t, t));
}
// acc + sum over a code word's four elements of (qc - c)^2: one VABSDIFF4 and one IDP.4A.
__device__ __forceinline__ uint32_t screen_word(uint32_t qc, uint32_t w, uint32_t acc) {
    const uint32_t d = __vabsdiffu4(w, qc);
    return __dp4a(d, d, acc);
}
// ... over the sixteen elements of a 16-byte word: one IDP.4A chain.
__device__ __forceinline__ uint32_t screen_words(const uint4& qc, const uint4& w, uint32_t acc) {
    return screen_word(qc.w, w.w, screen_word(qc.z, w.z, screen_word(qc.y, w.y, screen_word(qc.x, w.x, acc))));
}
// The screen's layout (DESIGN §4): a code row is read by a group of eight lanes, lane l taking the 16-byte words 4 (l & 7) + 32 j
// (j < CH) with one LDG.128 each, so each load instruction of the warp covers four rows.  D is an exact u32, so its adds give the same
// D in any order and on any lane: this layout need not follow the canonical distance's.  A lane holds screen_slots<CH>() rows (slots)
// of a batch: <= 32 code words in flight.
template <int CH>
__device__ __forceinline__ constexpr int screen_slots() { return CH == 1 ? 8 : CH == 2 ? 4 : CH <= 4 ? 2 : 1; }
// The query's words of the lane's slice: qc[j] = words 4 (lane & 7) + 32 j .. +3.  Warp-uniform call.
template <int CH>
__device__ __forceinline__ void screen_slice(uint4 (&qc)[CH], const ScreenQuery<CH>& sq, int lane) {
    const int src = 4 * (lane & 7);
#pragma unroll
    for (int j = 0; j < CH; ++j)
        qc[j] = make_uint4(__shfl_sync(kFullMask, sq.qc[j], src), __shfl_sync(kFullMask, sq.qc[j], src + 1),
                           __shfl_sync(kFullMask, sq.qc[j], src + 2), __shfl_sync(kFullMask, sq.qc[j], src + 3));
}
// The lane's code words of one row: 16-byte word j of a row lies past cwords (it is the next row's) unless cok[j].
template <int CH, bool kFull>
struct ScreenLane {
    const char* base;    // g.codes + 16 (lane & 7) bytes
    uint32_t row_bytes;  // 4 cwords
    bool cok[CH];
    __device__ __forceinline__ ScreenLane(const GraphView& g, int lane) {
        // The base address and the row stride stay in registers (as in batch_distances_impl): each row address is then ONE IMAD.WIDE,
        // where re-reading g.codes / g.cwords for every predicated row cost about a dozen instructions per row.
        base = reinterpret_cast<const char*>(g.codes) + 16 * (lane & 7);
        asm volatile("" : "+l"(base));
        row_bytes = kFull ? 128u * CH : g.cwords * 4u;
        if (!kFull) asm volatile("" : "+r"(row_bytes));
#pragma unroll
        for (int j = 0; j < CH; ++j) cok[j] = kFull || (uint32_t)(4 * (lane & 7) + 32 * j) < g.cwords;
    }
    __device__ __forceinline__ void load(uint4 (&w)[CH], uint32_t pid, bool ok) const {
        const char* row = base + (size_t)pid * row_bytes;
#pragma unroll
        for (int j = 0; j < CH; ++j) w[j] = (ok && cok[j]) ? __ldg(reinterpret_cast<const uint4*>(row + 128 * j)) : make_uint4(0u, 0u, 0u, 0u);
    }
};
// Drops the candidates in cpid[0, n_new) whose bound exceeds fdist (the distance of the ef-th key of nearest) and compacts the rest,
// in row order, to the front of cpid.  Returns how many are left.  Warp-uniform call.
// A batch is NS = 4 NSL rows; group grp = lane >> 3 holds rows b0 + NSL grp + i in its slots i < NSL.  After the eight-lane
// reduction lane l holds row b0 + NSL (l >> 3) + (l & (NSL - 1)) (row b0 + l at NSL = 8), and only lanes with l & 7 < NSL vote, so
// the ballot keeps the survivors in row order.
template <int CH, bool kFull>
__device__ __forceinline__ uint32_t screen_candidates(WarpState& s, const GraphView& g, const ScreenQuery<CH>& sq, uint32_t n_new,
                                                      float fdist, int lane) {
    uint32_t* cpid = s.cpid;
    constexpr int NSL = screen_slots<CH>(), NS = 4 * NSL;
    const ScreenLane<CH, kFull> sl(g, lane);
    uint4 qc[CH];
    screen_slice<CH>(qc, sq, lane);
    const uint32_t first = NSL * (uint32_t)(lane >> 3), sub = lane & 7;  // this group's first slot row, this lane's place in it
    uint32_t kept = 0;
#pragma unroll 1
    for (uint32_t b0 = 0; b0 < n_new; b0 += NS) {
        IDB_PHASE_COUNT(s, kPhScreenBatches, 1u);
        // Every slot is loaded and reduced, also in the last, part-filled batch: a warp-uniform skip of the slots no group has a row
        // in split the batch into blocks, and the headline cell spilled.
        uint4 w[NSL][CH];
#pragma unroll
        for (int i = 0; i < NSL; ++i) sl.load(w[i], cpid[b0 + first + i], b0 + first + i < n_new);  // (past n_new: stale ids, not loaded)
#ifdef IDB_K1_PHASES
        {
            uint32_t x = 0;
#pragma unroll
            for (int i = 0; i < NSL; ++i)
#pragma unroll
                for (int j = 0; j < CH; ++j) x ^= w[i][j].x ^ w[i][j].y ^ w[i][j].z ^ w[i][j].w;
            k1_phase_wait(s, x);
            IDB_PHASE(s, kPhScreenLoad);
        }
#endif
        const uint32_t mine = sub < (uint32_t)NSL && b0 + first + sub < n_new ? cpid[b0 + first + sub] : kInvalid;
        uint32_t p[NSL];
#pragma unroll
        for (int i = 0; i < NSL; ++i) {
            p[i] = 0u;
#pragma unroll
            for (int j = 0; j < CH; ++j) p[i] = screen_words(qc[j], w[i][j], p[i]);
        }
        const float bound = screen_bound_of(g, batch_butterfly<NSL, false, uint32_t, 8>(p, lane), sq.slack);
        const bool keep = mine != kInvalid && !(bound > fdist);
        const uint32_t m = __ballot_sync(kFullMask, keep);
        __syncwarp();  // every lane has read this batch's ids before any is overwritten (writes go to [kept, b0 + NS))
        if (keep) cpid[kept + __popc(m & ((1u << lane) - 1u))] = mine;
        kept += __popc(m);
        IDB_PHASE(s, kPhScreenMath);
    }
    __syncwarp();
    return kept;
}

// EXPERIMENT — the TMA staging north_star describes: every point row of a batch is fetched by ONE cp.async.bulk (1-D bulk copy,
// global -> shared, completion counted on an mbarrier) into a per-warp ring; no register staging (the 16 x float4 landing registers
// of batch_distances_impl are gone: more warps fit), distances computed from shared memory.  f32 rows only.  Same arithmetic and
// summation order as batch_distances_impl, so results are bit-identical.  A traversal row is used once by one warp, so the extra trip
// through shared memory buys nothing over the register gather; kept as an experiment, selected with IDB_VARIANT 5..8.
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
struct WarpState;
template <int CH, int NB>
__device__ __forceinline__ void batch_distances_tma(const GraphView& g, const float4 (&q)[CH], const uint32_t* cpid, uint64_t* ckey,
                                                    uint32_t n_new, int lane, WarpState& s);
// Rare path: something was evicted while its distance equals the new furthest distance.  Such an entry stays a
// live candidate in the reference (strict `>` at lib.rs:601) iff it is unexpanded and had been ADMITTED
// (pushed on `candidates`, lib.rs:719).  Admission of row entry j: rank_S(j) + #{i<j in row order, i in A, key_i < key_j} < ef.
template <int ROW_T, int EF_T>
__device__ __forceinline__ void collect_ties(WarpState& s, const uint64_t* old_near, uint32_t old_cnt, const uint32_t (&shift)[EF_T],
                                          const uint64_t (&keyg)[ROW_T], const uint32_t (&rank)[ROW_T], const bool (&inA)[ROW_T],
                                          const uint32_t (&less)[ROW_T], uint32_t ef_cur, uint32_t fbits, int lane) {
    // (a) evicted members of S
#pragma unroll
    for (int t = 0; t < EF_T; ++t) {
        uint32_t idx = lane + 32 * t;
        bool tie = false;
        uint64_t k = 0;
        if (idx < old_cnt) {
            k = old_near[idx];
            tie = (idx + shift[t] >= ef_cur) && !(k & kFlagExpanded) && key_dbits(k) == fbits;
        }
        uint32_t m = __ballot_sync(kFullMask, tie);
        if (m) {
            uint32_t pos = s.ntie + __popc(m & ((1u << lane) - 1));
            if (tie && pos < s.tie_cap) s.ties[pos] = k;
            s.ntie += __popc(m);
        }
    }
    // (b) evicted members of A that were admitted in row order
#pragma unroll
    for (int g = 0; g < ROW_T; ++g) {
        bool cand = inA[g] && (rank[g] + less[g] >= ef_cur) && key_dbits(keyg[g]) == fbits;
        uint32_t earlier = 0;
        // count A entries earlier in row order (compacted index c' = 32*g2 + lane' < c = 32*g + lane) with smaller key
#pragma unroll
        for (int g2 = 0; g2 < ROW_T; ++g2) {
            uint32_t mA = __ballot_sync(kFullMask, inA[g2]);
            while (mA) {
                int src = __ffs(mA) - 1;
                mA &= mA - 1;
                uint64_t ak = shfl64(keyg[g2], src);
                if ((32 * g2 + src) < (32 * g + lane) && ak < keyg[g]) earlier++;
            }
        }
        bool tie = cand && (rank[g] + earlier < ef_cur);
        uint32_t m = __ballot_sync(kFullMask, tie);
        if (m) {
            uint32_t pos = s.ntie + __popc(m & ((1u << lane) - 1));
            if (tie && pos < s.tie_cap) s.ties[pos] = keyg[g];
            s.ntie += __popc(m);
        }
    }
    if (s.ntie > s.tie_cap) { s.status = kQueryTieOverflow; s.ntie = s.tie_cap; }
    __threadfence_block();
    __syncwarp();
}

// Pop the smallest key of the tie list (BinaryHeap::pop order among ties).
__device__ __forceinline__ uint64_t pop_min_tie(WarpState& s, int lane) {
    uint64_t best = kKeyNone;
    uint32_t bi = 0;
    for (uint32_t i = lane; i < s.ntie; i += 32) {
        uint64_t k = s.ties[i];
        if (k < best) { best = k; bi = i; }
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        uint64_t ok = shfl64(best, lane ^ off);
        uint32_t oi = __shfl_xor_sync(kFullMask, bi, off);
        if (ok < best) { best = ok; bi = oi; }
    }
    if (lane == 0) s.ties[bi] = s.ties[s.ntie - 1];
    s.ntie--;
    __threadfence_block();
    __syncwarp();
    return best;
}

template <int CH, int NB>
__device__ __forceinline__ void batch_distances_tma(const GraphView& g, const float4 (&q)[CH], const uint32_t* cpid, uint64_t* ckey,
                                                    uint32_t n_new, int lane, WarpState& s) {
    const uint32_t row_bytes = g.nchunks * 16u;
    const uint32_t bar = smem_addr(s.mbar);
#pragma unroll 1
    for (uint32_t b0 = 0; b0 < n_new; b0 += NB) {
        const uint32_t nb = min(n_new - b0, (uint32_t)NB);
        if (lane == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(nb * row_bytes) : "memory");
        if ((uint32_t)lane < nb) {  // one bulk copy per row, issued by the lane of the same index
            const char* src = g.points + (size_t)cpid[b0 + lane] * row_bytes;
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                             smem_addr(s.ring + (size_t)lane * row_bytes)),
                         "l"(src), "r"(row_bytes), "r"(bar)
                         : "memory");
        }
        uint32_t done = 0;
        while (!done)
            asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                         : "=r"(done)
                         : "r"(bar), "r"(s.mbar_phase)
                         : "memory");
        s.mbar_phase ^= 1u;
        float p[NB];
#pragma unroll
        for (int i = 0; i < NB; ++i) {
            float4 v[CH];
#pragma unroll
            for (int j = 0; j < CH; ++j) {
                const uint32_t c = lane + 32 * j;
                v[j] = ((uint32_t)i < nb && c < g.nchunks) ? *reinterpret_cast<const float4*>(s.ring + (size_t)i * row_bytes + c * 16u)
                                                           : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            p[i] = lane_partial<CH>(q, v);
        }
        const float total = batch_butterfly<NB>(p, lane);
        if ((uint32_t)lane < nb && lane < NB) ckey[b0 + lane] = mk_key(total, cpid[b0 + lane]);
        __syncwarp();  // every lane has read the ring before the next batch's copies overwrite it
    }
}

// ---------------------------------------------------------------------------------------------------------
// search_layer (lib.rs:598-614) over one layer.
//   rows/width : adjacency table of this layer (fixed stride `width` u32 per node)
//   links      : `.take(links)` (lib.rs:606)
//   ef_cur     : Search::ef for this layer
// Pre: near[0..cnt) sorted, unexpanded entries are the enter points (candidates), visited holds them.
// kLive: rows may be rewritten concurrently (GPU build) -> read them through L2 (ld.global.cg), not the
// read-only/L1 path.
// ---------------------------------------------------------------------------------------------------------
// SCREEN: compile the screening pass in (K1's register flavours); it runs when g.codes is set.
template <int CH, int ROW_T, int EF_T, int B, bool kLive, class RT, bool FULL, bool TMA = false, bool SCREEN = false>
__device__ __forceinline__ void search_layer(const GraphView& g, WarpState& s, const QVec<CH>& q, const uint32_t* rows,
                                             uint32_t width, uint32_t links, uint32_t ef_cur, bool seed_entry, int lane) {
    const uint32_t lt_mask = (1u << lane) - 1;
#ifdef IDB_K1_PHASES
    k1_phase_begin(s);
#endif
    constexpr bool kScreen = SCREEN && CH > 0 && !kLive && !TMA && RT::kType != kRowQ8 && RT::kType != kRowBin;  // (no table, DESIGN §3c, §3d)
    ScreenQuery<kScreen ? CH : 1> sq;
    if constexpr (kScreen) {
        if (g.codes) screen_query<CH>(sq, g, q.r, lane);
    }
    for (;;) {
        uint64_t* near = (s.near_base + s.cur * s.near_len);
        uint32_t n_new = 0;
        if (seed_entry) {
            // push(PointId(0)) (lib.rs:364 / 444): the entry point is the only "row entry" of a pseudo expansion
            seed_entry = false;
            vis_insert(s.vis, 0u, lane == 0, lane);
            s.vis.count = 1;
            if (lane == 0) s.cpid[0] = 0u;
            n_new = 1;
            s.n_dist += 1;
            __syncwarp();
        } else {
            // ---- pop the min candidate: first unexpanded entry of nearest, else the smallest tie ----------
            int sel = -1, nxt = -1;  // first / second unexpanded entry (the second is the likely NEXT candidate)
#pragma unroll
            for (int t = 0; t < EF_T; ++t) {
                if (nxt < 0) {
                    uint32_t idx = lane + 32 * t;
                    bool un = idx < s.cnt && !(near[idx] & kFlagExpanded);
                    uint32_t m = __ballot_sync(kFullMask, un);
                    if (m && sel < 0) { sel = 32 * t + __ffs(m) - 1; m &= m - 1; }
                    if (m && sel >= 0 && nxt < 0) nxt = 32 * t + __ffs(m) - 1;
                }
            }
            if ((g.flags & kOptPrefetchNextRow) && nxt >= 0) {
                // just-in-time L2 prefetch of the adjacency row we will most likely expand next (~one expansion ahead:
                // short enough to survive the L2 turnover caused by the streaming point rows)
                const uint32_t* r = rows + (size_t)key_pid(near[nxt]) * width;
                if (lane == 0) prefetch_l2(r);
                if (lane == 1 && links > 32) prefetch_l2(r + 32);
            }
            uint32_t cpid;
            if (sel >= 0) {
                uint64_t ck = near[sel];
                cpid = key_pid(ck);
                __syncwarp();
                if (lane == 0) near[sel] = ck | kFlagExpanded;
                __syncwarp();
            } else if (s.ntie > 0) {
                cpid = key_pid(pop_min_tie(s, lane));  // dist == furthest dist by invariant -> not `>` -> expanded
            } else {
                break;  // heap empty, or its min is strictly beyond the furthest result (lib.rs:601-603)
            }
            s.n_expand++;
            IDB_PHASE(s, kPhPop);
            IDB_PHASE_COUNT(s, kPhExpansions, 1u);

            // ---- row of the candidate: NearestIter stops at the first INVALID (types.rs:178-191) ----------
            uint32_t ent[ROW_T];
            const uint32_t* row = rows + (size_t)cpid * width;
#pragma unroll
            for (int t = 0; t < ROW_T; ++t) {
                uint32_t e = lane + 32 * t;
                ent[t] = kInvalid;
                if (e < links) ent[t] = kLive ? __ldcg(row + e) : __ldg(row + e);
            }
            uint32_t count = 32 * ROW_T;
#pragma unroll
            for (int t = ROW_T - 1; t >= 0; --t) {
                uint32_t m = __ballot_sync(kFullMask, ent[t] == kInvalid);
                if (m) count = 32 * t + __ffs(m) - 1;
            }
            IDB_PHASE(s, kPhAdj);
            if (count == 0) continue;

            // ---- visited.insert for every row entry (lib.rs:705), compacted in row order ------------------
            if (!vis_reserve(s.vis, count, lane)) { s.status = kQueryVisitedOverflow; break; }
            if (s.vis.use_big && s.vis.mode == kVisB16) {
                // all home buckets of the row in flight at once (one 32-byte sector each); the inserts are plain stores
                // arbitrated inside the warp, so the row costs ONE L2 round trip and nothing waits for the stores
                Bucket8 bk[ROW_T];
                B16 tg[ROW_T];
#pragma unroll
                for (int t = 0; t < ROW_T; ++t) {
                    tg[t] = b16_of(s.vis, ent[t]);
                    bk[t].lo = bk[t].hi = make_uint4(0u, 0u, 0u, 0u);
                    if ((uint32_t)(lane + 32 * t) < count) { bk[t] = bucket_load(s.vis, tg[t].home); b16_tally_reset(s.vis, tg[t]); }
                }
                __syncwarp();
                bool ovf = false;
#pragma unroll
                for (int t = 0; t < ROW_T; ++t) {
                    const bool fresh = b16_commit<true>(s.vis, tg[t], ent[t], bk[t], (uint32_t)(lane + 32 * t) < count, lane, &ovf);
                    const uint32_t m = __ballot_sync(kFullMask, fresh);
                    if (fresh) s.cpid[n_new + __popc(m & lt_mask)] = ent[t];
                    n_new += __popc(m);
                }
                if (__any_sync(kFullMask, ovf)) { s.status = kQueryVisitedOverflow; break; }
            } else {
                VisProbe probe[ROW_T];
#pragma unroll
                for (int t = 0; t < ROW_T; ++t) probe[t] = vis_probe(s.vis, ent[t], (uint32_t)(lane + 32 * t) < count, lane);
#pragma unroll
                for (int t = 0; t < ROW_T; ++t) {
                    const bool fresh = vis_settle(s.vis, ent[t], (uint32_t)(lane + 32 * t) < count, probe[t]);
                    const uint32_t m = __ballot_sync(kFullMask, fresh);
                    if (fresh) s.cpid[n_new + __popc(m & lt_mask)] = ent[t];
                    n_new += __popc(m);
                }
            }
            s.vis.count += n_new;
            s.n_dist += n_new;
            IDB_PHASE(s, kPhVisit);
            if (n_new == 0) continue;
            __syncwarp();
            // ---- screen (DESIGN §4): with nearest full, a candidate whose code bound exceeds the furthest distance has a key
            // above the furthest key, so it would not be admitted; only the others are fetched in full, still in row order --------
            if constexpr (kScreen) {
                if (g.codes && s.cnt >= ef_cur) {
                    n_new = screen_candidates<CH, FULL>(s, g, sq, n_new, __uint_as_float(key_dbits(near[s.cnt - 1])), lane);
                    if (n_new == 0) continue;
                }
            }
        }
        s.n_full += n_new;

        // ---- distances (lib.rs:709-710) --------------------------------------------------------------------
        if constexpr (TMA) batch_distances_tma<CH, B>(g, q.r, s.cpid, s.ckey, n_new, lane, s);
        else batch_distances<CH, B, RT, FULL>(g, q, s.cpid, s.ckey, n_new, lane);
#ifdef IDB_K1_PHASES
        if constexpr (CH > 0 && !TMA) {
            for (uint32_t b0 = 0, w; b0 < n_new; b0 += w) {
                w = (uint32_t)batch_width<B, batch_floor<CH>()>(n_new - b0);
                IDB_PHASE_COUNT(s, kPhDistBatches, 1u);
                IDB_PHASE_COUNT(s, kPhDistSlots, w);
            }
            IDB_PHASE_COUNT(s, kPhDistRows, n_new);
        }
#endif
        uint64_t keyg[ROW_T];
#pragma unroll
        for (int gi = 0; gi < ROW_T; ++gi) {
            const uint32_t c = 32 * gi + lane;
            keyg[gi] = c < n_new ? s.ckey[c] : kKeyNone;
        }
        IDB_PHASE(s, kPhGather);

        // ---- admission (lib.rs:712-719): A = entries with rank_S < ef ----------------------------------
        const bool full = s.cnt >= ef_cur;
        const uint64_t furthest = s.cnt ? (near[s.cnt - 1] & kKeyMask) : 0ull;
        uint32_t rank[ROW_T];
        bool inA[ROW_T];
        uint32_t nA = 0;
#pragma unroll
        for (int gi = 0; gi < ROW_T; ++gi) {
            rank[gi] = 0;
            inA[gi] = false;
            if (keyg[gi] != kKeyNone && !(full && keyg[gi] > furthest)) {
                rank[gi] = lower_bound_keys(near, s.cnt, keyg[gi]);
                inA[gi] = rank[gi] < ef_cur;
            }
            nA += __popc(__ballot_sync(kFullMask, inA[gi]));
        }
        IDB_PHASE(s, kPhMerge);
        if (nA == 0) continue;

        // ---- merge S and A into the other buffer: pos = rank among the union ---------------------------
        uint32_t less[ROW_T];
        uint32_t shift[EF_T];
#pragma unroll
        for (int gi = 0; gi < ROW_T; ++gi) less[gi] = 0;
#pragma unroll
        for (int t = 0; t < EF_T; ++t) shift[t] = 0;
#pragma unroll
        for (int gi = 0; gi < ROW_T; ++gi) {
            uint32_t mA = __ballot_sync(kFullMask, inA[gi]);
            while (mA) {
                int src = __ffs(mA) - 1;
                mA &= mA - 1;
                uint64_t ak = shfl64(keyg[gi], src);
                uint32_t ar = __shfl_sync(kFullMask, rank[gi], src);
#pragma unroll
                for (int g2 = 0; g2 < ROW_T; ++g2) less[g2] += (ak < keyg[g2]) ? 1u : 0u;
#pragma unroll
                for (int t = 0; t < EF_T; ++t) shift[t] += (ar <= (uint32_t)(lane + 32 * t)) ? 1u : 0u;
            }
        }
        uint64_t* other = (s.near_base + (s.cur ^ 1) * s.near_len);
#pragma unroll
        for (int t = 0; t < EF_T; ++t) {
            uint32_t idx = lane + 32 * t;
            if (idx < s.cnt) {
                uint32_t p = idx + shift[t];
                if (p < ef_cur) other[p] = near[idx];
            }
        }
#pragma unroll
        for (int gi = 0; gi < ROW_T; ++gi) {
            if (inA[gi]) {
                uint32_t p = rank[gi] + less[gi];
                if (p < ef_cur) {
                    other[p] = keyg[gi];
                    if (g.flags & kOptPrefetchRows) {  // it will most likely be expanded: start fetching its adjacency row
                        const uint32_t* r = rows + (size_t)key_pid(keyg[gi]) * width;
                        prefetch_l2(r);
                        if (links > 32) prefetch_l2(r + 32);
                    }
                }
            }
        }
        __syncwarp();
        const uint32_t old_cnt = s.cnt;
        const uint32_t total = old_cnt + nA;
        s.cnt = min(total, ef_cur);
        s.cur ^= 1;
        IDB_PHASE(s, kPhMerge);

        // ---- candidates that fell off the end (lib.rs:612 truncate) -------------------------------------
        if (total > ef_cur) {
            const uint32_t fbits = key_dbits(other[ef_cur - 1]);
            if (s.ntie > 0 && fbits != key_dbits(furthest)) s.ntie = 0;  // their distance is now strictly beyond
            bool maybe = false;
#pragma unroll
            for (int t = 0; t < EF_T; ++t) {
                uint32_t idx = lane + 32 * t;
                if (idx < old_cnt && idx + shift[t] >= ef_cur) {
                    uint64_t k = near[idx];
                    maybe |= !(k & kFlagExpanded) && key_dbits(k) == fbits;
                }
            }
#pragma unroll
            for (int gi = 0; gi < ROW_T; ++gi)
                maybe |= inA[gi] && (rank[gi] + less[gi] >= ef_cur) && key_dbits(keyg[gi]) == fbits;
            if (__any_sync(kFullMask, maybe))
                collect_ties<ROW_T, EF_T>(s, near, old_cnt, shift, keyg, rank, inA, less, ef_cur, fbits, lane);
            IDB_PHASE(s, kPhTies);
            if (s.status != kQueryOk) break;
        }
    }
#ifdef IDB_K1_PHASES
    k1_phase_flush(s, lane);
#endif
}

// Search::cull (lib.rs:729-737): candidates := nearest; visited := {pids of nearest}.
template <int EF_T>
__device__ __forceinline__ void cull(WarpState& s, int lane, bool next_big) {
    uint64_t* near = (s.near_base + s.cur * s.near_len);
    s.ntie = 0;
    vis_clear(s.vis, lane, next_big);
#pragma unroll
    for (int t = 0; t < EF_T; ++t) {
        uint32_t idx = lane + 32 * t;
        bool have = idx < s.cnt;
        uint64_t k = have ? near[idx] : 0ull;
        if (have) near[idx] = k & kKeyMask;                 // every result is a candidate again
        vis_insert(s.vis, key_pid(k), have, lane);
    }
    s.vis.count = s.cnt;
    __syncwarp();
}

// Hnsw::search (lib.rs:352-383) when target_layer == 0 and ef_target == ef_search;
// Construction::insert's descent (lib.rs:443-463) when target_layer = the insert layer, ef_target = ef_construction.
// Layers above the target are searched on the UpperNode snapshots with ef = 1; the target layer on the zero table.
// On return nearest = (s.near_base + s.cur * s.near_len)[0..s.cnt).  counters (if non-null): {n_expand_upper, n_dist_upper, n_expand_target, n_dist_target}.
template <int CH, int ROW_T, int EF_T, int B, bool kLive, class RT = RowF32, bool FULL = false, bool TMA = false, bool SCREEN = false>
__device__ __forceinline__ void descend(const GraphView& g, WarpState& s, const QVec<CH>& q, uint32_t target_layer,
                                        uint32_t ef_target, int lane, uint32_t* counters4) {
    s.cur = 0;
    s.cnt = 0;
    s.ntie = 0;
    s.status = kQueryOk;
    s.n_expand = 0;
    s.n_dist = 0;
    s.n_full = 0;
    s.vis.count = 0;
    s.vis.use_big = (g.n_upper == target_layer);  // no ef=1 layer above the target: go straight to the big tier
    uint32_t up_expand = 0, up_dist = 0;

    bool seed = true;  // push(PointId(0)) (lib.rs:364 / 444) happens inside the first search_layer call
    for (uint32_t cur = g.n_upper;; --cur) {
        const bool above = cur > target_layer;
        const uint32_t* rows = above ? g.upper[cur - 1] : g.zero;
        const uint32_t width = above ? g.M : 2 * g.M;
        const uint32_t links = (above || target_layer != 0) ? g.M : 2 * g.M;  // lib.rs:445 / 366-369
        search_layer<CH, ROW_T, EF_T, B, kLive, RT, FULL, TMA, SCREEN>(g, s, q, rows, width, links, above ? 1u : ef_target, seed, lane);
        seed = false;
        if (!above || s.status != kQueryOk) break;
        cull<EF_T>(s, lane, /*next_big=*/(cur - 1 == target_layer));
        up_expand += s.n_expand;
        up_dist += s.n_dist;
        s.n_expand = 0;
        s.n_dist = 0;
    }
    if (counters4 && lane == 0) {
        counters4[0] = up_expand;
        counters4[1] = up_dist;
        counters4[2] = s.n_expand;
        counters4[3] = s.n_dist;
    }
}

// ---------------------------------------------------------------------------------------------------------
// Per-warp scratch tables (big visited tier, tie list) are a DEVICE-wide pool sized for the warps that can be resident at once
// (SMs x CTA slots per SM x warps per CTA), shared by every index, stream and kernel of this library on the device: a CTA claims
// a slot of the SM it runs on when it starts and returns it (tables clean) when it exits.  Any number of search / build kernels
// may therefore be in flight together — the next batch's CTAs move in as the previous batch's drain — without each needing its
// own ~75 MB of tables (which would no longer fit the persisting part of L2).
// ---------------------------------------------------------------------------------------------------------
struct TablePool {
    uint32_t* slot_masks;     // [word]: bit i set = slot i taken
    int32_t fixed_word;       // >= 0: claim from this word (the retry pool); < 0: from word %smid  (%smid < %nsmid, which may exceed
                              // the number of ENABLED SMs: the pool is sized by %nsmid)
    uint32_t word_base;       // subtracted from the word when the table index is formed (retry pool: its word; else 0)
    uint32_t slots_per_word;  // <= 32
    uint32_t* vis_tables;     // (word * slots_per_word + slot) * kWarpsPerCta + warp  ->  vis_stride words
    uint32_t vis_stride;
    uint32_t* vis_ext;        // b16 flavour: second segment of each table (ext_stride words), for tables beyond the first segment
    uint32_t ext_stride;
    uint64_t* tie_tables;     // same index -> tie_cap keys
    uint32_t tie_cap;
};
__device__ __forceinline__ uint32_t current_smid() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(r));
    return r;
}
// Block-uniform: returns the table index of warp 0 of this CTA (consecutive warps follow).  s_claim: 2 words of shared memory.
__device__ __forceinline__ uint32_t cta_tables_acquire(const TablePool& tp, uint32_t* s_claim, uint32_t warps_per_cta) {
    if (threadIdx.x == 0) {
        const uint32_t word = tp.fixed_word >= 0 ? (uint32_t)tp.fixed_word : current_smid();
        const uint32_t all = tp.slots_per_word >= 32u ? 0xFFFFFFFFu : ((1u << tp.slots_per_word) - 1u);
        uint32_t bit;
        for (;;) {
            const uint32_t freeb = ~atomicOr(tp.slot_masks + word, 0u) & all;
            if (!freeb) { __nanosleep(256); continue; }  // more co-resident CTAs than slots (a tuning variant): wait for one
            bit = __ffs(freeb) - 1;
            if (!(atomicOr(tp.slot_masks + word, 1u << bit) & (1u << bit))) break;
        }
        __threadfence();  // the previous holder's clean-up stores are visible before we touch the tables
        s_claim[0] = word;
        s_claim[1] = bit;
    }
    __syncthreads();
    return ((s_claim[0] - tp.word_base) * tp.slots_per_word + s_claim[1]) * warps_per_cta;
}
__device__ __forceinline__ void cta_tables_release(const TablePool& tp, const uint32_t* s_claim) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAnd(tp.slot_masks + s_claim[0], ~(1u << s_claim[1]));
    }
}

// Leave both visited tiers empty for the next query handled by this warp.
__device__ __forceinline__ void finish_query(WarpState& s, int lane) {
    vis_clear(s.vis, lane, false);
}

}  // namespace idb
