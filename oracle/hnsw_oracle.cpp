// hnsw_oracle.cpp — CPU ORACLE for the instant-distance HNSW hot path.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT. ***  Only tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference legs may load this library.  The product (libinstant_distance_b200.so)
// never links, loads or calls it; there is no CPU fallback in the product path.
//
// What it is: a restatement, function by function, of the reference's algorithm (the reference is Rust
// and cannot be compiled in this environment — no rustc/cargo, no network).  Citations are file:line
// under /root/reference/ with  core = instant-distance/src/lib.rs,  types = instant-distance/src/types.rs,
// py = instant-distance-py/src/lib.rs.
//
// Parity pins: the reference ships NO fixed-seed expected-id vectors.  Its own tests pin this path with
//   * tests/all.rs:9-39   `map`   exact distances/values for 5 collinear points   (seed independent)
//   * tests/all.rs:41-53  recall > 97/100 (heuristic) and > 90/100 (simple) on 1024 uniform 2-D points
//   * instant-distance-py/test/test.py:15-35   self-query returns own value first (1024 x 300)
// and the oracle is checked against all of them (tests/test_oracle_reference_pins.py).
// Third-party arithmetic that is NOT under /root/reference and is therefore **parity unpinned**:
//   * rand "0.10" SmallRng::seed_from_u64 + random_range (core:214,257-260): restated here from the
//     published algorithms (xoshiro256++ seeded by SplitMix64; widening-multiply range sampling with one
//     bias-reduction step, as in rand 0.9's UniformInt::sample_single_inclusive).  No reference test
//     pins the stream (seeds come from ThreadRng, tests/all.rs:17,56).  The generator core and its seeding ARE
//     pinned to the published known-answer vectors of xoshiro256++ (reference C implementation, state {1,2,3,4})
//     and of Xoshiro256PlusPlus::seed_from_u64(0) (orc_rng_kat); the range reduction remains unpinned.
//   * ordered-float "5.0" total order (types:231): NaN greatest and equal to itself, -0 == +0.
//   * rayon scheduling (core:316-318): threaded build order is nondeterministic by design.
//
// Distance: the reference's only f32-vector Point is FloatArray (py:378-421): SQUARED L2, fp32, FMA,
// fixed summation order (8 AVX lanes, dim fixed at 300).  We define ONE canonical fp32 summation order
// for any dim, shared bit-for-bit by this oracle and the CUDA kernels (see l2sq_canonical_scalar below);
// the gap to the reference's own AVX2 order is covered by north_star's 1e-4 relative tolerance.

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <thread>
#include <vector>

#if defined(__x86_64__)
#include <immintrin.h>
#endif

#define ORC_API extern "C" __attribute__((visibility("default")))

namespace {

constexpr uint32_t INVALID = 0xFFFFFFFFu;  // types:293

// ---------------------------------------------------------------------------------------------
// Canonical squared-L2 (shared with the GPU kernels, see DESIGN.md "canonical distance").
//   128 accumulators acc[i mod 128], each an fmaf chain over i = r, r+128, r+256, ... (ascending);
//   lane sums s[l] = (acc[4l]+acc[4l+1]) + (acc[4l+2]+acc[4l+3]), l = 0..31;
//   xor butterfly over l with offsets 1, 2, 4, 8, 16:  s[l] <- s[l] + s[l^off];  result s[0].
// ---------------------------------------------------------------------------------------------
float l2sq_canonical_scalar(const float* q, const float* x, uint32_t dim) {
    float acc[128];
    for (int i = 0; i < 128; ++i) acc[i] = 0.0f;
    for (uint32_t i = 0; i < dim; ++i) {
        float d = q[i] - x[i];
        acc[i & 127] = std::fmaf(d, d, acc[i & 127]);
    }
    float s[32], t[32];
    for (int l = 0; l < 32; ++l) s[l] = (acc[4 * l] + acc[4 * l + 1]) + (acc[4 * l + 2] + acc[4 * l + 3]);
    for (int off = 1; off <= 16; off <<= 1) {
        for (int l = 0; l < 32; ++l) t[l] = s[l] + s[l ^ off];
        for (int l = 0; l < 32; ++l) s[l] = t[l];
    }
    return s[0];
}

#if defined(__x86_64__)
__attribute__((target("avx512f,avx512dq,fma"))) float l2sq_canonical_avx512(const float* q, const float* x,
                                                                           uint32_t dim) {
    __m512 a0 = _mm512_setzero_ps(), a1 = a0, a2 = a0, a3 = a0, a4 = a0, a5 = a0, a6 = a0, a7 = a0;
    uint32_t i = 0;
#define ORC_STEP(A, OFF)                                                                  \
    {                                                                                     \
        __m512 d = _mm512_sub_ps(_mm512_loadu_ps(q + i + OFF), _mm512_loadu_ps(x + i + OFF)); \
        A = _mm512_fmadd_ps(d, d, A);                                                     \
    }
    for (; i + 128 <= dim; i += 128) {
        ORC_STEP(a0, 0) ORC_STEP(a1, 16) ORC_STEP(a2, 32) ORC_STEP(a3, 48)
        ORC_STEP(a4, 64) ORC_STEP(a5, 80) ORC_STEP(a6, 96) ORC_STEP(a7, 112)
    }
#undef ORC_STEP
    if (i < dim) {  // tail: masked lanes load 0 for both operands -> d = 0 -> fma(0,0,acc) == acc exactly
        uint32_t rem = dim - i;
        __m512* accs[8] = {&a0, &a1, &a2, &a3, &a4, &a5, &a6, &a7};
        for (int k = 0; k < 8 && rem > 0; ++k) {
            uint32_t take = rem >= 16 ? 16 : rem;
            __mmask16 m = (__mmask16)((1u << take) - 1u);
            __m512 d = _mm512_sub_ps(_mm512_maskz_loadu_ps(m, q + i + 16 * k), _mm512_maskz_loadu_ps(m, x + i + 16 * k));
            *accs[k] = _mm512_fmadd_ps(d, d, *accs[k]);
            rem -= take;
        }
    }
    // lane sums: within every group of 4 floats (a0+a1)+(a2+a3), replicated over the group
#define ORC_QUAD(V)                                                    \
    {                                                                  \
        __m512 t_ = _mm512_add_ps(V, _mm512_permute_ps(V, 0xB1)); /* [1,0,3,2] */ \
        V = _mm512_add_ps(t_, _mm512_permute_ps(t_, 0x4E));       /* [2,3,0,1] */ \
    }
    ORC_QUAD(a0) ORC_QUAD(a1) ORC_QUAD(a2) ORC_QUAD(a3) ORC_QUAD(a4) ORC_QUAD(a5) ORC_QUAD(a6) ORC_QUAD(a7)
#undef ORC_QUAD
    // zmm k holds lanes l = 4k+m, m = 128-bit lane index (each value x4).
    // butterfly off=1 <-> m^1, off=2 <-> m^2 (in-register lane swaps), off=4 <-> k^1, off=8 <-> k^2, off=16 <-> k^4
#define ORC_BF(V)                                                 \
    V = _mm512_add_ps(V, _mm512_shuffle_f32x4(V, V, 0xB1));       \
    V = _mm512_add_ps(V, _mm512_shuffle_f32x4(V, V, 0x4E));
    ORC_BF(a0) ORC_BF(a1) ORC_BF(a2) ORC_BF(a3) ORC_BF(a4) ORC_BF(a5) ORC_BF(a6) ORC_BF(a7)
#undef ORC_BF
    a0 = _mm512_add_ps(a0, a1); a2 = _mm512_add_ps(a2, a3); a4 = _mm512_add_ps(a4, a5); a6 = _mm512_add_ps(a6, a7);
    a0 = _mm512_add_ps(a0, a2); a4 = _mm512_add_ps(a4, a6);
    a0 = _mm512_add_ps(a0, a4);
    return _mm512_cvtss_f32(a0);
}
#endif

using dist_fn = float (*)(const float*, const float*, uint32_t);

dist_fn pick_l2sq() {
#if defined(__x86_64__)
    __builtin_cpu_init();
    if (__builtin_cpu_supports("avx512f") && __builtin_cpu_supports("avx512dq")) return l2sq_canonical_avx512;
#endif
    return l2sq_canonical_scalar;
}
dist_fn g_l2sq = pick_l2sq();

// Test-only metric restating tests/all.rs:93-97 (2-D Euclidean WITH sqrt), any dim, sequential sum.
float l2_sqrt_sequential(const float* a, const float* b, uint32_t dim) {
    float s = 0.0f;
    for (uint32_t i = 0; i < dim; ++i) {
        float d = a[i] - b[i];
        s = s + d * d;  // compiled with -ffp-contract=off: (a-b).powi(2) then add, like the test's Point
    }
    return std::sqrt(s);
}

// The reference's OWN summation order for its only f32-vector Point, FloatArray::distance (py:378-421): 8 AVX2 lanes, one FMA chain
// per lane over chunks_exact(8); upper half + lower half; the last 4 elements FMA'd into the 4 sums; then (s0+s2)+(s1+s3).
// The reference fixes DIMENSIONS = 300 (py:16) and asserts len % 8 == 4 (py:388); restated here for any dim with dim % 8 == 4.
// Used only to MEASURE how often results differ from the product's canonical order (tests/, scripts/summation_order_gap.py).
#define ORC_REF_ORDER_BODY                                                                                   \
    float acc8[8] = {0, 0, 0, 0, 0, 0, 0, 0};                                                                \
    const uint32_t body = dim / 8 * 8; /* chunks_exact(8) */                                                 \
    for (uint32_t i = 0; i < body; i += 8)                                                                   \
        for (int l = 0; l < 8; ++l) {                                                                        \
            const float d = a[i + l] - b[i + l];                                                             \
            acc8[l] = __builtin_fmaf(d, d, acc8[l]); /* _mm256_fmadd_ps (py:397) */                          \
        }                                                                                                    \
    float acc4[4];                                                                                           \
    for (int l = 0; l < 4; ++l) acc4[l] = acc8[4 + l] + acc8[l]; /* py:400-402 */                            \
    for (int l = 0; l < 4; ++l) {                                /* py:404-407: the LAST four elements */    \
        const float d = a[dim - 4 + l] - b[dim - 4 + l];                                                     \
        acc4[l] = __builtin_fmaf(d, d, acc4[l]);                                                             \
    }                                                                                                        \
    const float s0 = acc4[0] + acc4[2], s1 = acc4[1] + acc4[3]; /* movehl + add (py:409-410) */              \
    return s0 + s1;                                             /* shuffle + add_ss (py:411-413) */
float l2sq_reference_order_generic(const float* a, const float* b, uint32_t dim) { ORC_REF_ORDER_BODY }
#if defined(__x86_64__)
__attribute__((target("avx2,fma"))) float l2sq_reference_order_fma(const float* a, const float* b, uint32_t dim) { ORC_REF_ORDER_BODY }
#endif
#undef ORC_REF_ORDER_BODY
float l2sq_reference_avx2_order(const float* a, const float* b, uint32_t dim) {
#if defined(__x86_64__)
    static const bool have_fma = (__builtin_cpu_init(), __builtin_cpu_supports("fma") && __builtin_cpu_supports("avx2"));
    if (have_fma) return l2sq_reference_order_fma(a, b, dim);  // same IEEE results, hardware fma instead of libm's
#endif
    return l2sq_reference_order_generic(a, b, dim);
}

enum Metric : int { METRIC_L2SQ_CANONICAL = 0, METRIC_L2_SQRT_SEQ = 1, METRIC_L2SQ_REFERENCE_AVX2 = 2 };
dist_fn metric_fn(int metric) {
    if (metric == METRIC_L2_SQRT_SEQ) return l2_sqrt_sequential;
    if (metric == METRIC_L2SQ_REFERENCE_AVX2) return l2sq_reference_avx2_order;
    return g_l2sq;
}

// ---------------------------------------------------------------------------------------------
// Candidate ordering (types:228-234): derived lexicographic Ord on (OrderedFloat<f32>, PointId).
// Encoded as one u64 key: canonical distance bits (NaN -> 0x7fc00000 = greatest, -0 -> +0) << 32 | pid.
// Distances are non-negative, so unsigned compare of the bit pattern equals the float total order.
// ---------------------------------------------------------------------------------------------
inline uint32_t canon_bits(float d) {
    uint32_t b;
    std::memcpy(&b, &d, 4);
    if ((b & 0x7fffffffu) > 0x7f800000u) return 0x7fc00000u;
    if (b == 0x80000000u) return 0u;
    return b;
}
inline uint64_t mk_key(float d, uint32_t pid) { return ((uint64_t)canon_bits(d) << 32) | pid; }
inline uint32_t key_pid(uint64_t k) { return (uint32_t)k; }
inline uint32_t key_dbits(uint64_t k) { return (uint32_t)(k >> 32); }
inline float key_dist(uint64_t k) {
    uint32_t b = key_dbits(k);
    float f;
    std::memcpy(&f, &b, 4);
    return f;
}

// Visited (types:13-59): generation-stamped byte set.
struct Visited {
    std::vector<uint8_t> store;
    uint8_t generation = 1;
    void with_capacity(size_t cap) { store.assign(cap, 0); generation = 1; }
    void reserve_capacity(size_t cap) {  // types:26-30
        if (store.size() != cap) store.resize(cap, (uint8_t)(generation - 1));
    }
    bool insert(uint32_t pid) {  // types:32-40
        uint8_t& slot = store[pid];
        if (slot != generation) { slot = generation; return true; }
        return false;
    }
    void clear() {  // types:48-58
        if (generation < 249) { generation++; return; }
        std::fill(store.begin(), store.end(), 0);
        generation = 1;
    }
};

struct Counters {
    uint64_t n_expand_upper = 0, n_dist_upper = 0, n_expand_zero = 0, n_dist_zero = 0;
};

// Search (core:560-574)
struct Search {
    Visited visited;
    std::vector<uint64_t> candidates;  // min-heap (BinaryHeap<Reverse<Candidate>>)
    std::vector<uint64_t> nearest, working, discarded;
    size_t ef = 1;  // core:775
    // instrumentation (not in the reference): distance evaluations / expansions of the current call
    uint64_t n_dist = 0, n_expand = 0;

    void heap_push(uint64_t k) {
        candidates.push_back(k);
        std::push_heap(candidates.begin(), candidates.end(), std::greater<uint64_t>());
    }
    uint64_t heap_pop() {
        std::pop_heap(candidates.begin(), candidates.end(), std::greater<uint64_t>());
        uint64_t k = candidates.back();
        candidates.pop_back();
        return k;
    }
    void reset() {  // core:740-755 (ef untouched)
        visited.clear();
        candidates.clear();
        nearest.clear();
        working.clear();
        discarded.clear();
    }
    void cull() {  // core:729-737
        candidates.clear();
        for (uint64_t k : nearest) heap_push(k);
        visited.clear();
        for (uint64_t k : nearest) visited.insert(key_pid(k));
    }
};

struct RwSpin {  // stands in for parking_lot::RwLock around each ZeroNode (core:288)
    std::atomic<int32_t> s{0};
    void lock_shared() {
        for (;;) {
            int32_t v = s.load(std::memory_order_relaxed);
            if (v >= 0 && s.compare_exchange_weak(v, v + 1, std::memory_order_acquire)) return;
            if (v < 0) std::this_thread::yield();
        }
    }
    void unlock_shared() { s.fetch_sub(1, std::memory_order_release); }
    void lock() {
        for (;;) {
            int32_t v = 0;
            if (s.compare_exchange_weak(v, -1, std::memory_order_acquire)) return;
            std::this_thread::yield();
        }
    }
    void unlock() { s.store(0, std::memory_order_release); }
};

struct Points {
    const float* base = nullptr;
    size_t stride = 0;  // floats per row (dim rounded up to a multiple of 4, zero padded)
    uint32_t dim = 0;
    dist_fn fn = nullptr;
    const float* row(uint32_t pid) const { return base + (size_t)pid * stride; }
    float distance(const float* a, const float* b) const { return fn(a, b, dim); }
};

}  // namespace

struct orc_index {
    uint32_t M = 32;
    uint32_t dim = 0;
    size_t stride = 0;
    size_t n = 0;
    size_t ef_search = 100;
    int metric = METRIC_L2SQ_CANONICAL;
    float* points = nullptr;                      // n x stride, 64-byte aligned, PointId order
    std::vector<uint32_t> zero;                   // n x 2M      (ZeroNode, types:83-85)
    std::vector<std::vector<uint32_t>> layers;    // layers[l-1]: n_l x M (UpperNode, types:63)
    std::vector<uint64_t> layer_n;                // layer_n[l] = node count of layer l (layer_n[0] = n)
    Points pts() const {
        Points p;
        p.base = points; p.stride = stride; p.dim = dim;
        p.fn = metric_fn(metric);
        return p;
    }
    ~orc_index() { std::free(points); }
};

namespace {

// push (core:704-720).  NOTE: no truncation here; `nearest` may exceed ef until search() truncates.
inline void push(Search& s, uint32_t pid, const float* point, const Points& pts) {
    if (!s.visited.insert(pid)) return;
    float d = pts.distance(point, pts.row(pid));
    s.n_dist++;
    uint64_t key = mk_key(d, pid);
    size_t idx = std::lower_bound(s.nearest.begin(), s.nearest.end(), key) - s.nearest.begin();
    if (idx >= s.ef) return;  // Err(_) => return   (keys are unique, Ok(_) is unreachable: core:715)
    s.nearest.insert(s.nearest.begin() + idx, key);
    s.heap_push(key);
}

// search_layer (core:598-614).  row_fn(pid, links, buf) copies the row's valid prefix (NearestIter,
// types:172-192, + .take(links), core:606) into buf and returns its length.
template <class RowFn>
inline void search_layer(Search& s, const float* point, RowFn&& row_fn, const Points& pts, uint32_t links) {
    uint32_t buf[256];
    while (!s.candidates.empty()) {
        uint64_t cand = s.heap_pop();
        if (!s.nearest.empty() && key_dbits(cand) > key_dbits(s.nearest.back())) break;  // strict, distance only
        uint32_t cnt = row_fn(key_pid(cand), links, buf);
        s.n_expand++;
        for (uint32_t i = 0; i < cnt; ++i) push(s, buf[i], point, pts);
        if (s.nearest.size() > s.ef) s.nearest.resize(s.ef);  // core:612
    }
}

inline uint32_t copy_row(const uint32_t* row, uint32_t width, uint32_t links, uint32_t* buf) {
    uint32_t lim = std::min(width, links), c = 0;
    while (c < lim && row[c] != INVALID) { buf[c] = row[c]; ++c; }
    return c;
}

struct Heuristic { bool on = true, extend_candidates = false, keep_pruned = true; };

// select_heuristic (core:636-698).  full_row_fn has no `.take()` (core:649).
template <class RowFn>
inline void select_heuristic(Search& s, const float* point, RowFn&& full_row_fn, const Points& pts, uint32_t M,
                             const Heuristic& h) {
    s.working.clear();
    uint32_t buf[256];
    for (size_t i = 0; i < s.nearest.size(); ++i) {
        uint64_t cand = s.nearest[i];
        s.working.push_back(cand);
        if (h.extend_candidates) {
            uint32_t cnt = full_row_fn(key_pid(cand), 2 * M, buf);
            for (uint32_t j = 0; j < cnt; ++j) {
                if (!s.visited.insert(buf[j])) continue;
                float d = pts.distance(point, pts.row(buf[j]));
                s.n_dist++;
                s.working.push_back(mk_key(d, buf[j]));
            }
        }
    }
    if (h.extend_candidates) std::sort(s.working.begin(), s.working.end());
    s.nearest.clear();
    s.discarded.clear();
    for (uint64_t cand : s.working) {
        if (s.nearest.size() >= 2 * (size_t)M) break;  // always 2M (core:669)
        const float* cp = pts.row(key_pid(cand));
        bool keep = true;
        for (uint64_t r : s.nearest) {
            float d = pts.distance(cp, pts.row(key_pid(r)));
            s.n_dist++;
            if (canon_bits(d) < key_dbits(cand)) { keep = false; break; }  // strict < (core:678)
        }
        if (keep) s.nearest.push_back(cand); else s.discarded.push_back(cand);
    }
    s.working.clear();
    if (h.keep_pruned) {
        for (uint64_t cand : s.discarded) {
            if (s.nearest.size() >= 2 * (size_t)M) break;
            s.nearest.push_back(cand);
        }
    }
    s.discarded.clear();
}

// rust core::slice::binary_search_by (rustc >= 1.82 form; the reference's MSRV is 1.85, rust.yml:85).
// cmp(elem) returns -1 (Less), 0 (Equal), +1 (Greater).  Needed only for simple mode (core:500-512),
// whose closure violates the ordering contract, so the index depends on this exact probe sequence.
template <class Cmp>
inline size_t rust_binary_search_by(size_t len, Cmp&& cmp) {
    size_t size = len;
    if (size == 0) return 0;
    size_t base = 0;
    while (size > 1) {
        size_t half = size / 2, mid = base + half;
        int c = cmp(mid);
        base = (c > 0) ? base : mid;
        size -= half;
    }
    int c = cmp(base);
    if (c == 0) return base;  // Ok(base) -> unwrap_or_else(|e| e) gives the same index
    return base + (c < 0 ? 1 : 0);
}

struct Construction {
    orc_index* ix;
    std::vector<RwSpin> locks;
    uint32_t top;
    Heuristic heuristic;
    size_t ef_construction;
    Points pts;
    // SearchPool (core:531-554)
    RwSpin pool_lock;
    std::vector<std::pair<Search*, Search*>> pool;

    std::pair<Search*, Search*> pool_pop() {
        pool_lock.lock();
        if (!pool.empty()) {
            auto r = pool.back();
            pool.pop_back();
            pool_lock.unlock();
            return r;
        }
        pool_lock.unlock();
        auto* a = new Search();
        auto* b = new Search();
        a->visited.with_capacity(ix->n);
        b->visited.with_capacity(ix->n);
        return {a, b};
    }
    void pool_push(std::pair<Search*, Search*> p) {
        pool_lock.lock();
        pool.push_back(p);
        pool_lock.unlock();
    }

    uint32_t* zrow(uint32_t pid) { return ix->zero.data() + (size_t)pid * 2 * ix->M; }

    // Layer for &[RwLock<ZeroNode>] (types:142-151): read-lock the row while it is iterated.  We copy the
    // valid prefix under the lock and release — the same atomic snapshot the guard gives the reference.
    uint32_t live_row(uint32_t pid, uint32_t links, uint32_t* buf) {
        locks[pid].lock_shared();
        uint32_t c = copy_row(zrow(pid), 2 * ix->M, links, buf);
        locks[pid].unlock_shared();
        return c;
    }

    // insert (core:437-528)
    void insert(uint32_t neu, uint32_t layer) {
        const uint32_t M = ix->M;
        locks[neu].lock();  // core:438: write lock on the new node's row for the whole insert
        auto pr = pool_pop();
        Search& search = *pr.first;
        Search& insertion = *pr.second;
        insertion.ef = ef_construction;  // core:440

        const float* point = pts.row(neu);
        search.reset();
        push(search, 0, point, pts);  // core:444 (stale ef >= 1; nearest is empty)
        const uint32_t num = layer == 0 ? 2 * M : M;  // core:445

        for (uint32_t cur = top;; --cur) {  // core:447-463
            search.ef = cur <= layer ? ef_construction : 1;
            if (cur > layer) {
                const std::vector<uint32_t>& snap = ix->layers[cur - 1];
                search_layer(search, point,
                             [&](uint32_t pid, uint32_t links, uint32_t* buf) {
                                 return copy_row(snap.data() + (size_t)pid * M, M, links, buf);
                             },
                             pts, num);
                search.cull();
            } else {
                search_layer(search, point,
                             [&](uint32_t pid, uint32_t links, uint32_t* buf) { return live_row(pid, links, buf); },
                             pts, num);
                break;
            }
            if (cur == 0) break;
        }

        if (heuristic.on) {  // core:470-472
            select_heuristic(search, point,
                             [&](uint32_t pid, uint32_t links, uint32_t* buf) { return live_row(pid, links, buf); }, pts,
                             M, heuristic);
        } else {  // core:466-469
            if (search.nearest.size() > 2 * (size_t)M) search.nearest.resize(2 * (size_t)M);
        }
        const std::vector<uint64_t>& found = search.nearest;

        uint32_t* node = zrow(neu);
        uint32_t buf[256];
        for (size_t i = 0; i < found.size(); ++i) {  // core:481-517
            uint32_t pid = key_pid(found[i]);
            if (heuristic.on) {
                // add_neighbor_heuristic (core:616-631): candidates = {new} U row(pid), w.r.t. points[pid]
                const float* ppoint = pts.row(pid);
                insertion.reset();
                push(insertion, neu, ppoint, pts);
                uint32_t cnt = live_row(pid, 2 * M, buf);  // nearest_iter(pid) without take (core:487)
                for (uint32_t j = 0; j < cnt; ++j) push(insertion, buf[j], ppoint, pts);
                select_heuristic(insertion, ppoint,
                                 [&](uint32_t p, uint32_t links, uint32_t* b) {
                                     // extend_candidates would re-lock zero[new] here and deadlock in the
                                     // reference (core:438 vs core:649 via types:146); we read it unlocked.
                                     if (p == neu) return copy_row(zrow(p), 2 * M, links, b);
                                     return live_row(p, links, b);
                                 },
                                 pts, M, heuristic);
                // ZeroNode::rewrite (types:88-98)
                locks[pid].lock();
                uint32_t* row = zrow(pid);
                size_t it = 0;
                for (uint32_t sidx = 0; sidx < 2 * M; ++sidx) {
                    if (it < insertion.nearest.size()) row[sidx] = key_pid(insertion.nearest[it++]);
                    else if (row[sidx] != INVALID) row[sidx] = INVALID;
                    else break;
                }
                locks[pid].unlock();
            } else {
                // simple mode (core:497-515) incl. the reversed comparator at core:510
                const float* old = pts.row(pid);
                uint32_t dnew = key_dbits(found[i]);
                locks[pid].lock_shared();
                uint32_t* row = zrow(pid);
                size_t idx = rust_binary_search_by(2 * (size_t)M, [&](size_t k) -> int {
                    uint32_t third = row[k];
                    if (third == INVALID) return +1;  // Ordering::Greater (core:507)
                    uint32_t dt = canon_bits(pts.distance(old, pts.row(third)));
                    return dnew < dt ? -1 : (dnew > dt ? +1 : 0);  // distance.cmp(&third_distance) (core:510)
                });
                locks[pid].unlock_shared();
                locks[pid].lock();
                // ZeroNode::insert (types:100-113)
                if (idx < 2 * (size_t)M) {
                    if (row[idx] != INVALID) std::memmove(row + idx + 1, row + idx, (2 * M - 1 - idx) * sizeof(uint32_t));
                    row[idx] = neu;
                }
                locks[pid].unlock();
            }
            node[i] = pid;  // ZeroNode::set (types:115-117)
        }
        locks[neu].unlock();
        pool_push(pr);
    }
};

// rand restatement (parity unpinned, see header)
struct Xoshiro256pp {
    uint64_t s[4];
    explicit Xoshiro256pp(uint64_t seed) {  // SeedableRng::seed_from_u64 via SplitMix64
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
        uint64_t res = rotl(s[0] + s[3], 23) + s[0];
        uint64_t t = s[1] << 17;
        s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3];
        s[2] ^= t;
        s[3] = rotl(s[3], 45);
        return res;
    }
    uint32_t next_u32() { return (uint32_t)(next_u64() >> 32); }
    uint32_t random_range_u32(uint32_t range) {  // 0..range, range > 0
        uint64_t m = (uint64_t)next_u32() * range;
        uint32_t result = (uint32_t)(m >> 32), lo = (uint32_t)m;
        if (lo > (uint32_t)(0u - range)) {
            uint32_t new_hi = (uint32_t)(((uint64_t)next_u32() * range) >> 32);
            uint32_t sum = lo + new_hi;
            result += (sum < lo) ? 1u : 0u;  // carry
        }
        return result;
    }
};

std::vector<std::pair<uint64_t, uint64_t>> layer_sizes(uint64_t n, uint32_t M, float ml) {  // core:238-249
    std::vector<std::pair<uint64_t, uint64_t>> sizes;
    uint64_t num = n;
    for (;;) {
        float f = (float)num * ml;
        uint64_t next = f >= 1.8446744e19f ? UINT64_MAX : (f > 0.0f ? (uint64_t)f : 0);  // `as usize` saturates
        if (next < M) break;
        if (next >= num) break;  // ml >= 1 would never terminate in the reference; we stop (documented)
        sizes.push_back({num - next, num});
        num = next;
    }
    sizes.push_back({num, num});
    std::reverse(sizes.begin(), sizes.end());
    return sizes;
}

void shuffle_ids(uint64_t n, uint64_t seed, std::vector<uint32_t>& order /*rank -> orig*/, uint32_t* out /*orig -> pid*/) {
    Xoshiro256pp rng(seed);
    std::vector<std::pair<uint32_t, uint64_t>> sh(n);  // core:257-260
    for (uint64_t i = 0; i < n; ++i) sh[i] = {rng.random_range_u32((uint32_t)n), i};
    std::sort(sh.begin(), sh.end());
    order.resize(n);
    for (uint64_t r = 0; r < n; ++r) {
        order[r] = (uint32_t)sh[r].second;
        if (out) out[sh[r].second] = (uint32_t)r;  // core:267
    }
}

float* alloc_rows(size_t n, size_t stride) {
    size_t bytes = std::max<size_t>(64, n * stride * sizeof(float));
    bytes = (bytes + 63) / 64 * 64;
    float* p = (float*)std::aligned_alloc(64, bytes);
    if (p) std::memset(p, 0, bytes);
    return p;
}

template <class F>
void parallel_for(uint64_t begin, uint64_t end, int threads, uint64_t chunk, F&& f) {
    if (threads <= 1 || end - begin <= chunk) {
        for (uint64_t i = begin; i < end; ++i) f(i, 0);
        return;
    }
    std::atomic<uint64_t> next{begin};
    std::vector<std::thread> th;
    for (int t = 0; t < threads; ++t)
        th.emplace_back([&, t]() {
            for (;;) {
                uint64_t b = next.fetch_add(chunk);
                if (b >= end) return;
                uint64_t e = std::min(end, b + chunk);
                for (uint64_t i = b; i < e; ++i) f(i, t);
            }
        });
    for (auto& x : th) x.join();
}

}  // namespace

// ================================================================================================
// C API (used from Python via ctypes by tests/ and bench.py only)
// ================================================================================================
struct orc_params {
    uint32_t M;                // reference: const M = 32 (core:787); runtime here for BASELINE configs M=16/24
    uint32_t ef_construction;  // core:105
    uint32_t ef_search;        // core:104
    float ml;                  // core:107  (1/ln M)
    uint64_t seed;             // core:108
    int32_t heuristic;         // Some(Heuristic) / None   (core:106)
    int32_t extend_candidates; // core:124
    int32_t keep_pruned;       // core:125
    int32_t threads;           // 1 = strictly sequential (deterministic); >1 mimics rayon (core:316-318)
    int32_t metric;            // 0 canonical squared L2 (product); 1 sqrt-L2 sequential (reference's test Point)
};

ORC_API void orc_params_default(orc_params* p) {
    p->M = 32;
    p->ef_construction = 100;
    p->ef_search = 100;
    p->ml = 1.0f / std::log((float)32);
    p->seed = 0;
    p->heuristic = 1;
    p->extend_candidates = 0;
    p->keep_pruned = 1;
    p->threads = 1;
    p->metric = 0;
}

ORC_API float orc_default_ml(uint32_t M) { return 1.0f / std::log((float)M); }

ORC_API float orc_l2sq(const float* a, const float* b, uint32_t dim) { return g_l2sq(a, b, dim); }
ORC_API float orc_l2sq_reference_order(const float* a, const float* b, uint32_t dim) { return l2sq_reference_avx2_order(a, b, dim); }
ORC_API float orc_l2sq_scalar(const float* a, const float* b, uint32_t dim) { return l2sq_canonical_scalar(a, b, dim); }
ORC_API int orc_simd_level() { return g_l2sq == l2sq_canonical_scalar ? 0 : 512; }

// counts[l] = node count of layer l; returns number of layers (core:238-250, 275-281)
ORC_API uint32_t orc_layer_schedule(uint64_t n, uint32_t M, float ml, uint64_t* counts, uint32_t cap) {
    if (n == 0) return 0;
    auto sizes = layer_sizes(n, M, ml);
    uint32_t L = (uint32_t)sizes.size();
    for (uint32_t i = 0; i < L && (L - 1 - i) < cap; ++i) counts[L - 1 - i] = sizes[i].second;
    return L;
}

// out_ids[orig] = PointId (core:262-270)
// Known-answer access to the rand restatement: the first `count` next_u64 outputs from a raw state (`state` != null: the xoshiro256++
// reference implementation's own vector, s = {1,2,3,4}) or from seed_from_u64(seed) (SplitMix64 expansion).  Checked against the
// published vectors in tests/test_oracle_reference_pins.py.
ORC_API void orc_rng_kat(const uint64_t* state, uint64_t seed, uint64_t* out, uint32_t count) {
    Xoshiro256pp rng(seed);
    if (state) std::memcpy(rng.s, state, sizeof rng.s);
    for (uint32_t i = 0; i < count; ++i) out[i] = rng.next_u64();
}

ORC_API void orc_shuffle(uint64_t n, uint64_t seed, uint32_t* out_ids) {
    std::vector<uint32_t> order;
    shuffle_ids(n, seed, order, out_ids);
}

// Shared by orc_build and orc_build_batched, for n >= 1: layer schedule (core:238-249), shuffle and shuffled rows
// (core:257-270), an all-INVALID zero layer and empty snapshots.  Returns the (size, cumulative) pairs, top layer first.
static std::vector<std::pair<uint64_t, uint64_t>> init_index(orc_index* ix, const float* rows, uint64_t n, uint32_t dim,
                                                             const orc_params* p, uint32_t* out_ids) {
    const uint32_t M = p->M;
    auto sizes = layer_sizes(n, M, p->ml);
    const uint32_t num_layers = (uint32_t)sizes.size(), top = num_layers - 1;
    ix->layer_n.assign(num_layers, 0);
    for (uint32_t i = 0; i < num_layers; ++i) ix->layer_n[num_layers - 1 - i] = sizes[i].second;

    std::vector<uint32_t> order;
    shuffle_ids(n, p->seed, order, out_ids);
    ix->points = alloc_rows(n, ix->stride);
    int threads = std::max(1, p->threads);
    parallel_for(0, n, threads, 4096, [&](uint64_t r, int) {
        std::memcpy(ix->points + r * ix->stride, rows + (size_t)order[r] * dim, dim * sizeof(float));
    });

    ix->zero.assign(n * 2 * (size_t)M, INVALID);
    ix->layers.assign(top, {});
    return sizes;
}

// UpperNode::from_zero (types:65-71) for nodes [0, end) of a finished layer.
static void snapshot_layer(orc_index* ix, uint32_t layer, uint64_t end, int threads) {
    const uint32_t M = ix->M;
    auto& snap = ix->layers[layer - 1];
    snap.resize(end * (size_t)M);
    parallel_for(0, end, threads, 4096, [&](uint64_t v, int) {
        std::memcpy(snap.data() + v * M, ix->zero.data() + v * 2 * M, M * sizeof(uint32_t));
    });
}

ORC_API orc_index* orc_build(const float* rows, uint64_t n, uint32_t dim, const orc_params* p, uint32_t* out_ids) {
    auto* ix = new orc_index();
    ix->M = p->M;
    ix->dim = dim;
    ix->stride = ((size_t)dim + 3) / 4 * 4;
    ix->n = n;
    ix->ef_search = p->ef_search;
    ix->metric = p->metric;
    if (n == 0) return ix;  // core:224-234
    if (n >= 0xFFFFFFFFull) { delete ix; return nullptr; }  // core:256

    const auto sizes = init_index(ix, rows, n, dim, p, out_ids);
    const uint32_t num_layers = (uint32_t)sizes.size(), top = num_layers - 1;
    const int threads = std::max(1, p->threads);

    Construction st;
    st.ix = ix;
    st.locks = std::vector<RwSpin>(n);
    st.top = top;
    st.heuristic.on = p->heuristic != 0;
    st.heuristic.extend_candidates = p->extend_candidates != 0;
    st.heuristic.keep_pruned = p->keep_pruned != 0;
    st.ef_construction = p->ef_construction;
    st.pts = ix->pts();

    for (uint32_t i = 0; i < num_layers; ++i) {  // core:304-329
        uint32_t layer = num_layers - i - 1;
        uint64_t size = sizes[i].first, cumulative = sizes[i].second;
        uint64_t start = std::max<uint64_t>(cumulative - size, 1), end = cumulative;
        if (layer == top || threads <= 1) {
            for (uint64_t v = start; v < end; ++v) st.insert((uint32_t)v, layer);
        } else {
            parallel_for(start, end, threads, 16, [&](uint64_t v, int) { st.insert((uint32_t)v, layer); });
        }
        if (layer != 0) snapshot_layer(ix, layer, end, threads);
    }
    for (auto& pr : st.pool) { delete pr.first; delete pr.second; }
    return ix;
}

// ================================================================================================
// Batched build: a CPU statement of THIS LIBRARY's batch schedule (DESIGN.md §6, csrc/build.cu), not of the reference.
// The reference inserts concurrently under rayon and per-row locks, so its threaded graphs are not reproducible; the
// library replaces that with a deterministic schedule, and this section states that schedule with the oracle's own
// push / search_layer / select_heuristic, so batched GPU graphs can be checked bit for bit.  Per layer, top first:
//   schedule  b = 1 on the top layer, else min(max_batch, max(1, g0 / growth)), clipped to the end of the layer;
//   KA        every insert of a batch runs Construction::insert's descent against the zero layer as it stood when
//             the batch began (no row changes during the batch);
//   K2        each insert selects its own neighbours (select_heuristic, or the first min(len, 2M) in simple mode),
//             writes its whole row and emits (target <- new) link requests;
//   K2'       requests sorted by (target, new).  Heuristic mode: each target row is re-pruned in rounds of at most
//             kNewCap = 32 new ids, ascending; a round's candidates are its new ids followed by the row's valid prefix,
//             pushed in that order with ef = ef_construction (push admission, no truncation), then select_heuristic,
//             then the whole row is rewritten.  Simple mode: one request at a time in ascending `new` order, with the
//             reversed-comparator binary search and ZeroNode::insert of core:497-515.
// With max_batch = 1 this is exactly orc_build's sequential order.  Inserts of a batch and targets of a batch run on
// `threads` workers; each touches only its own output, so the graph does not depend on the thread count.
// ================================================================================================
struct orc_batch_stats {
    uint64_t batches;                   // batches over all layers
    uint64_t max_batch;                 // inserts in the largest batch
    uint64_t link_requests;             // (target <- new) pairs, over all batches
    uint64_t targets;                   // distinct target rows, summed over batches
    uint64_t max_target_requests;       // most requests one target received in one batch (the largest hub)
    uint64_t multi_new_rounds;          // heuristic re-prune rounds with more than one new id
    uint64_t multi_round_targets;       // heuristic targets that needed more than one round in one batch
    uint64_t admission_limited_rounds;  // heuristic rounds with ef_construction < C (push admission may reject)
    uint64_t simple_multi_targets;      // simple-mode targets with more than one request in one batch
    uint64_t max_insert_dist;           // most distance evaluations of one layer-0 insert on layer 0 (<= ids it visited there)
};

namespace {
constexpr uint32_t kNewCap = 32;  // new ids per re-prune round (build_kernels.cuh)

void merge_stats(orc_batch_stats& a, const orc_batch_stats& b) {
    a.link_requests += b.link_requests;
    a.targets += b.targets;
    a.max_target_requests = std::max(a.max_target_requests, b.max_target_requests);
    a.multi_new_rounds += b.multi_new_rounds;
    a.multi_round_targets += b.multi_round_targets;
    a.admission_limited_rounds += b.admission_limited_rounds;
    a.simple_multi_targets += b.simple_multi_targets;
    a.max_insert_dist = std::max(a.max_insert_dist, b.max_insert_dist);
}
}  // namespace

// out_batches (optional): (first PointId, inserts) of the first batch_cap batches, in build order.
// row_batch (optional, n entries): index of the last batch that wrote each zero row (INVALID: never written).
ORC_API orc_index* orc_build_batched(const float* rows, uint64_t n, uint32_t dim, const orc_params* p, uint32_t max_batch,
                                     uint32_t growth, orc_batch_stats* stats, uint64_t* out_batches, uint64_t batch_cap,
                                     uint32_t* row_batch, uint32_t* out_ids) {
    orc_batch_stats total;
    std::memset(&total, 0, sizeof(total));
    if (stats) *stats = total;
    if (row_batch) std::fill(row_batch, row_batch + n, INVALID);
    if (max_batch == 0 || growth == 0 || p->extend_candidates) return nullptr;  // the library rejects extend_candidates
    auto* ix = new orc_index();
    ix->M = p->M;
    ix->dim = dim;
    ix->stride = ((size_t)dim + 3) / 4 * 4;
    ix->n = n;
    ix->ef_search = p->ef_search;
    ix->metric = p->metric;
    if (n == 0) return ix;
    if (n >= 0xFFFFFFFFull) { delete ix; return nullptr; }

    const auto sizes = init_index(ix, rows, n, dim, p, out_ids);
    const uint32_t num_layers = (uint32_t)sizes.size(), top = num_layers - 1;
    const int threads = std::max(1, p->threads);
    const uint32_t M = p->M, cap = 2 * M;
    const size_t efc = p->ef_construction;
    Heuristic h;
    h.on = p->heuristic != 0;
    h.keep_pruned = p->keep_pruned != 0;
    const Points pts = ix->pts();
    auto zrow = [&](uint32_t pid) { return ix->zero.data() + (size_t)pid * cap; };
    auto no_rows = [](uint32_t, uint32_t, uint32_t*) { return 0u; };  // extend_candidates is off: no row is read

    std::vector<Search> searches(threads);
    for (auto& s : searches) s.visited.with_capacity(n);
    std::vector<orc_batch_stats> tstats(threads);
    std::vector<uint32_t> found;   // max_batch x 2M: own rows of the batch's inserts
    std::vector<uint64_t> pairs;   // (target << 32 | new)
    std::vector<uint64_t> seg;     // start index of each target's requests in `pairs`
    uint64_t batch_index = 0;

    for (uint32_t li = 0; li < num_layers; ++li) {
        const uint32_t layer = num_layers - li - 1;
        const uint64_t size = sizes[li].first, cumulative = sizes[li].second;
        const uint64_t start = std::max<uint64_t>(cumulative - size, 1), end = cumulative;
        const uint32_t num = layer == 0 ? 2 * M : M;  // core:445
        for (uint64_t g0 = start; g0 < end;) {
            uint64_t b = 1;
            if (layer != top) b = std::min<uint64_t>(max_batch, std::max<uint64_t>(1, g0 / growth));
            b = std::min<uint64_t>(b, end - g0);
            if (out_batches && batch_index < batch_cap) { out_batches[2 * batch_index] = g0; out_batches[2 * batch_index + 1] = b; }
            total.batches++;
            total.max_batch = std::max<uint64_t>(total.max_batch, b);
            for (auto& t : tstats) std::memset(&t, 0, sizeof(t));

            // ---- KA + K2: every insert against the zero layer as the batch found it ----
            found.assign(b * cap, INVALID);
            parallel_for(0, b, threads, 4, [&](uint64_t w, int t) {
                const uint32_t neu = (uint32_t)(g0 + w);
                const float* point = pts.row(neu);
                Search& s = searches[t];
                s.reset();
                push(s, 0, point, pts);  // core:444
                for (uint32_t cur = top;; --cur) {  // core:447-463
                    s.ef = cur <= layer ? efc : 1;
                    if (cur > layer) {
                        const uint32_t* snap = ix->layers[cur - 1].data();
                        search_layer(s, point, [&](uint32_t pid, uint32_t links, uint32_t* buf) {
                            return copy_row(snap + (size_t)pid * M, M, links, buf); }, pts, num);
                        s.cull();
                    } else {
                        s.n_dist = 0;
                        search_layer(s, point, [&](uint32_t pid, uint32_t links, uint32_t* buf) {
                            return copy_row(zrow(pid), cap, links, buf); }, pts, num);
                        if (layer == 0) tstats[t].max_insert_dist = std::max<uint64_t>(tstats[t].max_insert_dist, s.n_dist);
                        break;
                    }
                    if (cur == 0) break;
                }
                if (h.on) select_heuristic(s, point, no_rows, pts, M, h);  // core:470-472
                else if (s.nearest.size() > cap) s.nearest.resize(cap);  // core:466-469
                for (size_t i = 0; i < s.nearest.size(); ++i) found[w * cap + i] = key_pid(s.nearest[i]);
            });

            // ---- own rows and link requests, grouped by target ----
            pairs.clear();
            for (uint64_t w = 0; w < b; ++w) {
                const uint32_t neu = (uint32_t)(g0 + w);
                std::memcpy(zrow(neu), &found[w * cap], cap * sizeof(uint32_t));
                if (row_batch) row_batch[neu] = (uint32_t)batch_index;
                for (uint32_t i = 0; i < cap && found[w * cap + i] != INVALID; ++i)
                    pairs.push_back(((uint64_t)found[w * cap + i] << 32) | neu);
            }
            std::sort(pairs.begin(), pairs.end());
            seg.clear();
            for (size_t i = 0; i < pairs.size(); ++i)
                if (i == 0 || (pairs[i] >> 32) != (pairs[i - 1] >> 32)) seg.push_back(i);
            total.link_requests += pairs.size();
            total.targets += seg.size();

            // ---- K2': every target row, once per batch ----
            parallel_for(0, seg.size(), threads, 16, [&](uint64_t si, int t) {
                const size_t s0 = seg[si], s1 = si + 1 < seg.size() ? seg[si + 1] : pairs.size();
                const uint32_t tgt = (uint32_t)(pairs[s0] >> 32);
                const float* tpoint = pts.row(tgt);
                uint32_t* row = zrow(tgt);
                orc_batch_stats& ts = tstats[t];
                ts.max_target_requests = std::max<uint64_t>(ts.max_target_requests, s1 - s0);
                if (row_batch) row_batch[tgt] = (uint32_t)batch_index;
                if (!h.on) {
                    if (s1 - s0 > 1) ts.simple_multi_targets++;
                    for (size_t r = s0; r < s1; ++r) {  // core:497-515, ascending `new`
                        const uint32_t neu = (uint32_t)pairs[r];
                        const uint32_t dnew = canon_bits(pts.distance(tpoint, pts.row(neu)));
                        const size_t idx = rust_binary_search_by(cap, [&](size_t k) -> int {
                            const uint32_t third = row[k];
                            if (third == INVALID) return +1;
                            const uint32_t dt = canon_bits(pts.distance(tpoint, pts.row(third)));
                            return dnew < dt ? -1 : (dnew > dt ? +1 : 0);
                        });
                        if (idx < cap) {  // ZeroNode::insert (types:100-113)
                            if (row[idx] != INVALID) std::memmove(row + idx + 1, row + idx, (cap - 1 - idx) * sizeof(uint32_t));
                            row[idx] = neu;
                        }
                    }
                    return;
                }
                if (s1 - s0 > kNewCap) ts.multi_round_targets++;
                Search& s = searches[t];
                uint32_t buf[256];
                for (size_t r0 = s0; r0 < s1; r0 += kNewCap) {
                    const size_t r1 = std::min<size_t>(s1, r0 + kNewCap);
                    if (r1 - r0 > 1) ts.multi_new_rounds++;
                    s.reset();
                    s.ef = efc;
                    for (size_t r = r0; r < r1; ++r) push(s, (uint32_t)pairs[r], tpoint, pts);  // the new ids first (core:626)
                    const uint32_t cnt = copy_row(row, cap, cap, buf);
                    for (uint32_t j = 0; j < cnt; ++j) push(s, buf[j], tpoint, pts);  // then the row (core:627-629)
                    if (efc < (r1 - r0) + cnt) ts.admission_limited_rounds++;
                    select_heuristic(s, tpoint, no_rows, pts, M, h);
                    for (uint32_t i = 0; i < cap; ++i) row[i] = i < s.nearest.size() ? key_pid(s.nearest[i]) : INVALID;
                }
            });
            for (const auto& t : tstats) merge_stats(total, t);
            g0 += b;
            batch_index++;
        }
        if (layer != 0) snapshot_layer(ix, layer, end, threads);
    }
    if (stats) *stats = total;
    return ix;
}

// Wrap an existing graph ("search a given graph": the parity entry).  points are in PointId order.
ORC_API orc_index* orc_from_graph(const float* points, uint64_t n, uint32_t dim, uint32_t M, uint32_t ef_search,
                                  const uint32_t* zero, uint32_t n_upper, const uint32_t* const* upper,
                                  const uint64_t* upper_n, int32_t metric) {
    auto* ix = new orc_index();
    ix->M = M; ix->dim = dim; ix->stride = ((size_t)dim + 3) / 4 * 4; ix->n = n;
    ix->ef_search = ef_search; ix->metric = metric;
    if (n == 0) return ix;
    ix->points = alloc_rows(n, ix->stride);
    for (uint64_t r = 0; r < n; ++r) std::memcpy(ix->points + r * ix->stride, points + r * dim, dim * sizeof(float));
    ix->zero.assign(zero, zero + n * 2 * (size_t)M);
    ix->layers.resize(n_upper);
    ix->layer_n.assign(n_upper + 1, 0);
    ix->layer_n[0] = n;
    for (uint32_t l = 0; l < n_upper; ++l) {
        ix->layers[l].assign(upper[l], upper[l] + upper_n[l] * (size_t)M);
        ix->layer_n[l + 1] = upper_n[l];
    }
    return ix;
}

ORC_API void orc_free(orc_index* ix) { delete ix; }
ORC_API uint64_t orc_n(const orc_index* ix) { return ix->n; }
ORC_API uint32_t orc_dim(const orc_index* ix) { return ix->dim; }
ORC_API uint32_t orc_M(const orc_index* ix) { return ix->M; }
ORC_API uint32_t orc_num_layers(const orc_index* ix) { return ix->n == 0 ? 0 : (uint32_t)ix->layers.size() + 1; }
ORC_API uint64_t orc_layer_count(const orc_index* ix, uint32_t l) {
    if (l == 0) return ix->n;
    return ix->layers[l - 1].size() / ix->M;
}
ORC_API void orc_export_points(const orc_index* ix, float* out /* n x dim */) {
    for (size_t r = 0; r < ix->n; ++r) std::memcpy(out + r * ix->dim, ix->points + r * ix->stride, ix->dim * sizeof(float));
}
ORC_API void orc_export_zero(const orc_index* ix, uint32_t* out /* n x 2M */) {
    std::memcpy(out, ix->zero.data(), ix->zero.size() * sizeof(uint32_t));
}
ORC_API void orc_export_upper(const orc_index* ix, uint32_t l /*1-based*/, uint32_t* out /* n_l x M */) {
    std::memcpy(out, ix->layers[l - 1].data(), ix->layers[l - 1].size() * sizeof(uint32_t));
}

// Hnsw::search (core:352-383) for nq queries over `threads` workers, one Search per worker (the shape a
// rayon `par_iter().map_init(Search::default, ...)` harness would have; the reference itself is 1 query/call).
// out_ids/out_dist: nq x k_cap (first min(len,k_cap) of `nearest`); out_len[q] = len(nearest) (<= ef_search).
// counters (optional): nq x 4 = {n_expand_upper, n_dist_upper, n_expand_zero, n_dist_zero}.
ORC_API int orc_search(const orc_index* ix, const float* queries, uint64_t nq, uint32_t ef_search, uint32_t k_cap,
                       uint32_t* out_ids, float* out_dist, uint32_t* out_len, uint64_t* counters, int32_t threads) {
    const uint32_t M = ix->M, dim = ix->dim;
    const size_t qstride = ((size_t)dim + 3) / 4 * 4;
    Points pts = ix->pts();
    int T = std::max(1, threads);
    std::vector<Search> searches(T);
    std::vector<std::vector<float>> qbuf(T, std::vector<float>(qstride + 16, 0.0f));
    parallel_for(0, nq, T, 8, [&](uint64_t qi, int t) {
        Search& s = searches[t];
        float* q = qbuf[t].data();
        std::memcpy(q, queries + qi * dim, dim * sizeof(float));
        Counters c;
        s.reset();  // core:357
        if (ix->n != 0) {
            s.visited.reserve_capacity(ix->n);  // core:363
            s.n_dist = s.n_expand = 0;
            push(s, 0, q, pts);  // core:364
            for (uint32_t cur = (uint32_t)ix->layers.size();; --cur) {  // core:365
                s.ef = cur == 0 ? ef_search : 1;
                uint32_t num = cur == 0 ? 2 * M : M;
                if (cur == 0) {
                    const uint32_t* z = ix->zero.data();
                    search_layer(s, q, [&](uint32_t pid, uint32_t links, uint32_t* buf) {
                        return copy_row(z + (size_t)pid * 2 * M, 2 * M, links, buf); }, pts, num);
                    c.n_expand_zero = s.n_expand; c.n_dist_zero = s.n_dist;
                    break;
                }
                const uint32_t* u = ix->layers[cur - 1].data();
                search_layer(s, q, [&](uint32_t pid, uint32_t links, uint32_t* buf) {
                    return copy_row(u + (size_t)pid * M, M, links, buf); }, pts, num);
                s.cull();  // core:377-379
                c.n_expand_upper += s.n_expand; c.n_dist_upper += s.n_dist;
                s.n_expand = s.n_dist = 0;
            }
        }
        uint32_t len = (uint32_t)s.nearest.size();
        if (out_len) out_len[qi] = len;
        for (uint32_t j = 0; j < k_cap; ++j) {
            if (out_ids) out_ids[qi * k_cap + j] = j < len ? key_pid(s.nearest[j]) : INVALID;
            if (out_dist) out_dist[qi * k_cap + j] = j < len ? key_dist(s.nearest[j]) : INFINITY;
        }
        if (counters) {
            counters[qi * 4 + 0] = c.n_expand_upper; counters[qi * 4 + 1] = c.n_dist_upper;
            counters[qi * 4 + 2] = c.n_expand_zero;  counters[qi * 4 + 3] = c.n_dist_zero;
        }
    });
    return 0;
}

// Exact k-NN by exhaustive scan with the index's metric; ties by lower id.  Ground truth for recall.
ORC_API int orc_bruteforce(const float* points, uint64_t n, uint32_t dim, const float* queries, uint64_t nq, uint32_t k,
                           uint32_t* out_ids, float* out_dist, int32_t metric, int32_t threads) {
    dist_fn fn = metric_fn(metric);
    const size_t stride = ((size_t)dim + 3) / 4 * 4;
    float* prow = alloc_rows(n ? n : 1, stride);
    for (uint64_t r = 0; r < n; ++r) std::memcpy(prow + r * stride, points + r * dim, dim * sizeof(float));
    int T = std::max(1, threads);
    std::vector<std::vector<float>> qbuf(T, std::vector<float>(stride + 16, 0.0f));
    parallel_for(0, nq, T, 1, [&](uint64_t qi, int t) {
        float* q = qbuf[t].data();
        std::memcpy(q, queries + qi * dim, dim * sizeof(float));
        std::vector<uint64_t> heap;  // max-heap of the k smallest keys
        for (uint64_t r = 0; r < n; ++r) {
            uint64_t key = mk_key(fn(q, prow + r * stride, dim), (uint32_t)r);
            if (heap.size() < k) { heap.push_back(key); std::push_heap(heap.begin(), heap.end()); }
            else if (key < heap.front()) { std::pop_heap(heap.begin(), heap.end()); heap.back() = key; std::push_heap(heap.begin(), heap.end()); }
        }
        std::sort(heap.begin(), heap.end());
        for (uint32_t j = 0; j < k; ++j) {
            out_ids[qi * k + j] = j < heap.size() ? key_pid(heap[j]) : INVALID;
            if (out_dist) out_dist[qi * k + j] = j < heap.size() ? key_dist(heap[j]) : INFINITY;
        }
    });
    std::free(prow);
    return 0;
}

// One select_heuristic call in isolation (core:636-698), for unit-checking the GPU prune kernel.
// in: `cand_ids` (ascending by (dist,pid) w.r.t. `point`, as `nearest` is) -> out ids (<= 2M), returns count.
ORC_API uint32_t orc_select_heuristic(const orc_index* ix, const float* point, const uint32_t* cand_ids, uint32_t n_cand,
                                      int32_t keep_pruned, uint32_t* out_ids, float* out_dist) {
    Points pts = ix->pts();
    Search s;
    s.visited.with_capacity(ix->n);
    std::vector<float> q(ix->stride + 16, 0.0f);
    std::memcpy(q.data(), point, ix->dim * sizeof(float));
    for (uint32_t i = 0; i < n_cand; ++i)
        s.nearest.push_back(mk_key(pts.distance(q.data(), pts.row(cand_ids[i])), cand_ids[i]));
    Heuristic h;
    h.keep_pruned = keep_pruned != 0;
    select_heuristic(s, q.data(), [&](uint32_t, uint32_t, uint32_t*) { return 0u; }, pts, ix->M, h);
    for (size_t i = 0; i < s.nearest.size(); ++i) {
        out_ids[i] = key_pid(s.nearest[i]);
        if (out_dist) out_dist[i] = key_dist(s.nearest[i]);
    }
    return (uint32_t)s.nearest.size();
}
