// internal.cuh — host-side index object, per-device shared context and kernel argument blocks (not part of the public ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <functional>
#include <mutex>
#include <new>
#include <utility>
#include <vector>

#include "../../include/instant_distance_b200.h"
#include "hnsw_device.cuh"

namespace idb {

// Warps (= live queries / inserts) per CTA of the traversal kernels.  A CTA's resources are only handed to the next launch when ALL its
// warps have finished their last query, so fewer warps per CTA means the next batch moves in sooner at a batch boundary.
#ifndef IDB_WPC
#define IDB_WPC 4
#endif
constexpr int kSearchWarps = IDB_WPC;
constexpr int kSearchCtasPerSm = 16 / IDB_WPC;  // resident CTAs per SM -> 16 live queries per SM, <= 128 registers per thread
constexpr int kMaxCtasPerSm = 32 / IDB_WPC;     // upper bound for IDB_CTAS_PER_SM
constexpr int kRetryCtas = 32 / IDB_WPC;        // CTA slots of the (normally idle) overflow-retry pool -> 32 warps
constexpr int occ_for_warps(int warps_per_sm) { return warps_per_sm / IDB_WPC; }
constexpr uint32_t kRetrySlots = 1u << 18;  // hash slots per retry warp: 196k ids at 3/4 load (2M * ef <= 131k for M <= 64, ef <= 1024)
constexpr int kLanes = 4;              // submission lanes per index (own stream + per-call control state)

extern thread_local char g_err[512];
idb_status fail(idb_status st, const char* fmt, ...);

#define CUDA_TRY(expr)                                                                                         \
    do {                                                                                                       \
        cudaError_t e__ = (expr);                                                                              \
        if (e__ != cudaSuccess)                                                                                \
            return ::idb::fail(e__ == cudaErrorMemoryAllocation ? IDB_ERR_OOM : IDB_ERR_CUDA, "CUDA error %s at %s:%d (%s)", \
                               cudaGetErrorName(e__), __FILE__, __LINE__, cudaGetErrorString(e__));             \
    } while (0)

// Float4 chunks per lane of the traversal instantiation that serves rows of `nchunks` chunks: 1, 2, 3, 4, 6 or 8, and 0 for rows of
// more than 1024 elements (the long-row kernels, whose query lives in shared memory).
constexpr int kernel_ch(uint32_t nchunks) {
    const uint32_t c = (nchunks + 31) / 32;
    return c <= 4 ? (int)c : c <= 6 ? 6 : c <= 8 ? 8 : 0;
}

// The traversal cell of CH = kernel_ch(nchunks): B is its rows in flight per lane for f32 rows.  K1 and the graph range expansion
// take rows_in_flight<B, RT>() of it (search_kernel.cuh); KA, K2 / K2' and repair_kernel take B as is.
template <int CH_>
struct Cell {
    static constexpr int CH = CH_;
    static constexpr int B = CH == 1 ? 16 : CH == 2 ? 8 : CH == 3 || CH == 4 ? 4 : CH == 6 || CH == 8 ? 2 : kLongRowsInFlight;
};
// f(Cell<kernel_ch(nchunks)>()): the one switch from a row's chunk count to the cell compiled for it.
template <class F>
auto with_cell(uint32_t nchunks, F&& f) {
    switch (kernel_ch(nchunks)) {
        case 1: return f(Cell<1>());
        case 2: return f(Cell<2>());
        case 3: return f(Cell<3>());
        case 4: return f(Cell<4>());
        case 6: return f(Cell<6>());
        case 8: return f(Cell<8>());
        default: return f(Cell<0>());
    }
}

// The big visited tier a traversal's warps bind (Index::select_visited_tier, DeviceCtx::retry_tier).
struct VisTier {
    TablePool pool;                    // per-warp scratch tables, claimed per CTA (hnsw_device.cuh)
    uint32_t gslots, gshift;           // words in use per warp / hash flavour: 32 - log2(gslots)
    uint32_t mode;                     // flavour (hnsw_device.cuh VisMode)
    uint32_t b16_cap_ids;              // b16 flavour: ids per traversal before the retry pass takes over
    uint32_t b16_nb;                   // b16 flavour: buckets in use over both segments
};

// The work items of one traversal pass (K1 or KA) and where it reports on them.
struct TraversalWork {
    unsigned long long n_work;         // number of work items ...
    const uint32_t* n_work_dev;        // ... or, if non-null, read it from device memory (retry pass)
    const uint32_t* work_list;         // optional indirection: work item -> query / insert index
    unsigned long long* work_counter;
    uint32_t* status;                  // per query / insert: QueryStatus
    uint32_t* fail_count;
    uint32_t* fail_list;               // items whose visited table / tie list overflowed; null in the retry pass
};

// Device-side counters of one traversal pass, zeroed before it.
struct PassCtrl {
    unsigned long long work_counter;
    uint32_t fail_count;
};
// A search call's control block (Lane::ctrl).
struct SearchCtrl {
    PassCtrl main, retry;              // K1 and its retry pass
    unsigned long long full_fetches;   // rows fetched in full (the rows the screen did not drop), by both passes
};

struct SearchArgs {
    GraphView g;
    const float4* queries;             // nq x nchunks float4 (zero padded rows)
    TraversalWork work;
    uint32_t ef, k;
    uint32_t* out_ids;
    float* out_dist;
    uint32_t* out_len;
    uint32_t* counters;                // nq x 4 u32 or null
    VisTier tier;
    uint64_t* out_keys;                // optional: nq x k packed (distance bits << 32 | id_map[pid]) for the sharded all-gather
    const uint32_t* id_map;            // optional: PointId -> caller's global row id
    int variant;                       // tuning variant of the kernel template (0 = default)
    uint32_t metric;                   // Metric: how out_dist reports a key's distance (out_keys always carry the key's own bits)
    unsigned long long* full_tally;    // optional: += rows fetched in full (the rows the screen did not drop), over the call
    uint32_t* launched;                // HOST memory, optional: launch_search writes the K1 instantiation it launched (Lane::last_kernel)
};

// Persisting-L2 access-policy window attached to a launch (the b16 visited tables), or none.
struct LaunchWindow {
    void* base = nullptr;
    size_t bytes = 0;
    float hit_ratio = 1.0f;
};

// ---------------------------------------------------------------------------------------------------------
// One per CUDA device, shared by every index on it (reference-counted): the pool of per-warp scratch tables (sized for the
// warps that can be RESIDENT, not per index or per call), the retry pool, and the device's persisting-L2 reservation.
// ---------------------------------------------------------------------------------------------------------
struct DeviceCtx {
    int device = 0;
    int num_sms = 132;
    int sm_ids = 132;                      // %nsmid: SM ids are < sm_ids, which can exceed the number of enabled SMs
    int slots_per_sm = kSearchCtasPerSm;   // CTA slots per SM (IDB_CTAS_PER_SM)
    std::mutex mu;                         // held while tables are (re)allocated and while a launch that uses them is enqueued
    uint32_t* slot_masks = nullptr;        // sm_ids words + 1 (the retry pool)
    uint32_t n_tables = 0;                 // sm_ids * slots_per_sm * kSearchWarps (only those of enabled SMs are ever touched)
    uint32_t n_tables_live = 0;            // num_sms * slots_per_sm * kSearchWarps: how many can be in use at once
    // b16 tier: fixed stride per warp, a prefix of it in use per call
    uint32_t* b16_tables = nullptr;        // first segment of every table: what normal traversals use, under the persisting-L2 window
    uint32_t b16_stride = 0;               // u32 words per warp = b16_l2_bytes / 4
    uint32_t b16_l2_bytes = 32 * 1024;     // bytes per warp that keep all live tables inside the persisting part of L2
    uint32_t* b16_ext = nullptr;           // second segment (same size), used by traversals with a large ef; not under the window
    // atomic tiers (hash / bitmap): allocated on first use, regrown (device idle) when a call needs more
    uint32_t* big_tables = nullptr;
    uint32_t big_stride = 0;
    uint32_t* retry_tables = nullptr;      // kRetryCtas * kSearchWarps tables of kRetrySlots words
    uint64_t* tie_tables = nullptr;        // n_tables * kTieCap
    uint64_t* retry_ties = nullptr;        // kRetryCtas * kSearchWarps * kRetryTieCap
    int max_persist = 0, max_window = 0;
    size_t l2_reserved = 0;                // current cudaLimitPersistingL2CacheSize set by this library
    bool l2_allowed = false;               // idb_device_set_persisting_l2 / IDB_L2_PERSIST
    int refs = 0;

    static idb_status acquire(int device, DeviceCtx** out);
    static void release(DeviceCtx* c);
    idb_status ensure_big(uint32_t stride_words);          // caller holds mu
    idb_status reserve_l2(size_t bytes);                    // caller holds mu
    TablePool main_pool(bool b16) const;
    VisTier retry_tier() const;                             // the retry pool's 2^18-slot hash sets
    ~DeviceCtx();
};

// The arguments of the retry pass behind a main traversal pass `a` (device-side, unconditional, normally a no-op): a few warps re-run
// the items whose visited table or tie list overflowed, from a.work.fail_list, as many as the main pass counted on the device, with
// the retry pool's tables.  Failures of the retry pass are only counted in ctrl->fail_count (and visible in status).
template <class Args>
Args retry_pass(const Args& a, const DeviceCtx& c, PassCtrl* ctrl) {
    Args r = a;
    r.work.n_work = 0;
    r.work.n_work_dev = a.work.fail_count;
    r.work.work_list = a.work.fail_list;
    r.work.work_counter = &ctrl->work_counter;
    r.work.fail_count = &ctrl->fail_count;
    r.work.fail_list = nullptr;
    r.tier = c.retry_tier();
    return r;
}

// Per-call control state + host-API staging buffers; one per submission lane.  Calls on one lane are stream-ordered, so the
// buffers are reused without waiting; calls on different lanes overlap on the device.
struct Lane {
    std::mutex mu;
    cudaStream_t stream = nullptr;
    SearchCtrl* ctrl = nullptr;
    uint32_t* status = nullptr;   size_t status_cap = 0;
    uint32_t* fail_list = nullptr; size_t fail_cap = 0;
    uint32_t* counters = nullptr; size_t counters_cap = 0;
    float* q = nullptr;           size_t q_cap = 0;    // the call's queries in the kernel layout (Index::stage_queries)
    float* qn = nullptr;          size_t qn_cap = 0;   // a cosine call's normalised queries (Index::normalize_queries)
    uint32_t* ids = nullptr;      size_t ids_cap = 0;
    float* dist = nullptr;        size_t dist_cap = 0;
    uint32_t* len = nullptr;      size_t len_cap = 0;
    // sharded search
    uint64_t* keys_local = nullptr; size_t keys_local_cap = 0;
    uint64_t* keys_all = nullptr;   size_t keys_all_cap = 0;
    uint32_t* shard_ids = nullptr;  size_t shard_ids_cap = 0;   // the shard's K1 ids (its keys carry the results)
    // exact search: the (query, slice) k-lists of the current query chunk (exact.cu)
    uint64_t* exact_keys = nullptr; size_t exact_keys_cap = 0;
    // range search (range.cu): the appended (key, query) pairs, the keys gathered into their queries' segments, the host call's
    // offsets and the append counter, and CUB's scratch (in u64 words)
    uint64_t* range_keys = nullptr; size_t range_keys_cap = 0;
    uint32_t* range_qids = nullptr; size_t range_qids_cap = 0;
    uint64_t* range_seg = nullptr;  size_t range_seg_cap = 0;
    uint64_t* range_off = nullptr;  size_t range_off_cap = 0;
    uint64_t* range_tmp = nullptr;  size_t range_tmp_cap = 0;
    // graph range search (graph_range.cu): the seed search's keys, the main pass's per-warp frontiers and visited tables, its
    // control words and overflow list, and the retry pass's per-warp frontiers and bitmaps
    uint64_t* gr_seeds = nullptr;   size_t gr_seeds_cap = 0;
    uint64_t* gr_front = nullptr;   size_t gr_front_cap = 0;
    uint32_t* gr_vis = nullptr;     size_t gr_vis_cap = 0;
    uint32_t* gr_ctl = nullptr;     size_t gr_ctl_cap = 0;
    uint64_t* gr_retry = nullptr;   size_t gr_retry_cap = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    // host API: results land here first when the caller's output buffers are pageable (see read_back in api.cu)
    unsigned char* h_out = nullptr; size_t h_out_cap = 0;   // pinned
    // asynchronous read-back of the control block of the lane's last call (how many queries overflowed the b16 tables)
    SearchCtrl* h_ctrl = nullptr;    // pinned, 2 blocks: [0] the sampled overflow tally, [1] the host API's read-back (read_back)
    cudaEvent_t ev_ctrl = nullptr;
    bool ctrl_pending = false;
    int ctrl_b16 = 0;
    int last_b16 = 0;                // the lane's last call used the b16 visited flavour: 1 = first segment only, 2 = both segments
    void* win_base = nullptr;        // access-policy window currently attached to the stream (see Index::attach_window)
    size_t win_bytes = 0;
    uint32_t ctrl_ef = 0;
    uint64_t ctrl_nq = 0;
    uint64_t last_nq = 0;
    uint32_t last_launches = 0;
    // the template arguments of the lane's last main K1 launch: {CH, ROW_T, EF_T, B, RowType, FULL, TMA, IDB_VARIANT taken}
    uint32_t last_kernel[8] = {};
    void free_all();
};

// The stored rows as the export, the save and the screening table read them (Index::stored, rows.cu); K1, the build and the exact scan
// read them through the row traits of hnsw_device.cuh instead.
struct StoredRows {
    const void* rows;      // cap x stride elements of `type` (bin: cap x stride / 4 bytes)
    const float2* hdr;     // q8 row headers {o, s}
    uint32_t type, stride, dim;
};
// Element e (< stride) of stored row r, exactly as f32: bf16 by the 16-bit shift; fp16 by cvt.f32.f16, except that a NaN keeps its
// sign and payload (cvt.f32.f16 would return the canonical NaN), so an export or a save gives back the f32 value of every stored
// bit pattern; q8 as fmaf(c, s, o), and 0 past dim; bin as bit e % 4 of byte e / 4 (0 in the padding).
__device__ __forceinline__ float stored_elem(const StoredRows& s, uint64_t r, uint32_t e) {
    const size_t i = r * s.stride + e;
    if (s.type == kRowF32) return static_cast<const float*>(s.rows)[i];
    if (s.type == kRowBin) return (float)((static_cast<const uint8_t*>(s.rows)[r * (s.stride / 4) + e / 4] >> (e & 3u)) & 1u);
    if (s.type == kRowQ8) {
        const float2 h = s.hdr[r];
        return e < s.dim ? __fmaf_rn((float)static_cast<const uint8_t*>(s.rows)[i], h.y, h.x) : 0.f;
    }
    const uint32_t h = static_cast<const uint16_t*>(s.rows)[i];
    if (s.type == kRowBF16) return __uint_as_float(h << 16);
    return (h & 0x7fffu) > 0x7c00u ? __uint_as_float(((h & 0x8000u) << 16) | 0x7f800000u | ((h & 0x3ffu) << 13)) : widen_f16x2(h).x;
}

// An index's adjacency (DESIGN §2, graph.cu).  Move-only; frees what it holds.
struct Graph {
    uint32_t* zero = nullptr;                  // cap x 2M (rows past n: INVALID)
    std::vector<uint32_t*> upper;              // [l-1] -> n_l x M
    std::vector<uint64_t> upper_n;             // n >= n_1 >= ... >= 1
    const uint32_t** upper_ptrs = nullptr;     // device copy of `upper` (GraphView::upper)
    bool rows_distinct = true;                 // no adjacency row lists a PointId twice (checked for adopted graphs)

    Graph() = default;
    Graph(Graph&& o) noexcept { *this = std::move(o); }
    Graph& operator=(Graph&& o) noexcept;      // swaps: o frees what this held
    ~Graph();
    // On an empty Graph: zero of `cap` rows and one layer per entry of upper_n (contents unset), and the pointer table uploaded on st.
    cudaError_t alloc(uint64_t cap, uint32_t M, std::vector<uint64_t> upper_n, cudaStream_t st);
    // Rows [r0, r0 + m) of layer l (0 = zero) into host memory on st, then synchronises st.
    cudaError_t copy_out(uint32_t l, uint64_t r0, uint64_t m, uint32_t M, uint32_t* host, cudaStream_t st) const;
    // An adopted graph of n points: every entry INVALID or inside its layer (else IDB_ERR_INVALID_ARG), then rows_distinct.
    idb_status check(uint64_t n, uint32_t M, int num_sms, cudaStream_t st);
};

struct Index {
    int device = 0;
    int num_sms = 132;
    DeviceCtx* ctx = nullptr;
    Lane lanes[kLanes];
    cudaStream_t stream = nullptr;             // = lanes[0].stream: uploads, builds, the default lane
    std::mutex mu;                             // graph-level operations (build, export, id map)
    std::atomic<uint32_t> next_lane{0};        // host-API calls rotate over the lanes
    std::atomic<int> last_lane{0};

    std::atomic<uint64_t> n{0};                // written by an insert while other threads may read it (searches take a lane first)
    uint64_t cap = 0;                          // rows allocated for points, zero and the id map (>= n; grows by doubling on insert)
    uint32_t dim = 0, nchunks = 0, M = 32, ef_search = 100;
    void* d_rows = nullptr;                    // cap x nchunks*4 elements of row_type (PointId order): f32, bf16 / fp16, q8 codes or bin bits
    float2* d_hdr = nullptr;                   // cap q8 row headers {o, s} (DESIGN §3c), else null
    uint32_t row_type = kRowF32;               // RowType = the IDB_STORAGE_* the rows are stored as; set when the index is created
    uint32_t metric = kMetricL2Sq;             // kMetricCosine: the rows are canonically normalised, and so is every query (DESIGN §3a)
    Graph graph;
    uint32_t* d_id_map = nullptr;              // shard: PointId -> global row id (idb_index_set_id_map), cap entries
    // Screening table of the stored rows (DESIGN §2, §4): n x code_words(nchunks) u32 of 8-bit codes (zero padded to a multiple of
    // 16 bytes) + 3 x nchunks float4 (scale, offset, E),
    // one code step for every element and the bound on every row's coding error (GraphView::cstep / cerr).
    // Null when screening is off (IDB_SCREEN=0), the index is empty, or a stored value is not finite.
    uint32_t* d_codes = nullptr;
    float4* d_cparams = nullptr;
    float code_step = 0.f;
    float code_err = 0.f;
    bool screen = true;                        // IDB_SCREEN (default 1): build the table and let K1 screen with it; never changes results

    // tuning knobs (env IDB_OPT / IDB_VIS_MULT / IDB_VIS_TIER / IDB_B16_BYTES / IDB_VIS_SLOTS / IDB_VARIANT); none of them changes results
    uint32_t opt_flags = 0;       // L2 prefetch of rows/vectors (experiments; off by default)
    uint32_t vis_mult = 4;        // hash flavour: slots = next_pow2(vis_mult * 2M * ef): load <= ~0.15, probe chains ~1
    uint32_t vis_slots_override = 0; // IDB_VIS_SLOTS (tests): exact hash-table size, to force the overflow -> retry path
    uint32_t b16_bytes_override = 0; // IDB_B16_BYTES (tests / sweeps): exact b16 table bytes per warp in use
    uint32_t retry_slots_override = 0; // IDB_RETRY_SLOTS (tests): hash slots of the build's and the insert's KA retry pass
    uint32_t b16_cap_16ths = 11;     // IDB_B16_CAP (tests): hand a query to the retry pass beyond this many sixteenths of the slots
    int vis_tier = -1;            // IDB_VIS_TIER: -1 auto (b16 when exact for this n, else bitmap / hash), 0 hash, 1 bitmap, 2 b16
    int variant = 0;              // IDB_VARIANT: alternative (rows in flight, CTAs/SM) instantiations of K1
    uint64_t exact_scratch_keys = 0;  // IDB_EXACT_SCRATCH_KEYS (tests): keys of an exact call's list scratch per query chunk (0 = default)
    uint32_t graph_range_scratch = 0; // IDB_GRAPH_RANGE_SCRATCH (tests): hits per query the graph range search's main pass holds (0 = default)
    // Adaptive: when more than 1 in 1000 traversals of a call overflowed the b16 tables (data whose traversals visit more ids than
    // the tables were sized for), later calls with that ef or a larger one use the DRAM-resident atomic flavours instead of paying
    // for the retry pass.  Results are identical either way.
    std::atomic<uint32_t> b16_demote_ef[2] = {{0xFFFFFFFFu}, {0xFFFFFFFFu}};  // [0] first-segment tables, [1] two-segment tables
    int b16_level = 0;            // set by select_visited_tier (under ctx->mu): which b16 size the selected tier is (0 = not b16)
    void note_overflows(uint32_t ef, uint64_t n_work, uint32_t overflowed, int level);
    bool profiling = false;

    ~Index();
    idb_status init_device(int dev);
    // The graph of an index of n rows (cap = n, graph.cu): layer sizes checked, zero and upper allocated and copied (each upper layer
    // when given), adjacency entries checked.  The rows are put in by the caller (put_rows).
    idb_status upload(uint64_t n, uint32_t dim, uint32_t M, uint32_t ef, const uint32_t* zero, uint32_t n_upper,
                      const uint32_t* const* upper, const uint64_t* upper_n);
    GraphView view() const;
    // ---- the row storage (rows.cu) ----
    StoredRows stored() const;
    // Rows [r0, r0 + m) (r0 >= n, r0 + m <= cap) of the store.  fill(dst) writes them as nchunks * 4 f32 per row, zero padded (the
    // kernel layout), into the store itself for f32 rows, else into a staging buffer.  Then the storage's refusal (fp16, q8) runs
    // over the staged rows, naming the caller's row input_row[r] when given, else r; on a refusal nothing of the store is written.
    // Then they are narrowed (bf16, fp16) or quantised (q8) into the store.  An index without a store gets one of cap rows first.
    // Returns once the rows are stored.
    idb_status put_rows(uint64_t r0, uint64_t m, const uint32_t* input_row, const std::function<cudaError_t(float*)>& fill);
    // m x dim host floats -> dst (m rows of nchunks * 4 floats on the device, zero padded), enqueued on the index's stream.
    cudaError_t copy_rows_in(float* dst, const float* src, uint64_t m) const;
    // Storage for at least `rows` points: rows, zero and the id map move to buffers of max(rows, 2 cap) rows holding the same first
    // n rows.  Everything is allocated before anything is freed, so a failure leaves the index as it was.
    idb_status reserve_rows(uint64_t rows);
    size_t row_bytes() const;                                           // bytes of one stored row
    cudaError_t alloc_rows(uint64_t rows, void** pts, float2** hdr) const;  // a store of `rows` rows (and q8 headers); frees nothing
    idb_status copy_points_f32(float* host_out, uint64_t r0, uint64_t m);  // rows [r0, r0+m) widened to m x dim f32 on the host
    // ----
    // The zero rows of rows [r0, r0 + m) INVALID, and global_ids (m entries) into the id map when it exists (the insert, after
    // put_rows; graph.cu).
    idb_status stage_rows(uint64_t r0, uint64_t m, const uint32_t* global_ids);
    idb_status build_codes();                                            // (re)builds d_codes / d_cparams from the stored rows
    int search_grid() const;
    // The visited tier of a traversal with this ef, and its launch window.  Caller holds ctx->mu.
    idb_status select_visited_tier(uint32_t ef, VisTier& tier, LaunchWindow& win);
    // The persisting-L2 window on the b16 tables rides on every launch as a launch attribute; it is ALSO kept as a stream attribute,
    // because profilers that replay a kernel (ncu) re-launch it without its launch attributes.
    idb_status attach_window(Lane& ln, const LaunchWindow& win);
    idb_status ensure_lane_scratch(Lane& ln, uint64_t nq);
    // The caller's queries (dim floats per row, in host memory when `host`, else on the device) as the rows K1 and the exact scan
    // read: nchunks * 4 floats per row, zero padded, 16-byte aligned.  Device rows already laid out so are read where they are;
    // all others are copied into ln.q in one copy.  *out: the staged rows.
    idb_status stage_queries(Lane& ln, const float* queries, bool host, uint64_t nq, const float** out);
    // A cosine index normalises the staged rows *q once per call into ln.qn and points *q there; an L2 index reads them as staged.
    idb_status normalize_queries(Lane& ln, const float** q, uint64_t nq);
    // d_queries: staged rows (stage_queries).  map_ids = false: ids and keys carry PointIds even when the index has an id map.
    idb_status enqueue_search(Lane& ln, const float* d_queries, uint64_t nq, uint32_t ef, uint32_t k, uint32_t* d_ids, float* d_dist,
                              uint32_t* d_len, uint64_t* out_keys, bool map_ids = true);
    Lane& pick_lane();
    // For the idb_last_search_* queries: under the lane's lock, what the lane's last search left behind — its control block (`ctrl`,
    // once the lane's stream has drained) and its K1 instantiation (`kernel`, 8 words) — each optional, all zero when the lane has
    // run none.  `latest`: lane 0xFFFFFFFF names the lane of the last call issued on this index.
    idb_status last_search(uint32_t lane, bool latest, SearchCtrl* ctrl, uint32_t* kernel);
};

// The index held exclusively (&mut self) by a call that changes it (insert, remove, set_id_map): its mutex, then every lane's, in
// that order, so searches on other threads wait; then the index's device is set and every lane's stream drained, so what they
// enqueued before (and reads on the device) has run.  `drained` is that step's result, for the caller to report.
struct ExclusiveIndex {
    Index* ix;
    cudaError_t drained;
    explicit ExclusiveIndex(Index* index);
    ~ExclusiveIndex();
    ExclusiveIndex(const ExclusiveIndex&) = delete;
    ExclusiveIndex& operator=(const ExclusiveIndex&) = delete;
};

// The linking parameters of an insert or a removal: ef_construction in 1..1024, and no extend_candidates with the heuristic
// (IDB_ERR_UNSUPPORTED).  kNoExtendCandidates is the refusal's message, which the build shares.
extern const char kNoExtendCandidates[];
idb_status check_link_params(const idb_params* p);

constexpr uint32_t kExactMaxK = 1024;  // the exact search's largest k

// Fails with IDB_ERR_CUDA when the runtime sees no device (this library has no CPU fallback); else sets *count if given.
idb_status require_device(int* count = nullptr);

// The argument checks of a search entry, then require_device.  What differs between the entries: `exact` refuses k = 0 even when
// nq = 0 and caps k at kExactMaxK; `lane` (optional) must name a lane, even when nq = 0; `sharded` checks comm before anything else
// and the list of n_shards handles only when nq > 0 (the others check their one handle first).  nq = 0 passes once the checks that
// apply to it have, without the device check: there is nothing to do.
// `range` (the exact and the graph range search) takes no k; out_ids stands for its offsets, and `rc` carries what else it checks.
enum class Family { approx, exact, sharded, range };
struct RangeCheck {
    float radius;
    uint64_t capacity;
    const void* ids;
    bool device;                 // the device entry, which reports the total in *out_total
    const uint64_t* out_total;
    uint32_t ef_search;          // the graph range search's seed search width: 0 (the index's) or 1..kMaxEf; 0 for the exact one
};
constexpr uint32_t kMaxEf = 1024;                    // the largest ef_search a search takes
constexpr uint64_t kRangeMaxCapacity = 0x7fffffffu;  // CUB's sorts and scans take int sizes: capacity <= this, nq + 1 <= this
idb_status check_search_args(Family f, idb_index* const* shards, uint32_t n_shards, const void* comm, const uint32_t* lane,
                             const void* queries, uint64_t nq, const void* out_ids, uint32_t k, const RangeCheck* rc = nullptr);

// Empty result lists on the stream: ids INVALID, distances +inf, lengths 0, keys kKeyNone (each output optional but ids).
cudaError_t write_empty(cudaStream_t st, uint64_t nq, uint32_t k, uint32_t* ids, float* dist, uint32_t* len, uint64_t* keys);

// One approximate search on a lane (the caller holds ln.mu) of staged queries (`staged`) or of the caller's device queries (dim
// floats per row, any alignment); empty result lists for an empty index or ef_search = 0.
idb_status search_on_lane(Index* ix, Lane& ln, const float* queries, bool staged, uint64_t nq, uint32_t ef_search, uint32_t k,
                          uint32_t* d_ids, float* d_dist, uint32_t* d_len, uint64_t* d_keys, bool map_ids = true);

// Where a range search's collector puts its hits (range.cu): counts[q] (nq, zeroed) = query q's hits; each hit as a (key, query) pair at
// a position claimed from *total (zeroed), written only below `capacity`.
struct RangeSink {
    uint32_t* counts;
    unsigned long long* total;
    uint64_t capacity;
    uint64_t* keys;
    uint32_t* qids;
};
// A range search of nq queries on the lane (the caller holds ln.mu; DESIGN §9b, §9c): collect(sink) enqueues the kernels that append the
// hits; then the offsets (the exclusive scan of the counts), the total read back, the capacity check (IDB_ERR_CAPACITY, offsets and
// total written), the gather into each query's segment, the segmented sort by key and the ids (through the id map) and reported
// distances.  Host call: offsets, ids and dist are the caller's host buffers; device call: device buffers, the total goes to
// *out_total.  Returns once the lane has run the call.
idb_status range_on_lane(Index* ix, Lane& ln, bool host, uint64_t nq, uint64_t capacity, uint64_t* offsets, uint32_t* ids, float* dist,
                         uint64_t* out_total, const std::function<idb_status(const RangeSink&)>& collect);

// The end of a host call on lane ln: copies its results (ln.ids / dist / len, nq x k) to the caller's buffers (each but out_ids
// optional), reads the control block of each of `ctrl_lanes` whose last call ran K1 into its pinned h_ctrl[1], synchronises the
// stream, and fails with IDB_ERR_CAPACITY when queries overflowed even the retry pass of those calls.
idb_status read_back(Lane& ln, uint64_t nq, uint32_t k, uint32_t* out_ids, float* out_dist, uint32_t* out_len, Lane* const* ctrl_lanes,
                     uint32_t n_ctrl);
// Device-to-host copies on ln.stream (at most 4), each into the caller's buffer `user` (skipped when null), staged through the
// lane's pinned buffer when any of them is pageable; `also` enqueues more work behind them.  Then synchronises the stream.
struct HostCopy {
    void* user;
    const void* dev;
    size_t bytes;
};
idb_status copy_to_host(Lane& ln, const HostCopy* parts, int n_parts, const std::function<cudaError_t()>& also = nullptr);

cudaError_t fill_u32(uint32_t* p, size_t n, uint32_t v, cudaStream_t st);
static_assert(kRowF32 == IDB_STORAGE_F32 && kRowBF16 == IDB_STORAGE_BF16 && kRowF16 == IDB_STORAGE_F16 && kRowQ8 == IDB_STORAGE_Q8 &&
                  kRowBin == IDB_STORAGE_BIN,
              "RowType mirrors IDB_STORAGE_*");
// The storage values an index accepts (3 and 5..7 are not among them).
inline bool storage_known(uint32_t s) { return s <= IDB_STORAGE_F16 || s == IDB_STORAGE_Q8 || s == IDB_STORAGE_BIN; }
// bin rows take the squared L2 only (DESIGN §3d: normalised rows are not 0/1): IDB_ERR_UNSUPPORTED for cosine, else IDB_OK.
idb_status check_storage_metric(uint32_t storage, uint32_t metric);
// normalize_rows_kernel: dst[r] (nchunks * 4 floats, zero padded) = the canonical normalisation of src[r] (src_stride floats per row,
// dim used, any alignment), one warp per row.  dst may equal src when src_stride == nchunks * 4.
cudaError_t normalize_rows(const float* src, uint64_t src_stride, float* dst, uint64_t n, uint32_t dim, uint32_t nchunks, int num_sms,
                           cudaStream_t st);
// K4 (merge.cu): per query, the k smallest keys of G lists of k keys (G x nq x k; all ones = empty slot), written as ids / reported
// distances / lengths, or as keys when d_keys is set.  The merge holds a query's G x k keys per warp in shared memory: merge_fits
// refuses a merge larger than the device's opt-in shared memory per block and sets *max_smem to that limit, for launch_merge.
idb_status merge_fits(const Index* ix, uint64_t lists, uint32_t k, int* max_smem);
idb_status launch_merge(Index* ix, cudaStream_t st, const uint64_t* keys, uint32_t G, uint64_t nq, uint32_t k, uint32_t* d_ids,
                        float* d_dist, uint32_t* d_len, uint64_t* d_keys, int max_smem);

// idb_index_from_graph_ex, and idb_index_load_storage with from_file (argument errors of the file's graph become IDB_ERR_FORMAT).
idb_status adopt_graph(const float* points, uint64_t n, uint32_t dim, uint32_t M, uint32_t ef_search, const uint32_t* zero,
                       uint32_t n_upper, const uint32_t* const* upper, const uint64_t* upper_n, uint32_t storage, uint32_t metric,
                       int32_t device, idb_index** out_index, bool from_file);

cudaError_t ensure_u32(uint32_t*& p, size_t& cap, size_t need);
cudaError_t ensure_u64(uint64_t*& p, size_t& cap, size_t need);
cudaError_t ensure_f32(float*& p, size_t& cap, size_t need);

}  // namespace idb
