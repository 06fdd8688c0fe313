/*
 * instant_distance_b200.h — C ABI of the H100-native HNSW build-and-search engine.
 *
 * This is the drop-in boundary for djc/instant-distance's f32-vector hot path.  Every entry point below
 * names the reference interface it replaces (file:line under the reference tree; core =
 * instant-distance/src/lib.rs, types = instant-distance/src/types.rs, py = instant-distance-py/src/lib.rs).
 * A Rust `-sys` binding, the PyO3 module, or any other FFI binds exactly these symbols (INTEGRATION.md).
 *
 * Conventions
 *   - Plain C types only; all index state lives in GPU HBM behind an opaque handle.
 *   - Host-buffer calls copy in/out; the caller keeps ownership of every buffer it passes.
 *   - Every function returns an idb_status; idb_last_error() gives the thread-local message.
 *   - There is NO CPU fallback: without a CUDA device every compute call returns IDB_ERR_CUDA.
 *   - Points are f32 vectors under squared-L2 (the reference's FloatArray metric, py:378-421), any dim >= 1,
 *     computed in one canonical fp32 summation order (DESIGN.md) so results are bit-reproducible.  The entry points without an
 *     `_ex` suffix are squared-L2 indexes; the `_ex` ones also take IDB_METRIC_COSINE (DESIGN.md §3a).
 *   - PointIds are u32; IDB_INVALID (u32::MAX) is the reference's INVALID sentinel (types:293).
 */
#ifndef INSTANT_DISTANCE_B200_H
#define INSTANT_DISTANCE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define IDB_INVALID 0xFFFFFFFFu
#define IDB_STORAGE_F32 0u
#define IDB_STORAGE_BF16 1u
/* fp16 rows (DESIGN.md §3b): rounded to nearest even, subnormals kept, +-0 / +-inf / NaN kept; 11 significant bits against bf16's 8,
 * at the same 2 bytes per element.  A finite value that would round to +-inf (|x| >= 65520) is refused with IDB_ERR_INVALID_ARG,
 * naming its row and element, before the index changes.  Widened exactly to f32 for every distance, export and save. */
#define IDB_STORAGE_F16 2u
/* q8 rows (DESIGN.md §3c): one code byte per element and a per-row grid, so a row needs no trained parameters.  With e the smallest
 * power-of-two step (down to 2^-149, and no finer than 2^(ilogb(max|x|) - 23)) for which the row spans at most 255 steps,
 * b = floor(min x / 2^e) and c_i = rint(x_i / 2^e) - b (ties to even), element i is stored as (b + c_i) 2^e, an exact f32: the
 * header {b 2^e, 2^e} and c_i in [0, 255].  Quantising a stored row again gives the same row, and every distance, export and save
 * sees the dequantised row exactly.  A row with a NaN or infinite element, or whose header or dequantised values would overflow f32,
 * is refused with IDB_ERR_INVALID_ARG, naming its row and element, before the index changes.  A q8 index has no screening table.
 * (The value 3 is not a storage.) */
#define IDB_STORAGE_Q8 4u
/* Binary rows (DESIGN.md §3d): every element is 0 or 1, kept as one bit in one byte per 4 elements (element 4c + k is bit k of byte c,
 * the high nibble zero), a sixteenth of the f32 bytes.  A row element must be +0.0, -0.0 (stored as 0) or 1.0; any other value (0.5, 2,
 * -1, NaN, +-inf, a subnormal) is refused with IDB_ERR_INVALID_ARG, naming its row and element, before the index changes.  Metric
 * IDB_METRIC_L2SQ only (IDB_METRIC_COSINE with bin: IDB_ERR_UNSUPPORTED, normalised rows are not 0/1).  Queries are any f32 rows and
 * the reported distance is the canonical squared L2 to the 0/1 row; for a 0/1 query every partial sum is a small integer, so it is
 * exactly the Hamming distance.  Packed codes (8 elements per byte, most significant bit first) become queries and rows with
 * np.unpackbits(codes, axis=1).astype(np.float32).  A bin index has no screening table.  (The values 5 to 7 are not storages.) */
#define IDB_STORAGE_BIN 8u
/* Metrics (DESIGN.md §3a).  IDB_METRIC_COSINE: every row and every query is normalised in the canonical order (x / sqrt(sum x^2),
 * correctly rounded; a row whose sum of squares overflows becomes zeros and NaN), the traversal runs the canonical squared L2 on
 * the normalised rows, and the reported distance is half of it: 1 - cos(x, y) (0 .. 2).  An all-zero row stays zero, so it is at
 * 0.5 from every other row and at 0 from another zero row.  An index stores the normalised rows (bf16 / fp16: normalised in f32,
 * then rounded) and exports / saves them. */
#define IDB_METRIC_L2SQ 0u
#define IDB_METRIC_COSINE 1u

#if defined(__GNUC__)
#define IDB_API __attribute__((visibility("default")))
#else
#define IDB_API
#endif

typedef enum idb_status {
    IDB_OK = 0,
    IDB_ERR_INVALID_ARG = 1,   /* null pointer, dim == 0, N >= u32::MAX (core:256), unsupported M / ef ... */
    IDB_ERR_OOM = 2,           /* host or device allocation failed */
    IDB_ERR_CUDA = 3,          /* no device / CUDA runtime error (message has the CUDA error string) */
    IDB_ERR_NCCL = 4,
    IDB_ERR_IO = 5,
    IDB_ERR_FORMAT = 6,        /* malformed index file */
    IDB_ERR_CAPACITY = 7,      /* an internal per-query structure overflowed even after the retry pass; or a range search
                                  found more hits than its capacity */
    IDB_ERR_UNSUPPORTED = 8
} idb_status;

/* Opaque index handle: replaces `Hnsw<P>` (core:193-199) for P = f32 vector. */
typedef struct idb_index idb_index;

/* Builder (core:23-31) + Heuristic (core:115-119).  M is a compile-time const 32 in the reference
 * (core:787); it is a run-time field here because BASELINE.json's configs name M = 16 and M = 24. */
typedef struct idb_params {
    uint32_t M;                 /* reference: const M = 32 (core:787); supported 2..64 */
    uint32_t ef_construction;   /* Builder::ef_construction (core:35-38), default 100 (core:105) */
    uint32_t ef_search;         /* Builder::ef_search       (core:44-47), default 100 (core:104) */
    float    ml;                /* Builder::ml              (core:57-60), default 1/ln(M) (core:107) */
    uint64_t seed;              /* Builder::seed            (core:65-68) */
    int32_t  heuristic;         /* Builder::select_heuristic(Some/None) (core:49-52); default Some */
    int32_t  extend_candidates; /* Heuristic::extend_candidates (core:117), default false */
    int32_t  keep_pruned;       /* Heuristic::keep_pruned       (core:118), default true  */
    uint32_t insert_batch;      /* GPU build: concurrent inserts per step (rayon's worker count in the
                                   reference, core:316-318).  0 = auto, 1 = strictly sequential order. */
    int32_t  device;            /* CUDA device ordinal */
    uint32_t storage;           /* IDB_STORAGE_F32 (default), IDB_STORAGE_BF16 or IDB_STORAGE_F16: rows rounded to bf16 / fp16 (RNE)
                                   and kept in HBM at half the bytes; IDB_STORAGE_Q8: rows quantised to a per-row 8-bit grid, a
                                   quarter of the bytes plus 8 bytes per row; IDB_STORAGE_BIN: 0/1 rows at one byte per four
                                   elements.  Distances still accumulate in fp32 in the same canonical order.  An index with no
                                   rows records it for the rows a later insert adds. */
    /* Builder::progress(ProgressBar) (core:70-75; feature `indicatif`): called on the building thread with the number of
     * points whose insertion has been enqueued so far (set_position, core:519-525) and the total (set_length, core:216-222);
     * the last call has done == total (finish, core:331-334).  NULL = no reporting. */
    void (*progress)(uint64_t done, uint64_t total, void* user);
    void*    progress_user;
} idb_params;

/* Builder::default() (core:101-113) — except `seed`, which the reference draws from entropy; here 0. */
IDB_API idb_status idb_params_default(idb_params* p);

/* Builder::build_hnsw(points) -> (Hnsw, Vec<PointId>) (core:83-85 -> Hnsw::new core:209-345).
 * rows: n x dim row-major host f32.  out_ids[i] = PointId assigned to input row i (core:262-270); may be NULL. */
IDB_API idb_status idb_build_f32(const float* rows, uint64_t n, uint32_t dim, const idb_params* params,
                         idb_index** out_index, uint32_t* out_ids);
/* Same, for an index of metric `metric` (IDB_METRIC_*); idb_build_f32 = IDB_METRIC_L2SQ.  With IDB_METRIC_COSINE the rows are
 * normalised before the build (the caller's rows are not written).  (The metric is an argument rather than an idb_params field so
 * that idb_params keeps its size: callers compiled against an earlier header allocate it themselves.) */
IDB_API idb_status idb_build_ex(const float* rows, uint64_t n, uint32_t dim, const idb_params* params, uint32_t metric,
                                idb_index** out_index, uint32_t* out_ids);

/* Insert: append m host rows (m x dim f32) to an index of n0 points, each by Construction::insert(new, 0, layers) (core:437-528):
 * a descent from the top layer with ef = 1 on the layer snapshots, ef_construction on layer 0, select_heuristic (or the simple
 * selection), then the re-pruning of every target row.
 *   - PointIds: the new points get n0 .. n0+m-1 in input order (no shuffle); out_ids[i] = n0 + i (may be NULL).
 *   - Layer 0 only.  Layer l holds exactly PointIds [0, n_l) (core:275-281), so a new point could enter an upper layer only by
 *     renumbering existing ones, which this call does not do.  The upper layers, their snapshots and ef_search do not change: they
 *     stay a sample of the first n0 points, so navigation can degrade as m / n0 grows (DESIGN.md §6a: no recall loss measured up to
 *     m = n0 on sift-shaped rows).
 *   - Batches: the build's layer-0 schedule from g0 = n0, b = min(max_batch, max(1, g0 / growth)) with max_batch / growth from
 *     insert_batch (1 = the sequential reference order), else IDB_BUILD_MAXBATCH / IDB_BUILD_GROWTH (defaults 16384 / 8).  Unlike
 *     the build, an index with no upper layer is also inserted into in batches.  An empty index (n0 = 0) makes the first row its
 *     entry point, PointId 0.
 *   - Rows are stored as the build stores them: zero padded, normalised for a cosine index, then narrowed for a bf16 / fp16 one.
 *     An fp16 index refuses rows with a finite value that rounds to infinity (IDB_ERR_INVALID_ARG, naming the row i of `rows` and
 *     the element); the index's rows, graph and n stay as they were.
 *   - params: ef_construction (1..1024), heuristic, keep_pruned, insert_batch and progress (called with the rows inserted so far
 *     and m) are read; M must equal the index's M; extend_candidates is refused as by the build; seed, ml, ef_search, storage and
 *     device are ignored.  dim must equal the index's dim; n0 + m >= u32::MAX is refused (core:256); m = 0 does nothing.
 *   - global_ids (m entries): required when the index has an id map (idb_index_set_id_map), refused when it has none; appended to
 *     the map, so a shard keeps reporting global ids.
 *   - Exclusive (&mut self): searches on other threads wait until the insert has finished and see the index before or after it.
 *   - Failures: an argument error, a failed allocation or a CUDA error before the first batch leaves the index as it was.
 *     IDB_ERR_CAPACITY (an insert overflowed even the retry pass, e.g. in a cluster of thousands of identical rows): the index keeps
 *     the batches before the failing one — n is then that batch's first PointId — and stays searchable.  The traversals see
 *     n = n0 + m for the whole call.
 *   - Storage doubles when it grows, so repeated small inserts are not quadratic.  The screening table is rebuilt from all rows. */
IDB_API idb_status idb_index_insert_f32(idb_index* index, const float* rows, uint64_t m, uint32_t dim, const idb_params* params,
                                        const uint32_t* global_ids, uint32_t* out_ids);

/* Remove: take the m points pids[0..m) out of an index of n points (DESIGN.md §6b).
 *   - Repair: on every layer, each surviving row that lists a removed id is selected again.  Its candidates are its own entries
 *     and the entries of the row of each removed id it lists (one hop: removed ids in those rows are dropped, not followed), without
 *     the point itself and without removed ids.  The ef_construction nearest of them, by (distance, PointId), go through
 *     select_heuristic (core:636-698) with keep_pruned and the 2M cap, or in simple mode the first 2M are taken; an upper row keeps
 *     the first M (UpperNode::from_zero, types:65-71).  A row that lists no removed id is not touched.  An entry is any value other
 *     than INVALID.
 *   - Compaction, in order: new(x) = x - |{r in pids : r < x}|.  Every entry, the rows, the id map and the layer sizes follow:
 *     n' = n - m, n_l' = |[0, n_l) minus pids|, and the upper layers left with no point are dropped.  Layer l still holds
 *     [0, n_l'), and the entry point is the lowest surviving PointId.  out_new_ids (n entries, may be NULL) receives new(x), or
 *     INVALID for a removed point.
 *   - params: ef_construction (1..1024), heuristic and keep_pruned are read; M must equal the index's M; extend_candidates is
 *     refused as by the build; everything else is ignored.  A pid >= n or a repeated pid is IDB_ERR_INVALID_ARG, naming its position
 *     in pids.  m = 0 does nothing; m = n leaves an empty index of the same dim, storage and metric, which a later insert fills as
 *     it fills any empty index.
 *   - Exclusive (&mut self): searches on other threads wait until the removal has finished and see the index before or after it.
 *   - Failures: an argument error or a failed allocation leaves the index as it was (every buffer, the compacted storage included,
 *     is allocated before the first row is written, so the call needs room for a second copy of the index while it runs).
 *   - Known limits: a surviving point whose only in-links came from removed points can become unreachable; a row whose candidates
 *     were all removed ends up empty; the upper layers are not refilled from below.  The screening table is rebuilt from the rows
 *     that remain. */
IDB_API idb_status idb_index_remove(idb_index* index, const uint32_t* pids, uint64_t m, const idb_params* params,
                                    uint32_t* out_new_ids);

/* "Search a given graph": adopt a graph built elsewhere (the reference, the oracle, a loaded .idx file).
 * This is the parity entry point.  Mirrors the fields of `Hnsw` (core:194-199):
 *   points   n x dim, PointId order                       (Hnsw::points)
 *   zero     n x 2M u32, INVALID-terminated rows          (Hnsw::zero, ZeroNode types:83-85)
 *   upper[l] upper_n[l] x M u32 for layer l+1             (Hnsw::layers, UpperNode types:63) */
IDB_API idb_status idb_index_from_graph_f32(const float* points, uint64_t n, uint32_t dim, uint32_t M, uint32_t ef_search,
                                    const uint32_t* zero, uint32_t n_upper, const uint32_t* const* upper,
                                    const uint64_t* upper_n, int32_t device, idb_index** out_index);

/* Same, but the point rows are rounded to bf16 and stored that way (BASELINE config 4's data format).  Results equal the f32
 * engine / the reference algorithm run on the bf16-rounded points. */
IDB_API idb_status idb_index_from_graph_bf16(const float* points, uint64_t n, uint32_t dim, uint32_t M, uint32_t ef_search,
                                     const uint32_t* zero, uint32_t n_upper, const uint32_t* const* upper,
                                     const uint64_t* upper_n, int32_t device, idb_index** out_index);

/* Both of the above and the metric: storage = IDB_STORAGE_* (IDB_STORAGE_F16: the rows rounded to fp16, IDB_STORAGE_Q8: the rows
 * quantised, IDB_STORAGE_BIN: 0/1 rows, refused with IDB_METRIC_COSINE as IDB_ERR_UNSUPPORTED; results equal the reference
 * algorithm run on the rounded or dequantised points), metric = IDB_METRIC_*.  With IDB_METRIC_COSINE the points are taken as given
 * (normalising is not idempotent bit for bit, so an adopted graph keeps the exact rows it was built on): every row must be all zeros
 * or have |sum x^2 - 1| <= 1e-2 (which lets bf16- and fp16-rounded and q8-quantised unit rows through), else IDB_ERR_INVALID_ARG.
 * idb_normalize_f32 gives the canonical normalisation. */
IDB_API idb_status idb_index_from_graph_ex(const float* points, uint64_t n, uint32_t dim, uint32_t M, uint32_t ef_search,
                                           const uint32_t* zero, uint32_t n_upper, const uint32_t* const* upper,
                                           const uint64_t* upper_n, uint32_t storage, uint32_t metric, int32_t device,
                                           idb_index** out_index);

/* The canonical normalisation of n rows of dim f32 (DESIGN.md §3a) on the device: out (n x dim, host) = what a cosine index
 * stores for `rows` (before any bf16 / fp16 rounding).  For callers preparing rows for idb_index_from_graph_ex, and for parity tests. */
IDB_API idb_status idb_normalize_f32(const float* rows, uint64_t n, uint32_t dim, int32_t device, float* out);

/* Hnsw::search(point, &mut Search) (core:352-383), batched: one independent search per query row.
 * The reference returns the whole `nearest` list (<= ef_search items, ascending by (distance, pid));
 * callers take the first k.  Here: out_ids/out_dist are nq x k (row q holds the first min(len,k) items,
 * padded with IDB_INVALID / +inf), out_len[q] = len(nearest) (what `ExactSizeIterator::len` reports).
 * ef_search == 0 uses the index's own ef_search (Hnsw::ef_search, core:195).  out_dist / out_len may be NULL.
 * Thread safety: `Hnsw<P>: Sync` (core:352-356) — any number of host threads may call this on one index at once; each call
 * takes an idle submission lane (own CUDA stream and control state, idb_index_num_lanes() of them) so concurrent callers overlap on
 * the device.  Buffers may be pageable or pinned (idb_host_alloc); results for pageable output buffers are staged through pinned
 * memory inside the library, so one caller's read-back never stalls another caller's launches.
 * The per-warp visited tables of the traversal kernels live in a per-device pool shared by every index and are cached in L2 like any
 * other data.  idb_device_set_persisting_l2(device, 1) (or IDB_L2_PERSIST=1) makes the first search/build on a device reserve part
 * of the device's persisting-L2 set-aside for them (cudaLimitPersistingL2CacheSize, at most the device maximum), with an access-policy
 * window on every launch; results are identical, and on an H100 throughput is lower, because the set-aside takes most of the L2 away
 * from the graph.  The reservation is returned when the last index on the device is freed. */
IDB_API idb_status idb_search_batch_f32(idb_index* index, const float* queries, uint64_t nq, uint32_t ef_search, uint32_t k,
                                uint32_t* out_ids, float* out_dist, uint32_t* out_len);

/* Same, with queries and outputs already resident in HBM (device pointers, same device as the index;
 * d_queries is nq x dim row-major).  Enqueues on idb_index_stream(index) (= lane 0) and returns without syncing.
 * A query that overflows an internal per-query structure even in the retry pass gets out_len = 0 and IDB_INVALID ids;
 * idb_last_search_failures() reports how many did (the host-buffer call returns IDB_ERR_CAPACITY instead). */
IDB_API idb_status idb_search_batch_device(idb_index* index, const float* d_queries, uint64_t nq, uint32_t ef_search, uint32_t k,
                                   uint32_t* d_out_ids, float* d_out_dist, uint32_t* d_out_len);
/* The same on submission lane `lane` < idb_index_num_lanes(): calls on one lane are stream-ordered (idb_index_lane_stream), calls
 * on different lanes overlap — the next batch's thread blocks move in as the previous batch's drain, so back-to-back batches
 * issued alternately on two lanes keep the GPU full across batch boundaries. */
IDB_API idb_status idb_search_batch_device_lane(idb_index* index, uint32_t lane, const float* d_queries, uint64_t nq, uint32_t ef_search,
                                        uint32_t k, uint32_t* d_out_ids, float* d_out_dist, uint32_t* d_out_len);

/* Exact k-NN: for each query, the min(k, n) smallest (canonical distance, PointId) over ALL stored rows, in the index's metric and
 * row type; same output layout, padding, id map and distance reporting as idb_search_batch_f32.  1 <= k <= 1024.
 * Takes an idle submission lane, like idb_search_batch_f32 (any number of host threads, alongside approximate searches).
 * Ties are broken by the lower PointId and NaN distances order last, so the answer is unique and bit-reproducible: the ground truth
 * to measure an approximate search's recall against (DESIGN.md §9a).  Exact calls leave the approximate-search diagnostics
 * (idb_last_search_counters / _failures / _retried / _full_fetches / _kernel, idb_index_last_kernel_ms) describing the last
 * approximate search.  Null index / queries (nq > 0) / out_ids or k == 0: IDB_ERR_INVALID_ARG; k > 1024: IDB_ERR_UNSUPPORTED;
 * nq == 0: IDB_OK, nothing written. */
IDB_API idb_status idb_exact_search_batch_f32(idb_index* index, const float* queries, uint64_t nq, uint32_t k,
                                              uint32_t* out_ids, float* out_dist, uint32_t* out_len);
/* Same, device pointers on the index's device (d_queries: nq x dim at any alignment), enqueued on submission lane `lane` without
 * syncing (lane >= idb_index_num_lanes(): IDB_ERR_INVALID_ARG). */
IDB_API idb_status idb_exact_search_batch_device_lane(idb_index* index, uint32_t lane, const float* d_queries, uint64_t nq,
                                                      uint32_t k, uint32_t* d_out_ids, float* d_out_dist, uint32_t* d_out_len);

/* Exact range search (DESIGN.md §9b): every stored point within `radius` of each query.  Query q's hits are every PointId p whose
 * reported distance (squared L2, or 1 - cos for a cosine index, as the exact search reports it) is <= radius, in the exact search's
 * order (distance, then PointId; ids through the id map after ordering): a prefix of the query's full exact ordering.  A point at
 * exactly `radius` is a hit (radius = 0 finds exact duplicates), a NaN distance never is, radius = +inf finds every point whose
 * distance is not NaN, and a negative radius finds none.
 * The output is CSR: query q's hits are out_ids[out_offsets[q] .. out_offsets[q + 1]) (out_offsets: nq + 1 entries,
 * out_offsets[nq] = the total), with their distances at the same positions of out_dist (optional).  `capacity` is how many hits
 * out_ids / out_dist hold, and the size of the call's device scratch (20 bytes per hit).  When the total exceeds it the call returns
 * IDB_ERR_CAPACITY with out_offsets written and nothing else, so a caller can allocate exactly and call again; capacity = 0 is a
 * counting call.  The rows are scanned once per call.  capacity <= 2^31 - 1 and nq < 2^31 - 1 (IDB_ERR_UNSUPPORTED beyond:
 * the library's sort and scan take int sizes).  Takes an idle submission lane, like the exact search, and leaves the approximate-search
 * diagnostics as they are.  Null index / queries or out_offsets (nq > 0) / out_ids (capacity > 0), or a NaN radius:
 * IDB_ERR_INVALID_ARG.  nq == 0: IDB_OK, out_offsets[0] = 0 (when given). */
IDB_API idb_status idb_range_search_batch_f32(idb_index* index, const float* queries, uint64_t nq, float radius, uint64_t capacity,
                                              uint64_t* out_offsets, uint32_t* out_ids, float* out_dist);
/* Same, device pointers on the index's device (d_queries: nq x dim at any alignment; d_out_offsets 8-byte aligned), on submission
 * lane `lane` (>= idb_index_num_lanes(): IDB_ERR_INVALID_ARG, even at nq = 0).  The total goes to the HOST word *out_total (null:
 * IDB_ERR_INVALID_ARG), also with IDB_ERR_CAPACITY.  Unlike the other device entries this one returns only after the lane has run
 * the call: the hits are ordered by a sort whose size is the total, which the host has to know first.  nq == 0: IDB_OK,
 * *out_total = 0, nothing written on the device. */
IDB_API idb_status idb_range_search_batch_device_lane(idb_index* index, uint32_t lane, const float* d_queries, uint64_t nq,
                                                      float radius, uint64_t capacity, uint64_t* d_out_offsets,
                                                      uint32_t* d_out_ids, float* d_out_dist, uint64_t* out_total);

/* Graph range search (DESIGN.md §9c): the points within `radius` of each query that layer 0 reaches from the query's approximate
 * nearest neighbours, at a cost that follows the hits rather than the number of points.  The result may miss points the exact range
 * search finds, but it is a deterministic set:
 *   seeds: nearest(q) is what idb_search_batch_f32(index, q, 1, ef_search, k = ef) returns (PointIds before the id map), and the
 *     seeds are its members whose reported distance is <= radius;
 *   closure: the smallest set H(q) that holds the seeds and, with every point p, every layer-0 neighbour x of p (the entries of p's
 *     layer-0 row up to its first IDB_INVALID) whose reported distance is <= radius.
 * H(q) is a subset of the exact range search's result with the same distances, so its hits are a subsequence of that result.  The
 * radius edges, the order (distance, then PointId; ids through the id map after ordering), the CSR output, `capacity`, the counting
 * call, IDB_ERR_CAPACITY with out_offsets written, the size limits and the argument errors are those of idb_range_search_batch_f32.
 * ef_search: 0 = the index's, else 1..1024 (else IDB_ERR_INVALID_ARG).  The seed search is an approximate search and updates the
 * approximate-search diagnostics as one at the same ef_search would.  A query whose seed search overflowed even its retry pass makes
 * the call return IDB_ERR_CAPACITY with idb_last_search_failures(index, lane) > 0 (the results of the other queries are written
 * when the total fits).  The expansion itself never gives up on a query: the queries that overflow its per-query scratch are run
 * again with scratch for every point (up to 2 GB per call); only a failed allocation is an error (IDB_ERR_OOM).  Takes an idle
 * submission lane.  nq == 0: IDB_OK, out_offsets[0] = 0 (when given). */
IDB_API idb_status idb_graph_range_search_batch_f32(idb_index* index, const float* queries, uint64_t nq, uint32_t ef_search, float radius,
                                                    uint64_t capacity, uint64_t* out_offsets, uint32_t* out_ids, float* out_dist);
/* Same, device pointers, on submission lane `lane`, with the total in the HOST word *out_total: as idb_range_search_batch_device_lane,
 * it returns only after the lane has run the call. */
IDB_API idb_status idb_graph_range_search_batch_device_lane(idb_index* index, uint32_t lane, const float* d_queries, uint64_t nq,
                                                            uint32_t ef_search, float radius, uint64_t capacity,
                                                            uint64_t* d_out_offsets, uint32_t* d_out_ids, float* d_out_dist,
                                                            uint64_t* out_total);

IDB_API uint32_t idb_index_num_lanes(void);
IDB_API void* idb_index_lane_stream(idb_index* index, uint32_t lane);  /* cudaStream_t of that lane */
/* Waits for the last call on `lane` and reports how many of its queries failed even in the retry pass (0 = all results valid). */
IDB_API idb_status idb_last_search_failures(idb_index* index, uint32_t lane, uint32_t* out_failed);
/* Diagnostics: how many queries of the last call on `lane` overflowed their per-warp visited table / tie list in the main pass and were
 * re-run by the retry pass (their results are valid; a persistently non-zero figure costs throughput, and the library then switches the
 * index to its larger, DRAM-resident visited flavour by itself).  lane = 0xFFFFFFFF: the lane the last call on this index used. */
IDB_API idb_status idb_last_search_retried(idb_index* index, uint32_t lane, uint32_t* out_retried);
/* Diagnostics: how many candidate rows the last call on `lane` fetched in full, over all its queries (and its retry pass).  Without
 * screening that is the sum of the per-query distance counters; with it (the default, DESIGN §4) the rows whose 8-bit-code lower bound
 * already proves they would not be admitted are not fetched, so it is smaller.  Results are the same either way.
 * lane = 0xFFFFFFFF: the lane the last call on this index used. */
IDB_API idb_status idb_last_search_full_fetches(idb_index* index, uint32_t lane, uint64_t* out_rows);
/* Diagnostics: which instantiation of the search kernel the last call on `lane` launched (its main pass; the retry pass uses the same
 * one).  out (8 u32) = {CH (float4 chunks per lane of a row, 0 = the long-row kernel), ROW_T, EF_T, B (rows in flight per lane), the
 * row type (IDB_STORAGE_*: 0 f32, 1 bf16, 2 fp16, 4 q8, 8 bin), 1 if FULL (no chunk predicates), 1 if TMA, the IDB_VARIANT case taken (0 = the
 * default dispatch; the variants exist for f32 rows only)}; all zeros when the last call launched no kernel.  lane = 0xFFFFFFFF: the lane the last call on this index used. */
IDB_API idb_status idb_last_search_kernel(idb_index* index, uint32_t lane, uint32_t* out);
/* enabled = 1: reserve persisting L2 for the visited tables on `device` (see idb_search_batch_f32).  enabled = 0 (the default):
 * this library never touches the device's persisting-L2 limit nor attaches access-policy windows on `device`. */
IDB_API idb_status idb_device_set_persisting_l2(int32_t device, int32_t enabled);

/* Per-query traversal counters of the LAST search call issued on this index (whichever lane it used; for the roofline accounting,
 * SURVEY §8d): out is nq x 4 u64 = {n_expand_upper, n_dist_upper, n_expand_zero, n_dist_zero}. */
IDB_API idb_status idb_last_search_counters(idb_index* index, uint64_t nq, uint64_t* out);

/* Introspection: Hnsw::iter / Index<PointId> (core:386-391, types:269-275) and the graph itself. */
typedef struct idb_info {
    uint64_t n;
    uint32_t dim;
    uint32_t M;
    uint32_t ef_search;
    uint32_t n_layers;          /* 0 for an empty index, else 1 + number of upper layers */
    uint64_t layer_n[32];       /* node count per layer, [0] = n */
    int32_t  device;
    uint32_t storage;           /* IDB_STORAGE_* */
} idb_info;
IDB_API idb_status idb_index_info(const idb_index* index, idb_info* out);
/* The index's IDB_METRIC_* (a separate call, so that idb_info keeps its size). */
IDB_API idb_status idb_index_metric(const idb_index* index, uint32_t* out_metric);
IDB_API idb_status idb_index_export_points(const idb_index* index, float* out /* n x dim */);
IDB_API idb_status idb_index_export_zero(const idb_index* index, uint32_t* out /* n x 2M */);
IDB_API idb_status idb_index_export_upper(const idb_index* index, uint32_t layer /* 1-based */, uint32_t* out /* n_l x M */);

/* Hnsw::dump / Hnsw::load of the Python binding (py:121-137): bincode-1.3 layout of `Hnsw{ef_search, points, zero, layers}`
 * (core:193-199).  dim and M are not stored in the file (fixed-size arrays in the reference: dim = 300, M = 32), so load takes
 * them.  *out_values_offset (may be NULL) = file offset where an HnswMap's `values` begin (core:131-134), or the file size. */
IDB_API idb_status idb_index_save(const idb_index* index, const char* path);
IDB_API idb_status idb_index_load(const char* path, uint32_t dim, uint32_t M, int32_t device, idb_index** out_index, uint64_t* out_values_offset);
/* Same, as an index of metric `metric`; idb_index_load = IDB_METRIC_L2SQ.  The file format does not change and does not record the
 * metric: a cosine index saves its normalised rows, and loading them as cosine takes them as given (rows that are neither unit
 * length nor all zeros: IDB_ERR_FORMAT). */
IDB_API idb_status idb_index_load_ex(const char* path, uint32_t dim, uint32_t M, uint32_t metric, int32_t device, idb_index** out_index,
                                     uint64_t* out_values_offset);
/* Same, stored as `storage` (IDB_STORAGE_*); idb_index_load_ex = IDB_STORAGE_F32.  The file always holds f32 rows (a bf16, fp16 or
 * q8 index saves its rows widened or dequantised, exactly), so saving an index and loading it with its own storage gives back the
 * same rows (q8: the same codes and headers).  Unknown storage: IDB_ERR_INVALID_ARG; IDB_STORAGE_F16 and a row value that rounds to
 * infinity in fp16, or IDB_STORAGE_Q8 and a row q8 refuses, or IDB_STORAGE_BIN and a row element other than 0 or 1:
 * IDB_ERR_INVALID_ARG; IDB_STORAGE_BIN with IDB_METRIC_COSINE: IDB_ERR_UNSUPPORTED. */
IDB_API idb_status idb_index_load_storage(const char* path, uint32_t dim, uint32_t M, uint32_t metric, uint32_t storage, int32_t device,
                                          idb_index** out_index, uint64_t* out_values_offset);

/* Measurement hooks (bench.py): when enabled, CUDA events are recorded on the index stream immediately around the
 * dominant kernel of each call (K1 search_layer for searches); idb_index_last_kernel_ms waits for that kernel and
 * returns its duration and how many of this library's kernels the last call launched. */
IDB_API idb_status idb_index_set_profiling(idb_index* index, int32_t enabled);
IDB_API idb_status idb_index_last_kernel_ms(idb_index* index, float* out_ms, uint32_t* out_launches);

/* Measurement only: random point-row gathers in K1's launch shape and arithmetic (no visited set / adjacency / merge), to show
 * the gather ceiling of the device next to K1's own rate.  chain = independent 16-row batches between two dependent steps
 * (0 = all independent).  *out_bytes = bytes gathered per run. */
IDB_API idb_status idb_debug_gather_bench(idb_index* index, uint32_t n_items, uint32_t batches, uint32_t chain, uint32_t reps,
                                          float* out_ms, double* out_bytes);
/* Same with K1's second memory stream riding along: `atomics_per_batch` visited-style atomicAnd per 16-row batch on a per-warp
 * n-bit bitmap that is wiped after every item.  mode 1: atomics overlap the row loads (traffic-mix ceiling); mode 2: the row loads
 * wait for them (K1's dependency).  *out_bytes counts the ROW bytes only, like K1's algorithmic bytes. */
IDB_API idb_status idb_debug_gather_mix_bench(idb_index* index, uint32_t n_items, uint32_t batches, uint32_t chain, uint32_t reps,
                                              uint32_t atomics_per_batch, uint32_t mode, float* out_ms, double* out_bytes);
/* Measurement / test only: for each pair (query index, PointId) of `pairs` (npairs x 2), the screening bound K1 compares with the
 * furthest distance and the canonical distance (queries: nq x dim f32, used as given).  IDB_ERR_UNSUPPORTED when the index has no
 * screening table (IDB_SCREEN=0, an empty index, a non-finite stored value, or rows of more than 1024 elements). */
IDB_API idb_status idb_debug_screen_bound(idb_index* index, const float* queries, uint64_t nq, const uint32_t* pairs, uint64_t npairs,
                                          float* out_bound, float* out_dist);
/* Test only: the sharded search's merge kernel, with the same launch, on keys (G x nq x k u64, host) the caller supplies: per query, the
 * k smallest keys of its G lists (keys unique within a query; a slot of all ones is empty).  out_keys != NULL: the merged keys
 * (nq x k, padded with all ones), as a rank's pre-merge writes them; otherwise out_ids / out_dist (nq x k, the low 32 bits of each key
 * and its distance bits reported in the index's metric, padded with IDB_INVALID / +inf) and out_len (nq); out_dist / out_len may be
 * NULL.  IDB_ERR_UNSUPPORTED when G x k keys do not fit the device's opt-in shared memory per block, like the sharded search. */
IDB_API idb_status idb_debug_merge_topk(idb_index* index, const uint64_t* keys, uint32_t G, uint64_t nq, uint32_t k, uint32_t* out_ids,
                                        float* out_dist, uint32_t* out_len, uint64_t* out_keys);

IDB_API void* idb_index_stream(idb_index* index);      /* lane 0's cudaStream_t: builds, uploads and idb_search_batch_device run on it */
IDB_API idb_status idb_index_sync(idb_index* index);   /* cudaStreamSynchronize on every lane of the index */
IDB_API void idb_index_free(idb_index* index);         /* Drop for Hnsw */

/* ---- Index sharded by PointId range across the GPUs of one box (one process per GPU) ------------------------------
 * The reference has no distributed path; this is north_star's layout: every rank owns an independent index over its
 * contiguous range of the input rows, every query is searched on every shard, and ONE ncclAllGather of the per-shard
 * top-k (packed (distance, global id) keys) is followed by a merge kernel.  Results: the k smallest (distance, global id)
 * of the union of the shards' `nearest` lists; identical on every rank.
 * Metric: the shards of one call must share one metric (else IDB_ERR_INVALID_ARG).  Across ranks that cannot be checked without
 * another collective, so it is the caller's contract: every rank's shards must have the same metric. */
#define IDB_UNIQUE_ID_BYTES 128
typedef struct idb_comm idb_comm;
IDB_API idb_status idb_comm_unique_id(void* out_unique_id /* IDB_UNIQUE_ID_BYTES, made on one rank, shared by the host app */);
IDB_API idb_status idb_comm_create(const void* unique_id, int32_t rank, int32_t world, int32_t device, idb_comm** out);
IDB_API void idb_comm_free(idb_comm* comm);
/* global_ids[pid] = the caller's id of the row that became PointId pid on this shard (NULL clears the map).
 * Exclusive (&mut self): searches on other threads wait for it and see the map before or after it. */
IDB_API idb_status idb_index_set_id_map(idb_index* index, const uint32_t* global_ids);
/* Collective over `comm`: every rank passes the same queries.  out_ids are GLOBAL ids. */
IDB_API idb_status idb_sharded_search_batch_f32(idb_index* shard, idb_comm* comm, const float* queries, uint64_t nq, uint32_t ef_search,
                                        uint32_t k, uint32_t* out_ids, float* out_dist, uint32_t* out_len);
IDB_API idb_status idb_sharded_search_batch_device(idb_index* shard, idb_comm* comm, const float* d_queries, uint64_t nq,
                                           uint32_t ef_search, uint32_t k, uint32_t* d_out_ids, float* d_out_dist, uint32_t* d_out_len);
/* The same for a rank that holds SEVERAL shards on its device (e.g. 8 PointId ranges over 2 or 4 GPUs, or all 8 on one GPU: the
 * denominator of the 1 -> 8 GPU scaling figure).  The rank's shards are searched concurrently (one launch each, overlapping on the
 * device), their top-k lists pre-merged on the device, and the rank still contributes ONE k-list per query to the ONE all-gather. */
IDB_API idb_status idb_sharded_search_batch_f32_multi(idb_index* const* shards, uint32_t n_shards, idb_comm* comm, const float* queries,
                                              uint64_t nq, uint32_t ef_search, uint32_t k, uint32_t* out_ids, float* out_dist,
                                              uint32_t* out_len);
IDB_API idb_status idb_sharded_search_batch_device_multi(idb_index* const* shards, uint32_t n_shards, idb_comm* comm,
                                                 const float* d_queries, uint64_t nq, uint32_t ef_search, uint32_t k,
                                                 uint32_t* d_out_ids, float* d_out_dist, uint32_t* d_out_len);

/* The canonical squared-L2 of one pair, evaluated on the device (used by parity tests; FloatArray::distance, py:378-421). */
IDB_API idb_status idb_distance_f32(const float* a, const float* b, uint32_t dim, int32_t device, float* out);

/* Pinned host memory helpers for callers that want true async H2D/D2H. */
IDB_API idb_status idb_host_alloc(size_t bytes, void** out);
IDB_API void idb_host_free(void* p);

IDB_API const char* idb_last_error(void);
IDB_API const char* idb_version(void);
IDB_API int32_t idb_device_count(void);

#ifdef __cplusplus
}
#endif
#endif /* INSTANT_DISTANCE_B200_H */
