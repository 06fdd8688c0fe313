// build_kernels.cuh — construction-side kernels of Builder::build (instant-distance/src/lib.rs:209-345, 437-528).
//
//   KA  insert_search_kernel   Construction::insert's descent (lib.rs:443-463): one warp per concurrent insert runs the
//                              same `descend` as queries, with q = points[new], target = the insert layer, ef = ef_construction.
//   K2  select_new_kernel      Search::select_heuristic (Alg. 4, lib.rs:636-698) for every new node of the batch; writes the
//                              node's own row (ZeroNode::set, types.rs:115-117) and emits (neighbour <- new) link requests.
//   K2' relink_kernel          Search::add_neighbor_heuristic (lib.rs:616-631) + ZeroNode::rewrite (types.rs:88-98): one warp per
//                              distinct neighbour row that received link requests in this batch.
//   K5  snapshot_kernel        UpperNode::from_zero (types.rs:65-71) for a finished layer.
//   K6  gather_rows_kernel     the shuffled clone of the points (lib.rs:263-270).
//
// Concurrency model (replaces rayon + per-row RwLocks, lib.rs:316-318, 438, 494-496): inserts are processed in batches;
// within a batch every insert searches the graph as it stood when the batch began, then all link requests are grouped by
// target row (radix sort) and each target row is re-pruned once, by one warp, with all of its new candidates.  With
// batch = 1 this is exactly the reference's sequential order; for any batch schedule the result is deterministic.
#pragma once
#include "search_kernel.cuh"

namespace idb {

constexpr int kBuildWarps = 2;          // warps per CTA in the K2 kernels (each stages up to 2M rows in shared memory)
constexpr int kNewCap = 32;             // link requests folded into one re-prune of a row (more: several rounds)

struct BuildArgs {
    GraphView g;
    uint32_t* zero;                 // writable alias of g.zero
    uint32_t base;                  // first PointId of this batch
    uint32_t count;                 // inserts in this batch
    uint32_t layer;                 // insert layer (lib.rs:437)
    uint32_t efc;                   // ef_construction
    uint32_t cand_cap;              // keys per insert in cand_keys
    uint32_t keep_pruned;           // Heuristic::keep_pruned (lib.rs:118)
    uint64_t* cand_keys;            // count x cand_cap : `nearest` of each insert, ascending
    uint32_t* cand_cnt;             // count
    uint64_t* pairs;                // count x 2M : (target << 32 | new), kKeyNone when unused
    TraversalWork work;             // KA: the batch's inserts (n_work = count); K2', simple relink: work_counter only
    VisTier tier;                   // KA
    // relink
    const uint64_t* sorted_pairs;   // count*2M sorted ascending
    uint32_t n_pairs_cap;
    const uint32_t* seg_start;      // indices into sorted_pairs where a new target begins
    const uint32_t* n_seg;          // device counter
};

// ---------------------------------------------------------------------------------------------------------
// Warp-level Search::select_heuristic (lib.rs:636-698), extend_candidates = false.
//   cand[0..W)   candidate keys, ascending by (distance to the owner, pid)         (shared memory)
//   out[0..)     resulting row: kept candidates ascending, then (keep_pruned) the pruned ones ascending, capped at 2M
// A candidate is kept iff no already-kept r has  d(candidate, r) < d(owner, candidate)  (strict, lib.rs:676-679).
// Kept rows are staged in shared memory (kStage) so each is fetched from HBM/L2 once; the candidate's own row is the
// register-resident "query" of the canonical distance.
// ---------------------------------------------------------------------------------------------------------
template <int CH, int NB, bool kStage, class RT>
__device__ __forceinline__ uint32_t select_heuristic_warp(const GraphView& g, const uint64_t* cand, uint32_t W, uint32_t* out,
                                                          uint32_t* disc, float4* kept_vecs, uint32_t* kept_pid,
                                                          bool keep_pruned, int lane, QVec<CH>& q, uint64_t* key_scratch) {
    const uint32_t cap = 2 * g.M;
    // warm L2 with every candidate row (each is read once as a "query", kept ones again when not staged)
    {
        const uint32_t rb = g.nchunks * RT::kChunkBytes, lines = (rb + 127) / 128;
        for (uint32_t ln = 0; ln < lines; ++ln)
            for (uint32_t c = lane; c < W; c += 32) prefetch_l2(g.points + (size_t)key_pid(cand[c]) * rb + ln * 128u);
    }
    uint32_t kept = 0, nd = 0;
    bool cok[CH > 0 ? CH : 1];
#pragma unroll
    for (int j = 0; j < (CH > 0 ? CH : 1); ++j) cok[j] = (uint32_t)(lane + 32 * j) < g.nchunks;
    const uint32_t row_bytes = g.nchunks * RT::kChunkBytes;   // global rows (f32, bf16, fp16, q8 or bin)
    const uint32_t srow_bytes = g.nchunks * 16u;               // staged rows are always widened float4
    const char* gbase = g.points + lane * RT::kChunkBytes;
    const char* sbase = reinterpret_cast<const char*>(kept_vecs) + lane * 16;
    for (uint32_t i = 0; i < W; ++i) {
        if (kept >= cap) break;  // lib.rs:669
        const uint64_t ck = cand[i];
        const uint32_t cpid = key_pid(ck), cbits = key_dbits(ck);
        q_from_point<CH, RT>(q, g, cpid, lane);  // the candidate is the "query" of the distances below
        bool closer = false;
        if constexpr (CH == 0) {
#pragma unroll 1
            for (uint32_t b0 = 0; b0 < kept && !closer; b0 += kLongRowsInFlight) {
                const uint32_t nb = min(kept - b0, (uint32_t)kLongRowsInFlight);
                batch_distances_long<kLongRowsInFlight, RT>(g, q, kept_pid + b0, key_scratch, nb, lane);
                closer = __any_sync(kFullMask, (uint32_t)lane < nb && key_dbits(key_scratch[lane < kLongRowsInFlight ? lane : 0]) < cbits);
                __syncwarp();
            }
        } else {
#pragma unroll 1
        for (uint32_t b0 = 0; b0 < kept && !closer; b0 += NB) {
            const uint32_t nb = kept - b0;  // uniform
            float4 v[NB][CH > 0 ? CH : 1];
#pragma unroll
            for (int r = 0; r < NB; ++r) {
                const bool ok = (uint32_t)r < nb;  // branch-free: predicated loads, see batch_distances
                const uint32_t rp = ok ? kept_pid[b0 + r] : 0u;
                const char* row = kStage ? sbase + (size_t)(b0 + r) * srow_bytes : gbase + (size_t)rp * row_bytes;
                typename RT::Hdr h = typename RT::Hdr();
                if (!kStage) h = RT::hdr(g, rp);
#pragma unroll
                for (int j = 0; j < CH; ++j)
                    v[r][j] = (ok && cok[j]) ? (kStage ? *reinterpret_cast<const float4*>(row + j * 512)
                                                       : widen_chunk<RT>(g, RT::ld_raw(row + j * 32 * RT::kChunkBytes), h, lane + 32 * j))
                                             : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            float p[NB];
#pragma unroll
            for (int r = 0; r < NB; ++r) p[r] = lane_partial<(CH > 0 ? CH : 1)>(q.r, v[r]);
            const float total = batch_butterfly<NB>(p, lane);
            const bool hit = (uint32_t)lane < nb && lane < NB && canon_bits(total) < cbits;
            closer = __any_sync(kFullMask, hit);
        }
        }
        if (!closer) {
            if constexpr (kStage && CH > 0) {
#pragma unroll
                for (int j = 0; j < CH; ++j) {
                    const uint32_t c = lane + 32 * j;
                    if (c < g.nchunks) kept_vecs[(size_t)kept * g.nchunks + c] = q.r[j];
                }
            }
            if (lane == 0) { out[kept] = cpid; kept_pid[kept] = cpid; }
            kept++;
            __syncwarp();
        } else {
            if (lane == 0) disc[nd] = cpid;
            nd++;
        }
    }
    __syncwarp();
    uint32_t total = kept;
    if (keep_pruned) {  // lib.rs:687-695
        const uint32_t take = min(nd, cap - kept);
        for (uint32_t t = lane; t < take; t += 32) out[kept + t] = disc[t];
        total = kept + take;
    }
    __syncwarp();
    return total;
}

// Shared-memory carve-up of one K2 warp.
struct SelectSmem {
    uint64_t* cand;      // cand_cap keys
    uint32_t* out;       // 2M
    uint32_t* disc;      // cand_cap
    uint32_t* kept_pid;  // 2M
    uint32_t* cpid;      // 2M + kNewCap   (relink: ids whose distance to the owner is needed)
    uint64_t* ckey;      // 2M + kNewCap
    float4* kept_vecs;   // 2M x nchunks (kStage only) — or, for long rows (CH == 0), the warp's query buffer (long_q_bytes)
    __host__ __device__ static size_t bytes(uint32_t cand_cap, uint32_t M, uint32_t nchunks, bool stage) {
        size_t b = (size_t)cand_cap * 8 + 2 * M * 4 + (size_t)cand_cap * 4 + 2 * M * 4 + (2 * M + kNewCap) * 4 + (2 * M + kNewCap) * 8;
        b = (b + 15) / 16 * 16;
        if (stage) b += (size_t)2 * M * nchunks * 16;
        else if (nchunks > 256) b += long_q_bytes(nchunks);
        return b;
    }
    __device__ void carve(unsigned char* base, uint32_t cand_cap, uint32_t M, uint32_t nchunks) {
        unsigned char* p = base;
        cand = reinterpret_cast<uint64_t*>(p); p += (size_t)cand_cap * 8;
        ckey = reinterpret_cast<uint64_t*>(p); p += (size_t)(2 * M + kNewCap) * 8;
        out = reinterpret_cast<uint32_t*>(p); p += 2 * M * 4;
        disc = reinterpret_cast<uint32_t*>(p); p += (size_t)cand_cap * 4;
        kept_pid = reinterpret_cast<uint32_t*>(p); p += 2 * M * 4;
        cpid = reinterpret_cast<uint32_t*>(p); p += (2 * M + kNewCap) * 4;
        size_t off = (size_t)(p - base);
        off = (off + 15) / 16 * 16;
        kept_vecs = reinterpret_cast<float4*>(base + off);
    }
};

// ---------------------------------------------------------------------------------------------------------
// KA: descent of every insert of the batch (lib.rs:443-463).  Output: `nearest` (ascending keys) per insert.
// ---------------------------------------------------------------------------------------------------------
template <int CH, int ROW_T, int EF_T, int B, class RT>
__global__ void __launch_bounds__(kSearchWarps * 32, kSearchCtasPerSm) insert_search_kernel(BuildArgs a) {  // same occupancy as K1
    traverse<CH, ROW_T, EF_T, B, RT, false, false, false, uint32_t>(
        a.g, a.work, a.tier, a.layer, a.efc, nullptr,
        [&](uint32_t w, QVec<CH>& q, int lane) { q_from_point<CH, RT>(q, a.g, a.base + w, lane); },
        [&](uint32_t w, const uint64_t* near, uint32_t len, const WarpState&, int lane) {
            for (uint32_t j = lane; j < len; j += 32) a.cand_keys[(size_t)w * a.cand_cap + j] = near[j] & kKeyMask;
            if (lane == 0) a.cand_cnt[w] = len;
        });
}

// ---------------------------------------------------------------------------------------------------------
// K2: select_heuristic for the new nodes (lib.rs:465-473), own-row write (lib.rs:516) and link-request emission.
// ---------------------------------------------------------------------------------------------------------
template <int CH, int NB, bool kStage, class RT>
__global__ void __launch_bounds__(kBuildWarps * 32) select_new_kernel(BuildArgs a, uint32_t smem_per_warp) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    SelectSmem sm;
    sm.carve(smem_raw + (size_t)warp * smem_per_warp, a.cand_cap, a.g.M, a.g.nchunks);
    const uint32_t cap = 2 * a.g.M;
    for (uint32_t w = blockIdx.x * kBuildWarps + warp; w < a.count; w += gridDim.x * kBuildWarps) {
        const uint32_t neu = a.base + w;
        const uint32_t W = a.cand_cnt[w];
        for (uint32_t j = lane; j < W; j += 32) sm.cand[j] = a.cand_keys[(size_t)w * a.cand_cap + j];
        __syncwarp();
        QVec<CH> q;
        if constexpr (CH == 0) { q.s = sm.kept_vecs; q.ngroups = (a.g.nchunks + 31) / 32; }
        const uint32_t total = select_heuristic_warp<CH, NB, kStage, RT>(a.g, sm.cand, W, sm.out, sm.disc, sm.kept_vecs, sm.kept_pid,
                                                                         a.keep_pruned != 0, lane, q, sm.ckey);
        uint32_t* row = a.zero + (size_t)neu * cap;
        for (uint32_t t = lane; t < cap; t += 32) {
            const uint32_t pid = t < total ? sm.out[t] : kInvalid;
            row[t] = pid;
            a.pairs[(size_t)w * cap + t] = t < total ? (((uint64_t)pid << 32) | neu) : kKeyNone;
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------------------
// K2': add_neighbor_heuristic (lib.rs:616-631) + rewrite (types.rs:88-98) for every target row of the batch.
//   candidates = {new...} U row(p), distances w.r.t. points[p]; `push` admission with ef = ef_construction and
//   no truncation (lib.rs:704-720); then select_heuristic; then the row is rewritten.
// ---------------------------------------------------------------------------------------------------------
template <int CH, int NB, bool kStage, class RT>
__global__ void __launch_bounds__(kBuildWarps * 32) relink_kernel(BuildArgs a, uint32_t smem_per_warp) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    SelectSmem sm;
    sm.carve(smem_raw + (size_t)warp * smem_per_warp, a.cand_cap, a.g.M, a.g.nchunks);
    const uint32_t cap = 2 * a.g.M;
    const uint32_t n_seg = *a.n_seg;
    for (;;) {
        unsigned long long w = 0;
        if (lane == 0) w = atomicAdd(a.work.work_counter, 1ull);
        w = __shfl_sync(kFullMask, w, 0);
        if (w >= n_seg) break;
        uint32_t pos = a.seg_start[w];
        const uint32_t p = (uint32_t)(a.sorted_pairs[pos] >> 32);
        uint32_t* row = a.zero + (size_t)p * cap;
        QVec<CH> q;
        if constexpr (CH == 0) { q.s = sm.kept_vecs; q.ngroups = (a.g.nchunks + 31) / 32; }
        for (;;) {  // rounds of at most kNewCap link requests (one round unless p is a hub of this batch)
            // ---- gather: new ids first (push(new), lib.rs:626), then the row's valid prefix (lib.rs:627-629) ----
            uint32_t n_newc = 0;
            while (n_newc < kNewCap && pos + n_newc < a.n_pairs_cap && (uint32_t)(a.sorted_pairs[pos + n_newc] >> 32) == p) n_newc++;
            if (n_newc == 0) break;
            for (uint32_t t = lane; t < n_newc; t += 32) sm.cpid[t] = (uint32_t)a.sorted_pairs[pos + t];
            pos += n_newc;
            uint32_t rcount = cap;
            for (uint32_t t0 = 0; t0 < cap; t0 += 32) {
                const uint32_t e = t0 + lane;
                const uint32_t ent = e < cap ? __ldcg(row + e) : kInvalid;
                const uint32_t m = __ballot_sync(kFullMask, ent == kInvalid);
                if (!m || (uint32_t)(__ffs(m) - 1) > (uint32_t)lane) sm.cpid[n_newc + e] = ent;
                if (m) { rcount = t0 + __ffs(m) - 1; break; }
            }
            const uint32_t C = n_newc + rcount;
            __syncwarp();
            q_from_point<CH, RT>(q, a.g, p, lane);  // (per round: select_heuristic below reuses q for the candidates)
            batch_distances<CH, NB, RT>(a.g, q, sm.cpid, sm.ckey, C, lane);
            // ---- push admission (lib.rs:704-720, `nearest` is never truncated here): entry j, in push order, enters
            // iff fewer than ef earlier-pushed entries are smaller (counting earlier REJECTED entries is harmless: a
            // rejected entry already has >= ef smaller admitted ones).  Then sort the admitted keys by counting.
            uint32_t W = C;
            if (a.efc >= C) {  // everything is admitted (ef_construction >= row width + new ids): the common case
                for (uint32_t j0 = 0; j0 < C; j0 += 32) {
                    const uint32_t j = j0 + lane;
                    const uint64_t kj = j < C ? sm.ckey[j] : kKeyNone;
                    uint32_t r = 0;
                    for (uint32_t i = 0; i < C; ++i) r += (sm.ckey[i] < kj) ? 1u : 0u;
                    if (j < C) sm.cand[r] = kj;
                }
            } else {
                W = 0;
                for (uint32_t j0 = 0; j0 < C; j0 += 32) {
                    const uint32_t j = j0 + lane;
                    const uint64_t kj = j < C ? sm.ckey[j] : kKeyNone;
                    uint32_t earlier = 0;
                    for (uint32_t i = 0; i < C; ++i) earlier += (i < j && sm.ckey[i] < kj) ? 1u : 0u;
                    const bool adm = j < C && earlier < a.efc;
                    if (j < C) sm.disc[j] = adm ? 1u : 0u;
                    W += __popc(__ballot_sync(kFullMask, adm));
                }
                __syncwarp();
                for (uint32_t j0 = 0; j0 < C; j0 += 32) {
                    const uint32_t j = j0 + lane;
                    const uint64_t kj = j < C ? sm.ckey[j] : kKeyNone;
                    uint32_t r = 0;
                    for (uint32_t i = 0; i < C; ++i) r += (sm.disc[i] && sm.ckey[i] < kj) ? 1u : 0u;
                    if (j < C && sm.disc[j]) sm.cand[r] = kj;
                }
            }
            __syncwarp();
            const uint32_t total = select_heuristic_warp<CH, NB, kStage, RT>(a.g, sm.cand, W, sm.out, sm.disc, sm.kept_vecs,
                                                                             sm.kept_pid, a.keep_pruned != 0, lane, q, sm.ckey);
            for (uint32_t t = lane; t < cap; t += 32) __stcg(row + t, t < total ? sm.out[t] : kInvalid);  // rewrite
            __threadfence();
            __syncwarp();
        }
    }
}

// Simple mode reverse link (lib.rs:497-515, incl. the reversed comparator at lib.rs:510) for one (target, new) pair
// per warp, executed in ascending `new` order for every target (a target's requests are serialised by its warp).
template <int CH, class RT>
__global__ void __launch_bounds__(kBuildWarps * 32) relink_simple_kernel(BuildArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];  // long rows only: per warp the query buffer
    __shared__ uint32_t s_pid[kBuildWarps][4];
    __shared__ uint64_t s_key[kBuildWarps][kLongRowsInFlight];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const uint32_t cap = 2 * a.g.M;
    const uint32_t n_seg = *a.n_seg;
    for (;;) {
        unsigned long long w = 0;
        if (lane == 0) w = atomicAdd(a.work.work_counter, 1ull);
        w = __shfl_sync(kFullMask, w, 0);
        if (w >= n_seg) break;
        uint32_t pos = a.seg_start[w];
        const uint32_t p = (uint32_t)(a.sorted_pairs[pos] >> 32);
        uint32_t* row = a.zero + (size_t)p * cap;
        QVec<CH> q;
        if constexpr (CH == 0) {
            q.ngroups = (a.g.nchunks + 31) / 32;
            q.s = reinterpret_cast<float4*>(smem_raw + (size_t)warp * long_q_bytes(a.g.nchunks));
        }
        q_from_point<CH, RT>(q, a.g, p, lane);
        auto dist_to = [&](uint32_t pid) -> uint32_t {  // canonical distance bits from points[p] to points[pid]
            if constexpr (CH == 0) {
                __syncwarp();
                if (lane == 0) s_pid[warp][0] = pid;
                __syncwarp();
                batch_distances_long<kLongRowsInFlight, RT>(a.g, q, s_pid[warp], s_key[warp], 1u, lane);
                return key_dbits(s_key[warp][0]);
            } else {
                float4 v[CH > 0 ? CH : 1];
                load_row<(CH > 0 ? CH : 1), RT>(a.g, pid, lane, v);
                return canon_bits(butterfly_sum(lane_partial<(CH > 0 ? CH : 1)>(q.r, v)));
            }
        };
        while (pos < a.n_pairs_cap && (uint32_t)(a.sorted_pairs[pos] >> 32) == p) {
            const uint32_t neu = (uint32_t)a.sorted_pairs[pos++];
            const uint32_t dnew = dist_to(neu);
            // core::slice::binary_search_by (rustc >= 1.82) over the full 2M-wide row
            uint32_t size = cap, base = 0;
            auto cmp = [&](uint32_t k) -> int {
                const uint32_t third = __ldcg(row + k);
                if (third == kInvalid) return 1;                      // Ordering::Greater (lib.rs:507)
                const uint32_t dt = dist_to(third);
                return dnew < dt ? -1 : (dnew > dt ? 1 : 0);          // distance.cmp(&third_distance) (lib.rs:510)
            };
            while (size > 1) {
                const uint32_t half = size / 2, mid = base + half;
                base = cmp(mid) > 0 ? base : mid;
                size -= half;
            }
            const int c = cmp(base);
            const uint32_t idx = c == 0 ? base : base + (c < 0 ? 1u : 0u);
            // ZeroNode::insert (types.rs:100-113)
            if (idx < cap) {
                __syncwarp();
                if (__ldcg(row + idx) != kInvalid) {
                    uint32_t keep[4];
#pragma unroll
                    for (int t = 0; t < 4; ++t) {
                        const uint32_t e = lane + 32 * t;
                        keep[t] = (e >= idx && e + 1 < cap) ? __ldcg(row + e) : 0u;
                    }
                    __syncwarp();
#pragma unroll
                    for (int t = 0; t < 4; ++t) {
                        const uint32_t e = lane + 32 * t;
                        if (e >= idx && e + 1 < cap) __stcg(row + e + 1, keep[t]);
                    }
                }
                __syncwarp();
                if (lane == 0) __stcg(row + idx, neu);
                __threadfence();
                __syncwarp();
            }
        }
    }
}

}  // namespace idb
