// persist.cu — index files in the layout the reference's Python binding writes with bincode 1.3
// (instant-distance-py/src/lib.rs:58-75, 121-137): `Hnsw { ef_search, points, zero, layers }` (lib.rs:193-199) serialised
// field by field, little-endian, usize as u64, Vec<T> as u64 length + elements, fixed arrays ([f32; DIM], [PointId; 2M],
// [PointId; M]; types.rs:63, 83-85) with no length prefix.  For dim = 300 and M = 32 this is the reference's `.idx` body;
// other (dim, M) use the same scheme.  The layout is restated from bincode's documented encoding — no reference-written
// fixture exists in the reference tree, so byte-level parity with a real file is UNPINNED (DESIGN.md §7).
// An `HnswMap` file continues with `values` (lib.rs:131-134): idb_index_load reports the offset where they start.
// The file does not record the metric: a cosine index saves its (normalised) rows, and idb_index_load_ex takes them as given.
#include <cstdio>
#include <cstring>
#include <vector>

#include "internal.cuh"

using namespace idb;

namespace {
struct File {
    FILE* f = nullptr;
    ~File() { if (f) std::fclose(f); }
};
bool put(FILE* f, const void* p, size_t n) { return n == 0 || std::fwrite(p, 1, n, f) == n; }
bool get(FILE* f, void* p, size_t n) { return n == 0 || std::fread(p, 1, n, f) == n; }
bool put_u64(FILE* f, uint64_t v) { return put(f, &v, 8); }
bool get_u64(FILE* f, uint64_t* v) { return get(f, v, 8); }
}  // namespace

extern "C" {

idb_status idb_index_save(const idb_index* index, const char* path) {
    if (!index || !path) return fail(IDB_ERR_INVALID_ARG, "null argument");
    Index* ix = const_cast<Index*>(reinterpret_cast<const Index*>(index));
    std::lock_guard<std::mutex> lk(ix->mu);
    CUDA_TRY(cudaSetDevice(ix->device));
    File out;
    out.f = std::fopen(path, "wb");
    if (!out.f) return fail(IDB_ERR_IO, "cannot open %s for writing", path);
    const uint64_t n = ix->n;
    bool ok = put_u64(out.f, ix->ef_search) && put_u64(out.f, n);
    // points: n x [f32; dim]
    const uint64_t chunk = 1 << 16;
    std::vector<float> buf((size_t)chunk * ix->dim);
    for (uint64_t r0 = 0; ok && r0 < n; r0 += chunk) {
        const uint64_t m = std::min(chunk, n - r0);
        idb_status st = ix->copy_points_f32(buf.data(), r0, m);  // bf16- and fp16-stored rows are written widened (exact)
        if (st != IDB_OK) return st;
        ok = put(out.f, buf.data(), m * ix->dim * 4);
    }
    // zero: n x [u32; 2M]
    ok = ok && put_u64(out.f, n);
    std::vector<uint32_t> rows((size_t)chunk * 2 * ix->M);
    for (uint64_t r0 = 0; ok && r0 < n; r0 += chunk) {
        const uint64_t m = std::min(chunk, n - r0);
        CUDA_TRY(ix->graph.copy_out(0, r0, m, ix->M, rows.data(), ix->stream));
        ok = put(out.f, rows.data(), m * 2 * ix->M * 4);
    }
    // layers: Vec<Vec<UpperNode>>, layers[0] = layer 1
    ok = ok && put_u64(out.f, ix->graph.upper.size());
    for (uint32_t l = 1; ok && l <= ix->graph.upper.size(); ++l) {
        const uint64_t nl = ix->graph.upper_n[l - 1];
        ok = put_u64(out.f, nl);
        std::vector<uint32_t> u((size_t)nl * ix->M);
        CUDA_TRY(ix->graph.copy_out(l, 0, nl, ix->M, u.data(), ix->stream));
        ok = ok && put(out.f, u.data(), u.size() * 4);
    }
    if (!ok) return fail(IDB_ERR_IO, "short write to %s", path);
    return IDB_OK;
}

idb_status idb_index_load(const char* path, uint32_t dim, uint32_t M, int32_t device, idb_index** out_index, uint64_t* out_values_offset) {
    return idb_index_load_ex(path, dim, M, IDB_METRIC_L2SQ, device, out_index, out_values_offset);
}

idb_status idb_index_load_ex(const char* path, uint32_t dim, uint32_t M, uint32_t metric, int32_t device, idb_index** out_index,
                             uint64_t* out_values_offset) {
    return idb_index_load_storage(path, dim, M, metric, IDB_STORAGE_F32, device, out_index, out_values_offset);
}

idb_status idb_index_load_storage(const char* path, uint32_t dim, uint32_t M, uint32_t metric, uint32_t storage, int32_t device,
                                  idb_index** out_index, uint64_t* out_values_offset) {
    if (!path || !out_index) return fail(IDB_ERR_INVALID_ARG, "null argument");
    *out_index = nullptr;
    if (dim == 0 || M < 2 || M > 64) return fail(IDB_ERR_INVALID_ARG, "dim/M invalid");
    if (metric != IDB_METRIC_L2SQ && metric != IDB_METRIC_COSINE) return fail(IDB_ERR_INVALID_ARG, "unknown metric %u", metric);
    if (!storage_known(storage)) return fail(IDB_ERR_INVALID_ARG, "unknown storage %u", storage);
    if (idb_status s = check_storage_metric(storage, metric); s != IDB_OK) return s;
    File in;
    in.f = std::fopen(path, "rb");
    if (!in.f) return fail(IDB_ERR_IO, "cannot open %s", path);
    std::fseek(in.f, 0, SEEK_END);
    const uint64_t fsize = (uint64_t)std::ftell(in.f);
    std::fseek(in.f, 0, SEEK_SET);
    uint64_t ef = 0, n = 0, n2 = 0, nl = 0;
    if (!get_u64(in.f, &ef) || !get_u64(in.f, &n)) return fail(IDB_ERR_FORMAT, "%s: truncated header", path);
    if (n >= 0xFFFFFFFFull || fsize < 16 || n > (fsize - 16) / ((uint64_t)dim * 4)) return fail(IDB_ERR_FORMAT, "%s: point count %llu does not fit the file (dim %u?)", path, (unsigned long long)n, dim);
    std::vector<float> pts((size_t)n * dim);
    if (!get(in.f, pts.data(), pts.size() * 4) || !get_u64(in.f, &n2) || n2 != n)
        return fail(IDB_ERR_FORMAT, "%s: zero-layer length does not match the point count (wrong dim?)", path);
    std::vector<uint32_t> zero((size_t)n * 2 * M);
    if (!get(in.f, zero.data(), zero.size() * 4) || !get_u64(in.f, &nl) || nl > 31)
        return fail(IDB_ERR_FORMAT, "%s: bad layer table (wrong M?)", path);
    std::vector<std::vector<uint32_t>> upper(nl);
    std::vector<const uint32_t*> ptrs(nl);
    std::vector<uint64_t> counts(nl);
    for (uint64_t l = 0; l < nl; ++l) {
        uint64_t c = 0;
        if (!get_u64(in.f, &c) || c > n) return fail(IDB_ERR_FORMAT, "%s: bad layer %llu size", path, (unsigned long long)(l + 1));
        upper[l].resize((size_t)c * M);
        if (!get(in.f, upper[l].data(), upper[l].size() * 4)) return fail(IDB_ERR_FORMAT, "%s: truncated layer %llu", path, (unsigned long long)(l + 1));
        ptrs[l] = upper[l].data();
        counts[l] = c;
    }
    if (out_values_offset) *out_values_offset = (uint64_t)std::ftell(in.f);
    for (uint32_t v : zero)
        if (v != IDB_INVALID && v >= n) return fail(IDB_ERR_FORMAT, "%s: adjacency refers to PointId %u >= %llu", path, v, (unsigned long long)n);
    // the same checks as for any adopted graph (entries inside their layer, n >= n_1 >= ... >= 1; for cosine, unit rows); a file that
    // fails them is malformed.  The rows were saved widened, so narrowing them again to the storage they came from is exact.
    return adopt_graph(pts.data(), n, dim, M, (uint32_t)std::min<uint64_t>(ef, 0xFFFFFFFFu), zero.data(), (uint32_t)nl, ptrs.data(),
                       counts.data(), storage, metric, device, out_index, true);
}

}  // extern "C"
