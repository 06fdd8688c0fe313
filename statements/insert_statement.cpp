// insert_statement.cpp — CPU statement of the index insert (idb_index_insert_f32, csrc/build.cu insert_index), the GPU insert is
// checked against it bit for bit.  TEST INFRASTRUCTURE ONLY, like oracle/: never linked into the product.
//
// The oracle's translation unit is compiled into this one, so the statement runs on the oracle's own push / search_layer /
// select_heuristic / distance and its orc_index, and the oracle's C entry points (orc_from_graph, orc_export_*, orc_free) serve the
// handles made here.  On top of it:
//   ins_build_batched   the library's batched build (the schedule orc_build_batched states), with one batch body shared with the
//                       insert, and an optional stop: the layer-0 loop ends at the first batch boundary >= stop_at and the graph of
//                       that many points is returned (its upper layers are complete: they hold PointIds below layer 0's start);
//   ins_insert_batched  Construction::insert(new, 0, layers) (core:437-528) for m rows appended to an existing graph, in the layer-0
//                       schedule from g0 = n0: b = min(max_batch, max(1, g0 / growth)), also when the graph has no upper layer (the
//                       build inserts its only layer sequentially).  An empty graph takes its first row as PointId 0 and inserts
//                       from 1.
// With the same rows, a graph stopped at a layer-0 batch boundary n0 and then given rows [n0, n) by ins_insert_batched equals the
// full batched build: the insert's batches are exactly the build's remaining layer-0 batches.
#include "../oracle/hnsw_oracle.cpp"

namespace {

// One batch of the batched schedule (orc_build_batched's body): KA + K2 against the zero layer as the batch found it, the own rows
// and sorted link requests, then K2' on every target row once.
struct BatchBody {
    orc_index* ix = nullptr;
    uint32_t top = 0;
    size_t efc = 100;
    Heuristic h;
    int threads = 1;
    std::vector<Search> searches;
    std::vector<uint32_t> found;
    std::vector<uint64_t> pairs, seg;

    BatchBody(orc_index* index, const orc_params* p, uint64_t n_total) : ix(index), efc(p->ef_construction), threads(std::max(1, p->threads)) {
        top = (uint32_t)ix->layers.size();
        h.on = p->heuristic != 0;
        h.keep_pruned = p->keep_pruned != 0;
        searches.resize(threads);
        for (auto& s : searches) s.visited.with_capacity(n_total);
    }

    void run(uint64_t g0, uint64_t b, uint32_t layer) {
        const uint32_t M = ix->M, cap = 2 * M;
        const Points pts = ix->pts();
        auto zrow = [&](uint32_t pid) { return ix->zero.data() + (size_t)pid * cap; };
        auto no_rows = [](uint32_t, uint32_t, uint32_t*) { return 0u; };
        const uint32_t num = layer == 0 ? 2 * M : M;  // core:445
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
                    search_layer(s, point, [&](uint32_t pid, uint32_t links, uint32_t* buf) {
                        return copy_row(zrow(pid), cap, links, buf); }, pts, num);
                    break;
                }
                if (cur == 0) break;
            }
            if (h.on) select_heuristic(s, point, no_rows, pts, M, h);  // core:470-472
            else if (s.nearest.size() > cap) s.nearest.resize(cap);  // core:466-469
            for (size_t i = 0; i < s.nearest.size(); ++i) found[w * cap + i] = key_pid(s.nearest[i]);
        });
        pairs.clear();
        for (uint64_t w = 0; w < b; ++w) {
            const uint32_t neu = (uint32_t)(g0 + w);
            std::memcpy(zrow(neu), &found[w * cap], cap * sizeof(uint32_t));
            for (uint32_t i = 0; i < cap && found[w * cap + i] != INVALID; ++i) pairs.push_back(((uint64_t)found[w * cap + i] << 32) | neu);
        }
        std::sort(pairs.begin(), pairs.end());
        seg.clear();
        for (size_t i = 0; i < pairs.size(); ++i)
            if (i == 0 || (pairs[i] >> 32) != (pairs[i - 1] >> 32)) seg.push_back(i);
        parallel_for(0, seg.size(), threads, 16, [&](uint64_t si, int t) {
            const size_t s0 = seg[si], s1 = si + 1 < seg.size() ? seg[si + 1] : pairs.size();
            const uint32_t tgt = (uint32_t)(pairs[s0] >> 32);
            const float* tpoint = pts.row(tgt);
            uint32_t* row = zrow(tgt);
            if (!h.on) {
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
            Search& s = searches[t];
            uint32_t buf[256];
            for (size_t r0 = s0; r0 < s1; r0 += kNewCap) {  // rounds of at most kNewCap new ids
                const size_t r1 = std::min<size_t>(s1, r0 + kNewCap);
                s.reset();
                s.ef = efc;
                for (size_t r = r0; r < r1; ++r) push(s, (uint32_t)pairs[r], tpoint, pts);  // the new ids first (core:626)
                const uint32_t cnt = copy_row(row, cap, cap, buf);
                for (uint32_t j = 0; j < cnt; ++j) push(s, buf[j], tpoint, pts);  // then the row (core:627-629)
                select_heuristic(s, tpoint, no_rows, pts, M, h);
                for (uint32_t i = 0; i < cap; ++i) row[i] = i < s.nearest.size() ? key_pid(s.nearest[i]) : INVALID;
            }
        });
    }
};

uint64_t batch_size(uint64_t g0, uint32_t max_batch, uint32_t growth) {
    return std::min<uint64_t>(max_batch, std::max<uint64_t>(1, g0 / growth));
}

}  // namespace

// The batched build (orc_build_batched's graph for the same arguments).  stop_at < n: the layer-0 loop ends at the first batch
// boundary >= stop_at; the returned graph has that many points (orc_n), the rows and zero rows below it and every upper layer.
ORC_API orc_index* ins_build_batched(const float* rows, uint64_t n, uint32_t dim, const orc_params* p, uint32_t max_batch,
                                     uint32_t growth, uint64_t stop_at, uint32_t* out_ids) {
    if (max_batch == 0 || growth == 0 || p->extend_candidates || n == 0 || n >= 0xFFFFFFFFull) return nullptr;
    auto* ix = new orc_index();
    ix->M = p->M;
    ix->dim = dim;
    ix->stride = ((size_t)dim + 3) / 4 * 4;
    ix->n = n;
    ix->ef_search = p->ef_search;
    ix->metric = p->metric;
    const auto sizes = init_index(ix, rows, n, dim, p, out_ids);
    const uint32_t num_layers = (uint32_t)sizes.size(), top = num_layers - 1;
    BatchBody body(ix, p, n);
    // the layers are filled top first, but the descent reads the finished snapshots only: the body sees all `top` of them
    for (uint32_t li = 0; li < num_layers; ++li) {
        const uint32_t layer = num_layers - li - 1;
        const uint64_t size = sizes[li].first, cumulative = sizes[li].second;
        const uint64_t start = std::max<uint64_t>(cumulative - size, 1), end = cumulative;
        uint64_t g0 = start;
        while (g0 < end) {
            if (layer == 0 && g0 >= stop_at) break;
            const uint64_t b = std::min<uint64_t>(layer == top ? 1 : batch_size(g0, max_batch, growth), end - g0);
            body.run(g0, b, layer);
            g0 += b;
        }
        if (layer != 0) snapshot_layer(ix, layer, end, std::max(1, p->threads));
        if (layer == 0 && g0 < n) {  // stopped: keep the first g0 points
            ix->n = g0;
            ix->layer_n[0] = g0;
            ix->zero.resize(g0 * 2 * (size_t)ix->M);
        }
    }
    return ix;
}

// Appends m rows (m x dim, as the index stores them) to `ix` and inserts them on layer 0 in the insert's schedule.
ORC_API int ins_insert_batched(orc_index* ix, const float* rows, uint64_t m, const orc_params* p, uint32_t max_batch, uint32_t growth) {
    if (max_batch == 0 || growth == 0 || p->extend_candidates || p->M != ix->M || ix->n + m >= 0xFFFFFFFFull) return -1;
    if (m == 0) return 0;
    const uint64_t n0 = ix->n, n1 = n0 + m;
    float* pts = alloc_rows(n1, ix->stride);  // the row storage grows: old rows, then the new ones zero padded
    if (!pts) return -1;
    if (n0) std::memcpy(pts, ix->points, n0 * ix->stride * sizeof(float));
    for (uint64_t r = 0; r < m; ++r) std::memcpy(pts + (n0 + r) * ix->stride, rows + r * ix->dim, ix->dim * sizeof(float));
    std::free(ix->points);
    ix->points = pts;
    ix->zero.resize(n1 * 2 * (size_t)ix->M, INVALID);
    ix->n = n1;
    if (ix->layer_n.empty()) ix->layer_n.assign(1, 0);
    ix->layer_n[0] = n1;
    BatchBody body(ix, p, n1);  // visited capacity: every PointId after the insert
    for (uint64_t g0 = std::max<uint64_t>(n0, 1); g0 < n1;) {
        const uint64_t b = std::min<uint64_t>(batch_size(g0, max_batch, growth), n1 - g0);
        body.run(g0, b, 0);
        g0 += b;
    }
    return 0;
}
