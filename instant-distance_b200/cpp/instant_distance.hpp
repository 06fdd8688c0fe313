// instant_distance.hpp — C++17 host mirror of the reference crate's public surface (instant-distance/src/lib.rs) for f32
// vector points, forwarding to the C ABI (include/instant_distance_b200.h).  Same names, argument meaning and error
// behaviour as the Rust API so reference-side code reads the same:
//
//   auto [hnsw, ids] = instant_distance::Builder().ef_search(100).seed(42).build_hnsw(points);      // lib.rs:83-85
//   instant_distance::Search search;                                                                // lib.rs:767-778
//   for (auto item : hnsw.search(query, search)) use(item.distance, item.pid, *item.point);         // lib.rs:352-383
//
// The reference's API is infallible (panics on misuse); here misuse / device errors throw instant_distance::Error.
#pragma once
#include <cstdint>
#include <optional>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../../include/instant_distance_b200.h"

namespace instant_distance {

struct Error : std::runtime_error {
    idb_status status;
    Error(idb_status s, const std::string& m) : std::runtime_error(m), status(s) {}
};
inline void check(idb_status s) {
    if (s != IDB_OK) throw Error(s, idb_last_error());
}

// types.rs:236-267
struct PointId {
    uint32_t raw = IDB_INVALID;
    bool is_valid() const { return raw != IDB_INVALID; }
    uint32_t into_inner() const { return raw; }
    bool operator==(const PointId& o) const { return raw == o.raw; }
    bool operator<(const PointId& o) const { return raw < o.raw; }
};

// trait Point (lib.rs:780-782) for the one point type the GPU engine serves: an f32 vector under squared L2
// (FloatArray, instant-distance-py/src/lib.rs:359-421).  distance() is evaluated by the device library (canonical order).
struct Point {
    std::vector<float> v;
    Point() = default;
    Point(std::initializer_list<float> l) : v(l) {}
    explicit Point(std::vector<float> x) : v(std::move(x)) {}
    float distance(const Point& other) const {
        if (v.size() != other.v.size()) throw Error(IDB_ERR_INVALID_ARG, "points of different dimension");
        float d = 0.f;
        check(idb_distance_f32(v.data(), other.v.data(), (uint32_t)v.size(), 0, &d));
        return d;
    }
};

// lib.rs:115-128
struct Heuristic {
    bool extend_candidates = false;
    bool keep_pruned = true;
};

// lib.rs:399-403 / 175-180
struct Item {
    float distance;
    PointId pid;
    const Point* point;
};
template <class V>
struct MapItem {
    float distance;
    PointId pid;
    const Point* point;
    const V* value;
};

class Hnsw;
template <class V>
class HnswMap;

// lib.rs:560-574: result buffer of the last search (the traversal scratch lives on the device, owned by the index).
class Search {
    friend class Hnsw;
    std::vector<uint32_t> ids_;
    std::vector<float> dist_;
    uint32_t len_ = 0;

  public:
    Search() = default;  // Search::default()
    size_t len() const { return len_; }
};

class Builder;

// lib.rs:193-199
class Hnsw {
    friend class Builder;
    idb_index* raw_ = nullptr;
    std::vector<Point> points_;  // PointId order (lib.rs:263-270)
    size_t ef_search_ = 100;
    Hnsw() = default;

  public:
    Hnsw(const Hnsw&) = delete;
    Hnsw& operator=(const Hnsw&) = delete;
    Hnsw(Hnsw&& o) noexcept : raw_(o.raw_), points_(std::move(o.points_)), ef_search_(o.ef_search_) { o.raw_ = nullptr; }
    Hnsw& operator=(Hnsw&& o) noexcept {
        if (this != &o) { idb_index_free(raw_); raw_ = o.raw_; points_ = std::move(o.points_); ef_search_ = o.ef_search_; o.raw_ = nullptr; }
        return *this;
    }
    ~Hnsw() { idb_index_free(raw_); }
    static Builder builder();  // lib.rs:205-207

    // lib.rs:352-383: fills `search` and returns the whole `nearest` list (<= ef_search items, nearest first).
    std::vector<Item> search(const Point& point, Search& search) const {
        const uint32_t k = (uint32_t)(ef_search_ ? ef_search_ : 1);
        search.ids_.assign(k, IDB_INVALID);
        search.dist_.assign(k, 0.f);
        search.len_ = 0;
        if (!points_.empty() && point.v.size() != points_[0].v.size()) throw Error(IDB_ERR_INVALID_ARG, "query dimension differs from the index");
        if (ef_search_ && !points_.empty())
            check(idb_search_batch_f32(raw_, point.v.data(), 1, (uint32_t)ef_search_, k, search.ids_.data(), search.dist_.data(), &search.len_));
        std::vector<Item> out;
        for (uint32_t i = 0; i < search.len_ && i < k; ++i)
            out.push_back(Item{search.dist_[i], PointId{search.ids_[i]}, &points_[search.ids_[i]]});
        return out;
    }
    // Not in the reference: the points within `radius` of `point` that layer 0 reaches from its ef_search approximate nearest
    // neighbours through points within `radius` (idb_graph_range_search_batch_f32, DESIGN.md §9c; ef_search 0 = the index's), nearest
    // first, ties by lower PointId.  A subset of the exact range search's result, at a cost that follows the hits.
    std::vector<Item> search_range_graph(const Point& point, float radius, uint32_t ef_search = 0) const {
        if (!points_.empty() && point.v.size() != points_[0].v.size()) throw Error(IDB_ERR_INVALID_ARG, "query dimension differs from the index");
        uint64_t offsets[2] = {0, 0};
        std::vector<uint32_t> ids(1024);
        std::vector<float> dist(1024);
        idb_status st = idb_graph_range_search_batch_f32(raw_, point.v.data(), 1, ef_search, radius, ids.size(), offsets, ids.data(), dist.data());
        if (st == IDB_ERR_CAPACITY && offsets[1] > ids.size()) {  // once more, sized exactly
            ids.resize(offsets[1]);
            dist.resize(offsets[1]);
            st = idb_graph_range_search_batch_f32(raw_, point.v.data(), 1, ef_search, radius, ids.size(), offsets, ids.data(), dist.data());
        }
        check(st);
        std::vector<Item> out;
        for (uint64_t i = 0; i < offsets[1]; ++i) out.push_back(Item{dist[i], PointId{ids[i]}, &points_[ids[i]]});
        return out;
    }
    // #[doc(hidden)] get (lib.rs:394-396)
    std::optional<Item> get(size_t i, const Search& s) const {
        if (i >= s.len_) return std::nullopt;
        return Item{s.dist_[i], PointId{s.ids_[i]}, &points_[s.ids_[i]]};
    }
    // Not in the reference: Construction::insert (core:437-528) of each point on layer 0 (idb_index_insert_f32); returns their
    // PointIds, which continue from the current count in input order.  Like a `&mut self` method it invalidates the Items of
    // earlier searches (their points move when points_ grows).  On IDB_ERR_CAPACITY the index keeps the batches before the failing
    // one; their points are appended to points_ before the Error is thrown, so points_ always has one entry per PointId.
    std::vector<PointId> insert(std::vector<Point> points, size_t ef_construction = 100,
                                std::optional<Heuristic> heuristic = Heuristic{}) {
        idb_info info;
        check(idb_index_info(raw_, &info));
        std::vector<float> flat;
        flat.reserve(points.size() * info.dim);
        for (const Point& p : points) {
            if (p.v.size() != info.dim) throw Error(IDB_ERR_INVALID_ARG, "point dimension differs from the index");
            flat.insert(flat.end(), p.v.begin(), p.v.end());
        }
        idb_params p;
        check(idb_params_default(&p));
        p.M = info.M;
        p.ef_construction = (uint32_t)ef_construction;
        p.heuristic = heuristic ? 1 : 0;
        p.extend_candidates = heuristic && heuristic->extend_candidates;
        p.keep_pruned = !heuristic || heuristic->keep_pruned;
        std::vector<uint32_t> ids(points.size());
        const idb_status st = idb_index_insert_f32(raw_, flat.data(), points.size(), info.dim, &p, nullptr, ids.data());
        if (st != IDB_OK) {
            const Error err(st, idb_last_error());
            idb_info now;
            if (idb_index_info(raw_, &now) == IDB_OK)
                for (uint64_t i = 0; i < now.n - info.n && i < points.size(); ++i) points_.push_back(std::move(points[i]));
            throw err;
        }
        std::vector<PointId> out(points.size());
        for (size_t i = 0; i < points.size(); ++i) out[i] = PointId{ids[i]};
        for (Point& pt : points) points_.push_back(std::move(pt));
        return out;
    }
    // Not in the reference: removes the points `pids` (distinct PointIds, idb_index_remove).  The rows that listed a removed point
    // are selected again with ef_construction and the heuristic (nullopt: the simple selection); the other points keep their order
    // and are renumbered without gaps, so points_ drops the removed ones.  Returns, for each point the index had, its PointId
    // afterwards, or nullopt for a removed one.  Like a `&mut self` method it invalidates the Items of earlier searches.
    std::vector<std::optional<PointId>> remove(const std::vector<PointId>& pids, size_t ef_construction = 100,
                                               std::optional<Heuristic> heuristic = Heuristic{}) {
        idb_info info;
        check(idb_index_info(raw_, &info));
        idb_params p;
        check(idb_params_default(&p));
        p.M = info.M;
        p.ef_construction = (uint32_t)ef_construction;
        p.heuristic = heuristic ? 1 : 0;
        p.extend_candidates = heuristic && heuristic->extend_candidates;
        p.keep_pruned = !heuristic || heuristic->keep_pruned;
        std::vector<uint32_t> raw(pids.size()), new_ids(info.n);
        for (size_t i = 0; i < pids.size(); ++i) raw[i] = pids[i].raw;
        check(idb_index_remove(raw_, raw.data(), raw.size(), &p, new_ids.data()));
        std::vector<std::optional<PointId>> out(info.n);
        std::vector<Point> kept;
        for (size_t x = 0; x < info.n; ++x) {
            if (new_ids[x] == IDB_INVALID) continue;
            out[x] = PointId{new_ids[x]};
            kept.push_back(std::move(points_[x]));
        }
        points_ = std::move(kept);
        return out;
    }
    // lib.rs:386-391, types.rs:269-275
    const std::vector<Point>& iter() const { return points_; }
    const Point& operator[](PointId p) const { return points_.at(p.raw); }
    idb_index* raw() const { return raw_; }
};

// lib.rs:130-173
template <class V>
class HnswMap {
    friend class Builder;
    Hnsw hnsw_;

  public:
    std::vector<V> values;  // pub values (lib.rs:133), PointId order (lib.rs:144-149)
    HnswMap(Hnsw h, std::vector<V> v) : hnsw_(std::move(h)), values(std::move(v)) {}
    std::vector<MapItem<V>> search(const Point& point, Search& s) const {
        std::vector<MapItem<V>> out;
        for (const Item& it : hnsw_.search(point, s)) out.push_back(MapItem<V>{it.distance, it.pid, it.point, &values[it.pid.raw]});
        return out;
    }
    const std::vector<Point>& iter() const { return hnsw_.iter(); }
    // Hnsw::insert, with one value per point, appended in PointId order.
    std::vector<PointId> insert(std::vector<Point> points, std::vector<V> vals, size_t ef_construction = 100,
                                std::optional<Heuristic> heuristic = Heuristic{}) {
        if (vals.size() != points.size()) throw Error(IDB_ERR_INVALID_ARG, "points and values differ in length");
        const size_t n0 = hnsw_.iter().size();
        try {
            std::vector<PointId> ids = hnsw_.insert(std::move(points), ef_construction, heuristic);
            for (V& v : vals) values.push_back(std::move(v));
            return ids;
        } catch (const Error&) {  // values follow PointIds, also for the points a failed insert kept
            for (size_t i = 0; i < hnsw_.iter().size() - n0; ++i) values.push_back(std::move(vals[i]));
            throw;
        }
    }
    // Hnsw::remove; the values of the removed points are dropped, the others follow their points' new PointIds.
    std::vector<std::optional<PointId>> remove(const std::vector<PointId>& pids, size_t ef_construction = 100,
                                               std::optional<Heuristic> heuristic = Heuristic{}) {
        std::vector<std::optional<PointId>> new_ids = hnsw_.remove(pids, ef_construction, heuristic);
        std::vector<V> kept;
        for (size_t x = 0; x < new_ids.size(); ++x)
            if (new_ids[x]) kept.push_back(std::move(values[x]));
        values = std::move(kept);
        return new_ids;
    }
};

// lib.rs:21-113
class Builder {
    size_t ef_search_ = 100, ef_construction_ = 100;
    std::optional<Heuristic> heuristic_ = Heuristic{};
    float ml_;
    uint64_t seed_ = 0;
    uint32_t m_ = 32;
    int device_ = 0;
    uint32_t metric_ = IDB_METRIC_L2SQ;

  public:
    Builder() {
        idb_params p;
        check(idb_params_default(&p));
        ml_ = p.ml;
    }
    Builder& ef_construction(size_t v) { ef_construction_ = v; return *this; }
    Builder& ef_search(size_t v) { ef_search_ = v; return *this; }
    Builder& select_heuristic(std::optional<Heuristic> h) { heuristic_ = h; return *this; }
    Builder& ml(float v) { ml_ = v; return *this; }
    Builder& seed(uint64_t v) { seed_ = v; return *this; }
    Builder& device(int d) { device_ = d; return *this; }  // not in the reference: which GPU
    // Not in the reference: IDB_METRIC_L2SQ (default) or IDB_METRIC_COSINE — searches then report 1 - cos (DESIGN.md §3a);
    // Point::distance stays squared L2.
    Builder& metric(uint32_t m) { metric_ = m; return *this; }
    std::tuple<size_t, size_t, float, uint64_t> into_parts() const { return {ef_search_, ef_construction_, ml_, seed_}; }

    // Builder::build_hnsw (lib.rs:83-85)
    std::pair<Hnsw, std::vector<PointId>> build_hnsw(std::vector<Point> points) const {
        const uint32_t dim = points.empty() ? 1u : (uint32_t)points[0].v.size();
        std::vector<float> flat;
        flat.reserve(points.size() * dim);
        for (const Point& p : points) {
            if (p.v.size() != dim) throw Error(IDB_ERR_INVALID_ARG, "all points must have the same dimension");
            flat.insert(flat.end(), p.v.begin(), p.v.end());
        }
        idb_params p;
        check(idb_params_default(&p));
        p.M = m_;
        p.ef_construction = (uint32_t)ef_construction_;
        p.ef_search = (uint32_t)ef_search_;
        p.ml = ml_;
        p.seed = seed_;
        p.heuristic = heuristic_ ? 1 : 0;
        p.extend_candidates = heuristic_ && heuristic_->extend_candidates;
        p.keep_pruned = !heuristic_ || heuristic_->keep_pruned;
        p.device = device_;
        std::vector<uint32_t> ids(points.size());
        Hnsw h;
        check(idb_build_ex(flat.data(), points.size(), dim, &p, metric_, &h.raw_, ids.data()));
        h.ef_search_ = ef_search_;
        h.points_.resize(points.size());
        std::vector<PointId> out(points.size());
        for (size_t i = 0; i < points.size(); ++i) {
            out[i] = PointId{ids[i]};
            h.points_[ids[i]] = std::move(points[i]);
        }
        return {std::move(h), std::move(out)};
    }
    // Builder::build (lib.rs:78-80) -> HnswMap::new (lib.rs:141-152)
    template <class V>
    HnswMap<V> build(std::vector<Point> points, std::vector<V> values) const {
        if (values.size() != points.size()) throw Error(IDB_ERR_INVALID_ARG, "points and values differ in length");
        auto [h, ids] = build_hnsw(std::move(points));
        std::vector<V> by_pid(values.size());
        for (size_t i = 0; i < values.size(); ++i) by_pid[ids[i].raw] = std::move(values[i]);
        return HnswMap<V>(std::move(h), std::move(by_pid));
    }
};

inline Builder Hnsw::builder() { return Builder(); }

}  // namespace instant_distance
