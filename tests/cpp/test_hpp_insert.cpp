// Hnsw::insert / HnswMap::insert of the host mirror header when the insert fails part way (run with IDB_VIS_TIER=0,
// IDB_VIS_SLOTS=1024 and IDB_RETRY_SLOTS=1024, so that inserts with ef_construction = 200 overflow KA's retry pass once the index has
// grown): the Error carries IDB_ERR_CAPACITY, and points_ / values still have one entry per PointId of the index, so searches that
// return the points the index kept can dereference them.
#include <cstdio>
#include <random>
#include <string>

#include "../../instant-distance_b200/cpp/instant_distance.hpp"

using namespace instant_distance;

int main() {
    std::mt19937 rng(5);
    std::uniform_real_distribution<float> u(0.f, 1.f);
    std::vector<Point> base, more;
    std::vector<std::string> vals, more_vals;
    for (int i = 0; i < 6000; ++i) {
        Point p;
        for (int d = 0; d < 16; ++d) p.v.push_back(u(rng));
        (i < 500 ? base : more).push_back(p);
        (i < 500 ? vals : more_vals).push_back((i < 500 ? "b" : "d") + std::to_string(i));
    }
    auto map = Hnsw::builder().seed(3).ef_construction(200).build(base, vals);
    bool failed = false;
    try {
        map.insert(more, more_vals, 200);
    } catch (const Error& e) {
        failed = e.status == IDB_ERR_CAPACITY;
        if (!failed) { std::printf("FAIL: status %d (%s)\n", (int)e.status, e.what()); return 1; }
    }
    if (!failed) { std::puts("FAIL: the insert did not fail"); return 1; }
    const size_t n = map.iter().size();
    if (n <= 500 || n >= 6000 || map.values.size() != n) {
        std::printf("FAIL: %zu points, %zu values after the failed insert\n", n, map.values.size());
        return 1;
    }
    const Point& last = more[n - 501];
    Search s;
    auto items = map.search(last, s);
    if (items.empty() || items[0].pid.raw != n - 1 || items[0].point->v != last.v || *items[0].value != more_vals[n - 501]) {
        std::puts("FAIL: the last kept point is not found with its point and value");
        return 1;
    }
    for (const auto& it : items)
        if (it.pid.raw >= n) { std::puts("FAIL: PointId past the index"); return 1; }
    std::printf("OK %zu\n", n);
    return 0;
}
