// Hnsw::remove / HnswMap::remove of the host mirror header: the new PointIds are the ABI's (x minus the removed ids below x), and
// points_ / values follow them, so a search for a surviving point finds it with its own value.  Prints the new ids, one per line, for
// the Python test to compare with the ABI's.
#include <cstdio>
#include <random>
#include <string>

#include "../../instant-distance_b200/cpp/instant_distance.hpp"

using namespace instant_distance;

int main() {
    std::mt19937 rng(9);
    std::uniform_real_distribution<float> u(0.f, 1.f);
    std::vector<Point> pts;
    std::vector<std::string> vals;
    for (int i = 0; i < 800; ++i) {
        Point p;
        for (int d = 0; d < 12; ++d) p.v.push_back(u(rng));
        pts.push_back(p);
        vals.push_back("v" + std::to_string(i));
    }
    auto map = Hnsw::builder().seed(4).build(pts, vals);
    std::vector<PointId> gone;
    for (uint32_t x = 0; x < 800; x += 3) gone.push_back(PointId{x});
    const std::vector<Point> before = map.iter();
    const std::vector<std::string> vals_before = map.values;
    auto new_ids = map.remove(gone, 100);
    if (new_ids.size() != 800 || map.iter().size() != 800 - gone.size() || map.values.size() != map.iter().size()) {
        std::puts("FAIL: sizes");
        return 1;
    }
    uint32_t next = 0;
    for (uint32_t x = 0; x < 800; ++x) {
        if (x % 3 == 0) {
            if (new_ids[x]) { std::puts("FAIL: a removed point kept a PointId"); return 1; }
            continue;
        }
        if (!new_ids[x] || new_ids[x]->raw != next) { std::printf("FAIL: new id of %u\n", x); return 1; }
        if (map.iter()[next].v != before[x].v || map.values[next] != vals_before[x]) { std::printf("FAIL: point / value %u\n", x); return 1; }
        ++next;
    }
    Search s;
    auto items = map.search(before[1], s);
    if (items.empty() || items[0].distance != 0.f || *items[0].value != vals_before[1]) { std::puts("FAIL: search"); return 1; }
    std::puts("OK");
    return 0;
}
