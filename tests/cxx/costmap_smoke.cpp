// costmap_smoke.cpp -- the C++ facade's navigation costmaps (include/gem_b200/elevation_map.hpp costmapMarkMap,
// costmapMarkPoints, costmapUpdateOrigin, costmapCombine).  The grids and the records live in pinned host memory from
// gem_host_alloc, which the device reads and writes through unified addressing, so the program needs nothing but
// libgem_b200.  Prints "costmap ok" when a small local-costmap update behaves as the layers define it.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>

#include "gem_b200/elevation_map.hpp"

int main()
{
    const int L = 128;
    gem_b200::ElevationMap map(L, 0.1f, 2.5f, 0.7f, false);
    const int S = 75;
    void *lay = nullptr, *mas = nullptr, *pts = nullptr;
    if (gem_host_alloc(&lay, S * S) || gem_host_alloc(&mas, S * S) || gem_host_alloc(&pts, 4 * sizeof(gem_b200::PointXYZRGBICT))) return 1;
    unsigned char *layer = static_cast<unsigned char *>(lay), *master = static_cast<unsigned char *>(mas);
    std::memset(layer, GEM_COST_UNKNOWN, S * S);
    std::memset(master, GEM_COST_FREE, S * S);
    int failures = 0;
    // four records: two in one cell (the later one wins), one off the window, one NaN
    gem_b200::PointXYZRGBICT *p = static_cast<gem_b200::PointXYZRGBICT *>(pts);
    std::memset(p, 0, 4 * sizeof *p);
    p[0].x = 1.12f; p[0].y = 2.12f; p[0].travers = 0.9f;
    p[1].x = 1.15f; p[1].y = 2.15f; p[1].travers = 0.1f;
    p[2].x = -40.0f; p[2].y = 0.0f; p[2].travers = 0.9f;
    p[3].x = std::nanf(""); p[3].y = 1.0f; p[3].travers = 0.9f;
    gem_costmap_window w{-7.5, -7.5, 0.2, S, S};
    const double half = (S - 1 + 0.5) * 0.2 / 2;
    map.costmapUpdateOrigin(w, -7.5 + 0.15, -7.5 - 0.15, GEM_COST_UNKNOWN, layer); // less than a cell: no move
    if (w.origin_x != -7.5) failures++;
    map.costmapUpdateOrigin(w, 1.0 - half, 0.0 - half, GEM_COST_UNKNOWN, layer);
    const gem_costmap_marks mk = map.costmapMarkPoints(pts, 4, w, layer, 0.7);
    map.costmapCombine(GEM_COSTMAP_OVERWRITE, layer, master, S, S, 0, 0, S, S);
    map.sync();
    const int mx = (int)((1.15 - w.origin_x) / 0.2), my = (int)((2.15 - w.origin_y) / 0.2);
    if (mk.marked != 2 || mk.lethal != 1 || layer[my * S + mx] != GEM_COST_LETHAL || master[my * S + mx] != GEM_COST_LETHAL) failures++;
    if (mk.min_x != (double)1.12f || mk.max_y != (double)2.15f) failures++;
    bool threw = false;
    try {
        gem_costmap_window bad{0.0, 0.0, 0.0, S, S};
        map.costmapMarkPoints(pts, 4, bad, layer);
    } catch (const std::runtime_error &) {
        threw = true;
    }
    if (!threw) failures++;
    // the map source: an empty map has no shown cell, so with markUnknown every cell in the window is FREE
    map.sync();
    std::memset(layer, GEM_COST_UNKNOWN, S * S);
    gem_costmap_window lw{-7.0, -7.0, 0.2, S, S}; // holds the whole 12.8 m map
    const gem_costmap_marks mm = map.costmapMarkMap(lw, layer, 0.7, GEM_GRID_SHOWN, false);
    const gem_costmap_marks mu = map.costmapMarkMap(lw, layer, 0.7, GEM_GRID_SHOWN, true);
    if (mm.marked != 0 || mu.marked != (long long)L * L || mu.lethal != 0 || layer[S * S / 2] != GEM_COST_FREE) failures++;
    gem_host_free(lay);
    gem_host_free(mas);
    gem_host_free(pts);
    std::printf("marked=%lld lethal=%lld map marked=%lld/%lld failures=%d\n", mk.marked, mk.lethal, mm.marked, mu.marked, failures);
    if (failures == 0) std::printf("costmap ok\n");
    return failures == 0 ? 0 : 1;
}
