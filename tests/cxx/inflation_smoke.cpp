// inflation_smoke.cpp -- the C++ facade's costmapInflate (include/gem_b200/elevation_map.hpp): a small global-costmap update,
// PointMapLayer's overwrite of two records followed by the inflation of the master at costmap_2d's defaults.  The grids
// live in pinned host memory from gem_host_alloc, read and written by the device through unified addressing.  Prints
// "inflation ok" when the costs around the lethal cell are the ones InflationLayer defines.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>

#include "gem_b200/elevation_map.hpp"

int main()
{
    gem_b200::ElevationMap map(64, 0.1f, 2.5f, 0.7f, false);
    const int S = 40;
    void *lay = nullptr, *mas = nullptr, *pts = nullptr;
    if (gem_host_alloc(&lay, S * S) || gem_host_alloc(&mas, S * S) || gem_host_alloc(&pts, 2 * sizeof(gem_b200::PointXYZRGBICT))) return 1;
    unsigned char *layer = static_cast<unsigned char *>(lay), *master = static_cast<unsigned char *>(mas);
    std::memset(layer, GEM_COST_UNKNOWN, S * S);
    std::memset(master, GEM_COST_FREE, S * S);
    gem_b200::PointXYZRGBICT *p = static_cast<gem_b200::PointXYZRGBICT *>(pts);
    std::memset(p, 0, 2 * sizeof *p);
    p[0].x = 1.01f; p[0].y = 1.01f; p[0].travers = 0.1f; // lethal, cell (10, 10) of a 0.1 m grid from the origin
    p[1].x = 3.05f; p[1].y = 0.55f; p[1].travers = 0.9f; // free
    const gem_costmap_window w{0.0, 0.0, 0.1, S, S};
    const gem_costmap_marks mk = map.costmapMarkPoints(pts, 2, w, layer, 0.7);
    map.costmapCombine(GEM_COSTMAP_OVERWRITE, layer, master, S, S, 0, 0, S, S);
    const gem_costmap_inflation ip{0.55, 10.0, 0.2, 0};
    map.costmapInflate(w, ip, master, 10, 10, 11, 11);
    map.sync();
    int failures = 0;
    if (mk.marked != 2 || master[10 * S + 10] != GEM_COST_LETHAL) failures++;
    // distance 1 and 2 cells (0.1 m, 0.2 m) are within the inscribed radius; 3 cells: 252 * exp(-10 * 0.1) truncated
    if (master[10 * S + 11] != 253 || master[12 * S + 10] != 253) failures++;
    if (master[10 * S + 13] != (unsigned char)(252 * std::exp(-10.0 * (3 * 0.1 - 0.2)))) failures++;
    if (master[10 * S + 17] != GEM_COST_FREE || master[0] != GEM_COST_FREE) failures++; // beyond r = 6
    bool threw = false;
    try {
        const gem_costmap_inflation bad{-1.0, 10.0, 0.2, 0};
        map.costmapInflate(w, bad, master, 0, 0, S, S);
    } catch (const std::runtime_error &) {
        threw = true;
    }
    if (!threw) failures++;
    gem_host_free(lay);
    gem_host_free(mas);
    gem_host_free(pts);
    std::printf("marked=%lld failures=%d\n", mk.marked, failures);
    if (failures == 0) std::printf("inflation ok\n");
    return failures == 0 ? 0 : 1;
}
