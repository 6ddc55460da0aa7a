// prefilter_smoke.cpp -- the C++ facade's pre-filtered add (include/gem_b200/elevation_map.hpp Prefilter,
// addPointsFilteredStream, prefilterInfo) against the C ABI on a second handle.  The cloud lives in pinned host memory
// from gem_host_alloc, which the device reads through unified addressing.  Prints "prefilter ok" when both handles hold
// the same layers and step infos, and the facade refuses what the C ABI refuses.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <vector>

#include "gem_b200/elevation_map.hpp"

int main()
{
    const int L = 64, n = 4000;
    gem_b200::ElevationMap a(L, 0.1f, 2.5f, 0.7f, false), b(L, 0.1f, 2.5f, 0.7f, false);
    void *buf = nullptr;
    if (gem_host_alloc(&buf, (size_t)n * 16)) return 1;
    float *p = static_cast<float *>(buf);
    unsigned s = 12345u;
    for (int i = 0; i < n; i++) {
        for (int c = 0; c < 4; c++) {
            s = s * 1664525u + 1013904223u;
            const float u = (float)(s >> 8) / 16777216.0f;
            p[4 * i + c] = c < 2 ? 6.0f * u - 3.0f : (c == 2 ? 0.5f * u : 255.0f * u);
        }
    }
    const double T[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    const gem_frame f = gem_b200::makeFrame(T, gem_b200::LaserSensorProcessor());
    const gem_b200::ElevationMap::Prefilter pf = gem_b200::ElevationMap::Prefilter::filterKittiLaunch();
    int failures = 0;
    for (int k = 0; k < 3; k++) {
        a.addPointsFilteredStream(p, n, pf, nullptr, nullptr, f);
        if (gem_add_points_filtered_stream(b.handle(), p, n, &pf.c, nullptr, nullptr, &f) != GEM_OK) failures++;
    }
    a.sync();
    b.sync();
    const std::vector<gem_voxel_grid_info> ia = a.prefilterInfo(3);
    gem_voxel_grid_info ib[3];
    if (gem_prefilter_info(b.handle(), ib, 3) != GEM_OK) failures++;
    for (int j = 0; j < 3; j++)
        if (ia[j].count != ib[j].count || ia[j].used != ib[j].used || ia[j].passthrough != ib[j].passthrough) failures++;
    if (!(ia[2].count > 100 && ia[2].count < n)) failures++;
    std::vector<float> la((size_t)L * L), lb((size_t)L * L);
    for (int layer : {GEM_LAYER_ELEVATION, GEM_LAYER_VARIANCE}) {
        if (gem_get_layer(a.handle(), layer, la.data()) || gem_get_layer(b.handle(), layer, lb.data())) return 1;
        if (std::memcmp(la.data(), lb.data(), la.size() * sizeof(float)) != 0) failures++;
    }
    bool threw = false;
    gem_b200::ElevationMap::Prefilter bad = pf;
    bad.c.step[0].leaf_size[1] = 0.0f;
    try {
        a.addPointsFilteredStream(p, n, bad, nullptr, nullptr, f);
    } catch (const std::runtime_error &) {
        threw = true;
    }
    if (!threw) failures++;
    gem_host_free(buf);
    std::printf("count=%d used=%d failures=%d\n", ia[2].count, ia[0].used, failures);
    if (failures == 0) std::printf("prefilter ok\n");
    return failures == 0 ? 0 : 1;
}
