// color_octree_smoke.cpp -- the C++ facade's global-map octrees (include/gem_b200/elevation_map.hpp colorOctree,
// globalOctrees).  The split outputs go to pinned host memory from gem_host_alloc, which the device reads and writes
// through unified addressing, so the program needs nothing but libgem_b200.  Prints "color_octree ok" when the streams
// have the sizes their counts give and an empty cloud gives an empty stream.
#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "gem_b200/elevation_map.hpp"

int main()
{
    const int L = 128, N = 60000;
    gem_b200::ElevationMap map(L, 0.1f, 2.5f, 0.7f, false);
    std::vector<gem_b200::PointXYZRGBICT> cloud(N);
    uint64_t s = 13;
    auto rnd = [&s](double lo, double hi) {
        s = s * 6364136223846793005ull + 1442695040888963407ull;
        return lo + (hi - lo) * (double)(s >> 11) / 9007199254740992.0;
    };
    for (auto &p : cloud) {
        p.x = (float)rnd(-6.0, 6.0); p.y = (float)rnd(-7.0, -2.0); p.z = (float)rnd(-0.3, 0.3); p.pad = 1.0f;
        p.r = 200; p.g = 100; p.b = 50; p.a = 255;
        p.covariance = 0; p.intensity = 9.0f; p.travers = 0;
    }
    const double T[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0.2, 0, 0, 0, 1};
    const gem_frame f = gem_b200::makeFrame(T, gem_b200::LaserSensorProcessor());
    float pos[3] = {0.0f, 0.0f, 0.0f}, centre[2], shift[2];
    int start[2];
    map.move(pos, centre, start, shift);
    map.add(cloud.data(), cloud.size(), f);
    gem_b200::Layers layers;
    map.fuse(layers);
    map.snapshot();
    const int grid = map.gridCloud(GEM_GRID_SNAPSHOT, nullptr, 0);
    void *road = nullptr, *obstacle = nullptr;
    const unsigned long long bytes = (unsigned long long)(grid > 0 ? grid : 1) * sizeof(gem_b200::PointXYZRGBICT);
    if (gem_host_alloc(&road, bytes) || gem_host_alloc(&obstacle, bytes)) return 1;
    const gem_b200::GlobalOctrees g = map.globalOctrees(road, (size_t)grid, obstacle, (size_t)grid);
    int failures = 0;
    if (g.road.size() != (size_t)g.roadInfo.bytes || g.roadInfo.bytes != 8ll * g.roadInfo.nodes) failures++;
    if (g.obstacle.size() != (size_t)g.obstacleInfo.bytes || g.obstacleInfo.bytes != 8ll * g.obstacleInfo.nodes) failures++;
    if (g.roadInfo.inserted + g.roadInfo.skipped != g.split.road || g.obstacleInfo.inserted + g.obstacleInfo.skipped != g.split.obstacle)
        failures++;
    gem_octree e{};
    if (!map.colorOctree(nullptr, 0, 0.1, &e).empty() || e.nodes != 0) failures++;
    bool threw = false;
    try {
        map.colorOctree(road, 1, 0.0);
    } catch (const std::runtime_error &) {
        threw = true;
    }
    if (!threw) failures++;
    threw = false;
    try {
        map.colorOctree(road, (size_t)1 << 31, 0.1);   // a count that does not fit the C ABI's int
    } catch (const std::runtime_error &) {
        threw = true;
    }
    if (!threw) failures++;
    gem_host_free(road);
    gem_host_free(obstacle);
    std::printf("grid=%d road=%d/%d nodes obstacle=%d/%d nodes failures=%d\n", grid, g.split.road, g.roadInfo.nodes, g.split.obstacle,
                g.obstacleInfo.nodes, failures);
    if (failures == 0) std::printf("color_octree ok\n");
    return failures == 0 ? 0 : 1;
}
