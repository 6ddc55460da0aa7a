// grid_split_smoke.cpp -- the C++ facade's global-map filter (include/gem_b200/elevation_map.hpp gridCloudSplit), driven
// through size queries only (no device buffers), so the program needs nothing but libgem_b200.  Prints "grid_split ok"
// when the counts agree with the grid cloud.
#include <cstdint>
#include <cstdio>
#include <vector>

#include "gem_b200/elevation_map.hpp"

int main()
{
    const int L = 128, N = 60000;
    gem_b200::ElevationMap map(L, 0.1f, 2.5f, 0.7f, false);
    std::vector<gem_b200::PointXYZRGBICT> cloud(N);
    uint64_t s = 11;
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
    const gem_grid_split st = map.gridCloudSplit(GEM_GRID_SNAPSHOT, 20, 1.0, 0.0, nullptr, 0, nullptr, 0);
    int failures = 0;
    if (grid <= 0 || st.points != grid || st.valid != grid) failures++;
    if (st.road + st.obstacle > grid || st.road + st.obstacle < grid / 2 || !(st.threshold >= st.mean)) failures++;
    std::printf("grid=%d road=%d obstacle=%d mean=%g stddev=%g failures=%d\n", grid, st.road, st.obstacle, st.mean, st.stddev, failures);
    if (failures == 0) std::printf("grid_split ok\n");
    return failures == 0 ? 0 : 1;
}
