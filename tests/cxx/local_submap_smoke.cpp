// local_submap_smoke.cpp -- the C++ facade's local-submap calls (include/gem_b200/elevation_map.hpp): grid cloud, harvest
// into the device-resident local map, take / clear and the keyframe cut, driven through size queries only (no device
// buffers), so the program needs nothing but libgem_b200.  Prints "local_submap ok" when the sizes agree.
#include <cstdint>
#include <cstdio>
#include <vector>

#include "gem_b200/elevation_map.hpp"

int main()
{
    const int L = 128, N = 60000;
    gem_b200::ElevationMap map(L, 0.1f, 2.5f, 0.7f, false);
    std::vector<gem_b200::PointXYZRGBICT> cloud(N);
    uint64_t s = 7;
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
    int harvested = 0, failures = 0;
    for (int k = 0; k < 4; k++) {
        pos[0] = 0.7f * (float)k;
        map.move(pos, centre, start, shift);
        if (k > 0) {
            std::vector<gem_b200::PointXYZRGBICT> visual;
            harvested += map.harvestToLocalMap(centre, shift, &visual);
            if (visual.size() > (size_t)L * L) failures++;
        }
        map.add(cloud.data(), cloud.size(), f);
        gem_b200::Layers layers;
        map.fuse(layers);
        map.snapshot();
        map.clean();
    }
    const int grid = map.gridCloud(GEM_GRID_SHOWN, nullptr, 0), snap = map.gridCloud(GEM_GRID_SNAPSHOT, nullptr, 0);
    const int local = map.localMapTake(nullptr, 0);
    const int cut = map.cutSubmap(nullptr, 0); // too small: nothing written, nothing taken
    if (cut != local + grid || map.localMapTake(nullptr, 0) != local) failures++;
    if (local <= 0 || local > harvested || grid <= 0 || snap <= 0) failures++; // the ray clean-up ran after the snapshot
    map.localMapClear();
    if (map.localMapTake(nullptr, 0) != 0) failures++;
    std::printf("harvested=%d local=%d grid=%d snapshot=%d cut=%d failures=%d\n", harvested, local, grid, snap, cut, failures);
    if (failures == 0) std::printf("local_submap ok\n");
    return failures == 0 ? 0 : 1;
}
