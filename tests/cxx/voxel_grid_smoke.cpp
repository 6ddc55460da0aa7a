// voxel_grid_smoke.cpp -- the C++ facade's VoxelGrid pre-filter (include/gem_b200/elevation_map.hpp voxelGrid).  The clouds
// live in pinned host memory from gem_host_alloc, which the device reads and writes through unified addressing, so the
// program needs nothing but libgem_b200.  Prints "voxel grid ok" when a small filter.launch call behaves as f9 defines it.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>

#include "gem_b200/elevation_map.hpp"

int main()
{
    gem_b200::ElevationMap map(64, 0.1f, 2.5f, 0.7f, false);
    void *a = nullptr, *b = nullptr;
    if (gem_host_alloc(&a, 6 * 16) || gem_host_alloc(&b, 6 * 16)) return 1;
    float *in = static_cast<float *>(a), *out = static_cast<float *>(b);
    // two points in one 0.1 m voxel, one in another, one NaN, one beyond the x limit, one infinite intensity
    const float pts[6][4] = {{0.01f, 0.02f, 0.03f, 10.0f}, {0.05f, 0.06f, 0.07f, 20.0f}, {0.35f, 0.02f, 0.03f, 5.0f},
                             {std::nanf(""), 0.0f, 0.0f, 1.0f}, {12.0f, 0.0f, 0.0f, 1.0f}, {-0.45f, 0.0f, 0.0f, INFINITY}};
    std::memcpy(in, pts, sizeof pts);
    std::memset(out, 0xFF, 6 * 16);
    gem_voxel_grid_params p{};
    p.leaf_size[0] = p.leaf_size[1] = p.leaf_size[2] = 0.1f;
    p.field = GEM_VOXEL_FIELD_X;
    p.limit_min = -10.0;
    p.limit_max = 10.0;
    int failures = 0;
    const gem_voxel_grid_info q = map.voxelGrid(in, 6, p, nullptr, 0); // size query
    const gem_voxel_grid_info r = map.voxelGrid(in, 6, p, out, 6);
    if (q.count != 3 || r.count != 3 || r.used != 4 || r.passthrough != 0) failures++;
    // ascending voxel order: (-0.45, 0, 0), then the two-point voxel, then (0.35, ...)
    const float sx = 0.0f + 0.01f + 0.05f, si = 0.0f + 10.0f + 20.0f;
    if (out[0] != -0.45f || !std::isinf(out[3]) || out[4] != sx / 2.0f || out[7] != si / 2.0f || out[8] != 0.35f) failures++;
    bool threw = false;
    try {
        map.voxelGrid(in, 6, p, in + 4, 6); // overlapping ranges
    } catch (const std::runtime_error &) {
        threw = true;
    }
    if (!threw) failures++;
    gem_host_free(a);
    gem_host_free(b);
    std::printf("count=%d used=%d failures=%d\n", r.count, r.used, failures);
    if (failures == 0) std::printf("voxel grid ok\n");
    return failures == 0 ? 0 : 1;
}
