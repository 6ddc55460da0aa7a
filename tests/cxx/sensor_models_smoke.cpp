// sensor_models_smoke.cpp -- the C++ facade's stereo and perfect sensor processors (include/gem_b200/elevation_map.hpp).
// One organised 4 x 3 stereo cloud and one perfect point through ElevationMap::add (PCL records), checked against the
// model restated here, and the argument checks of the sensor model.  Prints "sensor models ok".
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <vector>

#include "gem_b200/elevation_map.hpp"

// StereoSensorProcessor.cpp:78-89 as include/gem_b200.h defines it (no rotation variance, sensor_jacobian = e_z: the
// height variance is vN)
static float stereo_vn(const gem_b200::StereoSensorProcessor &s, float z, int idx)
{
    const int row = s.cloud_width ? idx / s.cloud_width : 0, col = s.cloud_width ? idx % s.cloud_width : idx;
    const double disp = s.depth_to_disparity_factor / (double)z;
    const double a = s.depth_to_disparity_factor / (disp * disp);
    const double sj = ((s.p_3 * disp) + s.p_4) - (double)col;
    const double si = (double)(240 - row);
    return (float)((a * a) * ((((s.p_5 * disp) + s.p_2) * std::sqrt(sj * sj + si * si)) + s.p_1));
}

int main()
{
    const int L = 64;
    const float res = 0.1f;
    gem_b200::ElevationMap map(L, res, 2.5f, 0.7f, false);
    int failures = 0;
    gem_b200::StereoSensorProcessor stereo; // aslam.yaml
    stereo.p_1 = 0.03287; stereo.p_2 = -0.0001276; stereo.p_3 = 0.4850; stereo.p_4 = 399.1046; stereo.p_5 = 0.000006735;
    stereo.lateral_factor = 0.001376915; stereo.depth_to_disparity_factor = 47.3;
    stereo.cloud_width = 4;
    const double T[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    // 12 points, one per cell (0.3 m apart), at depths 0.5 .. 1.6 m
    std::vector<gem_b200::PointXYZRGBICT> cloud(12);
    for (int i = 0; i < 12; i++) {
        std::memset(&cloud[i], 0, sizeof cloud[i]);
        cloud[i].x = 0.3f * (float)(i % 4) - 0.45f;
        cloud[i].y = 0.3f * (float)(i / 4) - 0.45f;
        cloud[i].z = 0.5f + 0.1f * (float)i;
    }
    map.add(cloud.data(), cloud.size(), gem_b200::makeFrame(T, stereo));
    std::vector<float> var((size_t)L * L), elev((size_t)L * L);
    if (gem_get_layer(map.handle(), GEM_LAYER_VARIANCE, var.data()) || gem_get_layer(map.handle(), GEM_LAYER_ELEVATION, elev.data())) return 1;
    int found = 0;
    for (int i = 0; i < 12; i++) {
        const float vn = stereo_vn(stereo, cloud[i].z, i);
        const float want = (double)vn < 0.0001 ? (float)0.0001 : vn; // gpu.cu:533-534
        for (size_t c = 0; c < var.size(); c++)
            if (elev[c] == cloud[i].z) { found++; if (var[c] != want) { failures++; std::printf("point %d: var %.9g, want %.9g\n", i, var[c], want); } }
    }
    if (found != 12) failures++;
    // perfect: zero variance (floored), window +-inf whatever the base height
    gem_b200::ElevationMap pmap(L, res, 2.5f, 0.7f, false);
    gem_b200::PointXYZRGBICT p;
    std::memset(&p, 0, sizeof p);
    p.x = 0.05f; p.y = 0.05f; p.z = 100.0f;
    pmap.add(&p, 1, gem_b200::makeFrame(T, gem_b200::PerfectSensorProcessor{}, 1e6));
    if (gem_get_layer(pmap.handle(), GEM_LAYER_VARIANCE, var.data()) || gem_get_layer(pmap.handle(), GEM_LAYER_ELEVATION, elev.data())) return 1;
    int nperfect = 0;
    for (size_t c = 0; c < var.size(); c++)
        if (elev[c] == 100.0f) { nperfect++; if (var[c] != (float)0.0001) failures++; }
    if (nperfect != 1) failures++;
    // an unknown model or a negative width is refused, and nothing is written
    gem_frame bad = gem_b200::makeFrame(T, stereo);
    bad.sensor.type = 4;
    if (gem_add_cloud_pcl_host(map.handle(), cloud.data(), 12, &bad) != GEM_ERR_INVALID) failures++;
    bad.sensor.type = GEM_SENSOR_STEREO;
    bad.sensor.cloud_width = -1;
    if (gem_add_cloud_pcl_host(map.handle(), cloud.data(), 12, &bad) != GEM_ERR_INVALID) failures++;
    std::printf("failures=%d\n", failures);
    if (failures) return 1;
    std::printf("sensor models ok\n");
    return 0;
}
