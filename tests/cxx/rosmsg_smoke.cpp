// rosmsg_smoke.cpp -- the C++ facade's ROS messages (include/gem_b200/elevation_map.hpp rosGridMap / rosOrthomosaic /
// rosVisualPoints / rosCloud / rosSubmap).
//   rosmsg_smoke <records> <out_prefix> <layer_dir>
// builds the L33_opt_move state of tests/rosmsg_cases.py (the moves and the opt_move below, the layers from
// <layer_dir>/layer.<name>.bin), then writes each message to <out_prefix>.<kind>.bin from pinned buffers.  The records
// are read from <records> (raw 32-byte PointXYZRGBICT records) into pinned memory.  Prints "rosmsg ok".
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "gem_b200/elevation_map.hpp"

static std::string slurp(const std::string &path)
{
    std::string s;
    FILE *f = std::fopen(path.c_str(), "rb");
    if (!f) return s;
    char buf[65536];
    size_t k;
    while ((k = std::fread(buf, 1, sizeof buf, f)) > 0) s.append(buf, k);
    std::fclose(f);
    return s;
}

template <class Buffer> static bool spit(const std::string &path, const Buffer &b)
{
    FILE *f = std::fopen(path.c_str(), "wb");
    if (!f) return false;
    const bool ok = std::fwrite(b.data(), 1, b.size(), f) == b.size();
    return std::fclose(f) == 0 && ok;
}

int main(int argc, char **argv)
{
    if (argc != 4) return 2;
    const std::string raw = slurp(argv[1]), prefix = argv[2], dir = argv[3];
    const size_t n = raw.size() / sizeof(gem_b200::PointXYZRGBICT);
    gem_b200::ElevationMap map(33, 0.1f, 2.5f, 0.7f, false);
    const float p0[3] = {0.0f, 0.0f, 0.0f}, p1[3] = {0.75f, 0.42f, 0.0f};
    map.move(p0);
    map.move(p1);
    const char *names[6] = {"elevation", "variance", "intensity", "color_r", "color_g", "color_b"};
    for (int id = 0; id < 6; id++) {
        const std::string layer = slurp(dir + "/layer." + names[id] + ".bin");
        if (layer.size() != 33 * 33 * 4 || gem_set_layer(map.handle(), id, layer.data()) != GEM_OK) return 1;
    }
    const float opt[2] = {1.13f, 0.27f};
    float aligned[2];
    map.optMove(opt, 0.25f, aligned);
    if (gem_compute_features(map.handle()) != GEM_OK) return 1;

    void *rec = nullptr;
    if (gem_host_alloc(&rec, raw.size() + 32)) return 1;
    std::memcpy(rec, raw.data(), raw.size());
    const gem_ros_header h{1, 2, 3, "map"}, empty{0, 0, 0, ""};
    gem_b200::PinnedBytes msg;
    bool ok = true;
    ok = ok && map.rosGridMap(h, msg) == msg.size() && spit(prefix + ".grid_map.bin", msg);
    ok = ok && map.rosOrthomosaic(empty, msg) == msg.size() && spit(prefix + ".orthomosaic.bin", msg);
    ok = ok && map.rosVisualPoints(h, msg) == msg.size() && spit(prefix + ".visual_points.bin", msg);
    ok = ok && map.rosCloud(h, {gem_ros_part{rec, (long long)n}}, msg) == msg.size() && spit(prefix + ".cloud.bin", msg);
    const double pose[7] = {1.0, 2.0, 3.0, 0.0, 0.0, 0.0, 1.0};
    ok = ok && map.rosSubmap(h, rec, n, "keyframe", 8, pose, msg) == msg.size() && spit(prefix + ".submap.bin", msg);
    gem_host_free(rec);
    if (!ok) return 1;
    std::printf("rosmsg ok\n");
    return 0;
}
