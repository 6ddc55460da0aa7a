// colour_lookup_smoke.cpp -- the C++ facade's colour lookup mode (include/gem_b200/elevation_map.hpp setColourLookup;
// DESIGN.md f19).
//   colour_lookup_smoke <input> <out_prefix>
// <input>: T map<-sensor (16 doubles), T_camera (12), T_lidar (16), the position (3 floats), n (int32) and n float4
// {x, y, z, intensity}, width and height (int32), then the BGR8 image (height rows of 3 * width bytes).
// Checks that a mode other than IMAGE or NODE throws, then adds the cloud as a PointCloud2 with the image in NODE mode
// on a 200 x 0.1 m map with the laser model, and writes <out_prefix>.layers.bin: the nine layers fuse() exports.
// Prints "colour lookup ok".
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "gem_b200/elevation_map.hpp"

static bool slurp(const char *path, std::vector<uint8_t> &b)
{
    FILE *f = std::fopen(path, "rb");
    if (!f) return false;
    uint8_t buf[1 << 16];
    size_t k;
    while ((k = std::fread(buf, 1, sizeof buf, f)) > 0) b.insert(b.end(), buf, buf + k);
    return std::fclose(f) == 0;
}

int main(int argc, char **argv)
{
    if (argc != 3) return 2;
    std::vector<uint8_t> in;
    if (!slurp(argv[1], in)) return 3;
    size_t at = 0;
    auto take = [&](void *dst, size_t n) {
        if (at + n > in.size()) throw std::runtime_error("short input");
        std::memcpy(dst, in.data() + at, n);
        at += n;
    };
    double T[16];
    gem_camera_image img{};
    float pos[3];
    int32_t n = 0, W = 0, H = 0;
    take(T, sizeof T);
    take(img.T_camera, sizeof img.T_camera);
    take(img.T_lidar, sizeof img.T_lidar);
    take(pos, sizeof pos);
    take(&n, 4);
    std::vector<float> xyzi((size_t)n * 4);
    take(xyzi.data(), xyzi.size() * 4);
    take(&W, 4);
    take(&H, 4);
    std::vector<uint8_t> bgr((size_t)W * H * 3);
    take(bgr.data(), bgr.size());

    gem_b200::ElevationMap map(200, 0.1f, 2.5f, 0.7f, false);
    bool refused = false;
    try {
        map.setColourLookup(2);
    } catch (const std::runtime_error &) {
        refused = true;
    }
    if (!refused) return 4;
    map.setColourLookup(GEM_COLOUR_LOOKUP_NODE);

    gem_b200::PointCloud2Layout lay((unsigned)n, 1, 16, 16u * (unsigned)n);
    lay.addField("x", 0, GEM_PF_FLOAT32, 1);
    lay.addField("y", 4, GEM_PF_FLOAT32, 1);
    lay.addField("z", 8, GEM_PF_FLOAT32, 1);
    lay.addField("intensity", 12, GEM_PF_FLOAT32, 1);
    std::memcpy(img.encoding, "bgr8", 5);
    img.width = W;
    img.height = H;
    img.step = 3 * W;
    img.data = bgr.data();
    const gem_frame f = gem_b200::makeFrame(T, gem_b200::LaserSensorProcessor());
    map.move(pos);
    map.addPointCloud2HostAsync(lay, xyzi.data(), (unsigned long long)xyzi.size() * 4, &img, f);
    gem_b200::Layers out;
    map.fuse(out);
    FILE *o = std::fopen((std::string(argv[2]) + ".layers.bin").c_str(), "wb");
    if (!o) return 5;
    for (const auto *v : {&out.elevation, &out.variance, &out.rough, &out.slope, &out.traver, &out.color_r, &out.color_g,
                          &out.color_b, &out.intensity})
        if (std::fwrite(v->data(), 4, v->size(), o) != v->size()) return 6;
    if (std::fclose(o) != 0) return 7;
    std::printf("colour lookup ok: %d points\n", n);
    return 0;
}
