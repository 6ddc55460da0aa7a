// costmap_ingest_smoke.cpp -- the C++ facade's costmap plugins fed from their messages (include/gem_b200/elevation_map.hpp
// gridMapMsgParse / gridMapLayerFromFields / ElevationMapLayer / PointMapLayer; DESIGN.md f18).
//   costmap_ingest_smoke <out_prefix>
// Serialises a 20 x 12 grid_map_msgs/GridMap (layers elevation, traver; start index (3, 30)) into a pageable buffer and
// feeds it to an ElevationMapLayer (a second message while one is pending is dropped), marking a 40 x 30 window of
// 0.1 m; builds a 500-point PointXYZRGBICT PointCloud2 in pinned memory and feeds it to a PointMapLayer, marked twice.
// Writes <out_prefix>.msg.bin, .elev.bin (the elevation layer's grid), .cloud.bin and .point.bin (the point layer's grid).
// Prints "costmap ingest ok" with the marks.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "gem_b200/elevation_map.hpp"

static bool spit(const std::string &path, const void *b, size_t n)
{
    FILE *f = std::fopen(path.c_str(), "wb");
    if (!f) return false;
    const bool ok = n == 0 || std::fwrite(b, 1, n, f) == n;
    return std::fclose(f) == 0 && ok;
}

struct Writer {
    std::vector<uint8_t> b;
    void put(const void *p, size_t n) { b.insert(b.end(), (const uint8_t *)p, (const uint8_t *)p + n); }
    void u32(uint32_t v) { put(&v, 4); }
    void f64(double v) { put(&v, 8); }
    void str(const std::string &s) { u32((uint32_t)s.size()); put(s.data(), s.size()); }
};

// the deserialised message's fields, as roscpp's grid_map_msgs::GridMap names them
struct Dim { std::string label; uint32_t size, stride; };
struct Layout { std::vector<Dim> dim; uint32_t data_offset; };
struct Array { Layout layout; std::vector<float> data; };
struct Position { double x, y, z; };
struct Pose { Position position; };
struct Info { double resolution, length_x, length_y; Pose pose; };
struct GridMapMsg {
    Info info;
    std::vector<std::string> layers;
    std::vector<Array> data;
    uint16_t outer_start_index, inner_start_index;
};

int main(int argc, char **argv)
{
    if (argc != 2) return 2;
    const std::string prefix = argv[1];
    gem_b200::ElevationMap map(64, 0.1f, 2.5f, 0.7f, false);
    const int SX = 20, SY = 12;
    GridMapMsg m;
    m.info = Info{0.1, SX * 0.1 + 0.02, SY * 0.1, Pose{Position{0.55, -0.35, 0.0}}};
    m.layers = {"elevation", "traver"};
    m.outer_start_index = 3;
    m.inner_start_index = 30;
    for (int k = 0; k < 2; k++) {
        Array a;
        a.layout.dim = {Dim{"column_index", (uint32_t)SY, (uint32_t)(SX * SY)}, Dim{"row_index", (uint32_t)SX, (uint32_t)SX}};
        a.layout.data_offset = 0;
        for (int i = 0; i < SX * SY; i++) a.data.push_back(i % 17 == 0 ? NAN : (float)((i * 37 + k) % 100) / 100.0f);
        m.data.push_back(a);
    }
    Writer w;
    w.u32(1); w.u32(1700000000); w.u32(5); w.str("odom");
    w.f64(m.info.resolution); w.f64(m.info.length_x); w.f64(m.info.length_y);
    w.f64(m.info.pose.position.x); w.f64(m.info.pose.position.y); w.f64(0.0);
    w.f64(0.0); w.f64(0.0); w.f64(0.0); w.f64(1.0);
    w.u32(2); for (const auto &n : m.layers) w.str(n);
    w.u32(1); w.str("elevation");
    w.u32(2);
    for (const auto &a : m.data) {
        w.u32(2);
        for (const auto &d : a.layout.dim) { w.str(d.label); w.u32(d.size); w.u32(d.stride); }
        w.u32(0); w.u32((uint32_t)a.data.size()); w.put(a.data.data(), 4 * a.data.size());
    }
    uint16_t st[2] = {m.outer_start_index, m.inner_start_index};
    w.put(st, 4);

    const gem_grid_map_layer g = gem_b200::ElevationMap::gridMapMsgParse(w.b.data(), w.b.size());
    gem_grid_map_layer h;
    const float *floats = nullptr;
    bool ok = gem_b200::gridMapLayerFromFields(m, "traver", h, &floats) && floats == m.data[1].data.data();
    ok = ok && g.resolution == h.resolution && g.position_x == h.position_x && g.position_y == h.position_y &&
         g.length_x == h.length_x && g.length_y == h.length_y && g.size_x == h.size_x && g.size_y == h.size_y && g.size_x == SX &&
         g.size_y == SY && g.start_x == h.start_x && g.start_y == h.start_y && g.floats == h.floats && h.offset == 0 &&
         g.column_major == h.column_major;

    const gem_costmap_window win{-1.5, -1.5, 0.1, 40, 30};
    gem_b200::PinnedBytes elev(40 * 30, 0), point(40 * 30, 255);
    gem_b200::ElevationMapLayer el(map, 0.5);
    const gem_costmap_marks none = el.updateBounds(win, elev.data());
    ok = ok && none.marked == 0 && el.onMessage(w.b.data(), w.b.size()) && !el.onMessage(w.b.data(), w.b.size()) && el.available();
    const gem_costmap_marks me = el.updateBounds(win, elev.data());
    ok = ok && !el.available() && el.updateBounds(win, elev.data()).marked == 0;

    const int N = 500;
    std::vector<gem_b200::PointXYZRGBICT, gem_b200::PinnedAllocator<gem_b200::PointXYZRGBICT>> cloud(N);
    for (int i = 0; i < N; i++) {
        gem_b200::PointXYZRGBICT &p = cloud[i];
        std::memset(&p, 0, sizeof p);
        p.x = -1.4f + 0.0071f * (float)((i * 13) % 400);
        p.y = -1.4f + 0.0093f * (float)((i * 7) % 300);
        p.z = 0.1f * (float)(i % 5);
        p.pad = 1.0f;
        p.b = (unsigned char)i; p.g = 2; p.r = 3; p.a = 255;
        p.covariance = 0.01f; p.intensity = (float)i;
        p.travers = (float)((i * 29) % 100) / 100.0f;
    }
    gem_b200::PointCloud2Layout lay(N, 1, 32, 32 * N);
    const char *names[7] = {"x", "y", "z", "rgb", "intensity", "covariance", "travers"};
    const unsigned offs[7] = {0, 4, 8, 16, 24, 20, 28};
    for (int k = 0; k < 7; k++) lay.addField(names[k], offs[k], GEM_PF_FLOAT32, 1);
    gem_b200::PointMapLayer pl(map, 0.5);
    ok = ok && pl.updateBounds(win, point.data()).marked == 0;
    pl.onMessage(lay, cloud.data(), 32ull * N);
    gem_costmap_marks mp = pl.updateBounds(win, point.data());
    mp = pl.updateBounds(win, point.data());
    ok = ok && pl.points() == N && std::memcmp(pl.records(), cloud.data(), 32ull * N) == 0;

    ok = ok && spit(prefix + ".msg.bin", w.b.data(), w.b.size()) && spit(prefix + ".elev.bin", elev.data(), elev.size()) &&
         spit(prefix + ".cloud.bin", cloud.data(), 32ull * N) && spit(prefix + ".point.bin", point.data(), point.size());
    if (!ok) return 1;
    std::printf("costmap ingest ok elev=%lld,%lld,%.17g,%.17g,%.17g,%.17g point=%lld,%lld\n", me.marked, me.lethal, me.min_x, me.min_y,
                me.max_x, me.max_y, mp.marked, mp.lethal);
    return 0;
}
