// costmap_publish_smoke.cpp -- the C++ facade's costmap topics and footprint clearing (include/gem_b200/elevation_map.hpp
// rosCostmap / rosFootprint / costmapFootprint / CostmapPublisher; DESIGN.md f17).
//   costmap_publish_smoke <out_prefix>
// A 75 x 75 master grid holding (7 i + 3) mod 256 at cell i, in pinned memory (gem_host_alloc; the device reads it
// through unified addressing), published as full, update, none and forced full, then the footprint message and the
// footprint cleared in a FREE-initialised copy as the layer grid.  Each message goes to <out_prefix>.<k>.bin, the layer
// grid to <out_prefix>.layer.bin.  Prints "costmap publish ok" and the kinds.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "gem_b200/elevation_map.hpp"

template <class Buffer> static bool spit(const std::string &path, const Buffer &b, size_t n)
{
    FILE *f = std::fopen(path.c_str(), "wb");
    if (!f) return false;
    const bool ok = n == 0 || std::fwrite(&b[0], 1, n, f) == n;
    return std::fclose(f) == 0 && ok;
}

int main(int argc, char **argv)
{
    if (argc != 2) return 2;
    const std::string prefix = argv[1];
    const int S = 75;
    gem_b200::ElevationMap map(64, 0.1f, 2.5f, 0.7f, false);
    void *mas = nullptr, *lay = nullptr;
    if (gem_host_alloc(&mas, S * S) || gem_host_alloc(&lay, S * S)) return 1;
    unsigned char *master = static_cast<unsigned char *>(mas), *layer = static_cast<unsigned char *>(lay);
    for (int i = 0; i < S * S; i++) master[i] = (unsigned char)((7 * i + 3) % 256);
    std::memset(layer, 0, S * S);
    const gem_costmap_window w{-7.45, -7.45, 0.2, S, S};
    const gem_ros_header h{5, 6, 7, "odom"};
    gem_b200::CostmapPublisher pub;
    gem_b200::PinnedBytes msg;
    bool ok = true;
    int kinds[4] = {-1, -1, -1, -1};
    size_t n = map.rosCostmap(h, w, master, pub.state, msg, &kinds[0]);
    ok = ok && spit(prefix + ".0.bin", msg, n);
    pub.updateBounds(3, 20, 4, 9);
    n = map.rosCostmap(h, w, master, pub.state, msg, &kinds[1]);
    ok = ok && spit(prefix + ".1.bin", msg, n);
    n = map.rosCostmap(h, w, master, pub.state, msg, &kinds[2]);
    ok = ok && n == 0 && spit(prefix + ".2.bin", msg, n);
    pub.updateBounds(0, 1, 0, 1);
    n = map.rosCostmap(h, w, master, pub.state, msg, &kinds[3], true);
    ok = ok && spit(prefix + ".3.bin", msg, n);
    const std::vector<double> fp = {-0.64, -0.40, -0.64, 0.40, 0.64, 0.40, 0.64, -0.40};
    n = map.rosFootprint(h, fp, 0.03, -0.02, 0.7, msg);
    ok = ok && spit(prefix + ".footprint.bin", msg, n);
    const gem_costmap_marks mk = map.costmapFootprint(w, fp, 0.03, -0.02, 0.7, layer);
    map.sync();
    ok = ok && spit(prefix + ".layer.bin", layer, (size_t)(S * S));
    gem_host_free(mas);
    gem_host_free(lay);
    if (!ok) return 1;
    std::printf("costmap publish ok kinds=%d,%d,%d,%d marked=%lld bounds=%.17g,%.17g,%.17g,%.17g\n", kinds[0], kinds[1], kinds[2], kinds[3],
                mk.marked, mk.min_x, mk.min_y, mk.max_x, mk.max_y);
    return 0;
}
