// pcd_smoke.cpp -- the C++ facade's PCD writer (include/gem_b200/elevation_map.hpp savePcd / formatPcd / pcdHeader).
//   pcd_smoke <records> <out_prefix>
// reads raw 32-byte PointXYZRGBICT records from <records> and writes <out_prefix>.ascii.pcd (host records, one chunk),
// <out_prefix>.chunked.pcd (device-visible records, chunks of 7), <out_prefix>.binary.pcd and <out_prefix>.rgbu.pcd.
// The records live in pinned host memory from gem_host_alloc, which the device reads through unified addressing, so the
// program needs nothing but libgem_b200.  Prints "pcd ok" when the calls behave as f13 defines them.
#include <cstdio>
#include <cstring>
#include <stdexcept>
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

int main(int argc, char **argv)
{
    if (argc != 3) return 2;
    const std::string raw = slurp(argv[1]), prefix = argv[2];
    const size_t n = raw.size() / sizeof(gem_b200::PointXYZRGBICT);
    if (n == 0) return 2;
    gem_b200::ElevationMap map(64, 0.1f, 2.5f, 0.7f, false);
    void *pinned = nullptr;
    if (gem_host_alloc(&pinned, raw.size())) return 1;
    std::memcpy(pinned, raw.data(), raw.size());
    int failures = 0;
    map.savePcd(prefix + ".ascii.pcd", raw.data(), n, false);
    map.savePcd(prefix + ".chunked.pcd", pinned, n, true, false, false, 7);
    map.savePcd(prefix + ".binary.pcd", raw.data(), n, false, true);
    map.savePcd(prefix + ".rgbu.pcd", pinned, n, true, false, true, 5);
    if (slurp(prefix + ".ascii.pcd") != slurp(prefix + ".chunked.pcd")) failures++;
    const std::string bin = slurp(prefix + ".binary.pcd"), head = gem_b200::ElevationMap::pcdHeader((long long)n, true);
    if (bin.size() != head.size() + 28 * n || bin.compare(0, head.size(), head) != 0) failures++;
    // the size query, then a buffer one byte short: nothing is written
    const long long need = map.formatPcd(pinned, n, false, false, nullptr, 0);
    std::vector<char> out((size_t)need + 1, 'S');
    void *pout = nullptr;
    if (gem_host_alloc(&pout, (size_t)need)) return 1;
    std::memset(pout, 'S', (size_t)need);
    if (map.formatPcd(pinned, n, false, false, pout, (size_t)need - 1) != need) failures++;
    for (long long i = 0; i < need; i++)
        if (static_cast<char *>(pout)[i] != 'S') { failures++; break; }
    if (map.formatPcd(pinned, n, false, false, pout, (size_t)need) != need) failures++;
    const std::string ascii = slurp(prefix + ".ascii.pcd");
    if (ascii.compare(ascii.size() - (size_t)need, (size_t)need, static_cast<char *>(pout), (size_t)need) != 0) failures++;
    bool threw = false;
    try {
        map.savePcd(prefix + ".empty.pcd", raw.data(), 0, false); // PCL throws on an empty cloud
    } catch (const std::runtime_error &) {
        threw = true;
    }
    if (!threw || std::fopen((prefix + ".empty.pcd").c_str(), "rb") != nullptr) failures++;
    gem_host_free(pinned);
    gem_host_free(pout);
    std::printf("records=%zu bytes=%lld failures=%d\n", n, need, failures);
    if (failures == 0) std::printf("pcd ok\n");
    return failures == 0 ? 0 : 1;
}
