// mls_smoke.cpp -- the C++ facade's MLS densification (include/gem_b200/elevation_map.hpp mlsUpsample).  The records live
// in pinned host memory from gem_host_alloc, which the device reads and writes through unified addressing, so the program
// needs nothing but libgem_b200.  Prints "mls ok" when a small patch behaves as f10 defines it.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>

#include "gem_b200/elevation_map.hpp"

int main()
{
    gem_b200::ElevationMap map(64, 0.1f, 2.5f, 0.7f, false);
    const int N = 49, CAP = 4096;
    void *a = nullptr, *b = nullptr;
    if (gem_host_alloc(&a, N * sizeof(gem_b200::PointXYZRGBICT)) || gem_host_alloc(&b, CAP * sizeof(gem_b200::PointXYZRGBICT))) return 1;
    gem_b200::PointXYZRGBICT *in = static_cast<gem_b200::PointXYZRGBICT *>(a), *out = static_cast<gem_b200::PointXYZRGBICT *>(b);
    // a 7 x 7 lattice at 0.1 m on the plane z = 1: 49 neighbours for the centre, every point fitted by order 5
    for (int i = 0; i < N; i++) {
        gem_b200::PointXYZRGBICT &p = in[i];
        std::memset(&p, 0, sizeof p);
        p.x = 0.1f * (float)(i % 7 - 3);
        p.y = 0.1f * (float)(i / 7 - 3);
        p.z = 1.0f;
        p.pad = 1.0f;
        p.b = 10; p.g = 20; p.r = 30; p.a = 0;
        p.travers = 0.5f;
    }
    int failures = 0;
    gem_mls_params none = gem_b200::ElevationMap::gemMlsParams();
    none.upsampling = GEM_MLS_NONE;
    const gem_mls_info q = map.mlsUpsample(in, N, none, nullptr, 0); // size query
    const gem_mls_info r = map.mlsUpsample(in, N, none, out, CAP);
    if (q.count != N || r.count != N || r.processed != N || r.skipped != 0 || r.max_neighbours < 21) failures++;
    // a plane is its own MLS surface: every output lies on z = 1 within float rounding, carries the colour with a = 0xff
    for (int i = 0; i < N; i++)
        if (std::fabs(out[i].z - 1.0f) > 1e-5f || out[i].r != 30 || out[i].a != 0xff || out[i].travers != 0.5f) failures++;
    const gem_mls_info d = map.mlsUpsample(in, N, gem_b200::ElevationMap::gemMlsParams(7), out, CAP);
    if (d.count <= N || d.count > CAP) failures++;
    for (long long i = 0; i < d.count && i < CAP; i++)
        if (std::fabs(out[i].z - 1.0f) > 1e-5f) failures++;
    bool threw = false;
    try {
        map.mlsUpsample(in, N, none, in + 3, N); // overlapping ranges
    } catch (const std::runtime_error &) {
        threw = true;
    }
    if (!threw) failures++;
    gem_host_free(a);
    gem_host_free(b);
    std::printf("count=%lld dense=%lld fitted=%d failures=%d\n", r.count, d.count, r.fitted, failures);
    if (failures == 0) std::printf("mls ok\n");
    return failures == 0 ? 0 : 1;
}
