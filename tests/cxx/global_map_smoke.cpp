// global_map_smoke.cpp -- the C++ facade's global map (include/gem_b200/elevation_map.hpp globalMap* / saveSubmaps).
//   global_map_smoke <input> <out_dir/>
// <input>: int32 K, then K times {int32 n, 16 float pose, n 32-byte records}, then int32 k, k x 16 float opt poses,
// float64 resolution.  Pushes the K submaps, updates with the k poses, writes <out_dir>packed.bin (the packed stack),
// <out_dir>poses.bin (every keyframe's pose) and every submap through saveSubmaps; prints "fused=<n>" and
// "global_map ok".
#include <cuda_runtime.h>

#include <cstdio>
#include <string>
#include <vector>

#include "gem_b200/elevation_map.hpp"

int main(int argc, char **argv)
{
    if (argc != 3) return 2;
    FILE *f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    const std::string out = argv[2];
    gem_b200::ElevationMap map(64, 0.1f, 2.5f, 0.7f, false);
    map.globalMapReset();
    int K = 0;
    if (std::fread(&K, 4, 1, f) != 1) return 2;
    for (int s = 0; s < K; s++) {
        int n = 0;
        float pose[16];
        if (std::fread(&n, 4, 1, f) != 1 || std::fread(pose, 4, 16, f) != 16) return 2;
        std::vector<char> rec((size_t)n * 32);
        if (n && std::fread(rec.data(), 32, (size_t)n, f) != (size_t)n) return 2;
        void *d = nullptr;
        if (cudaMalloc(&d, rec.size() + 32) != cudaSuccess) return 1;
        cudaMemcpy(d, rec.data(), rec.size(), cudaMemcpyHostToDevice);
        map.globalMapPush(d, (size_t)n, pose);
        cudaFree(d);
    }
    int k = 0;
    double res = 0.0;
    if (std::fread(&k, 4, 1, f) != 1) return 2;
    std::vector<float> opt((size_t)k * 16);
    if ((k && std::fread(opt.data(), 4, opt.size(), f) != opt.size()) || std::fread(&res, 8, 1, f) != 1) return 2;
    std::fclose(f);
    const int fused = map.globalMapUpdate(opt.data(), k, res);
    long long total = 0;
    const void *all = map.globalMapRecords(&total);
    std::vector<char> host((size_t)total * 32);
    if (total) cudaMemcpy(host.data(), all, host.size(), cudaMemcpyDeviceToHost);
    FILE *g = std::fopen((out + "packed.bin").c_str(), "wb");
    if (!g || std::fwrite(host.data(), 1, host.size(), g) != host.size()) return 1;
    std::fclose(g);
    g = std::fopen((out + "poses.bin").c_str(), "wb");
    for (int i = 0; i <= map.globalMapSubmaps(); i++) {
        float pose[16], centre[2];
        map.globalMapPose(i, pose, centre);
        std::fwrite(pose, 4, 16, g);
    }
    std::fclose(g);
    map.saveSubmaps(out);
    long long sum = 0;
    for (int i = 0; i < map.globalMapSubmaps(); i++) {
        int n = 0;
        map.globalMapSubmap(i, &n);
        sum += n;
    }
    std::printf("fused=%d\n", fused);
    if (sum == total && map.globalMapSubmaps() == K) std::printf("global_map ok\n");
    return 0;
}
