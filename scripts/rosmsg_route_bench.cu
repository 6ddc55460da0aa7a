// rosmsg_route_bench.cu -- the two routes for grid_map's layer data (DESIGN.md f15), timed in one run on the c1, c3 and
// c2 map shapes (L = 200, 512, 1024) of a random map state, with a message that starts one byte past a 16-byte
// boundary and frame_id "map":
//   single   k_ros_grid_map: one pass from the map into the message at its misaligned offsets (the library's kernel);
//   simple   k_export_colmajor into device scratch, then one cudaMemcpyAsync per layer to its misaligned offset;
// each into device memory and into pinned host memory, and for pinned memory also
//   staged   the single pass into a device buffer at the same 16-byte phase, then one DMA copy of the message.
// The payload bytes of every route are checked equal.  CUDA events around each route, median of 20 after 3 warm-ups,
// the routes alternating within each iteration.  Prints one JSON line with the GPU name and the power limit.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -fmad=false -std=c++17 -o build/rosmsg_route_bench scripts/rosmsg_route_bench.cu
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../gem_b200/csrc/gem_kernels.cuh"
#include "../gem_b200/csrc/gem_rosmsg.cuh"

using namespace gem;

#define CK(x)                                                                                   \
    do {                                                                                        \
        cudaError_t e_ = (x);                                                                   \
        if (e_ != cudaSuccess) {                                                                \
            std::fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
            std::exit(1);                                                                       \
        }                                                                                       \
    } while (0)

__device__ __forceinline__ uint32_t hash32(uint32_t x)
{
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}
// a random map state: a fifth of the cells empty (-10), a few NaN traversabilities, colours and intensity bits at random
__global__ void k_fill(MapLayers ml, size_t n)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t a = hash32((uint32_t)i * 4 + 1), b = hash32((uint32_t)i * 4 + 2), c = hash32((uint32_t)i * 4 + 3);
        Cell &cl = ml.cell[i];
        cl.elev = (a % 5 == 0) ? -10.0f : (float)(a & 0xffff) * 1e-4f - 3.0f;
        cl.var = (float)(b & 0xfff) * 1e-5f;
        cl.inten = c;
        cl.rgb = b >> 8;
        ml.traver_out[i] = (c % 97 == 0) ? __int_as_float(0x7fc00000) : (float)(c & 0xff) / 255.0f;
        ml.rough[i] = (float)(a >> 20) * 1e-3f;
        ml.slope[i] = (float)(b >> 20) * 1e-3f;
    }
}

static double median(std::vector<float> v)
{
    std::sort(v.begin(), v.end());
    return v[v.size() / 2];
}

int main()
{
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    std::string power = "unknown";
    if (FILE *p = popen("nvidia-smi --query-gpu=power.limit --format=csv,noheader 2>/dev/null", "r")) {
        char buf[64] = {0};
        if (std::fgets(buf, sizeof buf, p)) power = std::string(buf, strcspn(buf, "\n"));
        pclose(p);
    }
    cudaStream_t st;
    CK(cudaStreamCreate(&st));
    std::printf("{\"gpu\": \"%s\", \"power_limit\": \"%s\", \"shapes\": [", prop.name, power.c_str());
    const int Ls[3] = {200, 512, 1024};
    for (int si = 0; si < 3; si++) {
        const int L = Ls[si];
        const size_t n = (size_t)L * L;
        const long long fid = 3, size = 737 + fid + 36ll * (long long)n, layer0 = 277 + fid, stride = 57 + 4ll * (long long)n;
        MapLayers ml{};
        CK(cudaMalloc(&ml.cell, n * sizeof(Cell)));
        CK(cudaMalloc(&ml.traver_out, n * 4));
        CK(cudaMalloc(&ml.rough, n * 4));
        CK(cudaMalloc(&ml.slope, n * 4));
        ml.traver = ml.traver_out;
        ml.lowest = ml.traver_out;
        k_fill<<<1024, 256, 0, st>>>(ml, n);
        CK(cudaGetLastError());
        float *scratch;
        unsigned char *dev_a, *dev_b, *stage, *pin_a, *pin_b, *pin_c;
        CK(cudaMalloc(&scratch, 9 * n * 4));
        CK(cudaMalloc(&dev_a, size + 16)); CK(cudaMalloc(&dev_b, size + 16)); CK(cudaMalloc(&stage, size + 16));
        CK(cudaMallocHost(&pin_a, size + 16)); CK(cudaMallocHost(&pin_b, size + 16)); CK(cudaMallocHost(&pin_c, size + 16));
        CK(cudaMemsetAsync(dev_a, 0, size + 16, st)); CK(cudaMemsetAsync(dev_b, 0, size + 16, st));
        CK(cudaMemsetAsync(stage, 0, size + 16, st));
        std::memset(pin_a, 0, size + 16); std::memset(pin_b, 0, size + 16); std::memset(pin_c, 0, size + 16);
        const int nch = (L + 31) / 32;
        const dim3 grid(nch, nch);
        auto single = [&](unsigned char *msg) { k_ros_grid_map<<<grid, 256, 0, st>>>(ml, L, msg + layer0, stride); };
        auto simple = [&](unsigned char *msg, cudaMemcpyKind kind) {
            k_export_colmajor<<<grid, 256, 0, st>>>(ml, L, scratch);
            for (int k = 0; k < 9; k++)
                CK(cudaMemcpyAsync(msg + layer0 + k * stride, scratch + k * n, n * 4, kind, st));
        };
        auto staged = [&](unsigned char *msg) {
            single(stage + 1);
            CK(cudaMemcpyAsync(msg, stage + 1, size, cudaMemcpyDeviceToHost, st));
        };
        const char *names[5] = {"single_device", "simple_device", "single_pinned", "simple_pinned", "staged_pinned"};
        std::vector<float> t[5];
        cudaEvent_t e0, e1;
        CK(cudaEventCreate(&e0));
        CK(cudaEventCreate(&e1));
        for (int it = 0; it < 23; it++) {
            for (int r0 = 0; r0 < 5; r0++) {
                const int r = (r0 + it) % 5;
                CK(cudaEventRecord(e0, st));
                switch (r) {
                case 0: single(dev_a + 1); break;
                case 1: simple(dev_b + 1, cudaMemcpyDeviceToDevice); break;
                case 2: single(pin_a + 1); break;
                case 3: simple(pin_b + 1, cudaMemcpyDeviceToHost); break;
                case 4: staged(pin_c + 1); break;
                }
                CK(cudaEventRecord(e1, st));
                CK(cudaEventSynchronize(e1));
                float ms;
                CK(cudaEventElapsedTime(&ms, e0, e1));
                if (it >= 3) t[r].push_back(ms);
            }
        }
        CK(cudaGetLastError());
        // the layer data of every route is the same
        std::vector<unsigned char> ha(size + 16), hb(size + 16);
        CK(cudaMemcpy(ha.data(), dev_a, size + 16, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(hb.data(), dev_b, size + 16, cudaMemcpyDeviceToHost));
        bool same = true;
        for (int k = 0; k < 9; k++) {
            const long long o = 1 + layer0 + k * stride;
            same = same && !std::memcmp(ha.data() + o, hb.data() + o, n * 4) && !std::memcmp(ha.data() + o, pin_a + o, n * 4) &&
                   !std::memcmp(ha.data() + o, pin_b + o, n * 4) && !std::memcmp(ha.data() + o, pin_c + o, n * 4);
        }
        std::printf("%s{\"L\": %d, \"message_bytes\": %lld, \"payloads_equal\": %s", si ? ", " : "", L, size, same ? "true" : "false");
        for (int r = 0; r < 5; r++) {
            const double ms = median(t[r]);
            std::printf(", \"%s\": {\"ms\": %.4f, \"GBps\": %.1f}", names[r], ms, (double)(36ll * n) / (ms * 1e6));
        }
        std::printf("}");
        CK(cudaFree(ml.cell)); CK(cudaFree(ml.traver_out)); CK(cudaFree(ml.rough)); CK(cudaFree(ml.slope));
        CK(cudaFree(scratch)); CK(cudaFree(dev_a)); CK(cudaFree(dev_b)); CK(cudaFree(stage));
        CK(cudaFreeHost(pin_a)); CK(cudaFreeHost(pin_b)); CK(cudaFreeHost(pin_c));
        CK(cudaEventDestroy(e0)); CK(cudaEventDestroy(e1));
    }
    std::printf("]}\n");
    CK(cudaStreamDestroy(st));
    return 0;
}
