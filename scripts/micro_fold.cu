// micro-benchmark of the serial fold step: cycles per record for one warp folding a list, alone on its SM and with
// busy neighbours on the same scheduler.   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -fmad=false -std=c++17 -I gem_b200/csrc -o scripts/micro_fold scripts/micro_fold.cu
#include <cstdio>
#include <vector>
#include "gem_add.cuh"
using namespace gem;

// mode 0: the general path alone (fold_chunk_general); 1: the library's fold_chunk, plain path first.  busy: warps 1..
// of the block spin on ALU work.
__global__ void k_micro(const uint4 *rec, int k, int mode, int busy_iters, float *out, long long *cyc)
{
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (w == 0) {
        CellState s;
        s.elev = 0.3f; s.var = 0.01f; s.src = 0; s.inten = 0; s.rgb = 0; s.ci_dirty = false; s.minh = 0; s.minhv = 0; s.any = false; s.low_old = 0; s.low_idx = 0;
        const long long t0 = clock64();
        for (int c0 = 0; c0 < k; c0 += 32) {
            uint4 r = make_uint4(0, 0, 0, 0);
            if (c0 + lane < k) r = rec[c0 + lane];
            if (mode == 0) { if (fold_chunk_general(s, r, min(32, k - c0))) s.elev += 1.0f; }
            else fold_chunk(s, r, min(32, k - c0), true);
        }
        const long long t1 = clock64();
        if (lane == 0) { out[blockIdx.x] = s.elev + s.var; cyc[blockIdx.x] = t1 - t0; }
    } else {
        float a = (float)threadIdx.x, b = 1.0001f;
        for (int i = 0; i < busy_iters; i++) { a = a * b + 0.5f; b = b * 0.9999f + 1e-4f; }
        if (a == 123.456f) out[0] = a;
    }
}

int main()
{
    const int k = 128;
    std::vector<uint4> h(k);
    for (int i = 0; i < k; i++) {
        float hh = 0.3f + 0.001f * (i % 17), vv = 0.001f + 1e-5f * (i % 5);
        h[i] = make_uint4(i, *(uint32_t *)&hh, *(uint32_t *)&vv, 0x01ffffffu);
    }
    uint4 *d; float *o; long long *c;
    cudaMalloc(&d, k * 16); cudaMalloc(&o, 1024 * 4); cudaMalloc(&c, 1024 * 8);
    cudaMemcpy(d, h.data(), k * 16, cudaMemcpyHostToDevice);
    for (int mode = 0; mode < 2; mode++)
        for (int nwarps : {1, 4, 8, 24})
            for (int busy : {0, 200000}) {
                if (nwarps == 1 && busy) continue;
                long long hc = 0;
                for (int rep = 0; rep < 3; rep++) {
                    k_micro<<<1, 32 * nwarps>>>(d, k, mode, busy, o, c);
                    cudaDeviceSynchronize();
                }
                cudaMemcpy(&hc, c, 8, cudaMemcpyDeviceToHost);
                printf("mode %d (%s) warps/block %2d busy %6d : %6.1f cycles/record (%lld cycles for k=%d) %s\n", mode, mode ? "fold_chunk" : "fold_chunk_general", nwarps, busy,
                       (double)hc / k, hc, k, cudaGetErrorString(cudaGetLastError()));
            }
    return 0;
}
