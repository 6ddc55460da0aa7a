// inflate_schedule_bench.cu -- the two schedules DESIGN.md f14 weighs for the inflation brushfire, timed on the same
// inputs: (A) the library's persistent cooperative kernel k_inflate, three grid barriers per distance bin; (B) one launch
// per phase and bin (3 per bin, plus the key reset), each of the same fixed size, captured once into a CUDA graph and
// replayed.  Both read the window of each bin from the bin starts on the device, so neither reads anything back.  The
// phase kernels below restate k_inflate's phases over gem_inflate.cuh's infl_entry / infl_wins; the outputs of A and B
// are checked equal.  Inputs: N x N grids with 1 % LETHAL cells (seeded), factor 10, inscribed 2 cells.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -fmad=false -std=c++17 -o /tmp/inflate_schedule_bench \
//        scripts/inflate_schedule_bench.cu && /tmp/inflate_schedule_bench
// Prints one JSON line: per workload the median of 50 calls of each schedule (CUDA events), bins and blocks.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <map>
#include <vector>

#include "../gem_b200/csrc/gem_inflate.cuh"

using namespace gem;

#define CK(x)                                                                                   \
    do {                                                                                        \
        cudaError_t e_ = (x);                                                                   \
        if (e_ != cudaSuccess) {                                                                \
            std::fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
            std::exit(1);                                                                       \
        }                                                                                       \
    } while (0)

__device__ __forceinline__ void phase_range(const InflateArgs &a, int q, long long &g0, long long &s0, long long &s1)
{
    long long nslots;
    g0 = 0;
    if (q == 0) {
        nslots = (long long)a.rw * a.rh;
    } else {
        g0 = __ldcg(&a.gstart[a.lo[q]]);
        nslots = 4ll * (__ldcg(&a.gstart[q]) - g0);
    }
    const long long chunk = ((nslots + gridDim.x - 1) / gridDim.x + INFL_BLOCK - 1) / INFL_BLOCK * INFL_BLOCK;
    s0 = (long long)blockIdx.x * chunk;
    s1 = s0 + chunk < nslots ? s0 + chunk : nslots;
}

__global__ void __launch_bounds__(INFL_BLOCK) k_phase1(InflateArgs a, int q)
{
    long long g0, s0, s1;
    phase_range(a, q, g0, s0, s1);
    int cell, src;
    unsigned long long k;
    for (long long s = s0 + threadIdx.x; s < s1; s += INFL_BLOCK)
        if (infl_entry(a, q, g0, s, cell, src, k) && __ldcg(&a.key[cell]) > k) atomicMin(&a.key[cell], k);
}

__global__ void __launch_bounds__(INFL_BLOCK) k_phase2(InflateArgs a, int q)
{
    long long g0, s0, s1;
    phase_range(a, q, g0, s0, s1);
    int cell, src, n = 0;
    for (long long t = s0; t < s1; t += INFL_BLOCK) {
        const long long s = t + threadIdx.x;
        n += __syncthreads_count(s < s1 && infl_wins(a, q, g0, s, cell, src));
    }
    if (threadIdx.x == 0) a.blk[blockIdx.x] = n;
}

__global__ void __launch_bounds__(INFL_BLOCK) k_phase3(InflateArgs a, int q)
{
    __shared__ int wsum[INFL_BLOCK / 32];
    __shared__ int s_base, s_total;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    long long g0, s0, s1;
    phase_range(a, q, g0, s0, s1);
    int before = 0, total = 0;
    for (int b = threadIdx.x; b < (int)gridDim.x; b += INFL_BLOCK) {
        const int c = __ldcg(&a.blk[b]);
        total += c;
        before += b < (int)blockIdx.x ? c : 0;
    }
    before = __reduce_add_sync(0xffffffffu, before);
    total = __reduce_add_sync(0xffffffffu, total);
    if (lane == 0) wsum[wid] = before;
    __syncthreads();
    if (threadIdx.x == 0) {
        int b = 0;
        for (int w = 0; w < INFL_BLOCK / 32; w++) b += wsum[w];
        s_base = b;
    }
    __syncthreads();
    if (lane == 0) wsum[wid] = total;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < INFL_BLOCK / 32; w++) t += wsum[w];
        s_total = t;
    }
    __syncthreads();
    const int gq = __ldcg(&a.gstart[q]);
    int pos = gq + s_base, cell, src;
    for (long long t = s0; t < s1; t += INFL_BLOCK) {
        const long long s = t + threadIdx.x;
        const bool win = s < s1 && infl_wins(a, q, g0, s, cell, src);
        const unsigned bal = __ballot_sync(0xffffffffu, win);
        __syncthreads();
        if (lane == 0) wsum[wid] = __popc(bal);
        __syncthreads();
        int off = 0, all = 0;
        for (int w = 0; w < INFL_BLOCK / 32; w++) {
            off += w < wid ? wsum[w] : 0;
            all += wsum[w];
        }
        if (win) {
            a.pops[pos + off + __popc(bal & ((1u << lane) - 1u))] = make_int2(cell, src);
            a.key[cell] = 0;
            const int my = cell / a.sx, mx = cell - my * a.sx, sy = src / a.sx, sx = src - sy * a.sx;
            const unsigned char c = a.cost[abs(mx - sx) * a.tw + abs(my - sy)];
            const unsigned char o = __ldcg(&a.master[cell]);
            if (o == COST_UNKNOWN && (a.inflate_unknown ? c > COST_FREE : c >= 253)) a.master[cell] = c;
            else a.master[cell] = o > c ? o : c;
        }
        pos += all;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) a.gstart[q + 1] = gq + s_total;
}

__global__ void k_reset(InflateArgs a)
{
    const int npop = __ldcg(&a.gstart[a.nbins]);
    for (int g = blockIdx.x * INFL_BLOCK + threadIdx.x; g < npop; g += gridDim.x * INFL_BLOCK) a.key[__ldcg(&a.pops[g]).x] = ~0ull;
}

// the library's host tables (gem_costmap_inflate): bin index per (i, j), cost, and the first bin that can push into each
static int tables(int r, double res, double weight, double inscribed, std::vector<int> &bin, std::vector<unsigned char> &cost,
                  std::vector<int> &lo)
{
    const int tw = r + 2;
    std::vector<double> dist((size_t)tw * tw);
    cost.assign((size_t)tw * tw, 0);
    for (int i = 0; i < tw; i++)
        for (int j = 0; j < tw; j++) {
            const double d = std::hypot((double)i, (double)j);
            dist[(size_t)i * tw + j] = d;
            cost[(size_t)i * tw + j] = d == 0 ? 254 : d * res <= inscribed ? 253
                                                      : (unsigned char)(252 * std::exp(-1.0 * weight * (d * res - inscribed)));
        }
    std::map<double, int> bins;
    for (double d : dist)
        if (!(d > r)) bins.emplace(d, 0);
    int nb = 0;
    for (auto &kv : bins) kv.second = nb++;
    bin.assign((size_t)tw * tw, -1);
    for (size_t t = 0; t < dist.size(); t++)
        if (!(dist[t] > r)) bin[t] = bins[dist[t]];
    lo.assign(nb, INT_MAX);
    for (int i = 0; i < tw; i++)
        for (int j = 0; j < tw; j++) {
            const int q = bin[(size_t)i * tw + j];
            if (q < 0) continue;
            const int n4[4][2] = {{i - 1, j}, {i + 1, j}, {i, j - 1}, {i, j + 1}};
            for (auto &n : n4)
                if (n[0] >= 0 && n[1] >= 0 && n[0] < tw && n[1] < tw) {
                    const int b = bin[(size_t)n[0] * tw + n[1]];
                    if (b >= 0 && b < lo[q]) lo[q] = b;
                }
        }
    for (int q = 0; q < nb; q++) lo[q] = std::min(lo[q], q);
    return nb;
}

int main()
{
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    int per_sm = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_inflate, INFL_BLOCK, 0));
    const int blocks = std::max(1, std::min(per_sm, 4) * prop.multiProcessorCount);
    cudaStream_t st;
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    std::printf("{\"gpu\": \"%s\", \"blocks\": %d, \"calls\": 50", prop.name, blocks);
    const int work[][2] = {{1000, 3}, {1000, 10}, {4000, 40}};
    bool all_equal = true;
    for (auto &wk : work) {
        const int N = wk[0], r = wk[1];
        const size_t cells = (size_t)N * N;
        std::vector<unsigned char> m0(cells, 0);
        unsigned long long x = 12345;
        for (size_t c = 0; c < cells; c++) {
            x = x * 6364136223846793005ull + 1442695040888963407ull;
            if ((x >> 33) % 100 == 0) m0[c] = 254;
        }
        std::vector<int> bin, lo;
        std::vector<unsigned char> cost;
        const int nb = tables(r, 1.0, 10.0 / r, 2.0, bin, cost, lo);
        const int tw = r + 2;
        unsigned char *d_m0, *d_m, *d_cost;
        int *d_bin, *d_lo, *d_gstart, *d_blk;
        unsigned long long *d_key;
        int2 *d_pops;
        CK(cudaMalloc(&d_m0, cells));
        CK(cudaMalloc(&d_m, cells));
        CK(cudaMalloc(&d_key, cells * 8));
        CK(cudaMalloc(&d_pops, cells * 8));
        CK(cudaMalloc(&d_bin, bin.size() * 4));
        CK(cudaMalloc(&d_cost, cost.size()));
        CK(cudaMalloc(&d_lo, lo.size() * 4));
        CK(cudaMalloc(&d_gstart, (nb + 1) * 4));
        CK(cudaMalloc(&d_blk, blocks * 4));
        CK(cudaMemcpy(d_m0, m0.data(), cells, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(d_bin, bin.data(), bin.size() * 4, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(d_cost, cost.data(), cost.size(), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(d_lo, lo.data(), lo.size() * 4, cudaMemcpyHostToDevice));
        CK(cudaMemset(d_key, 0xFF, cells * 8));
        InflateArgs a{d_m, N, N, 0, 0, N, N, d_bin, d_cost, d_lo, tw, nb, 0, d_key, d_pops, d_gstart, d_blk};
        // B's graph: the gstart reset, then 3 launches per bin (2 for bin 0) and the key reset
        cudaGraph_t graph;
        cudaGraphExec_t exec;
        CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        CK(cudaMemsetAsync(d_gstart, 0, 4, st));
        for (int q = 0; q < nb; q++) {
            if (q > 0) k_phase1<<<blocks, INFL_BLOCK, 0, st>>>(a, q);
            k_phase2<<<blocks, INFL_BLOCK, 0, st>>>(a, q);
            k_phase3<<<blocks, INFL_BLOCK, 0, st>>>(a, q);
        }
        k_reset<<<blocks, INFL_BLOCK, 0, st>>>(a);
        CK(cudaStreamEndCapture(st, &graph));
        CK(cudaGraphInstantiate(&exec, graph, 0));
        std::vector<unsigned char> outA(cells), outB(cells);
        double med[2];
        for (int sch = 0; sch < 2; sch++) {
            cudaEvent_t e0, e1;
            CK(cudaEventCreate(&e0));
            CK(cudaEventCreate(&e1));
            std::vector<float> t;
            for (int it = 0; it < 55; it++) {
                CK(cudaMemcpyAsync(d_m, d_m0, cells, cudaMemcpyDeviceToDevice, st));
                CK(cudaEventRecord(e0, st));
                if (sch == 0) {
                    CK(cudaMemsetAsync(d_gstart, 0, 4, st));
                    void *args[] = {&a};
                    CK(cudaLaunchCooperativeKernel((const void *)k_inflate, dim3(blocks), dim3(INFL_BLOCK), args, 0, st));
                } else {
                    CK(cudaGraphLaunch(exec, st));
                }
                CK(cudaEventRecord(e1, st));
                CK(cudaEventSynchronize(e1));
                float ms;
                CK(cudaEventElapsedTime(&ms, e0, e1));
                if (it >= 5) t.push_back(ms);
            }
            std::sort(t.begin(), t.end());
            med[sch] = t[t.size() / 2];
            CK(cudaMemcpy(sch == 0 ? outA.data() : outB.data(), d_m, cells, cudaMemcpyDeviceToHost));
        }
        const bool eq = outA == outB;
        all_equal &= eq;
        std::printf(", \"n%d_r%d\": {\"bins\": %d, \"persistent_ms\": %.4f, \"graph_ms\": %.4f, \"equal\": %s}", N, r, nb, med[0], med[1],
                    eq ? "true" : "false");
        CK(cudaGraphExecDestroy(exec));
        CK(cudaGraphDestroy(graph));
        for (void *p : {(void *)d_m0, (void *)d_m, (void *)d_key, (void *)d_pops, (void *)d_bin, (void *)d_cost, (void *)d_lo,
                        (void *)d_gstart, (void *)d_blk})
            CK(cudaFree(p));
    }
    std::printf(", \"outputs_equal\": %s}\n", all_equal ? "true" : "false");
    CK(cudaStreamDestroy(st));
    return all_equal ? 0 : 1;
}
