// gem_inflate.cuh -- costmap_2d's InflationLayer::updateCosts (navigation 1.14, unpinned) on the device (DESIGN.md f14).
//
// The reference is a brushfire over bins of increasing distance: std::map<double, std::vector<CellData>>, each bin taken
// in push order, each cell carrying the lethal source it was first reached from.  Its result depends on the order inside
// a bin, so it is reproduced exactly rather than replaced by a distance transform:
//   - every bin is known on the host: the distinct values of the distance table that are <= r (gem_api.cu);
//   - a push never lands in its parent's own bin (checked on the host when the tables are built) and a push into an
//     earlier bin is never processed, so once the bins before q are done, bin q holds all of its entries;
//   - every processed cell gets its global pop position G (the bins before it plus its rank in its bin).  The entry a
//     cell popped at G pushes in direction d (mx-1, my-1, mx+1, my+1) is slot 4G + d, so slot order is push order.  Seeds
//     (bin 0) are the rect's LETHAL cells in row-major order, which is their push order;
//   - bin q's entries are the slots of the pops of bins lo[q] .. q-1 (the only bins whose cells have neighbours in bin q)
//     whose child falls into bin q.  A cell's winner is its smallest slot, if the cell is still unseen; losers push
//     nothing.  The winners, compacted in slot order, are bin q's pops G.
// One persistent cooperative kernel runs every bin with three grid-wide barriers per bin: the atomicMin of the slot key per
// child cell, the per-block count of winners, then the ordered compaction that writes each winner's pop record and cost.
// No bin needs the host: the window of bin q is read from gstart[] on the device.
//
// key[cell] (u64, handle scratch): ~0 = unseen and no entry, 0 = seen, else 1 + the smallest slot that reached it in the
// current bin.  The kernel leaves every cell it popped at ~0 again, so the next call finds the buffer clear.
#pragma once
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "gem_costmap.cuh"

namespace gem {

constexpr int INFL_BLOCK = 256;

struct InflateArgs {
    unsigned char *master;
    int sx, sy;
    int ri0, rj0, rw, rh;              // the widened, clamped rect the seeds come from (I3)
    const int *bin;                    // [tw][tw]: bin index of dist[i][j], -1 beyond the radius
    const unsigned char *cost;         // [tw][tw]: computeCost(dist[i][j])
    const int *lo;                     // [nbins]: the first bin whose cells can push into bin q
    int tw, nbins, inflate_unknown;    // tw = r + 2 <= GEM_INFLATE_MAX_CELLS + 2: dx * tw + dy fits an int
    unsigned long long *key;           // [cells]
    int2 *pops;                        // [cells]: (cell, source) in pop order
    int *gstart;                       // [nbins + 1]: first pop of each bin
    int *blk;                          // [gridDim.x]: winners per block in the current bin
};

// Entry `s` of bin q: the child cell, its source and its slot key, or false when the slot pushes nothing into bin q.
__device__ __forceinline__ bool infl_entry(const InflateArgs &a, int q, long long g0, long long s, int &cell, int &src,
                                           unsigned long long &k)
{
    if (q == 0) { // seeds: the rect's cells in row-major order
        const int j = a.rj0 + (int)(s / a.rw), i = a.ri0 + (int)(s % a.rw);
        cell = j * a.sx + i;
        src = cell;
        k = 0;
        return __ldcg(&a.master[cell]) == COST_LETHAL;
    }
    const long long G = g0 + (s >> 2);
    const int d = (int)(s & 3);
    const int2 p = __ldcg(&a.pops[G]);
    const int my = p.x / a.sx, mx = p.x - my * a.sx;
    const int sy = p.y / a.sx, sx = p.y - sy * a.sx;
    int nx = mx, ny = my;
    if (d == 0) { if (mx == 0) return false; nx--; }
    else if (d == 1) { if (my == 0) return false; ny--; }
    else if (d == 2) { if (mx == a.sx - 1) return false; nx++; }
    else { if (my == a.sy - 1) return false; ny++; }
    const int dx = abs(nx - sx), dy = abs(ny - sy);
    if (dx >= a.tw || dy >= a.tw || a.bin[dx * a.tw + dy] != q) return false;
    cell = ny * a.sx + nx;
    src = p.y;
    k = 4ull * (unsigned long long)G + (unsigned long long)d + 1ull;
    return true;
}

__device__ __forceinline__ bool infl_wins(const InflateArgs &a, int q, long long g0, long long s, int &cell, int &src)
{
    unsigned long long k;
    if (!infl_entry(a, q, g0, s, cell, src, k)) return false;
    return q == 0 || __ldcg(&a.key[cell]) == k;
}

__global__ void __launch_bounds__(INFL_BLOCK) k_inflate(InflateArgs a)
{
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    __shared__ int wsum[INFL_BLOCK / 32];
    __shared__ int s_base, s_total;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int q = 0; q < a.nbins; q++) {
        long long g0 = 0, nslots;
        if (q == 0) {
            nslots = (long long)a.rw * a.rh;
        } else {
            g0 = __ldcg(&a.gstart[a.lo[q]]);
            nslots = 4ll * (__ldcg(&a.gstart[q]) - g0);
        }
        // each block owns one contiguous range of slots, so block order is slot order
        const long long chunk = ((nslots + gridDim.x - 1) / gridDim.x + INFL_BLOCK - 1) / INFL_BLOCK * INFL_BLOCK;
        const long long s0 = (long long)blockIdx.x * chunk, s1 = s0 + chunk < nslots ? s0 + chunk : nslots;
        int cell, src;
        unsigned long long k;
        if (q > 0) {
            // phase 1: the smallest slot per unseen child cell
            for (long long s = s0 + threadIdx.x; s < s1; s += INFL_BLOCK)
                if (infl_entry(a, q, g0, s, cell, src, k) && __ldcg(&a.key[cell]) > k) atomicMin(&a.key[cell], k);
            grid.sync();
        }
        // phase 2: winners per block
        int n = 0;
        for (long long t = s0; t < s1; t += INFL_BLOCK) {
            const long long s = t + threadIdx.x;
            n += __syncthreads_count(s < s1 && infl_wins(a, q, g0, s, cell, src));
        }
        if (threadIdx.x == 0) a.blk[blockIdx.x] = n;
        grid.sync();
        // phase 3: this block's offset among the winners, then the winners in slot order
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
        int pos = gq + s_base;
        for (long long t = s0; t < s1; t += INFL_BLOCK) {
            const long long s = t + threadIdx.x;
            const bool win = s < s1 && infl_wins(a, q, g0, s, cell, src);
            const unsigned bal = __ballot_sync(0xffffffffu, win);
            __syncthreads(); // wsum of the previous tile has been read
            if (lane == 0) wsum[wid] = __popc(bal);
            __syncthreads();
            int off = 0, all = 0;
            for (int w = 0; w < INFL_BLOCK / 32; w++) {
                off += w < wid ? wsum[w] : 0;
                all += wsum[w];
            }
            if (win) {
                a.pops[pos + off + __popc(bal & ((1u << lane) - 1u))] = make_int2(cell, src);
                a.key[cell] = 0; // seen
                // the cost of the cell from its source, and I4's write rule
                const int my = cell / a.sx, mx = cell - my * a.sx, sy = src / a.sx, sx = src - sy * a.sx;
                const unsigned char c = a.cost[abs(mx - sx) * a.tw + abs(my - sy)];
                const unsigned char o = __ldcg(&a.master[cell]);
                if (o == COST_UNKNOWN && (a.inflate_unknown ? c > COST_FREE : c >= 253)) a.master[cell] = c;
                else a.master[cell] = o > c ? o : c;
            }
            pos += all;
        }
        if (blockIdx.x == 0 && threadIdx.x == 0) a.gstart[q + 1] = gq + s_total;
        grid.sync();
    }
    // leave the key buffer clear for the next call: every cell that was given a key was popped
    const int npop = __ldcg(&a.gstart[a.nbins]);
    for (int g = blockIdx.x * INFL_BLOCK + threadIdx.x; g < npop; g += gridDim.x * INFL_BLOCK) a.key[__ldcg(&a.pops[g]).x] = ~0ull;
}

} // namespace gem
