// gem_costmap.cuh -- the navigation costmap layers of GEM's `layers/` package on the device (DESIGN.md f8):
// ElevationMapLayer::updateBounds (layers/src/elevationMap_layer.cpp:56-84) over the grid_map show() publishes,
// PointMapLayer::updateBounds (layers/src/pointMap_layer.cpp:54-81) over PointXYZRGBICT records, Costmap2D::updateOrigin
// (the rolling window) and the two ways a layer is combined into the master grid (CostmapLayer::updateWithMax and
// PointMapLayer::updateCosts, :86-100).  costmap_2d (navigation 1.14) is an unpinned dependency; its definitions are
// restated at the code and in DESIGN.md f8.
//
// A costmap grid is caller-owned device memory, uint8[size_y][size_x], cell (mx, my) at my * size_x + mx (getIndex).
// Costs: FREE_SPACE 0, LETHAL_OBSTACLE 254, NO_INFORMATION 255.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "gem_footprint.h"
#include "gem_kernels.cuh"

namespace gem {

constexpr unsigned char COST_FREE = 0, COST_LETHAL = 254, COST_UNKNOWN = 255;

struct CostWindow {
    double ox, oy, res;
    int sx, sy;
};

// Costmap2D::worldToMap (f8 item 4; gem_fp::world_to_map, shared with the host's footprint clearing)
__device__ __forceinline__ bool cm_world_to_map(const CostWindow &w, double wx, double wy, int &mx, int &my)
{
    return gem_fp::world_to_map(w.ox, w.oy, w.res, w.sx, w.sy, wx, wy, mx, my);
}

// Order-preserving integer encoding of a double (for atomicMin / atomicMax on the touch bounds).  touch() keeps
// min(x, min_x) etc.; the bounds are only ever compared, so a zero is reported as +0 (DEFINED: the reference's sign of a
// zero bound depends on which of two equal zeros came last).
__host__ __device__ __forceinline__ unsigned long long cm_key(double d)
{
    unsigned long long u;
    d = d + 0.0; // -0 -> +0
    memcpy(&u, &d, sizeof u);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__host__ __device__ __forceinline__ double cm_unkey(unsigned long long k)
{
    const unsigned long long u = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
    double d;
    memcpy(&d, &u, sizeof d);
    return d;
}

// what pass 1 accumulates: elements written (touch calls), of which LETHAL, and the encoded touch bounds
struct CostMarksDev {
    unsigned long long marked, lethal;
    unsigned long long minx, miny, maxx, maxy;
};

// Grid source: show()'s grid_map in GridMapIterator order (order = ix + iy * L over storage indices).  The value is
// show()'s traver (the feature output where the cell is shown, NaN elsewhere, ElevationMap.cpp:89,101), the position the
// grid_map cell centre in double.  ElevationMapLayer: is_obstacle = (double)value < travers_thresh (a float against a
// double), LETHAL if so, else FREE; NaN compares false, so a cleared cell is FREE, or writes nothing when
// mark_unknown == 0.  A chunk is 32 consecutive storage columns iy of one storage row ix: coalesced reads, and in a 0.05 m
// map neighbouring lanes usually fall into one costmap cell.
struct CostGridSrc {
    GridCloudSrc g;      // take() = show_valid on the live map; the snapshot already holds NaN where cleared
    double thresh;
    int mark_unknown;
    int nch;             // chunks per storage row
    __device__ __forceinline__ float value(int ix, int iy) const
    {
        return g.take(ix, iy) ? g.s.traver((size_t)ix * g.f.L + iy) : __int_as_float(0x7fc00000);
    }
    __device__ __forceinline__ bool element(long long chunk, int lane, int &order, double &wx, double &wy, unsigned char &cost) const
    {
        const int L = g.f.L;
        const int ix = (int)(chunk / nch), iy = (int)(chunk % nch) * 32 + lane;
        if (iy >= L) return false;
        const float v = value(ix, iy);
        if (v != v && !mark_unknown) return false;
        cost = ((double)v < thresh) ? COST_LETHAL : COST_FREE;
        wx = g.f.px(ix);
        wy = g.f.py(iy);
        order = ix + iy * L;
        return true;
    }
    __device__ __forceinline__ unsigned char cost_of(int order) const
    {
        const int L = g.f.L;
        return ((double)value(order % L, order / L) < thresh) ? COST_LETHAL : COST_FREE;
    }
};

// Point source: n 32-byte PointXYZRGBICT records {x, y, z, w, bgra, covariance, intensity, travers}, in record order.
// PointMapLayer: (double)x, (double)y through worldToMap; cost = (double)travers > travers_thresh ? FREE : LETHAL (so NaN
// and equality give LETHAL).
struct CostPointSrc {
    const float4 *p;
    int n;
    double thresh;
    __device__ __forceinline__ bool element(long long chunk, int lane, int &order, double &wx, double &wy, unsigned char &cost) const
    {
        const long long i = chunk * 32 + lane;
        if (i >= n) return false;
        const float4 a = p[2 * i];
        cost = cost_of((int)i);
        wx = (double)a.x;
        wy = (double)a.y;
        order = (int)i;
        return true;
    }
    __device__ __forceinline__ unsigned char cost_of(int order) const
    {
        const float t = reinterpret_cast<const float *>(p)[8 * (size_t)order + 7];
        return ((double)t > thresh) ? COST_FREE : COST_LETHAL;
    }
};

// Message-layer source (DESIGN.md f18): the floats of one grid_map_msgs/GridMap layer at any alignment, in G4 order
// (element k = the k-th float, buffer index (k % sx, k / sx)).  Positions are GridMapFrame's generalised to a rectangular
// map: (position + half) - res * unwrapped, half = 0.5 * length - 0.5 * res per axis, the start index already reduced
// into [0, size) on the host.  The cost rule and mark_unknown are CostGridSrc's.  A chunk is 32 consecutive floats.
struct CostMsgSrc {
    const unsigned char *p; // the layer's first float
    int aligned;            // p is 4-byte aligned: one 32-bit load per float, else four byte loads
    int sx, n;              // size_x, size_x * size_y
    int startx, starty;     // in [0, size_x) / [0, size_y)
    int sy;
    double ox, oy, res;     // ox = position_x + half_x, oy = position_y + half_y
    double thresh;
    int mark_unknown;
    __device__ __forceinline__ float value(int k) const
    {
        const unsigned char *q = p + 4 * (size_t)k;
        if (aligned) return __ldg(reinterpret_cast<const float *>(q));
        const uint32_t u = (uint32_t)__ldg(q) | ((uint32_t)__ldg(q + 1) << 8) | ((uint32_t)__ldg(q + 2) << 16) | ((uint32_t)__ldg(q + 3) << 24);
        return __uint_as_float(u);
    }
    __device__ __forceinline__ bool element(long long chunk, int lane, int &order, double &wx, double &wy, unsigned char &cost) const
    {
        const long long k = chunk * 32 + lane;
        if (k >= n) return false;
        const float v = value((int)k);
        if (v != v && !mark_unknown) return false;
        cost = ((double)v < thresh) ? COST_LETHAL : COST_FREE;
        const int ix = (int)(k % sx), iy = (int)(k / sx);
        const int ux = ix >= startx ? ix - startx : ix - startx + sx, uy = iy >= starty ? iy - starty : iy - starty + sy;
        wx = ox + res * (double)(-ux);
        wy = oy + res * (double)(-uy);
        order = (int)k;
        return true;
    }
    __device__ __forceinline__ unsigned char cost_of(int order) const { return ((double)value(order) < thresh) ? COST_LETHAL : COST_FREE; }
};

// Pass 1 of the deterministic last-writer scatter: one lane per source element (a warp per 32-element chunk, grid
// stride), worldToMap, then atomicMax(winner[cell], order).  Lanes of a warp hold increasing orders, so of each group of
// lanes with equal cells (__match_any_sync) only the highest lane issues the atomic.  The counts and the four touch
// bounds are reduced per warp and per block, then one atomic each per block.
constexpr int COST_BLOCK = 256;
template <class Src>
__global__ void __launch_bounds__(COST_BLOCK) k_costmap_scatter(Src s, long long nchunks, CostWindow w, int *winner, CostMarksDev *acc)
{
    __shared__ unsigned long long sh[COST_BLOCK / 32][6];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long nwarps = (long long)gridDim.x * (COST_BLOCK / 32);
    unsigned marked = 0, lethal = 0;
    unsigned long long kminx = cm_key(__longlong_as_double(0x7ff0000000000000ll)), kminy = kminx;
    unsigned long long kmaxx = cm_key(__longlong_as_double((long long)0xfff0000000000000ull)), kmaxy = kmaxx;
    for (long long k = (long long)blockIdx.x * (COST_BLOCK / 32) + wid; k < nchunks; k += nwarps) {
        int order = 0, mx = 0, my = 0;
        double wx = 0.0, wy = 0.0;
        unsigned char cost = 0;
        int cell = -1;
        if (s.element(k, lane, order, wx, wy, cost) && cm_world_to_map(w, wx, wy, mx, my)) cell = my * w.sx + mx;
        const unsigned grp = __match_any_sync(0xffffffffu, cell);
        if (cell >= 0) {
            marked++;
            lethal += cost == COST_LETHAL;
            const unsigned long long kx = cm_key(wx), ky = cm_key(wy);
            kminx = kx < kminx ? kx : kminx; kmaxx = kx > kmaxx ? kx : kmaxx;
            kminy = ky < kminy ? ky : kminy; kmaxy = ky > kmaxy ? ky : kmaxy;
            if (lane == 31 - __clz(grp)) atomicMax(&winner[cell], order);
        }
    }
    unsigned long long v[6] = {marked, lethal, kminx, kminy, kmaxx, kmaxy};
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        unsigned long long o[6];
#pragma unroll
        for (int q = 0; q < 6; q++) o[q] = __shfl_xor_sync(0xffffffffu, v[q], d);
        v[0] += o[0]; v[1] += o[1];
        v[2] = o[2] < v[2] ? o[2] : v[2]; v[3] = o[3] < v[3] ? o[3] : v[3];
        v[4] = o[4] > v[4] ? o[4] : v[4]; v[5] = o[5] > v[5] ? o[5] : v[5];
    }
    if (lane == 0) {
#pragma unroll
        for (int q = 0; q < 6; q++) sh[wid][q] = v[q];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int r = 1; r < COST_BLOCK / 32; r++) {
            v[0] += sh[r][0]; v[1] += sh[r][1];
            v[2] = sh[r][2] < v[2] ? sh[r][2] : v[2]; v[3] = sh[r][3] < v[3] ? sh[r][3] : v[3];
            v[4] = sh[r][4] > v[4] ? sh[r][4] : v[4]; v[5] = sh[r][5] > v[5] ? sh[r][5] : v[5];
        }
        if (v[0]) {
            atomicAdd(&acc->marked, v[0]);
            atomicAdd(&acc->lethal, v[1]);
            atomicMin(&acc->minx, v[2]); atomicMin(&acc->miny, v[3]);
            atomicMax(&acc->maxx, v[4]); atomicMax(&acc->maxy, v[5]);
        }
    }
}

// Pass 2: one thread per costmap cell; a cell with a winner gets the winner's cost, every other cell keeps its value
template <class Src> __global__ void __launch_bounds__(COST_BLOCK) k_costmap_store(Src s, const int *winner, int ncells, unsigned char *cost)
{
    const long long i = (long long)blockIdx.x * COST_BLOCK + threadIdx.x;
    if (i >= ncells) return;
    const int o = winner[i];
    if (o >= 0) cost[i] = s.cost_of(o);
}

// Costmap2D::updateOrigin's overlap copy, resetMaps and copy-back as one gather: new cell (i, j) holds old cell
// (i + cell_ox, j + cell_oy) when that lies inside the old grid, else the fill value.  `old` is a copy of the grid.
__global__ void __launch_bounds__(COST_BLOCK) k_costmap_roll(const unsigned char *old, unsigned char *cost, int sx, int sy, int cell_ox,
                                                             int cell_oy, unsigned char fill)
{
    const long long n = (long long)sx * sy;
    const long long i = (long long)blockIdx.x * COST_BLOCK + threadIdx.x;
    if (i >= n) return;
    const long long my = i / sx, mx = i - my * sx;
    const long long ox = mx + cell_ox, oy = my + cell_oy;
    cost[i] = (ox >= 0 && ox < sx && oy >= 0 && oy < sy) ? old[oy * sx + ox] : fill;
}

// One master byte from one layer byte.  Max (CostmapLayer::updateWithMax): a NO_INFORMATION layer cell is skipped,
// otherwise written when the master is NO_INFORMATION or below it.  Overwrite (PointMapLayer::updateCosts): every layer
// cell that is not NO_INFORMATION is copied.
__device__ __forceinline__ uint32_t cm_combine_byte(uint32_t l, uint32_t m, int mode)
{
    if (l == COST_UNKNOWN) return m;
    if (mode == 1) return l;
    return (m == COST_UNKNOWN || m < l) ? l : m;
}
__device__ __forceinline__ uint32_t cm_combine_word(uint32_t l, uint32_t m, int mode)
{
    uint32_t r = 0;
#pragma unroll
    for (int b = 0; b < 32; b += 8) r |= cm_combine_byte((l >> b) & 255u, (m >> b) & 255u, mode) << b;
    return r;
}
// Elementwise over the rect [i0, i1) x [j0, j1) (already clamped, non-empty).  Thread x of row j handles one 16-byte
// aligned block of the master row; a block wholly inside the rect goes as one 16-byte load / store of each grid when the
// layer has the master's alignment (vec), every other block byte by byte, touching only bytes inside the rect.
__global__ void __launch_bounds__(COST_BLOCK) k_costmap_combine(const unsigned char *layer, unsigned char *master, int sx, int i0, int i1,
                                                                int j0, int j1, int mode, int vec)
{
    const uintptr_t mb = (uintptr_t)master;
    for (int j = j0 + blockIdx.y; j < j1; j += gridDim.y) {
        const long long a = (long long)j * sx + i0, e = (long long)j * sx + i1; // row's byte range [a, e)
        const long long b0 = (long long)((mb + a) >> 4);
        const long long nb = (long long)((mb + e - 1) >> 4) - b0 + 1;
        for (long long q = (long long)blockIdx.x * COST_BLOCK + threadIdx.x; q < nb; q += (long long)gridDim.x * COST_BLOCK) {
            const long long lo = (long long)(((b0 + q) << 4) - mb); // first byte of the block, relative to master
            if (vec && lo >= a && lo + 16 <= e) {
                const uint4 l = *reinterpret_cast<const uint4 *>(layer + lo);
                uint4 m = *reinterpret_cast<const uint4 *>(master + lo);
                m.x = cm_combine_word(l.x, m.x, mode); m.y = cm_combine_word(l.y, m.y, mode);
                m.z = cm_combine_word(l.z, m.z, mode); m.w = cm_combine_word(l.w, m.w, mode);
                *reinterpret_cast<uint4 *>(master + lo) = m;
            } else {
                const long long s = lo > a ? lo : a, t = lo + 16 < e ? lo + 16 : e;
                for (long long k = s; k < t; k++) master[k] = (unsigned char)cm_combine_byte(layer[k], master[k], mode);
            }
        }
    }
}

} // namespace gem
