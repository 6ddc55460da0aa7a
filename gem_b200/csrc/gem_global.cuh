// gem_global.cuh -- the numeric block of composingGlobalMap (ElevationMapping.cpp:482-514) on the device: PCL's
// StatisticalOutlierRemoval (setMeanK, setStddevMulThresh; :1152-1156) over the grid cloud of gem_export_grid_cloud, and
// the split of the survivors into the road and obstacle clouds (:1161-1170).  DESIGN.md row f6.
//
// PARITY UNPINNED (PCL): the filter is restated from PCL 1.8 StatisticalOutlierRemoval<PointT>::applyFilterIndices with
// KdTreeFLANN (flann::L2_Simple<float>, exact search).  For every point with finite x, y, z: the mean_k + 1 smallest
// squared distances d2 to all points (itself included), each accumulated in float as FLANN does (r = 0; r += dx*dx;
// r += dy*dy; r += dz*dz, no contraction), sorted ascending, the first dropped, dist_sum (double) += sqrt(d2[k]) for
// k = 1..mean_k in that order, distance = (float)(dist_sum / mean_k).  Non-finite points get distance 0.  Which neighbour
// wins a tie does not matter: only the multiset of d2 values enters the sum.
//
// The grid cloud has at most one point per cell, at the cell centre, so the map grid is the spatial index:
//   * k_split_stage writes the z of every point with finite x, y, z into a GEOGRAPHIC-indexed array (NaN elsewhere) and
//     the float x of every geographic row, y of every column, from GridMapFrame::px/py exactly as ShownCells::emit
//     writes them into the records.  In geographic index space the storage wrap line does not exist: the neighbours of
//     a cell are the cells around it, clipped to [0, L).
//   * k_split_knn: one thread per geographic cell searches Chebyshev rings r = 1, 2, ... around it, keeping the
//     mean_k + 1 smallest d2 in sorted registers, and stops after ring r once it holds mean_k + 1 values and the largest
//     is <= split_ring_bound(r + 1), a lower bound on d2 for every cell of ring r+1 and beyond (proof there).  The z
//     array is 4 B per cell and a block's 16 x 16 tile plus four rings of halo is 24 x 24 floats, which stays in L1:
//     the loads go through the read-only path instead of an explicit shared-memory copy, which would add a barrier and
//     a halo loader without saving DRAM traffic.  A cell not finished within SPLIT_THREAD_RINGS rings is queued.
//   * k_split_knn_far: the queued cells (sparse maps, isolated cells, cells beside steps where dz dominates), the same
//     search restarted from ring 1 and run until it stops.  A ring can grow to the whole map: a queued cell costs O(L^2)
//     cell reads at worst.
//   * the distances are compacted into grid-cloud order with compact_cells (SplitDistSrc), and k_split_stats runs the
//     two double sums of applyFilterIndices as PCL's sequential loop, on one warp (DEFINED item 4).
//   * two more compact_cells passes write the kept points that go to the road and to the obstacle cloud (SplitSrc).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gem_kernels.cuh"

namespace gem {

constexpr int SPLIT_TILE = 16;         // k_split_knn: 16 x 16 geographic cells per block
constexpr int SPLIT_THREAD_RINGS = 4;  // rings searched per thread before a cell is queued for k_split_knn_far
constexpr int SPLIT_MAX_K = 64;

struct SplitStats { // device result of one gem_grid_cloud_split call: k_split_stats' fields and the three output counts
    double mean, stddev, threshold;
    int valid;
    int points, road, obstacle;
};

// d2 the FLANN way (flann::L2_Simple: r = 0; r += diff*diff per dimension, float, no contraction)
__device__ __forceinline__ float flann_d2(float ax, float ay, float az, float bx, float by, float bz)
{
    const float dx = __fsub_rn(ax, bx), dy = __fsub_rn(ay, by), dz = __fsub_rn(az, bz);
    float r = 0.0f;
    r = __fadd_rn(r, __fmul_rn(dx, dx));
    r = __fadd_rn(r, __fmul_rn(dy, dy));
    r = __fadd_rn(r, __fmul_rn(dz, dz));
    return r;
}

// Lower bound on the d2 of every cell at Chebyshev distance >= q from geographic cell (gx, gy); +inf when no such cell
// exists in [0, L)^2.
//
// Proof.  xg[g] = (float)(cx + half - res * g) with res > 0 is non-increasing in g (the double expression decreases and
// rounding to float is monotone), likewise yg.  A cell (g', h') at Chebyshev distance >= q has |g' - gx| >= q or
// |h' - gy| >= q; say g' <= gx - q.  Then xg[g'] >= xg[gx - q] >= xg[gx] = ax, so ax - xg[g'] <= ax - xg[gx - q] <= 0 in
// exact arithmetic and, rounding being monotone, fl(ax - xg[g']) <= fl(ax - xg[gx - q]) <= 0: |dx'| >= |dx_q| and
// fl(dx'^2) >= fl(dx_q^2).  The d2 of that cell is fl(fl(fl(0 + dx'^2) + dy'^2) + dz'^2): every addend is >= 0 and float
// addition of a non-negative addend never decreases a sum (monotone rounding of a + b >= a), so d2 >= fl(dx'^2) and,
// the same way, d2 >= fl(dy'^2).  The other three sides are symmetric.  The bound therefore holds for the ROUNDED
// positions: it is computed from the staged floats of the row / column at distance q, with the very operations of
// flann_d2, not from q * res -- far from the origin neighbouring centres round to equal floats and q * res would
// overestimate it.
__device__ __forceinline__ float split_ring_bound(const float *xg, const float *yg, int L, int gx, int gy, float ax, float ay, int q)
{
    float b = __int_as_float(0x7f800000);
    if (gx - q >= 0) { const float d = __fsub_rn(ax, xg[gx - q]); b = fminf(b, __fmul_rn(d, d)); }
    if (gx + q < L) { const float d = __fsub_rn(ax, xg[gx + q]); b = fminf(b, __fmul_rn(d, d)); }
    if (gy - q >= 0) { const float d = __fsub_rn(ay, yg[gy - q]); b = fminf(b, __fmul_rn(d, d)); }
    if (gy + q < L) { const float d = __fsub_rn(ay, yg[gy + q]); b = fminf(b, __fmul_rn(d, d)); }
    return b;
}

// the distance of a point from its sorted list: sqrt of each kept d2 but the first, in ascending order, in double
// (DEFINED item 1: the double sqrt of the float d2), then divided by mean_k
__device__ __forceinline__ float split_mean_distance(double dist_sum, int mean_k) { return (float)(dist_sum / (double)mean_k); }

// stage: zg[gx * L + gy] = z of the grid-cloud point of geographic cell (gx, gy) when x, y, z are finite, NaN otherwise
// (DEFINED item 2: a non-finite point is nobody's neighbour); xg / yg = the float x of every row, y of every column;
// dcell (storage-indexed) = 0, the distance of a point that gets none
__global__ void __launch_bounds__(256) k_split_stage(GridCloudSrc src, float *zg, float *xg, float *yg, float *dcell)
{
    const GridMapFrame &f = src.f;
    const int L = f.L;
    const size_t nc = (size_t)L * L;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += stride) {
        const int ix = (int)(c / L), iy = (int)(c - (size_t)ix * L);
        const int gx = (ix + L - f.sx) % L, gy = (iy + L - f.sy) % L;
        const float x = (float)f.px(ix), y = (float)f.py(iy); // ShownCells::emit
        if (iy == 0) xg[gx] = x;
        if (ix == 0) yg[gy] = y;
        const float z = src.s.elevation(c);
        const bool take = src.take(ix, iy); // the grid cloud's points (:1208)
        zg[(size_t)gx * L + gy] = (take && isfinite(x) && isfinite(y) && isfinite(z)) ? z : __int_as_float(0x7fc00000);
        dcell[c] = 0.0f;
    }
}

// KCAP >= mean_k + 1 register slots.  Slots [0, KCAP - K) hold -inf for good and the K live entries sit at the top, so
// the largest live entry is lst[KCAP - 1] and every index is static (no local memory).
template <int KCAP> struct SortedList {
    float v[KCAP];
    __device__ __forceinline__ void init(int K)
    {
#pragma unroll
        for (int j = 0; j < KCAP; j++) v[j] = j < KCAP - K ? __int_as_float(0xff800000) : __int_as_float(0x7f800000);
    }
    __device__ __forceinline__ float top() const { return v[KCAP - 1]; }
    // insert d, drop the largest: new[j] = old[j-1] if old[j-1] > d, else min(old[j], d)
    __device__ __forceinline__ void insert(float d)
    {
#pragma unroll
        for (int j = KCAP - 1; j > 0; j--) v[j] = v[j - 1] > d ? v[j - 1] : (v[j] < d ? v[j] : d);
        v[0] = v[0] < d ? v[0] : d;
    }
    __device__ __forceinline__ double sum_but_first(int K) const
    {
        double s = 0.0;
#pragma unroll
        for (int j = 0; j < KCAP; j++)
            if (j > KCAP - K) s += sqrt((double)v[j]);
        return s;
    }
};

// the ring search of one point at geographic cell (gx, gy) over rings 1..rmax (rmax >= L - 1: until it stops); false when
// it did not stop within rmax rings, else dist = its mean distance (NaN if the whole map holds fewer than K points)
template <int KCAP>
__device__ __forceinline__ bool split_search(const float *zg, const float *xg, const float *yg, int L, int gx, int gy, float az, int mean_k,
                                             int rmax, float &dist)
{
    const int K = mean_k + 1;
    const float ax = __ldg(xg + gx), ay = __ldg(yg + gy);
    SortedList<KCAP> lst;
    lst.init(K);
    lst.insert(0.0f); // the point itself
    int n = 1;        // candidates seen, capped at K
    for (int r = 1; r <= rmax; r++) {
        const int x0 = max(gx - r, 0), x1 = min(gx + r, L - 1);
        for (int x = x0; x <= x1; x++) {
            const float bx = __ldg(xg + x);
            const bool edge = x == gx - r || x == gx + r;
            const int y0 = edge ? max(gy - r, 0) : gy - r, y1 = edge ? min(gy + r, L - 1) : gy + r;
            const int step = edge ? 1 : 2 * r;
            for (int y = y0; y <= y1; y += step) {
                if (y < 0 || y >= L) continue;
                const float bz = __ldg(zg + (size_t)x * L + y);
                if (bz != bz) continue;
                const float d2 = flann_d2(ax, ay, az, bx, __ldg(yg + y), bz);
                n = min(n + 1, K);
                if (d2 < lst.top()) lst.insert(d2);
            }
        }
        const bool exhausted = gx - r - 1 < 0 && gx + r + 1 >= L && gy - r - 1 < 0 && gy + r + 1 >= L;
        if ((n == K && lst.top() <= split_ring_bound(xg, yg, L, gx, gy, ax, ay, r + 1)) || exhausted) {
            // fewer than mean_k + 1 points in the whole cloud (DEFINED item 3): NaN, k_split_stats handles the rest
            dist = n == K ? split_mean_distance(lst.sum_but_first(K), mean_k) : __int_as_float(0x7fc00000);
            return true;
        }
    }
    return false;
}

// one thread per geographic cell, rings 1..SPLIT_THREAD_RINGS; the cells not finished there are queued
template <int KCAP>
__global__ void __launch_bounds__(SPLIT_TILE * SPLIT_TILE) k_split_knn(const float *zg, const float *xg, const float *yg, int L, int sx, int sy,
                                                                        int mean_k, float *dcell, int *queue, int *counters /* {queued, finite} */)
{
    const int gx = blockIdx.y * SPLIT_TILE + threadIdx.x / SPLIT_TILE, gy = blockIdx.x * SPLIT_TILE + (threadIdx.x & (SPLIT_TILE - 1));
    const bool in = gx < L && gy < L;
    const float az = in ? __ldg(zg + (size_t)gx * L + gy) : __int_as_float(0x7fc00000);
    const bool pt = az == az;
    const unsigned m = __ballot_sync(0xffffffffu, pt); // warp-aggregated count of the points with a distance
    if ((threadIdx.x & 31u) == 0u && m) atomicAdd(&counters[1], __popc(m));
    if (!pt) return;
    float d;
    if (split_search<KCAP>(zg, xg, yg, L, gx, gy, az, mean_k, SPLIT_THREAD_RINGS, d))
        dcell[(size_t)((gx + sx) % L) * L + (gy + sy) % L] = d;
    else
        queue[atomicAdd(&counters[0], 1)] = gx * L + gy;
}

// the queued cells (sparse maps, isolated cells, cells beside steps where dz dominates): the same search, one thread per
// cell, restarted from ring 1 and run until it stops.  The queue's length stays on the device (a fixed grid strides
// over it).  A ring can grow to the whole map: a queued cell costs O(L^2) cell reads at worst.
template <int KCAP>
__global__ void __launch_bounds__(128) k_split_knn_far(const float *zg, const float *xg, const float *yg, int L, int sx, int sy, int mean_k,
                                                       float *dcell, const int *queue, const int *counters)
{
    const int nq = counters[0];
    for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += gridDim.x * blockDim.x) {
        const int cell = queue[q];
        const int gx = cell / L, gy = cell - gx * L;
        float d;
        split_search<KCAP>(zg, xg, yg, L, gx, gy, __ldg(zg + cell), mean_k, L, d); // stops by ring L - 1 at the latest (exhausted)
        dcell[(size_t)((gx + sx) % L) * L + (gy + sy) % L] = d;
    }
}

// the distances in grid-cloud order (the cells GridCloudSrc takes, GridMapIterator order), into the scratch the
// statistics read and into the first `capacity` entries of the caller's buffer
struct SplitDistSrc {
    GridCloudSrc g;
    const float *dcell;
    float *out;
    float *user;
    int capacity;
    __device__ __forceinline__ bool take(int ix, int iy) const { return g.take(ix, iy); }
    __device__ __forceinline__ void emit(int ix, int iy, int pos) const
    {
        const float d = dcell[(size_t)ix * g.f.L + iy];
        out[pos] = d;
        if (pos < capacity) user[pos] = d;
    }
};

// applyFilterIndices' statistics (DEFINED item 4: PCL's sequential loop in point order, bit for bit).  One warp: the
// lanes stage 1024 distances at a time in shared memory with coalesced loads, lane 0 runs the two dependent double
// chains.  With too few points the caller's distances (the first `capacity`) are overwritten with NaN.  points = the grid cloud's size, as the distance
// compaction left it on the device.  valid = the points with finite x, y, z; with at most mean_k of them (DEFINED
// item 3) every distance and statistic is NaN and valid = 0, which keeps every point (NaN > threshold is false).
constexpr int SPLIT_STATS_CHUNK = 1024;
__global__ void __launch_bounds__(32) k_split_stats(const float *dist, const int *points_dev, const int *counters, int mean_k, double stddev_mul,
                                                   SplitStats *out, float *user_dist, int capacity)
{
    __shared__ float buf[SPLIT_STATS_CHUNK];
    const unsigned lane = threadIdx.x;
    const int points = *points_dev, valid = counters[1];
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    if (valid <= mean_k) {
        for (int i = lane; i < min(points, capacity); i += 32) user_dist[i] = __int_as_float(0x7fc00000);
        if (lane == 0u) { out->mean = out->stddev = out->threshold = nan; out->valid = 0; }
        return;
    }
    double sum = 0.0, sq_sum = 0.0;
    for (int base = 0; base < points; base += SPLIT_STATS_CHUNK) {
        const int n = min(SPLIT_STATS_CHUNK, points - base);
        for (int i = lane; i < n; i += 32) buf[i] = dist[base + i];
        __syncwarp();
        if (lane == 0u) {
#pragma unroll 8
            for (int i = 0; i < n; i++) {
                const float d = buf[i];
                sum = __dadd_rn(sum, (double)d);
                sq_sum = __dadd_rn(sq_sum, (double)__fmul_rn(d, d)); // distances[i] * distances[i]: a float product
            }
        }
        __syncwarp();
    }
    if (lane == 0u) {
        const double v = (double)valid;
        const double mean = __ddiv_rn(sum, v);
        const double variance = __ddiv_rn(__dsub_rn(sq_sum, __ddiv_rn(__dmul_rn(sum, sum), v)), __dsub_rn(v, 1.0));
        const double stddev = __dsqrt_rn(variance);
        out->mean = mean;
        out->stddev = stddev;
        out->threshold = __dadd_rn(mean, __dmul_rn(stddev_mul, stddev));
        out->valid = valid;
    }
}

// the kept points of one output: taken, not removed (distance > threshold, float promoted to double), and
// (double)travers > travers_threshold (road) or not (obstacle: every grid-cloud traversability is non-NaN and != -10)
struct SplitSrc {
    GridCloudSrc g;
    const float *dcell;
    const SplitStats *st;
    double travers_threshold;
    int road;
    __device__ __forceinline__ bool take(int ix, int iy) const
    {
        if (!g.take(ix, iy)) return false;
        const size_t c = (size_t)ix * g.f.L + iy;
        if ((double)dcell[c] > st->threshold) return false;
        return ((double)g.s.traver(c) > travers_threshold) == (road != 0);
    }
    __device__ __forceinline__ void emit(int ix, int iy, int pos) const { g.emit(ix, iy, pos); }
};

} // namespace gem
