// gem_mls.cuh -- the moving-least-squares densification of GEM's dense_mapping signal on the device (DESIGN.md f10):
// pointcloudinterpolation (ElevationMapping.cpp:1072-1118), i.e. pcl::MovingLeastSquares<PointXYZRGB, PointXYZRGB>::process
// of PCL 1.7.2 (performProcessing / computeMLSPointNormal, KdTreeFLANN radius search, single-threaded), over n 32-byte
// PointXYZRGBICT records in device memory.  PCL is an unpinned dependency; its definitions are restated here, in
// include/gem_b200.h and in tests/orc_mls.c.  DEFINED marks what the library fixes where the reference leaves it open.
//
// M1 Input: of each record only x, y, z and the bgra word are read.  DEFINED: a record whose x, y or z is not finite is
//    nobody's neighbour and produces no output (FLANN is undefined there); it counts in skipped.
// M2 Neighbours (radiusSearch, L2_Simple<float>): d2 = ((dx dx) + dy dy) + dz dz in float, dx = x_j - x_i; j is a
//    neighbour iff d2 <= (float)(r r) (DEFINED inclusive), the query included, the list sorted by ascending d2 and ties by
//    ascending index (DEFINED), no cap.  Fewer than 3 neighbours: the point produces nothing.
// M3 Plane, in double and neighbour order: compute3DCentroid (sequential sums, then / n), the non-normalised
//    computeCovarianceMatrix in its update order ((1,1), (1,2), (2,2), then pt *= pt.x: (0,0), (0,1), (0,2)), eigen33's
//    smallest eigenpair (scale by the largest |entry|, computeRoots with its epsilon test and the computeRoots2 fallback,
//    also when the smallest root is <= 0, three row cross products, the largest squared norm in PCL's if-chain order),
//    d = -(n . centroid) with the Vector4d dot in Eigen's SSE2 packet order (a0b0 + a2b2) + (a1b1 + a3b3), and the
//    projection point = q - (q . n + d) n.  3-vector dots left to right (DEFINED).  atan2, sin, cos and exp are
//    gem_mathd.h's, shared with the oracle.
// M4 Fit, when polynomial_fit holds and n >= nr_coeff = (order + 1)(order + 2) / 2: de = p_j - point, d2f = (float)(de .
//    de), w = exp_d(-d2f / sqr_gauss), v_axis = n.unitOrthogonal() (Eigen: isMuchSmallerThan at 1e-12, 1 / |head<2>| or
//    1 / |tail<2>|), u_axis = n x v_axis, u = de . u_axis, v = de . v_axis, f = de . n, monomials in PCL's order (u power
//    outer, v power inner, running products).  A(a,b) = sum ((P(a) w) P(b)) for a >= b (the triangle LLT<Lower> reads)
//    and rhs(a) = sum ((P(a) w) f), each summed sequentially in neighbour order from +0 (DEFINED: Eigen's GEMM blocking
//    has no fixed order).  Left-looking Cholesky: L(i,j) = (A(i,j) - sum_{k<j} L(i,k) L(j,k)) / L(j,j), the diagonal the
//    square root of the same sum, k ascending; forward substitution y(i) = (rhs(i) - sum_{k<i} L(i,k) y(k)) / L(i,i),
//    back substitution c(i) = (y(i) - sum_{k>i} L(k,i) c(k)) / L(i,i), k ascending (DEFINED).  DEFINED: a pivot that is
//    not finite or not > 0 fails the fit, as PCL's !pcl_isfinite(c_vec[0]) does (Eigen would go on from a partial
//    factor); a non-finite c0 fails it too.  Reproduced from 1.7.2: the Darboux axes are set only inside the fit
//    (attempted, whatever its outcome); without one they are zero.
// M5 GEM_MLS_NONE: one output per processed point, point + c0 n when the fit succeeded, else the projection.
// M6 GEM_MLS_RANDOM_UNIFORM_DENSITY: k = (int)floor(point_density / 2.0 / n); k <= 0: M5's single output.  Otherwise k
//    samples: u, then v, floats in [-r/2, r/2), drawn again while u u + v v > r r / 4 (in double); the sample is
//    point + u u_axis + v v_axis, plus height(u, v) n when the fit succeeded, height = sum (u^a v^b) c_j in PCL's
//    monomial order with running products in double.  Without a fit all k samples land on the projection.  DEFINED
//    generator (the reference seeds boost::mt19937 with time(0)): draw j of input point i is splitmix64(seed ^ (i << 32)
//    ^ j), the float lo + (float)(x >> 40) 2^-24 (hi - lo) in float with hi = (float)(r / 2), lo = -hi; a rejected pair
//    consumes its two draws.
// M7 Output records: (float) of the double position, w = 1, bgra = the query's b, g, r with a = 0xff (DEFINED: the
//    alpha of PointXYZRGB's constructor), covariance, intensity and travers of the query (DEFINED: uninitialised in the
//    reference); input order, sample order within a point.
// M8 Info: processed (n >= 3), fitted, skipped (n < 3 or non-finite), max_neighbours (the longest list), count.
//
// The search grid: cells of edge r (1 + 2^-10) from the per-axis float minimum of the finite points, cell coordinates
// floor(((double)x - min) / edge) clamped to 2^21 - 1 and packed into a 63-bit key.  A neighbour (float d2 <= (float)r^2)
// lies within r (1 + 3e-7) in exact arithmetic, which is under one edge, so its cell differs from the query's by at most
// one on every axis; the clamp is monotone and keeps that true.  The 27 cells around a query therefore hold every
// neighbour; which cells they are only changes how many candidates are tested, never the list.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gem_kernels.cuh"
#include "gem_mathd.h"
#include "gem_voxel.cuh"

namespace gem {

constexpr int MLS_BLOCK = 128;         // four warps, one query each
constexpr int MLS_WARPS = MLS_BLOCK / 32;
constexpr int MLS_LIST = 512;          // a neighbour list of at most this many entries is sorted in shared memory
constexpr int MLS_CELL_BITS = 21;
constexpr unsigned long long MLS_CELL_MAX = (1ull << MLS_CELL_BITS) - 1;
constexpr int MLS_STAGE = 24;          // doubles per staged neighbour: 21 monomials, f, w, pad
constexpr int MLS_MAXC = 21;           // coefficients of order 5

struct MlsParams {
    double r, r2q, gauss, edge; // radius, r r / 4, sqr_gauss_param, cell edge
    float r2f, lo, hi;          // (float)(r r), the draw interval
    int fit, order, nc, upsampling, density;
    unsigned long long seed;
};

struct MlsAcc {
    unsigned mn[3];             // order-preserving encodings of the per-axis minimum of the finite points
    int nruns;                  // distinct keys after the sort (cells, plus one run of non-finite points)
    int nlong;                  // points whose list exceeds MLS_LIST
    int processed, skipped, fitted, max_nb;
    int pad;
};

__device__ __forceinline__ bool mls_finite(const float4 &p) { return isfinite(p.x) && isfinite(p.y) && isfinite(p.z); }
__device__ __forceinline__ float mls_d2(const float4 &p, const float4 &q)
{
    const float dx = p.x - q.x, dy = p.y - q.y, dz = p.z - q.z;
    return (dx * dx + dy * dy) + dz * dz;
}
__device__ __forceinline__ unsigned long long mls_cell1(float x, double mn, double edge)
{
    const double c = floor(((double)x - mn) / edge);
    return c >= (double)MLS_CELL_MAX ? MLS_CELL_MAX : (unsigned long long)c;
}
__device__ __forceinline__ void mls_cell(const float4 &p, const MlsAcc *acc, double edge, long long c[3])
{
    c[0] = (long long)mls_cell1(p.x, (double)vg_unkey(acc->mn[0]), edge);
    c[1] = (long long)mls_cell1(p.y, (double)vg_unkey(acc->mn[1]), edge);
    c[2] = (long long)mls_cell1(p.z, (double)vg_unkey(acc->mn[2]), edge);
}
__device__ __forceinline__ unsigned long long mls_key(long long cx, long long cy, long long cz)
{
    return ((unsigned long long)cz << (2 * MLS_CELL_BITS)) | ((unsigned long long)cy << MLS_CELL_BITS) | (unsigned long long)cx;
}

// Pass 1: the per-axis minimum of the finite points (order-preserving encodings; min is exact, so any order will do)
__global__ void __launch_bounds__(VOX_BLOCK) k_mls_bounds(const float4 *__restrict__ in, int n, MlsAcc *acc)
{
    __shared__ unsigned sh[VOX_BLOCK / 32][3];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned mn[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu};
    for (long long i = (long long)blockIdx.x * VOX_BLOCK + threadIdx.x; i < n; i += (long long)gridDim.x * VOX_BLOCK) {
        const float4 p = in[2 * i];
        if (mls_finite(p)) {
            mn[0] = min(mn[0], vg_key(p.x));
            mn[1] = min(mn[1], vg_key(p.y));
            mn[2] = min(mn[2], vg_key(p.z));
        }
    }
#pragma unroll
    for (int a = 0; a < 3; a++) mn[a] = __reduce_min_sync(0xffffffffu, mn[a]);
    if (lane == 0)
        for (int a = 0; a < 3; a++) sh[wid][a] = mn[a];
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < VOX_BLOCK / 32; w++)
            for (int a = 0; a < 3; a++) mn[a] = min(mn[a], sh[w][a]);
        for (int a = 0; a < 3; a++)
            if (mn[a] != 0xffffffffu) atomicMin(&acc->mn[a], mn[a]);
    }
}

// Pass 2: the cell key of each point (all ones for a non-finite one: it sorts last and no query looks it up), value =
// input index
__global__ void __launch_bounds__(VOX_BLOCK) k_mls_keys(const float4 *__restrict__ in, int n, MlsParams P, const MlsAcc *acc,
                                                        unsigned long long *__restrict__ key, int *__restrict__ idx)
{
    const long long i = (long long)blockIdx.x * VOX_BLOCK + threadIdx.x;
    if (i >= n) return;
    const float4 p = in[2 * i];
    unsigned long long k = ~0ull;
    if (mls_finite(p)) {
        long long c[3];
        mls_cell(p, acc, P.edge, c);
        k = mls_key(c[0], c[1], c[2]);
    }
    key[i] = k;
    idx[i] = (int)i;
}

// Pass 3: the points in cell order, {x, y, z, input index}, so that a cell's candidates are one contiguous run
__global__ void __launch_bounds__(VOX_BLOCK) k_mls_stage(const float4 *__restrict__ in, int n, const int *__restrict__ sidx,
                                                         float4 *__restrict__ spts)
{
    const long long s = (long long)blockIdx.x * VOX_BLOCK + threadIdx.x;
    if (s >= n) return;
    const int i = sidx[s];
    const float4 p = in[2 * (long long)i];
    spts[s] = make_float4(p.x, p.y, p.z, __int_as_float(i));
}

// The run of cell `key` among the sorted distinct keys, or an empty one
__device__ __forceinline__ void mls_cell_range(const unsigned long long *__restrict__ ukey, const int *__restrict__ uoff,
                                               const int *__restrict__ ucnt, int nruns, unsigned long long key, int &st, int &len)
{
    int lo = 0, hi = nruns;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ukey[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    st = 0;
    len = 0;
    if (lo < nruns && ukey[lo] == key) { st = uoff[lo]; len = ucnt[lo]; }
}

// Lane c < 27 of the warp finds the run of the c-th cell around the query (empty beyond the grid)
__device__ __forceinline__ void mls_lane_cell(const float4 &q, const MlsParams &P, const MlsAcc *acc, const unsigned long long *ukey,
                                              const int *uoff, const int *ucnt, int lane, int &st, int &len)
{
    st = 0;
    len = 0;
    if (lane >= 27) return;
    long long c[3];
    mls_cell(q, acc, P.edge, c);
    const long long x = c[0] + lane % 3 - 1, y = c[1] + (lane / 3) % 3 - 1, z = c[2] + lane / 9 - 1;
    if (x < 0 || y < 0 || z < 0 || x > (long long)MLS_CELL_MAX || y > (long long)MLS_CELL_MAX || z > (long long)MLS_CELL_MAX) return;
    mls_cell_range(ukey, uoff, ucnt, acc->nruns, mls_key(x, y, z), st, len);
}

// M6's per-point output count from the neighbour count
__device__ __forceinline__ int mls_samples(const MlsParams &P, int nb)
{
    return P.upsampling == 1 ? (int)floor((double)P.density / 2.0 / (double)nb) : 0;
}

// Pass 4: one warp per query (input order): M2's count over the 27 cells, the output count (0, 1 or k), the list of
// points too long for shared memory, and the per-block sums of processed, skipped and the longest list
__global__ void __launch_bounds__(MLS_BLOCK) k_mls_count(const float4 *__restrict__ in, int n, MlsParams P, MlsAcc *acc,
                                                         const float4 *__restrict__ spts, const unsigned long long *__restrict__ ukey,
                                                         const int *__restrict__ uoff, const int *__restrict__ ucnt,
                                                         int *__restrict__ nbr, long long *__restrict__ ocnt, int *__restrict__ long_list)
{
    __shared__ int s_proc, s_skip, s_max;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) { s_proc = 0; s_skip = 0; s_max = 0; }
    __syncthreads();
    const long long i = (long long)blockIdx.x * MLS_WARPS + wid;
    if (i < n) {
        const float4 q = in[2 * i];
        int cnt = 0;
        if (mls_finite(q)) {
            int st, len;
            mls_lane_cell(q, P, acc, ukey, uoff, ucnt, lane, st, len);
            for (int c = 0; c < 27; c++) {
                const int cs = __shfl_sync(0xffffffffu, st, c), cl = __shfl_sync(0xffffffffu, len, c);
                for (int s = cs + lane; s < cs + cl; s += 32) cnt += mls_d2(spts[s], q) <= P.r2f;
            }
            cnt = __reduce_add_sync(0xffffffffu, cnt);
        }
        if (lane == 0) {
            nbr[i] = cnt;
            long long oc = 0;
            if (cnt >= 3) {
                const int k = mls_samples(P, cnt);
                oc = k > 0 ? k : 1;
                atomicAdd(&s_proc, 1);
                if (cnt > MLS_LIST) long_list[atomicAdd(&acc->nlong, 1)] = (int)i;
            } else {
                atomicAdd(&s_skip, 1);
            }
            ocnt[i] = oc;
            atomicMax(&s_max, cnt);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        if (s_proc) atomicAdd(&acc->processed, s_proc);
        if (s_skip) atomicAdd(&acc->skipped, s_skip);
        if (s_max) atomicMax(&acc->max_nb, s_max);
    }
}

// Bitonic sort of K[0, m) (m a power of two) by one warp; __syncwarp orders the shared or global accesses between steps
__device__ __forceinline__ void mls_sort(unsigned long long *K, int m, int lane)
{
    for (int k = 2; k <= m; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < m; i += 32) {
                const int l = i ^ j;
                if (l > i) {
                    const unsigned long long a = K[i], b = K[l];
                    if ((a > b) == ((i & k) == 0)) { K[i] = b; K[l] = a; }
                }
            }
            __syncwarp();
        }
}

// M3's computeRoots (roots2: computeRoots2), ascending
__device__ __forceinline__ void mls_roots2(double b, double c, double *r)
{
    r[0] = 0.0;
    double d = b * b - 4.0 * c;
    if (d < 0.0) d = 0.0;
    const double sd = sqrt(d);
    r[2] = 0.5 * (b + sd);
    r[1] = 0.5 * (b - sd);
}
__device__ __forceinline__ void mls_roots3(const double *m, double *r) // m row-major 3 x 3
{
    const double m00 = m[0], m01 = m[1], m02 = m[2], m11 = m[4], m12 = m[5], m22 = m[8];
    const double c0 = m00 * m11 * m22 + 2.0 * m01 * m02 * m12 - m00 * m12 * m12 - m11 * m02 * m02 - m22 * m01 * m01;
    const double c1 = m00 * m11 - m01 * m01 + m00 * m22 - m02 * m02 + m11 * m22 - m12 * m12;
    const double c2 = m00 + m11 + m22;
    if (fabs(c0) < 2.220446049250313e-16) {
        mls_roots2(c2, c1, r);
        return;
    }
    const double s_inv3 = 1.0 / 3.0, s_sqrt3 = 1.7320508075688772; // sqrt(3.0), correctly rounded
    const double c2_over_3 = c2 * s_inv3;
    double a_over_3 = (c1 - c2 * c2_over_3) * s_inv3;
    if (a_over_3 > 0.0) a_over_3 = 0.0;
    const double half_b = 0.5 * (c0 + c2_over_3 * (2.0 * c2_over_3 * c2_over_3 - c1));
    double q = half_b * half_b + a_over_3 * a_over_3 * a_over_3;
    if (q > 0.0) q = 0.0;
    const double rho = sqrt(-a_over_3);
    const double theta = gem_atan2_d(sqrt(-q), half_b) * s_inv3;
    double sin_t, cos_t;
    gem_sincos_d(theta, &sin_t, &cos_t);
    r[0] = c2_over_3 + 2.0 * rho * cos_t;
    r[1] = c2_over_3 - rho * (cos_t + s_sqrt3 * sin_t);
    r[2] = c2_over_3 - rho * (cos_t - s_sqrt3 * sin_t);
    double t;
    if (r[0] >= r[1]) { t = r[0]; r[0] = r[1]; r[1] = t; }
    if (r[1] >= r[2]) {
        t = r[1]; r[1] = r[2]; r[2] = t;
        if (r[0] >= r[1]) { t = r[0]; r[0] = r[1]; r[1] = t; }
    }
    if (r[0] <= 0.0) mls_roots2(c2, c1, r);
}
__device__ __forceinline__ void mls_cross(const double *a, const double *b, double *c)
{
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ double mls_dot(const double *a, const double *b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
// eigen33: the unit eigenvector of the smallest eigenvalue of the symmetric s (row-major, overwritten)
__device__ __forceinline__ void mls_eigen33(double *s, double *ev)
{
    double scale = 0.0;
#pragma unroll
    for (int e = 0; e < 9; e++) scale = fabs(s[e]) > scale ? fabs(s[e]) : scale;
    if (scale <= 2.2250738585072014e-308) scale = 1.0;
#pragma unroll
    for (int e = 0; e < 9; e++) s[e] = s[e] / scale;
    double r[3];
    mls_roots3(s, r);
    s[0] -= r[0]; s[4] -= r[0]; s[8] -= r[0];
    double v1[3], v2[3], v3[3];
    mls_cross(s, s + 3, v1);
    mls_cross(s, s + 6, v2);
    mls_cross(s + 3, s + 6, v3);
    const double l1 = mls_dot(v1, v1), l2 = mls_dot(v2, v2), l3 = mls_dot(v3, v3);
    double v[3], l;
    if (l1 >= l2 && l1 >= l3) { v[0] = v1[0]; v[1] = v1[1]; v[2] = v1[2]; l = l1; }
    else if (l2 >= l1 && l2 >= l3) { v[0] = v2[0]; v[1] = v2[1]; v[2] = v2[2]; l = l2; }
    else { v[0] = v3[0]; v[1] = v3[1]; v[2] = v3[2]; l = l3; }
    const double sl = sqrt(l);
#pragma unroll
    for (int a = 0; a < 3; a++) ev[a] = v[a] / sl;
}

__device__ __forceinline__ unsigned long long mls_splitmix(unsigned long long x)
{
    unsigned long long z = x + 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ float mls_draw(const MlsParams &P, unsigned i, unsigned long long j)
{
    const unsigned long long x = mls_splitmix(P.seed ^ ((unsigned long long)i << 32) ^ j);
    return P.lo + ((float)(x >> 40) * 0x1p-24f) * (P.hi - P.lo);
}

// M7: one output record at `slot` if it lies below the capacity
__device__ __forceinline__ void mls_emit(float4 *__restrict__ out, long long capacity, long long slot, double x, double y, double z,
                                         const float4 &attr)
{
    if (slot >= capacity) return;
    out[2 * slot] = make_float4((float)x, (float)y, (float)z, 1.0f);
    out[2 * slot + 1] = make_float4(__uint_as_float(__float_as_uint(attr.x) | 0xff000000u), attr.y, attr.z, attr.w);
}

// Pass 5: M2's list, M3-M7 for one query per warp.  LONG = false: one warp per input point, lists of at most MLS_LIST
// entries sorted in shared memory (longer ones are skipped).  LONG = true: persistent warps over the long list, each
// sorting in its own global slice of `slice` keys.  Everything below runs in the order M3 and M4 define: the sequential
// chains (three centroid sums, six covariance sums, the nc (nc + 1) / 2 + nc normal-equation entries) are spread over
// the lanes, one chain per lane at a time, with 32 neighbours staged in shared memory per step.
template <bool LONG>
__global__ void __launch_bounds__(MLS_BLOCK) k_mls_fit(const float4 *__restrict__ in, int n, MlsParams P, MlsAcc *acc,
                                                       const float4 *__restrict__ spts, const unsigned long long *__restrict__ ukey,
                                                       const int *__restrict__ uoff, const int *__restrict__ ucnt,
                                                       const int *__restrict__ nbr, const long long *__restrict__ ooff,
                                                       const int *__restrict__ long_list, unsigned long long *__restrict__ gkeys,
                                                       int slice, float4 *__restrict__ out, long long capacity)
{
    __shared__ unsigned long long s_keys[LONG ? 1 : MLS_WARPS][LONG ? 1 : MLS_LIST];
    __shared__ double s_stage[MLS_WARPS][32 * MLS_STAGE];
    __shared__ double s_vec[MLS_WARPS][48]; // normal 0-2, point 3-5, u axis 6-8, v axis 9-11, rhs / y / c 12-32
    __shared__ int s_fitted;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_fitted = 0;
    __syncthreads();
    double *S = s_stage[wid], *V = s_vec[wid];
    const int nc = P.nc, ntri = nc * (nc + 1) / 2, ne = ntri + nc;
    // the normal-equation entries of this lane: e = lane + 32 t, A(a, b) for e < ntri (row-major lower triangle), rhs(a)
    // (b = the staged f) after it
    int ea[8], eb[8];
#pragma unroll
    for (int t = 0; t < 8; t++) {
        const int e = lane + 32 * t;
        ea[t] = -1;
        eb[t] = 0;
        if (e < ntri) {
            int a = 0;
            while ((a + 1) * (a + 2) / 2 <= e) a++;
            ea[t] = a;
            eb[t] = e - a * (a + 1) / 2;
        } else if (e < ne) {
            ea[t] = e - ntri;
            eb[t] = MLS_MAXC;
        }
    }
    const long long gw = (long long)blockIdx.x * MLS_WARPS + wid;
    const long long nq = LONG ? (long long)acc->nlong : (long long)n;
    const long long step = LONG ? (long long)gridDim.x * MLS_WARPS : nq;
    for (long long t0 = gw; t0 < nq; t0 += step) {
        const int i = LONG ? long_list[t0] : (int)t0;
        const int nb = nbr[i];
        if (nb < 3 || (!LONG && nb > MLS_LIST)) continue;
        unsigned long long *K = LONG ? gkeys + (size_t)gw * (size_t)slice : s_keys[LONG ? 0 : wid];
        const float4 q = in[2 * (long long)i];
        // M2: gather (d2, index) keys, then sort them; the padding sorts last
        {
            int st, len, pos = 0;
            mls_lane_cell(q, P, acc, ukey, uoff, ucnt, lane, st, len);
            for (int c = 0; c < 27; c++) {
                const int cs = __shfl_sync(0xffffffffu, st, c), cl = __shfl_sync(0xffffffffu, len, c);
                for (int b = 0; b < cl; b += 32) {
                    float d2 = 0.0f;
                    int j = 0;
                    bool hit = false;
                    if (b + lane < cl) {
                        const float4 p = spts[cs + b + lane];
                        d2 = mls_d2(p, q);
                        j = __float_as_int(p.w);
                        hit = d2 <= P.r2f;
                    }
                    const unsigned bal = __ballot_sync(0xffffffffu, hit);
                    if (hit) K[pos + __popc(bal & ((1u << lane) - 1u))] = ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned)j;
                    pos += __popc(bal);
                }
            }
            int m = 32;
            while (m < nb) m <<= 1;
            for (int e = nb + lane; e < m; e += 32) K[e] = ~0ull;
            __syncwarp();
            mls_sort(K, m, lane);
        }
        // M3: centroid (lanes 0-2), then covariance (lanes 0-5), 32 neighbours staged at a time
        float *F = reinterpret_cast<float *>(S);
        double c0 = 0.0, c1 = 0.0, c2 = 0.0;
        {
            double acc1 = 0.0;
            for (int b = 0; b < nb; b += 32) {
                const int mm = min(32, nb - b);
                if (lane < mm) {
                    const float4 p = in[2 * (long long)(unsigned)(K[b + lane] & 0xffffffffu)];
                    F[3 * lane] = p.x; F[3 * lane + 1] = p.y; F[3 * lane + 2] = p.z;
                }
                __syncwarp();
                if (lane < 3)
                    for (int k = 0; k < mm; k++) acc1 += F[3 * k + lane];
                __syncwarp();
            }
            acc1 = acc1 / (double)nb;
            c0 = __shfl_sync(0xffffffffu, acc1, 0);
            c1 = __shfl_sync(0xffffffffu, acc1, 1);
            c2 = __shfl_sync(0xffffffffu, acc1, 2);
        }
        double cov = 0.0;
        {
            // lanes 0-5: (1,1) y y, (1,2) y z, (2,2) z z, (0,0) x x, (0,1) y x, (0,2) z x
            const int ia = lane == 3 ? 0 : lane == 4 || lane == 1 || lane == 0 ? 1 : 2;
            const int ib = lane == 0 ? 1 : lane == 1 || lane == 2 ? 2 : 0;
            const double ca = ia == 0 ? c0 : ia == 1 ? c1 : c2, cb = ib == 0 ? c0 : ib == 1 ? c1 : c2;
            for (int b = 0; b < nb; b += 32) {
                const int mm = min(32, nb - b);
                if (lane < mm) {
                    const float4 p = in[2 * (long long)(unsigned)(K[b + lane] & 0xffffffffu)];
                    F[3 * lane] = p.x; F[3 * lane + 1] = p.y; F[3 * lane + 2] = p.z;
                }
                __syncwarp();
                if (lane < 6)
                    for (int k = 0; k < mm; k++) cov += (F[3 * k + ia] - ca) * (F[3 * k + ib] - cb);
                __syncwarp();
            }
        }
        const bool attempt = P.fit && nb >= nc;
        {
            const double c11 = __shfl_sync(0xffffffffu, cov, 0), c12 = __shfl_sync(0xffffffffu, cov, 1);
            const double c22 = __shfl_sync(0xffffffffu, cov, 2), c00 = __shfl_sync(0xffffffffu, cov, 3);
            const double c01 = __shfl_sync(0xffffffffu, cov, 4), c02 = __shfl_sync(0xffffffffu, cov, 5);
            if (lane == 0) {
                double m9[9] = {c00, c01, c02, c01, c11, c12, c02, c12, c22}, nv[3];
                mls_eigen33(m9, nv);
                const double d = -((nv[0] * c0 + nv[2] * c2) + (nv[1] * c1 + 0.0));
                const double qd[3] = {(double)q.x, (double)q.y, (double)q.z};
                const double dist = mls_dot(qd, nv) + d;
                for (int a = 0; a < 3; a++) { V[a] = nv[a]; V[3 + a] = qd[a] - dist * nv[a]; V[6 + a] = 0.0; V[9 + a] = 0.0; }
                if (attempt) {
                    // unitOrthogonal, then u = n x v
                    double va[3], ua[3];
                    const double prec = 1e-12;
                    if (!(fabs(nv[0]) <= fabs(nv[2]) * prec) || !(fabs(nv[1]) <= fabs(nv[2]) * prec)) {
                        const double inv = 1.0 / sqrt(nv[0] * nv[0] + nv[1] * nv[1]);
                        va[0] = -nv[1] * inv; va[1] = nv[0] * inv; va[2] = 0.0;
                    } else {
                        const double inv = 1.0 / sqrt(nv[1] * nv[1] + nv[2] * nv[2]);
                        va[0] = 0.0; va[1] = -nv[2] * inv; va[2] = nv[1] * inv;
                    }
                    mls_cross(nv, va, ua);
                    for (int a = 0; a < 3; a++) { V[6 + a] = ua[a]; V[9 + a] = va[a]; }
                }
            }
            __syncwarp();
        }
        const double nx = V[0], ny = V[1], nz = V[2], px = V[3], py = V[4], pz = V[5];
        const double ux = V[6], uy = V[7], uz = V[8], vx = V[9], vy = V[10], vz = V[11];
        bool fitted = false;
        if (attempt) {
            // M4: the normal equations, one sequential chain per entry
            double sum[8];
#pragma unroll
            for (int t = 0; t < 8; t++) sum[t] = 0.0;
            for (int b = 0; b < nb; b += 32) {
                const int mm = min(32, nb - b);
                __syncwarp();
                if (lane < mm) {
                    const float4 p = in[2 * (long long)(unsigned)(K[b + lane] & 0xffffffffu)];
                    const double de[3] = {p.x - px, p.y - py, p.z - pz};
                    const float d2f = (float)mls_dot(de, de);
                    const double w = gem_exp_d(-d2f / P.gauss);
                    const double u = (de[0] * ux + de[1] * uy) + de[2] * uz;
                    const double v = (de[0] * vx + de[1] * vy) + de[2] * vz;
                    const double f = (de[0] * nx + de[1] * ny) + de[2] * nz;
                    double *row = S + lane * MLS_STAGE;
                    int j = 0;
                    double upow = 1.0;
                    for (int ui = 0; ui <= P.order; ui++) {
                        double vpow = 1.0;
                        for (int vi = 0; vi <= P.order - ui; vi++) {
                            row[j++] = upow * vpow;
                            vpow *= v;
                        }
                        upow *= u;
                    }
                    row[MLS_MAXC] = f;
                    row[MLS_MAXC + 1] = w;
                }
                __syncwarp();
                for (int k = 0; k < mm; k++) {
                    const double *row = S + k * MLS_STAGE;
                    const double w = row[MLS_MAXC + 1];
#pragma unroll
                    for (int t = 0; t < 8; t++)
                        if (ea[t] >= 0) sum[t] += (row[ea[t]] * w) * row[eb[t]];
                }
            }
            __syncwarp();
            // A (lower triangle, row-major 21 x 21) and rhs into shared memory; S is free again
            double *L = S, *Y = V + 12;
#pragma unroll
            for (int t = 0; t < 8; t++)
                if (ea[t] >= 0) {
                    if (eb[t] == MLS_MAXC) Y[ea[t]] = sum[t];
                    else L[ea[t] * MLS_MAXC + eb[t]] = sum[t];
                }
            __syncwarp();
            // left-looking Cholesky, column by column, lane i owns row i
            bool ok = true;
            for (int jc = 0; jc < nc; jc++) {
                double s = 0.0;
                if (lane >= jc && lane < nc) {
                    s = L[lane * MLS_MAXC + jc];
                    for (int k = 0; k < jc; k++) s -= L[lane * MLS_MAXC + k] * L[jc * MLS_MAXC + k];
                }
                const double piv = __shfl_sync(0xffffffffu, s, jc);
                if (!(piv > 0.0) || !isfinite(piv)) { ok = false; break; }
                const double ljj = sqrt(piv);
                __syncwarp();
                if (lane == jc) L[jc * MLS_MAXC + jc] = ljj;
                else if (lane > jc && lane < nc) L[lane * MLS_MAXC + jc] = s / ljj;
                __syncwarp();
            }
            if (ok) {
                if (lane == 0) { // forward, then back substitution, both in place: Y holds rhs, then y, then c
                    for (int a = 0; a < nc; a++) {
                        double s = Y[a];
                        for (int k = 0; k < a; k++) s -= L[a * MLS_MAXC + k] * Y[k];
                        Y[a] = s / L[a * MLS_MAXC + a];
                    }
                    for (int a = nc - 1; a >= 0; a--) {
                        double s = Y[a];
                        for (int k = a + 1; k < nc; k++) s -= L[k * MLS_MAXC + a] * Y[k];
                        Y[a] = s / L[a * MLS_MAXC + a];
                    }
                }
                __syncwarp();
                fitted = isfinite(Y[0]);
            }
        }
        if (lane == 0 && fitted) atomicAdd(&s_fitted, 1);
        // M5 / M6 / M7
        const float4 attr = in[2 * (long long)i + 1];
        const long long base = ooff[i];
        const int k = mls_samples(P, nb);
        const double *C = V + 12;
        if (k <= 0) {
            if (lane == 0) {
                const double c = fitted ? C[0] : 0.0;
                if (fitted) mls_emit(out, capacity, base, px + c * nx, py + c * ny, pz + c * nz, attr);
                else mls_emit(out, capacity, base, px, py, pz, attr);
            }
        } else {
            // rejection sampling: lane l tests draw pair t0 + l; a ballot and a prefix count keep M6's draw order
            int got = 0;
            for (unsigned long long t = 0; got < k; t += 32) {
                const unsigned long long j = 2 * (t + lane);
                const float u = mls_draw(P, (unsigned)i, j), v = mls_draw(P, (unsigned)i, j + 1);
                const bool accept = !((double)u * (double)u + (double)v * (double)v > P.r2q);
                const unsigned bal = __ballot_sync(0xffffffffu, accept);
                const int rank = got + __popc(bal & ((1u << lane) - 1u));
                if (accept && rank < k) {
                    double x = (px + ux * u) + vx * v, y = (py + uy * u) + vy * v, z = (pz + uz * u) + vz * v;
                    if (fitted) {
                        double h = 0.0, upow = 1.0;
                        int jj = 0;
                        for (int ui = 0; ui <= P.order; ui++) {
                            double vpow = 1.0;
                            for (int vi = 0; vi <= P.order - ui; vi++) {
                                h += upow * vpow * C[jj++];
                                vpow *= v;
                            }
                            upow *= u;
                        }
                        x = x + nx * h;
                        y = y + ny * h;
                        z = z + nz * h;
                    }
                    mls_emit(out, capacity, base + rank, x, y, z, attr);
                }
                got += __popc(bal);
            }
        }
        __syncwarp();
    }
    __syncthreads();
    if (threadIdx.x == 0 && s_fitted) atomicAdd(&acc->fitted, s_fitted);
}

} // namespace gem
