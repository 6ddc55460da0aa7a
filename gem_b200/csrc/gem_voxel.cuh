// gem_voxel.cuh -- the VoxelGrid pre-filter of GEM's demo launches on the device (DESIGN.md f9): pcl_ros's VoxelGrid
// nodelet, i.e. pcl::VoxelGrid<pcl::PCLPointCloud2>::applyFilter of PCL 1.8 with downsample_all_data_ true, over
// n x float4 {x, y, z, intensity} in device memory.  PCL is an unpinned dependency; its definitions are restated here,
// in include/gem_b200.h and in tests/orc_voxel_grid.c.
//
// V1 Leaf: float leaf[3] (setLeafSize takes floats), inv[a] = 1.0f / leaf[a] in float.  A leaf that is not finite or
//    is <= 0 is an error (checked by the caller).
// V2 Index pass (which points are used): with a field selected, its float value v is cut when
//    (double)v > limit_max || (double)v < limit_min (negative = 0), or when (double)v < limit_max && (double)v > limit_min
//    (negative = 1); the limits are doubles, a NaN v passes.  A point that passes (every point without a field) is then
//    cut when x, y or z is not finite.  This specialisation tests finiteness without reading is_dense.
// V3 Bounds (getMinMax3D): the same two tests with the limits rounded to float and compared in float; min_p / max_p are
//    the per-axis float min / max over the survivors, from FLT_MAX / -FLT_MAX.  Every V2 survivor is a V3 survivor (no
//    float lies strictly between a double limit and its float rounding), so no voxel coordinate below is negative.
// V4 Overflow: d[a] = (int64)((max_p[a] - min_p[a]) * inv[a]) + 1, the product in float.  If d[0] d[1] d[2] > INT32_MAX
//    the output is the input unchanged (all n points in order, bit for bit).  DEFINED: a product that is not finite, or
//    a quotient >= 2^62, also counts as overflow (PCL's cast is undefined there); the product of the d is the
//    mathematical one (PCL's int64 product could wrap).
// V5 Nothing used (no V3 survivor, n = 0 included): count 0.  DEFINED: PCL casts -inf to int64 there.
// V6 Voxel and order: min_b[a] = floor(min_p[a] * inv[a]), max_b[a] likewise, ijk[a] = floor(p[a] * inv[a]) - min_b[a],
//    idx = ijk0 + ijk1 div0 + ijk2 div0 div1 with div[a] = max_b[a] - min_b[a] + 1; output in ascending idx, i.e.
//    lexicographic in (ijk2, ijk1, ijk0).  floor of a float product is exact whether it resolves to the float or the
//    double overload, so the overload changes nothing.  The subtraction is exact here (in double, as with the double
//    overload), and min_b stays a floor value rather than an int, so that coordinates beyond the int range with a small
//    span are defined.  DEFINED: when div0 div1 div2 exceeds 2^31 although V4 passed (PCL's int idx overflows), the order
//    is still lexicographic in (ijk2, ijk1, ijk0); the 64-bit mixed-radix key below is that order in every case.
// V7 Order inside a voxel: DEFINED as ascending input index (PCL's std::sort is not stable; its order inside a voxel
//    is libstdc++'s introsort and only changes the rounding of the sums).  The stable radix sort gives it.
// V8 Centroid: each of the four components starts at +0.0f, c += p in float point by point in V7 order, then one IEEE
//    division c /= (float)count per component.  Intensity is averaged like x, y, z; a single point at -0.0 gives +0.0.
// V9 Output: min(count, capacity) float4 into caller-owned device memory, count always reported.
//
// Every decision is taken on the device (DESIGN.md f20): a step reads its input count from device memory (the previous
// step's count in a chain), runs its kernels and its sort at a host-known upper bound N of that count, and leaves its
// count, V2 count and mode in its VoxStep.  Entries past the count take the cut points' key, so they join the run that
// is dropped.  The sort runs on the fixed width GEM_VOX_KEY_BITS (gem_voxgrid.h proves that every key fits).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "gem_kernels.cuh"
#include "gem_voxgrid.h"

namespace gem {

constexpr int VOX_BLOCK = 256;
constexpr int VOX_SHORT = 32; // a voxel of at most this many points is summed by its own lane, a longer one by its warp

struct VoxParams {
    float inv[3];
    int field;              // -1 none, 0..3: x, y, z, intensity
    double lmin, lmax;      // V2: the nodelet's double limits
    float flmin, flmax;     // V3: the same rounded to float
    int negative;
};

// what the bounds pass accumulates, and the run count of the sort
struct VoxAcc {
    unsigned mn[3], mx[3];  // order-preserving encodings of the V3 bounds
    int used, bounded;      // V2 survivors, V3 survivors
    int nruns;              // runs of the sorted keys (the last one holds the cut points when used < n)
    int pad;
};

// the voxel grid once V4 has passed: min_b as floor values, the mixed radix of the key, the key of a cut point
struct VoxGrid {
    double minb[3];
    unsigned long long div0, div01, cut_key;
};

// one step on the device: its bounds pass, its grid, and what it decided (mode GEM_VOX_*; count: output points; drop: the
// last run of the sorted keys holds cut points or entries past the count)
struct VoxStep {
    VoxAcc acc;
    VoxGrid grid;
    int mode, count, drop;
    int n; // step 0: its input count (k_vox_init); a later step reads its predecessor's count
};

// Order-preserving encoding of a float (min / max are exact, so the reduction order is free; -0 and +0 only differ in
// the sign of a bound, which floor and the differences below map to the same integers)
__host__ __device__ __forceinline__ unsigned vg_key(float f)
{
    unsigned u;
    memcpy(&u, &f, sizeof u);
    return (u >> 31) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float vg_unkey(unsigned k)
{
    const unsigned u = (k >> 31) ? (k & 0x7fffffffu) : ~k;
    float f;
    memcpy(&f, &u, sizeof f);
    return f;
}

__device__ __forceinline__ float vg_comp(const float4 &p, int a) { return a == 0 ? p.x : a == 1 ? p.y : a == 2 ? p.z : p.w; }
__device__ __forceinline__ bool vg_finite(const float4 &p) { return isfinite(p.x) && isfinite(p.y) && isfinite(p.z); }
// V2: used by the index pass
__device__ __forceinline__ bool vg_used(const VoxParams &P, const float4 &p)
{
    if (P.field >= 0) {
        const double v = (double)vg_comp(p, P.field);
        if (P.negative ? (v < P.lmax && v > P.lmin) : (v > P.lmax || v < P.lmin)) return false;
    }
    return vg_finite(p);
}
// V3: counted in the bounds
__device__ __forceinline__ bool vg_bounded(const VoxParams &P, const float4 &p)
{
    if (P.field >= 0) {
        const float v = vg_comp(p, P.field);
        if (P.negative ? (v < P.flmax && v > P.flmin) : (v > P.flmax || v < P.flmin)) return false;
    }
    return vg_finite(p);
}

// Pass 0: the steps' accumulators start empty (one thread per step); step 0 takes its input count n0
__global__ void k_vox_init(VoxStep *st, int nsteps, int n0)
{
    const int s = threadIdx.x;
    if (s >= nsteps) return;
    VoxStep z{};
    z.n = s == 0 ? n0 : 0;
    for (int a = 0; a < 3; a++) { z.acc.mn[a] = vg_key(3.402823466e38f); z.acc.mx[a] = vg_key(-3.402823466e38f); }
    st[s] = z;
}

// Pass 1: V2 count, V3 count and bounds.  Grid-stride over 16-byte loads; per warp __reduce_*_sync, per block through
// shared memory, then one atomic per quantity and block.
__global__ void __launch_bounds__(VOX_BLOCK) k_vox_bounds(const float4 *__restrict__ in, int N, const int *nin, VoxParams P, VoxAcc *acc)
{
    __shared__ unsigned sh[VOX_BLOCK / 32][8];
    const int n = min(N, *nin);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned mn[3], mx[3], used = 0, bounded = 0;
    for (int a = 0; a < 3; a++) { mn[a] = vg_key(3.402823466e38f); mx[a] = vg_key(-3.402823466e38f); }
    for (long long i = (long long)blockIdx.x * VOX_BLOCK + threadIdx.x; i < n; i += (long long)gridDim.x * VOX_BLOCK) {
        const float4 p = in[i];
        used += vg_used(P, p);
        if (vg_bounded(P, p)) {
            bounded++;
            const unsigned kx = vg_key(p.x), ky = vg_key(p.y), kz = vg_key(p.z);
            mn[0] = min(mn[0], kx); mx[0] = max(mx[0], kx);
            mn[1] = min(mn[1], ky); mx[1] = max(mx[1], ky);
            mn[2] = min(mn[2], kz); mx[2] = max(mx[2], kz);
        }
    }
    unsigned v[8] = {used, bounded, mn[0], mn[1], mn[2], mx[0], mx[1], mx[2]};
    v[0] = __reduce_add_sync(0xffffffffu, v[0]);
    v[1] = __reduce_add_sync(0xffffffffu, v[1]);
#pragma unroll
    for (int q = 2; q < 5; q++) v[q] = __reduce_min_sync(0xffffffffu, v[q]);
#pragma unroll
    for (int q = 5; q < 8; q++) v[q] = __reduce_max_sync(0xffffffffu, v[q]);
    if (lane == 0) {
#pragma unroll
        for (int q = 0; q < 8; q++) sh[wid][q] = v[q];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int r = 1; r < VOX_BLOCK / 32; r++) {
            v[0] += sh[r][0]; v[1] += sh[r][1];
            for (int q = 2; q < 5; q++) v[q] = min(v[q], sh[r][q]);
            for (int q = 5; q < 8; q++) v[q] = max(v[q], sh[r][q]);
        }
        if (v[0]) atomicAdd(&acc->used, (int)v[0]);
        if (v[1]) {
            atomicAdd(&acc->bounded, (int)v[1]);
            for (int a = 0; a < 3; a++) { atomicMin(&acc->mn[a], v[2 + a]); atomicMax(&acc->mx[a], v[5 + a]); }
        }
    }
}

// Between the passes, one thread: V5, V4 and V6 from the bounds (gem_voxgrid.h).  wide_passes: a GEM_VOX_WIDE grid
// passes the input through (the asynchronous chain, which cannot refuse); otherwise it stays GEM_VOX_WIDE, writes nothing
// and gem_voxel_grid refuses it.
__global__ void k_vox_decide(VoxParams P, int N, const int *nin, VoxStep *st, int wide_passes)
{
    const int n = min(N, *nin);
    VoxStep &S = *st;
    S.drop = S.acc.used < N ? 1 : 0;
    S.mode = GEM_VOX_EMPTY;
    S.count = 0;
    if (S.acc.bounded == 0) return; // V5
    float mn[3], mx[3];
    for (int a = 0; a < 3; a++) { mn[a] = vg_unkey(S.acc.mn[a]); mx[a] = vg_unkey(S.acc.mx[a]); }
    VoxGrid G{};
    const int mode = gem_vox_layout(mn, mx, P.inv, G.minb, &G.div0, &G.div01, &G.cut_key);
    if (mode == GEM_VOX_PASS || (mode == GEM_VOX_WIDE && wide_passes && S.acc.used > 0)) { // V4: the input unchanged
        S.mode = GEM_VOX_PASS;
        S.count = n;
    } else if (S.acc.used > 0) {
        S.mode = mode;
        S.grid = G; // count: k_vox_centroids
    }
}

// Pass 2: one key per point, V6's mixed-radix index of (ijk2, ijk1, ijk0) for a V2 survivor, cut_key (one past the
// largest voxel key) for a cut point, so that the cut points sort last as one run; the value is the input index.
// floorf of the float product is exact, the difference with the floor value min_b is exact in double, and lies in
// [0, div) because every survivor lies inside the V3 bounds.
// Entries past the step's count take cut_key as well; a step that is not GEM_VOX_GRID writes key 0 (its sort is not read).
__global__ void __launch_bounds__(VOX_BLOCK) k_vox_keys(const float4 *__restrict__ in, int N, const int *nin, VoxParams P,
                                                        const VoxStep *st, unsigned long long *__restrict__ key, int *__restrict__ idx)
{
    const long long i = (long long)blockIdx.x * VOX_BLOCK + threadIdx.x;
    if (i >= N) return;
    unsigned long long k = 0;
    if (st->mode == GEM_VOX_GRID) {
        const VoxGrid &G = st->grid;
        k = G.cut_key;
        if (i < *nin) {
            const float4 p = in[i];
            if (vg_used(P, p)) {
                const unsigned long long i0 = (unsigned long long)(long long)((double)floorf(p.x * P.inv[0]) - G.minb[0]);
                const unsigned long long i1 = (unsigned long long)(long long)((double)floorf(p.y * P.inv[1]) - G.minb[1]);
                const unsigned long long i2 = (unsigned long long)(long long)((double)floorf(p.z * P.inv[2]) - G.minb[2]);
                k = i0 + i1 * G.div0 + i2 * G.div01;
            }
        }
    }
    key[i] = k;
    idx[i] = (int)i;
}

// V8's sum with x86-64 (SSE) NaN results, DEFINED: IEEE 754 leaves NaN bits open, the reference's host gives c + p the
// first NaN operand (c, then p) quieted, and an invalid inf - inf the default NaN 0xFFC00000; once c is NaN it stays
// that NaN, and so does c / count.  The device's own NaN is canonical, so the chain of plain adds stays as it is and
// the bits of the first NaN it produces are recorded beside it, off the chain.
struct VgSum {
    float4 s = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    uint4 nan = make_uint4(0u, 0u, 0u, 0u);
};
__device__ __forceinline__ void vg_add1(float &s, unsigned &nb, float p)
{
    s = s + p;
    if (nb == 0u && s != s) nb = (p != p) ? (__float_as_uint(p) | 0x00400000u) : 0xffc00000u;
}
__device__ __forceinline__ void vg_add(VgSum &c, const float4 &p)
{
    vg_add1(c.s.x, c.nan.x, p.x); vg_add1(c.s.y, c.nan.y, p.y);
    vg_add1(c.s.z, c.nan.z, p.z); vg_add1(c.s.w, c.nan.w, p.w);
}
__device__ __forceinline__ void vg_add_plain(float4 &s, const float4 &p)
{
    s.x = s.x + p.x; s.y = s.y + p.y; s.z = s.z + p.z; s.w = s.w + p.w;
}
__device__ __forceinline__ bool vg_any_nan(const float4 &s) { return s.x != s.x || s.y != s.y || s.z != s.z || s.w != s.w; }
__device__ __forceinline__ float vg_div1(float s, unsigned nb, float d) { return nb ? __uint_as_float(nb) : s / d; }
__device__ __forceinline__ float4 vg_centroid(const VgSum &c, int count)
{
    const float d = (float)count;
    return make_float4(vg_div1(c.s.x, c.nan.x, d), vg_div1(c.s.y, c.nan.y, d), vg_div1(c.s.z, c.nan.z, d), vg_div1(c.s.w, c.nan.w, d));
}

// Pass 3 of a GEM_VOX_PASS step: the input copied, min(count, capacity) points
// Pass 3 of a GEM_VOX_GRID step: V8, one thread per voxel (run of the sorted keys; sidx holds each run's input indices in ascending order).  A
// voxel of at most VOX_SHORT points is summed by its own lane.  The longer voxels of a warp are taken one after another
// by the whole warp: the lanes gather 32 points at a time into shared memory (the next 32 are loaded while the current
// ones are summed) and lane 0 adds them in order, so the sequential chain is V8's and nothing longer.  The centroid goes
// straight to its voxel's output slot when that lies below the capacity.
__global__ void __launch_bounds__(VOX_BLOCK) k_vox_centroids(const float4 *__restrict__ in, const int *__restrict__ sidx,
                                                             const int *__restrict__ cnt, const int *__restrict__ off,
                                                             VoxStep *st, float4 *__restrict__ out, int capacity)
{
    __shared__ float4 stage[VOX_BLOCK / 32][32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long v = (long long)blockIdx.x * VOX_BLOCK + threadIdx.x;
    const int mode = st->mode;
    if (mode == GEM_VOX_PASS) {
        if (v < st->count && v < capacity) out[v] = in[v];
        return;
    }
    if (mode != GEM_VOX_GRID) return;
    const int nvox = st->acc.nruns - st->drop;
    if (v == 0) st->count = nvox;
    if ((long long)blockIdx.x * VOX_BLOCK >= nvox) return; // whole warps leave together below
    const int c = v < nvox ? cnt[v] : 0;
    const int o = v < nvox ? off[v] : 0;
    // NaN is sticky, so the chains below are plain adds; a stretch that turns a sum into NaN is summed once more with
    // the NaN bits recorded (vg_add), from the partial sum it started with
    if (c > 0 && c <= VOX_SHORT) {
        VgSum s;
#pragma unroll 4
        for (int j = 0; j < c; j++) vg_add_plain(s.s, in[sidx[o + j]]);
        if (vg_any_nan(s.s)) {
            s = VgSum();
            for (int j = 0; j < c; j++) vg_add(s, in[sidx[o + j]]);
        }
        if (v < capacity) out[v] = vg_centroid(s, c);
    }
    unsigned todo = __ballot_sync(0xffffffffu, c > VOX_SHORT);
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const int lc = __shfl_sync(0xffffffffu, c, src), lo = __shfl_sync(0xffffffffu, o, src);
        VgSum s;
        float4 p = in[sidx[lo + lane]]; // lc > 32: the first batch is full
        for (int base = 0; base < lc; base += 32) {
            stage[wid][lane] = p;
            __syncwarp();
            const int k = base + 32 + lane;
            if (k < lc) p = in[sidx[lo + k]];
            if (lane == 0) {
                const int m = lc - base < 32 ? lc - base : 32;
                const VgSum s0 = s;
                if (m == 32) { // unrolled, so that the shared loads run ahead of the chain of adds
#pragma unroll
                    for (int j = 0; j < 32; j++) vg_add_plain(s.s, stage[wid][j]);
                } else {
                    for (int j = 0; j < m; j++) vg_add_plain(s.s, stage[wid][j]);
                }
                if (vg_any_nan(s.s)) {
                    s = s0;
                    for (int j = 0; j < m; j++) vg_add(s, stage[wid][j]);
                }
            }
            __syncwarp();
        }
        const long long vs = v - lane + src;
        if (lane == 0 && vs < capacity) out[vs] = vg_centroid(s, lc);
    }
}

} // namespace gem
