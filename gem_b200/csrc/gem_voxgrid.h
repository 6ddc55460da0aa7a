/* gem_voxgrid.h -- the decision of one VoxelGrid step once its bounds are known (gem_voxel.cuh, V4-V6 of DESIGN.md f9),
 * in a form that both nvcc (the one-thread kernel k_vox_decide) and a C++ compiler (tests/voxgrid_host.cpp) accept.  The
 * float operations are spelled with __fsub_rn / __fmul_rn on the device, so that nothing is contracted, and are the
 * plain IEEE operations of a host without FMA elsewhere: both give the correctly rounded float results.
 *
 * Key width.  After V4 has passed, every voxel key lies below 2^GEM_VOX_KEY_BITS, so the sort can run on a fixed
 * width that no host read-back decides.  Proof, per axis a (drop a): let mn < mx be the float bounds, M = max(|mn|, |mx|),
 * s = mx - mn exactly and q = fl(fl(s) inv), so d = floor(q) + 1 > q.  Two distinct floats satisfy s >= ulp(M) / 2 >
 * M 2^-25 (same sign: the gap is at least the ulp of the lower binade; opposite signs: s >= M).  With A = fl(mx inv),
 * B = fl(mn inv) finite, div - 1 = floor(A) - floor(B) < A - B + 1 <= s inv + (ulp(A) + ulp(B)) / 2 + 1, and
 * ulp(A), ulp(B) <= 2^-23 M inv (1 + 2^-24) < 4.001 s inv.  Since fl(s) >= s (1 - 2^-24) and q >= fl(s) inv (1 - 2^-24),
 * s inv <= 1.001 q < 1.001 d, so div < 5.01 d + 2 <= 8 d (d >= 1; subnormal products give div <= 2 <= 8 d, and mn = mx
 * gives div = 1).  V4 leaves d0 d1 d2 <= 2^31 - 1, so cut_key = div0 div1 div2 < 2^9 2^31 = 2^40, and every key,
 * the cut key included, fits GEM_VOX_KEY_BITS = 40 bits.  tests/test_prefilter_cpu.py checks the bound on crafted clouds.
 * A product mn inv or mx inv that is not finite (a cloud at |x| near FLT_MAX with a span of few voxels) leaves no
 * integer voxel index: that is GEM_VOX_WIDE. */
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define GEM_VF static __host__ __device__ __forceinline__
#else
#define GEM_VF static inline
#endif

#define GEM_VOX_KEY_BITS 40

enum { GEM_VOX_EMPTY = 0, GEM_VOX_PASS = 1, GEM_VOX_GRID = 2, GEM_VOX_WIDE = 3 };

GEM_VF float gem_vox_sub(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}
GEM_VF float gem_vox_mul(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}

/* V4-V6 from the V3 bounds of a step with bounded > 0 survivors: GEM_VOX_PASS (V4's overflow), GEM_VOX_WIDE, or
 * GEM_VOX_GRID with min_b, the mixed radix div0 / div0 div1 and the cut points' key (one past the largest voxel key) */
GEM_VF int gem_vox_layout(const float mn[3], const float mx[3], const float inv[3], double minb[3], unsigned long long *div0,
                          unsigned long long *div01, unsigned long long *cut_key)
{
    /* V4: d[a] = (int64)((max_p - min_p) * inv) + 1, the product in float.  DEFINED: a product that is not finite or a
     * quotient >= 2^62 is an overflow; the product of the d is the mathematical one (each step below stays under 2^62) */
    long long d[3] = {0, 0, 0};
    int over = 0;
    for (int a = 0; a < 3; a++) {
        const float q = gem_vox_mul(gem_vox_sub(mx[a], mn[a]), inv[a]);
        if (!isfinite(q) || q >= 4611686018427387904.0f) over = 1;
        else d[a] = (long long)q + 1;
    }
    if (over || d[0] > INT32_MAX || d[1] > INT32_MAX || d[2] > INT32_MAX || d[0] * d[1] > INT32_MAX || d[0] * d[1] * d[2] > INT32_MAX)
        return GEM_VOX_PASS;
    /* V6: min_b, max_b as floor values of float products (exact in either overload), div from their exact difference */
    unsigned long long div[3];
    for (int a = 0; a < 3; a++) {
        const float lo = gem_vox_mul(mn[a], inv[a]), hi = gem_vox_mul(mx[a], inv[a]);
        if (!isfinite(lo) || !isfinite(hi)) return GEM_VOX_WIDE;
        minb[a] = floor((double)lo);
        div[a] = (unsigned long long)(floor((double)hi) - minb[a]) + 1;
    }
    *div0 = div[0];
    *div01 = div[0] * div[1];
    *cut_key = *div01 * div[2];
    return GEM_VOX_GRID;
}
