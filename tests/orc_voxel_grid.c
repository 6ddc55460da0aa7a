/* orc_voxel_grid.c -- oracle of gem_voxel_grid (DESIGN.md f9).  TEST INFRASTRUCTURE ONLY.
 *
 * A literal, single-threaded restatement of pcl::VoxelGrid<pcl::PCLPointCloud2>::applyFilter of PCL 1.8 with
 * downsample_all_data_ true (pcl_ros's VoxelGrid nodelet, GEM's filter.launch / filter_kitti.launch) on n float4
 * {x, y, z, intensity}: getMinMax3D, the overflow check, the index pass, the sort, the centroid loop.  PCL is unpinned and
 * not available; compiled with -ffp-contract=off.  The rules, where the reference is undefined the library's DEFINITIONS:
 *   V1 inv[a] = 1.0f / leaf[a] in float; a leaf that is not finite or is <= 0 is an error.
 *   V2 with a field: cut when (double)v > limit_max || (double)v < limit_min (negative 0), when (double)v < limit_max &&
 *      (double)v > limit_min (negative 1); NaN passes.  Then cut when x, y or z is not finite (is_dense is not read).
 *   V3 getMinMax3D: the same tests against the limits rounded to float, compared in float; float min / max per axis from
 *      FLT_MAX / -FLT_MAX (Eigen's cwiseMin / cwiseMax).
 *   V4 d[a] = (int64)((max_p[a] - min_p[a]) * inv[a]) + 1 with the product in float; d0 d1 d2 > INT32_MAX: the output is
 *      the input.  DEFINED: a product that is not finite or a quotient >= 2^62 is an overflow; the product of the d is
 *      the mathematical one.
 *   V5 no V3 survivor: count 0.  DEFINED (PCL casts -inf).
 *   V6 min_b = floor(min_p * inv) (the double floor of the float product: exact, as the float floor would be),
 *      ijk = floor(p * inv) - min_b (exact in double), idx = ijk0 + ijk1 div0 + ijk2 div0 div1 in 64 bits.  DEFINED: when
 *      div0 div1 div2 > 2^31 (PCL's int idx overflows) the order is lexicographic in (ijk2, ijk1, ijk0), which this idx is.
 *   V7 DEFINED: qsort on (idx, input index), a total order: ascending input index inside a voxel.
 *   V8 c = +0.0f per component, c += p in float in V7 order, c /= (float)count.  DEFINED: a NaN result has the bits
 *      x86-64 SSE gives it (the first NaN operand quieted; inf - inf the default NaN 0xFFC00000; NaN / count = that NaN).
 *   V9 min(count, capacity) float4 written, count always reported. */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { float leaf_size[3]; int field; double limit_min, limit_max; int limit_negative; } orc_voxel_params;
typedef struct { int count, used, passthrough; } orc_voxel_info;

typedef struct { unsigned long long idx; int cp; } entry; /* cloud_point_index_idx */

static int entry_cmp(const void *a, const void *b)
{
    const entry *x = (const entry *)a, *y = (const entry *)b;
    if (x->idx != y->idx) return x->idx < y->idx ? -1 : 1;
    return (x->cp > y->cp) - (x->cp < y->cp);
}

/* V8's c += p with the NaN bits of x86-64 SSE written out, so that they do not depend on the operand order the compiler
 * picks (DEFINED): the first NaN operand (c, then p) quieted; an invalid inf - inf gives the default NaN 0xFFC00000 */
static float quiet(float f)
{
    uint32_t u;
    memcpy(&u, &f, 4);
    u |= 0x00400000u;
    memcpy(&f, &u, 4);
    return f;
}
static float add_x86(float c, float p)
{
    const float s = c + p;
    if (s == s) return s;
    if (c != c) return quiet(c);
    if (p != p) return quiet(p);
    const uint32_t dn = 0xffc00000u;
    float r;
    memcpy(&r, &dn, 4);
    return r;
}

static int finite3(const float *pt) { return isfinite(pt[0]) && isfinite(pt[1]) && isfinite(pt[2]); }

/* V2 */
static int used(const orc_voxel_params *p, const float *pt)
{
    if (p->field >= 0) {
        const float v = pt[p->field];
        if (p->limit_negative) {
            if ((double)v < p->limit_max && (double)v > p->limit_min) return 0;
        } else {
            if ((double)v > p->limit_max || (double)v < p->limit_min) return 0;
        }
    }
    return finite3(pt);
}

/* V3 */
static int bounded(const orc_voxel_params *p, float lo, float hi, const float *pt)
{
    if (p->field >= 0) {
        const float v = pt[p->field];
        if (p->limit_negative) {
            if (v < hi && v > lo) return 0;
        } else {
            if (v > hi || v < lo) return 0;
        }
    }
    return finite3(pt);
}

/* 0, or -1 for an error (nothing written) */
int orc_voxel_grid(const float *in, int n, const orc_voxel_params *p, float *out, int capacity, orc_voxel_info *info)
{
    if (n < 0 || capacity < 0 || p->field < -1 || p->field > 3) return -1;
    for (int a = 0; a < 3; a++)
        if (!isfinite(p->leaf_size[a]) || !(p->leaf_size[a] > 0.0f)) return -1;
    info->count = info->used = info->passthrough = 0;
    if (n == 0) return 0;
    float inv[3];
    for (int a = 0; a < 3; a++) inv[a] = 1.0f / p->leaf_size[a];
    const float flo = (float)p->limit_min, fhi = (float)p->limit_max;
    float min_p[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, max_p[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    int nb = 0;
    for (int cp = 0; cp < n; cp++) {
        const float *pt = in + 4 * (size_t)cp;
        if (!bounded(p, flo, fhi, pt)) continue;
        nb++;
        for (int a = 0; a < 3; a++) {
            min_p[a] = (pt[a] < min_p[a]) ? pt[a] : min_p[a];
            max_p[a] = (max_p[a] < pt[a]) ? pt[a] : max_p[a];
        }
    }
    for (int cp = 0; cp < n; cp++) info->used += used(p, in + 4 * (size_t)cp);
    if (nb == 0) return 0; /* V5 */
    int over = 0;
    long long d[3] = {0, 0, 0};
    for (int a = 0; a < 3; a++) {
        const float q = (max_p[a] - min_p[a]) * inv[a];
        if (!isfinite(q) || q >= 0x1p62f) over = 1;
        else d[a] = (long long)q + 1;
    }
    if (!over) over = (__int128)d[0] * d[1] * d[2] > (__int128)INT32_MAX;
    if (over) {
        memcpy(out, in, (size_t)(n < capacity ? n : capacity) * 16);
        info->count = n;
        info->passthrough = 1;
        return 0;
    }
    double min_b[3];
    long long div[3];
    for (int a = 0; a < 3; a++) {
        min_b[a] = floor(min_p[a] * inv[a]);
        div[a] = (long long)(floor(max_p[a] * inv[a]) - min_b[a]) + 1;
    }
    entry *e = (entry *)malloc((size_t)n * sizeof *e);
    if (!e) return -1;
    int m = 0;
    for (int cp = 0; cp < n; cp++) {
        const float *pt = in + 4 * (size_t)cp;
        if (!used(p, pt)) continue;
        long long ijk[3];
        for (int a = 0; a < 3; a++) ijk[a] = (long long)(floor(pt[a] * inv[a]) - min_b[a]);
        e[m].idx = (unsigned long long)ijk[0] + (unsigned long long)ijk[1] * (unsigned long long)div[0] +
                   (unsigned long long)ijk[2] * (unsigned long long)div[0] * (unsigned long long)div[1];
        e[m].cp = cp;
        m++;
    }
    qsort(e, (size_t)m, sizeof *e, entry_cmp);
    int k = 0;
    for (int i = 0; i < m;) {
        int j = i;
        float c[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        while (j < m && e[j].idx == e[i].idx) {
            const float *pt = in + 4 * (size_t)e[j].cp;
            for (int q = 0; q < 4; q++) c[q] = add_x86(c[q], pt[q]);
            j++;
        }
        for (int q = 0; q < 4; q++) c[q] = (c[q] != c[q]) ? c[q] : c[q] / (float)(j - i); /* a NaN c stays that NaN */
        if (k < capacity) memcpy(out + 4 * (size_t)k, c, sizeof c);
        k++;
        i = j;
    }
    free(e);
    info->count = k;
    return 0;
}
