/* orc_global_map.c -- oracle of the gem_global_map_* calls (DESIGN.md f16).  TEST INFRASTRUCTURE ONLY.
 *
 * A literal restatement of the node's globalMap_ / trajectory_ / localMapLoc_ and of ElevationMapping::updateGlobalMap
 * (ElevationMapping.cpp:633-662, :688-707, :773-905) on top of the oracle's orc_transform_cloud and orc_refuse_submaps
 * (oracle/gem_oracle.c).  Each submap is a separate malloc'ed array, as globalMap_ holds separate clouds; the packed
 * stack of the device is their concatenation.  Compiled with -ffp-contract=off: the pose arithmetic is float, left to
 * right, without contraction. */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "gem_oracle.h"

typedef struct {
    int submaps, keyframes;
    float **rec;    /* rec[k]: 8 floats per record */
    int *n;         /* n[k] */
    float *poses;   /* 16 per keyframe, row-major */
    float *centres; /* 2 per keyframe */
} orc_gmap;

void orc_gmap_reset(orc_gmap *g)
{
    for (int k = 0; k < g->submaps; k++) free(g->rec[k]);
    free(g->rec);
    free(g->n);
    free(g->poses);
    free(g->centres);
    memset(g, 0, sizeof *g);
    /* :688-694: trajectory_ = {Identity}, localMapLoc_ = {(0, 0)} */
    g->keyframes = 1;
    g->poses = calloc(16, sizeof(float));
    g->poses[0] = g->poses[5] = g->poses[10] = g->poses[15] = 1.0f;
    g->centres = calloc(2, sizeof(float));
}

orc_gmap *orc_gmap_create(void)
{
    orc_gmap *g = calloc(1, sizeof *g);
    orc_gmap_reset(g);
    return g;
}

void orc_gmap_destroy(orc_gmap *g)
{
    orc_gmap_reset(g);
    free(g->poses);
    free(g->centres);
    free(g);
}

/* :636-642 then :660 */
void orc_gmap_push(orc_gmap *g, const float *rec, int n, const float pose[16])
{
    g->poses = realloc(g->poses, (size_t)(g->keyframes + 1) * 16 * sizeof(float));
    memcpy(g->poses + 16 * g->keyframes, pose, 16 * sizeof(float));
    g->centres = realloc(g->centres, (size_t)(g->keyframes + 1) * 2 * sizeof(float));
    g->centres[2 * g->keyframes] = pose[3];
    g->centres[2 * g->keyframes + 1] = pose[7];
    g->keyframes++;
    g->rec = realloc(g->rec, (size_t)(g->submaps + 1) * sizeof(float *));
    g->n = realloc(g->n, (size_t)(g->submaps + 1) * sizeof(int));
    g->rec[g->submaps] = malloc((size_t)(n > 0 ? n : 1) * 32);
    if (n > 0) memcpy(g->rec[g->submaps], rec, (size_t)n * 32);
    g->n[g->submaps] = n;
    g->submaps++;
}

/* optGlobalMapLoc_[i] * trajectory_[i].inverse() as Isometry3f: inverse = (R^T, -(R^T t)), product = (Rn Ri, Rn ti + tn) */
void orc_gmap_relative_pose(const float *pn, const float *po, float *T)
{
    float ri[3][3], ti[3];
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) ri[r][c] = po[4 * c + r];
    for (int r = 0; r < 3; r++) ti[r] = -((ri[r][0] * po[3] + ri[r][1] * po[7]) + ri[r][2] * po[11]);
    for (int r = 0; r < 3; r++) {
        for (int c = 0; c < 3; c++) T[4 * r + c] = (pn[4 * r] * ri[0][c] + pn[4 * r + 1] * ri[1][c]) + pn[4 * r + 2] * ri[2][c];
        T[4 * r + 3] = ((pn[4 * r] * ti[0] + pn[4 * r + 1] * ti[1]) + pn[4 * r + 2] * ti[2]) + pn[4 * r + 3];
    }
    T[12] = T[13] = T[14] = 0.0f;
    T[15] = 1.0f;
}

/* radiusSearch of centre i among the first K: d2 <= r^2 in float, sorted by (d2, index); returns the count */
static int radius_search(const float *c, int K, int i, float radius, int *idx, float *d2)
{
    int m = 0;
    for (int j = 0; j < K; j++) {
        const float dx = c[2 * j] - c[2 * i], dy = c[2 * j + 1] - c[2 * i + 1];
        const float d = dx * dx + dy * dy;
        if (d <= radius * radius) { idx[m] = j; d2[m] = d; m++; }
    }
    for (int a = 1; a < m; a++) /* insertion sort: stable, so equal distances stay in index order */
        for (int b = a; b > 0 && d2[b - 1] > d2[b]; b--) {
            const float t = d2[b]; d2[b] = d2[b - 1]; d2[b - 1] = t;
            const int u = idx[b]; idx[b] = idx[b - 1]; idx[b - 1] = u;
        }
    return m;
}

/* updateGlobalMap (:773-905) with optKeyframeNum = k; returns the fused count over all pairs */
int orc_gmap_update(orc_gmap *g, const float *opt_poses, int k, double res, double radius, int compat)
{
    const int K = k < g->submaps ? k : g->submaps; /* :784-786 */
    for (int i = 1; i < K; i++) {                  /* :791-809 */
        float T[16];
        orc_gmap_relative_pose(opt_poses + 16 * i, g->poses + 16 * i, T);
        orc_transform_cloud(g->rec[i], g->n[i], T);
        memcpy(g->poses + 16 * i, opt_poses + 16 * i, 16 * sizeof(float));
    }
    int total = 0;
    int *idx = malloc((size_t)(K > 0 ? K : 1) * sizeof(int));
    float *d2 = malloc((size_t)(K > 0 ? K : 1) * sizeof(float));
    for (int i = 0; i < K; i++) { /* :812-891 */
        const int m = radius_search(g->centres, K, i, (float)radius, idx, d2);
        if (m > 2) {
            for (int q = 1; q < m; q++) {
                const int j = idx[q];
                if (j == i) continue;
                total += orc_refuse_submaps(g->rec[j], &g->n[j], g->rec[i], &g->n[i], res, compat);
            }
        }
    }
    free(idx);
    free(d2);
    return total;
}

int orc_gmap_submaps(const orc_gmap *g) { return g->submaps; }
int orc_gmap_keyframes(const orc_gmap *g) { return g->keyframes; }
int orc_gmap_count(const orc_gmap *g, int k) { return g->n[k]; }
void orc_gmap_read(const orc_gmap *g, int k, float *out) { if (g->n[k] > 0) memcpy(out, g->rec[k], (size_t)g->n[k] * 32); }
void orc_gmap_pose(const orc_gmap *g, int i, float pose[16], float centre[2])
{
    memcpy(pose, g->poses + 16 * i, 16 * sizeof(float));
    centre[0] = g->centres[2 * i];
    centre[1] = g->centres[2 * i + 1];
}
