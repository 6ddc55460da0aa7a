/* orc_sensor_models.c -- CPU oracle of the stereo and perfect sensor models (GEM_SENSOR_STEREO / GEM_SENSOR_PERFECT):
 * the per-point step of G_pointsprocess (gpu.cu:384-455) with the variances of StereoSensorProcessor.cpp:78-90 and
 * PerfectSensorProcessor.cpp:84-101 in place of the laser model, and the `lowest` update.  TEST INFRASTRUCTURE ONLY:
 * compiled by tests/sensor_models_oracle.py next to the pinned oracle library (oracle/gem_oracle.c), which it leaves
 * untouched and whose index function (orc_points_to_index) and fold (orc_fuse) it shares.  Same conventions as the
 * oracle: -ffp-contract=off, literal evaluation order.
 *
 * PARITY UNPINNED (the reference's CPU code needs kindr and PCL): restated from computeVariances.  pow(v, 2) is
 * DEFINED as v * v, rounded once.  row / col = getI / getJ (Stereo.cpp:109-117) with indices_ = the point's position in
 * the cloud as received: no point is removed here, non-finite points fail the height window like every other
 * rejected point, so the remaining points keep their order. */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "gem_oracle.h"

typedef struct {
    int type;          /* 2 = stereo, 3 = perfect */
    double p[5];       /* p_1..p_5 */
    double lateral;    /* lateral_factor */
    double dtd;        /* depth_to_disparity_factor */
    int width;         /* pointCloud->width, 0 = unorganised (one row) */
} orc_sm_sensor;

/* returns varianceLateral, writes varianceNormal */
float orc_sm_variances(const orc_sm_sensor *s, float x, float y, float z, int idx, float *vN)
{
    if (s->type == 2) {
        const int row = s->width ? idx / s->width : 0, col = s->width ? idx % s->width : idx;
        const double disparity = s->dtd / (double)z;                 /* :78 */
        const double a = s->dtd / (disparity * disparity);            /* pow(disparity, 2) */
        const double sj = ((s->p[2] * disparity) + s->p[3]) - (double)col;
        const double si = (double)(240 - row);
        const float dist = sqrtf((x * x + y * y) + z * z);           /* :83 pointVector.norm() */
        const double l = s->lateral * (double)dist;
        *vN = (float)((a * a) * ((((s->p[4] * disparity) + s->p[1]) * sqrt(sj * sj + si * si)) + s->p[0])); /* :86-89 */
        return (float)(l * l);                                        /* :90 */
    }
    *vN = 0.0f; /* Perfect.cpp:87-88 */
    return 0.0f;
}

/* orc_process_points for the two models: the point i has index idx0 + i in the caller's cloud */
void orc_sm_process_points(orc_map *m, int n, const float *x, const float *y, const float *z, const float T[16],
                           double relLower, double relUpper, const orc_sm_sensor *sensor, const float sJ[3],
                           const float rotVar[9], const float C_SB_T[9], const float P[3], const float B_skew[9], int idx0,
                           int *key, float *var, float *x_ts, float *y_ts, float *z_ts)
{
    const size_t C = (size_t)m->L * m->L;
    float *minh = (float *)malloc(C * sizeof(float));
    int *argmin = (int *)malloc(C * sizeof(int));
    float *hvs = (float *)malloc((size_t)(n > 0 ? n : 1) * sizeof(float));
    int *touched = (int *)malloc((size_t)(n > 0 ? n : 1) * sizeof(int));
    int nt = 0, i, j;
    size_t c;
    for (c = 0; c < C; c++) argmin[c] = -1;
    for (i = 0; i < n; i++) {
        const float px = x[i], py = y[i], pz = z[i];
        const float h = ((T[8] * px + T[9] * py) + T[10] * pz) + T[11]; /* gpu.cu:389 */
        float hv = -1, xt = -1, yt = -1, zt = -1;                       /* :443-450 */
        int k = -1, geo = -1, flag = 0;
        if (m->compat_box_filter) /* gpu.cu:393 */
            if ((px > -1.5 && px < 1.5 && py > -1.5 && py < 1.5) || (py > -1 && py < 1) || py > 0) flag = 1;
        if (((double)h > relLower && (double)h < relUpper) && flag == 0) { /* gpu.cu:397 */
            float vN, vL, q[3], S[9], rotJ[3], A1[3], B1[3], SV[9], term1, term2;
            xt = ((T[0] * px + T[1] * py) + T[2] * pz) + T[3];
            yt = ((T[4] * px + T[5] * py) + T[6] * pz) + T[7];
            zt = h;
            vL = orc_sm_variances(sensor, px, py, pz, idx0 + i, &vN);
            for (j = 0; j < 3; j++) q[j] = (C_SB_T[3 * j] * px + C_SB_T[3 * j + 1] * py) + C_SB_T[3 * j + 2] * pz;
            S[0] = 0 + B_skew[0];     S[1] = -q[2] + B_skew[1]; S[2] = q[1] + B_skew[2];
            S[3] = q[2] + B_skew[3];  S[4] = 0 + B_skew[4];     S[5] = -q[0] + B_skew[5];
            S[6] = -q[1] + B_skew[6]; S[7] = q[0] + B_skew[7];  S[8] = 0 + B_skew[8];
            for (j = 0; j < 3; j++) rotJ[j] = (P[0] * S[j] + P[1] * S[3 + j]) + P[2] * S[6 + j];
            for (j = 0; j < 3; j++) A1[j] = (rotJ[0] * rotVar[j] + rotJ[1] * rotVar[3 + j]) + rotJ[2] * rotVar[6 + j];
            term1 = (A1[0] * rotJ[0] + A1[1] * rotJ[1]) + A1[2] * rotJ[2];
            memset(SV, 0, sizeof SV);
            SV[0] = vL; SV[4] = vL; SV[8] = vN;
            for (j = 0; j < 3; j++) B1[j] = (sJ[0] * SV[j] + sJ[1] * SV[3 + j]) + sJ[2] * SV[6 + j];
            term2 = (B1[0] * sJ[0] + B1[1] * sJ[1]) + B1[2] * sJ[2];
            hv = term1;
            hv += term2;
            geo = orc_points_to_index(m, xt, yt, &k); /* :430-431 */
            if (geo != -1) { /* lowest-scan: first index attaining the minimum */
                if (argmin[geo] < 0) { argmin[geo] = i; minh[geo] = h; touched[nt++] = geo; }
                else if (h < minh[geo]) { argmin[geo] = i; minh[geo] = h; }
            }
        }
        if (key) key[i] = k;
        if (var) var[i] = hv;
        if (x_ts) x_ts[i] = xt;
        if (y_ts) y_ts[i] = yt;
        if (z_ts) z_ts[i] = zt;
        hvs[i] = hv;
    }
    /* ORACLE DEFINITION of gpu.cu:432-438 (as orc_process_points): m = min h of the call's points in a geographic cell,
     * i* the first index attaining it: lowest = m + 3 * hv[i*] iff m <= lowest_old.  An inf / NaN hv goes in unchanged. */
    for (i = 0; i < nt; i++) {
        const int g = touched[i];
        if (minh[g] <= m->lowest[g]) m->lowest[g] = minh[g] + 3 * hvs[argmin[g]];
    }
    free(minh); free(argmin); free(hvs); free(touched);
}
