/* orc_mls.c -- oracle of gem_mls_upsample (DESIGN.md f10).  TEST INFRASTRUCTURE ONLY.
 *
 * A literal, single-threaded restatement of what pcl::MovingLeastSquares<PointXYZRGB, PointXYZRGB>::process computes in
 * GEM's pointcloudinterpolation (ElevationMapping.cpp:1072-1118) -- PCL 1.7.2's performProcessing /
 * computeMLSPointNormal with a KdTreeFLANN radius search -- over n 32-byte PointXYZRGBICT records.  PCL is unpinned and
 * not available; compiled with -ffp-contract=off.  exp, atan2, sin and cos come from gem_b200/csrc/gem_mathd.h, the
 * source the kernels include.  Items (DEFINED: the library fixes what the reference leaves open):
 *   M1 only x, y, z and the bgra word are read.  DEFINED: a record with a non-finite x, y or z is nobody's neighbour and
 *      produces nothing; it counts in skipped.
 *   M2 brute force: d2 = ((dx dx) + dy dy) + dz dz in float (dx = x_j - x_i), neighbour iff d2 <= (float)(r r) (DEFINED
 *      inclusive), the query included, sorted by (d2, index) (DEFINED ties), no cap; fewer than 3: nothing.
 *   M3 in double, in neighbour order: centroid = sequential sums / n; the non-normalised covariance in PCL's update
 *      order; eigen33's smallest eigenvector (scale, computeRoots / computeRoots2, three row cross products, the largest
 *      squared norm in PCL's if-chain order); d = -(n . centroid) with the Vector4d dot (a0b0 + a2b2) + (a1b1 + a3b3);
 *      point = q - (q . n + d) n.  3-vector dots left to right (DEFINED).
 *   M4 with polynomial_fit and n >= nr_coeff: de = p_j - point, d2f = (float)(de . de), w = exp_d(-d2f / sqr_gauss),
 *      v_axis = n.unitOrthogonal(), u_axis = n x v_axis, u = de . u_axis, v = de . v_axis, f = de . n, monomials in PCL's
 *      order; A(a,b) = sum ((P(a) w) P(b)) for a >= b, rhs(a) = sum ((P(a) w) f), sequential in neighbour order
 *      (DEFINED); left-looking Cholesky, forward and back substitution in the orders below (DEFINED); a pivot that is
 *      not finite or not > 0 fails the fit (DEFINED), as does a non-finite c0.  The axes are set only here (1.7.2).
 *   M5 NONE: point + c0 n when fitted, else point.
 *   M6 RANDOM_UNIFORM_DENSITY: k = (int)floor(density / 2.0 / n); k <= 0: M5's output; else k samples, u then v drawn
 *      as floats in [-r/2, r/2), redrawn while u u + v v > r r / 4 (double); sample = point + u u_axis + v v_axis
 *      (+ height(u, v) n when fitted).  DEFINED generator: draw j of point i is splitmix64(seed ^ (i << 32) ^ j), the float
 *      lo + (float)(x >> 40) 2^-24 (hi - lo) in float, lo = -(float)(r / 2), hi = (float)(r / 2).
 *   M7 records {(float)x, (float)y, (float)z, 1, b g r 0xff, covariance, intensity, travers of the query} (DEFINED: the
 *      last three and the alpha); input order, sample order within a point.
 *   M8 info: count, processed (n >= 3), fitted, skipped (n < 3 or non-finite), max_neighbours. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "gem_mathd.h"

typedef struct {
    double search_radius, sqr_gauss_param;
    int polynomial_fit, order, upsampling, point_density;
    unsigned long long seed;
} orc_mls_params;
typedef struct {
    long long count;
    int processed, fitted, skipped, max_neighbours;
} orc_mls_info;

double orc_mls_exp_d(double x) { return gem_exp_d(x); }
double orc_mls_atan2_d(double y, double x) { return gem_atan2_d(y, x); }
void orc_mls_sincos_d(double x, double *s, double *c) { gem_sincos_d(x, s, c); }

static int finite3(const float *p) { return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]); }

typedef struct { float d2; int idx; } nb_t;
static int nb_cmp(const void *a, const void *b)
{
    const nb_t *x = (const nb_t *)a, *y = (const nb_t *)b;
    if (x->d2 != y->d2) return x->d2 < y->d2 ? -1 : 1;
    return (x->idx > y->idx) - (x->idx < y->idx);
}

static double dot3(const double *a, const double *b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
static void cross3(const double *a, const double *b, double *c)
{
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

static void roots2(double b, double c, double *r)
{
    r[0] = 0.0;
    double d = b * b - 4.0 * c;
    if (d < 0.0) d = 0.0;
    const double sd = sqrt(d);
    r[2] = 0.5 * (b + sd);
    r[1] = 0.5 * (b - sd);
}

/* computeRoots: the roots of the characteristic polynomial in ascending order */
static void roots3(const double m[3][3], double *r)
{
    const double c0 = m[0][0] * m[1][1] * m[2][2] + 2.0 * m[0][1] * m[0][2] * m[1][2] - m[0][0] * m[1][2] * m[1][2] -
                      m[1][1] * m[0][2] * m[0][2] - m[2][2] * m[0][1] * m[0][1];
    const double c1 = m[0][0] * m[1][1] - m[0][1] * m[0][1] + m[0][0] * m[2][2] - m[0][2] * m[0][2] + m[1][1] * m[2][2] -
                      m[1][2] * m[1][2];
    const double c2 = m[0][0] + m[1][1] + m[2][2];
    if (fabs(c0) < 2.220446049250313e-16) {
        roots2(c2, c1, r);
        return;
    }
    const double s_inv3 = 1.0 / 3.0, s_sqrt3 = sqrt(3.0);
    const double c2_over_3 = c2 * s_inv3;
    double a_over_3 = (c1 - c2 * c2_over_3) * s_inv3;
    if (a_over_3 > 0.0) a_over_3 = 0.0;
    const double half_b = 0.5 * (c0 + c2_over_3 * (2.0 * c2_over_3 * c2_over_3 - c1));
    double q = half_b * half_b + a_over_3 * a_over_3 * a_over_3;
    if (q > 0.0) q = 0.0;
    const double rho = sqrt(-a_over_3);
    const double theta = gem_atan2_d(sqrt(-q), half_b) * s_inv3;
    double sin_theta, cos_theta;
    gem_sincos_d(theta, &sin_theta, &cos_theta);
    r[0] = c2_over_3 + 2.0 * rho * cos_theta;
    r[1] = c2_over_3 - rho * (cos_theta + s_sqrt3 * sin_theta);
    r[2] = c2_over_3 - rho * (cos_theta - s_sqrt3 * sin_theta);
    double t;
    if (r[0] >= r[1]) { t = r[0]; r[0] = r[1]; r[1] = t; }
    if (r[1] >= r[2]) {
        t = r[1]; r[1] = r[2]; r[2] = t;
        if (r[0] >= r[1]) { t = r[0]; r[0] = r[1]; r[1] = t; }
    }
    if (r[0] <= 0.0) roots2(c2, c1, r);
}

/* eigen33: the eigenvector of the smallest eigenvalue */
static void eigen33(const double cov[3][3], double *ev)
{
    double scale = 0.0;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++)
            if (fabs(cov[i][j]) > scale) scale = fabs(cov[i][j]);
    if (scale <= 2.2250738585072014e-308) scale = 1.0;
    double s[3][3];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) s[i][j] = cov[i][j] / scale;
    double r[3];
    roots3((const double(*)[3])s, r);
    for (int i = 0; i < 3; i++) s[i][i] -= r[0];
    double v1[3], v2[3], v3[3];
    cross3(s[0], s[1], v1);
    cross3(s[0], s[2], v2);
    cross3(s[1], s[2], v3);
    const double l1 = dot3(v1, v1), l2 = dot3(v2, v2), l3 = dot3(v3, v3);
    const double *v;
    double l;
    if (l1 >= l2 && l1 >= l3) { v = v1; l = l1; }
    else if (l2 >= l1 && l2 >= l3) { v = v2; l = l2; }
    else { v = v3; l = l3; }
    const double sl = sqrt(l);
    for (int a = 0; a < 3; a++) ev[a] = v[a] / sl;
}

/* Eigen's unitOrthogonal for a 3-vector */
static void unit_orthogonal(const double *n, double *v)
{
    const double prec = 1e-12;
    if (!(fabs(n[0]) <= fabs(n[2]) * prec) || !(fabs(n[1]) <= fabs(n[2]) * prec)) {
        const double inv = 1.0 / sqrt(n[0] * n[0] + n[1] * n[1]);
        v[0] = -n[1] * inv;
        v[1] = n[0] * inv;
        v[2] = 0.0;
    } else {
        const double inv = 1.0 / sqrt(n[1] * n[1] + n[2] * n[2]);
        v[0] = 0.0;
        v[1] = -n[2] * inv;
        v[2] = n[1] * inv;
    }
}

static uint64_t splitmix64(uint64_t x)
{
    uint64_t z = x + 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
static float draw(uint64_t seed, int i, uint64_t j, float lo, float hi)
{
    const uint64_t x = splitmix64(seed ^ ((uint64_t)(uint32_t)i << 32) ^ j);
    return lo + ((float)(x >> 40) * 0x1p-24f) * (hi - lo);
}

static void emit(float *out, long long capacity, long long slot, const double *pos, const float *q)
{
    if (slot >= capacity) return;
    float *o = out + 8 * (size_t)slot;
    uint32_t w;
    memcpy(&w, q + 4, 4);
    w |= 0xff000000u;
    o[0] = (float)pos[0];
    o[1] = (float)pos[1];
    o[2] = (float)pos[2];
    o[3] = 1.0f;
    memcpy(o + 4, &w, 4);
    o[5] = q[5];
    o[6] = q[6];
    o[7] = q[7];
}

/* what M2-M4 give one point; the test suite reads it through orc_mls_detail */
typedef struct {
    int nb, fitted, attempted;
    double normal[3], point[3], u_axis[3], v_axis[3], c[21];
} orc_mls_detail_t;

static int bad_params(const orc_mls_params *p)
{
    return !isfinite(p->search_radius) || !(p->search_radius > 0.0) || !isfinite(p->sqr_gauss_param) || !(p->sqr_gauss_param > 0.0) ||
           p->order < 1 || p->order > 5 || p->upsampling < 0 || p->upsampling > 1 || p->point_density < 0;
}

/* M2-M4 for point i (finite): nb (the sorted list) filled, d filled; d->nb < 3 leaves the rest unset */
static void mls_point(const float *in, int n, const orc_mls_params *p, int i, nb_t *nb, orc_mls_detail_t *D)
{
    const double r = p->search_radius;
    const float r2f = (float)(r * r);
    const int order = p->order, nc = (order + 1) * (order + 2) / 2;
    const float *q = in + 8 * (size_t)i;
    memset(D, 0, sizeof *D);
    int m = 0;
    for (int j = 0; j < n; j++) {
        const float *pj = in + 8 * (size_t)j;
        if (!finite3(pj)) continue;
        const float dx = pj[0] - q[0], dy = pj[1] - q[1], dz = pj[2] - q[2];
        const float d2 = (dx * dx + dy * dy) + dz * dz;
        if (d2 <= r2f) { nb[m].d2 = d2; nb[m].idx = j; m++; }
    }
    qsort(nb, (size_t)m, sizeof *nb, nb_cmp);
    D->nb = m;
    if (m < 3) return;
    /* M3 */
    double c[3] = {0.0, 0.0, 0.0};
    for (int k = 0; k < m; k++) {
        const float *pk = in + 8 * (size_t)nb[k].idx;
        c[0] += pk[0]; c[1] += pk[1]; c[2] += pk[2];
    }
    for (int a = 0; a < 3; a++) c[a] /= (double)m;
    double cov[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
    for (int k = 0; k < m; k++) {
        const float *pk = in + 8 * (size_t)nb[k].idx;
        const double x = pk[0] - c[0], y = pk[1] - c[1], z = pk[2] - c[2];
        cov[1][1] += y * y;
        cov[1][2] += y * z;
        cov[2][2] += z * z;
        cov[0][0] += x * x;
        cov[0][1] += y * x;
        cov[0][2] += z * x;
    }
    cov[1][0] = cov[0][1]; cov[2][0] = cov[0][2]; cov[2][1] = cov[1][2];
    double *nrm = D->normal, *pt = D->point, *uax = D->u_axis, *vax = D->v_axis, *cv = D->c;
    eigen33((const double(*)[3])cov, nrm);
    const double d = -((nrm[0] * c[0] + nrm[2] * c[2]) + (nrm[1] * c[1] + 0.0 * 1.0));
    const double qd[3] = {q[0], q[1], q[2]};
    const double dist = dot3(qd, nrm) + d;
    for (int a = 0; a < 3; a++) pt[a] = qd[a] - dist * nrm[a];
    /* M4 */
    if (!(p->polynomial_fit && m >= nc)) return;
    D->attempted = 1;
    unit_orthogonal(nrm, vax);
    cross3(nrm, vax, uax);
    double A[21][21], rhs[21], P[21];
    for (int a = 0; a < nc; a++) {
        rhs[a] = 0.0;
        for (int b = 0; b <= a; b++) A[a][b] = 0.0;
    }
    for (int k = 0; k < m; k++) {
        const float *pk = in + 8 * (size_t)nb[k].idx;
        const double de[3] = {pk[0] - pt[0], pk[1] - pt[1], pk[2] - pt[2]};
        const float d2f = (float)dot3(de, de);
        const double w = gem_exp_d(-d2f / p->sqr_gauss_param);
        const double u = dot3(de, uax), v = dot3(de, vax), f = dot3(de, nrm);
        int j = 0;
        double upow = 1.0;
        for (int ui = 0; ui <= order; ui++) {
            double vpow = 1.0;
            for (int vi = 0; vi <= order - ui; vi++) {
                P[j++] = upow * vpow;
                vpow *= v;
            }
            upow *= u;
        }
        for (int a = 0; a < nc; a++) {
            const double pw = P[a] * w;
            for (int b = 0; b <= a; b++) A[a][b] += pw * P[b];
            rhs[a] += pw * f;
        }
    }
    double L[21][21], y[21];
    for (int jc = 0; jc < nc; jc++) {
        for (int i2 = jc; i2 < nc; i2++) {
            double s = A[i2][jc];
            for (int k = 0; k < jc; k++) s -= L[i2][k] * L[jc][k];
            if (i2 == jc) {
                if (!(s > 0.0) || !isfinite(s)) return; /* the fit fails */
                L[jc][jc] = sqrt(s);
            } else {
                L[i2][jc] = s / L[jc][jc];
            }
        }
    }
    for (int i2 = 0; i2 < nc; i2++) {
        double s = rhs[i2];
        for (int k = 0; k < i2; k++) s -= L[i2][k] * y[k];
        y[i2] = s / L[i2][i2];
    }
    for (int i2 = nc - 1; i2 >= 0; i2--) {
        double s = y[i2];
        for (int k = i2 + 1; k < nc; k++) s -= L[k][i2] * cv[k];
        cv[i2] = s / L[i2][i2];
    }
    D->fitted = isfinite(cv[0]);
}

/* M2-M4 of point i; *nb_out receives the sorted neighbour indices (room for n).  0, or -1 for an error */
int orc_mls_detail(const float *in, int n, const orc_mls_params *p, int i, orc_mls_detail_t *D, int *nb_out)
{
    if (n < 0 || i < 0 || i >= n || bad_params(p)) return -1;
    memset(D, 0, sizeof *D);
    if (!finite3(in + 8 * (size_t)i)) return 0;
    nb_t *nb = (nb_t *)malloc((size_t)n * sizeof *nb);
    if (!nb) return -1;
    mls_point(in, n, p, i, nb, D);
    for (int k = 0; k < D->nb; k++) nb_out[k] = nb[k].idx;
    free(nb);
    return 0;
}

/* 0, or -1 for an error (nothing written).  capacity 0 is a size query: fitted = -1 (the fits are not run) */
int orc_mls_upsample(const float *in, int n, const orc_mls_params *p, float *out, long long capacity, orc_mls_info *info)
{
    if (n < 0 || capacity < 0 || bad_params(p)) return -1;
    memset(info, 0, sizeof *info);
    const double r = p->search_radius;
    const int order = p->order;
    const float tmp = (float)(r / 2.0), lo = -tmp, hi = tmp;
    nb_t *nb = (nb_t *)malloc((size_t)(n ? n : 1) * sizeof *nb);
    if (!nb) return -1;
    long long slot = 0;
    orc_mls_detail_t D;
    for (int i = 0; i < n; i++) {
        const float *q = in + 8 * (size_t)i;
        if (!finite3(q)) { info->skipped++; continue; }
        mls_point(in, n, p, i, nb, &D);
        const int m = D.nb;
        if (m > info->max_neighbours) info->max_neighbours = m;
        if (m < 3) { info->skipped++; continue; }
        info->processed++;
        info->fitted += D.fitted;
        const double *nrm = D.normal, *pt = D.point, *uax = D.u_axis, *vax = D.v_axis, *cv = D.c;
        const int fitted = D.fitted;
        /* M5 / M6 */
        const int k = p->upsampling == 1 ? (int)floor(p->point_density / 2.0 / (double)m) : 0;
        if (k <= 0) {
            double o[3];
            for (int a = 0; a < 3; a++) o[a] = fitted ? pt[a] + cv[0] * nrm[a] : pt[a];
            emit(out, capacity, slot++, o, q);
            continue;
        }
        uint64_t j = 0;
        for (int added = 0; added < k;) {
            const float u = draw(p->seed, i, j, lo, hi), v = draw(p->seed, i, j + 1, lo, hi);
            j += 2;
            if ((double)u * (double)u + (double)v * (double)v > r * r / 4.0) continue;
            double h = 0.0;
            if (fitted) {
                int jj = 0;
                double upow = 1.0;
                for (int ui = 0; ui <= order; ui++) {
                    double vpow = 1.0;
                    for (int vi = 0; vi <= order - ui; vi++) {
                        h += upow * vpow * cv[jj++];
                        vpow *= v;
                    }
                    upow *= u;
                }
            }
            double o[3];
            for (int a = 0; a < 3; a++) {
                o[a] = pt[a] + uax[a] * u + vax[a] * v;
                if (fitted) o[a] = o[a] + nrm[a] * h;
            }
            emit(out, capacity, slot++, o, q);
            added++;
        }
    }
    free(nb);
    info->count = slot;
    if (capacity == 0) info->fitted = -1;
    return 0;
}
