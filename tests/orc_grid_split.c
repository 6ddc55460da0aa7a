/* orc_grid_split.c -- CPU oracle of gem_grid_cloud_split: the numeric block of ElevationMapping::composingGlobalMap
 * (ElevationMapping.cpp:1146-1174): pcl::StatisticalOutlierRemoval (setMeanK, setStddevMulThresh) over the grid cloud,
 * then the survivors split by travers > travers_threshold into the road and the obstacle cloud.  TEST INFRASTRUCTURE
 * ONLY: compiled by tests/split_oracle.py with the oracle's flags (-ffp-contract=off), next to the pinned oracle library,
 * which it leaves untouched.
 *
 * PARITY UNPINNED (PCL): restated from PCL 1.8 StatisticalOutlierRemoval<PointT>::applyFilterIndices and KdTreeFLANN
 * (flann::L2_Simple<float>, exact search).  DEFINED (DESIGN.md f6): sqrt is the double sqrt of the float d2; a non-finite
 * point is nobody's neighbour; with at most mean_k finite points every point is kept and the distances and statistics
 * are NaN with valid = 0; the sums are the sequential loop in point order.
 *
 * The neighbour search does not use the map grid.  It sweeps the finite points sorted by x: a point j at sorted
 * distance beyond another point j' on the same side has |fl(x_i - x_j)| >= |fl(x_i - x_j')| (sorted floats, monotone
 * rounding), and its d2 = fl(fl(fl(0 + dx^2) + dy^2) + dz^2) >= fl(dx^2) (non-negative addends).  So once
 * fl(dx^2) exceeds the largest of the mean_k + 1 values held, no point further out on that side can enter. */
#include <math.h>
#include <stdlib.h>
#include <string.h>

static const float *g_x;
static int cmp_x(const void *a, const void *b)
{
    const int i = *(const int *)a, j = *(const int *)b;
    if (g_x[i] < g_x[j]) return -1;
    if (g_x[i] > g_x[j]) return 1;
    return (i > j) - (i < j);
}

static float flann_d2(const float *a, const float *b)
{
    float r = 0.0f, d;
    d = a[0] - b[0]; r += d * d;
    d = a[1] - b[1]; r += d * d;
    d = a[2] - b[2]; r += d * d;
    return r;
}

/* keep the K smallest values of a sorted list of *n entries */
static void push(float *lst, int *n, int K, float v)
{
    int p;
    if (*n == K && !(v < lst[K - 1])) return;
    p = *n < K ? (*n)++ : K - 1;
    while (p > 0 && lst[p - 1] > v) { lst[p] = lst[p - 1]; p--; }
    lst[p] = v;
}

/* recs: n PointXYZRGBICT records (8 floats).  dist[n] out; road_idx / obst_idx receive the indices of the kept points of
 * each output in input order; counts = {valid, road, obstacle}; stats = {mean, stddev, threshold} */
void orc_grid_split(int n, const float *recs, int mean_k, double stddev_mul, double travers_threshold, float *dist,
                    int *road_idx, int *obst_idx, int *counts, double *stats)
{
    const int K = mean_k + 1;
    float *xs = malloc((size_t)(n > 0 ? n : 1) * sizeof(float));
    float *pts = malloc((size_t)(n > 0 ? n : 1) * 3 * sizeof(float));
    int *order = malloc((size_t)(n > 0 ? n : 1) * sizeof(int));
    float lst[65];
    int nf = 0, i, s, valid = 0, nr = 0, no = 0;
    double sum = 0, sq_sum = 0, mean, variance, stddev, thr;
    for (i = 0; i < n; i++) {
        const float *r = recs + 8 * (size_t)i;
        memcpy(pts + 3 * (size_t)i, r, 3 * sizeof(float));
        xs[i] = r[0];
        if (isfinite(r[0]) && isfinite(r[1]) && isfinite(r[2])) order[nf++] = i;
    }
    g_x = xs;
    qsort(order, (size_t)nf, sizeof(int), cmp_x);
    for (i = 0; i < n; i++) dist[i] = 0.0f;
    for (s = 0; s < nf; s++) {
        const int q = order[s];
        const float *a = pts + 3 * (size_t)q;
        int cnt = 0, t, k, dir;
        double dist_sum = 0;
        push(lst, &cnt, K, 0.0f); /* the point itself */
        for (dir = -1; dir <= 1; dir += 2) {
            for (t = s + dir; t >= 0 && t < nf; t += dir) {
                const float *b = pts + 3 * (size_t)order[t];
                const float dx = a[0] - b[0], lb = dx * dx;
                if (cnt == K && lb > lst[K - 1]) break;
                push(lst, &cnt, K, flann_d2(a, b));
            }
        }
        if (cnt < K) continue;
        for (k = 1; k < K; k++) dist_sum += sqrt((double)lst[k]);
        dist[q] = (float)(dist_sum / mean_k);
        valid++;
    }
    if (nf <= mean_k) { /* DEFINED item 3 */
        for (i = 0; i < n; i++) dist[i] = (float)NAN;
        valid = 0;
        mean = stddev = thr = NAN;
    } else {
        for (i = 0; i < n; i++) {
            sum += dist[i];
            sq_sum += dist[i] * dist[i];
        }
        mean = sum / (double)valid;
        variance = (sq_sum - sum * sum / (double)valid) / ((double)valid - 1);
        stddev = sqrt(variance);
        thr = mean + stddev_mul * stddev;
    }
    for (i = 0; i < n; i++) {
        if (dist[i] > thr) continue;
        if ((double)recs[8 * (size_t)i + 7] > travers_threshold) road_idx[nr++] = i;
        else obst_idx[no++] = i;
    }
    counts[0] = valid; counts[1] = nr; counts[2] = no;
    stats[0] = mean; stats[1] = stddev; stats[2] = thr;
    free(xs); free(pts); free(order);
}
