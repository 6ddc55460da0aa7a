/* orc_costmap.c -- oracle of the gem_costmap_* calls (DESIGN.md f8).  TEST INFRASTRUCTURE ONLY.
 *
 * A literal, single-threaded restatement of the two plugin loops of GEM's layers/ package (ElevationMapLayer::updateBounds,
 * layers/src/elevationMap_layer.cpp:56-84; PointMapLayer::updateBounds and updateCosts, layers/src/pointMap_layer.cpp:54-100)
 * and of the costmap_2d functions they use (worldToMap, touch, updateOrigin with copyMapRegion / resetMaps, updateWithMax),
 * restated from navigation 1.14.  Compiled with -ffp-contract=off.  Where the reference is undefined the library's
 * DEFINITIONS are applied: a non-finite coordinate or a quotient >= 2^31 is not on the map; a zero bound is +0. */
#include <math.h>
#include <stdlib.h>
#include <string.h>

typedef struct { double origin_x, origin_y, resolution; int size_x, size_y; } orc_window;
typedef struct { long long marked, lethal; double min_x, min_y, max_x, max_y; } orc_marks;

enum { FREE_SPACE = 0, LETHAL_OBSTACLE = 254, NO_INFORMATION = 255 };

static int world_to_map(const orc_window *w, double wx, double wy, unsigned *mx, unsigned *my)
{
    if (wx < w->origin_x || wy < w->origin_y) return 0;
    const double qx = (wx - w->origin_x) / w->resolution, qy = (wy - w->origin_y) / w->resolution;
    if (!isfinite(wx) || !isfinite(wy) || !(qx < 2147483648.0) || !(qy < 2147483648.0)) return 0; /* DEFINED */
    *mx = (unsigned)(int)qx;
    *my = (unsigned)(int)qy;
    return *mx < (unsigned)w->size_x && *my < (unsigned)w->size_y;
}

static double dmin(double a, double b) { return (b < a) ? b : a; } /* std::min(a, b) */
static double dmax(double a, double b) { return (a < b) ? b : a; } /* std::max(a, b) */

static void touch(double x, double y, orc_marks *m)
{
    m->min_x = dmin(x, m->min_x);
    m->min_y = dmin(y, m->min_y);
    m->max_x = dmax(x, m->max_x);
    m->max_y = dmax(y, m->max_y);
}

static void marks_begin(orc_marks *m)
{
    m->marked = m->lethal = 0;
    m->min_x = m->min_y = INFINITY;
    m->max_x = m->max_y = -INFINITY;
}

static void marks_end(orc_marks *m)
{
    m->min_x += 0.0; m->min_y += 0.0; m->max_x += 0.0; m->max_y += 0.0; /* a zero bound is +0 */
}

/* ElevationMapLayer::updateBounds over show()'s grid_map.  traver: L x L, column-major (GridMapIterator linear index
 * ix + iy * L over storage indices), NaN where show() cleared the cell.  Positions: grid_map getPositionFromIndex with the
 * node's double resolution, around the float centre, with the circular buffer's start index. */
void orc_mark_map(int L, double grid_res, const float centre[2], const int start[2], const float *traver, const orc_window *w,
                  double travers_thresh, int mark_unknown, unsigned char *costmap, orc_marks *out)
{
    const double half = 0.5 * ((double)L * grid_res) - 0.5 * grid_res;
    marks_begin(out);
    for (int iy = 0; iy < L; iy++) {
        for (int ix = 0; ix < L; ix++) {
            const float v = traver[(size_t)iy * L + ix];
            if (!mark_unknown && isnan(v)) continue;
            const int is_obstacle = v < travers_thresh;
            const double px = (double)centre[0] + half - grid_res * (double)((ix + L - start[0]) % L);
            const double py = (double)centre[1] + half - grid_res * (double)((iy + L - start[1]) % L);
            unsigned mx, my;
            if (!world_to_map(w, px, py, &mx, &my)) continue;
            costmap[(size_t)my * w->size_x + mx] = is_obstacle ? LETHAL_OBSTACLE : FREE_SPACE;
            out->marked++;
            out->lethal += is_obstacle;
            touch(px, py, out);
        }
    }
    marks_end(out);
}

/* PointMapLayer::updateBounds over n 32-byte PointXYZRGBICT records (8 floats: x, y, z, w, bgra, covariance, intensity,
 * travers) */
void orc_mark_points(const float *rec, int n, const orc_window *w, double travers_thresh, unsigned char *costmap, orc_marks *out)
{
    marks_begin(out);
    for (int i = 0; i < n; i++) {
        const float *p = rec + 8 * (size_t)i;
        const double px = p[0], py = p[1];
        unsigned mx, my;
        if (!world_to_map(w, px, py, &mx, &my)) continue;
        const unsigned index = my * (unsigned)w->size_x + mx;
        if (p[7] > travers_thresh) {
            costmap[index] = FREE_SPACE;
        } else {
            costmap[index] = LETHAL_OBSTACLE;
            out->lethal++;
        }
        out->marked++;
        touch(px, py, out);
    }
    marks_end(out);
}

static void copy_map_region(const unsigned char *src, int sx0, int sy0, int src_size_x, unsigned char *dst, int dx0, int dy0,
                            int dst_size_x, int region_size_x, int region_size_y)
{
    const unsigned char *s = src + (size_t)sy0 * src_size_x + sx0;
    unsigned char *d = dst + (size_t)dy0 * dst_size_x + dx0;
    for (int i = 0; i < region_size_y; i++) {
        memcpy(d, s, (size_t)region_size_x);
        s += src_size_x;
        d += dst_size_x;
    }
}

static int imin(int a, int b) { return a < b ? a : b; }
static int imax(int a, int b) { return a > b ? a : b; }

/* Costmap2D::updateOrigin.  Returns 0, or -1 where the library defines an error (a shift that is not finite or does not fit
 * an int); then nothing changes. */
int orc_update_origin(orc_window *w, double new_origin_x, double new_origin_y, unsigned char fill, unsigned char *costmap)
{
    const double qx = (new_origin_x - w->origin_x) / w->resolution, qy = (new_origin_y - w->origin_y) / w->resolution;
    if (!(fabs(qx) < 2147483648.0) || !(fabs(qy) < 2147483648.0)) return -1;
    const int cell_ox = (int)qx, cell_oy = (int)qy;
    if (cell_ox == 0 && cell_oy == 0) return 0;
    const double new_grid_ox = w->origin_x + cell_ox * w->resolution;
    const double new_grid_oy = w->origin_y + cell_oy * w->resolution;
    const int size_x = w->size_x, size_y = w->size_y;
    /* the int sums of the reference, in long long so that a far shift does not overflow */
    const int lower_left_x = (int)imin(imax(cell_ox, 0), size_x);
    const int lower_left_y = (int)imin(imax(cell_oy, 0), size_y);
    const long long urx = (long long)cell_ox + size_x, ury = (long long)cell_oy + size_y;
    const int upper_right_x = (int)(urx < 0 ? 0 : urx > size_x ? size_x : urx);
    const int upper_right_y = (int)(ury < 0 ? 0 : ury > size_y ? size_y : ury);
    const int cell_size_x = upper_right_x - lower_left_x, cell_size_y = upper_right_y - lower_left_y;
    unsigned char *local_map = malloc((size_t)cell_size_x * cell_size_y + 1);
    copy_map_region(costmap, lower_left_x, lower_left_y, size_x, local_map, 0, 0, cell_size_x, cell_size_x, cell_size_y);
    memset(costmap, fill, (size_t)size_x * size_y); /* resetMaps */
    w->origin_x = new_grid_ox;
    w->origin_y = new_grid_oy;
    const int start_x = lower_left_x - cell_ox, start_y = lower_left_y - cell_oy;
    if (cell_size_x > 0 && cell_size_y > 0)
        copy_map_region(local_map, 0, 0, cell_size_x, costmap, start_x, start_y, size_x, cell_size_x, cell_size_y);
    free(local_map);
    return 0;
}

/* mode 0: CostmapLayer::updateWithMax; mode 1: PointMapLayer::updateCosts.  The rect is clamped to the grid. */
void orc_combine(int mode, const unsigned char *costmap, unsigned char *master, int size_x, int size_y, int min_i, int min_j,
                 int max_i, int max_j)
{
    min_i = imax(min_i, 0); min_j = imax(min_j, 0);
    max_i = imin(max_i, size_x); max_j = imin(max_j, size_y);
    for (int j = min_j; j < max_j; j++) {
        unsigned it = (unsigned)j * (unsigned)size_x + (unsigned)min_i;
        for (int i = min_i; i < max_i; i++) {
            if (costmap[it] == NO_INFORMATION) { it++; continue; }
            if (mode == 1) {
                master[it] = costmap[it];
            } else {
                const unsigned char old_cost = master[it];
                if (old_cost == NO_INFORMATION || old_cost < costmap[it]) master[it] = costmap[it];
            }
            it++;
        }
    }
}
