/* orc_footprint.c -- oracle of ObstacleLayer's footprint clearing (DESIGN.md f17 F1-F4): costmap_2d's transformFootprint,
 * Costmap2D::worldToMap, setConvexPolygonCost, convexFillCells, polygonOutlineCells, raytraceLine and bresenham2D, written
 * out as the reference's loops over plain arrays.  TEST INFRASTRUCTURE ONLY: compiled by tests/costmap_pub_oracle.py.
 *
 * F1 every vertex through worldToMap; one outside the window: nothing is filled.
 * F2 fewer than 3 vertices: nothing is filled.
 * F3 the outline: raytraceLine from vertex k to k + 1 and from the last back to the first; bresenham2D visits abs_da
 *    offsets and then the end one, each turned into (mx, my) by indexToCells.
 * F4 bubble sort by x (a swap steps i back), then the column walk pairing cells i, i + 1, widening by the cells of the
 *    same x, and appending (x, y) for min.y <= y < max.y to the list being walked. */
#include <math.h>
#include <stdlib.h>

typedef struct { unsigned x, y; } loc;

/* growable list of map locations */
typedef struct { loc *v; long n, cap; } list;
static void push(list *l, unsigned x, unsigned y)
{
    if (l->n == l->cap) {
        l->cap = l->cap ? 2 * l->cap : 64;
        l->v = (loc *)realloc(l->v, (size_t)l->cap * sizeof(loc));
    }
    l->v[l->n].x = x;
    l->v[l->n].y = y;
    l->n++;
}

static int world_to_map(const double w[3], const int size[2], double wx, double wy, unsigned *mx, unsigned *my)
{
    double qx, qy;
    if (!(wx >= w[0]) || !(wy >= w[1])) return 0;
    qx = (wx - w[0]) / w[2];
    qy = (wy - w[1]) / w[2];
    if (!(qx < 2147483648.0) || !(qy < 2147483648.0)) return 0;
    *mx = (unsigned)(int)qx;
    *my = (unsigned)(int)qy;
    return *mx < (unsigned)size[0] && *my < (unsigned)size[1];
}

static void bresenham2d(list *cells, unsigned size_x, unsigned abs_da, unsigned abs_db, int error_b, int offset_a, int offset_b,
                        unsigned offset, unsigned max_length)
{
    unsigned end = max_length < abs_da ? max_length : abs_da, i;
    for (i = 0; i < end; ++i) {
        push(cells, offset % size_x, offset / size_x);
        offset += offset_a;
        error_b += abs_db;
        if ((unsigned)error_b >= abs_da) {
            offset += offset_b;
            error_b -= abs_da;
        }
    }
    push(cells, offset % size_x, offset / size_x);
}

static int sgn(int x) { return x > 0 ? 1.0 : -1.0; }

static void raytrace_line(list *cells, unsigned size_x, unsigned x0, unsigned y0, unsigned x1, unsigned y1)
{
    unsigned max_length = 0xFFFFFFFFu;
    int dx = x1 - x0, dy = y1 - y0;
    unsigned abs_dx = abs(dx), abs_dy = abs(dy);
    int offset_dx = sgn(dx), offset_dy = sgn(dy) * size_x;
    unsigned offset = y0 * size_x + x0;
    double dist = hypot(dx, dy);
    double scale = (dist == 0.0) ? 1.0 : fmin(1.0, max_length / dist);
    if (abs_dx >= abs_dy) {
        int error_y = abs_dx / 2;
        bresenham2d(cells, size_x, abs_dx, abs_dy, error_y, offset_dx, offset_dy, offset, (unsigned)(scale * abs_dx));
        return;
    }
    int error_x = abs_dy / 2;
    bresenham2d(cells, size_x, abs_dy, abs_dx, error_x, offset_dy, offset_dx, offset, (unsigned)(scale * abs_dy));
}

/* convexFillCells after polygonOutlineCells: quick bubble sort by x, then the column walk over the growing list */
static void column_walk(list *pc)
{
    long i = 0;
    if (pc->n == 0) return;
    while (i < pc->n - 1) {
        if (pc->v[i].x > pc->v[i + 1].x) {
            loc t = pc->v[i];
            pc->v[i] = pc->v[i + 1];
            pc->v[i + 1] = t;
            if (i > 0) --i;
        } else {
            ++i;
        }
    }
    {
        loc min_pt, max_pt;
        unsigned min_x = pc->v[0].x, max_x = pc->v[pc->n - 1].x, x, y;
        i = 0;
        for (x = min_x; x <= max_x; ++x) {
            if (i >= pc->n - 1) break;
            if (pc->v[i].y < pc->v[i + 1].y) {
                min_pt = pc->v[i];
                max_pt = pc->v[i + 1];
            } else {
                min_pt = pc->v[i + 1];
                max_pt = pc->v[i];
            }
            i += 2;
            while (i < pc->n && pc->v[i].x == x) {
                if (pc->v[i].y < min_pt.y) min_pt = pc->v[i];
                else if (pc->v[i].y > max_pt.y) max_pt = pc->v[i];
                ++i;
            }
            for (y = min_pt.y; y < max_pt.y; ++y) push(pc, x, y);
        }
    }
}

/* the column walk alone on a crafted list of n (x, y) cells: the result into out_xy; returns its length (-2: capacity) */
long orc_column_walk(const unsigned *cells_xy, long n, unsigned *out_xy, long capacity)
{
    list pc = {0, 0, 0};
    long i, ret;
    for (i = 0; i < n; i++) push(&pc, cells_xy[2 * i], cells_xy[2 * i + 1]);
    column_walk(&pc);
    ret = pc.n > capacity ? -2 : pc.n;
    for (i = 0; ret >= 0 && i < pc.n; i++) {
        out_xy[2 * i] = pc.v[i].x;
        out_xy[2 * i + 1] = pc.v[i].y;
    }
    free(pc.v);
    return ret;
}

/* the footprint at the pose (double), the cells setConvexPolygonCost writes (into cells_xy, capacity pairs) and the
 * vertices' touch bounds.  Returns the number of cells (duplicates included), -1 when a vertex lies outside, -2 when the
 * list exceeds capacity. */
long orc_footprint(const double w[3], const int size[2], const double *spec_xy, int n, double rx, double ry, double yaw,
                   double *verts_xy, unsigned *cells_xy, long capacity)
{
    double c = cos(yaw), s = sin(yaw);
    list poly = {0, 0, 0}, pc = {0, 0, 0};
    long i, k, ret;
    for (k = 0; k < n; k++) {
        verts_xy[2 * k] = rx + (spec_xy[2 * k] * c - spec_xy[2 * k + 1] * s);
        verts_xy[2 * k + 1] = ry + (spec_xy[2 * k] * s + spec_xy[2 * k + 1] * c);
    }
    for (k = 0; k < n; k++) {
        unsigned mx, my;
        if (!world_to_map(w, size, verts_xy[2 * k], verts_xy[2 * k + 1], &mx, &my)) {
            free(poly.v);
            return -1;
        }
        push(&poly, mx, my);
    }
    if (poly.n >= 3) {
        /* polygonOutlineCells */
        for (i = 0; i < poly.n - 1; ++i) raytrace_line(&pc, size[0], poly.v[i].x, poly.v[i].y, poly.v[i + 1].x, poly.v[i + 1].y);
        raytrace_line(&pc, size[0], poly.v[poly.n - 1].x, poly.v[poly.n - 1].y, poly.v[0].x, poly.v[0].y);
        column_walk(&pc);
    }
    ret = pc.n;
    if (pc.n > capacity) ret = -2;
    else
        for (i = 0; i < pc.n; i++) {
            cells_xy[2 * i] = pc.v[i].x;
            cells_xy[2 * i + 1] = pc.v[i].y;
        }
    free(poly.v);
    free(pc.v);
    return ret;
}
