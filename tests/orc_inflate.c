/* orc_inflate.c -- oracle of gem_costmap_inflate (DESIGN.md f14).  TEST INFRASTRUCTURE ONLY.
 *
 * A literal, single-threaded restatement of costmap_2d's InflationLayer::updateCosts with computeCaches, costLookup and
 * enqueue (navigation 1.14, unpinned): a list of bins sorted by their double key, each a growable vector taken in push
 * order by index, so an entry pushed into the bin being walked would be walked too, and a bin created before the one
 * being walked is passed over, as std::map's iterator does.  Compiled with the flags of orc_costmap.c.  The library's
 * DEFINITIONS are applied: r is capped at ceil(hypot(size_x, size_y)) + 1.  Items I1-I4 of DESIGN.md f14 are marked at the
 * code below.  I5 (updateBounds), I6 (LayeredCostmap::updateMap with two plugins) and I7 (calculateMinAndMaxDistances) are
 * host arithmetic with no cell loop; they live in gem_b200/costmap.py and the tests restate them there:
 *   I5 on the first update and after a parameter change the incoming bounds are saved as last_* and the bounds become
 *      -+FLT_MAX; later, min = min(last_min, min) - inflation_radius, max = max(last_max, max) + inflation_radius, and
 *      last_* becomes the incoming bounds;
 *   I6 the layers' updateBounds in plugin order from +-1e30, the update rect, resetMap of the rect, then the layers'
 *      updateCosts in plugin order: the point layer's overwrite (or the elevation layer's max), then this inflation;
 *   I7 the inscribed radius is the least hypot from the origin to a vertex or an edge of the padded footprint, the
 *      projection parameter of distanceToLine clamped to [0, 1]. */
#include <math.h>
#include <stdlib.h>
#include <string.h>

enum { FREE_SPACE = 0, INSCRIBED_INFLATED_OBSTACLE = 253, LETHAL_OBSTACLE = 254, NO_INFORMATION = 255 };

typedef struct { int index, x, y, src_x, src_y; } cell_data;
typedef struct { double key; cell_data *v; size_t n, cap; } bin;
typedef struct { bin *b; size_t n, cap; } bin_list;

static bin *bin_at(bin_list *l, double key, size_t *walk)
{
    size_t lo = 0, hi = l->n;
    while (lo < hi) {
        const size_t mid = (lo + hi) / 2;
        if (l->b[mid].key < key) lo = mid + 1; else hi = mid;
    }
    if (lo < l->n && l->b[lo].key == key) return &l->b[lo];
    if (l->n == l->cap) {
        l->cap = l->cap ? 2 * l->cap : 16;
        l->b = realloc(l->b, l->cap * sizeof(bin));
    }
    memmove(&l->b[lo + 1], &l->b[lo], (l->n - lo) * sizeof(bin));
    l->b[lo] = (bin){key, NULL, 0, 0};
    l->n++;
    if (walk && lo <= *walk) (*walk)++; /* a key before the walked bin: the walk stays on its bin */
    return &l->b[lo];
}

static void push(bin *b, cell_data c)
{
    if (b->n == b->cap) {
        b->cap = b->cap ? 2 * b->cap : 16;
        b->v = realloc(b->v, b->cap * sizeof(cell_data));
    }
    b->v[b->n++] = c;
}

/* returns the number of cells popped */
long long orc_inflate(unsigned char *master, int size_x, int size_y, double resolution, double inflation_radius, double weight,
                      double inscribed_radius, int inflate_unknown, int min_i, int min_j, int max_i, int max_j)
{
    /* I1 cellDistance: r = (unsigned)max(0.0, ceil(inflation_radius / resolution)), with the DEFINED cap; r == 0 writes
     * nothing */
    double rd = ceil(inflation_radius / resolution);
    if (rd < 0.0) rd = 0.0;
    const double cap = ceil(hypot((double)size_x, (double)size_y)) + 1.0;
    if (rd > cap) rd = cap;
    const unsigned r = (unsigned)rd;
    if (r == 0) return 0;
    /* I2 computeCaches for 0 <= i, j <= r + 1: dist = hypot(i, j); cost 254 at 0, 253 when dist * resolution <= inscribed,
     * else (unsigned char)(252 * exp(-weight * (dist * resolution - inscribed))), with the host's libm */
    const unsigned tw = r + 2;
    double *dist = malloc((size_t)tw * tw * sizeof(double));
    unsigned char *cost = malloc((size_t)tw * tw);
    for (unsigned i = 0; i < tw; i++)
        for (unsigned j = 0; j < tw; j++) {
            const double d = hypot((double)i, (double)j);
            dist[i * tw + j] = d;
            unsigned char c;
            if (d == 0) c = LETHAL_OBSTACLE;
            else if (d * resolution <= inscribed_radius) c = INSCRIBED_INFLATED_OBSTACLE;
            else c = (unsigned char)((INSCRIBED_INFLATED_OBSTACLE - 1) * exp(-1.0 * weight * (d * resolution - inscribed_radius)));
            cost[i * tw + j] = c;
        }
    /* I3 the rect widened by r on every side and clamped to the grid; its LETHAL cells go into bin 0.0 in row-major order
     * (j outer, i inner), each its own source */
    long long mi = (long long)min_i - r, mj = (long long)min_j - r, xi = (long long)max_i + r, xj = (long long)max_j + r;
    if (mi < 0) mi = 0;
    if (mj < 0) mj = 0;
    if (xi > size_x) xi = size_x;
    if (xj > size_y) xj = size_y;
    unsigned char *seen = calloc((size_t)size_x * size_y, 1);
    bin_list bins = {NULL, 0, 0};
    bin *obs = bin_at(&bins, 0.0, NULL);
    for (long long j = mj; j < xj; j++)
        for (long long i = mi; i < xi; i++) {
            const int index = (int)(j * size_x + i);
            if (master[index] == LETHAL_OBSTACLE) push(obs, (cell_data){index, (int)i, (int)j, (int)i, (int)j});
        }
    /* I4 the bins in increasing key, each in push order: a seen cell is skipped; otherwise it is marked seen, takes
     * c = cost[|mx - sx|][|my - sy|] by the write rule, and pushes its four neighbours (inside the grid, unseen, same
     * source) into bin dist[|nx - sx|][|ny - sy|] unless that is > r.  seen is cleared per call. */
    long long popped = 0;
    for (size_t b = 0; b < bins.n; b++) {
        for (size_t k = 0; k < bins.b[b].n; k++) {
            const cell_data c = bins.b[b].v[k];
            const int index = c.index;
            if (seen[index]) continue;
            seen[index] = 1;
            popped++;
            const int mx = c.x, my = c.y, sx = c.src_x, sy = c.src_y;
            const unsigned char cc = cost[(unsigned)abs(mx - sx) * tw + (unsigned)abs(my - sy)];
            const unsigned char old = master[index];
            if (old == NO_INFORMATION && (inflate_unknown ? (cc > FREE_SPACE) : (cc >= INSCRIBED_INFLATED_OBSTACLE)))
                master[index] = cc;
            else
                master[index] = old > cc ? old : cc;
            /* enqueue(index, mx, my, src_x, src_y) of the four neighbours */
            const int nb[4][3] = {{mx > 0, index - 1, 0}, {my > 0, index - size_x, 1}, {mx < size_x - 1, index + 1, 2},
                                  {my < size_y - 1, index + size_x, 3}};
            for (int d = 0; d < 4; d++) {
                if (!nb[d][0]) continue;
                const int ni = nb[d][1];
                if (seen[ni]) continue;
                const int nx = mx + (d == 0 ? -1 : d == 2 ? 1 : 0), ny = my + (d == 1 ? -1 : d == 3 ? 1 : 0);
                const double dd = dist[(unsigned)abs(nx - sx) * tw + (unsigned)abs(ny - sy)];
                if (dd > r) continue;
                push(bin_at(&bins, dd, &b), (cell_data){ni, nx, ny, sx, sy});
            }
        }
    }
    for (size_t b = 0; b < bins.n; b++) free(bins.b[b].v);
    free(bins.b);
    free(seen);
    free(cost);
    free(dist);
    return popped;
}
