/* orc_gridmsg.c -- oracle of the f18 calls (DESIGN.md f18): gem_grid_map_msg_parse, gem_costmap_mark_grid and
 * gem_decode_pointcloud2_records.  TEST INFRASTRUCTURE ONLY.
 *
 * A literal, single-threaded restatement of what ElevationMapLayer::elevationMapCB / updateBounds
 * (layers/src/elevationMap_layer.cpp:31-84) compute from a serialised grid_map_msgs/GridMap, with grid_map 1.6's
 * fromMessage, setGeometry, GridMapIterator and getPositionFromIndex restated (unpinned):
 *   G1 size = (int)round(length / resolution), length = size * resolution, position = pose.position.{x, y}, start index
 *      = (outer_start_index, inner_start_index).
 *   G2 layer i goes with data[i]; the last layer of a repeated name wins (gridMap.add replaces).
 *   G3 dim[0].label "column_index" only; rows = dim[1].size, cols = dim[0].size; data_offset and floats beyond rows * cols
 *      ignored.
 *   G4 element k of the layer is buffer index (k % size_x, k / size_x); position (position + (0.5 length - 0.5 res)) +
 *      res * (-((index - start) mod size)), in double.
 *   Refused (return 1, nothing written), the library's DEFINITIONS: a truncated message, layers.size() != data.size(), the
 *   layer missing, fewer than two dims or dim[0] not "column_index", (rows, cols) != (size_x, size_y), fewer floats than
 *   rows * cols, a resolution or length <= 0 or not finite, a size or size_x * size_y above INT_MAX.
 * The message is deserialised whole first (every field into its own variable, as roscpp does), then fromMessage is run on
 * it.  The mark loop reuses tests/orc_costmap.c's worldToMap and touch; the records reuse tests/orc_pointcloud2.c.
 * Compiled with -ffp-contract=off. */
#include "orc_costmap.c"
#include "orc_pointcloud2.c"

#include <stdint.h>

typedef struct {
    double resolution, position_x, position_y, length_x, length_y;
    int size_x, size_y, start_x, start_y;
    unsigned long long offset;
    long long floats;
    int column_major;
} orc_grid_layer;

typedef struct { const unsigned char *p; unsigned long long n, at; int bad; } rd;

static int rd_need(rd *r, unsigned long long k)
{
    if (r->bad || r->n - r->at < k) { r->bad = 1; return 0; }
    return 1;
}
static uint32_t rd_u32(rd *r)
{
    uint32_t v = 0;
    if (rd_need(r, 4)) { memcpy(&v, r->p + r->at, 4); r->at += 4; }
    return v;
}
static uint16_t rd_u16(rd *r)
{
    uint16_t v = 0;
    if (rd_need(r, 2)) { memcpy(&v, r->p + r->at, 2); r->at += 2; }
    return v;
}
static double rd_f64(rd *r)
{
    double v = 0;
    if (rd_need(r, 8)) { memcpy(&v, r->p + r->at, 8); r->at += 8; }
    return v;
}
/* a string: its start and length, skipped */
static void rd_str(rd *r, unsigned long long *s, uint32_t *len)
{
    *len = rd_u32(r);
    *s = r->at;
    if (rd_need(r, *len)) r->at += *len;
}

typedef struct { unsigned long long name_at; uint32_t name_len; } orc_name;
typedef struct {
    uint32_t ndim;
    int dim0_column_index;
    uint32_t dim0_size, dim1_size;
    uint32_t nfloats;
    unsigned long long floats_at;
} orc_array;

int orc_grid_map_parse(const unsigned char *msg, unsigned long long bytes, const char *layer, orc_grid_layer *out)
{
    rd r = {msg, bytes, 0, 0};
    unsigned long long s;
    uint32_t len;
    /* deserialise */
    rd_u32(&r); rd_u32(&r); rd_u32(&r);
    rd_str(&r, &s, &len);
    const double resolution = rd_f64(&r), length_x = rd_f64(&r), length_y = rd_f64(&r);
    const double pos_x = rd_f64(&r), pos_y = rd_f64(&r);
    for (int k = 0; k < 5; k++) rd_f64(&r);
    const uint32_t nlayers = rd_u32(&r);
    if (r.bad || nlayers > (r.n - r.at) / 4) return 1;                    /* each string holds its 4-byte count at least */
    orc_name *names = (orc_name *)calloc(nlayers ? nlayers : 1, sizeof *names);
    for (uint32_t i = 0; i < nlayers && !r.bad; i++) rd_str(&r, &names[i].name_at, &names[i].name_len);
    const uint32_t nbasic = rd_u32(&r);
    for (uint32_t i = 0; i < nbasic && !r.bad; i++) rd_str(&r, &s, &len);
    const uint32_t ndata = rd_u32(&r);
    if (!r.bad && ndata > (r.n - r.at) / 12) r.bad = 1;                  /* each array holds 3 counts at least */
    orc_array *data = r.bad ? NULL : (orc_array *)calloc(ndata ? ndata : 1, sizeof *data);
    for (uint32_t i = 0; i < ndata && !r.bad; i++) {
        orc_array *a = &data[i];
        a->ndim = rd_u32(&r);
        for (uint32_t d = 0; d < a->ndim && !r.bad; d++) {
            rd_str(&r, &s, &len);
            const int col = !r.bad && len == 12 && memcmp(msg + s, "column_index", 12) == 0;
            const uint32_t size = rd_u32(&r);
            rd_u32(&r);
            if (d == 0) { a->dim0_column_index = col; a->dim0_size = size; }
            if (d == 1) a->dim1_size = size;
        }
        rd_u32(&r);
        a->nfloats = rd_u32(&r);
        a->floats_at = r.at;
        if (rd_need(&r, 4ull * a->nfloats)) r.at += 4ull * a->nfloats;
    }
    const int start_x = rd_u16(&r), start_y = rd_u16(&r);
    int rc = 1;
    if (r.bad) goto done;
    /* fromMessage: setGeometry (G1) */
    if (!(isfinite(resolution) && resolution > 0.0)) goto done;
    if (!(isfinite(length_x) && length_x > 0.0 && isfinite(length_y) && length_y > 0.0)) goto done;
    const double qx = round(length_x / resolution), qy = round(length_y / resolution);
    if (!(qx <= 2147483647.0 && qy <= 2147483647.0)) goto done;
    const int size_x = (int)qx, size_y = (int)qy;
    if ((long long)size_x * size_y > 2147483647ll) goto done;
    if (nlayers != ndata) goto done;
    /* the layers in order, a later one of the same name replacing an earlier one (G2) */
    long long found = -1;
    for (uint32_t i = 0; i < nlayers; i++)
        if (names[i].name_len == strlen(layer) && memcmp(msg + names[i].name_at, layer, names[i].name_len) == 0) found = i;
    if (found < 0) goto done;
    const orc_array *a = &data[found];
    if (a->ndim < 2 || !a->dim0_column_index) goto done;                  /* G3 */
    if (a->dim1_size != (uint32_t)size_x || a->dim0_size != (uint32_t)size_y) goto done;
    if ((unsigned long long)a->nfloats < (unsigned long long)a->dim1_size * a->dim0_size) goto done;
    memset(out, 0, sizeof *out);
    out->resolution = resolution;
    out->position_x = pos_x;
    out->position_y = pos_y;
    out->size_x = size_x;
    out->size_y = size_y;
    out->length_x = size_x * resolution;
    out->length_y = size_y * resolution;
    out->start_x = start_x;
    out->start_y = start_y;
    out->offset = a->floats_at;
    out->floats = (long long)size_x * size_y;
    out->column_major = 1;
    rc = 0;
done:
    free(names);
    free(data);
    return rc;
}

/* grid_map's getIndexFromBufferIndex: (index - start) wrapped into [0, size) */
static int unwrap(int index, int start, int size)
{
    long long u = ((long long)index - start) % size;
    return (int)(u < 0 ? u + size : u);
}

/* ElevationMapLayer::updateBounds over the layer's floats (G4 order), last writer wins */
void orc_mark_grid(const orc_grid_layer *g, const float *layer, const orc_window *w, double travers_thresh, int mark_unknown,
                   unsigned char *costmap, orc_marks *out)
{
    marks_begin(out);
    const double ox = g->position_x + (0.5 * g->length_x - 0.5 * g->resolution);
    const double oy = g->position_y + (0.5 * g->length_y - 0.5 * g->resolution);
    for (long long k = 0; k < g->floats; k++) {                          /* GridMapIterator: the linear index */
        const int ix = (int)(k % g->size_x), iy = (int)(k / g->size_x);
        const float v = layer[k];
        if (!mark_unknown && isnan(v)) continue;
        const int is_obstacle = v < travers_thresh;
        const double px = ox + g->resolution * (double)(-unwrap(ix, g->start_x, g->size_x));
        const double py = oy + g->resolution * (double)(-unwrap(iy, g->start_y, g->size_y));
        unsigned mx, my;
        if (!world_to_map(w, px, py, &mx, &my)) continue;
        costmap[(size_t)my * w->size_x + mx] = is_obstacle ? LETHAL_OBSTACLE : FREE_SPACE;
        out->marked++;
        out->lethal += is_obstacle;
        touch(px, py, out);
    }
    marks_end(out);
}

/* fromPCLPointCloud2 into whole records: tests/orc_pointcloud2.c's decode */
int orc_pc2_records(const orc_pointcloud2 *msg, const unsigned char *data, unsigned long long data_bytes, unsigned char *records)
{
    return orc_pc2_decode(msg, data, data_bytes, records, NULL);
}
