/* orc_pointcloud2.c -- oracle of gem_pointcloud2_mapping / gem_decode_pointcloud2 (DESIGN.md f12).  TEST INFRASTRUCTURE ONLY.
 *
 * A literal, single-threaded restatement of PCL 1.8's createMapping<PointXYZRGBICT> (FieldMapper, FieldMatches, the sort
 * and coalesce loop) and fromPCLPointCloud2 (the whole-point memcpy and the per-span memcpy loop).  PCL is unpinned and
 * not available.  The rules, where the reference is undefined the library's DEFINITIONS:
 *   M1 struct fields x 0, y 4, z 8, rgb 16, intensity 24, covariance 20, travers 28 in this order each take the first
 *      message field with an equal name, datatype FLOAT32 (7) and count 1 or 0.
 *   M2 sorted by message offset; j merges into i when j.ser - i.ser == j.str - i.str (uint32), i.size += (j.str + j.size)
 *      - (i.str + i.size).
 *   M3 one span at 0 / 0 with point_step == 32: every point's 32 bytes; else every span of every point, in span order,
 *      from row * row_step + col * point_step.
 *   DEFINED: the 32-byte records start as zero bytes (the reference's are stale heap memory).
 *   DEFINED: refused (return 1, nothing written): a datatype outside 1..8, width * height > INT_MAX, and with points: a
 *      matched field past point_step, two matched fields overlapping, row_step < width * point_step, data shorter than
 *      (height - 1) * row_step + width * point_step. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { char name[32]; unsigned offset; unsigned char datatype; unsigned count; } orc_pointfield;
typedef struct {
    unsigned width, height, point_step, row_step;
    unsigned char is_bigendian;
    int nfields;
    const orc_pointfield *fields;
} orc_pointcloud2;
typedef struct { unsigned serialized_offset, struct_offset, size; } orc_span;
typedef struct { int nspans; orc_span spans[7]; int fast_path; unsigned matched; long long points; unsigned long long bytes; } orc_pc2_mapping;

static const char *const NAMES[7] = {"x", "y", "z", "rgb", "intensity", "covariance", "travers"};
static const unsigned OFFSETS[7] = {0, 4, 8, 16, 24, 20, 28};

static int by_serialized(const void *a, const void *b)
{
    const orc_span *x = (const orc_span *)a, *y = (const orc_span *)b;
    return x->serialized_offset < y->serialized_offset ? -1 : x->serialized_offset > y->serialized_offset;
}

static int orc_map(const orc_pointcloud2 *msg, unsigned long long data_bytes, orc_pc2_mapping *out)
{
    orc_pc2_mapping r;
    memset(&r, 0, sizeof r);
    for (int f = 0; f < msg->nfields; f++)
        if (msg->fields[f].datatype < 1 || msg->fields[f].datatype > 8) return 1;
    const unsigned long long n = (unsigned long long)msg->width * msg->height;
    if (n > 2147483647ull) return 1;
    orc_span map[7];
    int nm = 0;
    for (int k = 0; k < 7; k++) {                                 /* FieldMapper: for_each_type in registration order */
        for (int f = 0; f < msg->nfields; f++) {
            const orc_pointfield *pf = &msg->fields[f];
            if (memchr(pf->name, 0, 32) == NULL || strcmp(pf->name, NAMES[k]) != 0) continue;
            if (pf->datatype != 7 || !(pf->count == 1 || pf->count == 0)) continue; /* FieldMatches, size 1 */
            map[nm].serialized_offset = pf->offset;
            map[nm].struct_offset = OFFSETS[k];
            map[nm].size = 4;
            nm++;
            r.matched |= 1u << k;
            break;
        }
    }
    qsort(map, (size_t)nm, sizeof map[0], by_serialized);         /* fieldOrdering */
    if (n > 0) {
        for (int i = 0; i < nm; i++)
            if ((unsigned long long)map[i].serialized_offset + map[i].size > msg->point_step) return 1;
        for (int i = 1; i < nm; i++)
            if ((unsigned long long)map[i - 1].serialized_offset + map[i - 1].size > map[i].serialized_offset) return 1;
        if ((unsigned long long)msg->row_step < (unsigned long long)msg->width * msg->point_step) return 1;
        r.bytes = (unsigned long long)(msg->height - 1) * msg->row_step + (unsigned long long)msg->width * msg->point_step;
        if (data_bytes < r.bytes) return 1;
    }
    /* coalesce: i = first, j = i + 1; merge and erase j, or advance both */
    int i = 0;
    for (int j = 1; j < nm; j++) {
        if (map[j].serialized_offset - map[i].serialized_offset == map[j].struct_offset - map[i].struct_offset) {
            map[i].size += (map[j].struct_offset + map[j].size) - (map[i].struct_offset + map[i].size);
        } else {
            i++;
            map[i] = map[j];
        }
    }
    r.nspans = nm ? i + 1 : 0;
    memcpy(r.spans, map, sizeof(orc_span) * (size_t)r.nspans);
    r.fast_path = r.nspans == 1 && r.spans[0].serialized_offset == 0 && r.spans[0].struct_offset == 0 && msg->point_step == 32;
    r.points = (long long)n;
    *out = r;
    return 0;
}

/* fromPCLPointCloud2 into n 32-byte records (zeroed first) */
int orc_pc2_decode(const orc_pointcloud2 *msg, const unsigned char *data, unsigned long long data_bytes, unsigned char *records,
                   orc_pc2_mapping *mapping_out)
{
    orc_pc2_mapping mp;
    if (orc_map(msg, data_bytes, &mp)) return 1;
    if (mapping_out) *mapping_out = mp;
    memset(records, 0, (size_t)mp.points * 32);
    unsigned char *cloud = records;
    if (mp.fast_path) {
        const size_t cloud_row_step = (size_t)32 * msg->width;
        for (unsigned row = 0; row < msg->height; row++)
            memcpy(cloud + row * cloud_row_step, data + (size_t)row * msg->row_step, cloud_row_step);
        return 0;
    }
    for (unsigned row = 0; row < msg->height; row++) {
        const unsigned char *row_data = data + (size_t)row * msg->row_step;
        for (unsigned col = 0; col < msg->width; col++) {
            const unsigned char *msg_data = row_data + (size_t)col * msg->point_step;
            for (int s = 0; s < mp.nspans; s++)
                memcpy(cloud + mp.spans[s].struct_offset, msg_data + mp.spans[s].serialized_offset, mp.spans[s].size);
            cloud += 32;
        }
    }
    return 0;
}
