// gem_gridmsg.h -- reading a serialised grid_map_msgs/GridMap (DESIGN.md f18): what GridMapRosConverter::fromMessage
// (grid_map 1.6, unpinned) derives from the message for ElevationMapLayer, and where one layer's floats are.  Host code
// only; the library and tests/gridmsg_host.cpp (built by the CPU suite with g++) compile the same definitions.  The
// rules G1-G4 are stated in include/gem_b200.h and restated in tests/orc_gridmsg.c and tests/gridmsg_oracle.py.
//
// The walk reads W1 / W2 of gem_rosfmt.h: header {seq, stamp, frame_id}, info {resolution, length_x, length_y, pose
// {position xyz, orientation xyzw}} (float64), layers (string[]), basic_layers (string[]), data (Float32MultiArray[]:
// layout {dim [{label, size, stride}], data_offset}, float32[]), outer_start_index, inner_start_index (uint16).
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../../include/gem_b200.h"

#if !defined(__BYTE_ORDER__) || __BYTE_ORDER__ != __ORDER_LITTLE_ENDIAN__
#error "gem_gridmsg.h reads ROS1's little-endian wire format with host loads"
#endif

namespace gem_gridmsg {

// a bounds-checked cursor over msg[0, n): every read fails once, and stays failed, when it would run past n
struct Reader {
    const unsigned char *p;
    unsigned long long n, at = 0;
    bool ok = true;
    bool take(unsigned long long k)
    {
        if (!ok || k > n - at) return ok = false;
        at += k;
        return true;
    }
    template <class T> T get()
    {
        T v{};
        const unsigned long long a = at;
        if (take(sizeof v)) memcpy(&v, p + a, sizeof v);
        return v;
    }
    // a string's bytes [*s, *s + *len) in the message
    bool str(unsigned long long *s, uint32_t *len)
    {
        *len = get<uint32_t>();
        *s = at;
        return take(*len);
    }
};

// G1 per axis: size = (int)round(length / resolution); false for a length or a quotient that is not finite, a size
// that does not fit an int (where the cast is undefined)
inline bool axis_size(double length, double resolution, int *size)
{
    if (!(isfinite(length) && length > 0.0)) return false;
    const double q = round(length / resolution);
    if (!(q <= 2147483647.0)) return false;
    *size = (int)q;
    return true;
}

// The descriptor of `layer` in msg[0, bytes) (G1-G3), or the reason it is refused (nothing written to *out)
inline const char *parse(const void *msg, unsigned long long bytes, const char *layer, gem_grid_map_layer *out)
{
    if (!msg || !layer || !out) return "bad argument";
    Reader r{static_cast<const unsigned char *>(msg), bytes};
    unsigned long long s;
    uint32_t len;
    r.get<uint32_t>(); r.get<uint32_t>(); r.get<uint32_t>(); // seq, stamp
    r.str(&s, &len);                                        // frame_id
    const double res = r.get<double>(), lx = r.get<double>(), ly = r.get<double>();
    const double px = r.get<double>(), py = r.get<double>();
    r.take(5 * 8);                                          // position.z, orientation: ignored (G1)
    const size_t want = strlen(layer);
    // G2: the last layer of the requested name
    const uint32_t nlayers = r.get<uint32_t>();
    long long match = -1;
    for (uint32_t i = 0; r.ok && i < nlayers; i++)
        if (r.str(&s, &len) && len == want && memcmp(r.p + s, layer, want) == 0) match = i;
    const uint32_t nbasic = r.get<uint32_t>();
    for (uint32_t i = 0; r.ok && i < nbasic; i++) r.str(&s, &len);
    const uint32_t ndata = r.get<uint32_t>();
    uint32_t ndim = 0, rows = 0, cols = 0, nfloats = 0;
    bool column_index = false;
    unsigned long long offset = 0;
    for (uint32_t i = 0; r.ok && i < ndata; i++) {
        const uint32_t nd = r.get<uint32_t>();
        for (uint32_t d = 0; r.ok && d < nd; d++) {
            r.str(&s, &len);
            const bool is_col = len == 12 && r.ok && memcmp(r.p + s, "column_index", 12) == 0;
            const uint32_t size = r.get<uint32_t>();
            r.get<uint32_t>();                              // stride
            if (i == match) {
                if (d == 0) column_index = is_col;
                if (d == 0) cols = size;
                if (d == 1) rows = size;
            }
        }
        r.get<uint32_t>();                                  // data_offset: ignored (G3)
        const uint32_t nf = r.get<uint32_t>();
        const unsigned long long at = r.at;
        r.take(4ull * nf);
        if (i == match) { ndim = nd; nfloats = nf; offset = at; }
    }
    const uint16_t sx = r.get<uint16_t>(), sy = r.get<uint16_t>();
    if (!r.ok) return "the message is truncated: a field, string or array runs past its end";
    if (nlayers != ndata) return "layers and data differ in length";
    if (match < 0) return "the layer is not in the message";
    if (ndim < 2 || !column_index) return "the layer's layout is not column-major (dim[0] \"column_index\", two dims)";
    if (!(isfinite(res) && res > 0.0)) return "the resolution is <= 0 or not finite";
    int size_x = 0, size_y = 0;
    if (!axis_size(lx, res, &size_x) || !axis_size(ly, res, &size_y))
        return "a length is <= 0 or not finite, or its size does not fit an int";
    if ((long long)size_x * size_y > 2147483647ll) return "size_x * size_y exceeds INT_MAX";
    if (rows != (uint32_t)size_x || cols != (uint32_t)size_y) return "the layer's rows and cols are not the map's size";
    if ((unsigned long long)nfloats < (unsigned long long)rows * cols) return "the layer holds fewer floats than rows * cols";
    gem_grid_map_layer g;
    memset(&g, 0, sizeof g);
    g.resolution = res;
    g.position_x = px;
    g.position_y = py;
    g.size_x = size_x;
    g.size_y = size_y;
    g.length_x = (double)size_x * res;
    g.length_y = (double)size_y * res;
    g.start_x = sx;
    g.start_y = sy;
    g.offset = offset;
    g.floats = (long long)size_x * size_y;
    g.column_major = 1;
    *out = g;
    return nullptr;
}

// what gem_costmap_mark_grid accepts of a descriptor (a caller may fill one by hand): G1 and G3's checks
inline bool layer_ok(const gem_grid_map_layer &g)
{
    return isfinite(g.resolution) && g.resolution > 0.0 && g.size_x >= 0 && g.size_y >= 0 &&
           (long long)g.size_x * g.size_y <= 2147483647ll && g.floats == (long long)g.size_x * g.size_y && g.column_major == 1 &&
           isfinite(g.length_x) && isfinite(g.length_y);
}

} // namespace gem_gridmsg
