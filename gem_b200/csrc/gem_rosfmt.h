// gem_rosfmt.h -- the framing of the ROS1 messages GEM's node publishes (DESIGN.md f15): every byte of a serialised
// message that is not map data, and where the data goes.  Host code only; the library and tests/rosmsg_fmt_host.cpp
// (built by the CPU suite with g++) compile the same definitions.  ROS, grid_map, PCL and cv_bridge are unpinned
// dependencies; the wire format is restated here, in include/gem_b200.h and in tests/rosmsg_oracle.py.
//
// W1 ROS1 serialisation: little-endian, unpadded.  string = uint32 byte count + bytes (no NUL); variable array = uint32
//    element count + elements; time = uint32 sec + uint32 nsec; bool = 1 byte; a nested message is its fields in order.
//    std_msgs/Header = seq, stamp, frame_id, written as the caller passes them.
// W2 grid_map_msgs/GridMap (grid_map 1.6 toMessage): info {header, resolution, length_x, length_y (float64), pose
//    {position (cx, cy, 0), orientation (0, 0, 0, 1)} (float64)}, layers (the 9 of ElevationMap.cpp:44), basic_layers
//    {"elevation"}, data: 9 Float32MultiArray {dim {"column_index", L, L^2}, {"row_index", L, L}, data_offset 0, L^2
//    floats (gem_export_layers' column-major layer)}, outer_start_index, inner_start_index (uint16).
//    737 + |frame_id| + 36 L^2 bytes; layer k's floats at 277 + |frame_id| + k (57 + 4 L^2).
// W3 sensor_msgs/Image: header, height = width = L, "bgr8", is_bigendian 0, step 3L, 3L^2 bytes.  41 + |frame_id| + 3 L^2.
// W4 sensor_msgs/PointCloud2 (pcl::toROSMsg): header, height 1, width n, fields {name, offset, datatype 7, count 1} in
//    registration order, is_bigendian 0, point_step 32, row_step 32n, 32n bytes, is_dense.  32n >= 2^32 is refused.
// W5 PointXYZRGBICT: fields x 0, y 4, z 8, rgb 16, intensity 24, covariance 20, travers 28.  165 + |frame_id| + 32n.
// W6 pcl::PointXYZRGB: fields x 0, y 4, z 8, rgb 16.  100 + |frame_id| + 32n.
// W7 octomap_msgs/Octomap (fullMapToMsg): header, binary 0, id "ColorOcTree", resolution (float64), int8[] stream.
//    44 + |frame_id| + bytes.
// W9-W11 and the publisher's decision P1-P4 (DESIGN.md f17, costmap_2d of navigation 1.14): below and in
//    include/gem_b200.h.
#pragma once
#include <stdint.h>
#include <string.h>

#include <string>

#include "../../include/gem_b200.h"

#if !defined(__BYTE_ORDER__) || __BYTE_ORDER__ != __ORDER_LITTLE_ENDIAN__
#error "gem_rosfmt.h writes ROS1's little-endian wire format with host stores"
#endif

#ifdef __CUDACC__
#define GEM_RF __host__ __device__ __forceinline__
#else
#define GEM_RF inline
#endif

namespace gem_ros {

constexpr int MAX_SEGS = 10;   // the grid map's: the part before layer 0's floats, 8 between layers, the start indices
constexpr int MAX_PAYLOADS = 9;
constexpr int GRID_LAYERS = 9;
constexpr long long U32_LIMIT = 1ll << 32;

// framing bytes bytes[src, src + len) belong at message offset `at`
struct Seg {
    long long at, src, len;
};

// A message as framing segments and payload runs, in message order.  The framing bytes are collected in `bytes`; a
// payload run is a hole the device fills (layer floats, image bytes, records, the octree stream).
struct Framing {
    std::string bytes;
    Seg seg[MAX_SEGS];
    int nseg = 0;
    long long payload_at[MAX_PAYLOADS], payload_len[MAX_PAYLOADS];
    int npayload = 0;
    long long size = 0;

    void put(const void *p, size_t n)
    {
        if (nseg == 0 || seg[nseg - 1].at + seg[nseg - 1].len != size) seg[nseg++] = Seg{size, (long long)bytes.size(), 0};
        bytes.append(static_cast<const char *>(p), n);
        seg[nseg - 1].len += (long long)n;
        size += (long long)n;
    }
    void u8(uint8_t v) { put(&v, 1); }
    void u16(uint16_t v) { put(&v, 2); }
    void u32(uint32_t v) { put(&v, 4); }
    void f64(double v) { put(&v, 8); }
    void str(const char *s, size_t n)
    {
        u32((uint32_t)n);
        if (n) put(s, n);
    }
    void str(const char *s) { str(s, strlen(s)); }
    void header(const gem_ros_header &h)
    {
        u32(h.seq);
        u32(h.stamp_sec);
        u32(h.stamp_nsec);
        str(h.frame_id);
    }
    void payload(long long n)
    {
        payload_at[npayload] = size;
        payload_len[npayload++] = n;
        size += n;
    }
};

// the header's frame_id may be any length that keeps the message's uint32 counts valid
inline bool header_ok(const gem_ros_header *h) { return h && h->frame_id && strlen(h->frame_id) < (size_t)(U32_LIMIT / 2); }

// W2
inline int grid_map(const gem_ros_header &h, int L, double res, double cx, double cy, int sx, int sy, Framing &f)
{
    static const char *const layers[GRID_LAYERS] = {"elevation", "variance", "rough", "slope", "traver",
                                                    "color_r", "color_g", "color_b", "intensity"};
    const long long cells = (long long)L * L;
    if (L <= 0 || 4 * cells >= U32_LIMIT) return GEM_ERR_INVALID;
    f.header(h);
    f.f64(res);
    f.f64((double)L * res);
    f.f64((double)L * res);
    f.f64(cx); f.f64(cy); f.f64(0.0);
    f.f64(0.0); f.f64(0.0); f.f64(0.0); f.f64(1.0);
    f.u32(GRID_LAYERS);
    for (const char *s : layers) f.str(s);
    f.u32(1);
    f.str("elevation");
    f.u32(GRID_LAYERS);
    for (int k = 0; k < GRID_LAYERS; k++) {
        f.u32(2);
        f.str("column_index"); f.u32((uint32_t)L); f.u32((uint32_t)cells);
        f.str("row_index"); f.u32((uint32_t)L); f.u32((uint32_t)L);
        f.u32(0);
        f.u32((uint32_t)cells);
        f.payload(4 * cells);
    }
    f.u16((uint16_t)sx);
    f.u16((uint16_t)sy);
    return GEM_OK;
}

// W3
inline int image(const gem_ros_header &h, int L, Framing &f)
{
    const long long bytes = 3ll * L * L;
    if (L <= 0 || bytes >= U32_LIMIT) return GEM_ERR_INVALID;
    f.header(h);
    f.u32((uint32_t)L);
    f.u32((uint32_t)L);
    f.str("bgr8");
    f.u8(0);
    f.u32((uint32_t)(3 * L));
    f.u32((uint32_t)bytes);
    f.payload(bytes);
    return GEM_OK;
}

enum CloudKind { CLOUD_XYZRGBICT = 0, CLOUD_XYZRGB = 1 };

// W4 with W5's or W6's fields
inline int cloud(const gem_ros_header &h, CloudKind kind, long long n, int is_dense, Framing &f)
{
    struct Field { const char *name; uint32_t offset; };
    static const Field ict[] = {{"x", 0}, {"y", 4}, {"z", 8}, {"rgb", 16}, {"intensity", 24}, {"covariance", 20}, {"travers", 28}};
    static const Field rgb[] = {{"x", 0}, {"y", 4}, {"z", 8}, {"rgb", 16}};
    if (n < 0 || 32 * n >= U32_LIMIT) return GEM_ERR_INVALID;
    const Field *fields = kind == CLOUD_XYZRGB ? rgb : ict;
    const int nf = kind == CLOUD_XYZRGB ? 4 : 7;
    f.header(h);
    f.u32(1);
    f.u32((uint32_t)n);
    f.u32((uint32_t)nf);
    for (int i = 0; i < nf; i++) {
        f.str(fields[i].name);
        f.u32(fields[i].offset);
        f.u8(7); // sensor_msgs::PointField::FLOAT32
        f.u32(1);
    }
    f.u8(0);
    f.u32(32);
    f.u32((uint32_t)(32 * n));
    f.u32((uint32_t)(32 * n));
    f.payload(32 * n);
    f.u8(is_dense ? 1 : 0);
    return GEM_OK;
}

// W7
inline int octomap(const gem_ros_header &h, double resolution, long long bytes, Framing &f)
{
    if (bytes < 0 || bytes >= U32_LIMIT) return GEM_ERR_INVALID;
    f.header(h);
    f.u8(0);
    f.str("ColorOcTree");
    f.f64(resolution);
    f.u32((uint32_t)bytes);
    f.payload(bytes);
    return GEM_OK;
}

// ---- the costmap topics (DESIGN.md f17) ----
// T, Costmap2DPublisher's cost_translation_table_: 0 -> 0, 253 -> 99, 254 -> 100, 255 -> -1, and 1..252 scaled into 1..98
// in integer arithmetic (the device's too: k_ros_costmap)
GEM_RF signed char cost_translate(unsigned c)
{
    if (c == 0) return 0;
    if (c == 253) return 99;
    if (c == 254) return 100;
    if (c == 255) return -1;
    return (signed char)(1 + (97 * ((int)c - 1)) / 251);
}

// W9 nav_msgs/OccupancyGrid (prepareGrid): the data (size_x size_y bytes) is the payload
inline int occupancy_grid(const gem_ros_header &h, const gem_costmap_window &w, Framing &f)
{
    const long long cells = (long long)w.size_x * w.size_y;
    if (w.size_x <= 0 || w.size_y <= 0 || cells >= U32_LIMIT) return GEM_ERR_INVALID;
    const double res = w.resolution;
    const double wx = w.origin_x + (0 + 0.5) * res, wy = w.origin_y + (0 + 0.5) * res; // mapToWorld(0, 0)
    f.header(h);
    f.u32(0); f.u32(0);          // map_load_time: never set
    const float fres = (float)res;
    f.put(&fres, 4);
    f.u32((uint32_t)w.size_x);
    f.u32((uint32_t)w.size_y);
    f.f64(wx - res / 2); f.f64(wy - res / 2); f.f64(0.0);
    f.f64(0.0); f.f64(0.0); f.f64(0.0); f.f64(1.0);
    f.u32((uint32_t)cells);
    f.payload(cells);
    return GEM_OK;
}

// W10 map_msgs/OccupancyGridUpdate of [x0, x0 + width) x [y0, y0 + height): the data (width height bytes) is the payload
inline int occupancy_grid_update(const gem_ros_header &h, int x0, int y0, int width, int height, Framing &f)
{
    const long long cells = (long long)width * height;
    if (width < 0 || height < 0 || cells >= U32_LIMIT) return GEM_ERR_INVALID;
    f.header(h);
    f.u32((uint32_t)x0);
    f.u32((uint32_t)y0);
    f.u32((uint32_t)width);
    f.u32((uint32_t)height);
    f.u32((uint32_t)cells);
    f.payload(cells);
    return GEM_OK;
}

// W11 geometry_msgs/PolygonStamped: every byte is framing (the transformed points as float32 x, y, z = 0)
inline int polygon_stamped(const gem_ros_header &h, const double *xy, int n, Framing &f)
{
    if (n < 0 || 12ll * n >= U32_LIMIT) return GEM_ERR_INVALID;
    f.header(h);
    f.u32((uint32_t)n);
    for (int i = 0; i < n; i++) {
        const float p[3] = {(float)xy[2 * i], (float)xy[2 * i + 1], 0.0f};
        f.put(p, 12);
    }
    return GEM_OK;
}

// P3 what a publish sends and the rectangle of its data (the whole grid for FULL); the publisher's state is not touched
struct CostmapPlan {
    int kind;                 // GEM_COSTMAP_PUB_*
    int x0, y0, width, height;
};
inline CostmapPlan costmap_plan(const gem_costmap_publisher &p, const gem_costmap_window &w, int force_full)
{
    CostmapPlan d{GEM_COSTMAP_PUB_NONE, 0, 0, 0, 0};
    const float res = (float)w.resolution; // Costmap2DPublisher compares the resolution as a float
    if (force_full || p.always_send_full || !p.saved || p.resolution != res || p.size_x != w.size_x || p.size_y != w.size_y ||
        p.origin_x != w.origin_x || p.origin_y != w.origin_y) {
        d.kind = GEM_COSTMAP_PUB_FULL;
        d.width = w.size_x;
        d.height = w.size_y;
    } else if (p.x0 < p.xn) { // y is not checked: an update of height 0 is sent
        d = CostmapPlan{GEM_COSTMAP_PUB_UPDATE, p.x0, p.y0, p.xn - p.x0, p.yn - p.y0};
    }
    return d;
}
// an UPDATE reads the grid inside the window only
inline bool costmap_plan_ok(const CostmapPlan &d, const gem_costmap_window &w)
{
    return d.kind != GEM_COSTMAP_PUB_UPDATE ||
           (d.x0 >= 0 && d.width > 0 && d.x0 + (long long)d.width <= w.size_x && d.y0 >= 0 && d.height >= 0 &&
            d.y0 + (long long)d.height <= w.size_y);
}
// P4, once the message is written: a FULL one saves the window; the bounds are reset to empty (x0 = size_x, y0 = size_y,
// xn = yn = 0; DEFINED y0 = size_y, which for GEM's square grids is also size_x), except after force_full
// (onNewSubscription publishes without touching them)
inline void costmap_commit(gem_costmap_publisher &p, const gem_costmap_window &w, const CostmapPlan &d, int force_full)
{
    if (d.kind == GEM_COSTMAP_PUB_FULL) {
        p.saved = 1;
        p.resolution = (float)w.resolution;
        p.size_x = w.size_x;
        p.size_y = w.size_y;
        p.origin_x = w.origin_x;
        p.origin_y = w.origin_y;
    }
    if (force_full) return;
    p.x0 = w.size_x;
    p.y0 = w.size_y;
    p.xn = p.yn = 0;
}
// A publish up to its first byte: the plan (P3), its framing (W9 / W10; NONE is an empty message), and whether the call
// writes: a size query (out NULL) or a capacity below the size writes nothing, and then the publisher must stay as it
// was (costmap_commit is not called).  GEM_ERR_INVALID for an UPDATE of bounds outside the grid.
inline int costmap_message(const gem_ros_header &h, const gem_costmap_window &w, const gem_costmap_publisher &p, int force_full,
                           bool size_query, long long capacity, CostmapPlan &d, Framing &f, bool &writes)
{
    writes = false;
    d = costmap_plan(p, w, force_full);
    if (!costmap_plan_ok(d, w)) return GEM_ERR_INVALID;
    int rc = GEM_OK;
    if (d.kind == GEM_COSTMAP_PUB_FULL) rc = occupancy_grid(h, w, f);
    else if (d.kind == GEM_COSTMAP_PUB_UPDATE) rc = occupancy_grid_update(h, d.x0, d.y0, d.width, d.height, f);
    if (rc) return rc;
    writes = !size_query && capacity >= f.size;
    return GEM_OK;
}

// P1, P2
inline void costmap_publisher_init(gem_costmap_publisher &p, int always_send_full)
{
    p = gem_costmap_publisher{};
    p.always_send_full = always_send_full ? 1 : 0;
    p.x0 = p.y0 = 0x7fffffff;
    p.xn = p.yn = 0;
}
inline void costmap_publisher_bounds(gem_costmap_publisher &p, int x0, int xn, int y0, int yn)
{
    p.x0 = x0 < p.x0 ? x0 : p.x0;
    p.xn = xn > p.xn ? xn : p.xn;
    p.y0 = y0 < p.y0 ? y0 : p.y0;
    p.yn = yn > p.yn ? yn : p.yn;
}

} // namespace gem_ros
