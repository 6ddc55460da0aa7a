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
#pragma once
#include <stdint.h>
#include <string.h>

#include <string>

#include "../../include/gem_b200.h"

#if !defined(__BYTE_ORDER__) || __BYTE_ORDER__ != __ORDER_LITTLE_ENDIAN__
#error "gem_rosfmt.h writes ROS1's little-endian wire format with host stores"
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

} // namespace gem_ros
