// costmap_pub_host.cpp -- the host build of the library's costmap topics and footprint clearing (gem_b200/csrc/
// gem_rosfmt.h W9-W11 and P1-P4, gem_b200/csrc/gem_footprint.h F1-F4), for tests/test_costmap_pub_cpu.py.  The data of
// W9 / W10 is T of a host master grid, here instead of on the device.
// TEST INFRASTRUCTURE ONLY: compiled by tests/costmap_pub_oracle.py into a temporary directory.
#include <string.h>

#include <vector>

#include "gem_footprint.h"
#include "gem_rosfmt.h"

static gem_ros_header hdr(unsigned seq, unsigned sec, unsigned nsec, const char *frame_id)
{
    gem_ros_header h;
    h.seq = seq; h.stamp_sec = sec; h.stamp_nsec = nsec; h.frame_id = frame_id;
    return h;
}

// the framing's segments and its one payload run (or none) in message order; -3 when they do not tile the message
static long long render(const gem_ros::Framing &f, const unsigned char *payload, unsigned char *out)
{
    long long at = 0;
    int s = 0, k = 0;
    while (at < f.size) {
        if (s < f.nseg && f.seg[s].at == at) {
            memcpy(out + at, f.bytes.data() + f.seg[s].src, (size_t)f.seg[s].len);
            at += f.seg[s++].len;
        } else if (k < f.npayload && f.payload_at[k] == at) {
            memcpy(out + at, payload, (size_t)f.payload_len[k]);
            at += f.payload_len[k++];
        } else {
            return -3;
        }
    }
    return at == f.size && s == f.nseg ? f.size : -3;
}

extern "C" {

int cp_translate(unsigned c) { return gem_ros::cost_translate(c); }

void cp_publisher_init(gem_costmap_publisher *p, int always_send_full) { gem_ros::costmap_publisher_init(*p, always_send_full); }
void cp_publisher_bounds(gem_costmap_publisher *p, int x0, int xn, int y0, int yn) { gem_ros::costmap_publisher_bounds(*p, x0, xn, y0, yn); }

// one publish as gem_ros_costmap makes it, the data translated on the host from `master` (size_y rows of size_x):
// returns the message size (written to out and committed when it fits and out is not NULL), -1 when refused.  *kind and
// rect[4] = (x0, y0, width, height) receive the plan.
long long cp_publish(unsigned seq, unsigned sec, unsigned nsec, const char *fid, const gem_costmap_window *w, const unsigned char *master,
                     gem_costmap_publisher *p, int force_full, unsigned char *out, long long capacity, int *kind, int *rect)
{
    gem_ros::CostmapPlan d;
    gem_ros::Framing f;
    bool writes = false;
    if (gem_ros::costmap_message(hdr(seq, sec, nsec, fid), *w, *p, force_full, !out, capacity, d, f, writes)) return -1;
    *kind = d.kind;
    rect[0] = d.x0; rect[1] = d.y0; rect[2] = d.width; rect[3] = d.height;
    if (!writes) return f.size;
    std::vector<unsigned char> data((size_t)d.width * d.height);
    for (int y = 0; y < d.height; y++)
        for (int x = 0; x < d.width; x++)
            data[(size_t)y * d.width + x] = (unsigned char)gem_ros::cost_translate(master[(size_t)(d.y0 + y) * w->size_x + d.x0 + x]);
    if (render(f, data.data(), out) != f.size) return -3;
    gem_ros::costmap_commit(*p, *w, d, force_full);
    return f.size;
}

long long cp_footprint_msg(unsigned seq, unsigned sec, unsigned nsec, const char *fid, const double *spec_xy, int n, double rx, double ry,
                           double yaw, unsigned char *out, long long capacity)
{
    std::vector<gem_fp::Point> pts;
    gem_fp::transform(spec_xy, n, rx, ry, yaw, pts);
    std::vector<double> xy;
    for (const gem_fp::Point &q : pts) {
        xy.push_back(q.x);
        xy.push_back(q.y);
    }
    gem_ros::Framing f;
    if (gem_ros::polygon_stamped(hdr(seq, sec, nsec, fid), xy.data(), n, f)) return -1;
    if (f.size > capacity) return -2;
    return render(f, nullptr, out);
}

// the transformed vertices (double) and the cells setConvexPolygonCost writes, as (x, y) pairs; returns the cell count,
// -1 when a vertex lies outside the window, -2 when capacity is too small
long long cp_footprint_cells(const gem_costmap_window *w, const double *spec_xy, int n, double rx, double ry, double yaw, double *verts_xy,
                             unsigned *cells_xy, long long capacity)
{
    std::vector<gem_fp::Point> pts;
    std::vector<gem_fp::Cell> cells;
    gem_fp::transform(spec_xy, n, rx, ry, yaw, pts);
    for (int i = 0; i < n; i++) {
        verts_xy[2 * i] = pts[i].x;
        verts_xy[2 * i + 1] = pts[i].y;
    }
    if (!gem_fp::polygon_cells(w->origin_x, w->origin_y, w->resolution, w->size_x, w->size_y, pts, cells)) return -1;
    if ((long long)cells.size() > capacity) return -2;
    for (size_t i = 0; i < cells.size(); i++) {
        cells_xy[2 * i] = cells[i].x;
        cells_xy[2 * i + 1] = cells[i].y;
    }
    return (long long)cells.size();
}

// F4's column walk alone on a crafted list of n (x, y) cells; returns the result's length (-2: capacity)
long long cp_column_walk(const unsigned *cells_xy, long long n, unsigned *out_xy, long long capacity)
{
    std::vector<gem_fp::Cell> cells;
    for (long long i = 0; i < n; i++) cells.push_back(gem_fp::Cell{cells_xy[2 * i], cells_xy[2 * i + 1]});
    gem_fp::column_walk(cells);
    if ((long long)cells.size() > capacity) return -2;
    for (size_t i = 0; i < cells.size(); i++) {
        out_xy[2 * i] = cells[i].x;
        out_xy[2 * i + 1] = cells[i].y;
    }
    return (long long)cells.size();
}

} // extern "C"
