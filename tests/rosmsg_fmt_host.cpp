// rosmsg_fmt_host.cpp -- the host build of the library's ROS message framing (gem_b200/csrc/gem_rosfmt.h): renders a
// whole message from its framing and a payload (the payload runs back to back), for tests/test_rosmsg_cpu.py.
// TEST INFRASTRUCTURE ONLY: compiled by tests/rosmsg_oracle.py into a temporary directory.
#include <string.h>

#include "gem_rosfmt.h"

// the framing's segments and the payload runs in message order into out; returns the size, -1 when the framing
// refuses, -2 when the message is larger than capacity, -3 when the segments and runs do not tile the message
static long long render(int rc, const gem_ros::Framing &f, const unsigned char *payload, unsigned char *out, long long capacity)
{
    if (rc) return -1;
    if (f.size > capacity) return -2;
    long long at = 0, p = 0;
    int s = 0, k = 0;
    while (at < f.size) {
        if (s < f.nseg && f.seg[s].at == at) {
            memcpy(out + at, f.bytes.data() + f.seg[s].src, (size_t)f.seg[s].len);
            at += f.seg[s++].len;
        } else if (k < f.npayload && f.payload_at[k] == at) {
            memcpy(out + at, payload + p, (size_t)f.payload_len[k]);
            p += f.payload_len[k];
            at += f.payload_len[k++];
        } else {
            return -3;
        }
    }
    return at == f.size && s == f.nseg ? f.size : -3;
}

static gem_ros_header hdr(unsigned seq, unsigned sec, unsigned nsec, const char *frame_id)
{
    gem_ros_header h;
    h.seq = seq; h.stamp_sec = sec; h.stamp_nsec = nsec; h.frame_id = frame_id;
    return h;
}

extern "C" {

long long ros_fmt_grid_map(unsigned seq, unsigned sec, unsigned nsec, const char *fid, int L, double res, double cx, double cy,
                           int sx, int sy, const unsigned char *payload, unsigned char *out, long long capacity)
{
    gem_ros::Framing f;
    const int rc = gem_ros::grid_map(hdr(seq, sec, nsec, fid), L, res, cx, cy, sx, sy, f);
    return render(rc, f, payload, out, capacity);
}

long long ros_fmt_image(unsigned seq, unsigned sec, unsigned nsec, const char *fid, int L, const unsigned char *payload,
                        unsigned char *out, long long capacity)
{
    gem_ros::Framing f;
    const int rc = gem_ros::image(hdr(seq, sec, nsec, fid), L, f);
    return render(rc, f, payload, out, capacity);
}

long long ros_fmt_cloud(unsigned seq, unsigned sec, unsigned nsec, const char *fid, int xyzrgb, long long n, int is_dense,
                        const unsigned char *payload, unsigned char *out, long long capacity)
{
    gem_ros::Framing f;
    const int rc = gem_ros::cloud(hdr(seq, sec, nsec, fid), xyzrgb ? gem_ros::CLOUD_XYZRGB : gem_ros::CLOUD_XYZRGBICT, n,
                                  is_dense, f);
    return render(rc, f, payload, out, capacity);
}

long long ros_fmt_octomap(unsigned seq, unsigned sec, unsigned nsec, const char *fid, double res, long long bytes,
                          const unsigned char *payload, unsigned char *out, long long capacity)
{
    gem_ros::Framing f;
    const int rc = gem_ros::octomap(hdr(seq, sec, nsec, fid), res, bytes, f);
    return render(rc, f, payload, out, capacity);
}

} // extern "C"
