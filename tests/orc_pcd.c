/* orc_pcd.c -- oracle of gem_pcd_header / gem_pcd_format (DESIGN.md f13): a literal C restatement of PCL's
 * pcl::PCDWriter::generateHeader<PointT>, writeASCII<PointT> and writeBinary<PointT> for PointXYZRGBICT, writing into
 * memory instead of a file.  PCL is not available to the tests, so this restatement is the definition (unpinned).
 * TEST INFRASTRUCTURE ONLY.
 *
 * getFields<PointXYZRGBICT> lists the fields in registration order (PointXYZRGBICT.hpp:50-58): x 0, y 4, z 8, rgb 16,
 * intensity 24, covariance 20, travers 28, each FLOAT32 count 1.  writeASCII streams each value with precision 8 in the
 * classic locale (libstdc++'s num_put calls vsnprintf("%.*g")), "nan" where pcl_isnan(value), one " " after every value,
 * then boost::trim of the line and "\n".  Newer PCL prints the rgb field as the uint32 of its bits (flag 2).
 * writeBinary copies each field's 4 bytes in the same order, right after the header. */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#define ORC_PCD_BINARY 1
#define ORC_PCD_RGB_UINT32 2

static const char *const NAMES[7] = {"x", "y", "z", "rgb", "intensity", "covariance", "travers"};
static const int OFFS[7] = {0, 4, 8, 16, 24, 20, 28};

/* generateHeader<PointT>(cloud) << "DATA ascii\n" / "DATA binary\n" for a cloud of width n, height 1; returns the length
 * or -1 (PCL throws on an empty cloud); writes only when it fits */
int orc_pcd_header(long long n, int flags, char *out, int cap)
{
    char h[1024];
    int o = 0;
    if (n <= 0 || (flags & ~3)) return -1;
    o += snprintf(h + o, sizeof h - o, "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS");
    for (int f = 0; f < 7; f++) o += snprintf(h + o, sizeof h - o, " %s", NAMES[f]);
    o += snprintf(h + o, sizeof h - o, "\nSIZE");
    for (int f = 0; f < 7; f++) o += snprintf(h + o, sizeof h - o, " %d", 4);
    o += snprintf(h + o, sizeof h - o, "\nTYPE");
    for (int f = 0; f < 7; f++) o += snprintf(h + o, sizeof h - o, " %c", 'F');
    o += snprintf(h + o, sizeof h - o, "\nCOUNT");
    for (int f = 0; f < 7; f++) o += snprintf(h + o, sizeof h - o, " %d", 1);
    o += snprintf(h + o, sizeof h - o, "\nWIDTH %lld\nHEIGHT %d\n", n, 1);
    /* sensor_origin_ (0, 0, 0) and sensor_orientation_ (w 1, x y z 0) of a default-constructed cloud */
    o += snprintf(h + o, sizeof h - o, "VIEWPOINT %d %d %d %d %d %d %d\n", 0, 0, 0, 1, 0, 0, 0);
    o += snprintf(h + o, sizeof h - o, "POINTS %lld\n", n);
    o += snprintf(h + o, sizeof h - o, (flags & ORC_PCD_BINARY) ? "DATA binary\n" : "DATA ascii\n");
    if (out && o <= cap) memcpy(out, h, (size_t)o);
    return o;
}

/* the data section of n records (32 bytes each); returns its bytes or -1 (empty cloud, bad flags); writes only when it
 * fits */
long long orc_pcd_data(const unsigned char *rec, long long n, int flags, char *out, long long cap)
{
    if (n <= 0 || (flags & ~3)) return -1;
    long long o = 0;
    char line[256], v[64];
    for (long long i = 0; i < n; i++) {
        const unsigned char *p = rec + 32 * i;
        if (flags & ORC_PCD_BINARY) {
            for (int d = 0; d < 7; d++) {
                if (out && o + 4 <= cap) memcpy(out + o, p + OFFS[d], 4);
                o += 4;
            }
            continue;
        }
        int l = 0;
        for (int d = 0; d < 7; d++) {
            if (d == 3 && (flags & ORC_PCD_RGB_UINT32)) {
                uint32_t u;
                memcpy(&u, p + OFFS[d], 4);
                snprintf(v, sizeof v, "%u", u);
            } else {
                float value;
                memcpy(&value, p + OFFS[d], 4);
                if (isnan(value)) snprintf(v, sizeof v, "nan");
                else snprintf(v, sizeof v, "%.8g", (double)value);
            }
            l += snprintf(line + l, sizeof line - l, "%s ", v);
        }
        while (l > 0 && line[l - 1] == ' ') l--; /* boost::trim */
        line[l++] = '\n';
        if (out && o + l <= cap) memcpy(out + o, line, (size_t)l);
        o += l;
    }
    return o;
}
