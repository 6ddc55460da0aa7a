/* orc_colour_lookup.c -- oracle of GEM_COLOUR_LOOKUP_NODE (DESIGN.md f19): the colour lookup loop of
 * ElevationMapping::Callback (ElevationMapping.cpp:349-381) written out literally, with cv::circle(img, midPoint, 1,
 * colour) as OpenCV's Circle() runs it at radius 1, thickness 1, LINE_8 and shift 0 (its inside and clipped branches,
 * not a closed form).  OpenCV is not available here: restated, unpinned.  TEST INFRASTRUCTURE ONLY.
 *
 * orc_colourise_node(xyzi, n, Tc, Tl, bgr, width, height, row_stride, rgba_out): like the oracle's orc_colourise, but the
 * points are taken in order against a working copy of the BGR8 image that each in-image point paints.  The caller's
 * image is not written.  Returns 0, or -1 when the working copy cannot be allocated. */
#include <stdlib.h>
#include <string.h>

/* cv::Point's int from a float: truncation toward zero, saturating, NaN to 0 (the library's __float2int_rz and the oracle's
 * f2i_rz; every value this changes lies outside the image either way) */
static int f2i_rz(float f)
{
    if (f != f) return 0;
    if (f >= 2147483648.0f) return 0x7fffffff;
    if (f <= -2147483648.0f) return (int)0x80000000u;
    return (int)f;
}

/* OpenCV's Circle(img, center, radius, color, fill = 0) for an 8UC3 image, drawing.cpp: the midpoint loop with its
 * `inside` fast branch and its clipped branch */
static void circle8(unsigned char *ptr, int width, int height, size_t step, int cx, int cy, int radius, const unsigned char color[3])
{
    const int pix_size = 3;
    int err = 0, dx = radius, dy = 0, plus = 1, minus = (radius << 1) - 1;
    const int inside = cx >= radius && cx < width - radius && cy >= radius && cy < height - radius;
#define PUT(row, x) memcpy((row) + (size_t)(x) * pix_size, color, pix_size)
    while (dx >= dy) {
        int mask;
        const int y11 = cy - dy, y12 = cy + dy, y21 = cy - dx, y22 = cy + dx;
        const int x11 = cx - dx, x12 = cx + dx, x21 = cx - dy, x22 = cx + dy;
        if (inside) {
            unsigned char *t0 = ptr + (size_t)y11 * step, *t1 = ptr + (size_t)y12 * step;
            PUT(t0, x11); PUT(t1, x11); PUT(t0, x12); PUT(t1, x12);
            t0 = ptr + (size_t)y21 * step;
            t1 = ptr + (size_t)y22 * step;
            PUT(t0, x21); PUT(t1, x21); PUT(t0, x22); PUT(t1, x22);
        } else if (x11 < width && x12 >= 0 && y21 < height && y22 >= 0) {
            if ((unsigned)y11 < (unsigned)height) {
                unsigned char *t = ptr + (size_t)y11 * step;
                if (x11 >= 0) PUT(t, x11);
                if (x12 < width) PUT(t, x12);
            }
            if ((unsigned)y12 < (unsigned)height) {
                unsigned char *t = ptr + (size_t)y12 * step;
                if (x11 >= 0) PUT(t, x11);
                if (x12 < width) PUT(t, x12);
            }
            if (x21 < width && x22 >= 0) {
                if ((unsigned)y21 < (unsigned)height) {
                    unsigned char *t = ptr + (size_t)y21 * step;
                    if (x21 >= 0) PUT(t, x21);
                    if (x22 < width) PUT(t, x22);
                }
                if ((unsigned)y22 < (unsigned)height) {
                    unsigned char *t = ptr + (size_t)y22 * step;
                    if (x21 >= 0) PUT(t, x21);
                    if (x22 < width) PUT(t, x22);
                }
            }
        }
        dy++;
        err += plus;
        plus += 2;
        mask = (err <= 0) - 1;
        err -= minus & mask;
        dx += mask;
        minus -= mask & 2;
    }
#undef PUT
}

int orc_colourise_node(float *xyzi, int n, const double Tc[12], const double Tl[16], const unsigned char *bgr, int width,
                       int height, int row_stride, unsigned char *rgba_out)
{
    double P[12];
    int i, j, k;
    const size_t bytes = (size_t)(height - 1) * (size_t)row_stride + 3 * (size_t)width;
    unsigned char *img = (unsigned char *)malloc(bytes); /* toCvCopy: the frame's own copy (:316) */
    if (!img) return -1;
    memcpy(img, bgr, bytes);
    for (i = 0; i < 3; i++) /* :347 P_lidar2img = Tcamera * TLidar */
        for (j = 0; j < 4; j++) {
            double a = Tc[4 * i + 0] * Tl[0 + j];
            for (k = 1; k < 4; k++) a = a + Tc[4 * i + k] * Tl[4 * k + j];
            P[4 * i + j] = a;
        }
    for (i = 0; i < n; i++) {
        const double x = (double)xyzi[4 * i], y = (double)xyzi[4 * i + 1], z = (double)xyzi[4 * i + 2];
        const double X = ((P[0] * x + P[1] * y) + P[2] * z) + P[3] * 1.0; /* :351-355 */
        const double Y = ((P[4] * x + P[5] * y) + P[6] * z) + P[7] * 1.0;
        const double Z = ((P[8] * x + P[9] * y) + P[10] * z) + P[11] * 1.0;
        const float Px = (float)(X / Z), Py = (float)(Y / Z); /* :359-360 */
        const int mx = f2i_rz(Px), my = f2i_rz(Py);           /* :362-365 */
        unsigned char *o = rgba_out + 4 * (size_t)i;
        if (mx > 0 && mx < width && my > 0 && my < height && Z > 0) { /* :368 */
            const unsigned char *px = img + (size_t)my * row_stride + 3 * (size_t)mx;
            const unsigned char colour[3] = {px[0], px[1], px[2]}; /* b, g, r (:369-371) */
            circle8(img, width, height, (size_t)row_stride, mx, my, 1, colour); /* :370 */
            o[0] = colour[2]; o[1] = colour[1]; o[2] = colour[0]; o[3] = 255;
        } else { /* :376-381 */
            o[0] = o[1] = o[2] = o[3] = 0;
            xyzi[4 * i + 3] = 0;
        }
    }
    free(img);
    return 0;
}
