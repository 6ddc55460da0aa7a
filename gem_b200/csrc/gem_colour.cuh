// gem_colour.cuh -- the node's colour lookup on the device (GEM_COLOUR_LOOKUP_NODE; DESIGN.md f19).  The loop of
// ElevationMapping::Callback (ElevationMapping.cpp:349-381) takes the points in cloud order against its copy of the
// image: an in-image point reads its pixel, then cv::circle(img, midPoint, 1, colour) paints that colour into the pixels
// (mx +- 1, my) and (mx, my +- 1) that lie inside the image (OpenCV's Circle() at radius 1, thickness 1, LINE_8, shift 0:
// no diagonals; painting the centre would write back the colour just read from it).  OpenCV is an unpinned dependency;
// the loop is restated here, in include/gem_b200.h and in tests/orc_colour_lookup.c.
//
// C1 Projection: project_pixel (gem_kernels.cuh), the arithmetic k_colourise uses.
// C4 Points outside the image: rgba 0,0,0,0 and intensity 0, as k_colourise writes them; they paint nothing.
// C5 Closed form: parent(i) is the largest j < i in the image whose pixel is a 4-neighbour of i's; following parent
//    links from i ends at a root r, and colour_i = image[pixel_r] with alpha 255.  (The working pixel i reads was last
//    painted by parent(i), with the colour parent(i) read, or never.)
//
// The device path: k_colour_keys writes a pixel key per point (the sentinel W * H outside the image); the stable radix
// sort of (key, index) and its runs (key_runs_enqueue) keep every pixel's points in ascending index; k_colour_parent
// finds parent(i) by two binary searches per neighbour pixel, the run and then the last index < i in it; at most
// ceil(log2 n) rounds of k_colour_jump turn the links into roots; k_colour_gather reads each root's pixel.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gem_kernels.cuh"

namespace gem {

// step 1: keys and indices for the sort; C4's outputs for the points outside the image
__global__ void __launch_bounds__(256)
k_colour_keys(float4 *xyzi, int n, const __grid_constant__ ProjParams pp, unsigned long long *key, int *idx, uchar4 *rgba_out)
{
    const unsigned long long outside = (unsigned long long)pp.width * (unsigned long long)pp.height;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)n; i += stride) {
        float4 p = xyzi[i];
        int mx, my;
        unsigned long long k = outside;
        if (project_pixel(p, pp, mx, my)) {
            k = (unsigned long long)my * (unsigned long long)pp.width + (unsigned long long)mx;
        } else {
            p.w = 0.0f;
            xyzi[i] = p;
            rgba_out[i] = make_uchar4(0, 0, 0, 0);
        }
        key[i] = k;
        idx[i] = (int)i;
    }
}

// the largest index < i among the points of pixel `k`, or -1: its run among the nruns distinct keys (ascending), then
// the last index below i in the run (the stable sort keeps a run's indices ascending)
__device__ __forceinline__ int last_before(unsigned long long k, int i, const unsigned long long *ukey, int nruns,
                                           const int *off, const int *cnt, const int *sidx)
{
    int lo = 0, hi = nruns;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ukey[mid] < k) lo = mid + 1;
        else hi = mid;
    }
    if (lo == nruns || ukey[lo] != k) return -1;
    const int first = off[lo];
    int a = first, b = first + cnt[lo];
    while (a < b) {
        const int mid = (a + b) >> 1;
        if (sidx[mid] < i) a = mid + 1;
        else b = mid;
    }
    return a == first ? -1 : sidx[a - 1];
}

// step 3: up[i] = parent(i), or i itself for a root and for a point outside the image
__global__ void __launch_bounds__(256)
k_colour_parent(const unsigned long long *key, int n, int width, int height, const unsigned long long *ukey, const int *nruns,
                const int *off, const int *cnt, const int *sidx, int *up)
{
    const unsigned long long W = (unsigned long long)width, outside = W * (unsigned long long)height;
    const int nr = *nruns;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < (size_t)n; t += stride) {
        const int i = (int)t;
        const unsigned long long k = key[i];
        int best = -1;
        if (k < outside) {
            const unsigned long long my = k / W, mx = k - my * W;
            // only neighbours inside the image can hold a point (row 0 and column 0 are painted, never read)
            if (mx > 1) best = max(best, last_before(k - 1, i, ukey, nr, off, cnt, sidx));
            if (mx + 1 < W) best = max(best, last_before(k + 1, i, ukey, nr, off, cnt, sidx));
            if (my > 1) best = max(best, last_before(k - W, i, ukey, nr, off, cnt, sidx));
            if (my + 1 < (unsigned long long)height) best = max(best, last_before(k + W, i, ukey, nr, off, cnt, sidx));
        }
        up[i] = best >= 0 ? best : i;
    }
}

// step 4: round r of pointer jumping, in place.  A read of another point's link sees its value before or after this
// round's write, an ancestor either way, so a round jumps at least as far as a synchronous one and ceil(log2 n) rounds
// reach every root.  moved[r] = 1 when round r changed a link; a round after one that changed none returns at once.
__global__ void __launch_bounds__(256) k_colour_jump(int *up, int n, int *moved, int r)
{
    if (r > 0 && *(volatile int *)&moved[r - 1] == 0) return;
    int changed = 0;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < (size_t)n; t += stride) {
        const int u = up[t], w = up[u];
        if (w != u) {
            up[t] = w;
            changed = 1;
        }
    }
    if (__syncthreads_or(changed) && threadIdx.x == 0) moved[r] = 1;
}

// step 5: each in-image point's colour from its root's pixel of the unmodified image
__global__ void __launch_bounds__(256)
k_colour_gather(const unsigned long long *key, const int *up, int n, int width, int height, int row_stride,
                const unsigned char *bgr, uchar4 *rgba_out)
{
    const unsigned long long W = (unsigned long long)width, outside = W * (unsigned long long)height;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)n; i += stride) {
        if (key[i] >= outside) continue;
        const unsigned long long k = key[up[i]], my = k / W, mx = k - my * W;
        const unsigned char *px = bgr + my * (unsigned long long)row_stride + 3 * mx;
        rgba_out[i] = make_uchar4(px[2], px[1], px[0], 255);
    }
}

} // namespace gem
