// gem_rosmsg.cuh -- the map's ROS messages written on the device (DESIGN.md f15): the payloads of GEM's visual_map,
// orthomosaic and visualpoints topics at their offsets in a serialised message, and the framing gem_rosfmt.h builds.
// The output may have any alignment (device memory; the library stages pinned outputs in device memory at the same
// 16-byte phase), so every store is either an aligned word that lies wholly inside the bytes one thread owns, or a
// single byte: no byte is written twice and no thread writes a word that holds another thread's bytes.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gem_kernels.cuh"
#include "gem_rosfmt.h"

namespace gem {

struct RosSegs { // gem_ros::Framing's segments, as a kernel parameter
    long long at[gem_ros::MAX_SEGS], src[gem_ros::MAX_SEGS], len[gem_ros::MAX_SEGS];
};

// the framing bytes (staged in device memory) at their offsets: one block per segment, byte by byte (a few hundred bytes)
__global__ void __launch_bounds__(256) k_ros_framing(const unsigned char *bytes, RosSegs s, unsigned char *out)
{
    const int k = blockIdx.x;
    for (long long i = threadIdx.x; i < s.len[k]; i += blockDim.x) out[s.at[k] + i] = bytes[s.src[k] + i];
}

// 16 bytes of the byte string that starts at shared word s (4-byte aligned), from byte offset o < its length - 15:
// funnel shifts of the five words that hold them; the fifth is read only when o is not a multiple of 4, and then it
// holds string bytes, so nothing past the string is read
__device__ __forceinline__ uint4 ros_bytes16(const uint32_t *s, int o)
{
    const uint32_t *p = s + (o >> 2);
    const unsigned sh = 8u * (unsigned)(o & 3);
    const uint32_t x0 = p[0], x1 = p[1], x2 = p[2], x3 = p[3], x4 = sh ? p[4] : 0u;
    return make_uint4(__funnelshift_r(x0, x1, sh), __funnelshift_r(x1, x2, sh), __funnelshift_r(x2, x3, sh), __funnelshift_r(x3, x4, sh));
}

// W2's data: k_export_colmajor's tile (the same gate and values, export_cell) transposed through shared memory, each
// column run of each layer stored at its place in the message.  A run of up to 128 bytes goes out as the aligned
// 16-byte words that lie inside it plus single bytes at its two ends, which share their words with the neighbouring
// run (another block's) or with the framing.  layer0: the first float of layer 0; stride: bytes from one layer's first
// float to the next one's (57 + 4 L^2).
constexpr int ROS_RUN_SLOTS = 10; // per run: the head bytes, up to 8 whole words, the tail bytes
__global__ void __launch_bounds__(256) k_ros_grid_map(MapLayers ml, int L, unsigned char *layer0, long long stride)
{
    __shared__ __align__(16) float tile[9][32][33]; // [layer][column][row]: a column run is contiguous, plus one word
    const int bx = blockIdx.x * 32, by = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int r = ty; r < 32; r += 8) {
        float v[9];
        export_cell(ml, L, bx + r, by + tx, v);
#pragma unroll
        for (int k = 0; k < 9; k++) tile[k][tx][r] = v[k];
    }
    __syncthreads();
    const int rows = min(32, L - bx), cols = min(32, L - by), len = 4 * rows;
    for (int t = threadIdx.x; t < 9 * cols * ROS_RUN_SLOTS; t += blockDim.x) {
        const int run = t / ROS_RUN_SLOTS, slot = t - run * ROS_RUN_SLOTS;
        const int k = run / cols, c = run - k * cols;
        unsigned char *dst = layer0 + k * stride + 4 * ((long long)(by + c) * L + bx);
        const unsigned char *s = reinterpret_cast<const unsigned char *>(&tile[k][c][0]);
        const int head = min(len, (int)((16u - ((uintptr_t)dst & 15u)) & 15u));
        const int words = (len - head) >> 4, tail = head + 16 * words;
        if (slot == 0) {
            for (int b = 0; b < head; b++) dst[b] = s[b];
        } else if (slot == ROS_RUN_SLOTS - 1) {
            for (int b = tail; b < len; b++) dst[b] = s[b];
        } else if (slot - 1 < words) {
            const int o = head + 16 * (slot - 1);
            *reinterpret_cast<uint4 *>(dst + o) = ros_bytes16(reinterpret_cast<const uint32_t *>(s), o);
        }
    }
}

// W3's data: ortho_pixel's image at any alignment.  Thread q owns the aligned 16-byte word q of the output range (about
// five pixels); the first and the last word, which the image may share with the framing, are written byte by byte.
__device__ __forceinline__ uint32_t ortho_pixel_or0(const MapGeom &g, const MapLayers &ml, long long p, long long npx)
{
    return p >= 0 && p < npx ? ortho_pixel(g, ml, (size_t)p) : 0u;
}
__global__ void __launch_bounds__(256) k_ros_orthomosaic(MapGeom g, MapLayers ml, unsigned char *img, long long nwords)
{
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nwords) return;
    const long long npx = (long long)g.L * g.L, nbytes = 3 * npx;
    const long long a = (long long)((uintptr_t)img & 15u);
    const long long b0 = 16 * q - a; // image byte at the word's first byte
    if (b0 >= 0 && b0 + 16 <= nbytes) {
        const long long p0 = b0 / 3;
        const unsigned d = (unsigned)(b0 - 3 * p0);
        uint32_t px[6]; // bytes 3 p0 .. 3 p0 + 17 hold the word's 16 (d <= 2)
#pragma unroll
        for (int i = 0; i < 6; i++) px[i] = ortho_pixel_or0(g, ml, p0 + i, npx);
        // the pixels' bytes from 3 p0 on as 4-byte words, then the 16 from byte d
        const uint32_t w0 = px[0] | (px[1] << 24), w1 = (px[1] >> 8) | (px[2] << 16), w2 = (px[2] >> 16) | (px[3] << 8);
        const uint32_t w3 = px[4] | (px[5] << 24), w4 = px[5] >> 8;
        const unsigned sh = 8u * d;
        *reinterpret_cast<uint4 *>(img + b0) = make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh),
                                                          __funnelshift_r(w2, w3, sh), __funnelshift_r(w3, w4, sh));
    } else {
        for (long long b = b0 < 0 ? 0 : b0; b < b0 + 16 && b < nbytes; b++) {
            const uint32_t p = ortho_pixel_or0(g, ml, b / 3, npx);
            img[b] = (unsigned char)(p >> (8 * (unsigned)(b % 3)));
        }
    }
}

// W9 / W10's data (DESIGN.md f17): T[cost] of the master grid's rectangle [x0, x0 + w) x [y0, ...) in row order, at any
// alignment, as k_ros_orthomosaic writes its image.  Thread q owns the aligned 16-byte word q of the output range and
// reads its 16 cells once (row by row at stride sx); the first and the last word, which the data may share with the
// framing, are written byte by byte.  T is gem_ros::cost_translate, computed in registers.
__device__ __forceinline__ unsigned char ros_cost_byte(const unsigned char *master, int sx, int x0, int y0, int w, long long d)
{
    const long long r = d / w, c = d - r * w;
    return (unsigned char)gem_ros::cost_translate(master[(y0 + r) * sx + x0 + c]);
}
__global__ void __launch_bounds__(256) k_ros_costmap(const unsigned char *master, int sx, int x0, int y0, int w, long long n,
                                                     unsigned char *data, long long nwords)
{
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nwords) return;
    const long long a = (long long)((uintptr_t)data & 15u);
    const long long d0 = 16 * q - a; // data byte at the word's first byte
    if (d0 >= 0 && d0 + 16 <= n) {
        long long r = d0 / w;
        int c = (int)(d0 - r * w);
        const unsigned char *row = master + (y0 + r) * sx + x0;
        uint32_t v[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int k = 0; k < 16; k++) {
            v[k >> 2] |= (uint32_t)(unsigned char)gem_ros::cost_translate(row[c]) << (8 * (k & 3));
            if (++c == w) {
                c = 0;
                row += sx;
            }
        }
        *reinterpret_cast<uint4 *>(data + d0) = make_uint4(v[0], v[1], v[2], v[3]);
    } else {
        for (long long d = d0 < 0 ? 0 : d0; d < d0 + 16 && d < n; d++) data[d] = ros_cost_byte(master, sx, x0, y0, w, d);
    }
}

// ObstacleLayer's footprint clearing: `value` into the layer grid at the n cell indices the host listed (gem_footprint.h)
__global__ void __launch_bounds__(256) k_costmap_cells(const int *cells, int n, unsigned char *grid, unsigned char value)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) grid[cells[i]] = value;
}

// W6's record of one shown cell: {x, y, z, 1.0f, b, g, r, 0xff, 12 zero bytes}, stored at any alignment (aligned
// 4-byte words inside the record, single bytes at its two ends)
__device__ __forceinline__ void ros_store_record(unsigned char *dst, const uint32_t (&w)[8])
{
    const unsigned a = (unsigned)((uintptr_t)dst & 3u);
    if (a == 0) {
        uint4 *d = reinterpret_cast<uint4 *>(dst);
        if (((uintptr_t)dst & 15u) == 0) {
            d[0] = make_uint4(w[0], w[1], w[2], w[3]);
            d[1] = make_uint4(w[4], w[5], w[6], w[7]);
        } else {
            uint32_t *d32 = reinterpret_cast<uint32_t *>(dst);
#pragma unroll
            for (int k = 0; k < 8; k++) d32[k] = w[k];
        }
        return;
    }
    const unsigned lead = 4u - a, sh = 8u * lead;
    for (unsigned b = 0; b < lead; b++) dst[b] = (unsigned char)(w[0] >> (8u * b));
    uint32_t *d32 = reinterpret_cast<uint32_t *>(dst + lead);
#pragma unroll
    for (int k = 0; k < 7; k++) d32[k] = __funnelshift_r(w[k], w[k + 1], sh);
    for (unsigned b = 0; b < a; b++) dst[28 + lead + b] = (unsigned char)(w[7] >> (sh + 8u * b));
}

// the visual cloud of ElevationMap::show as W6 records, in the order of gem_export_visual_points (VisualSrc)
struct RosVisualSrc {
    MapLayers ml;
    GridMapFrame f;
    unsigned char *out;
    __device__ __forceinline__ bool take(int ix, int iy) const
    {
        float e;
        return show_valid(ml, (size_t)ix * f.L + iy, e);
    }
    __device__ __forceinline__ void emit(int ix, int iy, int pos) const
    {
        const size_t c = (size_t)ix * f.L + iy;
        const uint32_t col = ml.cell[c].rgb;
        const uint32_t r = col & 255u, g = (col >> 8) & 255u, b = (col >> 16) & 255u;
        const uint32_t w[8] = {__float_as_uint((float)f.px(ix)), __float_as_uint((float)f.py(iy)), __float_as_uint(ml.cell[c].elev),
                               __float_as_uint(1.0f), b | (g << 8) | (r << 16) | 0xff000000u, 0u, 0u, 0u};
        ros_store_record(out + 32 * (size_t)pos, w);
    }
};

} // namespace gem
