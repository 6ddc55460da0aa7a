// gem_pcd.cuh -- the map's point clouds as PCD files (DESIGN.md f13): the data section pcl::io::savePCDFile writes for a
// pcl::PointCloud<PointXYZRGBICT> (savingMap, savingSubMap and pointcloudinterpolation, ElevationMapping.cpp:430-476,
// :1117), from 32-byte records in device memory.  PCL's PCDWriter::generateHeader / writeASCII / writeBinary are an
// unpinned dependency; their definitions are restated here, in include/gem_b200.h and in tests/orc_pcd.c.
//
// P1 Fields in registration order (PointXYZRGBICT.hpp:50-58): x, y, z, rgb, intensity, covariance, travers = record
//    words 0, 1, 2, 4, 6, 5, 7; word 3 (w) is never written.
// P2 ASCII: each value as gem_pcdfmt.h prints it (glibc's %.8g; "nan" for every NaN), rgb optionally as the uint32 of
//    its bits (GEM_PCD_RGB_UINT32, newer PCL); one space between values, '\n' after the last.
// P3 Binary: the seven words of P1 per record, 28 bytes, as they are in memory.
//
// ASCII takes two kernels around a scan.  k_pcd_len formats a tile of PCD_BLOCK records (one per thread) and stores the
// tile's byte count; an inclusive CUB scan turns the counts into tile ends; k_pcd_ascii formats the tile again, places
// each line in shared memory at its block-scanned offset, and the block stores the tile's bytes to its place in the
// output with aligned 16-byte stores.  Formatting twice costs arithmetic; staging fixed 105-byte slots instead would cost
// 105 bytes of device scratch per record against 8 bytes per tile here.  k_pcd_binary stages 28-byte records in shared
// memory the same way.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <cub/cub.cuh>

#include "../../include/gem_b200.h"
#include "gem_pcdfmt.h"

namespace gem {

constexpr int PCD_BLOCK = 256;                         // records per tile, one per thread
constexpr int PCD_FIELDS = 7;
constexpr int PCD_BINARY_RECORD = 28;
constexpr int PCD_SMEM = PCD_BLOCK * GEM_PCD_LINE_MAX + 16; // a tile's longest output, plus the word the store reads past it
static_assert(GEM_PCD_LINE_MAX == PCD_FIELDS * GEM_PCD_VALUE_MAX + PCD_FIELDS, "seven values, six spaces and a newline");

// the header of generateHeader<PointXYZRGBICT> for a cloud of width n, height 1, and its DATA line; returns its length
inline int pcd_header(long long n, int flags, char (&h)[GEM_PCD_HEADER_MAX])
{
    return snprintf(h, sizeof h,
                    "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z rgb intensity covariance travers\n"
                    "SIZE 4 4 4 4 4 4 4\nTYPE F F F F F F F\nCOUNT 1 1 1 1 1 1 1\nWIDTH %lld\nHEIGHT 1\n"
                    "VIEWPOINT 0 0 0 1 0 0 0\nPOINTS %lld\nDATA %s\n",
                    n, n, (flags & GEM_PCD_BINARY) ? "binary" : "ascii");
}

// P1: the seven values of record i (two 16-byte loads)
__device__ __forceinline__ void pcd_values(const float4 *rec, long long i, bool rgb_uint32, gem_pcd_val (&v)[PCD_FIELDS])
{
    const float4 a = rec[2 * i], b = rec[2 * i + 1];
    v[0] = gem_pcd_float(__float_as_uint(a.x));
    v[1] = gem_pcd_float(__float_as_uint(a.y));
    v[2] = gem_pcd_float(__float_as_uint(a.z));
    v[3] = rgb_uint32 ? gem_pcd_uint(__float_as_uint(b.x)) : gem_pcd_float(__float_as_uint(b.x));
    v[4] = gem_pcd_float(__float_as_uint(b.z));
    v[5] = gem_pcd_float(__float_as_uint(b.y));
    v[6] = gem_pcd_float(__float_as_uint(b.w));
}

__device__ __forceinline__ int pcd_line_len(const gem_pcd_val (&v)[PCD_FIELDS])
{
    int len = PCD_FIELDS; // six spaces and the newline
#pragma unroll
    for (int f = 0; f < PCD_FIELDS; f++) len += gem_pcd_len(v[f]);
    return len;
}

// the block stores s[0, len) (shared memory, 16-byte aligned, readable to len + 16) at dst, any alignment: bytewise up to
// the first 16-byte boundary of dst and after the last, aligned 16-byte stores in between (funnel shifts of the shared words)
__device__ __forceinline__ void pcd_store(const unsigned char *s, int len, unsigned char *dst)
{
    const int head = min(len, (int)((16u - ((uintptr_t)dst & 15u)) & 15u));
    const int words = (len - head) >> 4, tail = head + 16 * words;
    const uint32_t *s32 = reinterpret_cast<const uint32_t *>(s) + (head >> 2);
    const unsigned sh = 8u * (unsigned)(head & 3);
    uint4 *d16 = reinterpret_cast<uint4 *>(dst + head);
    for (int b = threadIdx.x; b < head; b += blockDim.x) dst[b] = s[b];
    for (int w = threadIdx.x; w < words; w += blockDim.x) {
        const uint32_t *p = s32 + 4 * w;
        const uint32_t x0 = p[0], x1 = p[1], x2 = p[2], x3 = p[3], x4 = p[4];
        d16[w] = make_uint4(__funnelshift_r(x0, x1, sh), __funnelshift_r(x1, x2, sh), __funnelshift_r(x2, x3, sh),
                            __funnelshift_r(x3, x4, sh));
    }
    for (int b = tail + threadIdx.x; b < len; b += blockDim.x) dst[b] = s[b];
}

// pass 1: the byte count of each tile's lines
__global__ void __launch_bounds__(PCD_BLOCK) k_pcd_len(const float4 *rec, int n, int rgb_uint32, long long *tile_bytes)
{
    using Reduce = cub::BlockReduce<int, PCD_BLOCK>;
    __shared__ typename Reduce::TempStorage tmp;
    const long long i = (long long)blockIdx.x * PCD_BLOCK + threadIdx.x;
    int len = 0;
    if (i < n) {
        gem_pcd_val v[PCD_FIELDS];
        pcd_values(rec, i, rgb_uint32 != 0, v);
        len = pcd_line_len(v);
    }
    const int sum = Reduce(tmp).Sum(len);
    if (threadIdx.x == 0) tile_bytes[blockIdx.x] = sum;
}

// pass 2: each tile's lines at tile_end[b - 1] (0 for the first tile)
__global__ void __launch_bounds__(PCD_BLOCK) k_pcd_ascii(const float4 *rec, int n, int rgb_uint32, const long long *tile_end,
                                                         unsigned char *out)
{
    using Scan = cub::BlockScan<int, PCD_BLOCK>;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ __align__(16) unsigned char s_out[PCD_SMEM];
    const long long i = (long long)blockIdx.x * PCD_BLOCK + threadIdx.x;
    gem_pcd_val v[PCD_FIELDS];
    int len = 0;
    if (i < n) {
        pcd_values(rec, i, rgb_uint32 != 0, v);
        len = pcd_line_len(v);
    }
    int off, total;
    Scan(tmp).ExclusiveSum(len, off, total);
    if (i < n) {
        char *p = reinterpret_cast<char *>(s_out) + off;
#pragma unroll
        for (int f = 0; f < PCD_FIELDS; f++) {
            p += gem_pcd_put(v[f], p);
            *p++ = f == PCD_FIELDS - 1 ? '\n' : ' ';
        }
    }
    __syncthreads();
    pcd_store(s_out, total, out + (blockIdx.x ? tile_end[blockIdx.x - 1] : 0ll));
}

// P3: 28 bytes per record, a tile at a time
__global__ void __launch_bounds__(PCD_BLOCK) k_pcd_binary(const float4 *rec, int n, unsigned char *out)
{
    __shared__ __align__(16) uint32_t s_out[(PCD_BLOCK * PCD_BINARY_RECORD + 16) / 4];
    const long long t0 = (long long)blockIdx.x * PCD_BLOCK, i = t0 + threadIdx.x;
    if (i < n) {
        const float4 a = rec[2 * i], b = rec[2 * i + 1];
        uint32_t *p = s_out + PCD_FIELDS * threadIdx.x;
        p[0] = __float_as_uint(a.x); p[1] = __float_as_uint(a.y); p[2] = __float_as_uint(a.z); p[3] = __float_as_uint(b.x);
        p[4] = __float_as_uint(b.z); p[5] = __float_as_uint(b.y); p[6] = __float_as_uint(b.w);
    }
    __syncthreads();
    const int cnt = (int)min((long long)PCD_BLOCK, (long long)n - t0);
    pcd_store(reinterpret_cast<const unsigned char *>(s_out), cnt * PCD_BINARY_RECORD, out + t0 * PCD_BINARY_RECORD);
}

} // namespace gem
