// gem_ingest.cuh -- raw sensor messages on the device (DESIGN.md f12): the sensor_msgs/PointCloud2 -> PointXYZRGBICT
// conversion the node does with pcl::fromPCLPointCloud2 (ElevationMapping.cpp:311-316) and cv_bridge's 8-bit image
// conversions to BGR8 (:317).  PCL 1.8's createMapping<PointXYZRGBICT> / fromPCLPointCloud2 are an unpinned dependency;
// their definitions are restated here, in include/gem_b200.h and in tests/orc_pointcloud2.c.
//
// M1 Match: struct fields in registration order (PointXYZRGBICT.hpp:50-58) x 0, y 4, z 8, rgb 16, intensity 24,
//    covariance 20, travers 28; each takes the first message field with an equal name, datatype FLOAT32 and count 1 or 0.
// M2 Coalesce: sorted by message offset, merged into the predecessor when the message and struct offset differences are
//    equal (the predecessor grows to the end of the later one, gap bytes included).
// M3 Copy: one span at 0 / 0 with point_step == 32 copies whole points; otherwise each span per point, in span order.
// DEFINED: struct bytes nothing writes are 0; layouts on which PCL reads out of bounds are refused (pc2_map).
//
// k_decode_pc2 only moves bytes: no float operation touches a value, so NaN payloads and -0 survive.  A block stages
// the message bytes of up to `tile` consecutive points of one row in shared memory with aligned 16-byte loads (the
// partial words at the two ends of the buffer bytewise), derives from the spans which message byte feeds each of the 16
// output bytes, and each thread then assembles its float4 from shared memory and stores it (coalesced).  Points wider
// than the shared-memory budget are gathered straight from global memory.  A second instantiation (REC 32, DESIGN.md
// f18) derives all 32 record bytes the same way and stores each point as two aligned 16-byte words.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../include/gem_b200.h"

namespace gem {

constexpr int PC2_BLOCK = 256;            // threads per block, and points per tile at most
constexpr unsigned PC2_SMEM = 32768;      // staged message bytes per block at most
constexpr unsigned PC2_RECORD = 32;       // sizeof(PointXYZRGBICT)

struct Pc2Params {
    const unsigned char *data;            // message bytes (any alignment)
    unsigned long long data_bytes;        // readable bytes from data
    unsigned long long row_step;          // bytes between rows (rows = 1 when the rows are contiguous)
    unsigned point_step;
    unsigned width;                       // points per row
    unsigned tiles_per_row;
    unsigned tile;                        // points per tile
    int staged;                           // 1: stage through shared memory (tile * point_step <= PC2_SMEM)
    int nspans;
    gem_pc2_span spans[GEM_PC2_FIELDS];   // M3's effective spans (the fast path as one 32-byte span)
    unsigned long long tiles;             // rows * tiles_per_row
};

// ---- M1-M3 on the host ----------------------------------------------------------------------------------------------
// returns nullptr and fills *out, or the reason the layout is refused
inline const char *pc2_map(const gem_pointcloud2 *L, unsigned long long data_bytes, gem_pc2_mapping *out)
{
    static const char *const names[GEM_PC2_FIELDS] = {"x", "y", "z", "rgb", "intensity", "covariance", "travers"};
    static const unsigned offs[GEM_PC2_FIELDS] = {0, 4, 8, 16, 24, 20, 28};
    if (!L || !out || L->nfields < 0 || (L->nfields > 0 && !L->fields)) return "bad argument";
    gem_pc2_mapping r;
    memset(&r, 0, sizeof r);
    for (int f = 0; f < L->nfields; f++)
        if (L->fields[f].datatype < GEM_PF_INT8 || L->fields[f].datatype > GEM_PF_FLOAT64) return "a field has a datatype outside 1..8";
    const unsigned long long n = (unsigned long long)L->width * L->height;
    if (n > 2147483647ull) return "width * height exceeds INT_MAX";
    // M1: FieldMapper in registration order, first matching message field
    gem_pc2_span m[GEM_PC2_FIELDS];
    int nm = 0;
    for (int k = 0; k < GEM_PC2_FIELDS; k++)
        for (int f = 0; f < L->nfields; f++) {
            const gem_pointfield &pf = L->fields[f];
            if (!memchr(pf.name, 0, sizeof pf.name) || strcmp(pf.name, names[k]) != 0) continue;
            if (pf.datatype != GEM_PF_FLOAT32 || (pf.count != 1 && pf.count != 0)) continue;
            m[nm++] = gem_pc2_span{pf.offset, offs[k], 4};
            r.matched |= 1u << k;
            break;
        }
    // M2: sort by message offset (insertion sort; equal offsets overlap and are refused below), then coalesce
    for (int i = 1; i < nm; i++)
        for (int j = i; j > 0 && m[j - 1].serialized_offset > m[j].serialized_offset; j--) { gem_pc2_span t = m[j]; m[j] = m[j - 1]; m[j - 1] = t; }
    if (n > 0) {
        for (int i = 0; i < nm; i++)
            if ((unsigned long long)m[i].serialized_offset + m[i].size > L->point_step) return "a matched field runs past point_step";
        for (int i = 1; i < nm; i++)
            if ((unsigned long long)m[i - 1].serialized_offset + m[i - 1].size > m[i].serialized_offset) return "two matched fields overlap";
        if ((unsigned long long)L->row_step < (unsigned long long)L->width * L->point_step) return "row_step < width * point_step";
        r.bytes = (unsigned long long)(L->height - 1) * L->row_step + (unsigned long long)L->width * L->point_step;
        if (data_bytes < r.bytes) return "data is shorter than (height - 1) * row_step + width * point_step";
    }
    int ns = 0;
    for (int j = 0; j < nm; j++) {
        if (ns > 0 && m[j].serialized_offset - r.spans[ns - 1].serialized_offset == m[j].struct_offset - r.spans[ns - 1].struct_offset) {
            gem_pc2_span &i = r.spans[ns - 1];
            i.size += (m[j].struct_offset + m[j].size) - (i.struct_offset + i.size);
        } else {
            r.spans[ns++] = m[j];
        }
    }
    r.nspans = ns;
    r.fast_path = ns == 1 && r.spans[0].serialized_offset == 0 && r.spans[0].struct_offset == 0 && L->point_step == PC2_RECORD;
    r.points = (long long)n;
    *out = r;
    return nullptr;
}

// kernel parameters for a validated layout: rows without padding are decoded as one row
inline Pc2Params pc2_params(const gem_pointcloud2 *L, const gem_pc2_mapping &mp, const void *data, unsigned long long data_bytes)
{
    Pc2Params p;
    memset(&p, 0, sizeof p);
    p.data = (const unsigned char *)data;
    p.data_bytes = data_bytes;
    p.point_step = L->point_step;
    const bool packed = L->height == 1 || (unsigned long long)L->row_step == (unsigned long long)L->width * L->point_step;
    const unsigned long long rows = packed ? (mp.points ? 1 : 0) : L->height;
    p.width = packed ? (unsigned)mp.points : L->width;
    p.row_step = packed ? 0 : L->row_step;
    p.staged = L->point_step > 0 && L->point_step <= PC2_SMEM;
    unsigned t = p.staged ? PC2_SMEM / L->point_step : PC2_BLOCK;
    p.tile = t < (unsigned)PC2_BLOCK ? t : PC2_BLOCK;
    p.tiles_per_row = p.width ? (p.width + p.tile - 1) / p.tile : 0;
    p.tiles = rows * p.tiles_per_row;
    if (mp.fast_path) {
        p.nspans = 1;
        p.spans[0] = gem_pc2_span{0, 0, PC2_RECORD};
    } else {
        p.nspans = mp.nspans;
        for (int k = 0; k < mp.nspans; k++) p.spans[k] = mp.spans[k];
    }
    return p;
}

// dynamic shared memory of k_decode_pc2: the tile's bytes plus the two partial words of the aligned window
inline size_t pc2_smem_bytes(const Pc2Params &p) { return p.staged ? ((size_t)p.tile * p.point_step + 47) / 16 * 16 : 0; }

// the 16-byte word of the message at address a; a word that is not wholly inside
// [data, data + data_bytes) are read bytewise, the bytes outside as 0
__device__ __forceinline__ uint4 pc2_load_word(uintptr_t a, uintptr_t lo, uintptr_t hi)
{
    if (a >= lo && a + 16 <= hi) return __ldg((const uint4 *)a);
    uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int b = 0; b < 16; b++)
        if (a + b >= lo && a + b < hi) w[b >> 2] |= (uint32_t)__ldg((const unsigned char *)(a + b)) << (8 * (b & 3));
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// the output float4 of one point as four words of its bytes: byte b from pt[src[b]], 0 where src[b] < 0
__device__ __forceinline__ uint4 pc2_assemble(const unsigned char *pt, const int (&src)[16])
{
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        uint32_t v = 0u;
#pragma unroll
        for (int b = 0; b < 4; b++)
            if (src[4 * k + b] >= 0) v |= (uint32_t)pt[src[4 * k + b]] << (8 * b);
        w[k] = v;
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// one decoded point at out[i]: REC 16, the float4 {x, y, z, intensity} (struct bytes 0-11, 24-27); REC 32, the whole
// record as two aligned 16-byte stores
template <int REC> __device__ __forceinline__ void pc2_store(uint4 *out, unsigned long long i, const unsigned char *pt, const int (&src)[REC]);
template <> __device__ __forceinline__ void pc2_store<16>(uint4 *out, unsigned long long i, const unsigned char *pt, const int (&src)[16])
{
    out[i] = pc2_assemble(pt, src);
}
template <> __device__ __forceinline__ void pc2_store<32>(uint4 *out, unsigned long long i, const unsigned char *pt, const int (&src)[32])
{
    out[2 * i] = pc2_assemble(pt, *reinterpret_cast<const int(*)[16]>(&src[0]));
    out[2 * i + 1] = pc2_assemble(pt, *reinterpret_cast<const int(*)[16]>(&src[16]));
}

// REC 16: gem_decode_pointcloud2's float4 xyzi; REC 32: gem_decode_pointcloud2_records' whole PointXYZRGBICT records (f18)
template <int REC> __global__ void __launch_bounds__(PC2_BLOCK) k_decode_pc2(const __grid_constant__ Pc2Params p, uint4 *out)
{
    extern __shared__ uint4 s_raw[];
    __shared__ int s_src[REC]; // per output byte: its byte in the point, or -1 (0)
    if (threadIdx.x < REC) {
        const unsigned sb = REC == 32 ? threadIdx.x : threadIdx.x < 12 ? threadIdx.x : threadIdx.x + 12; // struct bytes
        int src = -1;
        for (int k = 0; k < p.nspans; k++) // M3: in span order, a later span overwrites an earlier one
            if (sb >= p.spans[k].struct_offset && sb < p.spans[k].struct_offset + p.spans[k].size)
                src = (int)(p.spans[k].serialized_offset + (sb - p.spans[k].struct_offset));
        s_src[threadIdx.x] = src;
    }
    __syncthreads();
    int src[REC];
#pragma unroll
    for (int b = 0; b < REC; b++) src[b] = s_src[b];
    const uintptr_t lo = (uintptr_t)p.data, hi = lo + p.data_bytes;
    for (unsigned long long t = blockIdx.x; t < p.tiles; t += gridDim.x) {
        const unsigned long long row = t / p.tiles_per_row;
        const unsigned c0 = (unsigned)(t % p.tiles_per_row) * p.tile;
        const unsigned cnt = p.width - c0 < p.tile ? p.width - c0 : p.tile;
        const unsigned char *base = p.data + row * p.row_step + (unsigned long long)c0 * p.point_step;
        if (p.staged) {
            const uintptr_t a0 = (uintptr_t)base & ~(uintptr_t)15;
            const uintptr_t a1 = ((uintptr_t)base + (uintptr_t)cnt * p.point_step + 15) & ~(uintptr_t)15;
            const unsigned words = (unsigned)((a1 - a0) >> 4);
            for (unsigned w = threadIdx.x; w < words; w += blockDim.x) s_raw[w] = pc2_load_word(a0 + 16 * (uintptr_t)w, lo, hi);
            __syncthreads();
            if (threadIdx.x < cnt)
                pc2_store<REC>(out, row * p.width + c0 + threadIdx.x,
                               (const unsigned char *)s_raw + ((uintptr_t)base - a0) + (size_t)threadIdx.x * p.point_step, src);
            __syncthreads(); // the next tile overwrites the staged bytes
        } else if (threadIdx.x < cnt) {
            pc2_store<REC>(out, row * p.width + c0 + threadIdx.x, base + (size_t)threadIdx.x * p.point_step, src);
        }
    }
}

// ---- cv_bridge::toCvCopy(image, BGR8) for the byte-permutation encodings -----------------------------------------------
enum { IMG_BGR8 = 0, IMG_RGB8 = 1, IMG_BGRA8 = 2, IMG_RGBA8 = 3, IMG_MONO8 = 4 };
inline int image_encoding(const char *e)
{
    static const char *const names[] = {"bgr8", "rgb8", "bgra8", "rgba8", "mono8"};
    for (int k = 0; k < 5; k++)
        if (e && strcmp(e, names[k]) == 0) return k;
    return -1;
}
__host__ __device__ inline int image_channels(int enc) { return enc == IMG_MONO8 ? 1 : (enc == IMG_BGRA8 || enc == IMG_RGBA8) ? 4 : 3; }

// one thread per output pixel: bgr8 / bgra8 keep the first three bytes, rgb8 / rgba8 swap bytes 0 and 2, mono8 repeats
__global__ void k_image_to_bgr8(const unsigned char *src, int width, int height, long long step, int enc, unsigned char *dst,
                                long long dst_step)
{
    const int ch = image_channels(enc);
    const bool swap = enc == IMG_RGB8 || enc == IMG_RGBA8;
    const size_t n = (size_t)width * height, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const size_t y = i / (size_t)width, x = i % (size_t)width;
        const unsigned char *s = src + y * step + x * ch;
        unsigned char *d = dst + y * dst_step + 3 * x;
        if (enc == IMG_MONO8) {
            const unsigned char v = s[0];
            d[0] = v; d[1] = v; d[2] = v;
        } else {
            const unsigned char c0 = s[0], c1 = s[1], c2 = s[2];
            d[0] = swap ? c2 : c0; d[1] = c1; d[2] = swap ? c0 : c2;
        }
    }
}

} // namespace gem
