// gem_submap.cuh -- loop-closure re-fusion of submaps (SURVEY 8f row 4): what ElevationMapping::updateGlobalMap
// (ElevationMapping.cpp:773-905) does with pcl::transformPointCloud, two std::unordered_map's and a pairwise formula,
// on the device: rigid re-transform of a submap's PointXYZRGBICT records, and the pairwise fusion of two submaps through
// open-addressing hash tables of their cells.  DESIGN.md section "f4" lists, item by item, what is reproduced literally
// and what is DEFINED here because the reference leaves it to unordered_map iteration order or to uninitialised memory.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gem {

struct SubPoint { // PointXYZRGBICT.hpp:26-48, 32 bytes
    float x, y, z, w;
    uint32_t bgra;
    float covariance, intensity, travers;
};

static_assert(sizeof(SubPoint) == 32, "PointXYZRGBICT is 32 bytes");

// pcl::transformPointCloud (ElevationMapping.cpp:805): x' = t00 x + t01 y + t02 z + t03, left to right in float (the
// scalar code of PCL <= 1.9; PCL is an unpinned dependency of the reference).  T: row-major 4 x 4.
struct Rigid { float t[12]; };
__device__ __forceinline__ void rigid_apply(SubPoint &q, const Rigid &T)
{
    const float x = q.x, y = q.y, z = q.z;
    q.x = ((T.t[0] * x + T.t[1] * y) + T.t[2] * z) + T.t[3];
    q.y = ((T.t[4] * x + T.t[5] * y) + T.t[6] * z) + T.t[7];
    q.z = ((T.t[8] * x + T.t[9] * y) + T.t[10] * z) + T.t[11];
}
__global__ void __launch_bounds__(256) k_transform_cloud(SubPoint *p, int n, const __grid_constant__ Rigid T)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    rigid_apply(p[i], T);
}
// the same per point over the records [off[0], off[nseg]) of a packed stack: record r of segment s (off[s] <= r <
// off[s + 1]) is moved by T[s].  off and T are in device memory, nseg + 1 and nseg entries.
__global__ void __launch_bounds__(256) k_transform_segments(SubPoint *p, const int *off, const Rigid *T, int nseg)
{
    const int r = off[0] + (int)(blockIdx.x * blockDim.x + threadIdx.x);
    if (r >= off[nseg]) return;
    int lo = 0, hi = nseg - 1; // the last s with off[s] <= r
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= r) lo = mid; else hi = mid - 1;
    }
    rigid_apply(p[r], T[lo]);
}

// pointCloudtoHash (ElevationMapping.cpp:1180-1192): the cell of a point is the float pair
// (ceil(x / res) * res - res / 2, same for y), evaluated in double (resolution_ is a double) and stored to float;
// GridPointEqual compares the floats.
__device__ __forceinline__ unsigned long long cell_key(float x, float y, double res, float &rx, float &ry)
{
    rx = (float)(ceil((double)x / res) * res - res / 2.0);
    ry = (float)(ceil((double)y / res) * res - res / 2.0);
    if (rx == 0.0f) rx = 0.0f; // -0 == +0 for GridPointEqual
    if (ry == 0.0f) ry = 0.0f;
    return ((unsigned long long)__float_as_uint(rx) << 32) | (unsigned long long)__float_as_uint(ry);
}
constexpr unsigned long long HASH_EMPTY = 0xffffffffffffffffull; // NaN/NaN pattern: no real cell has it

__device__ __forceinline__ unsigned hash_slot(unsigned long long k, unsigned mask)
{
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return (unsigned)k & mask;
}
// umap::insert keeps the FIRST point of a cell: the table stores, per cell, the smallest point index
// The count of every cloud is read from device memory (n): a chain of pairs runs without host round trips.
__global__ void __launch_bounds__(256) k_hash_insert(const SubPoint *p, const int *n, double res, unsigned long long *keys, int *first, unsigned mask)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *n) return;
    float rx, ry;
    const unsigned long long k = cell_key(p[i].x, p[i].y, res, rx, ry);
    if (k == HASH_EMPTY || rx != rx || ry != ry) return; // a NaN position equals nothing, itself included: such points never meet another
    unsigned s = hash_slot(k, mask);
    for (;;) {
        const unsigned long long prev = atomicCAS(&keys[s], HASH_EMPTY, k);
        if (prev == HASH_EMPTY || prev == k) { atomicMin(&first[s], i); return; }
        s = (s + 1) & mask;
    }
}
__device__ __forceinline__ int hash_find(const unsigned long long *keys, const int *first, unsigned mask, unsigned long long k)
{
    unsigned s = hash_slot(k, mask);
    for (;;) {
        const unsigned long long q = keys[s];
        if (q == k) return first[s];
        if (q == HASH_EMPTY) return -1;
        s = (s + 1) & mask;
    }
}

// One thread per point of the OLD submap (submap i, "out_old"), launched before k_refuse_pair: keep_o[i] = 1 iff point i
// is the first of its cell (the point the hash map holds and localHashtoPointCloud emits); its position becomes the
// cell's (:1129-1130).  A launch of its own because k_refuse_pair overwrites whole old records with the cell's position,
// and a cell centre does not always key to its own cell: with res = 2^m, the coordinate 2^(m+23) + res is the only float
// of its cell, and its centre rounds (a tie, to even) to 2^(m+23), which lies in the cell below.  So the old side reads
// only unmodified positions.
__global__ void __launch_bounds__(256)
k_refuse_keep(SubPoint *po, const int *no, double res, const unsigned long long *ko, const int *fo, unsigned mo, unsigned char *keep_o)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *no) return;
    float rx, ry;
    const unsigned long long k = cell_key(po[i].x, po[i].y, res, rx, ry);
    const bool nan = rx != rx || ry != ry;
    const bool first = nan || hash_find(ko, fo, mo, k) == i;
    keep_o[i] = first ? 1 : 0;
    if (first) { po[i].x = rx; po[i].y = ry; po[i].w = 1.0f; }
}

// One thread per point of the NEW submap (the neighbour, "out_new"); `old` is submap i ("out_old"), its keep flags and
// positions already set by k_refuse_keep.  keep_n[i] = 1 iff point i is the first of its cell.
// ElevationMapping.cpp:847-870, with every cell present in both maps fused exactly ONCE (DEFINITION: the reference
// erases and re-inserts while iterating, so what it visits twice depends on libstdc++'s bucket order).
// compat != 0: the fused values as the reference's expression evaluates (C operator precedence, :862-863);
// compat == 0: the weighting the expression was written for.
__global__ void __launch_bounds__(256)
k_refuse_pair(SubPoint *pn, const int *nn, SubPoint *po, double res, const unsigned long long *kn, const int *fn, unsigned mn,
              const unsigned long long *ko, const int *fo, unsigned mo, unsigned char *keep_n, int compat, int *count)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *nn) return;
    float rx, ry;
    const unsigned long long k = cell_key(pn[i].x, pn[i].y, res, rx, ry);
    const bool nan = rx != rx || ry != ry;
    const bool first = nan || hash_find(kn, fn, mn, k) == i;
    keep_n[i] = first ? 1 : 0;
    if (!first) return;
    SubPoint a = pn[i];
    a.x = rx; a.y = ry; a.w = 1.0f;
    const int j = nan ? -1 : hash_find(ko, fo, mo, k);
    if (j >= 0) {
        const float vo = po[j].covariance, eo = po[j].z, vn = a.covariance, en = a.z;
        if (vo > 0.0f && vo < 1.0f) { // :857
            const double vn2 = (double)vn * (double)vn, vo2 = (double)vo * (double)vo; // pow(float, 2) in double: exact squares
            float ef, vf;
            if (compat) { // :862-863 as C parses them
                ef = (float)((vn2 * (double)eo + vo2 * (double)en / vo2) + vn2);
                vf = (float)(vo2 * vn2 / vo2 + vn2);
            } else {
                ef = (float)((vn2 * (double)eo + vo2 * (double)en) / (vo2 + vn2));
                vf = (float)(vo2 * vn2 / (vo2 + vn2));
            }
            a.z = ef;
            a.covariance = vf;
            SubPoint b = a; // both maps get the fused cell, with the NEW map's colour / intensity / travers (:856)
            po[j] = b;      // (x, y are the cell's position in both)
            atomicAdd(count, 1);
        }
    }
    pn[i] = a;
}

// ---- localMap_ on the device (ElevationMapping.cpp:740-747, localHashtoPointCloud :1124-1140) -----------------------
// The store is an append log of harvested PointXYZRGBICT records (2 x float4 each) plus an open-addressing index from a
// cell's key to the LATEST log position holding it.  GridPointEqual compares the float (x, y) of a grid_map cell centre;
// those are finite and never -0, so the key is their bit pattern.  find / erase / insert (:740-747) leaves the last write
// of a key, and it moves the key to the end of an insertion-ordered iteration: keeping log entry i iff the index points
// at i, in log order, is that iteration (DESIGN.md "local submap", order DEFINED).
__device__ __forceinline__ unsigned long long point_key(float x, float y)
{
    return ((unsigned long long)__float_as_uint(x) << 32) | (unsigned long long)__float_as_uint(y);
}
// index the log entries [from, to); a key's slot keeps the largest position (the later cell of one call, or a later call)
__global__ void __launch_bounds__(256) k_local_index(const float4 *log, int from, int to, unsigned long long *keys, int *latest, unsigned mask)
{
    const int i = from + (int)(blockIdx.x * blockDim.x + threadIdx.x);
    if (i >= to) return;
    const float4 p = log[2 * (size_t)i];
    const unsigned long long k = point_key(p.x, p.y);
    unsigned s = hash_slot(k, mask);
    for (;;) {
        const unsigned long long prev = atomicCAS(&keys[s], HASH_EMPTY, k);
        if (prev == HASH_EMPTY || prev == k) { atomicMax(&latest[s], i); return; }
        s = (s + 1) & mask;
    }
}
__device__ __forceinline__ bool local_kept(const float4 *log, int i, int n, const unsigned long long *keys, const int *latest, unsigned mask)
{
    if (i >= n) return false;
    const float4 p = log[2 * (size_t)i];
    return hash_find(keys, latest, mask, point_key(p.x, p.y)) == i;
}
// take, pass 1: kept entries per 32 log entries (one warp each); the counts are then scanned by k_compact_scan
constexpr int TAKE_BLOCK = 1024;
__global__ void __launch_bounds__(TAKE_BLOCK) k_local_count(const float4 *log, int n, const unsigned long long *keys, const int *latest,
                                                            unsigned mask, int *cnt)
{
    const int i = blockIdx.x * TAKE_BLOCK + threadIdx.x;
    const unsigned b = __ballot_sync(0xffffffffu, local_kept(log, i, n, keys, latest, mask));
    if ((threadIdx.x & 31u) == 0u && i < n) cnt[i >> 5] = __popc(b);
}
// take, pass 2: entry i goes to (totals of the scan segments in front) + (scanned count of its warp) + (rank in the warp)
__global__ void __launch_bounds__(TAKE_BLOCK) k_local_write(const float4 *log, int n, const unsigned long long *keys, const int *latest,
                                                            unsigned mask, const int *ofs, const int *segtot, int seg_size, float4 *out)
{
    const int i = blockIdx.x * TAKE_BLOCK + threadIdx.x;
    const unsigned lane = threadIdx.x & 31u;
    const bool keep = local_kept(log, i, n, keys, latest, mask);
    const unsigned b = __ballot_sync(0xffffffffu, keep);
    const int chunk = i >> 5, seg = chunk / seg_size;
    int pre = 0;
    for (int q = (int)lane; q < seg; q += 32) pre += segtot[q];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) pre += __shfl_xor_sync(0xffffffffu, pre, d);
    if (keep) {
        const size_t pos = (size_t)pre + ofs[chunk] + __popc(b & ((1u << lane) - 1u));
        out[2 * pos + 0] = log[2 * (size_t)i + 0];
        out[2 * pos + 1] = log[2 * (size_t)i + 1];
    }
}

// Order-preserving compaction of a re-fused cloud, with its count in device memory and a host-known upper bound ub on it
// (the count before the pair: a re-fusion only shrinks a cloud).  Pass 1 counts the kept records per 32 (and clears the
// flags in [*n, ub), so pass 2 needs no count), k_compact_scan scans those counts over many blocks, pass 2 writes every
// kept record to its rank and the new count to *n.
__global__ void __launch_bounds__(TAKE_BLOCK) k_keep_count(unsigned char *keep, const int *n, int ub, int *cnt)
{
    const int i = blockIdx.x * TAKE_BLOCK + threadIdx.x;
    bool k = false;
    if (i < ub) {
        if (i < *n) k = keep[i] != 0; else keep[i] = 0;
    }
    const unsigned b = __ballot_sync(0xffffffffu, k);
    if ((threadIdx.x & 31u) == 0u && i < ub) cnt[i >> 5] = __popc(b);
}
__global__ void __launch_bounds__(TAKE_BLOCK) k_keep_write(const SubPoint *in, const unsigned char *keep, int ub, const int *ofs,
                                                           const int *segtot, int nseg, int seg_size, SubPoint *out, int *n)
{
    const int i = blockIdx.x * TAKE_BLOCK + threadIdx.x;
    const unsigned lane = threadIdx.x & 31u;
    const bool k = i < ub && keep[i] != 0;
    const unsigned b = __ballot_sync(0xffffffffu, k);
    const int chunk = i >> 5, seg = chunk / seg_size;
    int pre = 0;
    for (int q = (int)lane; q < seg; q += 32) pre += segtot[q];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) pre += __shfl_xor_sync(0xffffffffu, pre, d);
    if (k) out[pre + ofs[chunk] + __popc(b & ((1u << lane) - 1u))] = in[i];
    if (i == 0) {
        int t = 0;
        for (int q = 0; q < nseg; q++) t += segtot[q];
        *n = t;
    }
}

// ---- the global map's submap stack (DESIGN.md f16) ----------------------------------------------------------------------
// Re-pack after an update: off_new[s] = exclusive prefix of the submaps' device counts (one thread: the stack holds
// hundreds of submaps, not millions), off_new[nseg] = the total
__global__ void k_pack_offsets(const int *cnt, int nseg, int *off_new)
{
    int t = 0;
    for (int s = 0; s < nseg; s++) { off_new[s] = t; t += cnt[s]; }
    off_new[nseg] = t;
}
// record r of segment s (off_old[s] <= r < off_old[s + 1]) goes to off_new[s] + (r - off_old[s]) if it is among the
// segment's first cnt[s]; src and dst are different buffers
__global__ void __launch_bounds__(256) k_pack_segments(const SubPoint *src, SubPoint *dst, const int *off_old, const int *off_new,
                                                       const int *cnt, int nseg)
{
    const int r = (int)(blockIdx.x * blockDim.x + threadIdx.x);
    if (r >= off_old[nseg]) return;
    int lo = 0, hi = nseg - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off_old[mid] <= r) lo = mid; else hi = mid - 1;
    }
    const int l = r - off_old[lo];
    if (l < cnt[lo]) dst[off_new[lo] + l] = src[r];
}

} // namespace gem
