// gem_add.cuh -- the add path of libgem_b200: Process_points + Fuse (gpu.cu:384-455, 477-537): one bin kernel, two fold
// kernels that run side by side (the few hundred cells with more than 40 records have a kernel of their own).
//
//   k_bin   1 thread/point : float4 load, SE(3), filters, sensor variance, cell key, per-cell arrival rank via one
//                            L2 atomic on the cell's own 32-byte record, 16-byte record {point index, h, var, rgb}
//                            stored straight to its slot.  Slots need NO allocation for ranks 0..39: ranks 0..7 live
//                            in a chunk addressed by the cell key, ranks 8..39 in a chunk addressed by the INDEX of
//                            the point that drew rank 8 (published in the cell record); only the few cells with more
//                            than 40 points take geometric chunks from a bump pool
//   k_fold  1 thread/touched cell with at most 8 records : order the cell's records by point index (== the order in
//                            which G_fuse's per-cell loop visits them), sequential Kalman fold with the 5-sigma gate,
//                            lowest-scan update, one 16 B write-back per cell.  The cells are found through a
//                            per-point mark array (point i drew rank 0 of cell c): no global list of touched cells
//   k_fold_long  1 warp/cell with more than 8 records, drawn from the two queues k_bin filled (one atomic per cell that
//                            reaches rank 8, one more per cell that reaches rank 40): a serial list runs 2-4x faster
//                            on a scheduler of its own than next to seven busy warps, and the longest list of a frame
//                            is the latency of the fold
//
// Round 1 had four kernels (transform+bin, per-cell allocation, scatter, fold) and five per-cell arrays; every
// touched cell cost five random 32-byte sectors per call.  Here a cell IS one sector and the allocation and scatter
// kernels are gone.  Measured on the way (profiles/r2_add_path_notes.md): a same-address atomic from different SMs
// costs ~1.4 ns at L2, so anything that takes one global counter per warp or per touched cell (a touched list, a
// list of long cells, a record allocator) serialises for microseconds; ld.acquire.gpu compiles to LDG + CCTL.IVALL
// (invalidates the SM's L1) and st.release.gpu to a MEMBAR.  Hence: no counters on the hot path, relaxed accesses.
#pragma once
#include "gem_kernels.cuh"

namespace gem {

// ---------------------------------------------------------------------------------------
// record chunks: level 0 = ranks 0..7 at chunk0[8 * key]; level 1 = ranks 8..39 at pool1[33 * i8] where i8 is the
// index of the point that drew rank 8 (slot 0 of a pool chunk is its header); level j >= 2 = 8 * 4^j ranks
// (128, 512, ...) bump-allocated from `pool` by the point that draws the level's first rank (40, 168, 680, ...).
// ---------------------------------------------------------------------------------------
constexpr int CHUNK0 = 8;
constexpr int CHUNK1_SLOTS = 33; // header + 32 records
__host__ __device__ __forceinline__ int level_base(int j) { return (CHUNK0 * ((1 << (2 * j)) - 1)) / 3; } // 8, 40, 168, 680, ...
__host__ __device__ __forceinline__ int level_cap(int j) { return CHUNK0 << (2 * j); }                    // 32, 128, 512, ...
__device__ __forceinline__ int level_of(int rank) // rank >= CHUNK0
{
    int j = 1;
    while (rank >= level_base(j + 1)) j++;
    return j;
}
constexpr int FOLD_LONG_FROM = 40;       // = level_base(2): a cell with more records is a "long" list, folded first

struct BinCounters { // one counter per 128-byte line
    int pool;     int pad0[31];  // pool slots handed out to chunks of level >= 2 (offset of the next chunk - 1)
    int nlong;    int pad1[31];  // cells with more than 40 records (the long-list queue, ~100 per frame)
    int next_long;int pad2[31];  // k_fold_long's draw counter (over the long-list queue, then the large-list queue)
    int ntouched; int pad3[31];  // statistics, accumulated by the folds: cells touched,
    int total;    int pad4[31];  //   points binned (accepted AND inside the grid / tile),
    int maxk;     int pad5[31];  //   longest per-cell list
    int nmarks;   int pad6[31];  // tiled maps: marks written by k_bin_peer (the fold's work list length)
    int nlarge;   int pad7[31];  // cells with more than 8 records (the large-list queue, a few hundred per frame)
};

static_assert(sizeof(BinCounters) == 8 * 128, "one counter per 128-byte line");
static_assert(sizeof(BinCounters) / sizeof(int) <= 256, "zero_next_counters: one thread per word of a 256-thread block");
static_assert(FOLD_LONG_FROM == CHUNK0 + 32 && CHUNK1_SLOTS == 33, "second chunk = header + ranks 8..39");

// the queues of k_fold_long hold {key, LIST_*, i8, p2}: i8 = index of the cell's rank-8 point, p2 = pool offset of its
// level-2 chunk (0 in a LIST_LARGE entry).  A cell with more than 40 records has an entry in both queues.
enum { LIST_LARGE = 2, LIST_LONG = 3 };

struct BinScratch { // one set per call parity
    int2 *mark;        // [P]   {key, index of the cell in the lowest layer} if point i drew rank 0 of cell `key`, else key = -1
    uint4 *chunk0;     // [8 * cells] records of rank 0..7 of cell `key`
    uint4 *pool1;      // [33 * P]    level-1 chunks, addressed by the index of the rank-8 point
    uint4 *pool;       // [pool_cap + 1] chunks of level >= 2; offset 0 is never handed out
    int4 *tlong;       // [long_cap]  {key, LIST_LONG, i8, p2} of the cells that reached rank 40: k_fold_long's first queue
    int4 *tlarge;      // [large_cap] {key, LIST_LARGE, i8, 0} of the cells that reached rank 8: its second queue
    BinCounters *ctr;      // counters of this call (zero when it starts)
    BinCounters *ctr_next; // zeroed by this call's bin kernel for the call after
    int par;           // which {counter, i8 + 1} pair of the cell records this call uses
    int pool_cap;
    int long_cap, large_cap; // entries of tlong / tlarge: P / 41 + 1 and P / 9 + 1 (at most as many as the map has cells, + 1)
    unsigned long long *stamps; // debug (gem_debug_stamps): %globaltimer marks of the kernels, else null
};

__device__ __forceinline__ unsigned long long globaltimer_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// slot 0/8: earliest start of k_bin / k_fold (stored as ~t so that one atomicMax serves); others: latest time a
// block's first warp passed the mark.  One thread per block: the marks themselves are same-address atomics.
__device__ __forceinline__ void stamp_start(const BinScratch &sc, int slot)
{
    if (sc.stamps && threadIdx.x == 0) atomicMax(&sc.stamps[slot], ~globaltimer_ns());
}
__device__ __forceinline__ void stamp_mark(const BinScratch &sc, int slot)
{
    if (sc.stamps && threadIdx.x == 0) atomicMax(&sc.stamps[slot], globaltimer_ns());
}
__device__ __forceinline__ void stamp_lane0(const BinScratch &sc, int slot, bool cond)
{
    if (sc.stamps && cond && (threadIdx.x & 31u) == 0u) atomicMax(&sc.stamps[slot], globaltimer_ns());
}
// longest time since t0 (one long list's own start) at which any long list passed the mark
__device__ __forceinline__ void stamp_since(const BinScratch &sc, int slot, unsigned long long t0)
{
    if (sc.stamps && t0 && (threadIdx.x & 31u) == 0u) atomicMax(&sc.stamps[slot], globaltimer_ns() - t0);
}

// Pointer publication between running blocks: RELAXED loads / stores at GPU scope (served by L2, no L1 involvement).
// Nothing but the pointer itself is communicated, so no acquire / release is needed -- and ld.acquire.gpu compiles to
// LDG + CCTL.IVALL (invalidate the SM's whole L1) and st.release.gpu to a MEMBAR; the first version of this kernel
// spent half its time in those (profiles/r2a_k_bin_hotspots.txt).
//   * cell.bin[par].y (index of the cell's rank-8 point + 1): a 32-bit word, 0 = not published, reset to 0 by the fold;
//   * the header of a pool chunk: the 64-bit word at byte 8 of its first slot = {next-level offset, CHUNK_TAG}.  A
//     stale RECORD in that slot carries {var bits, rgb | flag} there: bit 63 is clear; a stale header cannot exist
//     because the fold clears every header of the chunks it consumes and the pool starts zeroed.
constexpr unsigned long long CHUNK_TAG = 0x8000000000000000ull;
__device__ __forceinline__ int ld_relaxed(const int *p)
{
    int v;
    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed(int *p, int v)
{
    asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int spin_nonzero(const int *p)
{
    int v = ld_relaxed(p);
    while (v == 0) {
        __nanosleep(20);
        v = ld_relaxed(p);
    }
    return v;
}
__device__ __forceinline__ unsigned long long *chunk_header(uint4 *chunk) { return reinterpret_cast<unsigned long long *>(chunk) + 1; }
__device__ __forceinline__ void publish_next(uint4 *chunk, int next)
{
    const unsigned long long v = CHUNK_TAG | (unsigned long long)(unsigned)next;
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(chunk_header(chunk)), "l"(v) : "memory");
}
__device__ __forceinline__ int spin_next(uint4 *chunk)
{
    unsigned long long v;
    for (;;) {
        asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(chunk_header(chunk)) : "memory");
        if (v & CHUNK_TAG) break;
        __nanosleep(20);
    }
    return (int)(unsigned)(v & 0xffffffffull);
}
// the fold's view (the bin kernel has completed): next-level offset of a chunk whose successor exists
__device__ __forceinline__ int next_chunk(const uint4 *chunk) { return (int)chunk->z; }

// ---------------------------------------------------------------------------------------
// point sources of the bin kernel
// ---------------------------------------------------------------------------------------
enum { SRC_XYZI = 0, SRC_SOA = 1, SRC_PCL32 = 2, SRC_KEYS = 3, SRC_RECORDS = 4 };
// or-ed into SRC_XYZI / SRC_SOA / SRC_PCL32: the instantiation that runs every sensor model (transform_point<true>)
constexpr int SRC_ANY_MODEL = 8;
// or-ed into SRC_XYZI: the point count is min(n, *BinSource::n_dev), n the host's upper bound that sizes the grid (the
// asynchronous pre-filtered add, whose count only the device knows)
constexpr int SRC_DEVN = 16;

struct RouteRec { // 20 bytes on the wire between tiles (gem_route.cuh)
    int gkey;     // global geographic linear index gx*L+gy
    float h, var;
    uint32_t rgb;
    float intensity;
};
static_assert(sizeof(RouteRec) == 20, "20 bytes on the wire");

struct BinSource {
    // SRC_XYZI: float4 {x,y,z,intensity} + optional uchar4 rgba; SRC_PCL32: 2 x float4 per point (PointXYZRGBICT.hpp:26-48)
    const float4 *xyzi;
    const uchar4 *rgba;
    const float4 *pcl;
    // SRC_SOA (Process_points, gpu.cu:1085): inputs x, y, z; optional outputs = what Process_points returns
    const float *x, *y, *z;
    int *key_out;
    float *h_out, *hv_out, *xt_out, *yt_out;
    // SRC_KEYS (Fuse, gpu.cu:1154): map_index, height, var, R, G, B, intensity arrays
    const int *key_in, *R, *G, *B;
    const float *h_in, *hv_in, *inten_in;
    int ncells;
    // SRC_RECORDS (tiled maps): records received from the other tiles (gkey < 0 = padding)
    const RouteRec *rec;
    const int *n_dev; // SRC_DEVN
};

struct PointOut {
    int key;       // layer key or -1
    int geo;       // the cell's index in the lowest layer (geographic index; tiled handles: the key), or -1: derive it from the key
    float h, hv;
    uint32_t rgbf; // rgb | REC_COLOUR_OK
};

template <int SRC>
__device__ __forceinline__ PointOut bin_source_point(const MapGeom &g, const FrameParams &f, const BinSource &in, int i,
                                                     const SegTable *segs, const FrameParams *frames)
{
    constexpr bool ANY = (SRC & SRC_ANY_MODEL) != 0;
    constexpr int S = SRC & ~(SRC_ANY_MODEL | SRC_DEVN);
    PointOut o;
    o.key = -1; o.geo = -1; o.h = -1.0f; o.hv = -1.0f; o.rgbf = 0u;
    if (S == SRC_XYZI) {
        const float4 p = ld_stream_f4(in.xyzi + i);
        PtRes r;
        if (!ANY) {
            r = segs ? transform_point(g, frames[find_segment(*segs, i)], p.x, p.y, p.z) : transform_point(g, f, p.x, p.y, p.z);
        } else if (segs) { // the index restarts with every segment's cloud (idx0 = -offsets[s])
            const FrameParams &fs = frames[find_segment(*segs, i)];
            r = transform_point<true>(g, fs, p.x, p.y, p.z, fs.idx0 + i);
        } else {
            r = transform_point<true>(g, f, p.x, p.y, p.z, f.idx0 + i);
        }
        if (r.ingrid) { o.key = local_key(g, r.gx, r.gy); o.geo = g.tiled ? o.key : r.gx * g.L + r.gy; }
        o.h = r.h; o.hv = r.hv;
        uint32_t rgb = 0u;
        if (in.rgba) {
            const uchar4 c = in.rgba[i];
            rgb = pack_rgb(c.x, c.y, c.z);
        }
        o.rgbf = with_colour_flag(rgb, p.w);
    } else if (S == SRC_PCL32) {
        const float4 p = ld_stream_f4(in.pcl + 2 * (size_t)i);
        const float4 q = ld_stream_f4(in.pcl + 2 * (size_t)i + 1); // {rgb(b,g,r,a bytes), covariance, intensity, travers}
        const PtRes r = transform_point<ANY>(g, f, p.x, p.y, p.z, f.idx0 + i);
        if (r.ingrid) { o.key = local_key(g, r.gx, r.gy); o.geo = g.tiled ? o.key : r.gx * g.L + r.gy; }
        o.h = r.h; o.hv = r.hv;
        const uint32_t bgra = __float_as_uint(q.x);
        o.rgbf = with_colour_flag(pack_rgb((bgra >> 16) & 255, (bgra >> 8) & 255, bgra & 255), q.z);
    } else if (S == SRC_SOA) {
        const PtRes r = transform_point<ANY>(g, f, in.x[i], in.y[i], in.z[i], f.idx0 + i);
        if (r.ingrid) { o.key = local_key(g, r.gx, r.gy); o.geo = g.tiled ? o.key : r.gx * g.L + r.gy; }
        o.h = r.h; o.hv = r.hv;
        if (in.key_out) in.key_out[i] = o.key;
        if (in.h_out) in.h_out[i] = r.h;
        if (in.hv_out) in.hv_out[i] = r.hv;
        if (in.xt_out) { in.xt_out[i] = r.xt; in.yt_out[i] = r.yt; }
    } else if (S == SRC_KEYS) {
        int key = in.key_in[i];
        if (key < 0 || key >= in.ncells) key = -1; // no G_fuse thread has such a map_index
        o.key = key;
        o.h = in.h_in[i]; o.hv = in.hv_in[i];
        // the reference tests R,G,B != 0 on int values; channels are 8-bit by construction (PointXYZRGBICT r/g/b are
        // uint8, SPB.cpp:164-166).  A non-zero int whose low byte is zero is mapped to 255 in that byte so "!= 0" holds.
        const int r = in.R ? in.R[i] : 0, gg = in.G ? in.G[i] : 0, b = in.B ? in.B[i] : 0;
        const uint32_t rgb = pack_rgb((r != 0 && (r & 255) == 0) ? 255 : r, (gg != 0 && (gg & 255) == 0) ? 255 : gg,
                                      (b != 0 && (b & 255) == 0) ? 255 : b);
        o.rgbf = with_colour_flag(rgb, in.inten_in ? in.inten_in[i] : 0.0f);
    } else { // SRC_RECORDS
        const RouteRec r = in.rec[i];
        if (r.gkey >= 0) {
            const int gx = r.gkey / g.L, gy = r.gkey - gx * g.L;
            o.key = local_key(g, gx, gy);
            o.geo = g.tiled ? o.key : r.gkey;
        }
        o.h = r.h; o.hv = r.var;
        o.rgbf = with_colour_flag(r.rgb, r.intensity);
    }
    return o;
}

// ---------------------------------------------------------------------------------------
// the bin phase: U points per thread and iteration; every slot u of an iteration is a coalesced row of points
// (index base + u*nthreads + tid).
//
// Who waits for whom.  A point of rank 9..39 needs the index of the cell's rank-8 point, which that point publishes
// right after its own atomic returns (no waiting).  The rank-40 point (168, 680, ...) allocates the level-2 (3, 4,
// ...) chunk with one atomic on the pool counter and publishes it in the header of the chunk one level down, which it
// finds through the pointers of the lower levels; points of rank >= 40 wait for those headers.  Every wait is for a
// thread that drew a LOWER rank in the same cell -- it has executed its atomic, so it is resident and running -- and
// a publisher of level j waits only for publishers of levels < j: the wait-for graph is acyclic.  Publications of
// one thread are made level by level over all of its U points, so a thread never waits while it still owes a
// lower-level publication.
// ---------------------------------------------------------------------------------------
template <int SRC, int U>
__device__ __forceinline__ void bin_points(const MapGeom &g, const FrameParams &f, const BinSource &in, int n, Cell *cells,
                                           const BinScratch &sc, int tid, int nthreads, const SegTable *segs,
                                           const FrameParams *frames)
{
    const int par = sc.par;
    for (int base = 0; base < n; base += U * nthreads) {
        int key[U], rank[U], geo[U];
        uint4 rec[U];
        // ---- load, transform, arrival rank ---------------------------------------------------------------
#pragma unroll
        for (int u = 0; u < U; u++) {
            const int i = base + u * nthreads + tid;
            key[u] = -1;
            geo[u] = -1;
            rec[u] = make_uint4(0u, 0u, 0u, 0u);
            if (i < n) {
                const PointOut o = bin_source_point<SRC>(g, f, in, i, segs, frames);
                key[u] = o.key;
                geo[u] = o.geo;
                rec[u] = make_uint4((uint32_t)i, __float_as_uint(o.h), __float_as_uint(o.hv), o.rgbf);
            }
        }
#pragma unroll
        for (int u = 0; u < U; u++) rank[u] = (key[u] >= 0) ? atomicAdd(&cells[key[u]].bin[par].x, 1) : -1;
        // ---- marks; the rank-8 point publishes itself and queues the cell; allocators of level >= 2 reserve their chunk
        int lvl[U], myp[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const int i = base + u * nthreads + tid;
            lvl[u] = 0;
            myp[u] = 0;
            if (i >= n) continue;
            if (rank[u] == CHUNK0) {
                st_relaxed(&cells[key[u]].bin[par].y, i + 1);
                sc.tlarge[atomicAdd(&sc.ctr->nlarge, 1)] = make_int4(key[u], LIST_LARGE, i, 0); // a few hundred per frame
            } else if (rank[u] >= FOLD_LONG_FROM) {
                const int j = level_of(rank[u]);
                if (rank[u] == level_base(j)) {
                    lvl[u] = j;
                    myp[u] = 1 + atomicAdd(&sc.ctr->pool, level_cap(j) + 1); // one per 128+ records of one cell: rare
                }
            }
            sc.mark[i] = (rank[u] == 0) ? make_int2(key[u], geo[u]) : make_int2(-1, 0); // every point writes its mark (clears the previous call's)
        }
        // ---- chunk pointers of level >= 2, level by level ---------------------------------------------------------
        int maxl = 0;
#pragma unroll
        for (int u = 0; u < U; u++) maxl = max(maxl, lvl[u]);
        for (int l = 2; l <= maxl; l++) {
#pragma unroll
            for (int u = 0; u < U; u++) {
                if (lvl[u] != l) continue;
                const int i8 = spin_nonzero(&cells[key[u]].bin[par].y) - 1;
                uint4 *q = sc.pool1 + (size_t)CHUNK1_SLOTS * i8;
                for (int k = 2; k < l; k++) q = sc.pool + spin_next(q);
                if (l == 2) sc.tlong[atomicAdd(&sc.ctr->nlong, 1)] = make_int4(key[u], LIST_LONG, i8, myp[u]); // ~100 per frame
                publish_next(q, myp[u]);
            }
        }
        // ---- store the records -----------------------------------------------------------------------------------
#pragma unroll
        for (int u = 0; u < U; u++) {
            if (rank[u] < 0) continue;
            uint4 *dst;
            if (rank[u] < CHUNK0) {
                dst = sc.chunk0 + (size_t)CHUNK0 * key[u] + rank[u];
            } else {
                const int i8 = (rank[u] == CHUNK0) ? (base + u * nthreads + tid) : spin_nonzero(&cells[key[u]].bin[par].y) - 1;
                uint4 *q = sc.pool1 + (size_t)CHUNK1_SLOTS * i8;
                const int j = level_of(rank[u]);
                for (int k = 2; k <= j; k++) q = sc.pool + ((lvl[u] == k) ? myp[u] : spin_next(q));
                dst = q + 1 + (rank[u] - level_base(j));
            }
            *dst = rec[u];
        }
    }
}

__device__ __forceinline__ void zero_next_counters(const BinScratch &sc, int tid)
{
    if (tid < (int)(sizeof(BinCounters) / sizeof(int))) ((int *)sc.ctr_next)[tid] = 0; // 256 ints: the bin grids have >= 256 threads
}

template <int SRC, int U>
__global__ void __launch_bounds__(ADD_BLOCK)
k_bin(MapGeom g, MapLayers ml, FrameParams f, BinSource in, int n, BinScratch sc, const __grid_constant__ RegionOps ro, int point_blocks,
      const __grid_constant__ SegTable segs, const FrameParams *frames)
{
    if constexpr ((SRC & SRC_DEVN) != 0) n = min(n, *in.n_dev);
    if ((int)blockIdx.x < point_blocks) {
        stamp_start(sc, 0);
        zero_next_counters(sc, blockIdx.x * blockDim.x + threadIdx.x);
        bin_points<SRC, U>(g, f, in, n, ml.cell, sc, blockIdx.x * blockDim.x + threadIdx.x, point_blocks * blockDim.x,
                           frames ? &segs : nullptr, frames);
    } else { // extra blocks: deferred scroll clears + variance floor (only when no fold is in flight, see gem_api.cu)
        const size_t rb = gridDim.x - point_blocks;
        phase_regions(g, ml, ro, (size_t)(blockIdx.x - point_blocks) * blockDim.x + threadIdx.x, rb * blockDim.x);
    }
}

// =========================================================================================
// fold
// =========================================================================================
// where the fold finds the intensity of the point a cell finally takes its colour from: the record carries the
// point index, not the 4-byte intensity (a 16-byte record is one vector store and a cell's first 8 records are
// one 128-byte line); the input array is read once per cell instead
struct FoldSrc {
    const char *base; // intensity of point idx = *(const float *)(base + idx * stride); null: no intensities (0)
    int stride;       // xyzi: 16 (base = &xyzi[0].w), PointXYZRGBICT: 32, float array: 4, RouteRec: 20
};
__device__ __forceinline__ float fetch_intensity(const FoldSrc &s, uint32_t idx)
{
    return s.base ? *reinterpret_cast<const float *>(s.base + (size_t)idx * s.stride) : 0.0f;
}

struct CellState {
    float elev, var;
    uint32_t src;  // point index the cell last took intensity + colour from
    float inten;   // its intensity, when the caller prefetched the intensities of the list (else fetched at the end)
    uint32_t rgb;
    bool ci_dirty;
    float minh, minhv; // lowest-scan: min height and variance of the first point attaining it
    bool any;
    float low_old;     // lowest[cell] before this call, fetched with the cell state (off the tail of the cell)
    int low_idx;       // the cell's index in the (geographic) lowest layer
};

// lowest-scan of gpu.cu:432-438 (ORACLE DEFINITION): running minimum height of the call's points in
// the cell and the variance of the FIRST index attaining it.  Records must be offered in index order.
__device__ __forceinline__ void lowest_step(CellState &s, float h, float v)
{
    if (!s.any || h < s.minh) {
        s.minh = h;
        s.minhv = v;
        s.any = true;
    }
}

// The gate terms of one general step, shared by fold_step and fold_step_fast.
// gpu.cu:502-504: gate = RN(|h-e| / RN(sqrt(var))) > 5.  The fold is a serial dependency chain per cell, so the IEEE
// sqrt and divide are kept off it: the two roundings move the quotient by < 2.5e-7 relative, hence comparing d^2 with
// 25*var decides every case outside a +-1e-5 band exactly like the reference expression; inside the band, and for huge
// or non-finite values (`rare`), only the literal expression decides.
struct GateTerms {
    bool first;  // gpu.cu:484: the cell is empty
    float ov;    // the variance, floored
    float d;     // |h - e|
    bool hi, lo; // gate certainly true / certainly false
    bool rare;
};
__device__ __forceinline__ GateTerms gate_terms(const CellState &s, float h)
{
    GateTerms g;
    g.first = (s.elev == -10.0f);
    // gpu.cu:500-501: `var < 0.0001` compares in double; (float)0.0001 is the largest float below
    // the double literal, so the test is exactly `var <= 1e-4f`
    g.ov = (s.var <= 1e-4f) ? 1e-4f : s.var;
    g.d = fabsf(h - s.elev);
    const float dd = g.d * g.d, tv = 25.0f * g.ov;
    g.hi = dd > tv * 1.00001f;
    g.lo = dd < tv * 0.99999f;
    g.rare = !(dd < 1e30f && tv < 1e30f) | !(g.hi | g.lo);
    return g;
}

__device__ __forceinline__ void fold_step(CellState &s, float h, float v, uint32_t rgb, uint32_t idx, float inten, bool do_fuse)
{
    if (!do_fuse) return;
    const bool skip = (h == -1.0f); // gpu.cu:482
    const bool colour_ok = (rgb & REC_COLOUR_OK) != 0u; // gpu.cu:488, precomputed by the bin kernel
    const GateTerms g = gate_terms(s, h);
    const float oe = s.elev;
    bool gate = g.hi;
    if (g.rare) gate = (g.d / sqrtf(g.ov)) > 5.0f;
    // gpu.cu:518-519, computed speculatively (selected below)
    float qe, qv;
    div2_rn(g.ov * h + v * oe, v * g.ov, g.ov + v, qe, qv);
    const bool higher = oe < h; // gpu.cu:505
    const float ne = g.first ? h : (gate ? (higher ? h : oe) : qe);
    const float nv = g.first ? v : (gate ? (higher ? v : g.ov) : qv);
    const bool take = g.first || !gate || higher;
    if (!skip) {
        s.elev = ne;
        s.var = nv;
        if (take && colour_ok) {
            s.src = idx;
            s.inten = inten;
            s.rgb = rgb & 0xffffffu;
            s.ci_dirty = true;
        }
    }
}

// Branch-free twin of fold_step for the serial tail of long lists.  Same arithmetic, but no control flow inside the
// step: one warp folding one cell is in-order, so every branch of fold_step (gate band, division guard) puts the
// elevation-dependent gate chain IN FRONT of the variance-dependent reciprocal chain instead of beside it.  Here the
// step always takes the common path and only reports (returns true) when fold_step would have left it: gate inside
// the +-1e-5 band or non-finite, or division operands outside the guarded range.  The caller then redoes the chunk
// with fold_step from the saved state, so results are fold_step's bit for bit.
__device__ __forceinline__ bool fold_step_fast(CellState &s, float h, float v, uint32_t rgb, uint32_t idx, float inten)
{
    const bool skip = (h == -1.0f);
    const bool colour_ok = (rgb & REC_COLOUR_OK) != 0u;
    const GateTerms g = gate_terms(s, h);
    const float oe = s.elev, ov = g.ov;
    const float n0 = ov * h + v * oe, n1 = v * ov, den = ov + v;
    float qe, qv;
    div2_core(n0, n1, den, div2_rcp(den), qe, qv);
    const bool rare_div = !div2_fast_ok(n0, n1, den);
    const bool higher = oe < h;
    const float ne = g.first ? h : (g.hi ? (higher ? h : oe) : qe);
    const float nv = g.first ? v : (g.hi ? (higher ? v : ov) : qv);
    const bool take = (g.first | !g.hi | higher) & colour_ok & !skip;
    s.elev = skip ? s.elev : ne;
    s.var = skip ? s.var : nv;
    s.src = take ? idx : s.src;
    s.inten = take ? inten : s.inten;
    s.rgb = take ? (rgb & 0xffffffu) : s.rgb;
    s.ci_dirty = s.ci_dirty | take;
    return !skip & !g.first & (g.rare | (!g.hi & rare_div));
}

// the loads of a cell's state; issued before anything that depends on the list length
// low_idx < 0: derive the lowest index from the key (an integer division; the marks of short lists carry it instead)
__device__ __forceinline__ void cell_begin(CellState &s, const MapGeom &g, const MapLayers &ml, int key, bool do_lowest, int low_idx = -1)
{
    s.low_idx = (low_idx >= 0 || !do_lowest) ? low_idx : key_to_lowest(g, key);
    s.low_old = do_lowest ? ml.lowest[s.low_idx] : 0.0f;
    const float2 ev = load_ev(ml.cell, key);
    s.elev = ev.x; s.var = ev.y; s.src = 0u; s.inten = 0.0f; s.rgb = 0u; s.ci_dirty = false;
    s.minh = 0.0f; s.minhv = 0.0f; s.any = false;
}

// is the cell inside a scroll clear that the NEXT add call's Move has already decided?  (pipelined mode: this fold
// runs concurrently with the next call's bin kernel and carries that call's row / column clears, see gem_api.cu)
__device__ __forceinline__ bool in_clear_region(const MapGeom &g, const RegionOps &ro, int key)
{
    if (ro.count == 0) return false;
    const int row = key / g.cols, col = key - row * g.cols;
    bool hit = false;
#pragma unroll
    for (int r = 0; r < MAX_REGION_OPS; r++) {
        if (r < ro.count) {
            const RegionOp op = ro.op[r];
            if (op.kind == 1) hit |= (row >= op.start && row < op.start + op.n);
            else if (op.kind == 2) hit |= (col >= op.start && col < op.start + op.n);
        }
    }
    return hit;
}

// have_inten: s.inten is valid (the list's intensities were prefetched); else it is read from the input by point index
__device__ __forceinline__ void cell_end(CellState &s, const MapGeom &g, const MapLayers &ml, const BinScratch &sc, const FoldSrc &src,
                                         const RegionOps &ro_next, int key, bool do_fuse, bool do_lowest, bool have_inten)
{
    if (do_fuse) {
        if (in_clear_region(g, ro_next, key)) {
            // the cell scrolls out before anything can observe this fold: write what the clear writes (the region
            // blocks of this launch store the same bits, in either order)
            store_ev(ml.cell, key, make_float2(-10.0f, (float)0.0001));
            store_ci(ml.cell, key, make_uint2(0u, 0u));
        } else {
            if (s.var <= 1e-4f) s.var = 1e-4f; // gpu.cu:533-534 (same double-compare equivalence)
            store_ev(ml.cell, key, make_float2(s.elev, s.var));
            if (s.ci_dirty) store_ci(ml.cell, key, make_uint2(__float_as_uint(have_inten ? s.inten : fetch_intensity(src, s.src)), s.rgb));
        }
    }
    if (do_lowest && s.any) {
        // ORACLE DEFINITION of the racy gpu.cu:434-438 (SURVEY 8c): with m = min h of this
        // call's points in the cell and i* the first index attaining it,
        // lowest = m + 3*hv[i*] iff m <= lowest_old.
        if (s.minh <= s.low_old) ml.lowest[s.low_idx] = s.minh + 3.0f * s.minhv;
    }
    ml.cell[key].bin[sc.par] = make_int2(0, 0); // restore the all-zero invariant of this parity's {counter, slot}
}

// magnitude tests on bit patterns: |x| in [2^-40, 2^20)
__device__ __forceinline__ bool mag_ok(float x)
{
    const uint32_t u = __float_as_uint(x) & 0x7fffffffu;
    return (u - 0x2b800000u) < (0x49800000u - 0x2b800000u);
}

// The "plain" step (see fold_chunk for the argument): Kalman update or clear gate decision for ordinary magnitudes.
// Returns false when the step must be decided by the general or the literal code instead (the cell is empty, near
// the gate, numerator out of the guarded range); e / var then hold garbage and the caller redoes the list or chunk.
__device__ __forceinline__ bool plain_step(float &e, float &var, float h, float v, bool &take)
{
    // gpu.cu:484 on EVERY step: a state replaced by, or Kalman-averaged to, -10 earlier in the list is "empty", and the
    // literal step takes the next record as it is
    const bool empty = e == -10.0f;
    const float ov = (var <= 1e-4f) ? 1e-4f : var;
    const float den = ov + v, rc = div2_rcp(den);
    const float n1 = v * ov;
    const float n0 = ov * h + v * e; // gpu.cu:518 numerator, two roundings + one (no contraction)
    float qv, qe;
    div2_core(n1, n0, den, rc, qv, qe);
    const float d = fabsf(h - e), dd = d * d;
    const bool lo = dd < ov * 24.9995f, hi = dd > ov * 25.0005f, higher = e < h;
    const uint32_t u0 = __float_as_uint(n0) & 0x7fffffffu;
    const bool ok = (hi | (lo & num_ok(u0))) & !empty;
    take = lo | higher;
    e = lo ? qe : (higher ? h : e);
    var = lo ? qv : (higher ? v : ov); // an ignored lower point leaves the FLOORED variance behind (gpu.cu:500-501)
    return ok;
}
__device__ __forceinline__ bool plain_input(float h, float v)
{
    return h != -1.0f && (h == 0.0f || mag_ok(h)) && v >= 0x1p-40f && v < 0x1p20f;
}
__device__ __forceinline__ bool plain_state(float elev, float var)
{
    return elev != -10.0f && (elev == 0.0f || mag_ok(elev)) && ((var <= 1e-4f) ? 1e-4f : var) < 0x1p20f;
}

// 4-byte asynchronous copy global -> shared (no register holds the value in flight); cp.async.wait_all completes it
__device__ __forceinline__ void cp_async4(float *dst, const char *src)
{
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(src) : "memory");
}

// short lists (k <= 8): one thread per cell, records of chunk 0 held in registers, selection in index order.
// The cell's record, its lowest value (index from the mark) and all eight slots of chunk 0 (one 128-byte line; the
// slots beyond k hold stale bits and are masked) are requested together: one round trip after the mark.  The intensity
// of every record that may give the cell its colour is requested as soon as the records are there, into the thread's
// eight slots of s_int (s_int[e * ADD_BLOCK + threadIdx.x]), so it arrives under the fold instead of one round trip
// after it.  What counts besides those round trips is the instruction count: the plain step is tried first, the
// literal one only when a step leaves it.  Returns the list length (0 when the cell is k_fold_long's).
__device__ __forceinline__ int fold_small_cell(const MapGeom &g, const MapLayers &ml, const BinScratch &sc, const FoldSrc &src,
                                               const RegionOps &ro_next, int key, int low_idx, bool do_fuse, bool do_lowest,
                                               float *s_int)
{
    const uint4 *c0 = sc.chunk0 + (size_t)CHUNK0 * key;
    const int k = ml.cell[key].bin[sc.par].x;
    CellState s;
    cell_begin(s, g, ml, key, do_lowest, low_idx);
    uint4 rr[CHUNK0];
#pragma unroll
    for (int e = 0; e < CHUNK0; e++) rr[e] = c0[e];
    // k > 8: folded by a warp of k_fold_long.  k == 0: k_fold_long, which may run concurrently, has already folded the
    // cell and reset its counter -- a cell with a mark has at least one record until its owner resets it.  Either way
    // the cell is not this thread's: it must not even rewrite the state it loaded.
    if (k > CHUNK0 || k == 0) return 0;
#pragma unroll
    for (int e = 0; e < CHUNK0; e++) {
        if (e >= k) rr[e].x = 0x7fffffffu; // index padding: never selected
        if (e < k && do_fuse && src.base && (rr[e].w & REC_COLOUR_OK)) // lands in s_int without holding a register
            cp_async4(s_int + e * ADD_BLOCK + threadIdx.x, src.base + (size_t)rr[e].x * src.stride);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    const CellState s0 = s;
    const bool start_plain = do_fuse && plain_state(s.elev, s.var);
    bool plain = start_plain;
    for (int pass = 0; pass < 2; pass++) { // pass 0: plain steps; pass 1 (only if pass 0 left the plain path): literal
        int last = -1;
        for (int n = 0; n < k; n++) {
            int best = 0x7fffffff;
            uint4 b = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
            for (int e = 0; e < CHUNK0; e++) {
                const int ie = (int)rr[e].x;
                const bool c = ie > last && ie < best;
                if (c) { best = ie; b = rr[e]; }
            }
            last = best;
            const float h = __uint_as_float(b.y), v = __uint_as_float(b.z);
            lowest_step(s, h, v);
            if (plain) {
                bool take;
                plain = plain_input(h, v) && plain_step(s.elev, s.var, h, v, take);
                if (take && (b.w & REC_COLOUR_OK)) { s.src = b.x; s.rgb = b.w & 0xffffffu; s.ci_dirty = true; }
            } else {
                fold_step(s, h, v, b.w, b.x, 0.0f, do_fuse);
            }
        }
        if (pass == 0 && start_plain && !plain) { s = s0; continue; } // left the plain path: literal from the start
        break;
    }
    int se = 0;
#pragma unroll
    for (int e = 0; e < CHUNK0; e++) // the slot of the record the cell took its colour from (indices are unique)
        if (rr[e].x == s.src) se = e;
    asm volatile("cp.async.wait_all;" ::: "memory");
    s.inten = (src.base && s.ci_dirty) ? s_int[se * ADD_BLOCK + threadIdx.x] : 0.0f;
    cell_end(s, g, ml, sc, src, ro_next, key, do_fuse, do_lowest, true);
    return k;
}

constexpr int FOLD_KMAX = 1024;  // list length one warp sorts in shared memory
constexpr int FOLD_SLOT_BITS = 10; // sort key = (point index << 10) | rank: needs index < 2^22
constexpr int FOLD_INDEX_BITS = 32 - FOLD_SLOT_BITS; // = the largest launch (gem_create caps max_points)
constexpr int FOLD_RANK_K = 256; // lists up to this length are ordered by rank counting in shared memory

// order-preserving map float -> uint32 (for a warp min-reduction); -0 is folded onto +0
__device__ __forceinline__ uint32_t float_order_key(float f)
{
    const uint32_t u = __float_as_uint(f == 0.0f ? 0.0f : f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// The general path of fold_chunk: fold_step_fast on each of the chunk's m records.  Returns true (warp-uniform) when
// some step reported a rare case; s is then not fold_step's and the caller redoes the chunk from its saved state.
__device__ __forceinline__ bool fold_chunk_general(CellState &s, const uint4 r, int m)
{
    // broadcast record t+1 while record t is folded (in-order issue: keeps the shuffle latency off the serial chain)
    uint32_t nh = __shfl_sync(0xffffffffu, r.y, 0), nv = __shfl_sync(0xffffffffu, r.z, 0);
    uint32_t nc = __shfl_sync(0xffffffffu, r.w, 0), nx = __shfl_sync(0xffffffffu, r.x, 0);
    bool rare = false;
    for (int t = 0; t < m; t++) {
        const float h = __uint_as_float(nh), v = __uint_as_float(nv);
        const uint32_t rgb = nc, x = nx;
        const int tn = (t + 1) & 31;
        nh = __shfl_sync(0xffffffffu, r.y, tn);
        nv = __shfl_sync(0xffffffffu, r.z, tn);
        nc = __shfl_sync(0xffffffffu, r.w, tn);
        nx = __shfl_sync(0xffffffffu, r.x, tn);
        rare |= fold_step_fast(s, h, v, rgb, x, __uint_as_float(x));
    }
    return __any_sync(0xffffffffu, rare);
}

// Fold 32 records (one per lane, already in index order) into the cell state.  r = {x, h, var, rgb} where x is the
// record's intensity bits when the list's intensities were prefetched, else its point index (both views are carried:
// src = x, inten = bits of x; cell_end uses the valid one).
//
// A long list is ONE in-order warp walking it record by record (micro-benchmark scripts/micro_fold.cu: the general
// step below -- fold_step_fast, 85 instructions -- takes ~145 cycles per record on an otherwise idle SM).  Nearly every
// chunk of a long list is "plain": no record is skipped, the cell is not empty, no step is NEAR the 5-sigma gate, all
// magnitudes are ordinary.  Then a step is either the Kalman update (gpu.cu:517-529) or a clear gate decision
// (gpu.cu:504-516: replace by a higher point, ignore a lower one), and the step shrinks to the two quotient chains,
// one comparison and four selects (~35 instructions, ~90 cycles):
//   * magnitudes are tested once per chunk on the inputs (|h| in {0} U [2^-40, 2^20), var in [2^-40, 2^20), state
//     likewise): den = ov + v then lies in [2^-14, 2^21] and v*ov in [2^-54, 2^40], inside the ranges for which the
//     shared-reciprocal division is exact (div2_fast_ok); only the numerator ov*h + v*e, which can cancel, keeps its
//     per-step test;
//   * the gate is decided by comparing (h-e)^2 with 25 * ov as in gate_terms, but with a band of +-2e-5 that
//     plain_step leaves instead of evaluating the literal expression;
//   * the colour / intensity bookkeeping leaves the loop: a step takes the record's colour iff it is not an ignored
//     lower point, so the cell ends with the LAST taking record whose colour is valid (a bit mask, one clz).
// A chunk that is not plain, or leaves the plain path anywhere, is folded from its saved initial state by the
// general step (fold_step_fast), and if that reports a rare case, literally (fold_step): the result is always
// fold_step's, bit for bit.
__device__ __forceinline__ void fold_chunk(CellState &s, const uint4 r, int m, bool do_fuse)
{
    const unsigned lane = threadIdx.x & 31u;
    {   // lowest-scan of the chunk, off the serial chain: warp minimum of h, first lane attaining it
        // (lanes hold the records in index order), then the same strict-< update as lowest_step
        const uint32_t k = ((int)lane < m) ? float_order_key(__uint_as_float(r.y)) : 0xffffffffu;
        const uint32_t kmin = __reduce_min_sync(0xffffffffu, k);
        const int src = __ffs(__ballot_sync(0xffffffffu, k == kmin)) - 1;
        const float ch = __uint_as_float(__shfl_sync(0xffffffffu, r.y, src));
        const float cv = __uint_as_float(__shfl_sync(0xffffffffu, r.z, src));
        lowest_step(s, ch, cv);
    }
    if (!do_fuse) return;
    const CellState s0 = s;
    // ---- plain path ------------------------------------------------------------------------------------------------
    const bool lane_plain = ((int)lane >= m) || plain_input(__uint_as_float(r.y), __uint_as_float(r.z));
    const bool state_plain = plain_state(s.elev, s.var);
    if (__all_sync(0xffffffffu, lane_plain) && state_plain) {
        float e = s.elev, var = s.var;
        bool leave = false;
        unsigned takes = 0u;
        uint32_t nh = __shfl_sync(0xffffffffu, r.y, 0), nv = __shfl_sync(0xffffffffu, r.z, 0);
        for (int t = 0; t < m; t++) {
            const float h = __uint_as_float(nh), v = __uint_as_float(nv);
            const int tn = (t + 1) & 31;
            nh = __shfl_sync(0xffffffffu, r.y, tn);
            nv = __shfl_sync(0xffffffffu, r.z, tn);
            bool take;
            leave |= !plain_step(e, var, h, v, take); // off the serial chain: nothing reads `leave` before the end of the chunk
            takes |= (take ? 1u : 0u) << t;
        }
        if (!__any_sync(0xffffffffu, leave)) {
            s.elev = e;
            s.var = var;
            const unsigned cm = __ballot_sync(0xffffffffu, (int)lane < m && (r.w & REC_COLOUR_OK) != 0u) & takes;
            if (cm) { // the last taking record with a valid colour
                const int last = 31 - __clz((int)cm);
                const uint32_t x = __shfl_sync(0xffffffffu, r.x, last);
                s.src = x;
                s.inten = __uint_as_float(x);
                s.rgb = __shfl_sync(0xffffffffu, r.w, last) & 0xffffffu;
                s.ci_dirty = true;
            }
            return;
        }
        s = s0;
    }
    // ---- general path ----------------------------------------------------------------------------------------------
    if (fold_chunk_general(s, r, m)) { // some step left the common path: redo the chunk literally
        s = s0;
        for (int t = 0; t < m; t++) {
            const float h = __uint_as_float(__shfl_sync(0xffffffffu, r.y, t)), v = __uint_as_float(__shfl_sync(0xffffffffu, r.z, t));
            const uint32_t rgb = __shfl_sync(0xffffffffu, r.w, t), x = __shfl_sync(0xffffffffu, r.x, t);
            fold_step(s, h, v, rgb, x, __uint_as_float(x), true);
        }
    }
}

// chunk pointers of one cell, warp-uniform
struct ChunkRefs {
    int key;  // level 0: chunk0 + 8 * key
    int i8;   // level 1: pool1 + 33 * i8
    int p[5]; // pool offsets of levels 2..4 in p[2..4] (ranks < 2728); deeper levels are walked
};
__device__ __forceinline__ uint4 *chunk1(const BinScratch &sc, const ChunkRefs &c) { return sc.pool1 + (size_t)CHUNK1_SLOTS * c.i8; }
__device__ __forceinline__ const uint4 *record_ptr(const BinScratch &sc, const ChunkRefs &c, int rank)
{
    if (rank < CHUNK0) return sc.chunk0 + (size_t)CHUNK0 * c.key + rank;
    if (rank < level_base(2)) return chunk1(sc, c) + 1 + (rank - level_base(1));
    if (rank < level_base(3)) return sc.pool + c.p[2] + 1 + (rank - level_base(2));
    if (rank < level_base(4)) return sc.pool + c.p[3] + 1 + (rank - level_base(3));
    if (rank < level_base(5)) return sc.pool + c.p[4] + 1 + (rank - level_base(4));
    int j = 5, q = next_chunk(sc.pool + c.p[4]); // very long lists: walk the chain
    while (rank >= level_base(j + 1)) { q = next_chunk(sc.pool + q); j++; }
    return sc.pool + q + 1 + (rank - level_base(j));
}

// Warp-wide bitonic sort of 32*R keys held in registers: element i lives in lane i%32, register i/32.  Partners
// less than 32 apart are exchanged with one shuffle, the rest are in the same lane.  (A shared-memory network needs a
// store, a barrier and a load per stage; a shuffle stage needs none of them.)
template <int R>
__device__ __forceinline__ void warp_bitonic(uint32_t (&key)[R], unsigned lane)
{
#pragma unroll
    for (int size = 2; size <= 32 * R; size <<= 1) {
#pragma unroll
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            if (stride >= 32) {
                const int rs = stride >> 5;
#pragma unroll
                for (int r = 0; r < R; r++) {
                    if ((r & rs) == 0) {
                        const uint32_t a = key[r], b2 = key[r | rs];
                        const bool up = (((int)lane + 32 * r) & size) == 0;
                        const bool sw = (a > b2) == up;
                        key[r] = sw ? b2 : a;
                        key[r | rs] = sw ? a : b2;
                    }
                }
            } else {
#pragma unroll
                for (int r = 0; r < R; r++) {
                    const uint32_t a = key[r];
                    const uint32_t o = __shfl_xor_sync(0xffffffffu, a, stride);
                    const bool up = (((int)lane + 32 * r) & size) == 0;
                    const bool lower = ((int)lane & stride) == 0;
                    const uint32_t mn = min(a, o), mx = max(a, o);
                    key[r] = (lower == up) ? mn : mx;
                }
            }
        }
    }
}

// per-warp shared scratch of k_fold_long
struct WarpScratch {
    uint4 rec[FOLD_RANK_K];          // the records of a list of <= 256 (or the sort keys of a list of <= 1024)
    uint32_t idx[FOLD_RANK_K];       // their point indices, compact (read four at a time by the rank count)
    unsigned char perm[FOLD_RANK_K]; // position in index order -> rank
};

constexpr int FOLD_ROWS = 8; // 32-record rows a list may occupy in registers

// one warp folds one cell with more than 8 records.  info = the cell's queue entry {key, LIST_LARGE | LIST_LONG, i8, p2}.
// Returns the list length (0: not this entry's job).
//   k <= 256: the records are read ONCE, coalesced in rank order, into shared memory; the intensity of every record
//     is requested from the input as soon as the records are there (it arrives under the ordering work); every lane
//     counts, for each of its records, how many records of the list carry a smaller point index (16-byte broadcast
//     reads of the compact index array) -- that count is the record's position in G_fuse's visiting order;
//   k <= 1024: bitonic sort of packed (index, rank) keys in shared memory, records gathered per chunk;
//   longer: repeated selection of the next smallest index from global memory.
__device__ __noinline__ int fold_cell_warp(const MapGeom &g, const MapLayers &ml, const BinScratch &sc, const FoldSrc &src,
                                           const RegionOps &ro_next, bool do_fuse, bool do_lowest, WarpScratch &ws, int4 info)
{
    constexpr int ROWS = FOLD_ROWS;
    const unsigned lane = threadIdx.x & 31u;
    const bool from_long = info.y == LIST_LONG;
    const int key = info.x;
    ChunkRefs c;
    c.key = key; c.i8 = info.z; c.p[0] = 0; c.p[1] = 0; c.p[2] = info.w; c.p[3] = 0; c.p[4] = 0;
    const unsigned long long t0 = (sc.stamps && from_long) ? globaltimer_ns() : 0ull;
    // where the first 40 slots are follows from the entry alone (chunk0 by key, the second chunk by the index of the
    // rank-8 point), and so does the header of a long list's level-2 chunk: all are requested together with the cell
    // instead of one round trip later.  The slots beyond the list length hold stale bits and are masked once the length
    // has arrived; the header is used only by lists that have a level-3 chunk (pool offset 0, where a LARGE entry's p2
    // points, is never handed out and reads as zeros)
    const uint4 spec0 = *record_ptr(sc, c, (int)lane);
    uint4 spec1 = make_uint4(0u, 0u, 0u, 0u);
    if (lane < (unsigned)(FOLD_LONG_FROM - 32)) spec1 = *record_ptr(sc, c, (int)lane + 32);
    const int p3 = next_chunk(sc.pool + c.p[2]);
    const int k = ml.cell[key].bin[sc.par].x;
    CellState s;
    cell_begin(s, g, ml, key, do_lowest);
    // a LARGE entry whose cell also reached rank 40 is folded by its LONG entry; its counter reads > 40, or 0 once that
    // entry is done with it
    if (!from_long && (k > FOLD_LONG_FROM || k == 0)) return 0;
    if (k > 0) stamp_since(sc, 3, t0); // list length arrived
    if (k > level_base(3)) c.p[3] = p3;
    if (k > level_base(4)) c.p[4] = next_chunk(sc.pool + c.p[3]);
    bool have_inten = false;
    uint32_t *s_key = reinterpret_cast<uint32_t *>(ws.rec);
    if (k <= 32 * ROWS) {
        have_inten = true;
        const int rows = (k + 31) >> 5;
        uint4 rec[ROWS];
#pragma unroll
        for (int r = 0; r < ROWS; r++) { // all record loads first ...
            const int e = (int)lane + 32 * r;
            rec[r] = make_uint4(0x7fffffffu, 0u, 0u, 0u); // index padding: never smaller than a real index
            if (r < rows && e < k) rec[r] = (e < FOLD_LONG_FROM) ? (r == 0 ? spec0 : spec1) : *record_ptr(sc, c, e);
        }
        float it[ROWS];
#pragma unroll
        for (int r = 0; r < ROWS; r++) { // ... then the intensity requests, which depend on them
            const int e = (int)lane + 32 * r;
            it[r] = 0.0f;
            if (r < rows) {
                if (e < k && do_fuse && (rec[r].w & REC_COLOUR_OK)) it[r] = fetch_intensity(src, rec[r].x);
                ws.idx[e] = rec[r].x; // rows * 32 entries: the tail beyond k reads as 0x7fffffff (never smaller)
            }
        }
        __syncwarp();
        if (rec[0].y != 0x7fc12345u) stamp_since(sc, 4, t0); // records arrived, indices in shared memory
        if (k <= 64) {
            // position of a record = number of records with a smaller point index.  Indices are < 2^22 and the padding
            // is 0x7fffffff, so (x - mine) >> 31 is exactly [x < mine]: three independent instructions per comparison
            const int k4 = (k + 3) >> 2;
            const uint32_t m0 = rec[0].x, m1 = rec[1].x;
            uint32_t p0 = 0u, p1 = 0u;
            for (int q = 0; q < k4; q++) {
                const uint4 x = reinterpret_cast<const uint4 *>(ws.idx)[q];
                p0 += ((x.x - m0) >> 31) + ((x.y - m0) >> 31) + ((x.z - m0) >> 31) + ((x.w - m0) >> 31);
                p1 += ((x.x - m1) >> 31) + ((x.y - m1) >> 31) + ((x.z - m1) >> 31) + ((x.w - m1) >> 31);
            }
            if ((int)lane < k) ws.perm[p0] = (unsigned char)lane;
            if ((int)lane + 32 < k) ws.perm[p1] = (unsigned char)(lane + 32);
        } else {
            // register bitonic network on (index << 10 | rank) keys; the padding sorts last
            uint32_t key8[ROWS];
#pragma unroll
            for (int r = 0; r < 8; r++) key8[r] = 0xffffffffu;
#pragma unroll
            for (int r = 0; r < ROWS; r++) {
                const int e = (int)lane + 32 * r;
                key8[r] = (r < rows && e < k) ? ((rec[r].x << FOLD_SLOT_BITS) | (uint32_t)e) : 0xffffffffu;
            }
            if (k <= 128) {
                uint32_t key4[4] = {key8[0], key8[1], key8[2], key8[3]};
                warp_bitonic<4>(key4, lane);
#pragma unroll
                for (int r = 0; r < 4; r++) ws.perm[lane + 32 * r] = (unsigned char)(key4[r] & 255u);
            } else {
                warp_bitonic<8>(key8, lane);
#pragma unroll
                for (int r = 0; r < 8; r++) ws.perm[lane + 32 * r] = (unsigned char)(key8[r] & 255u);
            }
        }
        if (rec[0].y != 0x7fc12346u) stamp_since(sc, 7, t0); // order known
#pragma unroll
        for (int r = 0; r < ROWS; r++) {
            const int e = (int)lane + 32 * r;
            if (r < rows && e < k) {
                rec[r].x = __float_as_uint(it[r]); // the index has done its job: the slot now carries the intensity
                ws.rec[e] = rec[r];
            }
        }
        __syncwarp();
        stamp_since(sc, 5, t0); // ordered, intensities in place
    } else if (k <= FOLD_KMAX) {
        int P = 512;
        while (P < k) P <<= 1;
        for (int e = (int)lane; e < P; e += 32)
            s_key[e] = (e < k) ? ((record_ptr(sc, c, e)->x << FOLD_SLOT_BITS) | (uint32_t)e) : 0xffffffffu;
        __syncwarp();
        for (int size = 2; size <= P; size <<= 1) {
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                for (int i = (int)lane; i < (P >> 1); i += 32) {
                    const int lo = ((i & ~(stride - 1)) << 1) | (i & (stride - 1));
                    const int hi = lo + stride;
                    const uint32_t a = s_key[lo], b2 = s_key[hi];
                    const bool up = (lo & size) == 0;
                    if ((a > b2) == up) { s_key[lo] = b2; s_key[hi] = a; }
                }
                __syncwarp();
            }
        }
    }
    if (k <= FOLD_KMAX) { // the one chunk loop of the kernel (order the records by point index == G_fuse's visiting order)
        for (int c0 = 0; c0 < k; c0 += 32) {
            uint4 r = make_uint4(0u, 0u, 0u, 0u);
            if (c0 + (int)lane < k) {
                if (k <= 32 * ROWS) r = ws.rec[ws.perm[c0 + lane]];
                else r = *record_ptr(sc, c, (int)(s_key[c0 + lane] & ((1u << FOLD_SLOT_BITS) - 1u)));
            }
            fold_chunk(s, r, min(32, k - c0), do_fuse);
        }
        __syncwarp(); // the scratch is reused by this warp's next cell
    } else {
        uint32_t last = 0;
        bool have_last = false;
        for (int it = 0; it < k; it++) {
            uint32_t best = 0xffffffffu;
            int beste = -1;
            for (int e = (int)lane; e < k; e += 32) {
                const uint32_t v = record_ptr(sc, c, e)->x;
                if ((!have_last || v > last) && v < best) { best = v; beste = e; }
            }
            const uint32_t wbest = __reduce_min_sync(0xffffffffu, best);
            const unsigned who = __ballot_sync(0xffffffffu, best == wbest && beste >= 0);
            const int srcl = __ffs(who) - 1;
            const int e = __shfl_sync(0xffffffffu, beste, srcl);
            const uint4 r = *record_ptr(sc, c, e);
            lowest_step(s, __uint_as_float(r.y), __uint_as_float(r.z));
            fold_step(s, __uint_as_float(r.y), __uint_as_float(r.z), r.w, r.x, 0.0f, do_fuse);
            last = wbest;
            have_last = true;
        }
    }
    if (s.elev != 12345.678f) stamp_since(sc, 6, t0); // folded
    stamp_lane0(sc, 12, from_long && s.elev != 12345.678f);  // latest list of > 40 folded
    stamp_lane0(sc, 14, !from_long && s.elev != 12345.678f); // latest list of 9..40 folded
    if (lane == 0u) {
        cell_end(s, g, ml, sc, src, ro_next, key, do_fuse, do_lowest, have_inten);
        if (k > FOLD_LONG_FROM) { // clear the headers this list's chunks published (every chunk but the last): no stale tags
            uint4 *q = chunk1(sc, c);
            for (int l = 2; k > level_base(l); l++) {
                unsigned long long *hd = chunk_header(q);
                q = sc.pool + next_chunk(q);
                *hd = 0ull;
            }
        }
    }
    return k;
}

constexpr int FOLD_MARKS = 2; // marks per thread and pass: a block's slice is FOLD_MARKS * blockDim.x consecutive points

// k_fold: the cells with at most 8 records.  One block folds the cells whose marks lie in its slices of the point index
// range.  The marks of a slice are read coalesced and the touched cells queued in shared memory; the warps draw them 32
// at a time, one per thread (a cell with more records is skipped: k_fold_long folds it).  fold_blocks blocks fold;
// blocks beyond them execute `ro` (row / column clears of the NEXT call's Move, pipelined mode only: a cell inside such
// a region is written with the cleared value by whoever touches it, see cell_end).
__global__ void __launch_bounds__(ADD_BLOCK, 3)
k_fold(MapGeom g, MapLayers ml, BinScratch sc, FoldSrc src, const __grid_constant__ RegionOps ro, int n, int fold_blocks, int slice, int do_fuse_i, int do_lowest_i,
       const int *n_dev)
{
    if (n_dev) n = min(n, *n_dev); // tiled maps and pre-filtered adds: the number of marks is known on the device only
    extern __shared__ __align__(16) unsigned char s_dyn[]; // FOLD_SMEM_BYTES: the queue, the intensities (+ padding, see k_fold_long)
    int2 *s_first = reinterpret_cast<int2 *>(s_dyn);
    float *s_int = reinterpret_cast<float *>(s_first + FOLD_MARKS * ADD_BLOCK);
    __shared__ int s_nfirst, s_next_first, s_stat[3];
    if ((int)blockIdx.x >= fold_blocks) {
        const size_t rb = gridDim.x - fold_blocks;
        phase_regions(g, ml, ro, (size_t)(blockIdx.x - fold_blocks) * blockDim.x + threadIdx.x, rb * blockDim.x);
        return;
    }
    const bool do_fuse = do_fuse_i != 0, do_lowest = do_lowest_i != 0;
    const int w = threadIdx.x >> 5;
    const unsigned lane = threadIdx.x & 31u;
    stamp_start(sc, 8);
    if (threadIdx.x == 0) { s_stat[0] = 0; s_stat[1] = 0; s_stat[2] = 0; }
    // slice = points per block and pass (<= FOLD_MARKS * ADD_BLOCK, chosen by the host so that one pass covers a frame-sized call)
    for (int base = blockIdx.x * slice; base < n; base += fold_blocks * slice) {
        if (threadIdx.x == 0) { s_nfirst = 0; s_next_first = 0; }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < FOLD_MARKS; u++) {
            const int o = u * ADD_BLOCK + threadIdx.x, i = base + o;
            int2 mk = make_int2(-1, 0);
            if (o < slice && i < n) mk = sc.mark[i];
            const unsigned fm = __ballot_sync(0xffffffffu, mk.x >= 0);
            if (fm) { // warp-aggregated append of the touched cells {key, lowest index}
                int fb = 0;
                if (lane == 0u) fb = atomicAdd(&s_nfirst, __popc(fm));
                fb = __shfl_sync(0xffffffffu, fb, 0);
                if (mk.x >= 0) s_first[fb + __popc(fm & ((1u << lane) - 1u))] = mk;
            }
        }
        __syncthreads();
        const int nfirst = s_nfirst;
        stamp_mark(sc, 9); // marks of the slice read and queued
        int tk = 0, tsum = 0;
        for (;;) { // 32 cells per warp and draw, one per thread
            int j = 0;
            if (lane == 0u) j = atomicAdd(&s_next_first, 32);
            j = __shfl_sync(0xffffffffu, j, 0);
            if (j >= nfirst) break;
            if (j + (int)lane < nfirst) {
                const int2 c = s_first[j + lane];
                const int k = fold_small_cell(g, ml, sc, src, ro, c.x, c.y, do_fuse, do_lowest, s_int);
                tk = max(tk, k);
                tsum += k;
            }
        }
        stamp_mark(sc, 13); // the block's first warp has no cell left
        // statistics: points binned, longest list (cells touched = nfirst)
        int tmax = tk;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            tsum += __shfl_xor_sync(0xffffffffu, tsum, d);
            tmax = max(tmax, __shfl_xor_sync(0xffffffffu, tmax, d));
        }
        if (lane == 0u) {
            if (tsum) atomicAdd(&s_stat[1], tsum);
            atomicMax(&s_stat[2], tmax);
            if (w == 0) s_stat[0] += nfirst;
        }
        __syncthreads(); // the queue is reset by the next pass
    }
    if (threadIdx.x == 0) { // three reductions per block, no return value
        if (s_stat[0]) atomicAdd(&sc.ctr->ntouched, s_stat[0]);
        if (s_stat[1]) atomicAdd(&sc.ctr->total, s_stat[1]);
        if (s_stat[2]) atomicMax(&sc.ctr->maxk, s_stat[2]);
    }
    stamp_mark(sc, 10);
}
constexpr size_t FOLD_SMEM_USED = (size_t)FOLD_MARKS * ADD_BLOCK * sizeof(int2) + (size_t)CHUNK0 * ADD_BLOCK * sizeof(float);

// k_fold_long: the cells with more than 8 records, drawn from the two queues the bin kernel filled (one atomic per cell
// and queue, a few hundred per frame): the cells with more than 40 records first, so that the longest lists start
// first, then those with more than 8 (a cell on both queues is folded by its first entry).  A list is a serial chain of
// dependent steps per record, several times slower next to busy warps than with a scheduler to itself
// (scripts/micro_fold.cu measures both) -- and the longest list of a frame IS the latency of the fold.  So the lists
// get warps of their own, away from k_fold's short-list selection loops: blocks of four warps (one per scheduler).  With GEM_B200_EXCLUSIVE=1 they get SMs of their own as well: each block asks for so
// much shared memory (LONG_SMEM_BYTES, mostly unused) that no other block of this or a concurrently running kernel fits
// beside it (k_fold and k_bin then ask for at least BIN_SMEM_BYTES for exactly this reason).
constexpr int LONG_BLOCK = 128;
constexpr int LONG_BLOCKS = 32;
constexpr size_t LONG_SMEM_BYTES = 200 * 1024;
constexpr size_t BIN_SMEM_BYTES = 28 * 1024; // > 227 KB - LONG_SMEM_BYTES: keeps k_bin's blocks off k_fold_long's SMs
constexpr size_t FOLD_SMEM_BYTES = FOLD_SMEM_USED > BIN_SMEM_BYTES ? FOLD_SMEM_USED : BIN_SMEM_BYTES; // likewise k_fold's
__global__ void __launch_bounds__(LONG_BLOCK, 1)
k_fold_long(MapGeom g, MapLayers ml, BinScratch sc, FoldSrc src, const __grid_constant__ RegionOps ro, int do_fuse_i, int do_lowest_i)
{
    extern __shared__ __align__(16) unsigned char s_dyn[];
    WarpScratch *s_ws = reinterpret_cast<WarpScratch *>(s_dyn);
    const int w = threadIdx.x >> 5;
    const unsigned lane = threadIdx.x & 31u;
    const int nlong = sc.ctr->nlong, nall = nlong + sc.ctr->nlarge;
    int wk = 0, wtot = 0;
    for (;;) {
        int j = 0;
        if (lane == 0u) j = atomicAdd(&sc.ctr->next_long, 1);
        j = __shfl_sync(0xffffffffu, j, 0);
        if (j >= nall) break;
        const int4 info = (j < nlong) ? sc.tlong[j] : sc.tlarge[j - nlong];
        const int k = fold_cell_warp(g, ml, sc, src, ro, do_fuse_i != 0, do_lowest_i != 0, s_ws[w], info);
        wk = max(wk, k);
        wtot += k;
    }
    if (lane == 0u && wtot) { // the short-list statistics come from k_fold (these cells' marks count them as touched)
        atomicAdd(&sc.ctr->total, wtot);
        atomicMax(&sc.ctr->maxk, wk);
    }
}

} // namespace gem
