// gem_route.cuh -- point routing for spatially tiled maps (SURVEY.md 8e, BASELINE configs 4/5).
//
// The reference is single-GPU; a map that outgrows one GPU is cut into geographic tiles, one
// per rank.  Every rank transforms its share of the input, buckets the accepted in-grid
// points STABLY by owning tile, and the host side exchanges the buckets with one NCCL
// all-to-all (gem_b200/tiled.py).  Concatenating received buckets in (source rank, source
// order) reproduces the global point order, so the tiled result is bit-identical to the
// single-GPU result on the concatenated cloud.
#pragma once
#include "gem_add.cuh"

namespace gem {

constexpr int ROUTE_MAX_OWNERS = 64;
constexpr int ROUTE_BLOCK = 256;

// pass 1: transform, owner id, per-block owner histogram.  ANY: every sensor model (k_route_count_any)
template <bool ANY>
__device__ __forceinline__ void route_count(const MapGeom &g, const FrameParams &f, const float4 *xyzi, int n, int tile_h, int tile_w,
                                            int tiles_c, int n_owners, int *owner_out, int *gkey_out, float *h_out, float *hv_out,
                                            int *blockCounts)
{
    __shared__ int s_cnt[ROUTE_MAX_OWNERS];
    for (int o = threadIdx.x; o < n_owners; o += blockDim.x) s_cnt[o] = 0;
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    int owner = -1;
    if (i < n) {
        const float4 p = ld_stream_f4(xyzi + i);
        const PtRes r = transform_point<ANY>(g, f, p.x, p.y, p.z, i);
        int gkey = -1;
        if (r.ingrid) {
            owner = (r.gx / tile_h) * tiles_c + (r.gy / tile_w);
            gkey = r.gx * g.L + r.gy;
        }
        owner_out[i] = owner;
        gkey_out[i] = gkey;
        h_out[i] = r.h;
        hv_out[i] = r.hv;
    }
    if (owner >= 0) atomicAdd(&s_cnt[owner], 1);
    __syncthreads();
    for (int o = threadIdx.x; o < n_owners; o += blockDim.x) blockCounts[o * gridDim.x + blockIdx.x] = s_cnt[o];
}
__global__ void __launch_bounds__(ROUTE_BLOCK)
k_route_count(MapGeom g, FrameParams f, const float4 *xyzi, int n, int tile_h, int tile_w, int tiles_c,
              int n_owners, int *owner_out, int *gkey_out, float *h_out, float *hv_out, int *blockCounts /* [owners][blocks] */)
{
    route_count<false>(g, f, xyzi, n, tile_h, tile_w, tiles_c, n_owners, owner_out, gkey_out, h_out, hv_out, blockCounts);
}
__global__ void __launch_bounds__(ROUTE_BLOCK)
k_route_count_any(MapGeom g, FrameParams f, const float4 *xyzi, int n, int tile_h, int tile_w, int tiles_c,
                  int n_owners, int *owner_out, int *gkey_out, float *h_out, float *hv_out, int *blockCounts)
{
    route_count<true>(g, f, xyzi, n, tile_h, tile_w, tiles_c, n_owners, owner_out, gkey_out, h_out, hv_out, blockCounts);
}

// pass 2: one block scans blockCounts owner-major -> exclusive offsets; owner totals
__global__ void __launch_bounds__(1024) k_route_scan(int *blockCounts, int n_owners, int nblocks, int *counts_out)
{
    __shared__ int s_part[1024];
    __shared__ int s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    const int total = n_owners * nblocks;
    for (int base = 0; base < total; base += 1024) {
        const int idx = base + threadIdx.x;
        const int v = idx < total ? blockCounts[idx] : 0;
        s_part[threadIdx.x] = v;
        __syncthreads();
        for (int d = 1; d < 1024; d <<= 1) { // Hillis-Steele inclusive scan
            const int t = threadIdx.x >= d ? s_part[threadIdx.x - d] : 0;
            __syncthreads();
            s_part[threadIdx.x] += t;
            __syncthreads();
        }
        const int incl = s_part[threadIdx.x] + s_carry;
        if (idx < total) blockCounts[idx] = incl - v; // exclusive, global over (owner, block)
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = incl;
        __syncthreads();
    }
    // owner totals from consecutive owner starts
    __syncthreads();
    for (int o = threadIdx.x; o < n_owners; o += blockDim.x) {
        const int begin = blockCounts[o * nblocks];
        const int end = (o + 1 < n_owners) ? blockCounts[(o + 1) * nblocks] : s_carry;
        counts_out[o] = end - begin;
    }
}

// pass 3: stable in-block rank and record write
__global__ void __launch_bounds__(ROUTE_BLOCK)
k_route_write(const float4 *xyzi, const uchar4 *rgba, int n, int n_owners, const int *owner_in, const int *gkey_in,
              const float *h_in, const float *hv_in, const int *blockOffsets, RouteRec *out, int bucket_stride)
{
    __shared__ int s_wcnt[ROUTE_BLOCK / 32][ROUTE_MAX_OWNERS];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned lane = threadIdx.x & 31u;
    const int w = threadIdx.x >> 5;
    for (int o = (int)lane; o < n_owners; o += 32) s_wcnt[w][o] = 0;
    __syncwarp();
    const int owner = (i < n) ? owner_in[i] : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, owner);
    const int rank_in_warp = __popc(peers & ((1u << lane) - 1u));
    if (owner >= 0 && rank_in_warp == 0) s_wcnt[w][owner] = __popc(peers);
    __syncthreads();
    if (owner >= 0) {
        int before = 0;
        for (int ww = 0; ww < w; ww++) before += s_wcnt[ww][owner];
        int pos = blockOffsets[owner * gridDim.x + blockIdx.x] + before + rank_in_warp;
        // fixed-stride layout: bucket o starts at o*stride (padded all-to-all, no host-side split sizes)
        if (bucket_stride > 0) pos = pos - blockOffsets[owner * gridDim.x] + owner * bucket_stride;
        RouteRec r;
        r.gkey = gkey_in[i];
        r.h = h_in[i];
        r.var = hv_in[i];
        r.rgb = 0u;
        if (rgba) {
            const uchar4 c = rgba[i];
            r.rgb = pack_rgb(c.x, c.y, c.z);
        }
        r.intensity = xyzi[i].w;
        out[pos] = r;
    }
}

// per-point scratch of the routing passes
struct RouteScratch {
    int *owner, *gkey;
    float *h, *hv;
    int *blockCounts; // [owners][blocks]
    size_t blockCounts_capacity;
};
inline cudaError_t route_points(cudaStream_t st, const MapGeom &g, const FrameParams &fp, const float4 *xyzi,
                                const uchar4 *rgba, int n, int tiles_r, int tiles_c, const RouteScratch &sc,
                                RouteRec *out, int *counts_out, int bucket_stride)
{
    const int n_owners = tiles_r * tiles_c;
    const int nblocks = n > 0 ? (n + ROUTE_BLOCK - 1) / ROUTE_BLOCK : 1;
    if ((size_t)n_owners * nblocks > sc.blockCounts_capacity) return cudaErrorInvalidValue;
    const int tile_h = (g.L + tiles_r - 1) / tiles_r, tile_w = (g.L + tiles_c - 1) / tiles_c;
    (any_model(fp) ? k_route_count_any : k_route_count)<<<nblocks, ROUTE_BLOCK, 0, st>>>(
        g, fp, xyzi, n, tile_h, tile_w, tiles_c, n_owners, sc.owner, sc.gkey, sc.h, sc.hv, sc.blockCounts);
    k_route_scan<<<1, 1024, 0, st>>>(sc.blockCounts, n_owners, nblocks, counts_out);
    k_route_write<<<nblocks, ROUTE_BLOCK, 0, st>>>(xyzi, rgba, n, n_owners, sc.owner, sc.gkey, sc.h, sc.hv, sc.blockCounts, out, bucket_stride);
    return cudaGetLastError();
}

// =========================================================================================
// Peer path, round 2: route + exchange in ONE kernel, no collective library, no barrier kernel.
//
//   k_route_peer   (source rank r)  1 thread/point: transform, owner tile, stable position inside the block's
//                  sub-bucket, record stored straight into the owner's receive buffer over NVLink; every block also
//                  stores its per-owner count; the last block to finish raises this rank's flag on every peer
//   k_bin_peer     (owner rank)     one wave of blocks over the (source rank, source block) sub-buckets of 256 slots: waits
//                  for all peers' flags of this step, skips empty sub-buckets, bins the received records like k_bin does
//
// Determinism: rank r's block b owns slots [(r * nblk + b) * 256, +256) of every owner's buffer, filled in source
// order without a cross-block scan.  The slot index is monotone in (source rank, source point index), and it is the
// slot index that the fold sorts a cell's records by -- so the tiled map equals the single-GPU map of the rank-by-rank
// concatenated clouds bit for bit, although the buffer has holes.  The work list (marks) is dense and in no particular
// order (the fold's result does not depend on which thread folds a cell): a sub-bucket takes its range with one atomic.
// Step pipeline (gem_api.cu, gem_tiled_step).  Default, depth 2: the graph of call j runs {folds of step j-1 || route ->
// bin of step j}.  Depth 3 (GEM_B200_TILED_DEPTH=3, measured slower, kept as a switch): {folds of step j-2 || bin of step
// j-1 || route of step j}, all four kernels independent.
// Receive buffers: PEER_BUFS = 5 by step, sized for depth 3.  There peer p's route of step k+5 rewrites this rank's buffer
// k % 5, which this rank's fold of step k reads (intensities) in its graph k+2.  p's graph k+5 starts after p's graph k+4,
// whose bin of step k+3 waited for this rank's flag k+3, raised by this rank's route in ITS graph k+3, which started after
// its graph k+2 had completed.  (Four buffers would not do: flag k+2 is raised inside the very graph k+2 that still folds
// step k.)  Depth 2 needs three: the fold of step k runs in graph k+1; p's route of step k+3 follows p's bin of step k+2,
// which waited for this rank's flag k+2, raised in its graph k+2, i.e. after its graph k+1.
// =========================================================================================
constexpr int PEER_BUFS = 5;
struct PeerBufs { // device addresses valid on THIS device (own memory or peer mappings), per rank
    unsigned long long rec[ROUTE_MAX_OWNERS];   // uint4 [PEER_BUFS][world * cap]  {gkey, h, var, rgb}
    unsigned long long inten[ROUTE_MAX_OWNERS]; // float [PEER_BUFS][world * cap]
    unsigned long long cnt[ROUTE_MAX_OWNERS];   // int   [PEER_BUFS][world * nblk]
    unsigned long long flag[ROUTE_MAX_OWNERS];  // int   [world]: flag[o][r] = last step rank r has delivered to rank o
};

template <bool ANY>
__device__ __forceinline__ void route_peer(const MapGeom &g, const FrameParams &f, const float4 *xyzi, const uchar4 *rgba, int n, int tile_h,
                                           int tile_w, int tiles_c, int world, int my_rank, int nblk, int cap, int buf, int step,
                                           const PeerBufs &pb, int *ticket)
{
    __shared__ int s_wcnt[ROUTE_BLOCK / 32][ROUTE_MAX_OWNERS];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned lane = threadIdx.x & 31u;
    const int w = threadIdx.x >> 5;
    for (int o = (int)lane; o < world; o += 32) s_wcnt[w][o] = 0;
    __syncwarp();
    int owner = -1, gkey = -1;
    float h = 0.0f, hv = 0.0f, inten = 0.0f;
    uint32_t rgb = 0u;
    if (i < n) {
        const float4 p = ld_stream_f4(xyzi + i);
        const PtRes r = transform_point<ANY>(g, f, p.x, p.y, p.z, i);
        if (r.ingrid) {
            owner = (r.gx / tile_h) * tiles_c + (r.gy / tile_w);
            gkey = r.gx * g.L + r.gy;
            h = r.h; hv = r.hv; inten = p.w;
            if (rgba) { const uchar4 c = rgba[i]; rgb = pack_rgb(c.x, c.y, c.z); }
        }
    }
    const unsigned peers = __match_any_sync(0xffffffffu, owner);
    const int rank_in_warp = __popc(peers & ((1u << lane) - 1u));
    if (owner >= 0 && rank_in_warp == 0) s_wcnt[w][owner] = __popc(peers);
    __syncthreads();
    const size_t sub = (size_t)my_rank * nblk + blockIdx.x; // this block's sub-bucket in every owner's buffer
    if (owner >= 0) {
        int before = 0;
        for (int ww = 0; ww < w; ww++) before += s_wcnt[ww][owner];
        const size_t slot = (size_t)buf * world * cap + sub * ROUTE_BLOCK + before + rank_in_warp;
        reinterpret_cast<uint4 *>(pb.rec[owner])[slot] = make_uint4((uint32_t)gkey, __float_as_uint(h), __float_as_uint(hv), rgb); // NVLink
        reinterpret_cast<float *>(pb.inten[owner])[slot] = inten;
    }
    if ((int)threadIdx.x < world) { // this block's count for every owner (zero included: the owner must not read a stale one)
        int tot = 0;
        for (int ww = 0; ww < ROUTE_BLOCK / 32; ww++) tot += s_wcnt[ww][threadIdx.x];
        reinterpret_cast<int *>(pb.cnt[threadIdx.x])[(size_t)buf * world * nblk + sub] = tot;
    }
    // Visibility chain (PTX memory model; causality order composes across scopes):
    //   the block's peer stores -> barrier -> thread 0: fence at GPU scope -> ticket atomic            (every block)
    //   last block: ticket atomic (observes all others) -> ONE fence at system scope -> flag stores (relaxed.sys: fence + store = release)
    //   owner: flag load (acquire.sys) -> record loads.
    // A system-scope fence per block cost 44 % of this kernel's and k_bin_peer's stall samples together (MEMBAR.SYS drains
    // to every memory the SM could have written; profiles/r2_tiled_world1_kernels_full.txt: 17.4 us), one per thread twice that.
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("fence.acq_rel.gpu;" ::: "memory");
        const int t = atomicAdd(ticket, 1);
        if (t == (int)gridDim.x - 1) { // last block of this rank: everything is on its way -> raise the flag on every peer
            *ticket = 0;
            asm volatile("fence.acq_rel.sys;" ::: "memory");
            for (int o = 0; o < world; o++)
                asm volatile("st.relaxed.sys.global.s32 [%0], %1;" ::"l"(reinterpret_cast<int *>(pb.flag[o]) + my_rank), "r"(step) : "memory");
        }
    }
}
__global__ void __launch_bounds__(ROUTE_BLOCK)
k_route_peer(MapGeom g, FrameParams f, const float4 *xyzi, const uchar4 *rgba, int n, int tile_h, int tile_w, int tiles_c, int world,
             int my_rank, int nblk, int cap, int buf, int step, const __grid_constant__ PeerBufs pb, int *ticket)
{
    route_peer<false>(g, f, xyzi, rgba, n, tile_h, tile_w, tiles_c, world, my_rank, nblk, cap, buf, step, pb, ticket);
}
__global__ void __launch_bounds__(ROUTE_BLOCK) // every sensor model
k_route_peer_any(MapGeom g, FrameParams f, const float4 *xyzi, const uchar4 *rgba, int n, int tile_h, int tile_w, int tiles_c, int world,
                 int my_rank, int nblk, int cap, int buf, int step, const __grid_constant__ PeerBufs pb, int *ticket)
{
    route_peer<true>(g, f, xyzi, rgba, n, tile_h, tile_w, tiles_c, world, my_rank, nblk, cap, buf, step, pb, ticket);
}

// one point of the bin kernel, U = 1 (see bin_points for the argument why the waits cannot deadlock)
__device__ __forceinline__ void bin_one(Cell *cells, const BinScratch &sc, int key, int geo, uint4 rec, int i_rec, int i_mark)
{
    const int par = sc.par;
    const int rank = (key >= 0) ? atomicAdd(&cells[key].bin[par].x, 1) : -1;
    int lvl = 0, myp = 0;
    if (rank == CHUNK0) {
        st_relaxed(&cells[key].bin[par].y, i_rec + 1);
        sc.tlarge[atomicAdd(&sc.ctr->nlarge, 1)] = make_int4(key, LIST_LARGE, i_rec, 0);
    } else if (rank >= FOLD_LONG_FROM) {
        const int j = level_of(rank);
        if (rank == level_base(j)) { lvl = j; myp = 1 + atomicAdd(&sc.ctr->pool, level_cap(j) + 1); }
    }
    sc.mark[i_mark] = (rank == 0) ? make_int2(key, geo) : make_int2(-1, 0);
    if (rank < 0) return;
    uint4 *dst;
    if (rank < CHUNK0) {
        dst = sc.chunk0 + (size_t)CHUNK0 * key + rank;
    } else {
        const int i8 = (rank == CHUNK0) ? i_rec : spin_nonzero(&cells[key].bin[par].y) - 1;
        uint4 *q = sc.pool1 + (size_t)CHUNK1_SLOTS * i8;
        const int j = level_of(rank);
        if (lvl >= 2) { // publish the chunk this point allocated in the header of the level below
            uint4 *below = q;
            for (int k = 2; k < lvl; k++) below = sc.pool + spin_next(below);
            if (lvl == 2) sc.tlong[atomicAdd(&sc.ctr->nlong, 1)] = make_int4(key, LIST_LONG, i8, myp);
            publish_next(below, myp);
        }
        for (int k = 2; k <= j; k++) q = sc.pool + ((lvl == k) ? myp : spin_next(q));
        dst = q + 1 + (rank - level_base(j));
    }
    *dst = rec;
}

constexpr int BIN_PEER_MAX_BLOCKS = NUM_SMS * 8; // one wave of 256-thread blocks; a block takes sub-buckets blockIdx.x + q * gridDim.x
constexpr int BIN_PEER_MAX_PER_BLOCK = 32;
// k_bin_peer stages a block's sub-bucket counts in one round of BIN_PEER_MAX_PER_BLOCK.  What bounds nsub = world * nblk is
// gem_tiled_attach's world * cap <= max_points, and gem_create caps max_points at the fold's 2^22 point indices: at most
// 2^22 / 256 = 16384 sub-buckets, 16 per block.  A wider fold index must stage the counts in rounds first.
static_assert((1 << FOLD_INDEX_BITS) / ROUTE_BLOCK <= BIN_PEER_MAX_BLOCKS * BIN_PEER_MAX_PER_BLOCK,
              "k_bin_peer: more sub-buckets than one round of staged counts holds");

__global__ void __launch_bounds__(ROUTE_BLOCK)
k_bin_peer(MapGeom g, MapLayers ml, BinScratch sc, const uint4 *rec, const float *inten, const int *cnt, int nsub, const int *flags,
           int world, int step, int *n_marks)
{
    __shared__ int s_cnt[BIN_PEER_MAX_PER_BLOCK];
    __shared__ int s_base;
    if (blockIdx.x == 0) zero_next_counters(sc, threadIdx.x);
    if ((int)threadIdx.x < world) { // all peers have delivered this step (their records, counts and everything before the flag):
        int v;                      // one thread per peer, so the block waits for one round trip, not for `world` of them
        do {
            asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(flags + threadIdx.x) : "memory");
            if (v < step) __nanosleep(100);
        } while (v < step);
    }
    __syncthreads();
    const int nmine = (nsub - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x; // <= BIN_PEER_MAX_PER_BLOCK (static_assert above)
    if ((int)threadIdx.x < nmine) s_cnt[threadIdx.x] = cnt[blockIdx.x + threadIdx.x * gridDim.x];
    __syncthreads();
    for (int q = 0; q < nmine; q++) {
        const int c = s_cnt[q];
        if (c == 0) continue; // most sub-buckets of a large world are empty: a source's points land in few tiles
        const int sb = blockIdx.x + q * gridDim.x;
        // the marks are the fold's work list: any order will do as long as [0, *n_marks) is dense, so a sub-bucket takes its
        // range with one atomic (a few hundred per step) instead of summing the counts in front of it
        if (threadIdx.x == 0) s_base = atomicAdd(n_marks, c);
        __syncthreads();
        if ((int)threadIdx.x < c) {
            const int slot = sb * ROUTE_BLOCK + threadIdx.x; // monotone in (source rank, source point index): the fold's sort key
            const uint4 r = rec[slot];
            const int gkey = (int)r.x;
            const int gx = gkey / g.L, gy = gkey - gx * g.L;
            const int key = local_key(g, gx, gy);
            bin_one(ml.cell, sc, key, g.tiled ? key : gkey, make_uint4((uint32_t)slot, r.y, r.z, with_colour_flag(r.w, inten[slot])), slot, s_base + threadIdx.x);
        }
        __syncthreads(); // s_base is reused
    }
}

} // namespace gem
