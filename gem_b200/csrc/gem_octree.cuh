// gem_octree.cuh -- the octree step of composingGlobalMap (ElevationMapping.cpp:1146-1174, pointCloudtoOctomap) on the
// device: an octomap::ColorOcTree built from a cloud of 32-byte PointXYZRGBICT records (updateNode(p, true) and
// integrateNodeColor(p, r, g, b) per point in cloud order, :1161-1170, then updateInnerOccupancy, :1172-1173), written
// as the byte stream ColorOcTree::writeData produces (octomap_msgs::Octomap::data of fullMapToMsg).  DESIGN.md row f7.
//
// PARITY UNPINNED (octomap): restated from octomap 1.9 OccupancyOcTreeBase / ColorOcTree with default parameters; the
// oracle is tests/orc_color_octree.c.  Items O1-O6 (DESIGN.md f7; each is also at the code below):
//   O1 keys: s = floor((1.0 / resolution) * (double)c) per axis, inserted iff every s is in [-32768, 32767] (non-finite
//      coordinates DEFINED as skipped, octomap's cast is undefined there), key = (int)s + 32768.  Depth 16; the child
//      index at bit d is bit_d(kx) + 2 bit_d(ky) + 4 bit_d(kz), so the 48-bit Morton code below IS the path.
//   O2 hit = (float)log(0.7 / 0.3), max = (float)log(0.971 / 0.029), p(v) = 1 - 1 / (1 + exp((double)v)), all computed
//      on the host with its libm.  A node's value is one of the states v_1 = hit, v_k+1 = RN_f32(v_k + hit) clamped to
//      max (OctParams); the kernels carry the state index s (0 = just created, value 0) and read v and p from tables, so
//      no device exp / log enters the result.
//   O3 updateNode: early return when search(key) holds s == sat; missing children created (s 0, white); a childless,
//      not-just-created node expanded (8 copies); leaf s + 1; on the way up each node pruned when its 8 children exist,
//      are childless and have equal values (colour ignored); the pruned node copies child 0 and, if that colour is set,
//      takes the average colour of the children whose colour is set (ColorOcTree::pruneNode).
//   O4 integrateNodeColor on search(key): unset colour (255,255,255) is replaced; a set one mixed per channel as
//      (uint8_t)((double)prev * p + (double)new * (0.99 - p)), no contraction.
//   O5 updateInnerOccupancy: every node with children takes the max child value and the truncating mean of the set
//      child colours (white if none).
//   O6 stream: preorder, children 0..7, 8 bytes per node {float value, r, g, b, child bitset}; empty tree: 0 bytes.
//
// Parallel build.  Leaves only ever appear, and a pruned node stands for all 8^k leaves under it, so a node can be
// pruned only if every one of the 8^k leaf keys below it is inserted by the end: call such a node FULL.  A maximal full
// node (whose parent is not full) is never pruned into its parent, and every expansion, early return and colour
// integration on a pruned node inside it stays inside it.  Hence:
//   * k_oct_keys: O1 and the Morton code per point (skipped points get OCT_SKIP); CUB's stable radix sort by code keeps
//     each voxel's points in cloud order; run-length encoding gives the leaves and their point runs.
//   * k_oct_classify: per leaf, the largest k whose level-k ancestor is full (two binary searches per level over the
//     sorted leaf codes: full iff it holds 8^k leaves).  A leaf outside every full node is independent: its parent is
//     never pruned, so it is folded right there in point order (hit with early return at sat, then O4 on itself).  The
//     first leaf of each maximal full node opens a GROUP with a dense scratch subtree.
//   * k_oct_group_keys + a second sort: each group's points in cloud order; k_oct_group_sim simulates O3 / O4 literally,
//     one thread per group, on its dense subtree (in shared memory up to level OCT_SMEM_LEVEL) (a level-k group has 8^k distinct leaves, so the scratch is at most
//     8/7 of the leaf count), then O5 inside it and writes its final nodes.
//   * k_oct_upper, levels 0..16: the independent leaves, then per level the nodes above the groups (never pruned), with
//     O5 over their children (binary search for each child's first leaf).
//   * every node is written as a (preorder key, 8-byte record) pair; preorder is the order of (left-aligned code,
//     16 - level), so one more radix sort turns the records into the stream.
// The host synchronises twice: once for the sizes of the second phase, once for the counts of the result.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cub/cub.cuh>

namespace gem {

constexpr unsigned long long OCT_SKIP = 1ull << 48;   // sort key of a skipped point: above every 48-bit code
constexpr unsigned long long OCT_EMPTY = ~0ull;       // sort key of an unused node slot
constexpr int OCT_STATES = 8;
constexpr int OCT_SMEM_LEVEL = 5;                    // k_oct_group_sim: 37,449 slots, 146 KiB of shared memory
constexpr uint32_t OCT_WHITE = 0xFFFFFFu;             // packed node: r | g << 8 | b << 16 | s << 24 | flags
constexpr uint32_t OCT_EXISTS = 1u << 28, OCT_KIDS = 1u << 29;
constexpr uint32_t OCT_DATA = 0x0FFFFFFFu;            // colour and state

struct OctParams {                // O2, from the host: value, p and 0.99 - p of state s = 0..sat
    float v[OCT_STATES];
    double p[OCT_STATES], q[OCT_STATES];
    int sat;
};

struct OctCounters {
    int inserted, nruns, groups, upper, indep, grouped;
    unsigned long long dense;     // dense subtree nodes over every group
    int group_nodes, group_leaves, gp_pos, emit;
    int max_level;                // of every group
};

struct OctGroup {
    int head, level;              // first leaf (index into the sorted leaf codes), level of the maximal full node
    unsigned long long off;       // dense scratch offset
};

__host__ __device__ __forceinline__ unsigned long long oct_spread3(unsigned long long x)
{
    x &= 0xFFFFull;
    x = (x | x << 16) & 0x0000FF0000FFull;
    x = (x | x << 8) & 0x00F00F00F00Full;
    x = (x | x << 4) & 0x0C30C30C30C3ull;
    x = (x | x << 2) & 0x249249249249ull;
    return x;
}

// O1: false if the coordinate is skipped
__device__ __forceinline__ bool oct_key(double rf, float c, unsigned &key)
{
    const double s = floor(__dmul_rn(rf, (double)c));
    if (!(s >= -32768.0 && s <= 32767.0)) return false;   // NaN fails both
    key = (unsigned)((int)s + 32768);
    return true;
}

__device__ __forceinline__ unsigned long long oct_code(const float4 *pts, int p, double rf)
{
    const float4 a = __ldg(&pts[2 * (size_t)p]);
    unsigned kx, ky, kz;
    if (!oct_key(rf, a.x, kx) || !oct_key(rf, a.y, ky) || !oct_key(rf, a.z, kz)) return OCT_SKIP;
    return oct_spread3(kx) | oct_spread3(ky) << 1 | oct_spread3(kz) << 2;
}

__device__ __forceinline__ int oct_lower_bound(const unsigned long long *a, int lo, int hi, unsigned long long v)
{
    while (lo < hi) {
        const int mid = (int)(((unsigned)lo + (unsigned)hi) >> 1);
        if (a[mid] < v) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ unsigned oct_chan(uint32_t prev, uint32_t nw, double p, double q)
{
    return __double2uint_rz(__dadd_rn(__dmul_rn((double)prev, p), __dmul_rn((double)nw, q)));
}

// O4 on a packed node (colour bits only change) with the record's bgra word (r, g, b = bytes 2, 1, 0)
__device__ __forceinline__ uint32_t oct_integrate(uint32_t node, uint32_t bgra, const OctParams &P)
{
    const uint32_t r = (bgra >> 16) & 255, g = (bgra >> 8) & 255, b = bgra & 255;
    if ((node & OCT_WHITE) == OCT_WHITE) return (node & ~OCT_WHITE) | r | g << 8 | b << 16;
    const int s = (node >> 24) & 15;
    const double p = P.p[s], q = P.q[s];
    return (node & ~OCT_WHITE) | oct_chan(node & 255, r, p, q) | oct_chan((node >> 8) & 255, g, p, q) << 8 |
           oct_chan((node >> 16) & 255, b, p, q) << 16;
}

// O5 accumulator (also ColorOcTreeNode::getAverageChildColor for the pruned node of O3)
struct OctAvg {
    int r = 0, g = 0, b = 0, c = 0, s = 0;
    __device__ __forceinline__ void add(uint32_t node)
    {
        const int st = (node >> 24) & 15;
        s = st > s ? st : s;
        if ((node & OCT_WHITE) != OCT_WHITE) { r += node & 255; g += (node >> 8) & 255; b += (node >> 16) & 255; c++; }
    }
    __device__ __forceinline__ uint32_t colour() const
    {
        return c ? (uint32_t)(r / c) | (uint32_t)(g / c) << 8 | (uint32_t)(b / c) << 16 : OCT_WHITE;
    }
};

// the 8-byte stream record (O6) as a little-endian word: float value, r, g, b, child bitset
__device__ __forceinline__ unsigned long long oct_record(uint32_t node, unsigned bits, const OctParams &P)
{
    return (unsigned long long)__float_as_uint(P.v[(node >> 24) & 15]) | (unsigned long long)(node & OCT_WHITE) << 32 |
           (unsigned long long)bits << 56;
}

__device__ __forceinline__ unsigned long long oct_sort_key(unsigned long long left_code, int level)
{
    return left_code << 5 | (unsigned)(16 - level);
}

__device__ __forceinline__ int oct_warp_sum(int v)
{
    return __reduce_add_sync(0xFFFFFFFFu, v);
}

// a slot per calling thread from one counter, one atomic per warp
__device__ __forceinline__ int oct_warp_slot(int *ctr)
{
    const unsigned m = __activemask();
    const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
    int base = 0;
    if (lane == leader) base = atomicAdd(ctr, __popc(m));
    base = __shfl_sync(m, base, leader);
    return base + __popc(m & ((1u << lane) - 1));
}

__host__ __device__ __forceinline__ unsigned long long oct_dense_size(int level) // nodes of a complete level-k subtree
{
    return ((1ull << (3 * (level + 1))) - 1) / 7;
}

// O1 per point; the counter gets the inserted points
__global__ void k_oct_keys(const float4 *__restrict__ pts, int n, double rf, unsigned long long *__restrict__ code,
                           int *__restrict__ idx, OctCounters *ctr)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    int ins = 0;
    if (i < n) {
        const unsigned long long c = oct_code(pts, i, rf);
        code[i] = c;
        idx[i] = i;
        ins = c != OCT_SKIP;
    }
    ins = oct_warp_sum(ins);
    if ((threadIdx.x & 31) == 0 && ins) atomicAdd(&ctr->inserted, ins);
}

__device__ __forceinline__ int oct_leaf_count(const unsigned long long *U, const OctCounters *ctr)
{
    const int nr = ctr->nruns;
    return nr > 0 && U[nr - 1] == OCT_SKIP ? nr - 1 : nr;
}

// Per leaf j (sorted unique code U[j], points sidx[off[j] .. off[j] + cnt[j]) in cloud order): the level of its maximal
// full ancestor (0: independent), the independent fold, the group heads, and the counts of the second phase.
__global__ void k_oct_classify(const unsigned long long *__restrict__ U, const int *__restrict__ cnt,
                               const int *__restrict__ off, const int *__restrict__ sidx, const float4 *__restrict__ pts,
                               OctParams P, int *__restrict__ level, int *__restrict__ ghead, int *__restrict__ gid,
                               OctGroup *__restrict__ groups, uint32_t *__restrict__ val, OctCounters *ctr, int n)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const int nleaf = oct_leaf_count(U, ctr);
    int indep = 0, grouped = 0, upper = 0;
    if (j < nleaf && j < n) {
        const unsigned long long u = U[j];
        int g = 0, head = j;
        for (int k = 1; k <= 10 && (1ll << (3 * k)) <= (long long)nleaf; k++) {
            const unsigned long long pre = u >> (3 * k);
            const int lo = oct_lower_bound(U, 0, j + 1, pre << (3 * k));
            const int hi = oct_lower_bound(U, j, nleaf, (pre + 1) << (3 * k));
            if (hi - lo != (1 << (3 * k))) break;
            g = k;
            head = lo;
        }
        level[j] = g;
        ghead[j] = head;
        if (g == 0) { // independent leaf: its parent is never pruned (O3 on one leaf, O4 on itself)
            uint32_t node = OCT_WHITE;
            for (int t = 0, e = cnt[j], o = off[j]; t < e; t++) {
                int s = (node >> 24) & 15;
                if (s < P.sat) node = (node & ~(15u << 24)) | (uint32_t)(s + 1) << 24;   // early return at max
                const int p = sidx[o + t];
                node = oct_integrate(node, __float_as_uint(__ldg(&pts[2 * (size_t)p + 1]).x), P);
            }
            val[j] = node;
            indep = 1;
        } else {
            grouped = cnt[j];
            if (head == j) {
                const int gi = atomicAdd(&ctr->groups, 1);
                atomicMax(&ctr->max_level, g);
                groups[gi] = OctGroup{j, g, atomicAdd(&ctr->dense, oct_dense_size(g))};
                gid[j] = gi;
            }
        }
        for (int k = g + 1; k <= 16; k++) // the nodes above: counted at their first leaf
            upper += j == 0 || (U[j - 1] >> (3 * k)) != (u >> (3 * k));
    }
    indep = oct_warp_sum(indep);
    grouped = oct_warp_sum(grouped);
    upper = oct_warp_sum(upper);
    if ((threadIdx.x & 31) == 0) {
        if (indep) atomicAdd(&ctr->indep, indep);
        if (grouped) atomicAdd(&ctr->grouped, grouped);
        if (upper) atomicAdd(&ctr->upper, upper);
    }
}

// (group, point index) of every point in a group, for the second sort
__global__ void k_oct_group_keys(const unsigned long long *__restrict__ U, int nleaf, const int *__restrict__ cnt,
                                 const int *__restrict__ off, const int *__restrict__ sidx, const int *__restrict__ level,
                                 const int *__restrict__ ghead, const int *__restrict__ gid,
                                 unsigned long long *__restrict__ key2, OctCounters *ctr)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nleaf || level[j] == 0) return;
    const unsigned long long gi = (unsigned long long)gid[ghead[j]] << 32;
    const int e = cnt[j], o = off[j];
    const int base = atomicAdd(&ctr->gp_pos, e);
    for (int t = 0; t < e; t++) key2[base + t] = gi | (unsigned)sidx[o + t];
}

// O3 then O4 for one point of a group: `local` = the low 3 * g bits of its code (the path below the group root), on the
// dense subtree D of a level-g group
__device__ __forceinline__ void oct_group_point(uint32_t *D, int g, unsigned long long local, uint32_t bgra, const OctParams &P)
{
    // search(key): the leaf or the childless node on the path; -1 if the path ends at a missing node
    long long found = -1;
    if (D[0] & OCT_EXISTS) {
        long long at = 0, base = 0;
        for (int d = 0;; d++) {
            if (d == g || !(D[at] & OCT_KIDS)) { found = at; break; }
            base = base * 8 + 1;
            const long long c = base + (long long)(local >> (3 * (g - d - 1)));
            if (!(D[c] & OCT_EXISTS)) break;
            at = c;
        }
    }
    if (found < 0 || (int)((D[found] >> 24) & 15) < P.sat) { // O3 (early return when search holds max)
        bool just = false;
        if (!(D[0] & OCT_EXISTS)) { D[0] = OCT_EXISTS | OCT_WHITE; just = true; }
        long long at = 0, base = 0;
        for (int d = 0; d < g; d++) {
            const long long cbase = base * 8 + 1, idx = (long long)(local >> (3 * (g - d))), first = cbase + idx * 8;
            const long long c = cbase + (long long)(local >> (3 * (g - d - 1)));
            bool created = false;
            if (!(D[c] & OCT_EXISTS)) {
                if (!(D[at] & OCT_KIDS) && !just) { // expandNode: a pruned node becomes 8 copies
                    for (int i = 0; i < 8; i++) D[first + i] = OCT_EXISTS | (D[at] & OCT_DATA);
                } else {
                    D[c] = OCT_EXISTS | OCT_WHITE;
                    created = true;
                }
                D[at] |= OCT_KIDS;
            }
            just = created;
            at = c;
            base = cbase;
        }
        const uint32_t s = (D[at] >> 24) & 15;
        D[at] = (D[at] & ~(15u << 24)) | (s + 1) << 24; // s < sat here: a leaf at max returns early
        for (int d = g - 1; d >= 0; d--) { // pruneNode on the way up
            const long long dbase = (long long)((1ull << (3 * d)) - 1) / 7, idx = (long long)(local >> (3 * (g - d)));
            const long long n0 = dbase + idx, first = (long long)((1ull << (3 * (d + 1))) - 1) / 7 + idx * 8;
            const uint32_t c0 = D[first];
            bool ok = true;
            for (int i = 0; i < 8 && ok; i++) {
                const uint32_t ci = D[first + i];
                ok = (ci & OCT_EXISTS) && !(ci & OCT_KIDS) && ((ci >> 24) & 15) == ((c0 >> 24) & 15);
            }
            if (!ok) break; // a node above can only be collapsible if this one was just pruned
            uint32_t nd = OCT_EXISTS | (c0 & OCT_DATA);
            if ((c0 & OCT_WHITE) != OCT_WHITE) {
                OctAvg a;
                for (int i = 0; i < 8; i++) a.add(D[first + i]);
                nd = (nd & ~OCT_WHITE) | a.colour();
            }
            for (int i = 0; i < 8; i++) D[first + i] = 0;
            D[n0] = nd;
        }
    }
    // O4 on search(key), which exists now
    long long at = 0, base = 0;
    for (int d = 0; d < g && (D[at] & OCT_KIDS); d++) {
        base = base * 8 + 1;
        at = base + (long long)(local >> (3 * (g - d - 1)));
    }
    D[at] = oct_integrate(D[at], bgra, P);
}

// One warp per group, one thread of it simulating: O3 / O4 literally over the group's points in cloud order on a dense
// complete subtree (depth d from the group root holds 8^d slots from (8^d - 1) / 7), then O5 inside it, then its final
// nodes into the node list at node_base + the group's dense offset (unused slots keep OCT_EMPTY).  The simulation is a
// chain of dependent loads and stores on the subtree, so a subtree of at most smem_words slots lives in the block's
// shared memory (zeroed by the warp); a larger one uses its slots of `dense` (zeroed by the host), through L2.
__global__ void k_oct_group_sim(const OctGroup *__restrict__ groups, const unsigned long long *__restrict__ key2, int ngp,
                                const unsigned long long *__restrict__ U, const float4 *__restrict__ pts, double rf,
                                OctParams P, uint32_t *__restrict__ dense, int smem_words, unsigned long long *__restrict__ nkey,
                                unsigned long long *__restrict__ nrec, long long node_base, uint32_t *__restrict__ val,
                                OctCounters *ctr)
{
    extern __shared__ uint32_t oct_sub[];
    const int gi = blockIdx.x;
    const OctGroup G = groups[gi];
    const int g = G.level;
    const unsigned long long root = U[G.head] >> (3 * g) << (3 * g), lmask = (1ull << (3 * g)) - 1;
    uint32_t *D = dense + G.off;
    if ((long long)oct_dense_size(g) <= smem_words) {
        for (int i = threadIdx.x; i < (int)oct_dense_size(g); i += blockDim.x) oct_sub[i] = 0;
        __syncwarp();
        D = oct_sub;
    }
    // the warp fetches the next 32 points' paths and colours (independent loads, in flight together); lane 0 folds them
    __shared__ unsigned long long b_local[32];
    __shared__ uint32_t b_bgra[32];
    const int lane = threadIdx.x;
    const int lo = oct_lower_bound(key2, 0, ngp, (unsigned long long)gi << 32);
    const int hi = oct_lower_bound(key2, lo, ngp, (unsigned long long)(gi + 1) << 32);
    for (int t0 = lo; t0 < hi; t0 += 32) {
        if (t0 + lane < hi) {
            const int p = (int)(unsigned)key2[t0 + lane];
            b_local[lane] = oct_code(pts, p, rf) & lmask;
            b_bgra[lane] = __float_as_uint(__ldg(&pts[2 * (size_t)p + 1]).x);
        }
        __syncwarp();
        if (lane == 0)
            for (int u = 0, ue = min(32, hi - t0); u < ue; u++) oct_group_point(D, g, b_local[u], b_bgra[u], P);
        __syncwarp();
    }
    if (lane != 0) return;
    // O5 inside the group, bottom-up
    for (int d = g - 1; d >= 0; d--) {
        const long long dbase = (long long)((1ull << (3 * d)) - 1) / 7, cb = (long long)((1ull << (3 * (d + 1))) - 1) / 7;
        for (long long i = 0; i < (1ll << (3 * d)); i++) {
            const uint32_t nd = D[dbase + i];
            if (!(nd & OCT_KIDS)) continue;
            OctAvg a;
            for (int c = 0; c < 8; c++)
                if (D[cb + i * 8 + c] & OCT_EXISTS) a.add(D[cb + i * 8 + c]);
            D[dbase + i] = OCT_EXISTS | OCT_KIDS | (uint32_t)a.s << 24 | a.colour();
        }
    }
    // the final nodes
    int nodes = 0, leaves = 0;
    for (int d = 0; d <= g; d++) {
        const long long dbase = (long long)((1ull << (3 * d)) - 1) / 7, cb = (long long)((1ull << (3 * (d + 1))) - 1) / 7;
        for (long long i = 0; i < (1ll << (3 * d)); i++) {
            const uint32_t nd = D[dbase + i];
            if (!(nd & OCT_EXISTS)) continue;
            unsigned bits = 0;
            if (nd & OCT_KIDS)
                for (int c = 0; c < 8; c++) bits |= (D[cb + i * 8 + c] & OCT_EXISTS) ? 1u << c : 0u;
            const long long slot = node_base + (long long)G.off + dbase + i;
            nkey[slot] = oct_sort_key(root + ((unsigned long long)i << (3 * (g - d))), g - d);
            nrec[slot] = oct_record(nd, bits, P);
            nodes++;
            leaves += bits == 0;
        }
    }
    val[G.head] = D[0] & OCT_DATA;
    atomicAdd(&ctr->group_nodes, nodes);
    atomicAdd(&ctr->group_leaves, leaves);
}

// Level k = 0: the independent leaves.  Level k >= 1: the nodes above the groups (first leaf j, all its leaves at a
// lower group level), O5 over the children (each found by a binary search for its first leaf; val holds the child's
// packed node), into the node list at an atomic slot (the final sort orders them).
__global__ void k_oct_upper(const unsigned long long *__restrict__ U, int nleaf, const int *__restrict__ level, int k,
                            OctParams P, uint32_t *__restrict__ val, unsigned long long *__restrict__ nkey,
                            unsigned long long *__restrict__ nrec, OctCounters *ctr)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nleaf) return;
    const unsigned long long u = U[j];
    if (k == 0) {
        if (level[j] != 0) return;
        const int slot = oct_warp_slot(&ctr->emit);
        nkey[slot] = oct_sort_key(u, 0);
        nrec[slot] = oct_record(val[j], 0, P);
        return;
    }
    if (level[j] >= k || (j > 0 && (U[j - 1] >> (3 * k)) == (u >> (3 * k)))) return;
    const unsigned long long pre = u >> (3 * k);
    OctAvg a;
    unsigned bits = 0;
    int from = j;
    for (int c = 0; c < 8; c++) {
        const unsigned long long q = pre * 8 + c;
        const int h = oct_lower_bound(U, from, nleaf, q << (3 * (k - 1)));
        if (h < nleaf && (U[h] >> (3 * (k - 1))) == q) {
            a.add(val[h]);
            bits |= 1u << c;
            from = h;
        }
    }
    const uint32_t nd = (uint32_t)a.s << 24 | a.colour();
    val[j] = nd;
    const int slot = oct_warp_slot(&ctr->emit);
    nkey[slot] = oct_sort_key(pre << (3 * k), k);
    nrec[slot] = oct_record(nd, bits, P);
}

} // namespace gem
