// gem_api.cu -- host side of libgem_b200.so: the extern "C" ABI of include/gem_b200.h.
//
// Replaces the host wrappers of the reference's gpu_process.cu (Init_GPU_elevationmap :940,
// Move :1004, Process_points :1085, Mapvar_update :1146, Fuse :1154, Map_optmove :1215,
// Map_closeloop :1235, Map_feature :1256, Raytracing :1304).  Differences by design:
// per-handle state instead of __device__ globals, one stream per handle, zero per-call
// cudaMalloc/cudaFree (the reference does 8+7+9 per frame), geometry passed as kernel
// parameters instead of cudaMemcpyTo/FromSymbol round trips, int status codes, and every entry
// point takes the handle's mutex (the reference node enters libgpu.so from three threads,
// ElevationMapping.cpp:271-300,388-421, only partly under MapMutex_).
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/gem_b200.h"
#include "gem_add.cuh"
#include "gem_costmap.cuh"
#include "gem_kernels.cuh"
#include "gem_global.cuh"
#include "gem_mls.cuh"
#include "gem_octree.cuh"
#include "gem_route.cuh"
#include "gem_submap.cuh"
#include "gem_voxel.cuh"

using namespace gem;

namespace {

thread_local std::string g_create_error;

} // namespace

// one add call whose bin kernel has been issued and whose fold has not (pipelined mode)
struct PendingFold {
    bool active = false;
    BinScratch sc{};
    FoldSrc src{};
    MapGeom geom{};   // the geometry the call was binned with (a later Move must not change its lowest indices)
    int n = 0;        // marks of the call (tiled maps: their capacity; the count is *n_dev)
    const int *n_dev = nullptr;
};

struct TiledState { // gem_tiled_attach
    bool attached = false;
    int world = 0, my_rank = 0, tiles_r = 0, tiles_c = 0, cap = 0, nblk = 0;
    PeerBufs pb{};
    int *d_ticket = nullptr, *d_ntotal = nullptr; // [1], [2] (by call parity)
    int step = 0;
    int depth = 2;                                 // 2: {route j -> bin j || fold j-1} per call; 3: {route j || bin j-1 || fold j-2}
    struct { bool active = false; int step = 0, buf = 0; } routed; // depth 3: delivered to the owners, not binned yet
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    cudaGraphNode_t long_node = nullptr, fold_node = nullptr, route_node = nullptr, bin_node = nullptr;
};

struct OctBuf { // a device scratch buffer (octree, costmap and voxel-grid calls): grows on demand, never shrinks
    void *p = nullptr;
    size_t cap = 0;
    template <typename T> T *as() const { return static_cast<T *>(p); }
};
struct VoxScratch { // gem_voxel_grid (gem_voxel.cuh): keys and input indices before / after the sort, runs, offsets
    OctBuf key[2], idx[2], cnt, off, temp, acc;
};
struct MlsScratch { // gem_mls_upsample (gem_mls.cuh): cell keys and indices before / after the sort, the points in cell
                   // order, the distinct cells, neighbour and output counts, output offsets, the long lists and their keys
    OctBuf key[2], idx[2], spts, ukey, ucnt, uoff, nbr, ocnt, ooff, longs, lkeys, temp, acc;
};
struct OctScratch { // gem_color_octree (gem_octree.cuh); every buffer is consistent with its own capacity at all times
    OctBuf code[2], idx[2], leaf, cnt, off, level, ghead, gid, val, groups, ctr, temp, key2[2], nkey[2], nrec[2], dense;
    long long bytes = -1; // size of the last stream (in nrec[1]); -1: none
    gem_octree info{};
};

struct LocalStore { // localMap_ on the device (gem_harvest_to_local_map, gem_local_map_take / _clear; gem_submap.cuh)
    void *buf = nullptr;               // one allocation: log, index keys, index positions, take scratch
    float4 *log = nullptr;             // 2 x float4 per record, in harvest order
    unsigned long long *keys = nullptr; // open-addressing index, HASH_EMPTY = free slot
    int *latest = nullptr;             // per slot: the latest log position of its key
    int *cnt = nullptr;                // take: kept entries per 32 log entries, then the scan's segment totals
    int n = 0, cap = 0;                // records in the log, records it can hold
    size_t slots = 0;                  // index slots (a power of two >= 2 * cap)
};

struct FrameGraph { // {long lists || the other lists of the previous call || bin of this call} as one three-node CUDA graph
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    cudaGraphNode_t long_node = nullptr, fold_node = nullptr, bin_node = nullptr;
};

struct gem_map {
    std::recursive_mutex mu;
    gem_config cfg{};
    int dev = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int L = 0;
    size_t nc = 0; // cells held by this handle
    int P = 0;     // per-launch point capacity
    MapGeom geom{};
    MapLayers ml{};
    float sensorZ = 0.0f;
    // add path: two scratch sets (call parity), three counter buffers (the bin kernel of call i zeroes the
    // buffer of call i+1, last used by call i-2 whose fold is complete by then)
    BinScratch bs[2]{};
    BinCounters *ctr[3] = {nullptr, nullptr, nullptr};
    unsigned call_no = 0;
    BinCounters *ctr_last = nullptr; // counters of the last add call
    PendingFold pend;
    TiledState tiled;
    // tuning (scripts/pipe_sweep.sh sweeps them): GEM_B200_FOLD_BLOCKS, GEM_B200_LONG_BLOCKS,
    // GEM_B200_EXCLUSIVE=1 pads the kernels' shared memory so that k_fold_long's blocks get SMs of their own
    int fold_max_blocks = NUM_SMS * 2, long_blocks = LONG_BLOCKS;
    size_t bin_smem = 0, fold_smem = FOLD_SMEM_USED, long_smem = (LONG_BLOCK / 32) * sizeof(WarpScratch);
    int pipe_mode = 2;               // 0: never defer the fold; 1: two streams + events; 2: CUDA graph per call
    std::map<const void *, FrameGraph> graphs; // keyed by the bin kernel function
    cudaStream_t front_stream = nullptr;      // pipe_mode 1: the bin kernels run here
    cudaEvent_t ev_bin[2] = {nullptr, nullptr}, ev_fold[2] = {nullptr, nullptr}, ev_mark = nullptr;
    // deferred region operations (scroll clears of Move, the every-cell variance floor of
    // G_fuse): executed by the next add/fuse launch, or flushed before anything observes the map
    std::vector<RegionOp> pending;
    // staging (device), lazily allocated
    void *d_xyzi = nullptr, *d_rgba = nullptr, *d_pcl = nullptr;
    float *d_x = nullptr, *d_y = nullptr, *d_z = nullptr, *d_xt = nullptr, *d_yt = nullptr;
    int *d_keyin = nullptr, *d_keyout = nullptr, *d_R = nullptr, *d_G = nullptr, *d_B = nullptr;
    float *d_int = nullptr, *d_h = nullptr, *d_hv = nullptr;
    float *d_out = nullptr; // 9 * nc floats read-out staging
    int *d_owner_cnt = nullptr;
    RouteScratch route_sc{};
    float2 *prev_ev = nullptr;     // gem_snapshot_shown: prevMap_ (ElevationMapping.cpp:422) on the device
    uint2 *prev_ci = nullptr;
    float *prev_tr = nullptr;
    MapGeom prev_geom{};
    bool prev_valid = false;
    LocalStore local;
    int *d_viscnt = nullptr;       // visual-cloud export: per (column, row chunk) counts / offsets
    // gem_grid_cloud_split: geographic z, row x, column y, per-cell distance, compacted distances, queue, counters, stats
    float *split_zg = nullptr, *split_xg = nullptr, *split_yg = nullptr, *split_dcell = nullptr, *split_dist = nullptr;
    int *split_queue = nullptr, *split_ctr = nullptr;
    SplitStats *split_stats = nullptr;
    OctScratch oct;                // gem_color_octree: scratch and the last stream
    OctBuf cost_scratch;           // costmap calls: the winner per costmap cell (int), or the copy of a rolled grid
    CostMarksDev *cost_acc = nullptr; // costmap mark calls: counts and encoded touch bounds
    VoxScratch vox;                // gem_voxel_grid
    MlsScratch mls;                // gem_mls_upsample
    unsigned long long *d_stamps = nullptr; // gem_debug_stamps
    int *d_raylist = nullptr;      // ray clean-up: cells that cast a ray + their count
    uint32_t *d_bitmap = nullptr;  // ray clean-up: validity bitmap of the lowest layer (own tile / map-wide)
    size_t bitmap_words = 0;
    BinCounters *h_ctr = nullptr; // pinned
    // pipelined host ingest (gem_add_points_host_async): three staging sets (the fold of call i, issued with
    // call i+1, still reads call i's intensities)
    cudaEvent_t ev_export = nullptr, ev_export_done = nullptr; // gem_export_layers_begin / _end
    cudaStream_t copy_stream = nullptr;
    void *d_axyzi[3] = {nullptr, nullptr, nullptr}, *d_argba[3] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev_h2d[3] = {nullptr, nullptr, nullptr}, ev_done[3] = {nullptr, nullptr, nullptr};
    BinCounters *h_ctr_ring = nullptr; // pinned, 2 entries
    unsigned async_calls = 0;
    // gem_add_points_multi: ring of per-call FrameParams tables (pinned host + device)
    FrameParams *h_frames = nullptr, *d_frames = nullptr;
    cudaEvent_t ev_frames[4] = {nullptr, nullptr, nullptr, nullptr};
    unsigned multi_calls = 0;
    gem_stats stats{};
    std::string err;
    std::vector<void *> allocs;
    // launch accounting / optional per-kernel CUDA-event timing (gem_profile_*)
    long long launches = 0;
    bool profiling = false;
    struct Span { int cls; cudaEvent_t e0, e1; };
    std::vector<Span> spans;
    std::vector<cudaEvent_t> free_events;
    double prof_ms[GEM_PROF_CLASSES] = {0};
    long long prof_count[GEM_PROF_CLASSES] = {0};
};

namespace {

using Lock = std::lock_guard<std::recursive_mutex>;
// k_fold_long's grid (four warps per block, one list per warp and draw): a c2 lidar frame (125k points) has 330-420
// lists of more than 8 records and runs best with ~100-150 blocks; a c3 depth frame (307k points, ~13 per touched cell)
// has far more lists and runs faster the more blocks it gets, up to the cap (DESIGN.md section 4, decision 5)
inline int long_blocks_for(const gem_map *m, int n)
{
    const int b = n / 1024;
    return b < m->long_blocks ? m->long_blocks : (b > NUM_SMS * 4 ? NUM_SMS * 4 : b);
}
// points per block and pass of k_fold: an even share of the call, in whole warps, at most FOLD_MARKS marks per thread
inline int fold_slice(int n, int fold_blocks)
{
    int s = (n + fold_blocks - 1) / fold_blocks;
    s = (s + 31) / 32 * 32;
    if (s < ADD_BLOCK) s = ADD_BLOCK;
    if (s > FOLD_MARKS * ADD_BLOCK) s = FOLD_MARKS * ADD_BLOCK;
    return s;
}

int fail(gem_map *m, int code, const std::string &msg)
{
    if (m) m->err = msg; else g_create_error = msg;
    return code;
}

cudaEvent_t prof_event(gem_map *m)
{
    if (!m->free_events.empty()) {
        cudaEvent_t e = m->free_events.back();
        m->free_events.pop_back();
        return e;
    }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
}
// every kernel launch of the library goes through this macro: counts the launch and, when
// profiling is on, brackets it with CUDA events on the stream it is launched on
#define GEM_LAUNCH_ON(m, st, cls, ...)                           \
    do {                                                         \
        (m)->launches++;                                         \
        if ((m)->profiling) {                                    \
            gem_map::Span sp__{(cls), prof_event(m), prof_event(m)}; \
            cudaEventRecord(sp__.e0, (st));                      \
            __VA_ARGS__;                                         \
            cudaEventRecord(sp__.e1, (st));                      \
            (m)->spans.push_back(sp__);                          \
        } else {                                                 \
            __VA_ARGS__;                                         \
        }                                                        \
    } while (0)
#define GEM_LAUNCH(m, cls, ...) GEM_LAUNCH_ON(m, (m)->stream, cls, __VA_ARGS__)

#define GEM_CUDA(m, expr)                                                                      \
    do {                                                                                       \
        cudaError_t e__ = (expr);                                                              \
        if (e__ != cudaSuccess) {                                                              \
            return fail((m), GEM_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e__)); \
        }                                                                                      \
    } while (0)

template <typename T> int dev_alloc(gem_map *m, T **p, size_t count)
{
    void *q = nullptr;
    cudaError_t e = cudaMalloc(&q, count * sizeof(T) + 16);
    if (e != cudaSuccess) return fail(m, GEM_ERR_NOMEM, std::string("cudaMalloc: ") + cudaGetErrorString(e));
    m->allocs.push_back(q);
    *p = (T *)q;
    return GEM_OK;
}

// capacity of a per-call list of the cells holding MORE than k of a call's <= P records: at most P / (k + 1) such
// cells exist, and never more than the map has
inline size_t list_cap(size_t P, size_t nc, int k) { return std::min(nc, P / (size_t)(k + 1)) + 1; }
inline int blocks_for(size_t n, int bs, int cap = NUM_SMS * 16)
{
    size_t b = (n + bs - 1) / bs;
    if (b < 1) b = 1;
    if ((size_t)cap < b) b = cap;
    return (int)b;
}

// k_fold's grid: a frame-sized call gets one pass over an even share per block (at most fold_max_blocks blocks: the kernel
// is latency bound and few fat blocks leave room for the concurrently running bin kernel); a large call gets one block
// per full slice, scheduled in waves (a block's passes are serial latency chains, waves overlap them)
inline int fold_blocks_for(const gem_map *m, int n)
{
    if ((long long)n <= (long long)m->fold_max_blocks * FOLD_MARKS * ADD_BLOCK) return blocks_for((size_t)n, ADD_BLOCK, m->fold_max_blocks);
    return blocks_for((size_t)n, FOLD_MARKS * ADD_BLOCK, 1 << 30);
}

struct SetDev {
    int prev = -1;
    explicit SetDev(int d) { cudaGetDevice(&prev); if (prev != d) cudaSetDevice(d); else prev = -1; }
    ~SetDev() { if (prev >= 0) cudaSetDevice(prev); }
};

FrameParams make_frame(const gem_frame *f)
{
    FrameParams p;
    memset(&p, 0, sizeof p);
    for (int i = 0; i < 12; i++) p.T[i] = f->T[i];
    for (int i = 0; i < 3; i++) { p.sJ[i] = f->sensor_jacobian[i]; p.P[i] = f->P_mul_C_BM_transpose[i]; }
    p.has_rot = 0;
    for (int i = 0; i < 9; i++) {
        p.rotVar[i] = f->rotation_variance[i];
        p.CSBT[i] = f->C_SB_transpose[i];
        p.Bskew[i] = f->B_r_BS_skew[i];
        if (f->rotation_variance[i] != 0.0f) p.has_rot = 1;
    }
    p.lo = f->rel_lower;
    p.hi = f->rel_upper;
    p.sensor_type = f->sensor.type;
    p.min_r = f->sensor.min_radius;
    p.beam_a = f->sensor.beam_angle;
    p.beam_c = f->sensor.beam_constant;
    p.nf_a = f->sensor.normal_factor_a;
    p.nf_b = f->sensor.normal_factor_b;
    p.nf_c = f->sensor.normal_factor_c;
    p.nf_d = f->sensor.normal_factor_d;
    p.nf_e = f->sensor.normal_factor_e;
    p.lat = f->sensor.lateral_factor;
    p.cut_lo = (float)f->sensor.cutoff_min_depth; // pcl::PassThrough::setFilterLimits takes floats
    p.cut_hi = (float)f->sensor.cutoff_max_depth;
    return p;
}

size_t region_cells(const gem_map *m, const RegionOp &r)
{
    if (r.kind == 0) return m->nc;
    if (r.kind == 1) return (size_t)r.n * m->geom.cols;
    return (size_t)r.n * m->geom.rows;
}

int launch_regions(gem_map *m, const RegionOp *ops, int count)
{
    for (int i = 0; i < count; i += MAX_REGION_OPS) {
        RegionOps ro{};
        size_t cells = 0;
        ro.count = (count - i < MAX_REGION_OPS) ? (count - i) : MAX_REGION_OPS;
        for (int k = 0; k < ro.count; k++) { ro.op[k] = ops[i + k]; cells += region_cells(m, ops[i + k]); }
        GEM_LAUNCH(m, GEM_PROF_CLEAR, k_regions<<<blocks_for(cells, ADD_BLOCK), ADD_BLOCK, 0, m->stream>>>(m->geom, m->ml, ro));
    }
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}

// ---- the fold of a pipelined add call is issued with the NEXT call, or here ------------------------------------
int launch_fold(gem_map *m, cudaStream_t st, const PendingFold &p, const RegionOps &ro, int region_blocks, bool do_fuse, bool do_lowest)
{
    const int fb = fold_blocks_for(m, p.n);
    const int slice = fold_slice(p.n, fb);
    // the long lists first (their blocks claim whole SMs), then everything else; on one stream the two run back to back
    // (disjoint cells, so the order is free) -- the frame graph of the pipelined mode runs them side by side.  Both get
    // the next call's clears `ro`: a long list inside a cleared band must store the cleared value itself, because
    // k_fold's region blocks may clear the cell before k_fold_long writes it (cell_end)
    GEM_LAUNCH_ON(m, st, GEM_PROF_FOLD_LONG, k_fold_long<<<long_blocks_for(m, p.n), LONG_BLOCK, m->long_smem, st>>>(p.geom, m->ml, p.sc, p.src, ro, do_fuse ? 1 : 0, do_lowest ? 1 : 0));
    GEM_LAUNCH_ON(m, st, GEM_PROF_FOLD, k_fold<<<fb + region_blocks, ADD_BLOCK, m->fold_smem, st>>>(p.geom, m->ml, p.sc, p.src, ro, p.n, fb, slice, do_fuse ? 1 : 0, do_lowest ? 1 : 0, p.n_dev));
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}

// the bin kernel of a routed tiled step: its arguments and the fold it leaves behind; takes the call's scratch set
struct TiledBin {
    MapGeom gl;
    MapLayers ml;
    BinScratch sc;
    const uint4 *rec;
    const float *inten;
    const int *cnt, *flags;
    int nsub, world, step;
    int *ntotal;
    PendingFold fold;
};

TiledBin tiled_bin_of(gem_map *m, int step, int buf)
{
    TiledState &ts = m->tiled;
    const int par = (int)(m->call_no & 1u), c = (int)(m->call_no % 3u);
    TiledBin b{};
    b.gl = m->geom;
    b.ml = m->ml;
    b.sc = m->bs[par];
    b.sc.ctr = m->ctr[c];
    b.sc.ctr_next = m->ctr[(c + 1) % 3];
    b.sc.par = par;
    b.sc.stamps = nullptr;
    b.world = ts.world;
    b.nsub = ts.world * ts.nblk;
    b.step = step;
    b.rec = (const uint4 *)ts.pb.rec[ts.my_rank] + (size_t)buf * ts.world * ts.cap;
    b.inten = (const float *)ts.pb.inten[ts.my_rank] + (size_t)buf * ts.world * ts.cap;
    b.cnt = (const int *)ts.pb.cnt[ts.my_rank] + (size_t)buf * b.nsub;
    b.flags = (const int *)ts.pb.flag[ts.my_rank];
    b.ntotal = &b.sc.ctr->nmarks; // zero when the call starts (zeroed by the bin kernel of the call before)
    b.fold.active = true;
    b.fold.sc = b.sc;
    b.fold.geom = m->geom;
    b.fold.n = ts.world * ts.cap;
    b.fold.n_dev = b.ntotal;
    b.fold.src = FoldSrc{(const char *)b.inten, 4};
    m->ctr_last = b.sc.ctr;
    m->call_no++;
    return b;
}

static int bin_peer_blocks(int nsub) { return nsub < BIN_PEER_MAX_BLOCKS ? nsub : BIN_PEER_MAX_BLOCKS; }

int launch_tiled_bin(gem_map *m, const TiledBin &b)
{
    GEM_LAUNCH(m, GEM_PROF_BIN, k_bin_peer<<<bin_peer_blocks(b.nsub), ROUTE_BLOCK, 0, m->stream>>>(b.gl, b.ml, b.sc, b.rec, b.inten, b.cnt, b.nsub, b.flags, b.world, b.step, b.ntotal));
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}

int drain(gem_map *m)
{
    RegionOps none{};
    int rc;
    if (m->pend.active) {
        if (m->pipe_mode == 1) GEM_CUDA(m, cudaStreamWaitEvent(m->stream, m->ev_bin[m->pend.sc.par], 0));
        if ((rc = launch_fold(m, m->stream, m->pend, none, 0, true, true))) return rc;
        if (m->pipe_mode == 1) GEM_CUDA(m, cudaEventRecord(m->ev_fold[m->pend.sc.par], m->stream));
        m->pend.active = false;
    }
    if (m->tiled.routed.active) { // a tiled step that is routed but not binned: bin it, fold it
        const TiledBin b = tiled_bin_of(m, m->tiled.routed.step, m->tiled.routed.buf);
        m->tiled.routed.active = false;
        if ((rc = launch_tiled_bin(m, b)) || (rc = launch_fold(m, m->stream, b.fold, none, 0, true, true))) return rc;
    }
    return GEM_OK;
}

// something is about to read the layers: issue a deferred fold, then execute deferred clears (a clear is visible
// in the reference as soon as Move returns); floors stay pending until the next Fuse
int flush_for_observer(gem_map *m)
{
    int rc = drain(m);
    if (rc) return rc;
    std::vector<RegionOp> now;
    for (RegionOp &r : m->pending)
        if (r.clear) {
            RegionOp c = r;
            c.floor_ = 0;
            now.push_back(c);
            r.clear = 0;
        }
    if (now.empty()) return GEM_OK;
    return launch_regions(m, now.data(), (int)now.size());
}

// a Fuse-type call is starting with nothing in flight: hand the pending operations to its first kernel.
// The operations leave the pending list only once the kernel that executes them has been launched (commit_region_ops).
int take_region_ops(gem_map *m, RegionOps &ro, int &region_blocks)
{
    ro.count = 0;
    region_blocks = 0;
    const int np = (int)m->pending.size();
    if (np > MAX_REGION_OPS) { // rare: many moves without an add
        int rc = launch_regions(m, m->pending.data(), np - MAX_REGION_OPS);
        if (rc) return rc;
        m->pending.erase(m->pending.begin(), m->pending.end() - MAX_REGION_OPS);
    }
    size_t cells = 0;
    for (const RegionOp &r : m->pending) {
        ro.op[ro.count++] = r;
        cells += region_cells(m, r);
    }
    if (ro.count) region_blocks = blocks_for(cells, ADD_BLOCK * 4, NUM_SMS * 2);
    return GEM_OK;
}
void commit_region_ops(gem_map *m) { m->pending.clear(); }

// a Fuse with nothing to fold still applies clears + floor
int flush_all_pending(gem_map *m)
{
    int rc = drain(m);
    if (rc) return rc;
    if (m->pending.empty()) return GEM_OK;
    rc = launch_regions(m, m->pending.data(), (int)m->pending.size());
    if (rc == GEM_OK) m->pending.clear();
    return rc;
}

void pend_all_floor(gem_map *m)
{
    m->pending.clear();
    m->pending.push_back(RegionOp{0, 0, 0, 0, 1});
}

// points per thread in the bin kernel: one point per thread keeps a frame-sized call (1e5 points, < 1 wave)
// latency-optimal; large calls get 2 or 4 points per thread so that a thread has several independent DRAM/L2
// round trips in flight instead of running 3-4 waves of serial chains
inline int points_per_thread(int n) { return n >= 600000 ? 4 : (n >= 250000 ? 2 : 1); }

typedef void (*BinKernel)(MapGeom, MapLayers, FrameParams, BinSource, int, BinScratch, const RegionOps, int, const SegTable, const FrameParams *);
template <int SRC> BinKernel bin_kernel(int U)
{
    if (SRC == SRC_XYZI || SRC == SRC_RECORDS) {
        if (U == 4) return k_bin<SRC, 4>;
        if (U == 2) return k_bin<SRC, 2>;
    }
    return k_bin<SRC, 1>;
}

int read_counters(gem_map *m, long long n_in, bool accumulate)
{
    int rc = drain(m);
    if (rc) return rc;
    GEM_CUDA(m, cudaMemcpyAsync(m->h_ctr, m->ctr_last, sizeof(BinCounters), cudaMemcpyDeviceToHost, m->stream));
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    if (!accumulate) memset(&m->stats, 0, sizeof m->stats);
    m->stats.points_in += n_in;
    m->stats.points_binned += m->h_ctr->total;
    m->stats.cells_touched += m->h_ctr->ntouched;
    if (m->h_ctr->pool > m->bs[0].pool_cap) return fail(m, GEM_ERR_CUDA, "internal: record pool exhausted");
    if (m->h_ctr->nlong >= m->bs[0].long_cap || m->h_ctr->nlarge >= m->bs[0].large_cap) return fail(m, GEM_ERR_CUDA, "internal: list queue overflow");
    if (m->h_ctr->maxk > m->stats.max_points_per_cell) m->stats.max_points_per_cell = m->h_ctr->maxk;
    return GEM_OK;
}

int ensure_host_staging(gem_map *m)
{
    if (m->d_xyzi && m->d_rgba) return GEM_OK;
    int rc;
    if (!m->d_xyzi && (rc = dev_alloc(m, (float4 **)&m->d_xyzi, (size_t)m->P))) return rc;
    if (!m->d_rgba && (rc = dev_alloc(m, (uchar4 **)&m->d_rgba, (size_t)m->P))) return rc;
    return GEM_OK;
}
int ensure_pcl_staging(gem_map *m)
{
    if (m->d_pcl) return GEM_OK;
    return dev_alloc(m, (float4 **)&m->d_pcl, (size_t)m->P * 2);
}
int ensure_compat_staging(gem_map *m)
{
    int rc;
    const size_t P = (size_t)m->P;
    float **fp[] = {&m->d_x, &m->d_y, &m->d_z, &m->d_xt, &m->d_yt, &m->d_int, &m->d_h, &m->d_hv};
    int **ip[] = {&m->d_keyin, &m->d_keyout, &m->d_R, &m->d_G, &m->d_B};
    for (float **p : fp) if (!*p && (rc = dev_alloc(m, p, P))) return rc; // each buffer once, also after a partial failure
    for (int **p : ip) if (!*p && (rc = dev_alloc(m, p, P))) return rc;
    return GEM_OK;
}
int ensure_out_staging(gem_map *m)
{
    if (m->ev_export_done) cudaStreamWaitEvent(m->stream, m->ev_export_done, 0); // an asynchronous export may still be reading the staging buffer
    if (m->d_out) return GEM_OK;
    return dev_alloc(m, &m->d_out, m->nc * 9);
}

int ensure_ray_scratch(gem_map *m, size_t bitmap_cells)
{
    int rc;
    if (!m->d_raylist && (rc = dev_alloc(m, &m->d_raylist, m->nc + 1))) return rc; // every cell may cast a ray; [nc] = the count
    const size_t words = bitmap_cells / 32 + 1;
    if (!m->d_bitmap || m->bitmap_words < words) {
        if ((rc = dev_alloc(m, &m->d_bitmap, words))) return rc;
        m->bitmap_words = words;
    }
    return GEM_OK;
}
int ensure_route_scratch(gem_map *m)
{
    int rc;
    const size_t P = (size_t)m->P;
    RouteScratch &r = m->route_sc;
    if (!r.owner && (rc = dev_alloc(m, &r.owner, P))) return rc;
    if (!r.gkey && (rc = dev_alloc(m, &r.gkey, P))) return rc;
    if (!r.h && (rc = dev_alloc(m, &r.h, P))) return rc;
    if (!r.hv && (rc = dev_alloc(m, &r.hv, P))) return rc;
    if (!r.blockCounts) {
        r.blockCounts_capacity = (size_t)ROUTE_MAX_OWNERS * ((P + ROUTE_BLOCK - 1) / ROUTE_BLOCK);
        if ((rc = dev_alloc(m, &r.blockCounts, r.blockCounts_capacity))) return rc;
    }
    return GEM_OK;
}

int pipe_setup(gem_map *m)
{
    if (m->pipe_mode != 1) return GEM_OK;
    if (!m->front_stream) GEM_CUDA(m, cudaStreamCreateWithFlags(&m->front_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 2; i++) {
        if (!m->ev_bin[i]) GEM_CUDA(m, cudaEventCreateWithFlags(&m->ev_bin[i], cudaEventDisableTiming));
        if (!m->ev_fold[i]) {
            GEM_CUDA(m, cudaEventCreateWithFlags(&m->ev_fold[i], cudaEventDisableTiming));
            GEM_CUDA(m, cudaEventRecord(m->ev_fold[i], m->stream));
        }
    }
    if (!m->ev_mark) GEM_CUDA(m, cudaEventCreateWithFlags(&m->ev_mark, cudaEventDisableTiming));
    return GEM_OK;
}

// {long lists, other lists of the previous call || bin of this call} as a three-node graph, built once per bin kernel; per
// call only the node parameters change.  One cudaGraphLaunch replaces three launches, two event records and two stream waits.
int launch_frame_graph(gem_map *m, BinKernel bk, void **bin_args, int bin_grid, void **fold_args, int fold_grid, void **long_args, int long_grid)
{
    FrameGraph &fg = m->graphs[(const void *)bk];
    cudaKernelNodeParams kb{}, kf{}, kl{};
    kb.func = (void *)bk; kb.gridDim = dim3((unsigned)bin_grid); kb.blockDim = dim3(ADD_BLOCK); kb.sharedMemBytes = (unsigned)m->bin_smem; kb.kernelParams = bin_args;
    kf.func = (void *)k_fold; kf.gridDim = dim3((unsigned)fold_grid); kf.blockDim = dim3(ADD_BLOCK); kf.sharedMemBytes = (unsigned)m->fold_smem; kf.kernelParams = fold_args;
    kl.func = (void *)k_fold_long; kl.gridDim = dim3((unsigned)long_grid); kl.blockDim = dim3(LONG_BLOCK); kl.sharedMemBytes = (unsigned)m->long_smem; kl.kernelParams = long_args;
    if (!fg.exec) {
        GEM_CUDA(m, cudaGraphCreate(&fg.graph, 0));
        GEM_CUDA(m, cudaGraphAddKernelNode(&fg.long_node, fg.graph, nullptr, 0, &kl)); // first: its blocks want empty SMs
        GEM_CUDA(m, cudaGraphAddKernelNode(&fg.fold_node, fg.graph, nullptr, 0, &kf));
        GEM_CUDA(m, cudaGraphAddKernelNode(&fg.bin_node, fg.graph, nullptr, 0, &kb));
        GEM_CUDA(m, cudaGraphInstantiate(&fg.exec, fg.graph, 0));
    } else {
        GEM_CUDA(m, cudaGraphExecKernelNodeSetParams(fg.exec, fg.long_node, &kl));
        GEM_CUDA(m, cudaGraphExecKernelNodeSetParams(fg.exec, fg.fold_node, &kf));
        GEM_CUDA(m, cudaGraphExecKernelNodeSetParams(fg.exec, fg.bin_node, &kb));
    }
    GEM_CUDA(m, cudaGraphLaunch(fg.exec, m->stream));
    m->launches += 3;
    return GEM_OK;
}

// One add call on device-resident input.  pipelined == false: bin (+ deferred region operations) then fold, both
// on the handle's stream.  pipelined == true: the bin kernel of this call is issued together with the FOLD OF THE
// PREVIOUS pipelined call (which also carries the row / column clears this call's Move decided), and this call's
// fold stays pending until the next call or until anything observes the map (drain).
template <int SRC>
int enqueue_add(gem_map *m, const BinSource &in, const FoldSrc &fsrc, int n, const FrameParams &fp, const SegTable *segs,
                const FrameParams *frames, bool pipelined, bool do_fuse, bool do_lowest)
{
    int rc;
    if (m->profiling || m->pipe_mode == 0) pipelined = false; // per-kernel event timing needs the serial schedule
    if (pipelined && (rc = pipe_setup(m))) return rc;
    if (pipelined && m->pend.active) {
        // operations other than "clear + floor of a row / column band" cannot ride on a running fold
        bool mergeable = (int)m->pending.size() <= MAX_REGION_OPS;
        for (const RegionOp &r : m->pending) mergeable = mergeable && r.kind != 0 && r.clear && r.floor_;
        if (!mergeable && (rc = drain(m))) return rc;
    }
    if (!pipelined && (rc = drain(m))) return rc;
    const int par = (int)(m->call_no & 1u), c = (int)(m->call_no % 3u);
    BinScratch sc = m->bs[par];
    sc.ctr = m->ctr[c];
    sc.ctr_next = m->ctr[(c + 1) % 3];
    sc.par = par;
    sc.stamps = m->d_stamps;
    const int U = points_per_thread(n);
    BinKernel bk = bin_kernel<SRC>(U);
    const int pb = blocks_for((size_t)(n + U - 1) / U, ADD_BLOCK, NUM_SMS * 16);
    SegTable st{};
    if (segs) st = *segs;
    MapGeom g = m->geom;
    MapLayers ml = m->ml;
    FrameParams f = fp;
    BinSource bin = in;
    int nn = n;
    RegionOps ro{};
    int rb = 0;
    PendingFold cur;
    cur.active = true; cur.sc = sc; cur.src = fsrc; cur.geom = m->geom; cur.n = n;
    if (!pipelined || !m->pend.active) {
        // nothing in flight: the bin kernel carries the deferred region operations in spare blocks
        if ((rc = take_region_ops(m, ro, rb))) return rc;
        cudaStream_t st_bin = m->stream;
        if (pipelined && m->pipe_mode == 1) { // later bins of the pipeline run on the front stream: order it behind everything issued so far
            GEM_CUDA(m, cudaEventRecord(m->ev_mark, m->stream));
            GEM_CUDA(m, cudaStreamWaitEvent(m->front_stream, m->ev_mark, 0));
            st_bin = m->front_stream;
        }
        GEM_LAUNCH_ON(m, st_bin, GEM_PROF_BIN, bk<<<pb + rb, ADD_BLOCK, m->bin_smem, st_bin>>>(g, ml, f, bin, nn, sc, ro, pb, st, frames));
        GEM_CUDA(m, cudaGetLastError());
        commit_region_ops(m);
        if (pipelined && m->pipe_mode == 1) GEM_CUDA(m, cudaEventRecord(m->ev_bin[par], st_bin));
        if (!pipelined) {
            RegionOps none{};
            if ((rc = launch_fold(m, m->stream, cur, none, 0, do_fuse, do_lowest))) return rc;
        } else {
            m->pend = cur;
        }
    } else {
        // steady state of the pipeline
        if ((rc = take_region_ops(m, ro, rb))) return rc; // row / column clears of this call's Move: executed by the previous call's fold launch
        PendingFold prev = m->pend;
        const int fb = fold_blocks_for(m, prev.n);
        int slice = fold_slice(prev.n, fb);
        RegionOps none{};
        if (m->pipe_mode == 2) {
            int pbk = pb, one = 1, fbk = fb;
            void *bin_args[] = {&g, &ml, &f, &bin, &nn, &sc, &none, &pbk, &st, (void *)&frames};
            void *fold_args[] = {&prev.geom, &ml, &prev.sc, &prev.src, &ro, &prev.n, &fbk, &slice, &one, &one, (void *)&prev.n_dev};
            void *long_args[] = {&prev.geom, &ml, &prev.sc, &prev.src, &ro, &one, &one}; // the clears, like k_fold (launch_fold)
            if ((rc = launch_frame_graph(m, bk, bin_args, pb, fold_args, fb + rb, long_args, long_blocks_for(m, prev.n)))) return rc;
        } else {
            GEM_CUDA(m, cudaStreamWaitEvent(m->front_stream, m->ev_fold[par], 0)); // the fold that last used this parity's scratch
            GEM_LAUNCH_ON(m, m->front_stream, GEM_PROF_BIN, bk<<<pb, ADD_BLOCK, m->bin_smem, m->front_stream>>>(g, ml, f, bin, nn, sc, none, pb, st, frames));
            GEM_CUDA(m, cudaEventRecord(m->ev_bin[par], m->front_stream));
            GEM_CUDA(m, cudaStreamWaitEvent(m->stream, m->ev_bin[prev.sc.par], 0));
            if ((rc = launch_fold(m, m->stream, prev, ro, rb, true, true))) return rc;
            GEM_CUDA(m, cudaEventRecord(m->ev_fold[prev.sc.par], m->stream));
        }
        commit_region_ops(m);
        m->pend = cur;
    }
    m->ctr_last = sc.ctr;
    m->call_no++;
    return GEM_OK;
}

} // namespace

// =========================================================================================
static GridMapFrame grid_frame(const gem_map *m, float cx, float cy, int sx, int sy)
{
    GridMapFrame f;
    f.res = m->cfg.grid_resolution > 0.0 ? m->cfg.grid_resolution : (double)m->cfg.resolution;
    f.half = 0.5 * ((double)m->L * f.res) - 0.5 * f.res;
    f.cx = (double)cx; f.cy = (double)cy;
    f.L = m->L; f.sx = sx; f.sy = sy;
    return f;
}

// count -> scan -> write of the cells Src takes, in GridMapIterator order, issued on the handle's stream; the total is
// left in device memory (*d_total_out: the compaction scratch, valid until the next compaction)
template <class Src> static int compact_cells_issue(gem_map *m, const Src &src, int capacity, int **d_total_out)
{
    const int L = m->L, nch = (L + 31) / 32;
    int rc;
    const int n = L * nch, nseg = (n + SCAN_SEG - 1) / SCAN_SEG;
    if (!m->d_viscnt) { if ((rc = dev_alloc(m, &m->d_viscnt, (size_t)n + nseg + 1))) return rc; }
    int *d_segtot = m->d_viscnt + n, *d_total = d_segtot + nseg;
    const dim3 grid(nch, nch);
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_compact_count<Src><<<grid, 1024, 0, m->stream>>>(src, L, nch, m->d_viscnt));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_compact_scan<<<nseg, SCAN_SEG, 0, m->stream>>>(m->d_viscnt, n, d_segtot));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_compact_write<Src><<<grid, 1024, 0, m->stream>>>(src, L, nch, m->d_viscnt, d_segtot, nseg, d_total, capacity));
    GEM_CUDA(m, cudaGetLastError());
    *d_total_out = d_total;
    return GEM_OK;
}
// the same, host-synchronous; returns the total through *total_out
template <class Src> static int compact_cells(gem_map *m, const Src &src, int capacity, int *total_out)
{
    int *d_total = nullptr;
    const int rc = compact_cells_issue(m, src, capacity, &d_total);
    if (rc) return rc;
    GEM_CUDA(m, cudaMemcpyAsync(total_out, d_total, sizeof(int), cudaMemcpyDeviceToHost, m->stream));
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    return GEM_OK;
}

extern "C" {

int gem_version(void) { return GEM_B200_VERSION; }

const char *gem_last_error(const gem_map *m) { return m ? m->err.c_str() : g_create_error.c_str(); }

int gem_create(const gem_config *cfg, gem_map **out)
{
    if (!cfg || !out) return fail(nullptr, GEM_ERR_INVALID, "gem_create: null argument");
    *out = nullptr;
    if (cfg->length < 1 || cfg->length > 46340 || !(cfg->resolution > 0.0f))
        return fail(nullptr, GEM_ERR_INVALID, "gem_create: length must be in [1,46340] and resolution > 0");
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev < 1)
        return fail(nullptr, GEM_ERR_NO_DEVICE,
                    std::string("gem_create: no CUDA device (libgem_b200 has no CPU fallback): ") +
                        (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0"));
    int dev = cfg->device;
    if (dev < 0) {
        e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return fail(nullptr, GEM_ERR_NO_DEVICE, cudaGetErrorString(e));
    }
    if (dev >= ndev) return fail(nullptr, GEM_ERR_INVALID, "gem_create: device ordinal out of range");
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, dev);
    if (e != cudaSuccess) return fail(nullptr, GEM_ERR_NO_DEVICE, cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0)
        return fail(nullptr, GEM_ERR_NO_DEVICE,
                    "gem_create: this library carries sm_90a code only (found compute capability " +
                        std::to_string(prop.major) + "." + std::to_string(prop.minor) + ")");

    gem_map *m = new gem_map();
    m->cfg = *cfg;
    m->dev = dev;
    SetDev sd(dev);
    m->L = cfg->length;
    const bool tiled = cfg->tile_rows > 0 && cfg->tile_cols > 0;
    if (tiled) {
        if (cfg->tile_row0 < 0 || cfg->tile_col0 < 0 || cfg->tile_row0 + cfg->tile_rows > m->L ||
            cfg->tile_col0 + cfg->tile_cols > m->L) {
            delete m;
            return fail(nullptr, GEM_ERR_INVALID, "gem_create: tile outside the map");
        }
    }
    m->geom.L = m->L;
    m->geom.res = cfg->resolution;
    m->geom.cx = m->geom.cy = 0.0f; // gpu.cu:942
    m->geom.sx = m->geom.sy = 0;    // gpu.cu:943
    m->geom.box_filter = cfg->compat_box_filter ? 1 : 0;
    m->geom.tiled = tiled ? 1 : 0;
    m->geom.r0 = tiled ? cfg->tile_row0 : 0;
    m->geom.rows = tiled ? cfg->tile_rows : m->L;
    m->geom.c0 = tiled ? cfg->tile_col0 : 0;
    m->geom.cols = tiled ? cfg->tile_cols : m->L;
    m->nc = (size_t)m->geom.rows * m->geom.cols;
    m->P = cfg->max_points > 0 ? cfg->max_points : (1 << 20); // per point: 8 B mark + 528 B level-1 chunk space, x 2 parities
    // the fold's sort key packs the point index of a launch into 22 bits; larger calls are chunked
    if (m->P > (1 << FOLD_INDEX_BITS)) m->P = 1 << FOLD_INDEX_BITS;
    {
        const char *env = getenv("GEM_B200_PIPE"); // graph (default) | stream | off
        if (env && !strcmp(env, "stream")) m->pipe_mode = 1;
        else if (env && !strcmp(env, "off")) m->pipe_mode = 0;
        const char *e1 = getenv("GEM_B200_FOLD_BLOCKS"), *e2 = getenv("GEM_B200_LONG_BLOCKS"), *e3 = getenv("GEM_B200_EXCLUSIVE");
        if (e1 && atoi(e1) > 0) m->fold_max_blocks = atoi(e1);
        if (e2 && atoi(e2) > 0) m->long_blocks = atoi(e2);
        if (e3 && atoi(e3) == 1) { m->bin_smem = BIN_SMEM_BYTES; m->fold_smem = FOLD_SMEM_BYTES; m->long_smem = LONG_SMEM_BYTES; }
    }

    int rc = GEM_OK;
    auto bail = [&](int code) {
        std::string msg = m->err;
        gem_destroy(m);
        g_create_error = msg;
        return code;
    };
    if (cfg->stream) {
        m->stream = (cudaStream_t)cfg->stream;
    } else {
        e = cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking);
        if (e != cudaSuccess) { m->err = cudaGetErrorString(e); return bail(GEM_ERR_CUDA); }
        m->own_stream = true;
    }
    const size_t nc = m->nc, P = (size_t)m->P;
    if ((rc = dev_alloc(m, &m->ml.cell, nc)) || (rc = dev_alloc(m, &m->ml.traver, nc)) || (rc = dev_alloc(m, &m->ml.lowest, nc)) ||
        (rc = dev_alloc(m, &m->ml.rough, nc)) || (rc = dev_alloc(m, &m->ml.slope, nc)) || (rc = dev_alloc(m, &m->ml.traver_out, nc)) ||
        (rc = dev_alloc(m, &m->ctr[0], 3)))
        return bail(rc);
    for (int i = 1; i < 3; i++) m->ctr[i] = m->ctr[0] + i;
    m->ctr_last = m->ctr[0];
    for (int p = 0; p < 2; p++) {
        BinScratch &sc = m->bs[p];
        sc.par = p;
        // only cells with more than 40 records take pool chunks: at most 4k + 12 slots for a cell of k records
        sc.pool_cap = (int)std::min<size_t>(5 * P + 64, (size_t)0x7ffffff0);
        sc.long_cap = (int)list_cap(P, nc, FOLD_LONG_FROM);
        sc.large_cap = (int)list_cap(P, nc, CHUNK0);
        if ((rc = dev_alloc(m, &sc.mark, P)) || (rc = dev_alloc(m, &sc.chunk0, (size_t)CHUNK0 * nc)) ||
            (rc = dev_alloc(m, &sc.pool1, (size_t)CHUNK1_SLOTS * P)) || (rc = dev_alloc(m, &sc.pool, (size_t)sc.pool_cap + 1)) ||
            (rc = dev_alloc(m, &sc.tlong, (size_t)sc.long_cap)) || (rc = dev_alloc(m, &sc.tlarge, (size_t)sc.large_cap)))
            return bail(rc);
        // no stale chunk headers (the fold clears the ones it consumes); records and marks need no initialisation
        e = cudaMemsetAsync(sc.pool1, 0, (size_t)CHUNK1_SLOTS * P * sizeof(uint4), m->stream);
        if (e == cudaSuccess) e = cudaMemsetAsync(sc.pool, 0, ((size_t)sc.pool_cap + 1) * sizeof(uint4), m->stream);
        if (e != cudaSuccess) { m->err = cudaGetErrorString(e); return bail(GEM_ERR_CUDA); }
    }
    e = cudaHostAlloc((void **)&m->h_ctr, sizeof(BinCounters), cudaHostAllocDefault);
    if (e != cudaSuccess) { m->err = cudaGetErrorString(e); return bail(GEM_ERR_CUDA); }
    // G_Init_map gpu.cu:198-214
    GEM_LAUNCH(m, GEM_PROF_CLEAR, k_clear_range<<<blocks_for(nc, 256), 256, 0, m->stream>>>(m->ml, 0, nc, 2));
    GEM_LAUNCH(m, GEM_PROF_CLEAR, k_fill<<<blocks_for(nc, 256), 256, 0, m->stream>>>(m->ml.rough, nc, 0.0f));
    GEM_LAUNCH(m, GEM_PROF_CLEAR, k_fill<<<blocks_for(nc, 256), 256, 0, m->stream>>>(m->ml.slope, nc, 0.0f));
    GEM_LAUNCH(m, GEM_PROF_CLEAR, k_fill<<<blocks_for(nc, 256), 256, 0, m->stream>>>(m->ml.traver_out, nc, -10.0f));
    e = cudaMemsetAsync(m->ctr[0], 0, 3 * sizeof(BinCounters), m->stream);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(m->stream);
    if (e != cudaSuccess) {
        m->err = std::string("gem_create: init kernels failed (is the device sm_90?): ") + cudaGetErrorString(e);
        return bail(GEM_ERR_NO_DEVICE);
    }
    e = cudaFuncSetAttribute(k_fold, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FOLD_SMEM_BYTES); // > 48 KB: opt-in
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_fold_long, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LONG_SMEM_BYTES);
    if (e != cudaSuccess) { m->err = std::string("gem_create: k_fold shared memory: ") + cudaGetErrorString(e); return bail(GEM_ERR_CUDA); }
    pend_all_floor(m); // first Fuse floors every cell (gpu.cu:533-534)
    *out = m;
    return GEM_OK;
}

int gem_destroy(gem_map *m)
{
    if (!m) return GEM_OK;
    {
        Lock lk(m->mu);
        SetDev sd(m->dev);
        if (m->front_stream) cudaStreamSynchronize(m->front_stream);
        if (m->stream) cudaStreamSynchronize(m->stream);
        for (auto &kv : m->graphs) {
            if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
            if (kv.second.graph) cudaGraphDestroy(kv.second.graph);
        }
        if (m->tiled.exec) cudaGraphExecDestroy(m->tiled.exec);
        if (m->tiled.graph) cudaGraphDestroy(m->tiled.graph);
        for (auto &sp : m->spans) { cudaEventDestroy(sp.e0); cudaEventDestroy(sp.e1); }
        for (cudaEvent_t e : m->free_events) cudaEventDestroy(e);
        for (void *p : m->allocs) cudaFree(p);
        if (m->local.buf) cudaFree(m->local.buf);
        for (OctBuf *b : {&m->oct.code[0], &m->oct.code[1], &m->oct.idx[0], &m->oct.idx[1], &m->oct.leaf, &m->oct.cnt, &m->oct.off,
                          &m->oct.level, &m->oct.ghead, &m->oct.gid, &m->oct.val, &m->oct.groups, &m->oct.ctr, &m->oct.temp,
                          &m->oct.key2[0], &m->oct.key2[1], &m->oct.nkey[0], &m->oct.nkey[1], &m->oct.nrec[0], &m->oct.nrec[1],
                          &m->oct.dense, &m->cost_scratch, &m->vox.key[0], &m->vox.key[1], &m->vox.idx[0], &m->vox.idx[1],
                          &m->vox.cnt, &m->vox.off, &m->vox.temp, &m->vox.acc, &m->mls.key[0], &m->mls.key[1], &m->mls.idx[0],
                          &m->mls.idx[1], &m->mls.spts, &m->mls.ukey, &m->mls.ucnt, &m->mls.uoff, &m->mls.nbr, &m->mls.ocnt,
                          &m->mls.ooff, &m->mls.longs, &m->mls.lkeys, &m->mls.temp, &m->mls.acc})
            if (b->p) cudaFree(b->p);
        if (m->h_ctr) cudaFreeHost(m->h_ctr);
        if (m->h_ctr_ring) cudaFreeHost(m->h_ctr_ring);
        if (m->h_frames) cudaFreeHost(m->h_frames);
        for (int i = 0; i < 2; i++) {
            if (m->ev_bin[i]) cudaEventDestroy(m->ev_bin[i]);
            if (m->ev_fold[i]) cudaEventDestroy(m->ev_fold[i]);
        }
        if (m->ev_mark) cudaEventDestroy(m->ev_mark);
        if (m->ev_export) cudaEventDestroy(m->ev_export);
        if (m->ev_export_done) cudaEventDestroy(m->ev_export_done);
        if (m->front_stream) cudaStreamDestroy(m->front_stream);
        for (int i = 0; i < 4; i++) if (m->ev_frames[i]) cudaEventDestroy(m->ev_frames[i]);
        for (int i = 0; i < 3; i++) {
            if (m->ev_h2d[i]) cudaEventDestroy(m->ev_h2d[i]);
            if (m->ev_done[i]) cudaEventDestroy(m->ev_done[i]);
        }
        if (m->copy_stream) { cudaStreamSynchronize(m->copy_stream); cudaStreamDestroy(m->copy_stream); }
        if (m->own_stream && m->stream) cudaStreamDestroy(m->stream);
    }
    delete m;
    return GEM_OK;
}

void *gem_get_stream(gem_map *m) { return m ? (void *)m->stream : nullptr; }

int gem_debug_stamps(gem_map *m, int enable, unsigned long long out[16])
{
    if (!m) return GEM_ERR_INVALID;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = drain(m);
    if (rc) return rc;
    if (out && m->d_stamps) {
        GEM_CUDA(m, cudaMemcpyAsync(out, m->d_stamps, 16 * 8, cudaMemcpyDeviceToHost, m->stream));
        GEM_CUDA(m, cudaStreamSynchronize(m->stream));
        out[0] = ~out[0]; out[8] = ~out[8];
    }
    if (enable && !m->d_stamps && (rc = dev_alloc(m, &m->d_stamps, 16))) return rc;
    if (m->d_stamps) GEM_CUDA(m, cudaMemsetAsync(m->d_stamps, 0, 16 * 8, m->stream));
    if (!enable) m->d_stamps = nullptr; // (the 128 bytes stay allocated until gem_destroy)
    return GEM_OK;
}

int gem_flush(gem_map *m)
{
    if (!m) return GEM_ERR_INVALID;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    return drain(m);
}

int gem_sync(gem_map *m)
{
    if (!m) return GEM_ERR_INVALID;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = drain(m);
    if (rc) return rc;
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    return GEM_OK;
}

// ---- Move gpu.cu:1004-1083 -----------------------------------------------------------------
static int index_to_range(int index, int L)
{ // gpu.cu:916-921
    if (index < 0) index += ((-index / L) + 1) * L;
    return index % L;
}
static int d2i_host(double d)
{ // cvt.rzi semantics for the host-side casts of gpu.cu:897,998-999
    if (d != d) return 0;
    if (d >= 2147483648.0) return 2147483647;
    if (d <= -2147483649.0) return -2147483647 - 1;
    return (int)d;
}
static float position_to_range(float p, float shift, float resolution)
{ // gpu.cu:996-1002
    const int p_index = d2i_host((double)roundf(p / resolution));
    const int shift_index = d2i_host((double)roundf(shift / resolution));
    return (float)(p_index + shift_index) * resolution;
}
// scroll clears are deferred: the next add/fuse launch executes them (plus the variance
// floor that G_fuse would apply to the cleared cells), or flush_for_observer does
static void clear_rows(gem_map *m, int start, int n) { m->pending.push_back(RegionOp{1, start, n, 1, 1}); }
static void clear_cols(gem_map *m, int start, int n) { m->pending.push_back(RegionOp{2, start, n, 1, 1}); }

int gem_move(gem_map *m, const float pos[3], float centre_out[2], int start_out[2], float shift_out[2])
{
    if (!m || !pos) return fail(m, GEM_ERR_INVALID, "gem_move: null argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    const int L = m->L;
    m->sensorZ = pos[2]; // gpu.cu:1011-1012
    float aligned[2] = {0.0f, 0.0f};
    if (m->geom.tiled) {
        // tiled (multi-GPU) maps are global, non-scrolling maps (SURVEY 8d config 4)
        if (centre_out) { centre_out[0] = m->geom.cx; centre_out[1] = m->geom.cy; }
        if (start_out) { start_out[0] = 0; start_out[1] = 0; }
        if (shift_out) { shift_out[0] = 0.0f; shift_out[1] = 0.0f; }
        return GEM_OK;
    }
    float centre[2] = {m->geom.cx, m->geom.cy};
    int start[2] = {m->geom.sx, m->geom.sy};
    int indexShift[2];
    for (int i = 0; i < 2; i++) {
        const float ps = pos[i] - centre[i];
        indexShift[i] = d2i_host((double)(ps / m->geom.res) + 0.5 * (ps > 0 ? 1 : -1)); // gpu.cu:897
        aligned[i] = (float)indexShift[i] * m->geom.res;                                   // gpu.cu:909
    }
    for (int i = 0; i < 2; i++) {
        if (indexShift[i] != 0) {
            // |shift| >= L clears everything (the reference tests only the positive side,
            // gpu.cu:1033, and would write out of bounds for shift <= -L)
            if (indexShift[i] >= L || indexShift[i] <= -L) {
                { int rcd = drain(m); if (rcd) return rcd; }
                GEM_LAUNCH(m, GEM_PROF_CLEAR, k_clear_range<<<blocks_for(m->nc, 256), 256, 0, m->stream>>>(m->ml, 0, m->nc, 1));
                pend_all_floor(m);
            } else {
                const int sign = indexShift[i] > 0 ? 1 : -1;
                const int startIndex = start[i] - (sign > 0 ? 1 : 0);
                const int endIndex = startIndex + sign - indexShift[i];
                const int nCells = std::abs(indexShift[i]);
                int index = sign < 0 ? startIndex : endIndex;
                index = index_to_range(index, L);
                if (index + nCells <= L) {
                    if (i == 0) clear_rows(m, index, nCells); else clear_cols(m, index, nCells);
                } else {
                    const int firstn = L - index, secondn = nCells - firstn;
                    if (i == 0) { clear_rows(m, index, firstn); clear_rows(m, 0, secondn); }
                    else { clear_cols(m, index, firstn); clear_cols(m, 0, secondn); }
                }
            }
        }
        start[i] = index_to_range(start[i] - indexShift[i], L);
        centre[i] = position_to_range(centre[i], aligned[i], m->geom.res);
    }
    m->geom.cx = centre[0]; m->geom.cy = centre[1];
    m->geom.sx = start[0]; m->geom.sy = start[1];
    if (centre_out) { centre_out[0] = centre[0]; centre_out[1] = centre[1]; }
    if (start_out) { start_out[0] = start[0]; start_out[1] = start[1]; }
    if (shift_out) { shift_out[0] = aligned[0]; shift_out[1] = aligned[1]; }
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}


// ---- fused add -------------------------------------------------------------------------------
static BinSource xyzi_source(const void *xyzi, const void *rgba, int off)
{
    BinSource in{};
    in.xyzi = (const float4 *)xyzi + off;
    in.rgba = rgba ? (const uchar4 *)rgba + off : nullptr;
    return in;
}

int gem_add_points(gem_map *m, const void *xyzi, const void *rgba, int n, const gem_frame *frame)
{
    if (!m || !frame || n < 0 || (n > 0 && !xyzi)) return fail(m, GEM_ERR_INVALID, "gem_add_points: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = GEM_OK;
    const FrameParams fp = make_frame(frame);
    memset(&m->stats, 0, sizeof m->stats);
    if (n == 0) return flush_all_pending(m);
    for (int off = 0; off < n; off += m->P) {
        const int cn = (n - off < m->P) ? (n - off) : m->P;
        const BinSource in = xyzi_source(xyzi, rgba, off);
        const FoldSrc fs{in.xyzi ? (const char *)in.xyzi + 12 : nullptr, 16};
        if ((rc = enqueue_add<SRC_XYZI>(m, in, fs, cn, fp, nullptr, nullptr, false, true, true))) return rc;
        if (n > m->P && (rc = read_counters(m, cn, true))) return rc; // chunked: keep totals
    }
    if (n <= m->P) m->stats.points_in = n; // counters are fetched lazily by gem_get_stats
    return GEM_OK;
}

int gem_add_points_host(gem_map *m, const void *xyzi, const void *rgba, int n, const gem_frame *frame)
{
    if (!m || !frame || n < 0 || (n > 0 && !xyzi)) return fail(m, GEM_ERR_INVALID, "gem_add_points_host: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_host_staging(m);
    if (rc) return rc;
    const FrameParams fp = make_frame(frame);
    memset(&m->stats, 0, sizeof m->stats);
    if (n == 0) { if ((rc = flush_all_pending(m))) return rc; return gem_sync(m); }
    if ((rc = drain(m))) return rc; // the staging buffers may still feed a deferred fold
    for (int off = 0; off < n; off += m->P) {
        const int cn = (n - off < m->P) ? (n - off) : m->P;
        GEM_CUDA(m, cudaMemcpyAsync(m->d_xyzi, (const float4 *)xyzi + off, (size_t)cn * 16, cudaMemcpyHostToDevice, m->stream));
        if (rgba)
            GEM_CUDA(m, cudaMemcpyAsync(m->d_rgba, (const uchar4 *)rgba + off, (size_t)cn * 4, cudaMemcpyHostToDevice, m->stream));
        const BinSource in = xyzi_source(m->d_xyzi, rgba ? m->d_rgba : nullptr, 0);
        const FoldSrc fs{in.xyzi ? (const char *)in.xyzi + 12 : nullptr, 16};
        if ((rc = enqueue_add<SRC_XYZI>(m, in, fs, cn, fp, nullptr, nullptr, false, true, true))) return rc;
        if ((rc = read_counters(m, cn, true))) return rc; // also the host-visible completion point
    }
    return GEM_OK;
}

int gem_add_points_stream(gem_map *m, const void *xyzi, const void *rgba, int n, const gem_frame *frame)
{
    if (!m || !frame || n < 0 || (n > 0 && !xyzi)) return fail(m, GEM_ERR_INVALID, "gem_add_points_stream: bad argument");
    if (n > m->P) return fail(m, GEM_ERR_INVALID, "gem_add_points_stream: n exceeds max_points (use gem_add_points)");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    if (n == 0) return flush_all_pending(m);
    const FrameParams fp = make_frame(frame);
    const BinSource in = xyzi_source(xyzi, rgba, 0);
    const FoldSrc fs{in.xyzi ? (const char *)in.xyzi + 12 : nullptr, 16};
    int rc = enqueue_add<SRC_XYZI>(m, in, fs, n, fp, nullptr, nullptr, true, true, true);
    if (rc) return rc;
    memset(&m->stats, 0, sizeof m->stats);
    m->stats.points_in = n;
    return GEM_OK;
}

int gem_add_points_multi(gem_map *m, const void *xyzi, const void *rgba, int n_segments, const int *offsets,
                         const gem_frame *frames)
{
    if (!m || !xyzi || !offsets || !frames || n_segments < 1 || n_segments > MAX_SEGMENTS)
        return fail(m, GEM_ERR_INVALID, "gem_add_points_multi: bad argument");
    const int n = offsets[n_segments] - offsets[0];
    if (offsets[0] != 0 || n < 0 || n > m->P) return fail(m, GEM_ERR_INVALID, "gem_add_points_multi: offsets must start at 0 and n <= max_points");
    for (int s = 0; s < n_segments; s++)
        if (offsets[s + 1] < offsets[s]) return fail(m, GEM_ERR_INVALID, "gem_add_points_multi: offsets not monotone");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = GEM_OK;
    if (!m->h_frames) GEM_CUDA(m, cudaHostAlloc((void **)&m->h_frames, 4 * MAX_SEGMENTS * sizeof(FrameParams), cudaHostAllocDefault));
    if (!m->d_frames && (rc = dev_alloc(m, &m->d_frames, (size_t)4 * MAX_SEGMENTS))) return rc;
    for (int i = 0; i < 4; i++)
        if (!m->ev_frames[i]) GEM_CUDA(m, cudaEventCreateWithFlags(&m->ev_frames[i], cudaEventDisableTiming));
    if (n == 0) return flush_all_pending(m);
    const int slot = (int)(m->multi_calls++ & 3u);
    if (m->multi_calls > 4) GEM_CUDA(m, cudaEventSynchronize(m->ev_frames[slot])); // pinned slot free again
    FrameParams *hf = m->h_frames + (size_t)slot * MAX_SEGMENTS, *df = m->d_frames + (size_t)slot * MAX_SEGMENTS;
    SegTable st{};
    st.n = n_segments;
    for (int s = 0; s <= n_segments; s++) st.off[s] = offsets[s];
    for (int s = 0; s < n_segments; s++) hf[s] = make_frame(&frames[s]);
    GEM_CUDA(m, cudaMemcpyAsync(df, hf, (size_t)n_segments * sizeof(FrameParams), cudaMemcpyHostToDevice, m->stream));
    GEM_CUDA(m, cudaEventRecord(m->ev_frames[slot], m->stream));
    // GEM_B200_PIPE=stream: the steady-state bin runs on the front stream, which waits only for the fold that last used
    // its scratch (recorded before this copy was queued): it must not read the table before the copy lands
    if (m->pipe_mode == 1 && m->front_stream) GEM_CUDA(m, cudaStreamWaitEvent(m->front_stream, m->ev_frames[slot], 0));
    const BinSource in = xyzi_source(xyzi, rgba, 0);
    const FoldSrc fs{in.xyzi ? (const char *)in.xyzi + 12 : nullptr, 16};
    // pipelined like gem_add_points_stream: consecutive multi-sensor steps overlap bin(i+1) with fold(i)
    if ((rc = enqueue_add<SRC_XYZI>(m, in, fs, n, hf[0], &st, df, true, true, true))) return rc;
    memset(&m->stats, 0, sizeof m->stats);
    m->stats.points_in = n;
    return GEM_OK;
}

int gem_add_points_host_async(gem_map *m, const void *xyzi, const void *rgba, int n, const gem_frame *frame)
{
    if (!m || !frame || n < 0 || (n > 0 && !xyzi)) return fail(m, GEM_ERR_INVALID, "gem_add_points_host_async: bad argument");
    if (n > m->P) return fail(m, GEM_ERR_INVALID, "gem_add_points_host_async: n exceeds max_points (use gem_add_points_host)");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = GEM_OK;
    // lazy set-up (every handle created at most once, also after a partial failure): copy stream, three staging
    // sets, events, counter ring
    if (!m->copy_stream) GEM_CUDA(m, cudaStreamCreateWithFlags(&m->copy_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 3; i++) {
        if (!m->d_axyzi[i] && (rc = dev_alloc(m, (float4 **)&m->d_axyzi[i], (size_t)m->P))) return rc;
        if (!m->d_argba[i] && (rc = dev_alloc(m, (uchar4 **)&m->d_argba[i], (size_t)m->P))) return rc;
        if (!m->ev_h2d[i]) GEM_CUDA(m, cudaEventCreateWithFlags(&m->ev_h2d[i], cudaEventDisableTiming));
        if (!m->ev_done[i]) {
            GEM_CUDA(m, cudaEventCreateWithFlags(&m->ev_done[i], cudaEventDisableTiming));
            GEM_CUDA(m, cudaEventRecord(m->ev_done[i], m->stream));
        }
    }
    if (!m->h_ctr_ring) GEM_CUDA(m, cudaHostAlloc((void **)&m->h_ctr_ring, 2 * sizeof(BinCounters), cudaHostAllocDefault));
    if (n == 0) return flush_all_pending(m);
    const unsigned i = m->async_calls++;
    const int b = (int)(i % 3u);
    // copy stream: wait until the fold that last read staging set b (call i-3) has been issued and is done, then H2D
    GEM_CUDA(m, cudaStreamWaitEvent(m->copy_stream, m->ev_done[b], 0));
    GEM_CUDA(m, cudaMemcpyAsync(m->d_axyzi[b], xyzi, (size_t)n * 16, cudaMemcpyHostToDevice, m->copy_stream));
    if (rgba) GEM_CUDA(m, cudaMemcpyAsync(m->d_argba[b], rgba, (size_t)n * 4, cudaMemcpyHostToDevice, m->copy_stream));
    GEM_CUDA(m, cudaEventRecord(m->ev_h2d[b], m->copy_stream));
    // compute stream: wait for the copy, issue {fold of the previous call || bin of this one}
    GEM_CUDA(m, cudaStreamWaitEvent(m->stream, m->ev_h2d[b], 0));
    if (m->pipe_mode == 1 && m->front_stream) GEM_CUDA(m, cudaStreamWaitEvent(m->front_stream, m->ev_h2d[b], 0));
    const FrameParams fp = make_frame(frame);
    const BinSource in = xyzi_source(m->d_axyzi[b], rgba ? m->d_argba[b] : nullptr, 0);
    const FoldSrc fs{in.xyzi ? (const char *)in.xyzi + 12 : nullptr, 16};
    BinCounters *prev_ctr = m->pend.active ? m->pend.sc.ctr : nullptr;
    if ((rc = enqueue_add<SRC_XYZI>(m, in, fs, n, fp, nullptr, nullptr, true, true, true))) return rc;
    // the step's host-visible result: the counters of the newest call whose fold has been issued
    GEM_CUDA(m, cudaMemcpyAsync(&m->h_ctr_ring[i & 1u], prev_ctr ? prev_ctr : m->ctr_last, sizeof(BinCounters), cudaMemcpyDeviceToHost, m->stream));
    // staging set (i-1) % 3 was last read by the fold just issued (or by this call's own fold in the serial fallback)
    GEM_CUDA(m, cudaEventRecord(m->ev_done[(i + 2u) % 3u], m->stream));
    if (!m->pend.active) GEM_CUDA(m, cudaEventRecord(m->ev_done[b], m->stream));
    memset(&m->stats, 0, sizeof m->stats);
    m->stats.points_in = n; // the rest is fetched by gem_get_stats
    return GEM_OK;
}

int gem_add_cloud_pcl_host(gem_map *m, const void *pts, int n, const gem_frame *frame)
{
    if (!m || !frame || n < 0 || (n > 0 && !pts)) return fail(m, GEM_ERR_INVALID, "gem_add_cloud_pcl_host: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_pcl_staging(m);
    if (rc) return rc;
    const FrameParams fp = make_frame(frame);
    memset(&m->stats, 0, sizeof m->stats);
    if (n == 0) { if ((rc = flush_all_pending(m))) return rc; return gem_sync(m); }
    if ((rc = drain(m))) return rc;
    for (int off = 0; off < n; off += m->P) {
        const int cn = (n - off < m->P) ? (n - off) : m->P;
        GEM_CUDA(m, cudaMemcpyAsync(m->d_pcl, (const char *)pts + (size_t)off * 32, (size_t)cn * 32, cudaMemcpyHostToDevice, m->stream));
        BinSource in{};
        in.pcl = (const float4 *)m->d_pcl;
        const FoldSrc fs{(const char *)in.pcl + 24, 32};
        if ((rc = enqueue_add<SRC_PCL32>(m, in, fs, cn, fp, nullptr, nullptr, false, true, true))) return rc;
        if ((rc = read_counters(m, cn, true))) return rc;
    }
    return GEM_OK;
}

// ---- unfused reference calls ---------------------------------------------------------------
int gem_process_points(gem_map *m, int *map_index, const float *x, const float *y, const float *z, float *var,
                       float *x_ts, float *y_ts, float *z_ts, int n, const gem_frame *frame)
{
    if (!m || !frame || n < 0 || (n > 0 && (!x || !y || !z)))
        return fail(m, GEM_ERR_INVALID, "gem_process_points: bad argument");
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_process_points: not available on tiled handles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_compat_staging(m);
    if (rc) return rc;
    const FrameParams fp = make_frame(frame);
    memset(&m->stats, 0, sizeof m->stats);
    if ((rc = drain(m))) return rc;
    // Process_points does not fuse: clears/floors stay pending (they are handed to the bin kernel only by fusing calls)
    std::vector<RegionOp> keep;
    keep.swap(m->pending);
    for (int off = 0; off < n && rc == GEM_OK; off += m->P) {
        const int cn = (n - off < m->P) ? (n - off) : m->P;
        const size_t b = (size_t)cn * 4;
        cudaError_t e = cudaMemcpyAsync(m->d_x, x + off, b, cudaMemcpyHostToDevice, m->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(m->d_y, y + off, b, cudaMemcpyHostToDevice, m->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(m->d_z, z + off, b, cudaMemcpyHostToDevice, m->stream);
        if (e != cudaSuccess) { rc = fail(m, GEM_ERR_CUDA, cudaGetErrorString(e)); break; }
        BinSource in{};
        in.x = m->d_x; in.y = m->d_y; in.z = m->d_z;
        in.key_out = m->d_keyout; in.h_out = m->d_h; in.hv_out = m->d_hv; in.xt_out = m->d_xt; in.yt_out = m->d_yt;
        const FoldSrc fs{nullptr, 0};
        if ((rc = enqueue_add<SRC_SOA>(m, in, fs, cn, fp, nullptr, nullptr, false, false, true))) break; // lowest-scan only
        if (map_index && e == cudaSuccess) e = cudaMemcpyAsync(map_index + off, m->d_keyout, b, cudaMemcpyDeviceToHost, m->stream);
        if (var && e == cudaSuccess) e = cudaMemcpyAsync(var + off, m->d_hv, b, cudaMemcpyDeviceToHost, m->stream);
        if (z_ts && e == cudaSuccess) e = cudaMemcpyAsync(z_ts + off, m->d_h, b, cudaMemcpyDeviceToHost, m->stream);
        if (x_ts && e == cudaSuccess) e = cudaMemcpyAsync(x_ts + off, m->d_xt, b, cudaMemcpyDeviceToHost, m->stream);
        if (y_ts && e == cudaSuccess) e = cudaMemcpyAsync(y_ts + off, m->d_yt, b, cudaMemcpyDeviceToHost, m->stream);
        if (e != cudaSuccess) { rc = fail(m, GEM_ERR_CUDA, cudaGetErrorString(e)); break; }
        rc = read_counters(m, cn, true);
    }
    m->pending.insert(m->pending.begin(), keep.begin(), keep.end());
    return rc;
}

int gem_fuse(gem_map *m, int n, const int *index, const int *R, const int *G, const int *B, const float *intensity,
             const float *height, const float *var)
{
    if (!m || n < 0 || (n > 0 && (!index || !height || !var))) return fail(m, GEM_ERR_INVALID, "gem_fuse: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_compat_staging(m);
    if (rc) return rc;
    memset(&m->stats, 0, sizeof m->stats);
    if (n == 0) { if ((rc = flush_all_pending(m))) return rc; return gem_sync(m); }
    if ((rc = drain(m))) return rc;
    for (int off = 0; off < n; off += m->P) {
        const int cn = (n - off < m->P) ? (n - off) : m->P;
        const size_t b = (size_t)cn * 4;
        GEM_CUDA(m, cudaMemcpyAsync(m->d_keyin, index + off, b, cudaMemcpyHostToDevice, m->stream));
        GEM_CUDA(m, cudaMemcpyAsync(m->d_h, height + off, b, cudaMemcpyHostToDevice, m->stream));
        GEM_CUDA(m, cudaMemcpyAsync(m->d_hv, var + off, b, cudaMemcpyHostToDevice, m->stream));
        BinSource in{};
        in.key_in = m->d_keyin; in.h_in = m->d_h; in.hv_in = m->d_hv; in.ncells = (int)m->nc;
        if (R) { GEM_CUDA(m, cudaMemcpyAsync(m->d_R, R + off, b, cudaMemcpyHostToDevice, m->stream)); in.R = m->d_R; }
        if (G) { GEM_CUDA(m, cudaMemcpyAsync(m->d_G, G + off, b, cudaMemcpyHostToDevice, m->stream)); in.G = m->d_G; }
        if (B) { GEM_CUDA(m, cudaMemcpyAsync(m->d_B, B + off, b, cudaMemcpyHostToDevice, m->stream)); in.B = m->d_B; }
        if (intensity) {
            GEM_CUDA(m, cudaMemcpyAsync(m->d_int, intensity + off, b, cudaMemcpyHostToDevice, m->stream));
            in.inten_in = m->d_int;
        }
        const FoldSrc fs{(const char *)in.inten_in, 4};
        const FrameParams none{};
        if ((rc = enqueue_add<SRC_KEYS>(m, in, fs, cn, none, nullptr, nullptr, false, true, false))) return rc;
        if ((rc = read_counters(m, cn, true))) return rc;
    }
    return GEM_OK;
}

int gem_var_update(gem_map *m, float dv)
{
    if (!m) return GEM_ERR_INVALID;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    // x + 0.0f == x for every non-NaN x: the GEM node always passes 0 (ElevationMapping.cpp:944-945)
    if (dv == 0.0f) return GEM_OK;
    { int rcf = flush_for_observer(m); if (rcf) return rcf; }
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_var_update<<<blocks_for(m->nc, 256), 256, 0, m->stream>>>(m->ml, m->nc, dv));
    if (dv < 0.0f) pend_all_floor(m); // variances may drop below the floor: next Fuse floors every cell
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}

int gem_compute_features(gem_map *m)
{
    if (!m) return GEM_ERR_INVALID;
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_compute_features: tiled handles take the halo-padded tile: use gem_compute_features_tiled");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    { int rcf = flush_for_observer(m); if (rcf) return rcf; }
    GEM_LAUNCH(m, GEM_PROF_FEATURES, k_features<false><<<dim3((m->geom.cols + FEAT_TILE - 1) / FEAT_TILE, (m->geom.rows + FEAT_TILE - 1) / FEAT_TILE), FEAT_TILE * FEAT_TILE, 0, m->stream>>>(m->geom, m->ml, nullptr));
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}

static int copy_layer_out(gem_map *m, int layer, void *host, int slot)
{
    { int rcf = flush_for_observer(m); if (rcf) return rcf; }
    float *dst = m->d_out + (size_t)slot * m->nc;
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_unpack_layer<<<blocks_for(m->nc, 256), 256, 0, m->stream>>>(m->ml, m->nc, layer, dst));
    GEM_CUDA(m, cudaGetLastError());
    GEM_CUDA(m, cudaMemcpyAsync(host, dst, m->nc * 4, cudaMemcpyDeviceToHost, m->stream));
    return GEM_OK;
}

int gem_map_feature(gem_map *m, float *elevation, float *var, int *R, int *G, int *B, float *rough, float *slope,
                    float *traver, float *intensity)
{
    if (!m) return GEM_ERR_INVALID;
    Lock lk(m->mu);
    int rc = gem_compute_features(m);
    if (rc) return rc;
    SetDev sd(m->dev);
    if ((rc = ensure_out_staging(m))) return rc;
    struct { void *p; int layer; } outs[9] = {{elevation, 0}, {var, 1}, {R, 3}, {G, 4}, {B, 5},
                                              {rough, 8}, {slope, 9}, {traver, 10}, {intensity, 2}};
    for (int k = 0; k < 9; k++)
        if (outs[k].p && (rc = copy_layer_out(m, outs[k].layer, outs[k].p, k))) return rc;
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    return GEM_OK;
}

int gem_get_layer_device(gem_map *m, int layer, void *out_device)
{
    if (!m || !out_device || layer < 0 || layer > 10) return fail(m, GEM_ERR_INVALID, "gem_get_layer_device: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    { int rcf = flush_for_observer(m); if (rcf) return rcf; }
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_unpack_layer<<<blocks_for(m->nc, 256), 256, 0, m->stream>>>(m->ml, m->nc, layer, out_device));
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}

int gem_compute_features_tiled(gem_map *m, const float *padded_elevation)
{
    if (!m || !padded_elevation) return fail(m, GEM_ERR_INVALID, "gem_compute_features_tiled: bad argument");
    if (!m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_compute_features_tiled: handle is not tiled");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    { int rcf = flush_for_observer(m); if (rcf) return rcf; }
    GEM_LAUNCH(m, GEM_PROF_FEATURES, k_features<true><<<dim3((m->geom.cols + FEAT_TILE - 1) / FEAT_TILE, (m->geom.rows + FEAT_TILE - 1) / FEAT_TILE), FEAT_TILE * FEAT_TILE, 0, m->stream>>>(m->geom, m->ml, padded_elevation));
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}

int gem_raytracing_tiled(gem_map *m, const float *global_lowest)
{
    if (!m || !global_lowest) return fail(m, GEM_ERR_INVALID, "gem_raytracing_tiled: bad argument");
    if (!m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_raytracing_tiled: handle is not tiled");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    { int rcf = flush_for_observer(m); if (rcf) return rcf; }
    const size_t ng = (size_t)m->L * m->L;
    { int rc = ensure_ray_scratch(m, ng); if (rc) return rc; }
    int *ray_count = m->d_raylist + m->nc;
    GEM_CUDA(m, cudaMemsetAsync(ray_count, 0, sizeof(int), m->stream));
    MapLayers mlg = m->ml;
    mlg.lowest = const_cast<float *>(global_lowest); // rays probe the replicated, map-wide lowest layer
    GEM_LAUNCH(m, GEM_PROF_RAYTRACE, k_ray_collect<<<blocks_for(m->nc, 256, 1 << 30), 256, 0, m->stream>>>(m->geom, m->ml, m->cfg.obstacle_threshold, m->d_raylist, ray_count));
    GEM_LAUNCH(m, GEM_PROF_RAYTRACE, k_lowest_bitmap<<<blocks_for(ng, 256, 1 << 30), 256, 0, m->stream>>>(global_lowest, (int)ng, m->d_bitmap));
    GEM_LAUNCH(m, GEM_PROF_RAYTRACE, k_ray_trace<<<NUM_SMS * 8, 256, 0, m->stream>>>(m->geom, mlg, m->d_bitmap, m->sensorZ, m->d_raylist, ray_count));
    GEM_LAUNCH(m, GEM_PROF_CLEAR, k_fill<<<blocks_for(m->nc, 256), 256, 0, m->stream>>>(m->ml.lowest, m->nc, 10.0f)); // own tile's lowest
    GEM_CUDA(m, cudaGetLastError());
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    return GEM_OK;
}

int gem_raytracing(gem_map *m)
{
    if (!m) return GEM_ERR_INVALID;
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_raytracing: tiled handles take the map-wide lowest layer: use gem_raytracing_tiled");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    { int rcf = flush_for_observer(m); if (rcf) return rcf; }
    { int rc = ensure_ray_scratch(m, m->nc); if (rc) return rc; }
    int *ray_count = m->d_raylist + m->nc; // the list's length lives behind it
    GEM_CUDA(m, cudaMemsetAsync(ray_count, 0, sizeof(int), m->stream));
    GEM_LAUNCH(m, GEM_PROF_RAYTRACE, k_ray_collect<<<blocks_for(m->nc, 256, 1 << 30), 256, 0, m->stream>>>(m->geom, m->ml, m->cfg.obstacle_threshold, m->d_raylist, ray_count));
    uint32_t *bitmap = m->d_bitmap;
    GEM_LAUNCH(m, GEM_PROF_RAYTRACE, k_lowest_bitmap<<<blocks_for(m->nc, 256, 1 << 30), 256, 0, m->stream>>>(m->ml.lowest, (int)m->nc, bitmap));
    GEM_LAUNCH(m, GEM_PROF_RAYTRACE, k_ray_trace<<<NUM_SMS * 8, 256, 0, m->stream>>>(m->geom, m->ml, bitmap, m->sensorZ, m->d_raylist, ray_count));
    GEM_LAUNCH(m, GEM_PROF_CLEAR, k_fill<<<blocks_for(m->nc, 256), 256, 0, m->stream>>>(m->ml.lowest, m->nc, 10.0f)); // G_Clear_maplowest
    GEM_CUDA(m, cudaGetLastError());
    GEM_CUDA(m, cudaStreamSynchronize(m->stream)); // gpu.cu:1312
    return GEM_OK;
}

int gem_opt_move(gem_map *m, const float opt_p[2], float height_update, float aligned_out[2])
{
    if (!m || !opt_p) return GEM_ERR_INVALID;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    float c[2] = {m->geom.cx, m->geom.cy};
    for (int i = 0; i < 2; i++) { // alignedPosition gpu.cu:1203-1213
        const float ps = opt_p[i] - c[i];
        const int is = d2i_host((double)(ps / m->geom.res) + 0.5 * (ps > 0 ? 1 : -1));
        c[i] = c[i] + m->geom.res * (float)is;
        if (aligned_out) aligned_out[i] = c[i];
    }
    m->geom.cx = c[0]; m->geom.cy = c[1];
    { int rcf = flush_for_observer(m); if (rcf) return rcf; }
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_add_height<<<blocks_for(m->nc, 256), 256, 0, m->stream>>>(m->ml, m->nc, height_update));
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}

int gem_closeloop(gem_map *m, const float up[2], float height_update)
{
    if (!m || !up) return GEM_ERR_INVALID;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    float c[2] = {m->geom.cx, m->geom.cy};
    for (int i = 0; i < 2; i++) { // gpu.cu:1242-1247
        const float ps = up[i] - c[i];
        const int is = d2i_host((double)(ps / m->geom.res) + 0.5 * (ps > 0 ? 1 : -1));
        const float aligned = (float)is * m->geom.res;
        c[i] = position_to_range(c[i], aligned, m->geom.res);
    }
    m->geom.cx = c[0]; m->geom.cy = c[1];
    { int rcf = flush_for_observer(m); if (rcf) return rcf; }
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_add_height<<<blocks_for(m->nc, 256), 256, 0, m->stream>>>(m->ml, m->nc, height_update));
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}

int gem_colourise_points(gem_map *m, void *xyzi, int n, const double Tc[12], const double Tl[16], const unsigned char *bgr,
                         int width, int height, int row_stride, void *rgba_out)
{
    if (!m || n < 0 || (n > 0 && (!xyzi || !rgba_out)) || !Tc || !Tl || !bgr || width < 1 || height < 1 || row_stride < 3 * width)
        return fail(m, GEM_ERR_INVALID, "gem_colourise_points: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    ProjParams pp;
    for (int i = 0; i < 3; i++) // P_lidar2img = Tcamera * TLidar (ElevationMapping.cpp:347), double, left-to-right sums
        for (int j = 0; j < 4; j++) {
            double a = Tc[4 * i + 0] * Tl[0 + j];
            for (int k = 1; k < 4; k++) a = a + Tc[4 * i + k] * Tl[4 * k + j];
            pp.P[4 * i + j] = a;
        }
    pp.width = width; pp.height = height; pp.row_stride = row_stride;
    if (n > 0)
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_colourise<<<blocks_for((size_t)n, 256), 256, 0, m->stream>>>((float4 *)xyzi, n, pp, bgr, (uchar4 *)rgba_out));
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}

int gem_export_layers(gem_map *m, float *host_layers[9])
{
    if (!m || !host_layers) return GEM_ERR_INVALID;
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_export_layers: not available on tiled handles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_out_staging(m);
    if (rc) return rc;
    if ((rc = flush_for_observer(m))) return rc;
    dim3 grid((m->L + 31) / 32, (m->L + 31) / 32);
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_export_colmajor<<<grid, 256, 0, m->stream>>>(m->ml, m->L, m->d_out));
    GEM_CUDA(m, cudaGetLastError());
    for (int k = 0; k < 9; k++)
        if (host_layers[k])
            GEM_CUDA(m, cudaMemcpyAsync(host_layers[k], m->d_out + (size_t)k * m->nc, m->nc * 4, cudaMemcpyDeviceToHost, m->stream));
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    return GEM_OK;
}

// The write-back in two halves: _begin runs the export kernel and starts the device-to-host copies on the copy stream,
// _end waits for them.  Between the two the caller can issue work that does not change what was exported -- the node
// calls Raytracing right after Map_feature + show() (ElevationMapping.cpp:404-421), and the ray clean-up does not
// touch the staging buffer -- so the 4 * 9 * L^2 bytes cross PCIe while the rays are traced.
int gem_export_layers_begin(gem_map *m, float *host_layers[9])
{
    if (!m || !host_layers) return GEM_ERR_INVALID;
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_export_layers_begin: not available on tiled handles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_out_staging(m);
    if (rc) return rc;
    if ((rc = flush_for_observer(m))) return rc;
    if (!m->copy_stream) GEM_CUDA(m, cudaStreamCreateWithFlags(&m->copy_stream, cudaStreamNonBlocking));
    if (!m->ev_export) GEM_CUDA(m, cudaEventCreateWithFlags(&m->ev_export, cudaEventDisableTiming));
    if (!m->ev_export_done) GEM_CUDA(m, cudaEventCreateWithFlags(&m->ev_export_done, cudaEventDisableTiming));
    dim3 grid((m->L + 31) / 32, (m->L + 31) / 32);
    GEM_CUDA(m, cudaStreamWaitEvent(m->stream, m->ev_export_done, 0)); // the previous export's copies have left the staging buffer
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_export_colmajor<<<grid, 256, 0, m->stream>>>(m->ml, m->L, m->d_out));
    GEM_CUDA(m, cudaGetLastError());
    GEM_CUDA(m, cudaEventRecord(m->ev_export, m->stream));
    GEM_CUDA(m, cudaStreamWaitEvent(m->copy_stream, m->ev_export, 0));
    for (int k = 0; k < 9; k++)
        if (host_layers[k])
            GEM_CUDA(m, cudaMemcpyAsync(host_layers[k], m->d_out + (size_t)k * m->nc, m->nc * 4, cudaMemcpyDeviceToHost, m->copy_stream));
    GEM_CUDA(m, cudaEventRecord(m->ev_export_done, m->copy_stream));
    return GEM_OK;
}
int gem_export_layers_end(gem_map *m)
{
    if (!m) return GEM_ERR_INVALID;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    if (m->ev_export_done) GEM_CUDA(m, cudaEventSynchronize(m->ev_export_done));
    return GEM_OK;
}

int gem_export_orthomosaic(gem_map *m, unsigned char *host_bgr)
{
    if (!m || !host_bgr) return fail(m, GEM_ERR_INVALID, "gem_export_orthomosaic: null argument");
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_export_orthomosaic: not available on tiled handles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_out_staging(m);
    if (rc) return rc;
    if ((rc = flush_for_observer(m))) return rc;
    unsigned char *d_img = reinterpret_cast<unsigned char *>(m->d_out);
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_orthomosaic<<<blocks_for((m->nc + 3) / 4, 256, 1 << 30), 256, 0, m->stream>>>(m->geom, m->ml, d_img));
    GEM_CUDA(m, cudaGetLastError());
    GEM_CUDA(m, cudaMemcpyAsync(host_bgr, d_img, m->nc * 3, cudaMemcpyDeviceToHost, m->stream));
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    return GEM_OK;
}

int gem_export_visual_points(gem_map *m, float *host_xyz, unsigned char *host_rgb, int capacity, int *count_out)
{
    if (!m || !count_out || capacity < 0 || (capacity > 0 && (!host_xyz || !host_rgb)))
        return fail(m, GEM_ERR_INVALID, "gem_export_visual_points: bad argument");
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_export_visual_points: not available on tiled handles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_out_staging(m);
    if (rc) return rc;
    if ((rc = flush_for_observer(m))) return rc;
    // staging (9 floats per cell): xyz = 3 floats per cell, rgb = 3 bytes per cell behind it
    VisualSrc src;
    src.ml = m->ml;
    src.f = grid_frame(m, m->geom.cx, m->geom.cy, m->geom.sx, m->geom.sy);
    src.xyz = m->d_out;
    src.rgb = reinterpret_cast<unsigned char *>(m->d_out + 3 * m->nc);
    const int cap = (int)std::min<size_t>((size_t)capacity, m->nc);
    int total = 0;
    if ((rc = compact_cells(m, src, cap, &total))) return rc;
    *count_out = total; // the number of shown cells; only min(total, capacity) points are written
    const size_t n = (size_t)std::min(total, cap);
    if (n) {
        GEM_CUDA(m, cudaMemcpyAsync(host_xyz, src.xyz, n * 12, cudaMemcpyDeviceToHost, m->stream));
        GEM_CUDA(m, cudaMemcpyAsync(host_rgb, src.rgb, n * 3, cudaMemcpyDeviceToHost, m->stream));
        GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    }
    return GEM_OK;
}

int gem_snapshot_shown(gem_map *m)
{
    if (!m) return GEM_ERR_INVALID;
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_snapshot_shown: not available on tiled handles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc;
    if ((rc = flush_for_observer(m))) return rc;
    if (!m->prev_ev) {
        if ((rc = dev_alloc(m, &m->prev_ev, m->nc)) || (rc = dev_alloc(m, &m->prev_ci, m->nc)) || (rc = dev_alloc(m, &m->prev_tr, m->nc))) return rc;
    }
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_snapshot_shown<<<blocks_for(m->nc, 256), 256, 0, m->stream>>>(m->ml, m->nc, m->prev_ev, m->prev_ci, m->prev_tr));
    GEM_CUDA(m, cudaGetLastError());
    m->prev_geom = m->geom;
    m->prev_valid = true;
    return GEM_OK;
}

// the harvest of :716-765 into the read-out staging buffer (the first `cap` records); the caller holds the lock
static int harvest_to_staging(gem_map *m, const float current_xy[2], const float shift_xy[2], int cap, int *total)
{
    int rc = ensure_out_staging(m);
    if (rc) return rc;
    HarvestSrc src;
    src.s = snapshot_cells(m->prev_ev, m->prev_ci, m->prev_tr);
    src.f = grid_frame(m, m->prev_geom.cx, m->prev_geom.cy, m->prev_geom.sx, m->prev_geom.sy);
    // :727-734: current_x (float) -+ length_ * resolution_ / 2 with the node's double resolution_
    const double halfwin = (double)m->L * src.f.res / 2;
    src.lox = (double)current_xy[0] - halfwin; src.hix = (double)current_xy[0] + halfwin;
    src.loy = (double)current_xy[1] - halfwin; src.hiy = (double)current_xy[1] + halfwin;
    src.dx = shift_xy[0]; src.dy = shift_xy[1];
    src.out = reinterpret_cast<float4 *>(m->d_out); // 8 of the 9 staging floats per cell
    return compact_cells(m, src, cap, total);
}

int gem_harvest_scrolled_out(gem_map *m, const float current_xy[2], const float shift_xy[2], void *host_points32,
                             int capacity, int *count_out)
{
    if (!m || !current_xy || !shift_xy || !count_out || capacity < 0 || (capacity > 0 && !host_points32))
        return fail(m, GEM_ERR_INVALID, "gem_harvest_scrolled_out: bad argument");
    if (!m->prev_valid) return fail(m, GEM_ERR_INVALID, "gem_harvest_scrolled_out: no snapshot (call gem_snapshot_shown first)");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    const int cap = (int)std::min<size_t>((size_t)capacity, m->nc);
    int total = 0, rc;
    if ((rc = harvest_to_staging(m, current_xy, shift_xy, cap, &total))) return rc;
    *count_out = total;
    const size_t n = (size_t)std::min(total, cap);
    if (n) {
        GEM_CUDA(m, cudaMemcpyAsync(host_points32, m->d_out, n * 32, cudaMemcpyDeviceToHost, m->stream));
        GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    }
    return GEM_OK;
}

int gem_export_grid_cloud(gem_map *m, int source, void *points32_device, int capacity, int *count_out)
{
    if (!m || !count_out || capacity < 0 || (capacity > 0 && !points32_device) || (source != GEM_GRID_SHOWN && source != GEM_GRID_SNAPSHOT))
        return fail(m, GEM_ERR_INVALID, "gem_export_grid_cloud: bad argument");
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_export_grid_cloud: not available on tiled handles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    if (source == GEM_GRID_SNAPSHOT && !m->prev_valid)
        return fail(m, GEM_ERR_INVALID, "gem_export_grid_cloud: no snapshot (call gem_snapshot_shown first)");
    int rc = flush_for_observer(m);
    if (rc) return rc;
    GridCloudSrc src;
    const MapGeom &g = source == GEM_GRID_SHOWN ? m->geom : m->prev_geom;
    src.s = source == GEM_GRID_SHOWN ? live_cells(m->ml) : snapshot_cells(m->prev_ev, m->prev_ci, m->prev_tr);
    src.f = grid_frame(m, g.cx, g.cy, g.sx, g.sy);
    src.out = reinterpret_cast<float4 *>(points32_device);
    int total = 0;
    if ((rc = compact_cells(m, src, (int)std::min<size_t>((size_t)capacity, m->nc), &total))) return rc;
    *count_out = total; // the number of cells taken; min(total, capacity) records are written
    return GEM_OK;
}

// composingGlobalMap's numeric block (ElevationMapping.cpp:1152-1170): statistical outlier removal over the grid cloud,
// then the road / obstacle split of the survivors (gem_global.cuh, DESIGN.md f6)
int gem_grid_cloud_split(gem_map *m, int source, int mean_k, double stddev_mul, double travers_threshold,
                         void *road_points32_device, int road_capacity, void *obstacle_points32_device, int obstacle_capacity,
                         float *mean_distance_device, int distance_capacity, gem_grid_split *out)
{
    if (!m || !out || (source != GEM_GRID_SHOWN && source != GEM_GRID_SNAPSHOT) || road_capacity < 0 || obstacle_capacity < 0 ||
        distance_capacity < 0 || (road_capacity > 0 && !road_points32_device) || (obstacle_capacity > 0 && !obstacle_points32_device) ||
        (distance_capacity > 0 && !mean_distance_device))
        return fail(m, GEM_ERR_INVALID, "gem_grid_cloud_split: bad argument");
    if (mean_k < 1 || mean_k > SPLIT_MAX_K) return fail(m, GEM_ERR_INVALID, "gem_grid_cloud_split: mean_k must be in [1, 64]");
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_grid_cloud_split: not available on tiled handles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    if (source == GEM_GRID_SNAPSHOT && !m->prev_valid)
        return fail(m, GEM_ERR_INVALID, "gem_grid_cloud_split: no snapshot (call gem_snapshot_shown first)");
    int rc = flush_for_observer(m);
    if (rc) return rc;
    const int L = m->L;
    if (!m->split_stats) { // the scratch is published only once every buffer exists (a failed call leaves it unset)
        float *zg, *xg, *yg, *dcell, *dist;
        int *queue, *ctr;
        SplitStats *st;
        if ((rc = dev_alloc(m, &zg, m->nc)) || (rc = dev_alloc(m, &xg, (size_t)L)) || (rc = dev_alloc(m, &yg, (size_t)L)) ||
            (rc = dev_alloc(m, &dcell, m->nc)) || (rc = dev_alloc(m, &dist, m->nc)) || (rc = dev_alloc(m, &queue, m->nc)) ||
            (rc = dev_alloc(m, &ctr, 2)) || (rc = dev_alloc(m, &st, 1)))
            return rc;
        m->split_zg = zg; m->split_xg = xg; m->split_yg = yg; m->split_dcell = dcell; m->split_dist = dist;
        m->split_queue = queue; m->split_ctr = ctr; m->split_stats = st;
    }
    GridCloudSrc g;
    const MapGeom &geo = source == GEM_GRID_SHOWN ? m->geom : m->prev_geom;
    g.s = source == GEM_GRID_SHOWN ? live_cells(m->ml) : snapshot_cells(m->prev_ev, m->prev_ci, m->prev_tr);
    g.f = grid_frame(m, geo.cx, geo.cy, geo.sx, geo.sy);
    g.out = nullptr;
    GEM_CUDA(m, cudaMemsetAsync(m->split_ctr, 0, 2 * sizeof(int), m->stream));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_split_stage<<<blocks_for(m->nc, 256), 256, 0, m->stream>>>(g, m->split_zg, m->split_xg, m->split_yg, m->split_dcell));
    const int nt = (L + SPLIT_TILE - 1) / SPLIT_TILE;
    const dim3 grid(nt, nt);
    const int K = mean_k + 1;
    // the queue's length stays on the device: k_split_knn_far's fixed grid strides over it
#define GEM_SPLIT_KNN(KC)                                                                                                              \
    do {                                                                                                                               \
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_split_knn<KC><<<grid, SPLIT_TILE * SPLIT_TILE, 0, m->stream>>>(m->split_zg, m->split_xg, m->split_yg, L, geo.sx, geo.sy, mean_k, m->split_dcell, m->split_queue, m->split_ctr)); \
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_split_knn_far<KC><<<NUM_SMS * 4, 128, 0, m->stream>>>(m->split_zg, m->split_xg, m->split_yg, L, geo.sx, geo.sy, mean_k, m->split_dcell, m->split_queue, m->split_ctr)); \
    } while (0)
    if (K <= 8) GEM_SPLIT_KNN(8);
    else if (K <= 24) GEM_SPLIT_KNN(24);
    else GEM_SPLIT_KNN(SPLIT_MAX_K + 1);
#undef GEM_SPLIT_KNN
    GEM_CUDA(m, cudaGetLastError());
    // distances in cloud order -> statistics -> road -> obstacle, all on the stream; the three counts are copied beside
    // the statistics on the device, and the call waits once, for the one small read-back
    SplitStats *dst = m->split_stats;
    int *d_total = nullptr;
    SplitDistSrc ds{g, m->split_dcell, m->split_dist, mean_distance_device, distance_capacity};
    if ((rc = compact_cells_issue(m, ds, (int)m->nc, &d_total))) return rc;
    GEM_CUDA(m, cudaMemcpyAsync(&dst->points, d_total, sizeof(int), cudaMemcpyDeviceToDevice, m->stream));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_split_stats<<<1, 32, 0, m->stream>>>(m->split_dist, &dst->points, m->split_ctr, mean_k, stddev_mul, dst,
                                                                         mean_distance_device, distance_capacity));
    GEM_CUDA(m, cudaGetLastError());
    SplitSrc rs{g, m->split_dcell, dst, travers_threshold, 1};
    rs.g.out = reinterpret_cast<float4 *>(road_points32_device);
    if ((rc = compact_cells_issue(m, rs, (int)std::min<size_t>((size_t)road_capacity, m->nc), &d_total))) return rc;
    GEM_CUDA(m, cudaMemcpyAsync(&dst->road, d_total, sizeof(int), cudaMemcpyDeviceToDevice, m->stream));
    SplitSrc os{g, m->split_dcell, dst, travers_threshold, 0};
    os.g.out = reinterpret_cast<float4 *>(obstacle_points32_device);
    if ((rc = compact_cells_issue(m, os, (int)std::min<size_t>((size_t)obstacle_capacity, m->nc), &d_total))) return rc;
    GEM_CUDA(m, cudaMemcpyAsync(&dst->obstacle, d_total, sizeof(int), cudaMemcpyDeviceToDevice, m->stream));
    SplitStats st;
    GEM_CUDA(m, cudaMemcpyAsync(&st, dst, sizeof st, cudaMemcpyDeviceToHost, m->stream));
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    out->points = st.points;
    out->valid = st.valid;
    out->road = st.road;
    out->obstacle = st.obstacle;
    out->mean = st.mean;
    out->stddev = st.stddev;
    out->threshold = st.threshold;
    return GEM_OK;
}

// Grow a device scratch buffer (octree, costmap, voxel grid) to at least `bytes`, with a quarter of slack and at least
// 4 KiB so that slowly growing inputs do not reallocate on every call.  The new buffer is allocated before the old one is
// released, so a failed growth leaves the buffer as it was; the stream is drained before the old buffer goes, because
// work queued on it (an update_origin, say) may still read it.
static int scratch_grow(gem_map *m, OctBuf &b, size_t bytes, const char *what)
{
    if (b.cap >= bytes) return GEM_OK;
    bytes = std::max(bytes + bytes / 4, (size_t)4096);
    void *q = nullptr;
    const cudaError_t e = cudaMalloc(&q, bytes);
    if (e != cudaSuccess) return fail(m, GEM_ERR_NOMEM, std::string(what) + ": cudaMalloc: " + cudaGetErrorString(e));
    if (b.p) {
        cudaStreamSynchronize(m->stream);
        cudaFree(b.p);
    }
    b.p = q;
    b.cap = bytes;
    return GEM_OK;
}
static int oct_grow(gem_map *m, OctBuf &b, size_t bytes) { return scratch_grow(m, b, bytes, "gem_color_octree"); }

// pointCloudtoOctomap's tree (ElevationMapping.cpp:1157-1174) as the ColorOcTree::writeData stream (gem_octree.cuh,
// DESIGN.md f7)
int gem_color_octree(gem_map *m, const void *points32_device, int n, double resolution, gem_octree *info)
{
    if (!m || !info || n < 0 || (n > 0 && !points32_device)) return fail(m, GEM_ERR_INVALID, "gem_color_octree: bad argument");
    if (!std::isfinite(resolution) || !(resolution > 0.0))
        return fail(m, GEM_ERR_INVALID, "gem_color_octree: resolution must be finite and positive");
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_color_octree: not available on tiled handles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    OctScratch &S = m->oct;
    S.bytes = -1; // the buffers of the last stream are overwritten from here on
    gem_octree r{};
    if (n == 0) {
        S.bytes = 0;
        S.info = r;
        *info = r;
        return GEM_OK;
    }
    // O2: the constants and the value states, with the host's libm as octomap computes them
    OctParams P{};
    {
        const float hit = (float)std::log(0.7 / 0.3), vmax = (float)std::log(0.971 / 0.029);
        float v = 0.0f;
        int s = 0;
        while (!(v >= vmax) && s + 1 < OCT_STATES) {
            v = v + hit;
            if (v > vmax) v = vmax;
            P.v[++s] = v;
            P.p[s] = 1.0 - 1.0 / (1.0 + std::exp((double)v));
            P.q[s] = 0.99 - P.p[s];
        }
        P.sat = s;
    }
    const double rf = 1.0 / resolution;
    const size_t N = (size_t)n;
    using u64 = unsigned long long;
    cudaStream_t st = m->stream;
    int rc;
    // phase 1: keys, the sort by code, the leaves and their runs, the classification (sizes of phase 2)
    size_t t_sort = 0, t_rle = 0, t_scan = 0;
    GEM_CUDA(m, cub::DeviceRadixSort::SortPairs(nullptr, t_sort, (u64 *)nullptr, (u64 *)nullptr, (int *)nullptr, (int *)nullptr, n, 0, 49, st));
    GEM_CUDA(m, cub::DeviceRunLengthEncode::Encode(nullptr, t_rle, (u64 *)nullptr, (u64 *)nullptr, (int *)nullptr, (int *)nullptr, n, st));
    GEM_CUDA(m, cub::DeviceScan::ExclusiveSum(nullptr, t_scan, (int *)nullptr, (int *)nullptr, n, st));
    if ((rc = oct_grow(m, S.code[0], N * 8)) || (rc = oct_grow(m, S.code[1], N * 8)) || (rc = oct_grow(m, S.idx[0], N * 4)) ||
        (rc = oct_grow(m, S.idx[1], N * 4)) || (rc = oct_grow(m, S.leaf, N * 8)) || (rc = oct_grow(m, S.cnt, N * 4)) ||
        (rc = oct_grow(m, S.off, N * 4)) || (rc = oct_grow(m, S.level, N * 4)) || (rc = oct_grow(m, S.ghead, N * 4)) ||
        (rc = oct_grow(m, S.gid, N * 4)) || (rc = oct_grow(m, S.val, N * 4)) ||
        (rc = oct_grow(m, S.groups, (N / 8 + 1) * sizeof(OctGroup))) || (rc = oct_grow(m, S.ctr, sizeof(OctCounters))) ||
        (rc = oct_grow(m, S.temp, std::max(t_sort, std::max(t_rle, t_scan)))))
        return rc;
    const float4 *pts = static_cast<const float4 *>(points32_device);
    OctCounters *ctr = S.ctr.as<OctCounters>();
    u64 *leaf = S.leaf.as<u64>();
    int *cnt = S.cnt.as<int>(), *off = S.off.as<int>(), *level = S.level.as<int>(), *sidx = S.idx[1].as<int>();
    uint32_t *val = S.val.as<uint32_t>();
    size_t tcap = S.temp.cap;
    GEM_CUDA(m, cudaMemsetAsync(ctr, 0, sizeof(OctCounters), st));
    // the run-length encoding writes nruns <= n counts (a device-side number); the scan below runs over all n, so the
    // rest must be defined
    GEM_CUDA(m, cudaMemsetAsync(cnt, 0, N * sizeof(int), st));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_oct_keys<<<blocks_for(N, 256, 1 << 30), 256, 0, st>>>(pts, n, rf, S.code[0].as<u64>(), S.idx[0].as<int>(), ctr));
    GEM_CUDA(m, cudaGetLastError());
    GEM_CUDA(m, cub::DeviceRadixSort::SortPairs(S.temp.p, tcap, S.code[0].as<u64>(), S.code[1].as<u64>(), S.idx[0].as<int>(), sidx, n, 0, 49, st));
    GEM_CUDA(m, cub::DeviceRunLengthEncode::Encode(S.temp.p, tcap, S.code[1].as<u64>(), leaf, cnt, &ctr->nruns, n, st));
    GEM_CUDA(m, cub::DeviceScan::ExclusiveSum(S.temp.p, tcap, cnt, off, n, st));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_oct_classify<<<blocks_for(N, 256, 1 << 30), 256, 0, st>>>(leaf, cnt, off, sidx, pts, P, level, S.ghead.as<int>(), S.gid.as<int>(),
                                                                                             S.groups.as<OctGroup>(), val, ctr, n));
    GEM_CUDA(m, cudaGetLastError());
    OctCounters hc;
    GEM_CUDA(m, cudaMemcpyAsync(&hc, ctr, sizeof hc, cudaMemcpyDeviceToHost, st));
    GEM_CUDA(m, cudaStreamSynchronize(st));
    // phase 2: the groups, the nodes above them, the preorder sort
    const int nleaf = hc.inserted > 0 ? hc.nruns - (hc.inserted < n) : 0;
    const size_t ngp = (size_t)hc.grouped, nnode = (size_t)hc.upper + (size_t)hc.indep + (size_t)hc.dense;
    if (nnode > (size_t)INT32_MAX) return fail(m, GEM_ERR_INVALID, "gem_color_octree: too many nodes");
    if (nnode > 0) {
        int gbits = 0;
        while ((1ll << gbits) < (long long)hc.groups) gbits++;
        size_t t_keys = 0, t_nodes = 0;
        GEM_CUDA(m, cub::DeviceRadixSort::SortKeys(nullptr, t_keys, (u64 *)nullptr, (u64 *)nullptr, (int)ngp, 0, 32 + gbits, st));
        GEM_CUDA(m, cub::DeviceRadixSort::SortPairs(nullptr, t_nodes, (u64 *)nullptr, (u64 *)nullptr, (u64 *)nullptr, (u64 *)nullptr, (int)nnode, 0, 53, st));
        if ((rc = oct_grow(m, S.key2[0], ngp * 8)) || (rc = oct_grow(m, S.key2[1], ngp * 8)) || (rc = oct_grow(m, S.nkey[0], nnode * 8)) ||
            (rc = oct_grow(m, S.nkey[1], nnode * 8)) || (rc = oct_grow(m, S.nrec[0], nnode * 8)) || (rc = oct_grow(m, S.nrec[1], nnode * 8)) ||
            (rc = oct_grow(m, S.dense, (size_t)hc.dense * 4)) || (rc = oct_grow(m, S.temp, std::max(t_keys, t_nodes))))
            return rc;
        tcap = S.temp.cap;
        u64 *nkey = S.nkey[0].as<u64>(), *nrec = S.nrec[0].as<u64>();
        GEM_CUDA(m, cudaMemsetAsync(nkey, 0xFF, nnode * 8, st)); // OCT_EMPTY: unused group slots sort last
        if (ngp) {
            GEM_CUDA(m, cudaMemsetAsync(S.dense.p, 0, (size_t)hc.dense * 4, st));
            GEM_LAUNCH(m, GEM_PROF_OTHER, k_oct_group_keys<<<blocks_for((size_t)nleaf, 256, 1 << 30), 256, 0, st>>>(leaf, nleaf, cnt, off, sidx, level, S.ghead.as<int>(),
                                                                                                                    S.gid.as<int>(), S.key2[0].as<u64>(), ctr));
            GEM_CUDA(m, cub::DeviceRadixSort::SortKeys(S.temp.p, tcap, S.key2[0].as<u64>(), S.key2[1].as<u64>(), (int)ngp, 0, 32 + gbits, st));
            // every subtree up to level OCT_SMEM_LEVEL is simulated in shared memory sized for the largest such group
            const int smem_words = (int)oct_dense_size(std::min(hc.max_level, OCT_SMEM_LEVEL));
            const size_t smem = (size_t)smem_words * sizeof(uint32_t);
            if (smem > 48 * 1024) GEM_CUDA(m, cudaFuncSetAttribute(k_oct_group_sim, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            GEM_LAUNCH(m, GEM_PROF_OTHER, k_oct_group_sim<<<hc.groups, 32, smem, st>>>(S.groups.as<OctGroup>(), S.key2[1].as<u64>(), (int)ngp, leaf, pts, rf, P,
                                                                                       S.dense.as<uint32_t>(), smem_words, nkey, nrec, (long long)hc.upper + hc.indep, val, ctr));
        }
        for (int k = 0; k <= 16; k++)
            GEM_LAUNCH(m, GEM_PROF_OTHER, k_oct_upper<<<blocks_for((size_t)nleaf, 256, 1 << 30), 256, 0, st>>>(leaf, nleaf, level, k, P, val, nkey, nrec, ctr));
        GEM_CUDA(m, cudaGetLastError());
        GEM_CUDA(m, cub::DeviceRadixSort::SortPairs(S.temp.p, tcap, nkey, S.nkey[1].as<u64>(), nrec, S.nrec[1].as<u64>(), (int)nnode, 0, 53, st));
        GEM_CUDA(m, cudaMemcpyAsync(&hc, ctr, sizeof hc, cudaMemcpyDeviceToHost, st));
        GEM_CUDA(m, cudaStreamSynchronize(st));
    }
    r.nodes = hc.upper + hc.indep + hc.group_nodes;
    r.leaves = hc.indep + hc.group_leaves;
    r.bytes = 8ll * r.nodes;
    r.inserted = hc.inserted;
    r.skipped = n - hc.inserted;
    S.bytes = r.bytes;
    S.info = r;
    *info = r;
    return GEM_OK;
}

int gem_color_octree_read(gem_map *m, void *out, long long capacity)
{
    if (!m) return GEM_ERR_INVALID;
    Lock lk(m->mu);
    const long long bytes = m->oct.bytes;
    if (bytes < 0) return fail(m, GEM_ERR_INVALID, "gem_color_octree_read: no octree has been built");
    if (capacity < bytes || (bytes > 0 && !out)) return fail(m, GEM_ERR_INVALID, "gem_color_octree_read: capacity < bytes");
    if (bytes == 0) return GEM_OK;
    SetDev sd(m->dev);
    GEM_CUDA(m, cudaMemcpyAsync(out, m->oct.nrec[1].p, (size_t)bytes, cudaMemcpyDefault, m->stream));
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    return GEM_OK;
}

// ---- navigation costmaps (gem_costmap.cuh, DESIGN.md f8) ---------------------------------------------------------
// a window every costmap call accepts: sizes > 0 with fewer than 2^31 cells, a finite positive resolution
static bool cost_sizes_ok(int sx, int sy) { return sx > 0 && sy > 0 && (long long)sx * sy < (1ll << 31); }
static bool cost_window_ok(const gem_costmap_window *w)
{
    return w && cost_sizes_ok(w->size_x, w->size_y) && std::isfinite(w->resolution) && w->resolution > 0.0;
}
static int cost_grow(gem_map *m, size_t bytes) { return scratch_grow(m, m->cost_scratch, bytes, "costmap scratch"); }
// the last-writer scatter of both mark calls (pass 1, pass 2), then the marks back to the host
extern "C++" {
template <class Src> static int cost_mark(gem_map *m, const Src &src, long long nchunks, const gem_costmap_window *w, unsigned char *cost,
                                         gem_costmap_marks *out)
{
    const int ncells = w->size_x * w->size_y;
    int rc;
    if ((rc = cost_grow(m, (size_t)ncells * sizeof(int)))) return rc;
    if (!m->cost_acc && (rc = dev_alloc(m, &m->cost_acc, 1))) return rc;
    const CostWindow cw{w->origin_x, w->origin_y, w->resolution, w->size_x, w->size_y};
    CostMarksDev init{0, 0, cm_key(INFINITY), cm_key(INFINITY), cm_key(-INFINITY), cm_key(-INFINITY)};
    int *winner = m->cost_scratch.as<int>();
    GEM_CUDA(m, cudaMemsetAsync(winner, 0xFF, (size_t)ncells * sizeof(int), m->stream)); // -1: no writer
    GEM_CUDA(m, cudaMemcpyAsync(m->cost_acc, &init, sizeof init, cudaMemcpyHostToDevice, m->stream));
    if (nchunks > 0) {
        const int grid = (int)std::min<long long>((nchunks + COST_BLOCK / 32 - 1) / (COST_BLOCK / 32), NUM_SMS * 8);
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_costmap_scatter<Src><<<grid, COST_BLOCK, 0, m->stream>>>(src, nchunks, cw, winner, m->cost_acc));
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_costmap_store<Src><<<(unsigned)(((long long)ncells + COST_BLOCK - 1) / COST_BLOCK), COST_BLOCK, 0, m->stream>>>(src, winner, ncells, cost));
        GEM_CUDA(m, cudaGetLastError());
    }
    CostMarksDev r;
    GEM_CUDA(m, cudaMemcpyAsync(&r, m->cost_acc, sizeof r, cudaMemcpyDeviceToHost, m->stream));
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    out->marked = (long long)r.marked;
    out->lethal = (long long)r.lethal;
    out->min_x = cm_unkey(r.minx); out->min_y = cm_unkey(r.miny);
    out->max_x = cm_unkey(r.maxx); out->max_y = cm_unkey(r.maxy);
    return GEM_OK;
}
} // extern "C++"

int gem_costmap_mark_map(gem_map *m, int source, const gem_costmap_window *w, double travers_thresh, int mark_unknown,
                         unsigned char *cost_device, gem_costmap_marks *out)
{
    if (!m || !cost_device || !out || (source != GEM_GRID_SHOWN && source != GEM_GRID_SNAPSHOT))
        return fail(m, GEM_ERR_INVALID, "gem_costmap_mark_map: bad argument");
    if (!cost_window_ok(w)) return fail(m, GEM_ERR_INVALID, "gem_costmap_mark_map: bad window");
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_costmap_mark_map: not available on tiled handles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    if (source == GEM_GRID_SNAPSHOT && !m->prev_valid)
        return fail(m, GEM_ERR_INVALID, "gem_costmap_mark_map: no snapshot (call gem_snapshot_shown first)");
    int rc = flush_for_observer(m);
    if (rc) return rc;
    CostGridSrc src;
    const MapGeom &g = source == GEM_GRID_SHOWN ? m->geom : m->prev_geom;
    src.g.s = source == GEM_GRID_SHOWN ? live_cells(m->ml) : snapshot_cells(m->prev_ev, m->prev_ci, m->prev_tr);
    src.g.f = grid_frame(m, g.cx, g.cy, g.sx, g.sy);
    src.g.out = nullptr;
    src.thresh = travers_thresh;
    src.mark_unknown = mark_unknown ? 1 : 0;
    src.nch = (m->L + 31) / 32;
    return cost_mark(m, src, (long long)m->L * src.nch, w, cost_device, out);
}

int gem_costmap_mark_points(gem_map *m, const void *points32_device, int n, const gem_costmap_window *w, double travers_thresh,
                            unsigned char *cost_device, gem_costmap_marks *out)
{
    if (!m || !cost_device || !out || n < 0 || (n > 0 && !points32_device))
        return fail(m, GEM_ERR_INVALID, "gem_costmap_mark_points: bad argument");
    if (!cost_window_ok(w)) return fail(m, GEM_ERR_INVALID, "gem_costmap_mark_points: bad window");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    CostPointSrc src{static_cast<const float4 *>(points32_device), n, travers_thresh};
    return cost_mark(m, src, ((long long)n + 31) / 32, w, cost_device, out);
}

int gem_costmap_update_origin(gem_map *m, gem_costmap_window *w, double new_origin_x, double new_origin_y, unsigned char fill,
                              unsigned char *cost_device)
{
    if (!m || !cost_device) return fail(m, GEM_ERR_INVALID, "gem_costmap_update_origin: bad argument");
    if (!cost_window_ok(w)) return fail(m, GEM_ERR_INVALID, "gem_costmap_update_origin: bad window");
    // Costmap2D::updateOrigin: cell_ox = (int)((new_ox - origin_x) / resolution), truncating toward zero.  DEFINED: a shift
    // that is not finite or does not fit an int (where the cast is undefined) is an error.
    const double qx = (new_origin_x - w->origin_x) / w->resolution, qy = (new_origin_y - w->origin_y) / w->resolution;
    if (!(std::fabs(qx) < 2147483648.0) || !(std::fabs(qy) < 2147483648.0))
        return fail(m, GEM_ERR_INVALID, "gem_costmap_update_origin: the shift in cells is not finite or does not fit an int");
    const int cell_ox = (int)qx, cell_oy = (int)qy;
    if (cell_ox == 0 && cell_oy == 0) return GEM_OK; // nothing to update: the origin stays
    Lock lk(m->mu);
    SetDev sd(m->dev);
    const size_t ncells = (size_t)w->size_x * w->size_y;
    int rc;
    if ((rc = cost_grow(m, ncells))) return rc;
    // the copy, then the gather of k_costmap_roll, both ordered on the stream
    GEM_CUDA(m, cudaMemcpyAsync(m->cost_scratch.p, cost_device, ncells, cudaMemcpyDefault, m->stream));
    // |cell_ox| >= size_x leaves nothing of the old grid: clamp, so that the kernel's index sums cannot overflow
    const int cx = std::max(-w->size_x, std::min(w->size_x, cell_ox)), cy = std::max(-w->size_y, std::min(w->size_y, cell_oy));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_costmap_roll<<<(unsigned)((ncells + COST_BLOCK - 1) / COST_BLOCK), COST_BLOCK, 0, m->stream>>>(
                                      m->cost_scratch.as<unsigned char>(), cost_device, w->size_x, w->size_y, cx, cy, fill));
    GEM_CUDA(m, cudaGetLastError());
    // the new origin is grid-aligned: origin + cell_o * resolution (an int times a double, then the sum)
    const double dx = (double)cell_ox * w->resolution, dy = (double)cell_oy * w->resolution;
    w->origin_x = w->origin_x + dx;
    w->origin_y = w->origin_y + dy;
    return GEM_OK;
}

int gem_costmap_combine(gem_map *m, int mode, const unsigned char *layer_device, unsigned char *master_device, int size_x, int size_y,
                        int min_i, int min_j, int max_i, int max_j)
{
    if (!m || !layer_device || !master_device || (mode != GEM_COSTMAP_MAX && mode != GEM_COSTMAP_OVERWRITE))
        return fail(m, GEM_ERR_INVALID, "gem_costmap_combine: bad argument");
    if (!cost_sizes_ok(size_x, size_y)) return fail(m, GEM_ERR_INVALID, "gem_costmap_combine: bad grid size");
    const int i0 = std::max(min_i, 0), i1 = std::min(max_i, size_x), j0 = std::max(min_j, 0), j1 = std::min(max_j, size_y);
    if (i0 >= i1 || j0 >= j1) return GEM_OK;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    const int vec = (((uintptr_t)layer_device - (uintptr_t)master_device) & 15u) == 0 ? 1 : 0;
    const long long blocks_x = ((long long)(i1 - i0) / 16 + 2 + COST_BLOCK - 1) / COST_BLOCK;
    const dim3 grid((unsigned)std::min<long long>(blocks_x, 1024), (unsigned)std::min(j1 - j0, 65535));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_costmap_combine<<<grid, COST_BLOCK, 0, m->stream>>>(layer_device, master_device, size_x, i0, i1, j0, j1,
                                                                                    mode, vec));
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}

// ---- the VoxelGrid pre-filter of GEM's demo launches (gem_voxel.cuh, DESIGN.md f9) ------------------------------------
int gem_voxel_grid(gem_map *m, const void *xyzi_device, int n, const gem_voxel_grid_params *p, void *out_xyzi_device, int capacity,
                   gem_voxel_grid_info *info)
{
    if (!m || !p || !info || n < 0 || (n > 0 && !xyzi_device) || capacity < 0 || (capacity > 0 && !out_xyzi_device))
        return fail(m, GEM_ERR_INVALID, "gem_voxel_grid: bad argument");
    if (p->field < GEM_VOXEL_FIELD_NONE || p->field > GEM_VOXEL_FIELD_INTENSITY) return fail(m, GEM_ERR_INVALID, "gem_voxel_grid: bad field id");
    for (int a = 0; a < 3; a++) // V1
        if (!std::isfinite(p->leaf_size[a]) || !(p->leaf_size[a] > 0.0f))
            return fail(m, GEM_ERR_INVALID, "gem_voxel_grid: every leaf size must be finite and positive");
    // V9: input and output ranges may not overlap (chained calls alternate between two buffers)
    const uintptr_t i0 = (uintptr_t)xyzi_device, i1 = i0 + (size_t)n * sizeof(float4);
    const uintptr_t o0 = (uintptr_t)out_xyzi_device, o1 = o0 + (size_t)capacity * sizeof(float4);
    if (n > 0 && capacity > 0 && i0 < o1 && o0 < i1) return fail(m, GEM_ERR_INVALID, "gem_voxel_grid: the input and output ranges overlap");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    gem_voxel_grid_info r{};
    if (n == 0) { // V5
        *info = r;
        return GEM_OK;
    }
    VoxParams P{};
    for (int a = 0; a < 3; a++) P.inv[a] = 1.0f / p->leaf_size[a];
    P.field = p->field;
    P.lmin = p->limit_min;
    P.lmax = p->limit_max;
    P.flmin = (float)p->limit_min; // getMinMax3D takes the limits as floats
    P.flmax = (float)p->limit_max;
    P.negative = p->limit_negative ? 1 : 0;
    using u64 = unsigned long long;
    const size_t N = (size_t)n;
    cudaStream_t st = m->stream;
    VoxScratch &S = m->vox;
    // every buffer is sized before the first write (the sort's temporary for the widest key), so that a failed growth
    // writes nothing
    size_t t_sort = 0, t_rle = 0, t_scan = 0;
    GEM_CUDA(m, cub::DeviceRadixSort::SortPairs(nullptr, t_sort, (u64 *)nullptr, (u64 *)nullptr, (int *)nullptr, (int *)nullptr, n, 0, 64, st));
    GEM_CUDA(m, cub::DeviceRunLengthEncode::Encode(nullptr, t_rle, (u64 *)nullptr, (u64 *)nullptr, (int *)nullptr, (int *)nullptr, n, st));
    GEM_CUDA(m, cub::DeviceScan::ExclusiveSum(nullptr, t_scan, (int *)nullptr, (int *)nullptr, n, st));
    const char *what = "gem_voxel_grid";
    int rc;
    if ((rc = scratch_grow(m, S.key[0], N * 8, what)) || (rc = scratch_grow(m, S.key[1], N * 8, what)) ||
        (rc = scratch_grow(m, S.idx[0], N * 4, what)) || (rc = scratch_grow(m, S.idx[1], N * 4, what)) ||
        (rc = scratch_grow(m, S.cnt, N * 4, what)) || (rc = scratch_grow(m, S.off, N * 4, what)) ||
        (rc = scratch_grow(m, S.temp, std::max(t_sort, std::max(t_rle, t_scan)), what)) || (rc = scratch_grow(m, S.acc, sizeof(VoxAcc), what)))
        return rc;
    const float4 *in = static_cast<const float4 *>(xyzi_device);
    float4 *out = static_cast<float4 *>(out_xyzi_device);
    VoxAcc *acc = S.acc.as<VoxAcc>();
    VoxAcc h{};
    for (int a = 0; a < 3; a++) { h.mn[a] = vg_key(FLT_MAX); h.mx[a] = vg_key(-FLT_MAX); }
    GEM_CUDA(m, cudaMemcpyAsync(acc, &h, sizeof h, cudaMemcpyHostToDevice, st));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_vox_bounds<<<blocks_for(N, VOX_BLOCK, NUM_SMS * 8), VOX_BLOCK, 0, st>>>(in, n, P, acc));
    GEM_CUDA(m, cudaGetLastError());
    // synchronisation 1: V4, V5 and the key layout are decided on the host from the counts and the bounds
    GEM_CUDA(m, cudaMemcpyAsync(&h, acc, sizeof h, cudaMemcpyDeviceToHost, st));
    GEM_CUDA(m, cudaStreamSynchronize(st));
    r.used = h.used;
    if (h.bounded == 0) { // V5
        *info = r;
        return GEM_OK;
    }
    // V4: d[a] = (int64)((max_p - min_p) * inv) + 1, the product in float.  DEFINED: a product that is not finite or a
    // quotient >= 2^62 is an overflow; the product of the d is the mathematical one (each step below stays under 2^62)
    float mn[3], mx[3];
    long long d[3] = {0, 0, 0};
    bool over = false;
    for (int a = 0; a < 3; a++) {
        mn[a] = vg_unkey(h.mn[a]);
        mx[a] = vg_unkey(h.mx[a]);
        const float q = (mx[a] - mn[a]) * P.inv[a];
        if (!std::isfinite(q) || q >= 4611686018427387904.0f) over = true;
        else d[a] = (long long)q + 1;
    }
    over = over || d[0] > INT32_MAX || d[1] > INT32_MAX || d[2] > INT32_MAX || d[0] * d[1] > INT32_MAX || d[0] * d[1] * d[2] > INT32_MAX;
    if (over) { // the input unchanged: PCL's output = *input_
        const size_t k = std::min(N, (size_t)capacity);
        if (k) GEM_CUDA(m, cudaMemcpyAsync(out, in, k * sizeof(float4), cudaMemcpyDeviceToDevice, st));
        GEM_CUDA(m, cudaStreamSynchronize(st)); // synchronisation 2: the call is host-synchronous
        r.count = n;
        r.passthrough = 1;
        *info = r;
        return GEM_OK;
    }
    if (h.used == 0) {
        *info = r;
        return GEM_OK;
    }
    // V6: min_b, max_b as floor values of float products (exact in either overload), div from their exact difference; the
    // mixed-radix key ijk0 + ijk1 div0 + ijk2 div0 div1 in 64 bits is PCL's idx where that fits an int and the DEFINED
    // lexicographic order where it does not
    VoxGrid G{};
    u64 div[3];
    for (int a = 0; a < 3; a++) {
        G.minb[a] = std::floor((double)(mn[a] * P.inv[a]));
        div[a] = (u64)(std::floor((double)(mx[a] * P.inv[a])) - G.minb[a]) + 1;
    }
    // with V4 passed the voxel count stays far below 2^62 (each div[a] is within a few times d[a]); guarded all the same
    if (!((double)div[0] * (double)div[1] * (double)div[2] < 4.0e18))
        return fail(m, GEM_ERR_INVALID, "gem_voxel_grid: the voxel grid needs keys wider than 62 bits");
    G.div0 = div[0];
    G.div01 = div[0] * div[1];
    G.cut_key = G.div01 * div[2]; // one past the largest voxel key: the cut points' run sorts last
    int bits = 1;
    while ((1ull << bits) <= G.cut_key) bits++;
    u64 *key0 = S.key[0].as<u64>(), *key1 = S.key[1].as<u64>();
    int *idx0 = S.idx[0].as<int>(), *idx1 = S.idx[1].as<int>(), *cnt = S.cnt.as<int>(), *off = S.off.as<int>();
    size_t tcap = S.temp.cap;
    // the run-length encoding writes nruns <= n counts; the scan runs over all n, so the rest must be defined
    GEM_CUDA(m, cudaMemsetAsync(cnt, 0, N * sizeof(int), st));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_vox_keys<<<(unsigned)((N + VOX_BLOCK - 1) / VOX_BLOCK), VOX_BLOCK, 0, st>>>(in, n, P, G, key0, idx0));
    GEM_CUDA(m, cudaGetLastError());
    // V7: the stable sort keeps each voxel's points in input order
    GEM_CUDA(m, cub::DeviceRadixSort::SortPairs(S.temp.p, tcap, key0, key1, idx0, idx1, n, 0, bits, st));
    GEM_CUDA(m, cub::DeviceRunLengthEncode::Encode(S.temp.p, tcap, key1, key0, cnt, &acc->nruns, n, st));
    GEM_CUDA(m, cub::DeviceScan::ExclusiveSum(S.temp.p, tcap, cnt, off, n, st));
    const int drop = h.used < n ? 1 : 0;
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_vox_centroids<<<(unsigned)(((size_t)h.used + VOX_BLOCK - 1) / VOX_BLOCK), VOX_BLOCK, 0, st>>>(
                                      in, idx1, cnt, off, acc, drop, out, capacity));
    GEM_CUDA(m, cudaGetLastError());
    // synchronisation 2: the voxel count
    GEM_CUDA(m, cudaMemcpyAsync(&h.nruns, &acc->nruns, sizeof(int), cudaMemcpyDeviceToHost, st));
    GEM_CUDA(m, cudaStreamSynchronize(st));
    r.count = h.nruns - drop;
    *info = r;
    return GEM_OK;
}

// ---- the MLS densification of the dense_mapping signal (gem_mls.cuh, DESIGN.md f10) -----------------------------------
int gem_mls_upsample(gem_map *m, const void *points32_device, int n, const gem_mls_params *p, void *out_points32_device,
                     long long capacity, gem_mls_info *info)
{
    if (!m || !p || !info || n < 0 || (n > 0 && !points32_device) || capacity < 0 || (capacity > 0 && !out_points32_device))
        return fail(m, GEM_ERR_INVALID, "gem_mls_upsample: bad argument");
    if (!std::isfinite(p->search_radius) || !(p->search_radius > 0.0) || !std::isfinite(p->sqr_gauss_param) || !(p->sqr_gauss_param > 0.0))
        return fail(m, GEM_ERR_INVALID, "gem_mls_upsample: the search radius and the Gauss parameter must be finite and positive");
    if (p->order < 1 || p->order > 5) return fail(m, GEM_ERR_INVALID, "gem_mls_upsample: the polynomial order must lie in 1..5");
    if (p->upsampling != GEM_MLS_NONE && p->upsampling != GEM_MLS_RANDOM_UNIFORM_DENSITY)
        return fail(m, GEM_ERR_INVALID, "gem_mls_upsample: unknown upsampling method");
    if (p->point_density < 0) return fail(m, GEM_ERR_INVALID, "gem_mls_upsample: point_density < 0");
    const uintptr_t i0 = (uintptr_t)points32_device, i1 = i0 + (size_t)n * 32;
    const uintptr_t o0 = (uintptr_t)out_points32_device, o1 = o0 + (size_t)capacity * 32;
    if (n > 0 && capacity > 0 && i0 < o1 && o0 < i1) return fail(m, GEM_ERR_INVALID, "gem_mls_upsample: the input and output ranges overlap");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    gem_mls_info r{};
    if (n == 0) {
        r.fitted = capacity == 0 ? -1 : 0; // M8: a size query reports no fit count
        *info = r;
        return GEM_OK;
    }
    MlsParams P{};
    P.r = p->search_radius;
    P.r2q = P.r * P.r / 4.0;
    P.gauss = p->sqr_gauss_param;
    P.edge = P.r * (1.0 + 1.0 / 1024.0); // the search grid (gem_mls.cuh): a neighbour is always less than one edge away
    P.r2f = (float)(P.r * P.r);
    P.hi = (float)(P.r / 2.0);
    P.lo = -P.hi;
    P.fit = p->polynomial_fit ? 1 : 0;
    P.order = p->order;
    P.nc = (p->order + 1) * (p->order + 2) / 2;
    P.upsampling = p->upsampling;
    P.density = p->point_density;
    P.seed = p->seed;
    using u64 = unsigned long long;
    const size_t N = (size_t)n;
    cudaStream_t st = m->stream;
    MlsScratch &S = m->mls;
    // every buffer the first synchronisation needs is sized before the first launch, so that a failed growth writes nothing
    size_t t_sort = 0, t_rle = 0, t_scan = 0, t_scan64 = 0;
    GEM_CUDA(m, cub::DeviceRadixSort::SortPairs(nullptr, t_sort, (u64 *)nullptr, (u64 *)nullptr, (int *)nullptr, (int *)nullptr, n, 0, 64, st));
    GEM_CUDA(m, cub::DeviceRunLengthEncode::Encode(nullptr, t_rle, (u64 *)nullptr, (u64 *)nullptr, (int *)nullptr, (int *)nullptr, n, st));
    GEM_CUDA(m, cub::DeviceScan::ExclusiveSum(nullptr, t_scan, (int *)nullptr, (int *)nullptr, n, st));
    GEM_CUDA(m, cub::DeviceScan::ExclusiveSum(nullptr, t_scan64, (long long *)nullptr, (long long *)nullptr, n, st));
    const char *what = "gem_mls_upsample";
    int rc;
    if ((rc = scratch_grow(m, S.key[0], N * 8, what)) || (rc = scratch_grow(m, S.key[1], N * 8, what)) ||
        (rc = scratch_grow(m, S.idx[0], N * 4, what)) || (rc = scratch_grow(m, S.idx[1], N * 4, what)) ||
        (rc = scratch_grow(m, S.spts, N * 16, what)) || (rc = scratch_grow(m, S.ukey, N * 8, what)) ||
        (rc = scratch_grow(m, S.ucnt, N * 4, what)) || (rc = scratch_grow(m, S.uoff, N * 4, what)) ||
        (rc = scratch_grow(m, S.nbr, N * 4, what)) || (rc = scratch_grow(m, S.ocnt, N * 8, what)) ||
        (rc = scratch_grow(m, S.ooff, N * 8, what)) || (rc = scratch_grow(m, S.longs, N * 4, what)) ||
        (rc = scratch_grow(m, S.temp, std::max(std::max(t_sort, t_rle), std::max(t_scan, t_scan64)), what)) ||
        (rc = scratch_grow(m, S.acc, sizeof(MlsAcc), what)))
        return rc;
    const float4 *in = static_cast<const float4 *>(points32_device);
    float4 *out = static_cast<float4 *>(out_points32_device);
    MlsAcc *acc = S.acc.as<MlsAcc>();
    u64 *key0 = S.key[0].as<u64>(), *key1 = S.key[1].as<u64>(), *ukey = S.ukey.as<u64>();
    int *idx0 = S.idx[0].as<int>(), *idx1 = S.idx[1].as<int>(), *ucnt = S.ucnt.as<int>(), *uoff = S.uoff.as<int>();
    int *nbr = S.nbr.as<int>(), *longs = S.longs.as<int>();
    long long *ocnt = S.ocnt.as<long long>(), *ooff = S.ooff.as<long long>();
    float4 *spts = S.spts.as<float4>();
    size_t tcap = S.temp.cap;
    MlsAcc h{};
    h.mn[0] = h.mn[1] = h.mn[2] = 0xffffffffu;
    GEM_CUDA(m, cudaMemcpyAsync(acc, &h, sizeof h, cudaMemcpyHostToDevice, st));
    // the run-length encoding writes nruns <= n counts; the scan runs over all n, so the rest must be defined
    GEM_CUDA(m, cudaMemsetAsync(ucnt, 0, N * sizeof(int), st));
    const unsigned gb = (unsigned)((N + VOX_BLOCK - 1) / VOX_BLOCK), gq = (unsigned)((N + MLS_WARPS - 1) / MLS_WARPS);
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_mls_bounds<<<blocks_for(N, VOX_BLOCK, NUM_SMS * 8), VOX_BLOCK, 0, st>>>(in, n, acc));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_mls_keys<<<gb, VOX_BLOCK, 0, st>>>(in, n, P, acc, key0, idx0));
    GEM_CUDA(m, cudaGetLastError());
    GEM_CUDA(m, cub::DeviceRadixSort::SortPairs(S.temp.p, tcap, key0, key1, idx0, idx1, n, 0, 64, st));
    GEM_CUDA(m, cub::DeviceRunLengthEncode::Encode(S.temp.p, tcap, key1, ukey, ucnt, &acc->nruns, n, st));
    GEM_CUDA(m, cub::DeviceScan::ExclusiveSum(S.temp.p, tcap, ucnt, uoff, n, st));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_mls_stage<<<gb, VOX_BLOCK, 0, st>>>(in, n, idx1, spts));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_mls_count<<<gq, MLS_BLOCK, 0, st>>>(in, n, P, acc, spts, ukey, uoff, ucnt, nbr, ocnt, longs));
    GEM_CUDA(m, cudaGetLastError());
    GEM_CUDA(m, cub::DeviceScan::ExclusiveSum(S.temp.p, tcap, ocnt, ooff, n, st));
    // synchronisation 1: the output count (last offset + last count), the longest list and the number of long lists
    long long tail[2] = {0, 0};
    GEM_CUDA(m, cudaMemcpyAsync(&tail[0], ooff + (N - 1), sizeof(long long), cudaMemcpyDeviceToHost, st));
    GEM_CUDA(m, cudaMemcpyAsync(&tail[1], ocnt + (N - 1), sizeof(long long), cudaMemcpyDeviceToHost, st));
    GEM_CUDA(m, cudaMemcpyAsync(&h, acc, sizeof h, cudaMemcpyDeviceToHost, st));
    GEM_CUDA(m, cudaStreamSynchronize(st));
    r.count = tail[0] + tail[1];
    // the long lists: persistent warps, each sorting in its own global slice of a power of two >= the longest list; as
    // many warps as fit in 256 MiB, at least one block's worth
    int slice = 32, lwarps = 0;
    if (h.nlong > 0) {
        while (slice < h.max_nb) slice <<= 1;
        const size_t per = (size_t)slice * 8;
        size_t w = std::max((size_t)MLS_WARPS, ((size_t)256 << 20) / per / MLS_WARPS * MLS_WARPS);
        w = std::min(w, (size_t)NUM_SMS * 16);
        w = std::min(w, ((size_t)h.nlong + MLS_WARPS - 1) / MLS_WARPS * MLS_WARPS);
        lwarps = (int)w;
        if ((rc = scratch_grow(m, S.lkeys, w * per, what))) return rc;
    }
    if (capacity == 0) { // a size query stops here: the fits are not run
        r.processed = h.processed;
        r.fitted = -1;
        r.skipped = h.skipped;
        r.max_neighbours = h.max_nb;
        *info = r;
        return GEM_OK;
    }
    if (r.count > 0) {
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_mls_fit<false><<<gq, MLS_BLOCK, 0, st>>>(in, n, P, acc, spts, ukey, uoff, ucnt, nbr, ooff, longs,
                                                                                 nullptr, 0, out, capacity));
        if (lwarps)
            GEM_LAUNCH(m, GEM_PROF_OTHER, k_mls_fit<true><<<lwarps / MLS_WARPS, MLS_BLOCK, 0, st>>>(
                                              in, n, P, acc, spts, ukey, uoff, ucnt, nbr, ooff, longs, S.lkeys.as<u64>(), slice, out, capacity));
        GEM_CUDA(m, cudaGetLastError());
    }
    // synchronisation 2: the info
    GEM_CUDA(m, cudaMemcpyAsync(&h, acc, sizeof h, cudaMemcpyDeviceToHost, st));
    GEM_CUDA(m, cudaStreamSynchronize(st));
    r.processed = h.processed;
    r.fitted = h.fitted;
    r.skipped = h.skipped;
    r.max_neighbours = h.max_nb;
    *info = r;
    return GEM_OK;
}

// ---- localMap_ on the device ----------------------------------------------------------------------------------------
// Grow the store to hold `need` records (capacity doubles from LOCAL_MIN_RECORDS).  Everything is allocated before
// anything is released, so a failed growth leaves the store as it was.
static constexpr int LOCAL_MIN_RECORDS = 1024;
static int local_reserve(gem_map *m, long long need)
{
    LocalStore &s = m->local;
    if (need <= s.cap) return GEM_OK;
    long long cap = s.cap > 0 ? s.cap : LOCAL_MIN_RECORDS;
    while (cap < need) cap *= 2;
    if (cap > (1 << 30)) return fail(m, GEM_ERR_NOMEM, "local map: more than 2^30 records");
    size_t slots = 64;
    while (slots < 2 * (size_t)cap) slots <<= 1;
    const size_t nchunk = (size_t)cap / 32 + 1, nseg = nchunk / SCAN_SEG + 1;
    const size_t bytes = (size_t)cap * 32 + slots * (8 + 4) + (nchunk + nseg) * 4;
    void *buf = nullptr;
    cudaError_t e = cudaMalloc(&buf, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(m, GEM_ERR_NOMEM, std::string("local map: cudaMalloc: ") + cudaGetErrorString(e));
    }
    LocalStore t;
    t.buf = buf;
    t.log = (float4 *)buf;
    t.keys = (unsigned long long *)(t.log + 2 * (size_t)cap);
    t.latest = (int *)(t.keys + slots);
    t.cnt = t.latest + slots;
    t.n = s.n; t.cap = (int)cap; t.slots = slots;
    e = cudaMemsetAsync(t.keys, 0xff, slots * 8, m->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(t.latest, 0xff, slots * 4, m->stream);
    if (e == cudaSuccess && s.n) e = cudaMemcpyAsync(t.log, s.log, (size_t)s.n * 32, cudaMemcpyDeviceToDevice, m->stream);
    if (e == cudaSuccess && s.n) {
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_local_index<<<blocks_for((size_t)s.n, 256, 1 << 30), 256, 0, m->stream>>>(t.log, 0, s.n, t.keys, t.latest, (unsigned)(slots - 1)));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(m->stream);
    if (e != cudaSuccess) {
        cudaFree(buf);
        return fail(m, GEM_ERR_CUDA, std::string("local map: growth: ") + cudaGetErrorString(e));
    }
    if (s.buf) cudaFree(s.buf);
    s = t;
    return GEM_OK;
}

// forget every record: the index back to all-free slots
static int local_reset(gem_map *m)
{
    LocalStore &s = m->local;
    s.n = 0;
    if (!s.buf) return GEM_OK;
    GEM_CUDA(m, cudaMemsetAsync(s.keys, 0xff, s.slots * 8, m->stream));
    GEM_CUDA(m, cudaMemsetAsync(s.latest, 0xff, s.slots * 4, m->stream));
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    return GEM_OK;
}

int gem_local_map_reserve(gem_map *m, int records)
{
    if (!m || records < 0) return fail(m, GEM_ERR_INVALID, "gem_local_map_reserve: bad argument");
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_local_map_reserve: not available on tiled handles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    return local_reserve(m, records);
}

int gem_harvest_to_local_map(gem_map *m, const float current_xy[2], const float shift_xy[2], void *host_points32, int capacity,
                             int *count_out)
{
    if (!m || !current_xy || !shift_xy || !count_out || capacity < 0 || (capacity > 0 && !host_points32))
        return fail(m, GEM_ERR_INVALID, "gem_harvest_to_local_map: bad argument");
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_harvest_to_local_map: not available on tiled handles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    if (!m->prev_valid) return fail(m, GEM_ERR_INVALID, "gem_harvest_to_local_map: no snapshot (call gem_snapshot_shown first)");
    int total = 0, rc;
    if ((rc = harvest_to_staging(m, current_xy, shift_xy, (int)m->nc, &total))) return rc;
    if ((rc = local_reserve(m, (long long)m->local.n + total))) return rc;
    LocalStore &s = m->local;
    if (total) { // append, then point every key of this call at its latest position (:740-747)
        GEM_CUDA(m, cudaMemcpyAsync(s.log + 2 * (size_t)s.n, m->d_out, (size_t)total * 32, cudaMemcpyDeviceToDevice, m->stream));
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_local_index<<<blocks_for((size_t)total, 256, 1 << 30), 256, 0, m->stream>>>(s.log, s.n, s.n + total, s.keys, s.latest, (unsigned)(s.slots - 1)));
        GEM_CUDA(m, cudaGetLastError());
        s.n += total;
    }
    const size_t n = (size_t)std::min(total, capacity);
    if (n) GEM_CUDA(m, cudaMemcpyAsync(host_points32, m->d_out, n * 32, cudaMemcpyDeviceToHost, m->stream));
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    *count_out = total;
    return GEM_OK;
}

int gem_local_map_take(gem_map *m, void *points32_device, int capacity, int *count_out)
{
    if (!m || !count_out || capacity < 0 || (capacity > 0 && !points32_device))
        return fail(m, GEM_ERR_INVALID, "gem_local_map_take: bad argument");
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_local_map_take: not available on tiled handles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    LocalStore &s = m->local;
    if (s.n == 0) { *count_out = 0; return GEM_OK; }
    // the kept entries (those the index points at) in log order: count per warp -> multi-block scan -> write
    const int nchunk = (s.n + 31) / 32, nseg = (nchunk + SCAN_SEG - 1) / SCAN_SEG, nb = (s.n + TAKE_BLOCK - 1) / TAKE_BLOCK;
    const unsigned mask = (unsigned)(s.slots - 1);
    int *segtot = s.cnt + nchunk;
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_local_count<<<nb, TAKE_BLOCK, 0, m->stream>>>(s.log, s.n, s.keys, s.latest, mask, s.cnt));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_compact_scan<<<nseg, SCAN_SEG, 0, m->stream>>>(s.cnt, nchunk, segtot));
    GEM_CUDA(m, cudaGetLastError());
    std::vector<int> h((size_t)nseg);
    GEM_CUDA(m, cudaMemcpyAsync(h.data(), segtot, (size_t)nseg * 4, cudaMemcpyDeviceToHost, m->stream));
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    long long total = 0;
    for (int v : h) total += v;
    *count_out = (int)total;
    if (total > capacity) return GEM_OK; // nothing written, the store is kept: *count_out is the size needed
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_local_write<<<nb, TAKE_BLOCK, 0, m->stream>>>(s.log, s.n, s.keys, s.latest, mask, s.cnt, segtot, SCAN_SEG,
                                                                                 reinterpret_cast<float4 *>(points32_device)));
    GEM_CUDA(m, cudaGetLastError());
    return local_reset(m);
}

int gem_local_map_clear(gem_map *m)
{
    if (!m) return GEM_ERR_INVALID;
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_local_map_clear: not available on tiled handles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    return local_reset(m);
}

int gem_get_layer(gem_map *m, int layer, void *host_out)
{
    if (!m || !host_out || layer < 0 || layer > 9) return fail(m, GEM_ERR_INVALID, "gem_get_layer: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_out_staging(m);
    if (rc) return rc;
    if ((rc = copy_layer_out(m, layer, host_out, 0))) return rc;
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    return GEM_OK;
}

int gem_set_layer(gem_map *m, int layer, const void *host_in)
{
    if (!m || !host_in || layer < 0 || layer > 9) return fail(m, GEM_ERR_INVALID, "gem_set_layer: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_out_staging(m);
    if (rc) return rc;
    if ((rc = flush_for_observer(m))) return rc;
    GEM_CUDA(m, cudaMemcpyAsync(m->d_out, host_in, m->nc * 4, cudaMemcpyHostToDevice, m->stream));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_pack_layer<<<blocks_for(m->nc, 256), 256, 0, m->stream>>>(m->ml, m->nc, layer, m->d_out));
    GEM_CUDA(m, cudaGetLastError());
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    if (layer == GEM_LAYER_VARIANCE) pend_all_floor(m);
    return GEM_OK;
}

int gem_get_state(gem_map *m, float centre[2], int start[2], float *sensor_z)
{
    if (!m) return GEM_ERR_INVALID;
    Lock lk(m->mu);
    if (centre) { centre[0] = m->geom.cx; centre[1] = m->geom.cy; }
    if (start) { start[0] = m->geom.sx; start[1] = m->geom.sy; }
    if (sensor_z) *sensor_z = m->sensorZ;
    return GEM_OK;
}

int gem_get_stats(gem_map *m, gem_stats *out)
{
    if (!m || !out) return GEM_ERR_INVALID;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    if (m->stats.points_in > 0 && m->stats.cells_touched == 0 && m->stats.points_binned == 0) {
        // device-pointer call: counters not fetched yet
        const long long n_in = m->stats.points_in;
        int rc = read_counters(m, 0, false);
        if (rc) return rc;
        m->stats.points_in = n_in;
    }
    *out = m->stats;
    return GEM_OK;
}

int gem_profile_enable(gem_map *m, int on)
{
    if (!m) return GEM_ERR_INVALID;
    Lock lk(m->mu);
    if (on && !m->profiling) { int rc = drain(m); if (rc) return rc; }
    m->profiling = on != 0;
    return GEM_OK;
}

int gem_profile_read(gem_map *m, gem_profile *out, int reset)
{
    if (!m || !out) return GEM_ERR_INVALID;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    { int rc = drain(m); if (rc) return rc; }
    if (m->front_stream) GEM_CUDA(m, cudaStreamSynchronize(m->front_stream));
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    for (auto &sp : m->spans) {
        float ms = 0.0f;
        if (cudaEventElapsedTime(&ms, sp.e0, sp.e1) == cudaSuccess) {
            m->prof_ms[sp.cls] += ms;
            m->prof_count[sp.cls]++;
        }
        m->free_events.push_back(sp.e0);
        m->free_events.push_back(sp.e1);
    }
    m->spans.clear();
    out->launches = m->launches;
    for (int i = 0; i < GEM_PROF_CLASSES; i++) {
        out->ms[i] = m->prof_ms[i];
        out->count[i] = m->prof_count[i];
    }
    if (reset) {
        m->launches = 0;
        for (int i = 0; i < GEM_PROF_CLASSES; i++) { m->prof_ms[i] = 0.0; m->prof_count[i] = 0; }
    }
    return GEM_OK;
}

int gem_selftest_division(gem_map *m, unsigned long long seed, unsigned long long n, unsigned long long *mismatches_out,
                          unsigned long long *fast_out)
{
    if (!m || !mismatches_out) return GEM_ERR_INVALID;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    unsigned long long *d = nullptr;
    GEM_CUDA(m, cudaMalloc((void **)&d, 16));
    GEM_CUDA(m, cudaMemsetAsync(d, 0, 16, m->stream));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_div_selftest<<<NUM_SMS * 8, 256, 0, m->stream>>>(seed, (size_t)n, d, d + 1));
    unsigned long long h[2] = {0, 0};
    GEM_CUDA(m, cudaMemcpyAsync(h, d, 16, cudaMemcpyDeviceToHost, m->stream));
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    cudaFree(d);
    *mismatches_out = h[0];
    if (fast_out) *fast_out = h[1];
    return GEM_OK;
}

int gem_host_alloc(void **out, unsigned long long bytes)
{
    if (!out) return GEM_ERR_INVALID;
    return cudaHostAlloc(out, (size_t)bytes, cudaHostAllocDefault) == cudaSuccess ? GEM_OK : GEM_ERR_NOMEM;
}
int gem_host_free(void *p) { return cudaFreeHost(p) == cudaSuccess ? GEM_OK : GEM_ERR_CUDA; }

// ---- multi-GPU routing -----------------------------------------------------------------------
int gem_route_points(gem_map *m, const void *xyzi, const void *rgba, int n, const gem_frame *frame, int tiles_r,
                     int tiles_c, void *rec_out, int *counts_out, int bucket_stride)
{
    if (!m || !frame || n < 0 || tiles_r < 1 || tiles_c < 1 || !rec_out || !counts_out || (n > 0 && !xyzi))
        return fail(m, GEM_ERR_INVALID, "gem_route_points: bad argument");
    if (n > m->P) return fail(m, GEM_ERR_INVALID, "gem_route_points: n exceeds max_points");
    if (tiles_r * tiles_c > ROUTE_MAX_OWNERS) return fail(m, GEM_ERR_INVALID, "gem_route_points: too many tiles");
    if (bucket_stride > 0 && bucket_stride < n) // one owner may receive all n records
        return fail(m, GEM_ERR_INVALID, "gem_route_points: bucket_stride must be 0 (packed) or >= n");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    const FrameParams fp = make_frame(frame);
    MapGeom gg = m->geom;
    gg.tiled = 0; // routing works on global geographic indices
    if (bucket_stride > 0) // padded layout: unused slots must read as "no record" (gkey = -1)
        GEM_CUDA(m, cudaMemsetAsync(rec_out, 0xff, (size_t)tiles_r * tiles_c * bucket_stride * sizeof(RouteRec), m->stream));
    { int rc = ensure_route_scratch(m); if (rc) return rc; }
    const cudaError_t e = route_points(m->stream, gg, fp, (const float4 *)xyzi, (const uchar4 *)rgba, n, tiles_r,
                                       tiles_c, m->route_sc, (RouteRec *)rec_out, counts_out, bucket_stride);
    m->launches += 3;
    if (e != cudaSuccess) return fail(m, GEM_ERR_CUDA, std::string("gem_route_points: ") + cudaGetErrorString(e));
    return GEM_OK;
}

static int fuse_records_impl(gem_map *m, const void *rec, int n, const int *src_counts, int stride);

int gem_fuse_records(gem_map *m, const void *rec, int n) { return fuse_records_impl(m, rec, n, nullptr, 1); }

int gem_fuse_records_counted(gem_map *m, const void *rec, const int *src_counts, int n_sources, int bucket_stride)
{
    if (!m || !rec || !src_counts || n_sources < 1 || bucket_stride < 1) return fail(m, GEM_ERR_INVALID, "gem_fuse_records_counted: bad argument");
    if ((long long)n_sources * bucket_stride > m->P) return fail(m, GEM_ERR_INVALID, "gem_fuse_records_counted: n_sources*bucket_stride exceeds max_points");
    return fuse_records_impl(m, rec, n_sources * bucket_stride, src_counts, bucket_stride);
}

int gem_route_points_peer(gem_map *m, const void *xyzi, const void *rgba, int n, const gem_frame *frame, int tiles_r, int tiles_c,
                          const unsigned long long *peer_recv, const unsigned long long *peer_counts, int my_rank, int bucket_stride)
{
    const int no = tiles_r * tiles_c;
    if (!m || !frame || n < 0 || tiles_r < 1 || tiles_c < 1 || !peer_recv || !peer_counts || (n > 0 && !xyzi) || bucket_stride < n ||
        my_rank < 0 || my_rank >= no)
        return fail(m, GEM_ERR_INVALID, "gem_route_points_peer: bad argument (bucket_stride must be >= n)");
    if (n > m->P) return fail(m, GEM_ERR_INVALID, "gem_route_points_peer: n exceeds max_points");
    if (no > ROUTE_MAX_OWNERS) return fail(m, GEM_ERR_INVALID, "gem_route_points_peer: too many tiles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = GEM_OK;
    if (!m->d_owner_cnt && (rc = dev_alloc(m, &m->d_owner_cnt, ROUTE_MAX_OWNERS))) return rc;
    const FrameParams fp = make_frame(frame);
    MapGeom gg = m->geom;
    gg.tiled = 0;
    PeerTable pt;
    memset(&pt, 0, sizeof pt);
    for (int o = 0; o < no; o++) { pt.recv[o] = peer_recv[o]; pt.counts[o] = peer_counts[o]; }
    if ((rc = ensure_route_scratch(m))) return rc;
    const cudaError_t e = route_points(m->stream, gg, fp, (const float4 *)xyzi, (const uchar4 *)rgba, n, tiles_r, tiles_c,
                                       m->route_sc, nullptr, m->d_owner_cnt, bucket_stride, &pt, my_rank);
    m->launches += 3;
    if (e != cudaSuccess) return fail(m, GEM_ERR_CUDA, std::string("gem_route_points_peer: ") + cudaGetErrorString(e));
    return GEM_OK;
}

// ---- loop-closure submap re-fusion (SURVEY 8f row 4, gem_submap.cuh) -------------------------------------------------------
int gem_transform_cloud(gem_map *m, void *points32, int n, const float T[16])
{
    if (!m || n < 0 || (n > 0 && !points32) || !T) return fail(m, GEM_ERR_INVALID, "gem_transform_cloud: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    Rigid r;
    for (int i = 0; i < 12; i++) r.t[i] = T[i];
    if (n > 0) GEM_LAUNCH(m, GEM_PROF_OTHER, k_transform_cloud<<<blocks_for((size_t)n, 256, 1 << 30), 256, 0, m->stream>>>((SubPoint *)points32, n, r));
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}

int gem_refuse_submaps(gem_map *m, void *new_points32, int *n_new, void *old_points32, int *n_old, double resolution, int compat,
                       int *fused_out)
{
    if (!m || !n_new || !n_old || *n_new < 0 || *n_old < 0 || (*n_new > 0 && !new_points32) || (*n_old > 0 && !old_points32) || !(resolution > 0.0))
        return fail(m, GEM_ERR_INVALID, "gem_refuse_submaps: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    const int nn = *n_new, no = *n_old;
    auto pow2 = [](size_t v) { size_t p = 64; while (p < v) p <<= 1; return p; };
    const size_t cn = pow2(2 * (size_t)nn + 2), co = pow2(2 * (size_t)no + 2);
    // one scratch block: two hash tables (keys + first index), keep flags, compaction outputs, counters
    const size_t bytes = (cn + co) * (8 + 4) + (size_t)nn + no + 64 + ((size_t)nn + no) * sizeof(SubPoint) + 64;
    char *d = nullptr;
    GEM_CUDA(m, cudaMalloc((void **)&d, bytes));
    unsigned long long *kn = (unsigned long long *)d, *ko = kn + cn;
    int *fn = (int *)(ko + co), *fo = fn + cn;
    int *cnts = fo + co; // [0] fused, [1] kept new, [2] kept old
    SubPoint *outn = (SubPoint *)(((uintptr_t)(cnts + 4) + 31) & ~(uintptr_t)31), *outo = outn + nn;
    unsigned char *keepn = (unsigned char *)(outo + no), *keepo = keepn + nn;
    auto done = [&](int rc) { cudaFree(d); return rc; };
    cudaError_t e = cudaMemsetAsync(kn, 0xff, (cn + co) * 8, m->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(fn, 0x7f, (cn + co) * 4, m->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(cnts, 0, 16, m->stream);
    if (e != cudaSuccess) return done(fail(m, GEM_ERR_CUDA, cudaGetErrorString(e)));
    SubPoint *pn = (SubPoint *)new_points32, *po = (SubPoint *)old_points32;
    if (nn) GEM_LAUNCH(m, GEM_PROF_OTHER, k_hash_insert<<<blocks_for((size_t)nn, 256, 1 << 30), 256, 0, m->stream>>>(pn, nn, resolution, kn, fn, (unsigned)(cn - 1)));
    if (no) GEM_LAUNCH(m, GEM_PROF_OTHER, k_hash_insert<<<blocks_for((size_t)no, 256, 1 << 30), 256, 0, m->stream>>>(po, no, resolution, ko, fo, (unsigned)(co - 1)));
    const int nmax = nn > no ? nn : no;
    if (nmax) GEM_LAUNCH(m, GEM_PROF_OTHER, k_refuse_pair<<<blocks_for((size_t)nmax, 256, 1 << 30), 256, 0, m->stream>>>(pn, nn, po, no, resolution, kn, fn, (unsigned)(cn - 1), ko, fo, (unsigned)(co - 1), keepn, keepo, compat, cnts));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_compact_points<<<1, 1024, 0, m->stream>>>(pn, keepn, nn, outn, cnts + 1));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_compact_points<<<1, 1024, 0, m->stream>>>(po, keepo, no, outo, cnts + 2));
    int h[4] = {0, 0, 0, 0};
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(h, cnts, 16, cudaMemcpyDeviceToHost, m->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(m->stream);
    if (e == cudaSuccess && h[1] > 0) e = cudaMemcpyAsync(pn, outn, (size_t)h[1] * sizeof(SubPoint), cudaMemcpyDeviceToDevice, m->stream);
    if (e == cudaSuccess && h[2] > 0) e = cudaMemcpyAsync(po, outo, (size_t)h[2] * sizeof(SubPoint), cudaMemcpyDeviceToDevice, m->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(m->stream);
    if (e != cudaSuccess) return done(fail(m, GEM_ERR_CUDA, std::string("gem_refuse_submaps: ") + cudaGetErrorString(e)));
    *n_new = h[1];
    *n_old = h[2];
    if (fused_out) *fused_out = h[0];
    return done(GEM_OK);
}

// ---- tiled maps, peer path (gem_route.cuh "Peer path, round 2") --------------------------------------------------------
int gem_tiled_attach(gem_map *m, const gem_tiled_peers *p)
{
    if (!m || !p) return fail(m, GEM_ERR_INVALID, "gem_tiled_attach: null argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    if (!m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_tiled_attach: handle is not tiled");
    const int world = p->tiles_r * p->tiles_c;
    if (world < 1 || world > ROUTE_MAX_OWNERS || p->my_rank < 0 || p->my_rank >= world || p->bucket_capacity < 1)
        return fail(m, GEM_ERR_INVALID, "gem_tiled_attach: bad geometry");
    const int nblk = (p->bucket_capacity + ROUTE_BLOCK - 1) / ROUTE_BLOCK, cap = nblk * ROUTE_BLOCK;
    if ((long long)world * cap > m->P) return fail(m, GEM_ERR_INVALID, "gem_tiled_attach: world * bucket_capacity exceeds max_points");
    int rc = drain(m);
    if (rc) return rc;
    TiledState &ts = m->tiled;
    ts.world = world; ts.my_rank = p->my_rank; ts.tiles_r = p->tiles_r; ts.tiles_c = p->tiles_c; ts.cap = cap; ts.nblk = nblk;
    for (int o = 0; o < world; o++) {
        ts.pb.rec[o] = p->recv_records[o]; ts.pb.inten[o] = p->recv_intensity[o];
        ts.pb.cnt[o] = p->recv_counts[o]; ts.pb.flag[o] = p->flags[o];
    }
    if (!ts.d_ticket && (rc = dev_alloc(m, &ts.d_ticket, 4))) return rc;
    ts.d_ntotal = ts.d_ticket + 1;
    GEM_CUDA(m, cudaMemsetAsync(ts.d_ticket, 0, 4 * sizeof(int), m->stream));
    ts.step = 0;
    ts.routed.active = false;
    if (const char *e = getenv("GEM_B200_TILED_DEPTH")) ts.depth = (atoi(e) == 3) ? 3 : 2;
    if (ts.exec) { cudaGraphExecDestroy(ts.exec); cudaGraphDestroy(ts.graph); ts.exec = nullptr; ts.graph = nullptr; }
    ts.attached = true;
    return GEM_OK;
}

// One step of a tiled map: route this rank's cloud to the owning tiles (peer stores), bin what the peers delivered,
// fold.  Pipelined three deep: call j issues ONE graph with four independent kernels {fold_long, fold of step j-2 || bin
// of step j-1 || route of step j}; what is outstanding after the last call is issued by whatever reads the map next
// (gem_flush).  Every rank must make the same sequence of gem_tiled_step calls (a bin waits for every peer's flag of
// its step).  GEM_B200_TILED_DEPTH=2: {fold_long, fold of step j-1 || route -> bin of step j}.
int gem_tiled_step(gem_map *m, const void *xyzi, const void *rgba, int n, const gem_frame *frame)
{
    if (!m || !frame || n < 0 || (n > 0 && !xyzi)) return fail(m, GEM_ERR_INVALID, "gem_tiled_step: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    TiledState &ts = m->tiled;
    if (!ts.attached) return fail(m, GEM_ERR_INVALID, "gem_tiled_step: gem_tiled_attach first");
    if (n > ts.cap) return fail(m, GEM_ERR_INVALID, "gem_tiled_step: cloud larger than bucket_capacity");
    int rc;
    const bool serial = m->profiling || m->pipe_mode == 0;
    if (serial && (rc = drain(m))) return rc;
    if (!m->pending.empty()) { // tiled maps do not scroll: only the first-fuse floor can be pending
        if ((rc = drain(m)) || (rc = flush_all_pending(m))) return rc;
    }
    ts.step++;
    const int world = ts.world;
    MapGeom gg = m->geom;
    gg.tiled = 0; // routing works on global geographic indices
    FrameParams fp = make_frame(frame);
    int th = (m->L + ts.tiles_r - 1) / ts.tiles_r, tw = (m->L + ts.tiles_c - 1) / ts.tiles_c;
    const float4 *px = (const float4 *)xyzi;
    const uchar4 *pr = (const uchar4 *)rgba;
    int nn = n, tiles_c = ts.tiles_c, my_rank = ts.my_rank, nblk = ts.nblk, cap = ts.cap, bufv = ts.step % PEER_BUFS, stepv = ts.step, worldv = world;
    int *ticket = ts.d_ticket;
    PeerBufs pb = ts.pb;
    void *route_args[] = {&gg, &fp, &px, &pr, &nn, &th, &tw, &tiles_c, &worldv, &my_rank, &nblk, &cap, &bufv, &stepv, &pb, &ticket};
    auto launch_route = [&]() -> int {
        GEM_LAUNCH(m, GEM_PROF_ROUTE, k_route_peer<<<nblk, ROUTE_BLOCK, 0, m->stream>>>(gg, fp, px, pr, nn, th, tw, tiles_c, worldv, my_rank, nblk, cap, bufv, stepv, pb, ticket));
        GEM_CUDA(m, cudaGetLastError());
        return GEM_OK;
    };
    memset(&m->stats, 0, sizeof m->stats);
    m->stats.points_in = n;
    RegionOps none{};
    int one = 1;
    const bool graphs = !serial && m->pipe_mode == 2;
    if (!graphs || ts.depth == 2) {
        // route -> bin of this step on the stream or in one graph with the previous step's folds
        if (!graphs || !m->pend.active) {
            if ((rc = drain(m)) || (rc = launch_route())) return rc;
            const TiledBin b = tiled_bin_of(m, stepv, bufv);
            if ((rc = launch_tiled_bin(m, b))) return rc;
            if (serial) return launch_fold(m, m->stream, b.fold, none, 0, true, true);
            m->pend = b.fold;
            return GEM_OK;
        }
    } else if (!ts.routed.active || !m->pend.active) {
        // depth 3, pipeline filling (first two calls, or after a flush): plain launches, one after the other
        if (!ts.routed.active) {
            if ((rc = drain(m)) || (rc = launch_route())) return rc;
        } else {
            const TiledBin b = tiled_bin_of(m, ts.routed.step, ts.routed.buf);
            if ((rc = launch_tiled_bin(m, b)) || (rc = launch_route())) return rc;
            m->pend = b.fold;
        }
        ts.routed.active = true; ts.routed.step = stepv; ts.routed.buf = bufv;
        return GEM_OK;
    }
    // steady state: one graph
    PendingFold prev = m->pend;
    TiledBin b = (ts.depth == 2) ? tiled_bin_of(m, stepv, bufv) : tiled_bin_of(m, ts.routed.step, ts.routed.buf);
    const int fb = fold_blocks_for(m, prev.n);
    int slice = fold_slice(prev.n, fb), fbk = fb;
    void *fold_args[] = {&prev.geom, &b.ml, &prev.sc, &prev.src, &none, &prev.n, &fbk, &slice, &one, &one, (void *)&prev.n_dev};
    void *long_args[] = {&prev.geom, &b.ml, &prev.sc, &prev.src, &none, &one, &one};
    void *bin_args[] = {&b.gl, &b.ml, &b.sc, &b.rec, &b.inten, &b.cnt, &b.nsub, &b.flags, &b.world, &b.step, &b.ntotal};
    cudaKernelNodeParams kl{}, kf{}, kr{}, kb{};
    kl.func = (void *)k_fold_long; kl.gridDim = dim3((unsigned)long_blocks_for(m, prev.n / world)); kl.blockDim = dim3(LONG_BLOCK); kl.sharedMemBytes = (unsigned)m->long_smem; kl.kernelParams = long_args;
    kf.func = (void *)k_fold; kf.gridDim = dim3((unsigned)fb); kf.blockDim = dim3(ADD_BLOCK); kf.sharedMemBytes = (unsigned)m->fold_smem; kf.kernelParams = fold_args;
    kr.func = (void *)k_route_peer; kr.gridDim = dim3((unsigned)nblk); kr.blockDim = dim3(ROUTE_BLOCK); kr.sharedMemBytes = 0; kr.kernelParams = route_args;
    kb.func = (void *)k_bin_peer; kb.gridDim = dim3((unsigned)bin_peer_blocks(b.nsub)); kb.blockDim = dim3(ROUTE_BLOCK); kb.sharedMemBytes = 0; kb.kernelParams = bin_args;
    if (!ts.exec) {
        GEM_CUDA(m, cudaGraphCreate(&ts.graph, 0));
        GEM_CUDA(m, cudaGraphAddKernelNode(&ts.long_node, ts.graph, nullptr, 0, &kl));
        GEM_CUDA(m, cudaGraphAddKernelNode(&ts.route_node, ts.graph, nullptr, 0, &kr));
        GEM_CUDA(m, cudaGraphAddKernelNode(&ts.fold_node, ts.graph, nullptr, 0, &kf));
        if (ts.depth == 2) GEM_CUDA(m, cudaGraphAddKernelNode(&ts.bin_node, ts.graph, &ts.route_node, 1, &kb));
        else GEM_CUDA(m, cudaGraphAddKernelNode(&ts.bin_node, ts.graph, nullptr, 0, &kb));
        GEM_CUDA(m, cudaGraphInstantiate(&ts.exec, ts.graph, 0));
    } else {
        GEM_CUDA(m, cudaGraphExecKernelNodeSetParams(ts.exec, ts.long_node, &kl));
        GEM_CUDA(m, cudaGraphExecKernelNodeSetParams(ts.exec, ts.route_node, &kr));
        GEM_CUDA(m, cudaGraphExecKernelNodeSetParams(ts.exec, ts.fold_node, &kf));
        GEM_CUDA(m, cudaGraphExecKernelNodeSetParams(ts.exec, ts.bin_node, &kb));
    }
    GEM_CUDA(m, cudaGraphLaunch(ts.exec, m->stream));
    m->launches += 4;
    m->pend = b.fold;
    if (ts.depth != 2) { ts.routed.active = true; ts.routed.step = stepv; ts.routed.buf = bufv; }
    return GEM_OK;
}

static int fuse_records_impl(gem_map *m, const void *rec, int n, const int *src_counts, int stride)
{
    if (!m || n < 0 || (n > 0 && !rec)) return fail(m, GEM_ERR_INVALID, "gem_fuse_records: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = GEM_OK;
    memset(&m->stats, 0, sizeof m->stats);
    if (n == 0) return flush_all_pending(m);
    for (int off = 0; off < n; off += m->P) {
        const int cn = (n - off < m->P) ? (n - off) : m->P;
        BinSource in{};
        in.rec = (const RouteRec *)rec + off;
        in.src_counts = src_counts; // counted buffers are never chunked (n <= max_points is checked by the caller)
        in.stride = stride;
        const FoldSrc fs{(const char *)in.rec + 16, (int)sizeof(RouteRec)};
        const FrameParams none{};
        if ((rc = enqueue_add<SRC_RECORDS>(m, in, fs, cn, none, nullptr, nullptr, false, true, true))) return rc;
        if (n > m->P && (rc = read_counters(m, cn, true))) return rc;
    }
    if (n <= m->P) m->stats.points_in = n;
    return GEM_OK;
}

} // extern "C"
