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
#include <utility>
#include <vector>

#include "../../include/gem_b200.h"
#include "gem_add.cuh"
#include "gem_colour.cuh"
#include "gem_costmap.cuh"
#include "gem_gridmsg.h"
#include "gem_inflate.cuh"
#include "gem_kernels.cuh"
#include "gem_global.cuh"
#include "gem_globalmap.h"
#include "gem_ingest.cuh"
#include "gem_mls.cuh"
#include "gem_octree.cuh"
#include "gem_pcd.cuh"
#include "gem_rosmsg.cuh"
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

// Owners of the handle's CUDA resources: each releases what it holds when it is reset, assigned over or destroyed, so
// deleting the handle releases everything it holds.  Move-only.
template <typename H, auto Release> struct Owned {
    H p = nullptr;
    Owned() = default;
    Owned(Owned &&o) noexcept : p(std::exchange(o.p, nullptr)) {}
    Owned &operator=(Owned &&o) noexcept { if (this != &o) { reset(); p = std::exchange(o.p, nullptr); } return *this; }
    ~Owned() { reset(); }
    void reset() { if (p) Release(p); p = nullptr; }
};
using Event = Owned<cudaEvent_t, cudaEventDestroy>;
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
template <typename T> using Pinned = Owned<T *, cudaFreeHost>;
struct Graph { // a CUDA graph and its executable instance
    Owned<cudaGraph_t, cudaGraphDestroy> graph;
    Owned<cudaGraphExec_t, cudaGraphExecDestroy> exec;
    void reset() { exec.reset(); graph.reset(); }
};

struct DevBuf { // a device buffer and its capacity in bytes; scratch buffers grow on demand (scratch_grow), never shrink
    void *p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(DevBuf &&o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
    DevBuf &operator=(DevBuf &&o) noexcept
    {
        if (this != &o) { reset(); p = std::exchange(o.p, nullptr); cap = std::exchange(o.cap, 0); }
        return *this;
    }
    ~DevBuf() { reset(); }
    void reset() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <typename T> T *as() const { return static_cast<T *>(p); }
};

struct TiledState { // gem_tiled_attach
    bool attached = false;
    int world = 0, my_rank = 0, tiles_r = 0, tiles_c = 0, cap = 0, nblk = 0;
    PeerBufs pb{};
    int *d_ticket = nullptr, *d_ntotal = nullptr; // [1], [2] (by call parity)
    int step = 0;
    int depth = 2;                                 // 2: {route j -> bin j || fold j-1} per call; 3: {route j || bin j-1 || fold j-2}
    struct { bool active = false; int step = 0, buf = 0; } routed; // depth 3: delivered to the owners, not binned yet
    Graph g;
    cudaGraphNode_t long_node = nullptr, fold_node = nullptr, route_node = nullptr, bin_node = nullptr;
    const void *route_func = nullptr; // the route kernel the graph was built with (k_route_peer or k_route_peer_any)
};
struct KeyRuns { // records bucketed by a 64-bit key (key_runs_grow, key_runs_enqueue): keys and record indices before /
                 // after the sort, the run lengths and their offsets, the temporary of the sort, the encoding and the scan
    DevBuf key[2], idx[2], cnt, off, temp;
};
struct VoxScratch { // gem_voxel_grid and the pre-filter (gem_voxel.cuh): the voxel keys' runs, the steps' device state
                   // (GEM_PREFILTER_MAX_STEPS VoxStep per ring slot, then gem_voxel_grid's), the pre-filter's two buffers
    KeyRuns kr;
    DevBuf acc, buf[2];
    int n = 0; // points kr and buf are sized for
};
struct MlsScratch { // gem_mls_upsample (gem_mls.cuh): the cell keys' runs, the points in cell order, the distinct cells,
                   // neighbour and output counts, output offsets, the long lists and their keys
    KeyRuns kr;
    DevBuf spts, ukey, nbr, ocnt, ooff, longs, lkeys, acc;
};
struct InflScratch { // gem_costmap_inflate (gem_inflate.cuh): per-cell keys and pop records, the tables, bin starts, block counts
    DevBuf key, pops, tab, gstart, blk;
    // the tables in `tab` were built for these parameters (r < 0: none)
    long long r = -1;
    double res = 0.0, weight = 0.0, inscribed = 0.0;
    int nbins = 0, blocks = 0;
    bool key_dirty = false; // `key` was (re)allocated and its clearing memset has not been enqueued yet
};
struct ColourScratch { // GEM_COLOUR_LOOKUP_NODE (gem_colour.cuh): the pixel keys' runs, the distinct keys, the links, and
                      // the run count followed by one changed-a-link flag per jumping round
    KeyRuns kr;
    DevBuf ukey, up, ctl;
    int n = 0; // points every buffer is sized for
};
struct SplitScratch { // gem_grid_cloud_split: geographic z, row x, column y, per-cell distance, compacted distances, queue,
                      // counters, stats
    DevBuf zg, xg, yg, dcell, dist, queue, ctr, stats;
};
struct PcdScratch { // gem_pcd_format (gem_pcd.cuh): per-tile byte counts, their inclusive scan, the scan's temporary
    DevBuf bytes, ends, temp;
};
struct OctScratch { // gem_color_octree (gem_octree.cuh); every buffer is consistent with its own capacity at all times
    KeyRuns kr;          // the leaf codes' runs; kr.temp also serves the phase-2 sorts
    DevBuf leaf, level, ghead, gid, val, groups, ctr, key2[2], nkey[2], nrec[2], dense;
    long long bytes = -1; // size of the last stream (in nrec[1]); -1: none
    double res = 0.0;     // the resolution it was built at
    gem_octree info{};
};

struct LocalStore { // localMap_ on the device (gem_harvest_to_local_map, gem_local_map_take / _clear; gem_submap.cuh)
    DevBuf buf;                        // one allocation: log, index keys, index positions, take scratch
    float4 *log = nullptr;             // 2 x float4 per record, in harvest order
    unsigned long long *keys = nullptr; // open-addressing index, HASH_EMPTY = free slot
    int *latest = nullptr;             // per slot: the latest log position of its key
    int *cnt = nullptr;                // take: kept entries per 32 log entries, then the scan's segment totals
    int n = 0, cap = 0;                // records in the log, records it can hold
    size_t slots = 0;                  // index slots (a power of two >= 2 * cap)
};

struct GlobalStore { // globalMap_, trajectory_ and localMapLoc_ on the device (gem_global_map_*; DESIGN.md f16)
    std::mutex mu;                     // the stack's own lock: no call on it takes the handle's mutex except a push, briefly
    Stream stream;                     // the stack's own stream
    Event ev;                          // push: the handle's stream -> the stack's stream
    DevBuf arena[2];                   // arena[cur]: the submaps back to back in push order; the other: the re-pack target
    int cur = 0;
    long long cap = 0;                 // records each arena buffer holds
    DevBuf meta;                       // update: counts, old and new offsets, fused count, the re-pose table
    int meta_submaps = 0;              // submaps `meta` is laid out for
    DevBuf pair;                       // update: one pair's hash tables, keep flags, scan counts and compaction output
    std::vector<int> cnt, off{0};      // host mirror: per submap its count, and its offset (one entry more)
    std::vector<float> poses{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}; // trajectory_: 16 floats per keyframe
    std::vector<float> centres{0.0f, 0.0f};                                  // localMapLoc_: x, y per keyframe
};

struct FrameGraph { // {long lists || the other lists of the previous call || bin of this call} as one three-node CUDA graph
    Graph g;
    cudaGraphNode_t long_node = nullptr, fold_node = nullptr, bin_node = nullptr;
};

struct gem_map {
    std::recursive_mutex mu;
    gem_config cfg{};
    int dev = 0;
    cudaStream_t stream = nullptr; // cfg->stream, or own_stream
    Stream own_stream;             // the stream gem_create made when the caller gave none
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
    std::map<const void *, FrameGraph> graphs; // keyed by the bin kernel function
    // deferred region operations (scroll clears of Move, the every-cell variance floor of
    // G_fuse): executed by the next add/fuse launch, or flushed before anything observes the map
    std::vector<RegionOp> pending;
    // staging (device), lazily allocated
    void *d_xyzi = nullptr, *d_rgba = nullptr, *d_pcl = nullptr;
    float *d_x = nullptr, *d_y = nullptr, *d_z = nullptr, *d_xt = nullptr, *d_yt = nullptr;
    int *d_keyin = nullptr, *d_keyout = nullptr, *d_R = nullptr, *d_G = nullptr, *d_B = nullptr;
    float *d_int = nullptr, *d_h = nullptr, *d_hv = nullptr;
    float *d_out = nullptr; // 9 * nc floats read-out staging
    RouteScratch route_sc{};
    float2 *prev_ev = nullptr;     // gem_snapshot_shown: prevMap_ (ElevationMapping.cpp:422) on the device
    uint2 *prev_ci = nullptr;
    float *prev_tr = nullptr;
    MapGeom prev_geom{};
    bool prev_valid = false;
    LocalStore local;
    int *d_viscnt = nullptr;       // visual-cloud export: per (column, row chunk) counts / offsets
    SplitScratch split;            // gem_grid_cloud_split
    OctScratch oct;                // gem_color_octree: scratch and the last stream
    DevBuf cost_scratch;           // costmap calls: the winner per costmap cell (int), or the copy of a rolled grid
    CostMarksDev *cost_acc = nullptr; // costmap mark calls: counts and encoded touch bounds
    VoxScratch vox;                // gem_voxel_grid
    MlsScratch mls;                // gem_mls_upsample
    PcdScratch pcd;                // gem_pcd_format
    int colour_lookup = GEM_COLOUR_LOOKUP_IMAGE; // gem_set_colour_lookup
    ColourScratch colour;          // gem_colourise_points / gem_add_pointcloud2_host_async in GEM_COLOUR_LOOKUP_NODE
    // the newest pre-filtered add: its ring slot and step count (gem_prefilter_info), and its filtered count on the
    // device until gem_get_stats fetches it (while call_no is still pf_call)
    int pf_slot = -1, pf_nsteps = 0;
    const int *pf_count = nullptr;
    unsigned pf_call = 0;
    DevBuf ros_framing;            // gem_ros_*: the framing bytes of the call, staged for k_ros_framing
    DevBuf ros_stage;              // gem_ros_* map messages for pinned outputs, written here and copied over in one DMA
    DevBuf cost_cells;             // gem_costmap_footprint: the cell indices the host listed
    InflScratch infl;              // gem_costmap_inflate
    DevBuf refuse;                 // gem_refuse_submaps: one pair's scratch (pair_layout)
    GlobalStore gmap;              // gem_global_map_*
    unsigned long long *d_stamps = nullptr; // gem_debug_stamps
    int *d_raylist = nullptr;      // ray clean-up: cells that cast a ray + their count
    DevBuf ray_bitmap;             // ray clean-up: validity bitmap of the lowest layer (own tile / map-wide)
    DevBuf divtest;                // gem_selftest_division: mismatch and fast-path counters
    Pinned<BinCounters> h_ctr;
    // pipelined host ingest (gem_add_points_host_async): three staging sets (the fold of call i, issued with
    // call i+1, still reads call i's intensities)
    Event ev_export, ev_export_done; // gem_export_layers_begin / _end
    Stream copy_stream;
    void *d_axyzi[3] = {nullptr, nullptr, nullptr}, *d_argba[3] = {nullptr, nullptr, nullptr};
    Event ev_h2d[3], ev_done[3];
    Pinned<BinCounters> h_ctr_ring; // 2 entries
    unsigned async_calls = 0;
    // gem_add_pointcloud2_host_async: per ring slot the message bytes and the camera image as they arrive (copy
    // stream), and one BGR8 conversion target (handle's stream); grown on demand
    DevBuf pc2_raw[3], pc2_img[3], pc2_bgr;
    // gem_add_points_multi: ring of per-call FrameParams tables (pinned host + device)
    Pinned<FrameParams> h_frames;
    FrameParams *d_frames = nullptr;
    Event ev_frames[4];
    unsigned multi_calls = 0;
    gem_stats stats{};
    std::string err;
    std::vector<DevBuf> allocs;
    // launch accounting / optional per-kernel CUDA-event timing (gem_profile_*)
    long long launches = 0;
    bool profiling = false;
    struct Span { int cls; Event e0, e1; };
    std::vector<Span> spans;
    std::vector<Event> free_events;
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

Event prof_event(gem_map *m)
{
    Event e;
    if (!m->free_events.empty()) {
        e = std::move(m->free_events.back());
        m->free_events.pop_back();
    } else {
        cudaEventCreate(&e.p);
    }
    return e;
}
// every kernel launch of the library goes through this macro: counts the launch and, when
// profiling is on, brackets it with CUDA events on the handle's stream
#define GEM_LAUNCH(m, cls, ...)                                  \
    do {                                                         \
        (m)->launches++;                                         \
        if ((m)->profiling) {                                    \
            gem_map::Span sp__{(cls), prof_event(m), prof_event(m)}; \
            cudaEventRecord(sp__.e0.p, (m)->stream);             \
            __VA_ARGS__;                                         \
            cudaEventRecord(sp__.e1.p, (m)->stream);             \
            (m)->spans.push_back(std::move(sp__));               \
        } else {                                                 \
            __VA_ARGS__;                                         \
        }                                                        \
    } while (0)

#define GEM_CUDA(m, expr)                                                                      \
    do {                                                                                       \
        cudaError_t e__ = (expr);                                                              \
        if (e__ != cudaSuccess) {                                                              \
            return fail((m), GEM_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e__)); \
        }                                                                                      \
    } while (0)

// a buffer that lives as long as the handle (the handle keeps it in m->allocs)
template <typename T> int dev_alloc(gem_map *m, T **p, size_t count)
{
    DevBuf b;
    cudaError_t e = cudaMalloc(&b.p, count * sizeof(T) + 16);
    if (e != cudaSuccess) {
        cudaGetLastError(); // a failed cudaMalloc stays recorded as the last error, which the next launch check would report
        return fail(m, GEM_ERR_NOMEM, std::string("cudaMalloc: ") + cudaGetErrorString(e));
    }
    *p = b.as<T>();
    m->allocs.push_back(std::move(b));
    return GEM_OK;
}
// pinned host memory, with dev_alloc's contract
template <typename T> int host_alloc(gem_map *m, Pinned<T> &h, size_t count)
{
    void *q = nullptr;
    cudaError_t e = cudaHostAlloc(&q, count * sizeof(T), cudaHostAllocDefault);
    if (e != cudaSuccess) {
        cudaGetLastError(); // as in dev_alloc
        return fail(m, GEM_ERR_NOMEM, std::string("cudaHostAlloc: ") + cudaGetErrorString(e));
    }
    h.p = static_cast<T *>(q);
    return GEM_OK;
}

// Grow a device scratch buffer to at least `bytes`, with a quarter of slack and at least 4 KiB so that slowly growing
// inputs do not reallocate on every call.  The new buffer is allocated before the old one is released, so a failed
// growth leaves the buffer as it was; `stream` (the one the buffer's users run on) is drained before the old buffer
// goes, because work queued on it (an update_origin, say) may still read it.
int scratch_grow(gem_map *m, DevBuf &b, size_t bytes, const char *what, cudaStream_t stream)
{
    if (b.cap >= bytes) return GEM_OK;
    bytes = std::max(bytes + bytes / 4, (size_t)4096);
    DevBuf q;
    const cudaError_t e = cudaMalloc(&q.p, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError(); // as in dev_alloc
        return fail(m, GEM_ERR_NOMEM, std::string(what) + ": cudaMalloc: " + cudaGetErrorString(e));
    }
    q.cap = bytes;
    if (b.p) cudaStreamSynchronize(stream);
    b = std::move(q);
    return GEM_OK;
}

// Size every buffer of `k` for n records, its temporary for the sort (up to 64 key bits), the run-length encoding, the
// scan of the run lengths and `temp_bytes` more that the caller needs later.  Every buffer is sized before the first
// write, so that a failed growth writes nothing.
int key_runs_grow(gem_map *m, KeyRuns &k, int n, size_t temp_bytes, const char *what)
{
    using u64 = unsigned long long;
    const size_t N = (size_t)n;
    cudaStream_t st = m->stream;
    size_t t_sort = 0, t_rle = 0, t_scan = 0;
    GEM_CUDA(m, cub::DeviceRadixSort::SortPairs(nullptr, t_sort, (u64 *)nullptr, (u64 *)nullptr, (int *)nullptr, (int *)nullptr, n, 0, 64, st));
    GEM_CUDA(m, cub::DeviceRunLengthEncode::Encode(nullptr, t_rle, (u64 *)nullptr, (u64 *)nullptr, (int *)nullptr, (int *)nullptr, n, st));
    GEM_CUDA(m, cub::DeviceScan::ExclusiveSum(nullptr, t_scan, (int *)nullptr, (int *)nullptr, n, st));
    int rc;
    if ((rc = scratch_grow(m, k.key[0], N * 8, what, st)) || (rc = scratch_grow(m, k.key[1], N * 8, what, st)) ||
        (rc = scratch_grow(m, k.idx[0], N * 4, what, st)) || (rc = scratch_grow(m, k.idx[1], N * 4, what, st)) ||
        (rc = scratch_grow(m, k.cnt, N * 4, what, st)) || (rc = scratch_grow(m, k.off, N * 4, what, st)))
        return rc;
    return scratch_grow(m, k.temp, std::max(std::max(t_sort, t_rle), std::max(t_scan, temp_bytes)), what, st);
}

// Bucket the n records whose keys and indices the caller wrote to k.key[0] and k.idx[0]: the stable sort on key bits
// [0, bits) into k.key[1] / k.idx[1], the runs of equal keys (their keys to `unique`, their lengths to k.cnt, their number
// to *nruns, all on the device) and the runs' offsets in k.off, issued on the handle's stream
int key_runs_enqueue(gem_map *m, KeyRuns &k, int n, int bits, unsigned long long *unique, int *nruns)
{
    using u64 = unsigned long long;
    cudaStream_t st = m->stream;
    size_t tcap = k.temp.cap;
    // the run-length encoding writes nruns <= n counts; the scan runs over all n, so the rest must be defined
    GEM_CUDA(m, cudaMemsetAsync(k.cnt.p, 0, (size_t)n * sizeof(int), st));
    GEM_CUDA(m, cub::DeviceRadixSort::SortPairs(k.temp.p, tcap, k.key[0].as<u64>(), k.key[1].as<u64>(), k.idx[0].as<int>(), k.idx[1].as<int>(), n, 0, bits, st));
    GEM_CUDA(m, cub::DeviceRunLengthEncode::Encode(k.temp.p, tcap, k.key[1].as<u64>(), unique, k.cnt.as<int>(), nruns, n, st));
    GEM_CUDA(m, cub::DeviceScan::ExclusiveSum(k.temp.p, tcap, k.cnt.as<int>(), k.off.as<int>(), n, st));
    return GEM_OK;
}

bool ranges_meet(const void *a, size_t na, const void *b, size_t nb)
{
    const uintptr_t a0 = (uintptr_t)a, b0 = (uintptr_t)b;
    return na > 0 && nb > 0 && a0 < b0 + nb && b0 < a0 + na;
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
    for (int i = 0; i < 9; i++) {
        p.rotVar[i] = f->rotation_variance[i];
        p.CSBT[i] = f->C_SB_transpose[i];
        p.Bskew[i] = f->B_r_BS_skew[i];
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
    for (int i = 0; i < 5; i++) p.sp[i] = f->sensor.stereo_p[i];
    p.dtd = f->sensor.depth_to_disparity_factor;
    p.width = f->sensor.cloud_width;
    p.idx0 = 0;
    return p;
}
// a sensor model the kernels implement: an unknown type must not run as a laser
bool sensor_ok(const gem_sensor_model &s)
{
    return s.type >= GEM_SENSOR_LASER && s.type <= GEM_SENSOR_PERFECT && s.cloud_width >= 0;
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
int launch_fold(gem_map *m, const PendingFold &p, const RegionOps &ro, int region_blocks, bool do_fuse, bool do_lowest)
{
    const int fb = fold_blocks_for(m, p.n);
    const int slice = fold_slice(p.n, fb);
    // the long lists first (their blocks claim whole SMs), then everything else; on one stream the two run back to back
    // (disjoint cells, so the order is free) -- the frame graph of the pipelined mode runs them side by side.  Both get
    // the next call's clears `ro`: a long list inside a cleared band must store the cleared value itself, because
    // k_fold's region blocks may clear the cell before k_fold_long writes it (cell_end)
    GEM_LAUNCH(m, GEM_PROF_FOLD_LONG, k_fold_long<<<long_blocks_for(m, p.n), LONG_BLOCK, m->long_smem, m->stream>>>(p.geom, m->ml, p.sc, p.src, ro, do_fuse ? 1 : 0, do_lowest ? 1 : 0));
    GEM_LAUNCH(m, GEM_PROF_FOLD, k_fold<<<fb + region_blocks, ADD_BLOCK, m->fold_smem, m->stream>>>(p.geom, m->ml, p.sc, p.src, ro, p.n, fb, slice, do_fuse ? 1 : 0, do_lowest ? 1 : 0, p.n_dev));
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
        if ((rc = launch_fold(m, m->pend, none, 0, true, true))) return rc;
        m->pend.active = false;
    }
    if (m->tiled.routed.active) { // a tiled step that is routed but not binned: bin it, fold it
        const TiledBin b = tiled_bin_of(m, m->tiled.routed.step, m->tiled.routed.buf);
        m->tiled.routed.active = false;
        if ((rc = launch_tiled_bin(m, b)) || (rc = launch_fold(m, b.fold, none, 0, true, true))) return rc;
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
// any: a frame uses the stereo or perfect model -> the every-model instantiation, one point per thread
template <int SRC> BinKernel bin_kernel(int U, bool any)
{
    constexpr int S = SRC & ~SRC_DEVN;
    if constexpr (S == SRC_XYZI || S == SRC_SOA || S == SRC_PCL32) {
        if (any) return k_bin<SRC | SRC_ANY_MODEL, 1>;
    }
    if (S == SRC_XYZI || S == SRC_RECORDS) {
        if (U == 4) return k_bin<SRC, 4>;
        if (U == 2) return k_bin<SRC, 2>;
    }
    return k_bin<SRC, 1>;
}

int read_counters(gem_map *m, long long n_in, bool accumulate)
{
    int rc = drain(m);
    if (rc) return rc;
    GEM_CUDA(m, cudaMemcpyAsync(m->h_ctr.p, m->ctr_last, sizeof(BinCounters), cudaMemcpyDeviceToHost, m->stream));
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    if (!accumulate) memset(&m->stats, 0, sizeof m->stats);
    m->stats.points_in += n_in;
    m->stats.points_binned += m->h_ctr.p->total;
    m->stats.cells_touched += m->h_ctr.p->ntouched;
    if (m->h_ctr.p->pool > m->bs[0].pool_cap) return fail(m, GEM_ERR_CUDA, "internal: record pool exhausted");
    if (m->h_ctr.p->nlong >= m->bs[0].long_cap || m->h_ctr.p->nlarge >= m->bs[0].large_cap) return fail(m, GEM_ERR_CUDA, "internal: list queue overflow");
    if (m->h_ctr.p->maxk > m->stats.max_points_per_cell) m->stats.max_points_per_cell = m->h_ctr.p->maxk;
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
    if (m->ev_export_done.p) cudaStreamWaitEvent(m->stream, m->ev_export_done.p, 0); // an asynchronous export may still be reading the staging buffer
    if (m->d_out) return GEM_OK;
    return dev_alloc(m, &m->d_out, m->nc * 9);
}

int ensure_ray_scratch(gem_map *m, size_t bitmap_cells)
{
    int rc;
    if (!m->d_raylist && (rc = dev_alloc(m, &m->d_raylist, m->nc + 1))) return rc; // every cell may cast a ray; [nc] = the count
    return scratch_grow(m, m->ray_bitmap, (bitmap_cells / 32 + 1) * sizeof(uint32_t), "raytracing", m->stream);
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

// {long lists, other lists of the previous call || bin of this call} as a three-node graph, built once per bin kernel; per
// call only the node parameters change.  One cudaGraphLaunch runs the three side by side on the handle's stream.
int launch_frame_graph(gem_map *m, BinKernel bk, void **bin_args, int bin_grid, void **fold_args, int fold_grid, void **long_args, int long_grid)
{
    FrameGraph &fg = m->graphs[(const void *)bk];
    Graph &g = fg.g;
    cudaKernelNodeParams kb{}, kf{}, kl{};
    kb.func = (void *)bk; kb.gridDim = dim3((unsigned)bin_grid); kb.blockDim = dim3(ADD_BLOCK); kb.sharedMemBytes = (unsigned)m->bin_smem; kb.kernelParams = bin_args;
    kf.func = (void *)k_fold; kf.gridDim = dim3((unsigned)fold_grid); kf.blockDim = dim3(ADD_BLOCK); kf.sharedMemBytes = (unsigned)m->fold_smem; kf.kernelParams = fold_args;
    kl.func = (void *)k_fold_long; kl.gridDim = dim3((unsigned)long_grid); kl.blockDim = dim3(LONG_BLOCK); kl.sharedMemBytes = (unsigned)m->long_smem; kl.kernelParams = long_args;
    if (!g.exec.p) {
        g.reset(); // what a build that failed part way left
        GEM_CUDA(m, cudaGraphCreate(&g.graph.p, 0));
        GEM_CUDA(m, cudaGraphAddKernelNode(&fg.long_node, g.graph.p, nullptr, 0, &kl)); // first: its blocks want empty SMs
        GEM_CUDA(m, cudaGraphAddKernelNode(&fg.fold_node, g.graph.p, nullptr, 0, &kf));
        GEM_CUDA(m, cudaGraphAddKernelNode(&fg.bin_node, g.graph.p, nullptr, 0, &kb));
        GEM_CUDA(m, cudaGraphInstantiate(&g.exec.p, g.graph.p, 0));
    } else {
        GEM_CUDA(m, cudaGraphExecKernelNodeSetParams(g.exec.p, fg.long_node, &kl));
        GEM_CUDA(m, cudaGraphExecKernelNodeSetParams(g.exec.p, fg.fold_node, &kf));
        GEM_CUDA(m, cudaGraphExecKernelNodeSetParams(g.exec.p, fg.bin_node, &kb));
    }
    GEM_CUDA(m, cudaGraphLaunch(g.exec.p, m->stream));
    m->launches += 3;
    return GEM_OK;
}

// One add call on device-resident input.  pipelined == false: bin (+ deferred region operations) then fold, both
// on the handle's stream.  pipelined == true: the bin kernel of this call is issued together with the FOLD OF THE
// PREVIOUS pipelined call (which also carries the row / column clears this call's Move decided), and this call's
// fold stays pending until the next call or until anything observes the map (drain).
// any_segment: some segment of a multi-cloud call uses the stereo or perfect model (fp is segment 0's frame)
template <int SRC>
int enqueue_add(gem_map *m, const BinSource &in, const FoldSrc &fsrc, int n, const FrameParams &fp, const SegTable *segs,
                const FrameParams *frames, bool pipelined, bool do_fuse, bool do_lowest, bool any_segment = false,
                const int *n_dev = nullptr)
{
    int rc;
    if (m->profiling) pipelined = false; // per-kernel event timing needs the serial schedule
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
    const bool any = any_segment || any_model(fp);
    const int U = any ? 1 : points_per_thread(n);
    BinKernel bk = bin_kernel<SRC>(U, any);
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
    cur.active = true; cur.sc = sc; cur.src = fsrc; cur.geom = m->geom; cur.n = n; cur.n_dev = n_dev;
    if (!pipelined || !m->pend.active) {
        // nothing in flight: the bin kernel carries the deferred region operations in spare blocks
        if ((rc = take_region_ops(m, ro, rb))) return rc;
        GEM_LAUNCH(m, GEM_PROF_BIN, bk<<<pb + rb, ADD_BLOCK, m->bin_smem, m->stream>>>(g, ml, f, bin, nn, sc, ro, pb, st, frames));
        GEM_CUDA(m, cudaGetLastError());
        commit_region_ops(m);
        if (!pipelined) {
            RegionOps none{};
            if ((rc = launch_fold(m, cur, none, 0, do_fuse, do_lowest))) return rc;
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
        int pbk = pb, one = 1, fbk = fb;
        void *bin_args[] = {&g, &ml, &f, &bin, &nn, &sc, &none, &pbk, &st, (void *)&frames};
        void *fold_args[] = {&prev.geom, &ml, &prev.sc, &prev.src, &ro, &prev.n, &fbk, &slice, &one, &one, (void *)&prev.n_dev};
        void *long_args[] = {&prev.geom, &ml, &prev.sc, &prev.src, &ro, &one, &one}; // the clears, like k_fold (launch_fold)
        if ((rc = launch_frame_graph(m, bk, bin_args, pb, fold_args, fb + rb, long_args, long_blocks_for(m, prev.n)))) return rc;
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

// the cells and the geometry of the shown map or of the snapshot gem_snapshot_shown took (out = nullptr)
static GridCloudSrc grid_cells(const gem_map *m, int source)
{
    const MapGeom &g = source == GEM_GRID_SHOWN ? m->geom : m->prev_geom;
    GridCloudSrc src;
    src.s = source == GEM_GRID_SHOWN ? live_cells(m->ml) : snapshot_cells(m->prev_ev, m->prev_ci, m->prev_tr);
    src.f = grid_frame(m, g.cx, g.cy, g.sx, g.sy);
    src.out = nullptr;
    return src;
}

// the grid a call `what` reads (GEM_GRID_SHOWN or GEM_GRID_SNAPSHOT), ready to be read; the caller holds the lock
static int grid_source(gem_map *m, int source, const char *what, GridCloudSrc *src)
{
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, std::string(what) + ": not available on tiled handles");
    if (source == GEM_GRID_SNAPSHOT && !m->prev_valid)
        return fail(m, GEM_ERR_INVALID, std::string(what) + ": no snapshot (call gem_snapshot_shown first)");
    const int rc = flush_for_observer(m);
    if (rc) return rc;
    *src = grid_cells(m, source);
    return GEM_OK;
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
        e = cudaStreamCreateWithFlags(&m->own_stream.p, cudaStreamNonBlocking);
        if (e != cudaSuccess) { m->err = cudaGetErrorString(e); return bail(GEM_ERR_CUDA); }
        m->stream = m->own_stream.p;
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
    if (host_alloc(m, m->h_ctr, 1)) return bail(GEM_ERR_CUDA);
    // G_Init_map gpu.cu:198-214.  A call that failed earlier on this thread (any handle; it was reported then) leaves its
    // error behind: clear it, so that the launch check below sees this handle's launches only
    cudaGetLastError();
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
    SetDev sd(m->dev); // the owners release on the handle's device
    {
        Lock lk(m->mu);
        // every stream the handle issues work to is drained before any owner runs: nothing queued may still use what
        // the owners release
        for (cudaStream_t s : {m->stream, m->copy_stream.p, m->gmap.stream.p})
            if (s) cudaStreamSynchronize(s);
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
    if (!m || !frame || n < 0 || (n > 0 && !xyzi) || !sensor_ok(frame->sensor)) return fail(m, GEM_ERR_INVALID, "gem_add_points: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = GEM_OK;
    FrameParams fp = make_frame(frame);
    memset(&m->stats, 0, sizeof m->stats);
    if (n == 0) return flush_all_pending(m);
    for (int off = 0; off < n; off += m->P) {
        const int cn = (n - off < m->P) ? (n - off) : m->P;
        const BinSource in = xyzi_source(xyzi, rgba, off);
        fp.idx0 = off; // the stereo model indexes the caller's cloud
        const FoldSrc fs{in.xyzi ? (const char *)in.xyzi + 12 : nullptr, 16};
        if ((rc = enqueue_add<SRC_XYZI>(m, in, fs, cn, fp, nullptr, nullptr, false, true, true))) return rc;
        if (n > m->P && (rc = read_counters(m, cn, true))) return rc; // chunked: keep totals
    }
    if (n <= m->P) m->stats.points_in = n; // counters are fetched lazily by gem_get_stats
    return GEM_OK;
}

int gem_add_points_host(gem_map *m, const void *xyzi, const void *rgba, int n, const gem_frame *frame)
{
    if (!m || !frame || n < 0 || (n > 0 && !xyzi) || !sensor_ok(frame->sensor)) return fail(m, GEM_ERR_INVALID, "gem_add_points_host: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_host_staging(m);
    if (rc) return rc;
    FrameParams fp = make_frame(frame);
    memset(&m->stats, 0, sizeof m->stats);
    if (n == 0) { if ((rc = flush_all_pending(m))) return rc; return gem_sync(m); }
    if ((rc = drain(m))) return rc; // the staging buffers may still feed a deferred fold
    for (int off = 0; off < n; off += m->P) {
        const int cn = (n - off < m->P) ? (n - off) : m->P;
        fp.idx0 = off;
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
    if (!m || !frame || n < 0 || (n > 0 && !xyzi) || !sensor_ok(frame->sensor)) return fail(m, GEM_ERR_INVALID, "gem_add_points_stream: bad argument");
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
    bool any = false;
    for (int s = 0; s < n_segments; s++) {
        if (!sensor_ok(frames[s].sensor)) return fail(m, GEM_ERR_INVALID, "gem_add_points_multi: bad sensor model");
        any = any || frames[s].sensor.type == GEM_SENSOR_STEREO || frames[s].sensor.type == GEM_SENSOR_PERFECT;
    }
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = GEM_OK;
    if (!m->h_frames.p && (rc = host_alloc(m, m->h_frames, (size_t)4 * MAX_SEGMENTS))) return rc;
    if (!m->d_frames && (rc = dev_alloc(m, &m->d_frames, (size_t)4 * MAX_SEGMENTS))) return rc;
    for (int i = 0; i < 4; i++)
        if (!m->ev_frames[i].p) GEM_CUDA(m, cudaEventCreateWithFlags(&m->ev_frames[i].p, cudaEventDisableTiming));
    if (n == 0) return flush_all_pending(m);
    const int slot = (int)(m->multi_calls++ & 3u);
    if (m->multi_calls > 4) GEM_CUDA(m, cudaEventSynchronize(m->ev_frames[slot].p)); // pinned slot free again
    FrameParams *hf = m->h_frames.p + (size_t)slot * MAX_SEGMENTS, *df = m->d_frames + (size_t)slot * MAX_SEGMENTS;
    SegTable st{};
    st.n = n_segments;
    for (int s = 0; s <= n_segments; s++) st.off[s] = offsets[s];
    for (int s = 0; s < n_segments; s++) {
        hf[s] = make_frame(&frames[s]);
        hf[s].idx0 = -offsets[s]; // every segment is a cloud of its own
    }
    GEM_CUDA(m, cudaMemcpyAsync(df, hf, (size_t)n_segments * sizeof(FrameParams), cudaMemcpyHostToDevice, m->stream));
    GEM_CUDA(m, cudaEventRecord(m->ev_frames[slot].p, m->stream));
    const BinSource in = xyzi_source(xyzi, rgba, 0);
    const FoldSrc fs{in.xyzi ? (const char *)in.xyzi + 12 : nullptr, 16};
    // pipelined like gem_add_points_stream: consecutive multi-sensor steps overlap bin(i+1) with fold(i)
    if ((rc = enqueue_add<SRC_XYZI>(m, in, fs, n, hf[0], &st, df, true, true, true, any))) return rc;
    memset(&m->stats, 0, sizeof m->stats);
    m->stats.points_in = n;
    return GEM_OK;
}

// gem_add_points_host_async / gem_add_pointcloud2_host_async: lazy set-up of the shared ring (every handle created at most
// once, also after a partial failure): copy stream, three staging sets, events, counter ring
static int ensure_async_ring(gem_map *m)
{
    int rc = GEM_OK;
    if (!m->copy_stream.p) GEM_CUDA(m, cudaStreamCreateWithFlags(&m->copy_stream.p, cudaStreamNonBlocking));
    for (int i = 0; i < 3; i++) {
        if (!m->d_axyzi[i] && (rc = dev_alloc(m, (float4 **)&m->d_axyzi[i], (size_t)m->P))) return rc;
        if (!m->d_argba[i] && (rc = dev_alloc(m, (uchar4 **)&m->d_argba[i], (size_t)m->P))) return rc;
        if (!m->ev_h2d[i].p) GEM_CUDA(m, cudaEventCreateWithFlags(&m->ev_h2d[i].p, cudaEventDisableTiming));
        if (!m->ev_done[i].p) {
            GEM_CUDA(m, cudaEventCreateWithFlags(&m->ev_done[i].p, cudaEventDisableTiming));
            GEM_CUDA(m, cudaEventRecord(m->ev_done[i].p, m->stream));
        }
    }
    if (!m->h_ctr_ring.p) return host_alloc(m, m->h_ctr_ring, 2);
    return GEM_OK;
}

// the pipelined add of ring call i, whose points are in staging set i % 3 on the handle's stream
// (n_dev: the count is min(n, *n_dev), known on the device only)
static int async_add_slot(gem_map *m, unsigned i, int n, bool rgba, const gem_frame *frame, const int *n_dev = nullptr)
{
    const int b = (int)(i % 3u);
    const FrameParams fp = make_frame(frame);
    BinSource in = xyzi_source(m->d_axyzi[b], rgba ? m->d_argba[b] : nullptr, 0);
    in.n_dev = n_dev;
    const FoldSrc fs{in.xyzi ? (const char *)in.xyzi + 12 : nullptr, 16};
    BinCounters *prev_ctr = m->pend.active ? m->pend.sc.ctr : nullptr;
    int rc = n_dev ? enqueue_add<SRC_XYZI | SRC_DEVN>(m, in, fs, n, fp, nullptr, nullptr, true, true, true, false, n_dev)
                   : enqueue_add<SRC_XYZI>(m, in, fs, n, fp, nullptr, nullptr, true, true, true);
    if (rc) return rc;
    // the step's host-visible result: the counters of the newest call whose fold has been issued
    GEM_CUDA(m, cudaMemcpyAsync(&m->h_ctr_ring.p[i & 1u], prev_ctr ? prev_ctr : m->ctr_last, sizeof(BinCounters), cudaMemcpyDeviceToHost, m->stream));
    // staging set (i-1) % 3 was last read by the fold just issued (or by this call's own fold in the serial fallback)
    GEM_CUDA(m, cudaEventRecord(m->ev_done[(i + 2u) % 3u].p, m->stream));
    if (!m->pend.active) GEM_CUDA(m, cudaEventRecord(m->ev_done[b].p, m->stream));
    memset(&m->stats, 0, sizeof m->stats);
    m->stats.points_in = n; // the rest is fetched by gem_get_stats
    m->pf_count = n_dev;    // ... and a device count with it
    m->pf_call = m->call_no;
    return GEM_OK;
}

int gem_add_points_host_async(gem_map *m, const void *xyzi, const void *rgba, int n, const gem_frame *frame)
{
    if (!m || !frame || n < 0 || (n > 0 && !xyzi) || !sensor_ok(frame->sensor)) return fail(m, GEM_ERR_INVALID, "gem_add_points_host_async: bad argument");
    if (n > m->P) return fail(m, GEM_ERR_INVALID, "gem_add_points_host_async: n exceeds max_points (use gem_add_points_host)");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_async_ring(m);
    if (rc) return rc;
    if (n == 0) return flush_all_pending(m);
    const unsigned i = m->async_calls++;
    const int b = (int)(i % 3u);
    // copy stream: wait until the fold that last read staging set b (call i-3) has been issued and is done, then H2D
    GEM_CUDA(m, cudaStreamWaitEvent(m->copy_stream.p, m->ev_done[b].p, 0));
    GEM_CUDA(m, cudaMemcpyAsync(m->d_axyzi[b], xyzi, (size_t)n * 16, cudaMemcpyHostToDevice, m->copy_stream.p));
    if (rgba) GEM_CUDA(m, cudaMemcpyAsync(m->d_argba[b], rgba, (size_t)n * 4, cudaMemcpyHostToDevice, m->copy_stream.p));
    GEM_CUDA(m, cudaEventRecord(m->ev_h2d[b].p, m->copy_stream.p));
    // compute stream: wait for the copy, issue {fold of the previous call || bin of this one}
    GEM_CUDA(m, cudaStreamWaitEvent(m->stream, m->ev_h2d[b].p, 0));
    return async_add_slot(m, i, n, rgba != nullptr, frame);
}

int gem_add_cloud_pcl_host(gem_map *m, const void *pts, int n, const gem_frame *frame)
{
    if (!m || !frame || n < 0 || (n > 0 && !pts) || !sensor_ok(frame->sensor)) return fail(m, GEM_ERR_INVALID, "gem_add_cloud_pcl_host: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_pcl_staging(m);
    if (rc) return rc;
    FrameParams fp = make_frame(frame);
    memset(&m->stats, 0, sizeof m->stats);
    if (n == 0) { if ((rc = flush_all_pending(m))) return rc; return gem_sync(m); }
    if ((rc = drain(m))) return rc;
    for (int off = 0; off < n; off += m->P) {
        const int cn = (n - off < m->P) ? (n - off) : m->P;
        fp.idx0 = off;
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
    if (!m || !frame || n < 0 || (n > 0 && (!x || !y || !z)) || !sensor_ok(frame->sensor))
        return fail(m, GEM_ERR_INVALID, "gem_process_points: bad argument");
    if (m->geom.tiled) return fail(m, GEM_ERR_INVALID, "gem_process_points: not available on tiled handles");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_compat_staging(m);
    if (rc) return rc;
    FrameParams fp = make_frame(frame);
    memset(&m->stats, 0, sizeof m->stats);
    if ((rc = drain(m))) return rc;
    // Process_points does not fuse: clears/floors stay pending (they are handed to the bin kernel only by fusing calls)
    std::vector<RegionOp> keep;
    keep.swap(m->pending);
    for (int off = 0; off < n && rc == GEM_OK; off += m->P) {
        const int cn = (n - off < m->P) ? (n - off) : m->P;
        const size_t b = (size_t)cn * 4;
        fp.idx0 = off;
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
    GEM_LAUNCH(m, GEM_PROF_RAYTRACE, k_lowest_bitmap<<<blocks_for(ng, 256, 1 << 30), 256, 0, m->stream>>>(global_lowest, (int)ng, m->ray_bitmap.as<uint32_t>()));
    GEM_LAUNCH(m, GEM_PROF_RAYTRACE, k_ray_trace<<<NUM_SMS * 8, 256, 0, m->stream>>>(m->geom, mlg, m->ray_bitmap.as<uint32_t>(), m->sensorZ, m->d_raylist, ray_count));
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
    uint32_t *bitmap = m->ray_bitmap.as<uint32_t>();
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

static ProjParams proj_params(const double Tc[12], const double Tl[16], int width, int height, int row_stride)
{
    ProjParams pp;
    for (int i = 0; i < 3; i++) // P_lidar2img = Tcamera * TLidar (ElevationMapping.cpp:347), double, left-to-right sums
        for (int j = 0; j < 4; j++) {
            double a = Tc[4 * i + 0] * Tl[0 + j];
            for (int k = 1; k < 4; k++) a = a + Tc[4 * i + k] * Tl[4 * k + j];
            pp.P[4 * i + j] = a;
        }
    pp.width = width; pp.height = height; pp.row_stride = row_stride;
    return pp;
}

int gem_set_colour_lookup(gem_map *m, int mode)
{
    if (!m) return GEM_ERR_INVALID;
    if (mode != GEM_COLOUR_LOOKUP_IMAGE && mode != GEM_COLOUR_LOOKUP_NODE)
        return fail(m, GEM_ERR_INVALID, "gem_set_colour_lookup: mode is not GEM_COLOUR_LOOKUP_IMAGE or GEM_COLOUR_LOOKUP_NODE");
    Lock lk(m->mu);
    m->colour_lookup = mode;
    return GEM_OK;
}

// rounds of k_colour_jump that reach the root of a chain of n points: 2^R >= n - 1 links
static int colour_rounds(int n)
{
    int r = 0;
    while ((1ll << r) < (long long)n - 1) r++;
    return r;
}

// size the NODE lookup's scratch for n points before anything is enqueued (a failed growth writes nothing)
static int colour_grow(gem_map *m, int n, const char *what)
{
    ColourScratch &S = m->colour;
    if (S.n >= n) return GEM_OK;
    const size_t N = (size_t)n;
    int rc;
    if ((rc = key_runs_grow(m, S.kr, n, 0, what)) || (rc = scratch_grow(m, S.ukey, N * 8, what, m->stream)) ||
        (rc = scratch_grow(m, S.up, N * 4, what, m->stream)) ||
        (rc = scratch_grow(m, S.ctl, (size_t)(colour_rounds(n) + 1) * sizeof(int), what, m->stream)))
        return rc;
    S.n = n;
    return GEM_OK;
}

// colour n > 0 points from a BGR8 image on the handle's stream by the handle's lookup mode: k_colourise (IMAGE), or the
// node's painted lookup of gem_colour.cuh (NODE; colour_grow(n) first)
static int colourise_enqueue(gem_map *m, float4 *xyzi, int n, const ProjParams &pp, const unsigned char *bgr, uchar4 *rgba)
{
    cudaStream_t st = m->stream;
    const int blocks = blocks_for((size_t)n, 256);
    if (m->colour_lookup == GEM_COLOUR_LOOKUP_IMAGE) {
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_colourise<<<blocks, 256, 0, st>>>(xyzi, n, pp, bgr, rgba));
        GEM_CUDA(m, cudaGetLastError());
        return GEM_OK;
    }
    using u64 = unsigned long long;
    ColourScratch &S = m->colour;
    const u64 keys = (u64)pp.width * (u64)pp.height + 1; // the pixels and the sentinel
    int bits = 0;
    while ((1ull << bits) < keys) bits++;
    const int rounds = colour_rounds(n);
    int *ctl = S.ctl.as<int>();
    GEM_CUDA(m, cudaMemsetAsync(ctl, 0, (size_t)(rounds + 1) * sizeof(int), st));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_colour_keys<<<blocks, 256, 0, st>>>(xyzi, n, pp, S.kr.key[0].as<u64>(), S.kr.idx[0].as<int>(), rgba));
    GEM_CUDA(m, cudaGetLastError());
    int rc = key_runs_enqueue(m, S.kr, n, bits, S.ukey.as<u64>(), ctl);
    if (rc) return rc;
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_colour_parent<<<blocks, 256, 0, st>>>(S.kr.key[0].as<u64>(), n, pp.width, pp.height,
                                                                             S.ukey.as<u64>(), ctl, S.kr.off.as<int>(),
                                                                             S.kr.cnt.as<int>(), S.kr.idx[1].as<int>(), S.up.as<int>()));
    for (int r = 0; r < rounds; r++)
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_colour_jump<<<blocks, 256, 0, st>>>(S.up.as<int>(), n, ctl + 1, r));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_colour_gather<<<blocks, 256, 0, st>>>(S.kr.key[0].as<u64>(), S.up.as<int>(), n, pp.width,
                                                                             pp.height, pp.row_stride, bgr, rgba));
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
    const ProjParams pp = proj_params(Tc, Tl, width, height, row_stride);
    if (n == 0) {
        GEM_CUDA(m, cudaGetLastError());
        return GEM_OK;
    }
    if (m->colour_lookup == GEM_COLOUR_LOOKUP_NODE) {
        const int rc = colour_grow(m, n, "gem_colourise_points");
        if (rc) return rc;
    }
    return colourise_enqueue(m, (float4 *)xyzi, n, pp, bgr, (uchar4 *)rgba_out);
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
    if (!m->copy_stream.p) GEM_CUDA(m, cudaStreamCreateWithFlags(&m->copy_stream.p, cudaStreamNonBlocking));
    if (!m->ev_export.p) GEM_CUDA(m, cudaEventCreateWithFlags(&m->ev_export.p, cudaEventDisableTiming));
    if (!m->ev_export_done.p) GEM_CUDA(m, cudaEventCreateWithFlags(&m->ev_export_done.p, cudaEventDisableTiming));
    dim3 grid((m->L + 31) / 32, (m->L + 31) / 32);
    GEM_CUDA(m, cudaStreamWaitEvent(m->stream, m->ev_export_done.p, 0)); // the previous export's copies have left the staging buffer
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_export_colmajor<<<grid, 256, 0, m->stream>>>(m->ml, m->L, m->d_out));
    GEM_CUDA(m, cudaGetLastError());
    GEM_CUDA(m, cudaEventRecord(m->ev_export.p, m->stream));
    GEM_CUDA(m, cudaStreamWaitEvent(m->copy_stream.p, m->ev_export.p, 0));
    for (int k = 0; k < 9; k++)
        if (host_layers[k])
            GEM_CUDA(m, cudaMemcpyAsync(host_layers[k], m->d_out + (size_t)k * m->nc, m->nc * 4, cudaMemcpyDeviceToHost, m->copy_stream.p));
    GEM_CUDA(m, cudaEventRecord(m->ev_export_done.p, m->copy_stream.p));
    return GEM_OK;
}
int gem_export_layers_end(gem_map *m)
{
    if (!m) return GEM_ERR_INVALID;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    if (m->ev_export_done.p) GEM_CUDA(m, cudaEventSynchronize(m->ev_export_done.p));
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
    const GridCloudSrc snap = grid_cells(m, GEM_GRID_SNAPSHOT);
    HarvestSrc src;
    src.s = snap.s;
    src.f = snap.f;
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
    Lock lk(m->mu);
    SetDev sd(m->dev);
    GridCloudSrc src;
    int rc = grid_source(m, source, "gem_export_grid_cloud", &src);
    if (rc) return rc;
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
    Lock lk(m->mu);
    SetDev sd(m->dev);
    GridCloudSrc g;
    int rc = grid_source(m, source, "gem_grid_cloud_split", &g);
    if (rc) return rc;
    const int L = m->L;
    SplitScratch &s = m->split;
    const char *what = "gem_grid_cloud_split";
    const size_t fn = m->nc * sizeof(float), fl = (size_t)L * sizeof(float);
    if ((rc = scratch_grow(m, s.zg, fn, what, m->stream)) || (rc = scratch_grow(m, s.xg, fl, what, m->stream)) ||
        (rc = scratch_grow(m, s.yg, fl, what, m->stream)) || (rc = scratch_grow(m, s.dcell, fn, what, m->stream)) ||
        (rc = scratch_grow(m, s.dist, fn, what, m->stream)) || (rc = scratch_grow(m, s.queue, m->nc * sizeof(int), what, m->stream)) ||
        (rc = scratch_grow(m, s.ctr, 2 * sizeof(int), what, m->stream)) || (rc = scratch_grow(m, s.stats, sizeof(SplitStats), what, m->stream)))
        return rc;
    float *zg = s.zg.as<float>(), *xg = s.xg.as<float>(), *yg = s.yg.as<float>(), *dcell = s.dcell.as<float>(), *dist = s.dist.as<float>();
    int *queue = s.queue.as<int>(), *ctr = s.ctr.as<int>();
    GEM_CUDA(m, cudaMemsetAsync(ctr, 0, 2 * sizeof(int), m->stream));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_split_stage<<<blocks_for(m->nc, 256), 256, 0, m->stream>>>(g, zg, xg, yg, dcell));
    const int nt = (L + SPLIT_TILE - 1) / SPLIT_TILE;
    const dim3 grid(nt, nt);
    const int K = mean_k + 1;
    // the queue's length stays on the device: k_split_knn_far's fixed grid strides over it
#define GEM_SPLIT_KNN(KC)                                                                                                              \
    do {                                                                                                                               \
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_split_knn<KC><<<grid, SPLIT_TILE * SPLIT_TILE, 0, m->stream>>>(zg, xg, yg, L, g.f.sx, g.f.sy, mean_k, dcell, queue, ctr)); \
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_split_knn_far<KC><<<NUM_SMS * 4, 128, 0, m->stream>>>(zg, xg, yg, L, g.f.sx, g.f.sy, mean_k, dcell, queue, ctr)); \
    } while (0)
    if (K <= 8) GEM_SPLIT_KNN(8);
    else if (K <= 24) GEM_SPLIT_KNN(24);
    else GEM_SPLIT_KNN(SPLIT_MAX_K + 1);
#undef GEM_SPLIT_KNN
    GEM_CUDA(m, cudaGetLastError());
    // distances in cloud order -> statistics -> road -> obstacle, all on the stream; the three counts are copied beside
    // the statistics on the device, and the call waits once, for the one small read-back
    SplitStats *dst = s.stats.as<SplitStats>();
    int *d_total = nullptr;
    SplitDistSrc ds{g, dcell, dist, mean_distance_device, distance_capacity};
    if ((rc = compact_cells_issue(m, ds, (int)m->nc, &d_total))) return rc;
    GEM_CUDA(m, cudaMemcpyAsync(&dst->points, d_total, sizeof(int), cudaMemcpyDeviceToDevice, m->stream));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_split_stats<<<1, 32, 0, m->stream>>>(dist, &dst->points, ctr, mean_k, stddev_mul, dst,
                                                                         mean_distance_device, distance_capacity));
    GEM_CUDA(m, cudaGetLastError());
    SplitSrc rs{g, dcell, dst, travers_threshold, 1};
    rs.g.out = reinterpret_cast<float4 *>(road_points32_device);
    if ((rc = compact_cells_issue(m, rs, (int)std::min<size_t>((size_t)road_capacity, m->nc), &d_total))) return rc;
    GEM_CUDA(m, cudaMemcpyAsync(&dst->road, d_total, sizeof(int), cudaMemcpyDeviceToDevice, m->stream));
    SplitSrc os{g, dcell, dst, travers_threshold, 0};
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
        S.res = resolution;
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
    const char *what = "gem_color_octree";
    if ((rc = key_runs_grow(m, S.kr, n, 0, what)) || (rc = scratch_grow(m, S.leaf, N * 8, what, st)) ||
        (rc = scratch_grow(m, S.level, N * 4, what, st)) || (rc = scratch_grow(m, S.ghead, N * 4, what, st)) ||
        (rc = scratch_grow(m, S.gid, N * 4, what, st)) || (rc = scratch_grow(m, S.val, N * 4, what, st)) ||
        (rc = scratch_grow(m, S.groups, (N / 8 + 1) * sizeof(OctGroup), what, st)) || (rc = scratch_grow(m, S.ctr, sizeof(OctCounters), what, st)))
        return rc;
    const float4 *pts = static_cast<const float4 *>(points32_device);
    OctCounters *ctr = S.ctr.as<OctCounters>();
    u64 *leaf = S.leaf.as<u64>();
    int *cnt = S.kr.cnt.as<int>(), *off = S.kr.off.as<int>(), *level = S.level.as<int>(), *sidx = S.kr.idx[1].as<int>();
    uint32_t *val = S.val.as<uint32_t>();
    GEM_CUDA(m, cudaMemsetAsync(ctr, 0, sizeof(OctCounters), st));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_oct_keys<<<blocks_for(N, 256, 1 << 30), 256, 0, st>>>(pts, n, rf, S.kr.key[0].as<u64>(), S.kr.idx[0].as<int>(), ctr));
    GEM_CUDA(m, cudaGetLastError());
    if ((rc = key_runs_enqueue(m, S.kr, n, 49, leaf, &ctr->nruns))) return rc;
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
        if ((rc = scratch_grow(m, S.key2[0], ngp * 8, what, st)) || (rc = scratch_grow(m, S.key2[1], ngp * 8, what, st)) ||
            (rc = scratch_grow(m, S.nkey[0], nnode * 8, what, st)) || (rc = scratch_grow(m, S.nkey[1], nnode * 8, what, st)) ||
            (rc = scratch_grow(m, S.nrec[0], nnode * 8, what, st)) || (rc = scratch_grow(m, S.nrec[1], nnode * 8, what, st)) ||
            (rc = scratch_grow(m, S.dense, (size_t)hc.dense * 4, what, st)) || (rc = scratch_grow(m, S.kr.temp, std::max(t_keys, t_nodes), what, st)))
            return rc;
        size_t tcap = S.kr.temp.cap;
        u64 *nkey = S.nkey[0].as<u64>(), *nrec = S.nrec[0].as<u64>();
        GEM_CUDA(m, cudaMemsetAsync(nkey, 0xFF, nnode * 8, st)); // OCT_EMPTY: unused group slots sort last
        if (ngp) {
            GEM_CUDA(m, cudaMemsetAsync(S.dense.p, 0, (size_t)hc.dense * 4, st));
            GEM_LAUNCH(m, GEM_PROF_OTHER, k_oct_group_keys<<<blocks_for((size_t)nleaf, 256, 1 << 30), 256, 0, st>>>(leaf, nleaf, cnt, off, sidx, level, S.ghead.as<int>(),
                                                                                                                    S.gid.as<int>(), S.key2[0].as<u64>(), ctr));
            GEM_CUDA(m, cub::DeviceRadixSort::SortKeys(S.kr.temp.p, tcap, S.key2[0].as<u64>(), S.key2[1].as<u64>(), (int)ngp, 0, 32 + gbits, st));
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
        GEM_CUDA(m, cub::DeviceRadixSort::SortPairs(S.kr.temp.p, tcap, nkey, S.nkey[1].as<u64>(), nrec, S.nrec[1].as<u64>(), (int)nnode, 0, 53, st));
        GEM_CUDA(m, cudaMemcpyAsync(&hc, ctr, sizeof hc, cudaMemcpyDeviceToHost, st));
        GEM_CUDA(m, cudaStreamSynchronize(st));
    }
    r.nodes = hc.upper + hc.indep + hc.group_nodes;
    r.leaves = hc.indep + hc.group_leaves;
    r.bytes = 8ll * r.nodes;
    r.inserted = hc.inserted;
    r.skipped = n - hc.inserted;
    S.bytes = r.bytes;
    S.res = resolution;
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
// the last-writer scatter of both mark calls (pass 1, pass 2), then the marks back to the host
extern "C++" {
template <class Src> static int cost_mark(gem_map *m, const Src &src, long long nchunks, const gem_costmap_window *w, unsigned char *cost,
                                         gem_costmap_marks *out)
{
    const int ncells = w->size_x * w->size_y;
    int rc;
    if ((rc = scratch_grow(m, m->cost_scratch, (size_t)ncells * sizeof(int), "costmap scratch", m->stream))) return rc;
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
    Lock lk(m->mu);
    SetDev sd(m->dev);
    CostGridSrc src;
    const int rc = grid_source(m, source, "gem_costmap_mark_map", &src.g);
    if (rc) return rc;
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

// ---- the plugins fed from their subscribed messages (gem_gridmsg.h G1-G4; f18) -----------------------------------------
int gem_grid_map_msg_parse(const void *msg, unsigned long long bytes, const char *layer, gem_grid_map_layer *out)
{
    const char *why = gem_gridmsg::parse(msg, bytes, layer, out);
    return why ? fail(nullptr, GEM_ERR_INVALID, std::string("gem_grid_map_msg_parse: ") + why) : GEM_OK;
}

int gem_costmap_mark_grid(gem_map *m, const gem_grid_map_layer *g, const void *layer_device, const gem_costmap_window *w,
                          double travers_thresh, int mark_unknown, unsigned char *cost_device, gem_costmap_marks *out)
{
    if (!m || !g || !cost_device || !out || (g->floats > 0 && !layer_device))
        return fail(m, GEM_ERR_INVALID, "gem_costmap_mark_grid: bad argument");
    if (!cost_window_ok(w)) return fail(m, GEM_ERR_INVALID, "gem_costmap_mark_grid: bad window");
    if (!gem_gridmsg::layer_ok(*g)) return fail(m, GEM_ERR_INVALID, "gem_costmap_mark_grid: bad layer descriptor");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    CostMsgSrc src;
    src.p = static_cast<const unsigned char *>(layer_device);
    src.aligned = ((uintptr_t)layer_device & 3u) == 0;
    src.sx = g->size_x;
    src.sy = g->size_y;
    src.n = (int)g->floats;
    // G4: the start index wrapped into [0, size) once, here; the positions' constant part in double as grid_map adds it
    src.startx = g->size_x ? (int)(((long long)g->start_x % g->size_x + g->size_x) % g->size_x) : 0;
    src.starty = g->size_y ? (int)(((long long)g->start_y % g->size_y + g->size_y) % g->size_y) : 0;
    src.ox = g->position_x + (0.5 * g->length_x - 0.5 * g->resolution);
    src.oy = g->position_y + (0.5 * g->length_y - 0.5 * g->resolution);
    src.res = g->resolution;
    src.thresh = travers_thresh;
    src.mark_unknown = mark_unknown ? 1 : 0;
    return cost_mark(m, src, ((long long)src.n + 31) / 32, w, cost_device, out);
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
    if ((rc = scratch_grow(m, m->cost_scratch, ncells, "costmap scratch", m->stream))) return rc;
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

// InflationLayer::updateCosts (gem_inflate.cuh, DESIGN.md f14).  The host builds I2's tables with its libm, the bins (the
// distinct table values <= r, in increasing order) and, per bin, the first bin that can push into it; one cooperative
// kernel then runs the whole brushfire on the stream.
int gem_costmap_inflate(gem_map *m, const gem_costmap_window *w, const gem_costmap_inflation *p, unsigned char *master_device,
                        int min_i, int min_j, int max_i, int max_j)
{
    if (!m || !p || !master_device) return fail(m, GEM_ERR_INVALID, "gem_costmap_inflate: bad argument");
    if (!cost_window_ok(w)) return fail(m, GEM_ERR_INVALID, "gem_costmap_inflate: bad window");
    if (!std::isfinite(p->inflation_radius) || p->inflation_radius < 0.0 || !std::isfinite(p->cost_scaling_factor) ||
        p->cost_scaling_factor < 0.0 || !std::isfinite(p->inscribed_radius) || p->inscribed_radius < 0.0)
        return fail(m, GEM_ERR_INVALID, "gem_costmap_inflate: the radius, weight and inscribed radius must be finite and >= 0");
    if (p->inflate_unknown != 0 && p->inflate_unknown != 1) return fail(m, GEM_ERR_INVALID, "gem_costmap_inflate: bad inflate_unknown");
    const int sx = w->size_x, sy = w->size_y;
    const double res = w->resolution;
    // I1, with the DEFINED cap
    const double cap = std::ceil(std::hypot((double)sx, (double)sy)) + 1.0;
    const long long r = (long long)std::min(std::max(0.0, std::ceil(p->inflation_radius / res)), cap);
    if (r == 0) return GEM_OK;
    // DEFINED: the host tables grow with r^2, so r is bounded (a 16.8 M-entry table; 204 m at 0.05 m, 819 m at 0.2 m)
    if (r > GEM_INFLATE_MAX_CELLS)
        return fail(m, GEM_ERR_INVALID, "gem_costmap_inflate: the radius exceeds GEM_INFLATE_MAX_CELLS cells");
    // I3: the widened rect, clamped
    const long long i0 = std::max(0ll, (long long)min_i - r), i1 = std::min((long long)sx, (long long)max_i + r);
    const long long j0 = std::max(0ll, (long long)min_j - r), j1 = std::min((long long)sy, (long long)max_j + r);
    if (i0 >= i1 || j0 >= j1) return GEM_OK; // no seed
    Lock lk(m->mu);
    SetDev sd(m->dev);
    InflScratch &S = m->infl;
    const int tw = (int)r + 2;
    const size_t T = (size_t)tw * tw;
    const bool same = S.r == r && S.res == res && S.weight == p->cost_scaling_factor && S.inscribed == p->inscribed_radius;
    std::vector<int> bin, lo;
    std::vector<unsigned char> cost;
    int nbins = S.nbins;
    if (!same) try {
        // I2: computeCaches
        std::vector<double> dist(T);
        cost.resize(T);
        for (int i = 0; i < tw; i++)
            for (int j = 0; j < tw; j++) {
                const double d = std::hypot((double)i, (double)j);
                dist[(size_t)i * tw + j] = d;
                unsigned char c;
                if (d == 0) c = COST_LETHAL;
                else if (d * res <= p->inscribed_radius) c = 253;
                else c = (unsigned char)(252 * std::exp(-1.0 * p->cost_scaling_factor * (d * res - p->inscribed_radius)));
                cost[(size_t)i * tw + j] = c;
            }
        std::map<double, int> bins;
        for (size_t t = 0; t < T; t++)
            if (!(dist[t] > (double)r)) bins.emplace(dist[t], 0);
        nbins = 0;
        for (auto &kv : bins) kv.second = nbins++;
        bin.assign(T, -1);
        for (size_t t = 0; t < T; t++)
            if (!(dist[t] > (double)r)) bin[t] = bins[dist[t]];
        // lo[q]: the smallest bin holding a table neighbour of a cell of bin q (a push changes one |offset| by one)
        lo.assign(nbins, INT32_MAX);
        for (int i = 0; i < tw; i++)
            for (int j = 0; j < tw; j++) {
                const int q = bin[(size_t)i * tw + j];
                if (q < 0) continue;
                const int nb[4][2] = {{i - 1, j}, {i + 1, j}, {i, j - 1}, {i, j + 1}};
                for (auto &n : nb) {
                    if (n[0] < 0 || n[1] < 0 || n[0] >= tw || n[1] >= tw) continue;
                    const int b = bin[(size_t)n[0] * tw + n[1]];
                    if (b == q) return fail(m, GEM_ERR_INVALID, "gem_costmap_inflate: the distance table pushes a cell into its own bin");
                    if (b >= 0 && b < lo[q]) lo[q] = b;
                }
            }
        for (int q = 0; q < nbins; q++) lo[q] = std::min(lo[q], q);
    } catch (const std::bad_alloc &) {
        return fail(m, GEM_ERR_NOMEM, "gem_costmap_inflate: host memory for the distance tables");
    }
    // scratch, all grown before anything is written
    const size_t ncells = (size_t)sx * sy;
    const size_t tab_bytes = T * sizeof(int) + ((T + 15) / 16) * 16 + (size_t)nbins * sizeof(int);
    if (!S.blocks) {
        int per_sm = 0, sms = 0;
        GEM_CUDA(m, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_inflate, INFL_BLOCK, 0));
        GEM_CUDA(m, cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, m->dev));
        S.blocks = std::max(1, std::min(per_sm, 4) * sms);
    }
    // A failed growth returns GEM_ERR_NOMEM, and a later call must still find consistent state: the tables are marked
    // stale before `tab` may be replaced, and a replaced key buffer stays marked until its clearing memset is enqueued.
    if (!same) S.r = -1;
    void *old_key = S.key.p;
    int rc = scratch_grow(m, S.key, ncells * 8, "gem_costmap_inflate", m->stream);
    if (S.key.p != old_key) S.key_dirty = true;
    if (rc || (rc = scratch_grow(m, S.pops, ncells * 8, "gem_costmap_inflate", m->stream)) ||
        (rc = scratch_grow(m, S.tab, tab_bytes, "gem_costmap_inflate", m->stream)) ||
        (rc = scratch_grow(m, S.gstart, ((size_t)nbins + 1) * sizeof(int), "gem_costmap_inflate", m->stream)) ||
        (rc = scratch_grow(m, S.blk, (size_t)S.blocks * sizeof(int), "gem_costmap_inflate", m->stream)))
        return rc;
    if (S.key_dirty) {
        GEM_CUDA(m, cudaMemsetAsync(S.key.p, 0xFF, S.key.cap, m->stream)); // every cell unseen
        S.key_dirty = false;
    }
    int *d_bin = S.tab.as<int>();
    unsigned char *d_cost = reinterpret_cast<unsigned char *>(d_bin + T);
    int *d_lo = reinterpret_cast<int *>(d_cost + ((T + 15) / 16) * 16);
    if (!same) {
        GEM_CUDA(m, cudaMemcpyAsync(d_bin, bin.data(), T * sizeof(int), cudaMemcpyHostToDevice, m->stream));
        GEM_CUDA(m, cudaMemcpyAsync(d_cost, cost.data(), T, cudaMemcpyHostToDevice, m->stream));
        GEM_CUDA(m, cudaMemcpyAsync(d_lo, lo.data(), (size_t)nbins * sizeof(int), cudaMemcpyHostToDevice, m->stream));
        // from pageable memory each copy returns once its source is staged, so the vectors may go when this call returns
        S.r = r;
        S.res = res;
        S.weight = p->cost_scaling_factor;
        S.inscribed = p->inscribed_radius;
        S.nbins = nbins;
    }
    GEM_CUDA(m, cudaMemsetAsync(S.gstart.p, 0, sizeof(int), m->stream));
    InflateArgs a{master_device, sx, sy, (int)i0, (int)j0, (int)(i1 - i0), (int)(j1 - j0), d_bin, d_cost, d_lo, tw, nbins,
                  p->inflate_unknown, S.key.as<unsigned long long>(), S.pops.as<int2>(), S.gstart.as<int>(), S.blk.as<int>()};
    void *args[] = {&a};
    GEM_LAUNCH(m, GEM_PROF_OTHER, GEM_CUDA(m, cudaLaunchCooperativeKernel((const void *)k_inflate, dim3((unsigned)S.blocks), dim3(INFL_BLOCK), args, 0, m->stream)));
    return GEM_OK;
}

// ---- the VoxelGrid pre-filter of GEM's demo launches (gem_voxel.cuh, DESIGN.md f9, f20) -------------------------------
static const char *vox_params_bad(const gem_voxel_grid_params *p)
{
    if (p->field < GEM_VOXEL_FIELD_NONE || p->field > GEM_VOXEL_FIELD_INTENSITY) return "bad field id";
    for (int a = 0; a < 3; a++) // V1
        if (!std::isfinite(p->leaf_size[a]) || !(p->leaf_size[a] > 0.0f)) return "every leaf size must be finite and positive";
    return nullptr;
}

static VoxParams vox_params(const gem_voxel_grid_params *p)
{
    VoxParams P{};
    for (int a = 0; a < 3; a++) P.inv[a] = 1.0f / p->leaf_size[a];
    P.field = p->field;
    P.lmin = p->limit_min;
    P.lmax = p->limit_max;
    P.flmin = (float)p->limit_min; // getMinMax3D takes the limits as floats
    P.flmax = (float)p->limit_max;
    P.negative = p->limit_negative ? 1 : 0;
    return P;
}

// the steps' scratch is sized for n points (with the pre-filter's two buffers when bufs)
static bool vox_fits(const gem_map *m, int n, bool bufs)
{
    const VoxScratch &S = m->vox;
    return S.acc.p && S.n >= n && (!bufs || S.buf[1].cap >= (size_t)n * 16);
}
// size it before anything is enqueued (a failed growth writes nothing)
static int vox_grow(gem_map *m, int n, bool bufs, const char *what)
{
    VoxScratch &S = m->vox;
    int rc;
    if ((rc = scratch_grow(m, S.acc, (size_t)4 * GEM_PREFILTER_MAX_STEPS * sizeof(VoxStep), what, m->stream))) return rc;
    if (bufs && ((rc = scratch_grow(m, S.buf[0], (size_t)n * 16, what, m->stream)) ||
                 (rc = scratch_grow(m, S.buf[1], (size_t)n * 16, what, m->stream))))
        return rc;
    if (S.n >= n) return GEM_OK;
    if ((rc = key_runs_grow(m, S.kr, n, 0, what))) return rc;
    S.n = n;
    return GEM_OK;
}

// the device state of ring slot `slot` (0..2), or gem_voxel_grid's (3)
static VoxStep *vox_steps(gem_map *m, int slot) { return m->vox.acc.as<VoxStep>() + (size_t)slot * GEM_PREFILTER_MAX_STEPS; }

// k > 0 steps on the handle's stream, no host read-back: step 0 reads n points of `in` (n > 0 host-known), step j > 0
// the count step j-1 left in st[j-1]; the steps alternate between the scratch buffers, the last one writes up to
// `capacity` points to `out`.  Every kernel and sort runs at n, the upper bound of every step's count.  vox_grow(n) first.
static int vox_chain_enqueue(gem_map *m, const gem_voxel_grid_params *steps, int k, const float4 *in, int n, float4 *out,
                             int capacity, VoxStep *st, bool wide_passes)
{
    using u64 = unsigned long long;
    VoxScratch &S = m->vox;
    cudaStream_t s = m->stream;
    const size_t N = (size_t)n;
    const unsigned blocks = (unsigned)((N + VOX_BLOCK - 1) / VOX_BLOCK);
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_vox_init<<<1, 32, 0, s>>>(st, k, n));
    const float4 *src = in;
    for (int j = 0; j < k; j++) {
        const VoxParams P = vox_params(&steps[j]);
        const int *nin = j == 0 ? &st[0].n : &st[j - 1].count;
        float4 *dst = j == k - 1 ? out : S.buf[j & 1].as<float4>();
        const int cap = j == k - 1 ? capacity : n;
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_vox_bounds<<<blocks_for(N, VOX_BLOCK, NUM_SMS * 8), VOX_BLOCK, 0, s>>>(src, n, nin, P, &st[j].acc));
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_vox_decide<<<1, 1, 0, s>>>(P, n, nin, &st[j], wide_passes ? 1 : 0));
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_vox_keys<<<blocks, VOX_BLOCK, 0, s>>>(src, n, nin, P, &st[j], S.kr.key[0].as<u64>(), S.kr.idx[0].as<int>()));
        GEM_CUDA(m, cudaGetLastError());
        // V7: the stable sort keeps each voxel's points in input order; every key fits GEM_VOX_KEY_BITS (gem_voxgrid.h)
        int rc = key_runs_enqueue(m, S.kr, n, GEM_VOX_KEY_BITS, S.kr.key[0].as<u64>(), &st[j].acc.nruns);
        if (rc) return rc;
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_vox_centroids<<<blocks, VOX_BLOCK, 0, s>>>(src, S.kr.idx[1].as<int>(), S.kr.cnt.as<int>(),
                                                                                  S.kr.off.as<int>(), &st[j], dst, cap));
        GEM_CUDA(m, cudaGetLastError());
        src = dst;
    }
    return GEM_OK;
}

static gem_voxel_grid_info vox_info(const VoxStep &h)
{
    gem_voxel_grid_info r{};
    r.count = h.count;
    r.used = h.acc.used;
    r.passthrough = h.mode == GEM_VOX_PASS ? 1 : 0;
    return r;
}

int gem_voxel_grid(gem_map *m, const void *xyzi_device, int n, const gem_voxel_grid_params *p, void *out_xyzi_device, int capacity,
                   gem_voxel_grid_info *info)
{
    if (!m || !p || !info || n < 0 || (n > 0 && !xyzi_device) || capacity < 0 || (capacity > 0 && !out_xyzi_device))
        return fail(m, GEM_ERR_INVALID, "gem_voxel_grid: bad argument");
    if (const char *why = vox_params_bad(p)) return fail(m, GEM_ERR_INVALID, std::string("gem_voxel_grid: ") + why);
    // V9: input and output ranges may not overlap (chained calls alternate between two buffers)
    if (ranges_meet(xyzi_device, (size_t)n * sizeof(float4), out_xyzi_device, (size_t)capacity * sizeof(float4)))
        return fail(m, GEM_ERR_INVALID, "gem_voxel_grid: the input and output ranges overlap");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    if (n == 0) { // V5
        *info = gem_voxel_grid_info{};
        return GEM_OK;
    }
    int rc;
    if ((rc = vox_grow(m, n, false, "gem_voxel_grid"))) return rc;
    VoxStep *st = vox_steps(m, 3);
    if ((rc = vox_chain_enqueue(m, p, 1, static_cast<const float4 *>(xyzi_device), n, static_cast<float4 *>(out_xyzi_device),
                                capacity, st, false)))
        return rc;
    // the one synchronisation: the step's decision and counts
    VoxStep h{};
    GEM_CUDA(m, cudaMemcpyAsync(&h, st, sizeof h, cudaMemcpyDeviceToHost, m->stream));
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    if (h.mode == GEM_VOX_WIDE) return fail(m, GEM_ERR_INVALID, "gem_voxel_grid: the bounds times 1 / leaf are not finite (no voxel index)");
    *info = vox_info(h);
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
    if (ranges_meet(points32_device, (size_t)n * 32, out_points32_device, (size_t)capacity * 32))
        return fail(m, GEM_ERR_INVALID, "gem_mls_upsample: the input and output ranges overlap");
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
    size_t t_scan64 = 0;
    GEM_CUDA(m, cub::DeviceScan::ExclusiveSum(nullptr, t_scan64, (long long *)nullptr, (long long *)nullptr, n, st));
    const char *what = "gem_mls_upsample";
    int rc;
    if ((rc = key_runs_grow(m, S.kr, n, t_scan64, what)) || (rc = scratch_grow(m, S.spts, N * 16, what, st)) ||
        (rc = scratch_grow(m, S.ukey, N * 8, what, st)) || (rc = scratch_grow(m, S.nbr, N * 4, what, st)) ||
        (rc = scratch_grow(m, S.ocnt, N * 8, what, st)) || (rc = scratch_grow(m, S.ooff, N * 8, what, st)) ||
        (rc = scratch_grow(m, S.longs, N * 4, what, st)) || (rc = scratch_grow(m, S.acc, sizeof(MlsAcc), what, st)))
        return rc;
    const float4 *in = static_cast<const float4 *>(points32_device);
    float4 *out = static_cast<float4 *>(out_points32_device);
    MlsAcc *acc = S.acc.as<MlsAcc>();
    u64 *ukey = S.ukey.as<u64>();
    int *idx1 = S.kr.idx[1].as<int>(), *ucnt = S.kr.cnt.as<int>(), *uoff = S.kr.off.as<int>();
    int *nbr = S.nbr.as<int>(), *longs = S.longs.as<int>();
    long long *ocnt = S.ocnt.as<long long>(), *ooff = S.ooff.as<long long>();
    float4 *spts = S.spts.as<float4>();
    MlsAcc h{};
    h.mn[0] = h.mn[1] = h.mn[2] = 0xffffffffu;
    GEM_CUDA(m, cudaMemcpyAsync(acc, &h, sizeof h, cudaMemcpyHostToDevice, st));
    const unsigned gb = (unsigned)((N + VOX_BLOCK - 1) / VOX_BLOCK), gq = (unsigned)((N + MLS_WARPS - 1) / MLS_WARPS);
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_mls_bounds<<<blocks_for(N, VOX_BLOCK, NUM_SMS * 8), VOX_BLOCK, 0, st>>>(in, n, acc));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_mls_keys<<<gb, VOX_BLOCK, 0, st>>>(in, n, P, acc, S.kr.key[0].as<u64>(), S.kr.idx[0].as<int>()));
    GEM_CUDA(m, cudaGetLastError());
    if ((rc = key_runs_enqueue(m, S.kr, n, 64, ukey, &acc->nruns))) return rc;
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_mls_stage<<<gb, VOX_BLOCK, 0, st>>>(in, n, idx1, spts));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_mls_count<<<gq, MLS_BLOCK, 0, st>>>(in, n, P, acc, spts, ukey, uoff, ucnt, nbr, ocnt, longs));
    GEM_CUDA(m, cudaGetLastError());
    size_t tcap = S.kr.temp.cap;
    GEM_CUDA(m, cub::DeviceScan::ExclusiveSum(S.kr.temp.p, tcap, ocnt, ooff, n, st));
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
        if ((rc = scratch_grow(m, S.lkeys, w * per, what, st))) return rc;
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
    LocalStore t;
    cudaError_t e = cudaMalloc(&t.buf.p, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(m, GEM_ERR_NOMEM, std::string("local map: cudaMalloc: ") + cudaGetErrorString(e));
    }
    t.buf.cap = bytes;
    t.log = t.buf.as<float4>();
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
    if (e != cudaSuccess) return fail(m, GEM_ERR_CUDA, std::string("local map: growth: ") + cudaGetErrorString(e));
    s = std::move(t);
    return GEM_OK;
}

// forget every record: the index back to all-free slots
static int local_reset(gem_map *m)
{
    LocalStore &s = m->local;
    s.n = 0;
    if (!s.buf.p) return GEM_OK;
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
    if (m->pf_count && m->pf_call == m->call_no) { // a pre-filtered add: its counters and its filtered count
        int rc = read_counters(m, 0, false);
        if (rc) return rc;
        int c = 0;
        GEM_CUDA(m, cudaMemcpyAsync(&c, m->pf_count, sizeof c, cudaMemcpyDeviceToHost, m->stream));
        GEM_CUDA(m, cudaStreamSynchronize(m->stream));
        m->stats.points_in = c;
        m->pf_count = nullptr;
    } else if (m->stats.points_in > 0 && m->stats.cells_touched == 0 && m->stats.points_binned == 0) {
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
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    for (auto &sp : m->spans) {
        float ms = 0.0f;
        if (cudaEventElapsedTime(&ms, sp.e0.p, sp.e1.p) == cudaSuccess) {
            m->prof_ms[sp.cls] += ms;
            m->prof_count[sp.cls]++;
        }
        m->free_events.push_back(std::move(sp.e0));
        m->free_events.push_back(std::move(sp.e1));
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
    const int rc = scratch_grow(m, m->divtest, 16, "gem_selftest_division", m->stream);
    if (rc) return rc;
    unsigned long long *d = m->divtest.as<unsigned long long>();
    GEM_CUDA(m, cudaMemsetAsync(d, 0, 16, m->stream));
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_div_selftest<<<NUM_SMS * 8, 256, 0, m->stream>>>(seed, (size_t)n, d, d + 1));
    unsigned long long h[2] = {0, 0};
    GEM_CUDA(m, cudaMemcpyAsync(h, d, 16, cudaMemcpyDeviceToHost, m->stream));
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    *mismatches_out = h[0];
    if (fast_out) *fast_out = h[1];
    return GEM_OK;
}

int gem_host_alloc(void **out, unsigned long long bytes)
{
    if (!out) return GEM_ERR_INVALID;
    if (cudaHostAlloc(out, (size_t)bytes, cudaHostAllocDefault) == cudaSuccess) return GEM_OK;
    cudaGetLastError(); // as in dev_alloc
    return GEM_ERR_NOMEM;
}
int gem_host_free(void *p) { return cudaFreeHost(p) == cudaSuccess ? GEM_OK : GEM_ERR_CUDA; }

// ---- multi-GPU routing -----------------------------------------------------------------------
int gem_route_points(gem_map *m, const void *xyzi, const void *rgba, int n, const gem_frame *frame, int tiles_r,
                     int tiles_c, void *rec_out, int *counts_out, int bucket_stride)
{
    if (!m || !frame || n < 0 || tiles_r < 1 || tiles_c < 1 || !rec_out || !counts_out || (n > 0 && !xyzi) || !sensor_ok(frame->sensor))
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

int gem_fuse_records(gem_map *m, const void *rec, int n)
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
        const FoldSrc fs{(const char *)in.rec + 16, (int)sizeof(RouteRec)};
        const FrameParams none{};
        if ((rc = enqueue_add<SRC_RECORDS>(m, in, fs, cn, none, nullptr, nullptr, false, true, true))) return rc;
        if (n > m->P && (rc = read_counters(m, cn, true))) return rc;
    }
    if (n <= m->P) m->stats.points_in = n;
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

// One pair's scratch, laid out in one buffer for clouds of at most nn and no records: two hash tables (keys + first index),
// the keep flags, the scan counts of the compaction, its output and four counters.
struct PairScratch {
    unsigned long long *kn, *ko;
    int *fn, *fo, *cnt, *ctr;
    unsigned char *keepn, *keepo;
    SubPoint *out;
    size_t cn, co, nchunk;
};
static size_t hash_slots(int n) { size_t p = 64; while (p < 2 * (size_t)n + 2) p <<= 1; return p; }
static PairScratch pair_layout(void *base, int nn, int no, size_t *bytes = nullptr)
{
    PairScratch s;
    const int big = std::max(nn, no);
    s.cn = hash_slots(nn);
    s.co = hash_slots(no);
    s.nchunk = ((size_t)big + 31) / 32 + 1;
    const size_t nseg = s.nchunk / SCAN_SEG + 1;
    char *p = (char *)base;
    size_t at = 0;
    auto take = [&](size_t n) { char *q = p + at; at = (at + n + 31) & ~(size_t)31; return q; };
    s.out = (SubPoint *)take((size_t)big * sizeof(SubPoint));
    s.kn = (unsigned long long *)take((s.cn + s.co) * 8);
    s.ko = s.kn + s.cn;
    s.fn = (int *)take((s.cn + s.co) * 4);
    s.fo = s.fn + s.cn;
    s.cnt = (int *)take((s.nchunk + nseg) * 4);
    s.ctr = (int *)take(16);
    s.keepn = (unsigned char *)take((size_t)nn + no);
    s.keepo = s.keepn + nn;
    if (bytes) *bytes = at;
    return s;
}
static size_t pair_bytes(int nn, int no)
{
    size_t b = 0;
    pair_layout(nullptr, nn, no, &b);
    return b;
}

// compact p[0, *n) by its keep flags, in order and in place (through s.out); ub >= *n is known on the host
static cudaError_t enqueue_compact(cudaStream_t st, const PairScratch &s, SubPoint *p, unsigned char *keep, int ub, int *n, int &launches)
{
    if (ub == 0) return cudaSuccess;
    const int nchunk = (ub + 31) / 32, nseg = (nchunk + SCAN_SEG - 1) / SCAN_SEG, nb = (ub + TAKE_BLOCK - 1) / TAKE_BLOCK;
    int *segtot = s.cnt + s.nchunk;
    k_keep_count<<<nb, TAKE_BLOCK, 0, st>>>(keep, n, ub, s.cnt);
    k_compact_scan<<<nseg, SCAN_SEG, 0, st>>>(s.cnt, nchunk, segtot);
    k_keep_write<<<nb, TAKE_BLOCK, 0, st>>>(p, keep, ub, s.cnt, segtot, nseg, SCAN_SEG, s.out, n);
    launches += 3;
    return cudaMemcpyAsync(p, s.out, (size_t)ub * sizeof(SubPoint), cudaMemcpyDeviceToDevice, st);
}

// One pass of :847-883 for the pair (new = pn, old = po), enqueued on `st` with no allocation and no host synchronisation:
// the counts *nn / *no stay in device memory and come back updated, ubn / ubo are host-known upper bounds on them (the
// tables, flags and grids are sized from those), fused cells are added to *fused.  s = pair_layout for (ubn, ubo) or more.
static cudaError_t enqueue_pair(cudaStream_t st, const PairScratch &s, SubPoint *pn, int ubn, int *nn, SubPoint *po, int ubo, int *no,
                                double res, int compat, int *fused, int &launches)
{
    cudaError_t e = cudaMemsetAsync(s.kn, 0xff, (s.cn + s.co) * 8, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(s.fn, 0x7f, (s.cn + s.co) * 4, st);
    if (e != cudaSuccess) return e;
    const unsigned mn = (unsigned)(s.cn - 1), mo = (unsigned)(s.co - 1);
    if (ubn) k_hash_insert<<<blocks_for((size_t)ubn, 256, 1 << 30), 256, 0, st>>>(pn, nn, res, s.kn, s.fn, mn);
    if (ubo) k_hash_insert<<<blocks_for((size_t)ubo, 256, 1 << 30), 256, 0, st>>>(po, no, res, s.ko, s.fo, mo);
    if (ubo) k_refuse_keep<<<blocks_for((size_t)ubo, 256, 1 << 30), 256, 0, st>>>(po, no, res, s.ko, s.fo, mo, s.keepo);
    if (ubn) k_refuse_pair<<<blocks_for((size_t)ubn, 256, 1 << 30), 256, 0, st>>>(pn, nn, po, res, s.kn, s.fn, mn, s.ko, s.fo, mo, s.keepn, compat, fused);
    launches += (ubn ? 2 : 0) + (ubo ? 2 : 0);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if ((e = enqueue_compact(st, s, pn, s.keepn, ubn, nn, launches)) != cudaSuccess) return e;
    if ((e = enqueue_compact(st, s, po, s.keepo, ubo, no, launches)) != cudaSuccess) return e;
    return cudaGetLastError();
}

int gem_refuse_submaps(gem_map *m, void *new_points32, int *n_new, void *old_points32, int *n_old, double resolution, int compat,
                       int *fused_out)
{
    if (!m || !n_new || !n_old || *n_new < 0 || *n_old < 0 || (*n_new > 0 && !new_points32) || (*n_old > 0 && !old_points32) || !(resolution > 0.0))
        return fail(m, GEM_ERR_INVALID, "gem_refuse_submaps: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    const int nn = *n_new, no = *n_old;
    int rc = scratch_grow(m, m->refuse, pair_bytes(nn, no), "gem_refuse_submaps", m->stream);
    if (rc) return rc;
    const PairScratch s = pair_layout(m->refuse.p, nn, no);
    int h[4] = {0, nn, no, 0}; // fused, n_new, n_old
    int launches = 0;
    cudaError_t e = cudaMemcpyAsync(s.ctr, h, 16, cudaMemcpyHostToDevice, m->stream);
    if (e == cudaSuccess)
        e = enqueue_pair(m->stream, s, (SubPoint *)new_points32, nn, s.ctr + 1, (SubPoint *)old_points32, no, s.ctr + 2, resolution, compat,
                         s.ctr, launches);
    m->launches += launches;
    if (e == cudaSuccess) e = cudaMemcpyAsync(h, s.ctr, 16, cudaMemcpyDeviceToHost, m->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(m->stream);
    if (e != cudaSuccess) return fail(m, GEM_ERR_CUDA, std::string("gem_refuse_submaps: ") + cudaGetErrorString(e));
    *n_new = h[1];
    *n_old = h[2];
    if (fused_out) *fused_out = h[0];
    return GEM_OK;
}

// ---- the global map: keyframe submap stack, poses and updateGlobalMap (DESIGN.md f16) ----------------------------------
using GLock = std::lock_guard<std::mutex>;

// the stack's stream and event, created on first use (caller holds g.mu)
static int gmap_ready(gem_map *m)
{
    GlobalStore &g = m->gmap;
    if (!g.stream.p) GEM_CUDA(m, cudaStreamCreateWithFlags(&g.stream.p, cudaStreamNonBlocking));
    if (!g.ev.p) GEM_CUDA(m, cudaEventCreateWithFlags(&g.ev.p, cudaEventDisableTiming));
    return GEM_OK;
}
// room for `need` records in both arena buffers (capacity doubles from 1024).  Both are allocated before anything is
// released, so a failed growth leaves the stack as it was.
static int gmap_reserve_records(gem_map *m, long long need)
{
    GlobalStore &g = m->gmap;
    if (need <= g.cap) return GEM_OK;
    long long cap = g.cap > 0 ? g.cap : 1024;
    while (cap < need) cap *= 2;
    if (cap > (1 << 30)) return fail(m, GEM_ERR_NOMEM, "global map: more than 2^30 records");
    DevBuf q[2];
    for (int b = 0; b < 2; b++) {
        const cudaError_t e = cudaMalloc(&q[b].p, (size_t)cap * sizeof(SubPoint));
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(m, GEM_ERR_NOMEM, std::string("global map: cudaMalloc: ") + cudaGetErrorString(e));
        }
        q[b].cap = (size_t)cap * sizeof(SubPoint);
    }
    const int total = g.off.back();
    cudaError_t e = total ? cudaMemcpyAsync(q[0].p, g.arena[g.cur].p, (size_t)total * sizeof(SubPoint), cudaMemcpyDeviceToDevice, g.stream.p)
                          : cudaSuccess;
    if (e == cudaSuccess) e = cudaStreamSynchronize(g.stream.p);
    if (e != cudaSuccess) return fail(m, GEM_ERR_CUDA, std::string("global map: growth: ") + cudaGetErrorString(e));
    for (int b = 0; b < 2; b++) g.arena[b] = std::move(q[b]);
    g.cur = 0;
    g.cap = cap;
    return GEM_OK;
}
// the update's device bookkeeping for K submaps: counts [K], old offsets [K + 1], new offsets [K + 1], counters [4],
// then the re-pose table Rigid [K]
static size_t gmap_meta_ints(int K) { return ((3 * (size_t)K + 6) + 3) & ~(size_t)3; }
static int gmap_reserve_meta(gem_map *m, int K)
{
    GlobalStore &g = m->gmap;
    if (K <= g.meta_submaps) return GEM_OK;
    int cap = std::max(g.meta_submaps * 2, 64);
    while (cap < K) cap *= 2;
    const int rc = scratch_grow(m, g.meta, gmap_meta_ints(cap) * 4 + (size_t)cap * sizeof(Rigid), "global map", g.stream.p);
    if (rc == GEM_OK) g.meta_submaps = cap;
    return rc;
}

int gem_global_map_reset(gem_map *m)
{
    if (!m) return GEM_ERR_INVALID;
    GlobalStore &g = m->gmap;
    GLock lk(g.mu);
    g.cnt.clear();
    g.off.assign(1, 0);
    g.poses.assign({1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1});
    g.centres.assign({0.0f, 0.0f});
    return GEM_OK;
}

int gem_global_map_reserve(gem_map *m, long long records, int submaps)
{
    if (!m || records < 0 || submaps < 0) return fail(m, GEM_ERR_INVALID, "gem_global_map_reserve: bad argument");
    if (records > (1 << 30)) return fail(m, GEM_ERR_NOMEM, "gem_global_map_reserve: more than 2^30 records");
    GlobalStore &g = m->gmap;
    GLock lk(g.mu);
    SetDev sd(m->dev);
    int rc;
    if ((rc = gmap_ready(m)) || (rc = gmap_reserve_records(m, records)) || (rc = gmap_reserve_meta(m, submaps))) return rc;
    // one pair of the largest submaps the arena can hold
    const int big = (int)std::min<long long>(records, g.cap);
    return scratch_grow(m, g.pair, pair_bytes(big, big), "gem_global_map_reserve", g.stream.p);
}

int gem_global_map_push(gem_map *m, const void *records_device, int n, const float pose[16])
{
    if (!m || n < 0 || !pose || (n > 0 && !records_device)) return fail(m, GEM_ERR_INVALID, "gem_global_map_push: bad argument");
    SetDev sd(m->dev);
    if (n > 0) {
        cudaPointerAttributes a{};
        if (cudaPointerGetAttributes(&a, records_device) != cudaSuccess || (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged)) {
            cudaGetLastError();
            return fail(m, GEM_ERR_INVALID, "gem_global_map_push: the records are not in device memory");
        }
    }
    GlobalStore &g = m->gmap;
    GLock lk(g.mu);
    int rc;
    const long long total = g.off.back();
    if ((rc = gmap_ready(m)) || (rc = gmap_reserve_records(m, total + n))) return rc;
    { // a cut_submap issued just before on the handle's stream is complete before the copy reads it
        Lock hl(m->mu);
        GEM_CUDA(m, cudaEventRecord(g.ev.p, m->stream));
    }
    GEM_CUDA(m, cudaStreamWaitEvent(g.stream.p, g.ev.p, 0));
    if (n) GEM_CUDA(m, cudaMemcpyAsync(g.arena[g.cur].as<SubPoint>() + total, records_device, (size_t)n * sizeof(SubPoint),
                                       cudaMemcpyDeviceToDevice, g.stream.p));
    GEM_CUDA(m, cudaStreamSynchronize(g.stream.p));
    // :636-642, then :660: the keyframe (pose, centre = its translation x, y) first, then its submap
    g.poses.insert(g.poses.end(), pose, pose + 16);
    g.centres.push_back(pose[3]);
    g.centres.push_back(pose[7]);
    g.cnt.push_back(n);
    g.off.push_back((int)(total + n));
    return GEM_OK;
}

int gem_global_map_update(gem_map *m, const float *opt_poses, int k, double resolution, double radius, int compat, int *fused_out)
{
    if (!m || k < 0 || (k > 0 && !opt_poses) || !(resolution > 0.0) || !std::isfinite(resolution) || !(radius >= 0.0))
        return fail(m, GEM_ERR_INVALID, "gem_global_map_update: bad argument");
    GlobalStore &g = m->gmap;
    GLock lk(g.mu);
    SetDev sd(m->dev);
    int rc;
    if ((rc = gmap_ready(m))) return rc;
    const int K = (int)g.cnt.size(), Kp = std::min(k, K); // :784-786
    // :791-809 on the host: the re-pose of submaps 1 .. K'-1 (submap 0 keeps its pose)
    std::vector<Rigid> T((size_t)std::max(Kp, 1));
    for (int i = 1; i < Kp; i++) {
        float t[16];
        gem_gmap::relative_pose(opt_poses + 16 * (size_t)i, &g.poses[16 * (size_t)i], t);
        for (int q = 0; q < 12; q++) T[i].t[q] = t[q];
    }
    // :812-891's pairs from the pushed centres (localMapLoc_ is never updated)
    std::vector<std::pair<int, int>> pairs;
    gem_gmap::pair_schedule(g.centres.data(), Kp, radius, pairs);
    int big = 0;
    for (int i = 0; i < Kp; i++) big = std::max(big, g.cnt[i]);
    if ((rc = gmap_reserve_meta(m, std::max(K, 1))) || (rc = scratch_grow(m, g.pair, pair_bytes(big, big), "gem_global_map_update", g.stream.p))) return rc;
    int *d_cnt = g.meta.as<int>(), *d_off = d_cnt + K, *d_off_new = d_off + K + 1, *d_ctr = d_off_new + K + 1;
    Rigid *d_T = (Rigid *)(g.meta.as<int>() + gmap_meta_ints(g.meta_submaps));
    std::vector<int> h((size_t)3 * K + 6, 0);
    std::copy(g.cnt.begin(), g.cnt.end(), h.begin());
    std::copy(g.off.begin(), g.off.end(), h.begin() + K);
    GEM_CUDA(m, cudaMemcpyAsync(d_cnt, h.data(), h.size() * 4, cudaMemcpyHostToDevice, g.stream.p));
    SubPoint *arena = g.arena[g.cur].as<SubPoint>();
    if (Kp > 1) {
        GEM_CUDA(m, cudaMemcpyAsync(d_T, T.data(), (size_t)Kp * sizeof(Rigid), cudaMemcpyHostToDevice, g.stream.p));
        const int n = g.off[Kp] - g.off[1];
        if (n > 0) k_transform_segments<<<blocks_for((size_t)n, 256, 1 << 30), 256, 0, g.stream.p>>>(arena, d_off + 1, d_T + 1, Kp - 1);
        GEM_CUDA(m, cudaGetLastError());
    }
    int launches = 0;
    for (const auto &pr : pairs) { // each pair's scratch laid out for its own two upper bounds (within pair_bytes(big, big))
        const int j = pr.first, i = pr.second;
        const cudaError_t e = enqueue_pair(g.stream.p, pair_layout(g.pair.p, g.cnt[j], g.cnt[i]), arena + g.off[j], g.cnt[j], d_cnt + j, arena + g.off[i], g.cnt[i], d_cnt + i,
                                           resolution, compat, d_ctr, launches);
        if (e != cudaSuccess) return fail(m, GEM_ERR_CUDA, std::string("gem_global_map_update: ") + cudaGetErrorString(e));
    }
    if (!pairs.empty()) { // the stack back to back again, into the other arena buffer
        k_pack_offsets<<<1, 1, 0, g.stream.p>>>(d_cnt, K, d_off_new);
        k_pack_segments<<<blocks_for((size_t)g.off[K], 256, 1 << 30), 256, 0, g.stream.p>>>(arena, g.arena[g.cur ^ 1].as<SubPoint>(), d_off,
                                                                                          d_off_new, d_cnt, K);
        GEM_CUDA(m, cudaGetLastError());
    }
    GEM_CUDA(m, cudaMemcpyAsync(h.data(), d_cnt, h.size() * 4, cudaMemcpyDeviceToHost, g.stream.p));
    GEM_CUDA(m, cudaStreamSynchronize(g.stream.p));
    if (!pairs.empty()) g.cur ^= 1;
    for (int i = 0; i < K; i++) {
        g.cnt[i] = h[i];
        g.off[i + 1] = g.off[i] + h[i];
    }
    for (int i = 1; i < Kp; i++) std::copy(opt_poses + 16 * (size_t)i, opt_poses + 16 * (size_t)(i + 1), &g.poses[16 * (size_t)i]);
    if (fused_out) *fused_out = h[3 * (size_t)K + 2];
    return GEM_OK;
}

int gem_global_map_info(gem_map *m, int *submaps, int *keyframes, long long *records)
{
    if (!m) return GEM_ERR_INVALID;
    GlobalStore &g = m->gmap;
    GLock lk(g.mu);
    if (submaps) *submaps = (int)g.cnt.size();
    if (keyframes) *keyframes = (int)(g.centres.size() / 2);
    if (records) *records = g.off.back();
    return GEM_OK;
}

int gem_global_map_submap(gem_map *m, int i, void **records_out, int *count_out)
{
    if (!m || !records_out || !count_out) return fail(m, GEM_ERR_INVALID, "gem_global_map_submap: bad argument");
    GlobalStore &g = m->gmap;
    GLock lk(g.mu);
    if (i < 0 || i >= (int)g.cnt.size()) return fail(m, GEM_ERR_INVALID, "gem_global_map_submap: no such submap");
    *records_out = g.arena[g.cur].as<SubPoint>() + g.off[i];
    *count_out = g.cnt[i];
    return GEM_OK;
}

int gem_global_map_records(gem_map *m, void **records_out, long long *count_out)
{
    if (!m || !records_out || !count_out) return fail(m, GEM_ERR_INVALID, "gem_global_map_records: bad argument");
    GlobalStore &g = m->gmap;
    GLock lk(g.mu);
    *records_out = g.arena[g.cur].p;
    *count_out = g.off.back();
    return GEM_OK;
}

int gem_global_map_pose(gem_map *m, int i, float pose_out[16], float centre_out[2])
{
    if (!m) return GEM_ERR_INVALID;
    GlobalStore &g = m->gmap;
    GLock lk(g.mu);
    if (i < 0 || i >= (int)(g.centres.size() / 2)) return fail(m, GEM_ERR_INVALID, "gem_global_map_pose: no such keyframe");
    if (pose_out) std::copy(&g.poses[16 * (size_t)i], &g.poses[16 * (size_t)i] + 16, pose_out);
    if (centre_out) { centre_out[0] = g.centres[2 * (size_t)i]; centre_out[1] = g.centres[2 * (size_t)i + 1]; }
    return GEM_OK;
}

void *gem_global_map_stream(gem_map *m)
{
    if (!m) return nullptr;
    GlobalStore &g = m->gmap;
    GLock lk(g.mu);
    SetDev sd(m->dev);
    return gmap_ready(m) == GEM_OK ? (void *)g.stream.p : nullptr;
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
    if ((long long)world * cap > m->P) // (this also bounds k_bin_peer's sub-buckets, gem_route.cuh)
        return fail(m, GEM_ERR_INVALID, "gem_tiled_attach: world * bucket_capacity (rounded up to 256) = " + std::to_string((long long)world * cap) +
                                            " exceeds max_points = " + std::to_string(m->P) + " (at most 2^" + std::to_string(FOLD_INDEX_BITS) + ")");
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
    ts.g.reset();
    ts.attached = true;
    return GEM_OK;
}

// One step of a tiled map: route this rank's cloud to the owning tiles (peer stores), bin what the peers delivered,
// fold.  Pipelined two deep by default: call j issues ONE graph {fold_long, fold of step j-1 || route -> bin of step j}.
// GEM_B200_TILED_DEPTH=3 pipelines three deep: four independent kernels {fold_long, fold of step j-2 || bin of step j-1
// || route of step j}.  What is outstanding after the last call is issued by whatever reads the map next (gem_flush).
// Every rank must make the same sequence of gem_tiled_step calls (a bin waits for every peer's flag of its step).
int gem_tiled_step(gem_map *m, const void *xyzi, const void *rgba, int n, const gem_frame *frame)
{
    if (!m || !frame || n < 0 || (n > 0 && !xyzi) || !sensor_ok(frame->sensor)) return fail(m, GEM_ERR_INVALID, "gem_tiled_step: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    TiledState &ts = m->tiled;
    if (!ts.attached) return fail(m, GEM_ERR_INVALID, "gem_tiled_step: gem_tiled_attach first");
    if (n > ts.cap) return fail(m, GEM_ERR_INVALID, "gem_tiled_step: cloud larger than bucket_capacity");
    int rc;
    const bool serial = m->profiling;
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
    // stereo / perfect frames take the every-model instantiation (gem_route.cuh)
    auto *route_kernel = any_model(fp) ? k_route_peer_any : k_route_peer;
    void *route_args[] = {&gg, &fp, &px, &pr, &nn, &th, &tw, &tiles_c, &worldv, &my_rank, &nblk, &cap, &bufv, &stepv, &pb, &ticket};
    auto launch_route = [&]() -> int {
        GEM_LAUNCH(m, GEM_PROF_ROUTE, route_kernel<<<nblk, ROUTE_BLOCK, 0, m->stream>>>(gg, fp, px, pr, nn, th, tw, tiles_c, worldv, my_rank, nblk, cap, bufv, stepv, pb, ticket));
        GEM_CUDA(m, cudaGetLastError());
        return GEM_OK;
    };
    memset(&m->stats, 0, sizeof m->stats);
    m->stats.points_in = n;
    RegionOps none{};
    int one = 1;
    const bool graphs = !serial;
    if (!graphs || ts.depth == 2) {
        // route -> bin of this step on the stream or in one graph with the previous step's folds
        if (!graphs || !m->pend.active) {
            if ((rc = drain(m)) || (rc = launch_route())) return rc;
            const TiledBin b = tiled_bin_of(m, stepv, bufv);
            if ((rc = launch_tiled_bin(m, b))) return rc;
            if (serial) return launch_fold(m, b.fold, none, 0, true, true);
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
    kr.func = (void *)route_kernel; kr.gridDim = dim3((unsigned)nblk); kr.blockDim = dim3(ROUTE_BLOCK); kr.sharedMemBytes = 0; kr.kernelParams = route_args;
    kb.func = (void *)k_bin_peer; kb.gridDim = dim3((unsigned)bin_peer_blocks(b.nsub)); kb.blockDim = dim3(ROUTE_BLOCK); kb.sharedMemBytes = 0; kb.kernelParams = bin_args;
    Graph &tg = ts.g;
    if (!tg.exec.p || ts.route_func != kr.func) { // (re)build: a node's kernel cannot be swapped for the other sensor kind's
        tg.reset();
        ts.route_func = kr.func;
        GEM_CUDA(m, cudaGraphCreate(&tg.graph.p, 0));
        GEM_CUDA(m, cudaGraphAddKernelNode(&ts.long_node, tg.graph.p, nullptr, 0, &kl));
        GEM_CUDA(m, cudaGraphAddKernelNode(&ts.route_node, tg.graph.p, nullptr, 0, &kr));
        GEM_CUDA(m, cudaGraphAddKernelNode(&ts.fold_node, tg.graph.p, nullptr, 0, &kf));
        if (ts.depth == 2) GEM_CUDA(m, cudaGraphAddKernelNode(&ts.bin_node, tg.graph.p, &ts.route_node, 1, &kb));
        else GEM_CUDA(m, cudaGraphAddKernelNode(&ts.bin_node, tg.graph.p, nullptr, 0, &kb));
        GEM_CUDA(m, cudaGraphInstantiate(&tg.exec.p, tg.graph.p, 0));
    } else {
        GEM_CUDA(m, cudaGraphExecKernelNodeSetParams(tg.exec.p, ts.long_node, &kl));
        GEM_CUDA(m, cudaGraphExecKernelNodeSetParams(tg.exec.p, ts.route_node, &kr));
        GEM_CUDA(m, cudaGraphExecKernelNodeSetParams(tg.exec.p, ts.fold_node, &kf));
        GEM_CUDA(m, cudaGraphExecKernelNodeSetParams(tg.exec.p, ts.bin_node, &kb));
    }
    GEM_CUDA(m, cudaGraphLaunch(tg.exec.p, m->stream));
    m->launches += 4;
    m->pend = b.fold;
    if (ts.depth != 2) { ts.routed.active = true; ts.routed.step = stepv; ts.routed.buf = bufv; }
    return GEM_OK;
}

// ---- raw sensor messages: PointCloud2 decode, cv_bridge's 8-bit conversions, the one-call frame (gem_ingest.cuh; f12) ----
int gem_pointcloud2_mapping(const gem_pointcloud2 *layout, unsigned long long data_bytes, gem_pc2_mapping *out)
{
    const char *why = pc2_map(layout, data_bytes, out);
    return why ? fail(nullptr, GEM_ERR_INVALID, std::string("gem_pointcloud2_mapping: ") + why) : GEM_OK;
}

// rec 16: float4 xyzi; rec 32: whole PointXYZRGBICT records
static int launch_decode(gem_map *m, const gem_pointcloud2 *layout, const gem_pc2_mapping &mp, const void *data, void *out, int rec = 16)
{
    if (mp.points == 0) return GEM_OK;
    const Pc2Params p = pc2_params(layout, mp, data, mp.bytes); // the kernel reads no byte past the last point's
    const int blocks = p.tiles < (unsigned long long)NUM_SMS * 16 ? (int)p.tiles : NUM_SMS * 16;
    if (rec == 32) GEM_LAUNCH(m, GEM_PROF_OTHER, k_decode_pc2<32><<<blocks, PC2_BLOCK, pc2_smem_bytes(p), m->stream>>>(p, (uint4 *)out));
    else GEM_LAUNCH(m, GEM_PROF_OTHER, k_decode_pc2<16><<<blocks, PC2_BLOCK, pc2_smem_bytes(p), m->stream>>>(p, (uint4 *)out));
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}

int gem_decode_pointcloud2(gem_map *m, const gem_pointcloud2 *layout, const void *data, unsigned long long data_bytes, void *xyzi_out)
{
    if (!m) return GEM_ERR_INVALID;
    gem_pc2_mapping mp;
    const char *why = pc2_map(layout, data_bytes, &mp);
    if (why) return fail(m, GEM_ERR_INVALID, std::string("gem_decode_pointcloud2: ") + why);
    if (mp.points > 0 && ((mp.bytes > 0 && !data) || !xyzi_out || ((uintptr_t)xyzi_out & 15u)))
        return fail(m, GEM_ERR_INVALID, "gem_decode_pointcloud2: NULL pointer, or the output is not 16-byte aligned");
    if (mp.points > 0 && ranges_meet(data, mp.bytes, xyzi_out, (size_t)mp.points * 16))
        return fail(m, GEM_ERR_INVALID, "gem_decode_pointcloud2: the message and output ranges overlap");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    return launch_decode(m, layout, mp, data, xyzi_out);
}

// f18: the same decode into whole 32-byte records
int gem_decode_pointcloud2_records(gem_map *m, const gem_pointcloud2 *layout, const void *data, unsigned long long data_bytes,
                                   void *points32_out)
{
    if (!m) return GEM_ERR_INVALID;
    gem_pc2_mapping mp;
    const char *why = pc2_map(layout, data_bytes, &mp);
    if (why) return fail(m, GEM_ERR_INVALID, std::string("gem_decode_pointcloud2_records: ") + why);
    if (mp.points > 0 && ((mp.bytes > 0 && !data) || !points32_out || ((uintptr_t)points32_out & 15u)))
        return fail(m, GEM_ERR_INVALID, "gem_decode_pointcloud2_records: NULL pointer, or the output is not 16-byte aligned");
    if (mp.points > 0 && ranges_meet(data, mp.bytes, points32_out, (size_t)mp.points * PC2_RECORD))
        return fail(m, GEM_ERR_INVALID, "gem_decode_pointcloud2_records: the message and output ranges overlap");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    return launch_decode(m, layout, mp, data, points32_out, (int)PC2_RECORD);
}

static int launch_image(gem_map *m, int enc, const void *src, int width, int height, long long step, void *dst, long long dst_step)
{
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_image_to_bgr8<<<blocks_for((size_t)width * height, 256), 256, 0, m->stream>>>(
                                      (const unsigned char *)src, width, height, step, enc, (unsigned char *)dst, dst_step));
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}

// bytes of a width x height image with `channels` bytes per pixel and rows `step` bytes apart (the last row unpadded)
static size_t image_bytes(int width, int height, long long step, int channels)
{
    return (size_t)(height - 1) * (size_t)step + (size_t)channels * width;
}

int gem_image_to_bgr8(gem_map *m, const char *encoding, const void *src, int width, int height, int step, void *dst, int dst_step)
{
    if (!m) return GEM_ERR_INVALID;
    const int enc = image_encoding(encoding);
    if (enc < 0) return fail(m, GEM_ERR_INVALID, "gem_image_to_bgr8: encoding is not bgr8, rgb8, bgra8, rgba8 or mono8");
    const int ch = image_channels(enc);
    if (!src || !dst || width < 1 || height < 1 || (long long)step < (long long)ch * width || (long long)dst_step < 3ll * width)
        return fail(m, GEM_ERR_INVALID, "gem_image_to_bgr8: bad argument");
    if (ranges_meet(src, image_bytes(width, height, step, ch), dst, image_bytes(width, height, dst_step, 3)))
        return fail(m, GEM_ERR_INVALID, "gem_image_to_bgr8: the source and destination ranges overlap");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    return launch_image(m, enc, src, width, height, step, dst, dst_step);
}

// the pre-filter's steps are ones gem_voxel_grid takes, and the frame's sensor is unorganised
static const char *prefilter_bad(const gem_prefilter *pf, const gem_frame *frame)
{
    if (pf->nsteps < 0 || pf->nsteps > GEM_PREFILTER_MAX_STEPS) return "nsteps outside 0..GEM_PREFILTER_MAX_STEPS";
    for (int j = 0; j < pf->nsteps; j++)
        if (const char *why = vox_params_bad(&pf->step[j])) return why;
    if (frame->sensor.cloud_width != 0) return "the filtered cloud is unorganised: sensor.cloud_width must be 0";
    return nullptr;
}

// ring call i on n > 0 points at `in` (device; n is the upper bound): the pre-filter's steps into staging set i % 3 (or a
// copy when there are none; pf == NULL: an unfiltered call), the colour lookup (bgr != NULL) and the pipelined add, with
// no host read-back.  vox_grow first.
static int filtered_slot(gem_map *m, unsigned i, const float4 *in, int n, const gem_prefilter *pf, const ProjParams *pp,
                         const unsigned char *bgr, const gem_frame *frame)
{
    const int b = (int)(i % 3u), k = pf ? pf->nsteps : 0;
    float4 *slot = (float4 *)m->d_axyzi[b];
    const int *n_dev = nullptr;
    int rc;
    if (pf) {
        m->pf_slot = b;
        m->pf_nsteps = k;
    }
    if (k > 0) {
        VoxStep *st = vox_steps(m, b);
        if ((rc = vox_chain_enqueue(m, pf->step, k, in, n, slot, n, st, true))) return rc;
        n_dev = &st[k - 1].count;
    } else if (in != slot) {
        GEM_CUDA(m, cudaMemcpyAsync(slot, in, (size_t)n * 16, cudaMemcpyDeviceToDevice, m->stream));
    }
    // a point's colour depends only on the points before it (gem_colour.cuh, C5), so colouring the n entries of the slot
    // leaves the filtered ones as colouring the filtered count would; the entries past it are never binned
    if (bgr && (rc = colourise_enqueue(m, slot, n, *pp, bgr, (uchar4 *)m->d_argba[b]))) return rc;
    return async_add_slot(m, i, n, bgr != nullptr, frame, n_dev);
}

// gem_add_pointcloud2_host_async (pf == NULL) and gem_add_pointcloud2_filtered_host_async
static int pc2_host_async(gem_map *m, const gem_pointcloud2 *layout, const void *data, unsigned long long data_bytes,
                          const gem_camera_image *img, const gem_prefilter *pf, const gem_frame *frame, const char *what)
{
    const std::string w = std::string(what) + ": ";
    if (!m || !frame || !sensor_ok(frame->sensor)) return fail(m, GEM_ERR_INVALID, w + "bad argument");
    if (pf)
        if (const char *why = prefilter_bad(pf, frame)) return fail(m, GEM_ERR_INVALID, w + why);
    gem_pc2_mapping mp;
    const char *why = pc2_map(layout, data_bytes, &mp);
    if (why) return fail(m, GEM_ERR_INVALID, w + why);
    if (mp.bytes > 0 && !data) return fail(m, GEM_ERR_INVALID, w + "NULL data");
    if (mp.points > m->P) return fail(m, GEM_ERR_INVALID, w + "width * height exceeds max_points");
    int enc = -1;
    size_t img_bytes = 0;
    if (img) {
        char e[sizeof img->encoding + 1];
        memcpy(e, img->encoding, sizeof img->encoding);
        e[sizeof img->encoding] = 0;
        if ((enc = image_encoding(e)) < 0)
            return fail(m, GEM_ERR_INVALID, w + "encoding is not bgr8, rgb8, bgra8, rgba8 or mono8");
        if (!img->data || img->width < 1 || img->height < 1 || (long long)img->step < (long long)image_channels(enc) * img->width)
            return fail(m, GEM_ERR_INVALID, w + "bad image");
        img_bytes = image_bytes(img->width, img->height, img->step, image_channels(enc));
    }
    const int n = (int)mp.points;
    const bool filter = pf && pf->nsteps > 0;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_async_ring(m);
    if (rc) return rc;
    if (n == 0) return flush_all_pending(m);
    const unsigned i = m->async_calls;
    const int b = (int)(i % 3u);
    // growth before anything is enqueued: both streams drained, so no queued copy or kernel uses a buffer that goes
    const size_t bgr_bytes = img && enc != IMG_BGR8 ? (size_t)3 * img->width * img->height : 0;
    const bool node = img && m->colour_lookup == GEM_COLOUR_LOOKUP_NODE;
    if (m->pc2_raw[b].cap < mp.bytes || m->pc2_img[b].cap < img_bytes || m->pc2_bgr.cap < bgr_bytes || (node && m->colour.n < n) ||
        (filter && !vox_fits(m, n, true))) {
        GEM_CUDA(m, cudaStreamSynchronize(m->copy_stream.p));
        GEM_CUDA(m, cudaStreamSynchronize(m->stream));
        if ((rc = scratch_grow(m, m->pc2_raw[b], mp.bytes, what, m->stream)) ||
            (rc = scratch_grow(m, m->pc2_img[b], img_bytes, what, m->stream)) ||
            (rc = scratch_grow(m, m->pc2_bgr, bgr_bytes, what, m->stream)) ||
            (node && (rc = colour_grow(m, n, what))) || (filter && (rc = vox_grow(m, n, true, what))))
            return rc;
    }
    m->async_calls++;
    // copy stream: the slot's last reader (call i-3) is done (see gem_add_points_host_async); pageable sources are staged
    // by CUDA before cudaMemcpyAsync returns
    GEM_CUDA(m, cudaStreamWaitEvent(m->copy_stream.p, m->ev_done[b].p, 0));
    if (mp.bytes > 0) GEM_CUDA(m, cudaMemcpyAsync(m->pc2_raw[b].p, data, mp.bytes, cudaMemcpyHostToDevice, m->copy_stream.p));
    if (img) GEM_CUDA(m, cudaMemcpyAsync(m->pc2_img[b].p, img->data, img_bytes, cudaMemcpyHostToDevice, m->copy_stream.p));
    GEM_CUDA(m, cudaEventRecord(m->ev_h2d[b].p, m->copy_stream.p));
    GEM_CUDA(m, cudaStreamWaitEvent(m->stream, m->ev_h2d[b].p, 0));
    // decode into staging set b (with the filter: into the second step buffer, which the first step does not write), then
    // the filter, and (with an image) BGR8 and the colourisation of ElevationMapping.cpp:331-381 by the handle's lookup mode
    float4 *dec = filter ? m->vox.buf[1].as<float4>() : (float4 *)m->d_axyzi[b];
    if ((rc = launch_decode(m, layout, mp, m->pc2_raw[b].p, dec))) return rc;
    const void *bgr = nullptr;
    ProjParams pp{};
    if (img) {
        bgr = m->pc2_img[b].p;
        int stride = img->step;
        if (enc != IMG_BGR8) {
            if ((rc = launch_image(m, enc, m->pc2_img[b].p, img->width, img->height, img->step, m->pc2_bgr.p, 3ll * img->width))) return rc;
            bgr = m->pc2_bgr.p;
            stride = 3 * img->width;
        }
        pp = proj_params(img->T_camera, img->T_lidar, img->width, img->height, stride);
    }
    return filtered_slot(m, i, dec, n, pf, &pp, (const unsigned char *)bgr, frame);
}

int gem_add_pointcloud2_host_async(gem_map *m, const gem_pointcloud2 *layout, const void *data, unsigned long long data_bytes,
                                   const gem_camera_image *img, const gem_frame *frame)
{
    return pc2_host_async(m, layout, data, data_bytes, img, nullptr, frame, "gem_add_pointcloud2_host_async");
}

int gem_add_pointcloud2_filtered_host_async(gem_map *m, const gem_pointcloud2 *layout, const void *data, unsigned long long data_bytes,
                                            const gem_camera_image *img, const gem_prefilter *prefilter, const gem_frame *frame)
{
    if (!prefilter) return fail(m, GEM_ERR_INVALID, "gem_add_pointcloud2_filtered_host_async: bad argument");
    return pc2_host_async(m, layout, data, data_bytes, img, prefilter, frame, "gem_add_pointcloud2_filtered_host_async");
}

int gem_add_points_filtered_stream(gem_map *m, const void *xyzi, int n, const gem_prefilter *pf, const void *bgr,
                                   const gem_projection *proj, const gem_frame *frame)
{
    const char *what = "gem_add_points_filtered_stream";
    if (!m || !frame || !pf || n < 0 || (n > 0 && !xyzi) || !sensor_ok(frame->sensor) ||
        (bgr && (!proj || proj->width < 1 || proj->height < 1 || proj->row_stride < 3 * proj->width)))
        return fail(m, GEM_ERR_INVALID, std::string(what) + ": bad argument");
    if (const char *why = prefilter_bad(pf, frame)) return fail(m, GEM_ERR_INVALID, std::string(what) + ": " + why);
    if (n > m->P) return fail(m, GEM_ERR_INVALID, std::string(what) + ": n exceeds max_points");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    int rc = ensure_async_ring(m);
    if (rc) return rc;
    if (n == 0) return flush_all_pending(m);
    const bool node = bgr && m->colour_lookup == GEM_COLOUR_LOOKUP_NODE;
    if ((node && m->colour.n < n) || (pf->nsteps > 0 && !vox_fits(m, n, true))) {
        GEM_CUDA(m, cudaStreamSynchronize(m->copy_stream.p));
        GEM_CUDA(m, cudaStreamSynchronize(m->stream));
        if ((node && (rc = colour_grow(m, n, what))) || (pf->nsteps > 0 && (rc = vox_grow(m, n, true, what)))) return rc;
    }
    // staging set i % 3 is written on the handle's stream, after the fold of call i-3 that last read it
    const unsigned i = m->async_calls++;
    ProjParams pp{};
    if (bgr) pp = proj_params(proj->T_camera, proj->T_lidar, proj->width, proj->height, proj->row_stride);
    return filtered_slot(m, i, static_cast<const float4 *>(xyzi), n, pf, &pp, static_cast<const unsigned char *>(bgr), frame);
}

int gem_prefilter_info(gem_map *m, gem_voxel_grid_info *out, int nsteps)
{
    if (!m) return GEM_ERR_INVALID;
    if (nsteps < 0 || nsteps > GEM_PREFILTER_MAX_STEPS || (nsteps > 0 && !out)) return fail(m, GEM_ERR_INVALID, "gem_prefilter_info: bad argument");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    VoxStep h[GEM_PREFILTER_MAX_STEPS] = {};
    const int k = m->pf_slot < 0 ? 0 : std::min(nsteps, m->pf_nsteps);
    if (k > 0) {
        GEM_CUDA(m, cudaMemcpyAsync(h, vox_steps(m, m->pf_slot), (size_t)k * sizeof(VoxStep), cudaMemcpyDeviceToHost, m->stream));
        GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    }
    for (int j = 0; j < nsteps; j++) out[j] = j < k ? vox_info(h[j]) : gem_voxel_grid_info{};
    return GEM_OK;
}

// ---- point clouds as PCD files: PCL's generateHeader / writeASCII / writeBinary (gem_pcd.cuh; f13) ----------------------
int gem_pcd_header(long long n, int flags, char *out, int capacity, int *len_out)
{
    if (len_out) *len_out = 0;
    if (!len_out || capacity < 0 || (capacity > 0 && !out)) return fail(nullptr, GEM_ERR_INVALID, "gem_pcd_header: bad argument");
    if (n < 0 || (flags & ~(GEM_PCD_BINARY | GEM_PCD_RGB_UINT32))) return fail(nullptr, GEM_ERR_INVALID, "gem_pcd_header: n < 0 or unknown flags");
    if (n == 0) return fail(nullptr, GEM_ERR_INVALID, "gem_pcd_header: the cloud is empty (PCL writes no file)");
    char h[GEM_PCD_HEADER_MAX];
    const int len = pcd_header(n, flags, h);
    *len_out = len;
    if (capacity > len) memcpy(out, h, (size_t)len + 1);
    return GEM_OK;
}

int gem_pcd_format(gem_map *m, const void *points32_device, int n, int flags, void *out_device, long long capacity, long long *bytes_out)
{
    if (bytes_out) *bytes_out = 0;
    if (!m) return GEM_ERR_INVALID;
    if (!bytes_out || capacity < 0 || (capacity > 0 && !out_device)) return fail(m, GEM_ERR_INVALID, "gem_pcd_format: bad argument");
    if (n < 0 || (flags & ~(GEM_PCD_BINARY | GEM_PCD_RGB_UINT32))) return fail(m, GEM_ERR_INVALID, "gem_pcd_format: n < 0 or unknown flags");
    if (n == 0) return fail(m, GEM_ERR_INVALID, "gem_pcd_format: the cloud is empty (PCL writes no file)");
    if (!points32_device || ((uintptr_t)points32_device & 15u))
        return fail(m, GEM_ERR_INVALID, "gem_pcd_format: the records are NULL or not 16-byte aligned");
    const float4 *rec = static_cast<const float4 *>(points32_device);
    unsigned char *out = static_cast<unsigned char *>(out_device);
    const size_t N = (size_t)n, tiles = (N + PCD_BLOCK - 1) / PCD_BLOCK;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    cudaStream_t st = m->stream;
    long long bytes = (long long)N * PCD_BINARY_RECORD;
    if (!(flags & GEM_PCD_BINARY)) {
        PcdScratch &S = m->pcd;
        const char *what = "gem_pcd_format";
        size_t t_scan = 0;
        GEM_CUDA(m, cub::DeviceScan::InclusiveSum(nullptr, t_scan, (long long *)nullptr, (long long *)nullptr, (int)tiles, st));
        int rc;
        if ((rc = scratch_grow(m, S.bytes, tiles * 8, what, m->stream)) || (rc = scratch_grow(m, S.ends, tiles * 8, what, m->stream)) ||
            (rc = scratch_grow(m, S.temp, t_scan, what, m->stream)))
            return rc;
        long long *tb = S.bytes.as<long long>(), *te = S.ends.as<long long>();
        size_t tcap = S.temp.cap;
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_pcd_len<<<(unsigned)tiles, PCD_BLOCK, 0, st>>>(rec, n, flags & GEM_PCD_RGB_UINT32, tb));
        GEM_CUDA(m, cudaGetLastError());
        GEM_CUDA(m, cub::DeviceScan::InclusiveSum(S.temp.p, tcap, tb, te, (int)tiles, st));
        GEM_CUDA(m, cudaMemcpyAsync(&bytes, te + (tiles - 1), sizeof bytes, cudaMemcpyDeviceToHost, st));
        GEM_CUDA(m, cudaStreamSynchronize(st));
    }
    *bytes_out = bytes;
    if (capacity < bytes) return GEM_OK; // a size query, or too small: nothing is written
    if (ranges_meet(points32_device, N * 32, out_device, (size_t)bytes))
        return fail(m, GEM_ERR_INVALID, "gem_pcd_format: the records and the output overlap");
    if (flags & GEM_PCD_BINARY)
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_pcd_binary<<<(unsigned)tiles, PCD_BLOCK, 0, st>>>(rec, n, out));
    else
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_pcd_ascii<<<(unsigned)tiles, PCD_BLOCK, 0, st>>>(rec, n, flags & GEM_PCD_RGB_UINT32,
                                                                                     m->pcd.ends.as<long long>(), out));
    GEM_CUDA(m, cudaGetLastError());
    GEM_CUDA(m, cudaStreamSynchronize(st));
    return GEM_OK;
}

// ---- the node's map topics as serialised ROS1 messages (gem_rosfmt.h, gem_rosmsg.cuh; f15) -----------------------------
// the checks every gem_ros_* call makes first.  *pinned: out is page-locked host memory (the kernels may store to
// device, managed and pinned memory; pageable host memory is refused, since a store to it from the device faults)
static int ros_args(gem_map *m, const gem_ros_header *h, void *out, long long capacity, long long *bytes_out, const char *what,
                    bool *pinned, bool reads_map = true)
{
    if (bytes_out) *bytes_out = 0;
    if (!m) return GEM_ERR_INVALID;
    if (!bytes_out || capacity < 0 || (capacity > 0 && !out)) return fail(m, GEM_ERR_INVALID, std::string(what) + ": bad argument");
    if (!gem_ros::header_ok(h)) return fail(m, GEM_ERR_INVALID, std::string(what) + ": NULL header or frame_id");
    if (reads_map && m->geom.tiled) return fail(m, GEM_ERR_INVALID, std::string(what) + ": not available on tiled handles");
    *pinned = false;
    if (out) {
        cudaPointerAttributes a{};
        if (cudaPointerGetAttributes(&a, out) != cudaSuccess) {
            cudaGetLastError(); // an unknown pointer: treated as pageable
            a.type = cudaMemoryTypeUnregistered;
        }
        if (a.type == cudaMemoryTypeUnregistered)
            return fail(m, GEM_ERR_INVALID, std::string(what) + ": out is pageable host memory (device or pinned memory only)");
        *pinned = a.type == cudaMemoryTypeHost;
    }
    return GEM_OK;
}

// Where a map message's kernels write: device memory directly; for pinned host memory a device staging buffer at the
// same 16-byte phase (so the kernels take the same paths and write the same bytes), copied to `out` in one DMA transfer
// by ros_unstage.  The kernels' own stores across PCIe were measured slower than the copy (DESIGN.md f15).
static int ros_stage(gem_map *m, unsigned char *out, long long size, bool pinned, unsigned char **dst)
{
    *dst = out;
    if (!pinned) return GEM_OK;
    const int rc = scratch_grow(m, m->ros_stage, (size_t)size + 16, "gem_ros staging", m->stream);
    if (rc) return rc;
    *dst = m->ros_stage.as<unsigned char>() + ((uintptr_t)out & 15u);
    return GEM_OK;
}
static int ros_unstage(gem_map *m, unsigned char *out, const unsigned char *dst, long long size, bool pinned)
{
    if (pinned) GEM_CUDA(m, cudaMemcpyAsync(out, dst, (size_t)size, cudaMemcpyDeviceToHost, m->stream));
    return GEM_OK;
}

// the framing bytes into their places in `out`; the caller holds the lock.  They go to the device from pageable memory,
// which CUDA copies to its staging memory before cudaMemcpyAsync returns, so `f` may go as soon as this returns, and the
// device buffer is reused in stream order.
static int ros_put_framing(gem_map *m, const gem_ros::Framing &f, unsigned char *out)
{
    const int rc = scratch_grow(m, m->ros_framing, f.bytes.size(), "gem_ros framing", m->stream);
    if (rc) return rc;
    GEM_CUDA(m, cudaMemcpyAsync(m->ros_framing.p, f.bytes.data(), f.bytes.size(), cudaMemcpyHostToDevice, m->stream));
    RosSegs s{};
    for (int k = 0; k < f.nseg; k++) {
        s.at[k] = f.seg[k].at;
        s.src[k] = f.seg[k].src;
        s.len[k] = f.seg[k].len;
    }
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_ros_framing<<<f.nseg, 256, 0, m->stream>>>(m->ros_framing.as<unsigned char>(), s, out));
    GEM_CUDA(m, cudaGetLastError());
    return GEM_OK;
}

int gem_ros_grid_map(gem_map *m, const gem_ros_header *h, void *out, long long capacity, long long *bytes_out)
{
    bool pinned = false;
    int rc = ros_args(m, h, out, capacity, bytes_out, "gem_ros_grid_map", &pinned);
    if (rc) return rc;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    const GridMapFrame gf = grid_frame(m, m->geom.cx, m->geom.cy, m->geom.sx, m->geom.sy);
    gem_ros::Framing f;
    if (gem_ros::grid_map(*h, m->L, gf.res, gf.cx, gf.cy, m->geom.sx, m->geom.sy, f))
        return fail(m, GEM_ERR_INVALID, "gem_ros_grid_map: a layer of more than 2^32 bytes");
    if (capacity < f.size) { // a size query, or too small: nothing is written
        *bytes_out = f.size;
        return GEM_OK;
    }
    unsigned char *o = nullptr;
    if ((rc = ros_stage(m, static_cast<unsigned char *>(out), f.size, pinned, &o)) || (rc = flush_for_observer(m)) ||
        (rc = ros_put_framing(m, f, o)))
        return rc;
    const int nch = (m->L + 31) / 32;
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_ros_grid_map<<<dim3(nch, nch), 256, 0, m->stream>>>(m->ml, m->L, o + f.payload_at[0],
                                                                                         f.payload_at[1] - f.payload_at[0]));
    GEM_CUDA(m, cudaGetLastError());
    if ((rc = ros_unstage(m, static_cast<unsigned char *>(out), o, f.size, pinned))) return rc;
    *bytes_out = f.size;
    return GEM_OK;
}

int gem_ros_orthomosaic(gem_map *m, const gem_ros_header *h, void *out, long long capacity, long long *bytes_out)
{
    bool pinned = false;
    int rc = ros_args(m, h, out, capacity, bytes_out, "gem_ros_orthomosaic", &pinned);
    if (rc) return rc;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    gem_ros::Framing f;
    if (gem_ros::image(*h, m->L, f)) return fail(m, GEM_ERR_INVALID, "gem_ros_orthomosaic: an image of more than 2^32 bytes");
    if (capacity < f.size) {
        *bytes_out = f.size;
        return GEM_OK;
    }
    unsigned char *o = nullptr;
    if ((rc = ros_stage(m, static_cast<unsigned char *>(out), f.size, pinned, &o)) || (rc = flush_for_observer(m)) ||
        (rc = ros_put_framing(m, f, o)))
        return rc;
    unsigned char *img = o + f.payload_at[0];
    const long long nwords = ((long long)((uintptr_t)img & 15u) + f.payload_len[0] + 15) / 16;
    GEM_LAUNCH(m, GEM_PROF_OTHER, k_ros_orthomosaic<<<(unsigned)((nwords + 255) / 256), 256, 0, m->stream>>>(m->geom, m->ml, img, nwords));
    GEM_CUDA(m, cudaGetLastError());
    if ((rc = ros_unstage(m, static_cast<unsigned char *>(out), o, f.size, pinned))) return rc;
    *bytes_out = f.size;
    return GEM_OK;
}

int gem_ros_visual_points(gem_map *m, const gem_ros_header *h, void *out, long long capacity, long long *bytes_out)
{
    bool pinned = false;
    int rc = ros_args(m, h, out, capacity, bytes_out, "gem_ros_visual_points", &pinned);
    if (rc) return rc;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    if ((rc = flush_for_observer(m))) return rc;
    RosVisualSrc src;
    src.ml = m->ml;
    src.f = grid_frame(m, m->geom.cx, m->geom.cy, m->geom.sx, m->geom.sy);
    src.out = nullptr;
    int n = 0;
    if ((rc = compact_cells(m, src, 0, &n))) return rc; // the count alone
    gem_ros::Framing f;
    if (gem_ros::cloud(*h, gem_ros::CLOUD_XYZRGB, n, 1, f))
        return fail(m, GEM_ERR_INVALID, "gem_ros_visual_points: 32 n >= 2^32 (PointCloud2's data length is a uint32)");
    if (capacity < f.size) {
        *bytes_out = f.size;
        return GEM_OK;
    }
    unsigned char *o = nullptr;
    if ((rc = ros_stage(m, static_cast<unsigned char *>(out), f.size, pinned, &o)) || (rc = ros_put_framing(m, f, o))) return rc;
    src.out = o + f.payload_at[0];
    int *d_total = nullptr;
    if ((rc = compact_cells_issue(m, src, n, &d_total)) || (rc = ros_unstage(m, static_cast<unsigned char *>(out), o, f.size, pinned)))
        return rc;
    GEM_CUDA(m, cudaStreamSynchronize(m->stream));
    *bytes_out = f.size;
    return GEM_OK;
}

int gem_ros_cloud(gem_map *m, const gem_ros_header *h, const gem_ros_part *parts, int nparts, int is_dense, void *out,
                  long long capacity, long long *bytes_out)
{
    bool pinned = false;
    int rc = ros_args(m, h, out, capacity, bytes_out, "gem_ros_cloud", &pinned);
    if (rc) return rc;
    if (nparts < 0 || (nparts > 0 && !parts)) return fail(m, GEM_ERR_INVALID, "gem_ros_cloud: nparts < 0 or no parts");
    long long n = 0;
    for (int i = 0; i < nparts; i++) {
        if (parts[i].n < 0 || (parts[i].n > 0 && !parts[i].points32))
            return fail(m, GEM_ERR_INVALID, "gem_ros_cloud: a part with n < 0 or without records");
        n += std::min(parts[i].n, gem_ros::U32_LIMIT); // no overflow; any sum this large is refused below
    }
    gem_ros::Framing f;
    if (gem_ros::cloud(*h, gem_ros::CLOUD_XYZRGBICT, n, is_dense, f))
        return fail(m, GEM_ERR_INVALID, "gem_ros_cloud: 32 n >= 2^32 (PointCloud2's data length is a uint32)");
    if (capacity < f.size) {
        *bytes_out = f.size;
        return GEM_OK;
    }
    for (int i = 0; i < nparts; i++)
        if (parts[i].n > 0 && ranges_meet(parts[i].points32, (size_t)parts[i].n * 32, out, (size_t)f.size))
            return fail(m, GEM_ERR_INVALID, "gem_ros_cloud: the output overlaps a part");
    Lock lk(m->mu);
    SetDev sd(m->dev);
    unsigned char *o = static_cast<unsigned char *>(out);
    if ((rc = ros_put_framing(m, f, o))) return rc;
    long long at = f.payload_at[0];
    for (int i = 0; i < nparts; i++) {
        if (parts[i].n == 0) continue;
        GEM_CUDA(m, cudaMemcpyAsync(o + at, parts[i].points32, (size_t)parts[i].n * 32, cudaMemcpyDefault, m->stream));
        at += 32 * parts[i].n;
    }
    *bytes_out = f.size;
    return GEM_OK;
}

int gem_ros_octomap(gem_map *m, const gem_ros_header *h, void *out, long long capacity, long long *bytes_out)
{
    bool pinned = false;
    int rc = ros_args(m, h, out, capacity, bytes_out, "gem_ros_octomap", &pinned);
    if (rc) return rc;
    Lock lk(m->mu);
    SetDev sd(m->dev);
    const long long bytes = m->oct.bytes;
    if (bytes < 0) return fail(m, GEM_ERR_INVALID, "gem_ros_octomap: no octree has been built");
    gem_ros::Framing f;
    if (gem_ros::octomap(*h, m->oct.res, bytes, f)) return fail(m, GEM_ERR_INVALID, "gem_ros_octomap: a stream of 2^32 bytes or more");
    if (capacity < f.size) {
        *bytes_out = f.size;
        return GEM_OK;
    }
    unsigned char *o = static_cast<unsigned char *>(out);
    if ((rc = ros_put_framing(m, f, o))) return rc;
    if (bytes) GEM_CUDA(m, cudaMemcpyAsync(o + f.payload_at[0], m->oct.nrec[1].p, (size_t)bytes, cudaMemcpyDefault, m->stream));
    *bytes_out = f.size;
    return GEM_OK;
}


// ---- the costmap topics and footprint clearing (gem_rosfmt.h W9-W11 and P1-P4, gem_footprint.h F1-F4; f17) --------------
int gem_costmap_publisher_init(gem_costmap_publisher *p, int always_send_full)
{
    if (!p) return GEM_ERR_INVALID;
    gem_ros::costmap_publisher_init(*p, always_send_full);
    return GEM_OK;
}

int gem_costmap_publisher_bounds(gem_costmap_publisher *p, int x0, int xn, int y0, int yn)
{
    if (!p) return GEM_ERR_INVALID;
    gem_ros::costmap_publisher_bounds(*p, x0, xn, y0, yn);
    return GEM_OK;
}

// a footprint and pose the f17 calls accept: n >= 0 (x, y) pairs, every value finite
static bool footprint_ok(const double *spec_xy, int n, double rx, double ry, double yaw)
{
    if (n < 0 || (n > 0 && !spec_xy) || !std::isfinite(rx) || !std::isfinite(ry) || !std::isfinite(yaw)) return false;
    for (int i = 0; i < 2 * n; i++)
        if (!std::isfinite(spec_xy[i])) return false;
    return true;
}

int gem_ros_costmap(gem_map *m, const gem_ros_header *h, const gem_costmap_window *w, const unsigned char *master_device,
                    gem_costmap_publisher *p, int force_full, void *out, long long capacity, long long *bytes_out, int *kind_out)
{
    if (kind_out) *kind_out = GEM_COSTMAP_PUB_NONE;
    bool pinned = false;
    int rc = ros_args(m, h, out, capacity, bytes_out, "gem_ros_costmap", &pinned, false);
    if (rc) return rc;
    if (!kind_out || !p || !master_device || (force_full != 0 && force_full != 1))
        return fail(m, GEM_ERR_INVALID, "gem_ros_costmap: bad argument");
    if (!cost_window_ok(w)) return fail(m, GEM_ERR_INVALID, "gem_ros_costmap: bad window");
    gem_ros::CostmapPlan d;
    gem_ros::Framing f;
    bool writes = false;
    if (gem_ros::costmap_message(*h, *w, *p, force_full, !out, capacity, d, f, writes))
        return fail(m, GEM_ERR_INVALID, "gem_ros_costmap: the accumulated bounds lie outside the grid");
    *kind_out = d.kind;
    if (!writes) { // a size query, or too small: nothing is written and the publisher stays as it was
        *bytes_out = f.size;
        return GEM_OK;
    }
    const size_t cells = (size_t)w->size_x * w->size_y;
    if (f.size > 0 && ranges_meet(master_device, cells, out, (size_t)f.size))
        return fail(m, GEM_ERR_INVALID, "gem_ros_costmap: the output overlaps the master grid");
    if (d.kind != GEM_COSTMAP_PUB_NONE) {
        Lock lk(m->mu);
        SetDev sd(m->dev);
        unsigned char *o = nullptr;
        if ((rc = ros_stage(m, static_cast<unsigned char *>(out), f.size, pinned, &o)) || (rc = ros_put_framing(m, f, o))) return rc;
        unsigned char *data = o + f.payload_at[0];
        const long long n = f.payload_len[0];
        if (n > 0) {
            const long long nwords = ((long long)((uintptr_t)data & 15u) + n + 15) / 16;
            GEM_LAUNCH(m, GEM_PROF_OTHER, k_ros_costmap<<<(unsigned)((nwords + 255) / 256), 256, 0, m->stream>>>(
                                              master_device, w->size_x, d.x0, d.y0, d.width, n, data, nwords));
            GEM_CUDA(m, cudaGetLastError());
        }
        if ((rc = ros_unstage(m, static_cast<unsigned char *>(out), o, f.size, pinned))) return rc;
    }
    gem_ros::costmap_commit(*p, *w, d, force_full);
    *bytes_out = f.size;
    return GEM_OK;
}

int gem_ros_footprint(gem_map *m, const gem_ros_header *h, const double *spec_xy, int n, double robot_x, double robot_y,
                      double robot_yaw, void *out, long long capacity, long long *bytes_out)
{
    bool pinned = false;
    int rc = ros_args(m, h, out, capacity, bytes_out, "gem_ros_footprint", &pinned, false);
    if (rc) return rc;
    if (!footprint_ok(spec_xy, n, robot_x, robot_y, robot_yaw))
        return fail(m, GEM_ERR_INVALID, "gem_ros_footprint: n < 0, no footprint, or a value that is not finite");
    std::vector<gem_fp::Point> pts;
    gem_fp::transform(spec_xy, n, robot_x, robot_y, robot_yaw, pts);
    std::vector<double> xy;
    for (const gem_fp::Point &q : pts) {
        xy.push_back(q.x);
        xy.push_back(q.y);
    }
    gem_ros::Framing f;
    if (gem_ros::polygon_stamped(*h, xy.data(), n, f)) return fail(m, GEM_ERR_INVALID, "gem_ros_footprint: a polygon of 2^32 bytes or more");
    if (!out || capacity < f.size) {
        *bytes_out = f.size;
        return GEM_OK;
    }
    Lock lk(m->mu);
    SetDev sd(m->dev);
    if ((rc = ros_put_framing(m, f, static_cast<unsigned char *>(out)))) return rc;
    *bytes_out = f.size;
    return GEM_OK;
}

// ObstacleLayer::updateFootprint's bounds and updateCosts' setConvexPolygonCost(FREE_SPACE) on the layer grid.  The
// reference fills at updateCosts; this fills at bounds time, which gives the same bytes: nothing reads the layer grid in
// between, and with a vertex touched the bounds are never empty, so LayeredCostmap::updateMap always reaches updateCosts.
int gem_costmap_footprint(gem_map *m, const gem_costmap_window *w, const double *spec_xy, int n, double robot_x, double robot_y,
                          double robot_yaw, unsigned char *layer_device, gem_costmap_marks *out)
{
    if (!m || !layer_device || !out) return fail(m, GEM_ERR_INVALID, "gem_costmap_footprint: bad argument");
    if (!cost_window_ok(w)) return fail(m, GEM_ERR_INVALID, "gem_costmap_footprint: bad window");
    if (!footprint_ok(spec_xy, n, robot_x, robot_y, robot_yaw))
        return fail(m, GEM_ERR_INVALID, "gem_costmap_footprint: n < 0, no footprint, or a value that is not finite");
    std::vector<gem_fp::Point> pts;
    std::vector<gem_fp::Cell> cells;
    gem_fp::transform(spec_xy, n, robot_x, robot_y, robot_yaw, pts);
    gem_costmap_marks r{0, 0, INFINITY, INFINITY, -INFINITY, -INFINITY};
    for (const gem_fp::Point &q : pts) { // touch(), a zero reported as +0 (f8)
        r.min_x = std::min(r.min_x, q.x + 0.0); r.min_y = std::min(r.min_y, q.y + 0.0);
        r.max_x = std::max(r.max_x, q.x + 0.0); r.max_y = std::max(r.max_y, q.y + 0.0);
    }
    gem_fp::polygon_cells(w->origin_x, w->origin_y, w->resolution, w->size_x, w->size_y, pts, cells);
    std::vector<int> idx(cells.size());
    for (size_t i = 0; i < cells.size(); i++) idx[i] = (int)(cells[i].y * (unsigned)w->size_x + cells[i].x);
    if (!idx.empty()) {
        Lock lk(m->mu);
        SetDev sd(m->dev);
        int rc;
        if ((rc = scratch_grow(m, m->cost_cells, idx.size() * sizeof(int), "costmap footprint cells", m->stream))) return rc;
        // from pageable memory the copy returns once its source is staged, so idx may go when this call returns
        GEM_CUDA(m, cudaMemcpyAsync(m->cost_cells.p, idx.data(), idx.size() * sizeof(int), cudaMemcpyHostToDevice, m->stream));
        GEM_LAUNCH(m, GEM_PROF_OTHER, k_costmap_cells<<<(unsigned)((idx.size() + 255) / 256), 256, 0, m->stream>>>(
                                          m->cost_cells.as<int>(), (int)idx.size(), layer_device, COST_FREE));
        GEM_CUDA(m, cudaGetLastError());
    }
    r.marked = (long long)idx.size();
    *out = r;
    return GEM_OK;
}

} // extern "C"
