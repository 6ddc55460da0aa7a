/*
 * gem_b200.h -- C ABI of libgem_b200.so: the H100-native (sm_90a) replacement for GEM's
 * GPU map library `libgpu.so` (reference: elevation_mapping/elevation_mapping/cuda/
 * gpu_process.cu, "gpu.cu" below; ZJU-Robotics-Lab/GEM @ d7ec953).
 *
 * The reference boundary is 9 C++-mangled free functions declared ad hoc by their callers
 * (ElevationMapping.cpp:44-50, SensorProcessorBase.cpp:34, RobotMotionMapUpdater.cpp:18)
 * with Eigen types by value and one process-global map.  This header is the C-ABI they bind
 * to instead: plain pointers and sizes, an opaque per-map handle, int status codes.
 * compat/gpu_process_shim.cpp re-exports the 9 original symbols on top of it (needs Eigen,
 * compiled inside the catkin workspace), see INTEGRATION.md.
 *
 * Conventions
 *   - every function returns GEM_OK (0) or a GEM_ERR_* code; gem_last_error() gives text;
 *   - "device" pointers are CUDA device pointers on the handle's device, "host" pointers
 *     are ordinary (pageable or pinned) host memory;
 *   - all work of one handle is ordered on one CUDA stream; functions taking device
 *     pointers are asynchronous on that stream, functions taking host pointers return
 *     after the result is visible to the host (like the reference wrappers, which are all
 *     host-synchronous);
 *   - a handle is thread-safe: every entry point takes the handle's (recursive) mutex, so the
 *     reference node's three threads (processpoints: Process_points OUTSIDE MapMutex_ and Fuse
 *     inside, ElevationMapping.cpp:271-282; processmapcells :286-300; the spinner's Move /
 *     Map_feature / Raytracing :388-421) may enter concurrently; calls are serialised, and
 *     what one call enqueued is ordered before the next on the handle's stream;
 *   - there is NO CPU fallback: gem_create fails with GEM_ERR_NO_DEVICE without a GPU.
 *
 * Layer layout seen through this ABI is the reference's: row-major L*L arrays, index
 * x*L+y; elevation/variance/intensity/colour/traver are indexed by STORAGE index (circular
 * buffer), lowest by GEOGRAPHIC index (gpu.cu:430-431, SURVEY appendix A).  Empty cell
 * sentinels: elevation == -10, variance == -10, traver == -10 (gpu.cu:203-210).
 */
#ifndef GEM_B200_H
#define GEM_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define GEM_B200_VERSION 100

enum {
    GEM_OK = 0,
    GEM_ERR_INVALID = 1,   /* bad argument                                   */
    GEM_ERR_CUDA = 2,      /* CUDA runtime error (text in gem_last_error)    */
    GEM_ERR_NO_DEVICE = 3, /* no usable CUDA device / kernels not loadable   */
    GEM_ERR_NOMEM = 4
};

typedef struct gem_map gem_map; /* opaque */

/* Replaces the arguments of Init_GPU_elevationmap (gpu.cu:940) + the hard-coded knobs. */
typedef struct gem_config {
    int length;                  /* cells per side L (gpu.cu:35)                          */
    float resolution;            /* metres per cell (gpu.cu:36)                           */
    float mahalanobis_threshold; /* uploaded but unused by the reference (gate is 5)      */
    float obstacle_threshold;    /* ElevationMapping.cpp:194 hard-codes 0.7               */
    int compat_box_filter;       /* 1: apply the sensor-frame box filter of gpu.cu:393    */
    int max_points;              /* per-launch capacity; larger calls are chunked. 0=auto */
    int device;                  /* CUDA ordinal, -1 = current device                     */
    void *stream;                /* cudaStream_t to run on; NULL = library-owned stream   */
    /* spatial tile owned by this handle (multi-GPU tiling, SURVEY 8e).  All zero = whole
     * map.  Tiled handles do not scroll (gem_move keeps start index 0). */
    int tile_row0, tile_rows, tile_col0, tile_cols;
    /* The node keeps its resolution as a double (ElevationMapping.hpp:314) and grid_map computes cell-centre
     * positions with it, while the CUDA side gets the float.  Used only for the positions emitted by
     * gem_export_visual_points / gem_harvest_scrolled_out; 0 = (double)resolution. */
    double grid_resolution;
} gem_config;

enum { GEM_SENSOR_LASER = 0, GEM_SENSOR_STRUCTURED_LIGHT = 1 };

/* Sensor noise model: laser = gpu.cu:410-411 (C_min_r, C_beam_a, C_beam_c);
 * structured light = StructuredLightSensorProcessor.cpp:129-139 (doubles), plus the depth
 * pass-through of its cleanPointCloud (:51-66). */
typedef struct gem_sensor_model {
    int type;
    float min_radius, beam_angle, beam_constant;
    double normal_factor_a, normal_factor_b, normal_factor_c, normal_factor_d, normal_factor_e;
    double lateral_factor;
    /* structured light only: cleanPointCloud's pcl::PassThrough on the sensor-frame z
     * (StructuredLightSensorProcessor.cpp:51-66, realsense_d435.yaml 0.2 / 3.25; the node's defaults are
     * DBL_MIN / DBL_MAX, :39-40).  PCL converts the limits to float and drops a point when it is not finite or
     * z < min || z > max.  Always applied for GEM_SENSOR_STRUCTURED_LIGHT by the fused add calls (a dropped point
     * is a rejected point: the order of the remaining ones is unchanged); ignored for the laser model, whose
     * cleanPointCloud only removes non-finite points (LaserSensorProcessor.cpp:50-59) -- those never pass the
     * height window of gpu.cu:397 anyway. */
    double cutoff_min_depth, cutoff_max_depth;
} gem_sensor_model;

/* Per-frame constants = the by-value arguments of Process_points (gpu.cu:1085), derived by
 * SensorProcessorBase::GPUPointCloudprocess / readcomputerparam (SPB.cpp:171-206,270-290).
 * Matrices are row-major. */
typedef struct gem_frame {
    float T[16];                 /* map <- sensor (Eigen::Matrix4f transform)             */
    float sensor_jacobian[3];    /* row 3 of R_map<-sensor (SPB.cpp:275)                  */
    float rotation_variance[9];  /* Sigma_q, all zero in GEM (SPB.cpp:202-204)            */
    float C_SB_transpose[9];     /* SPB.cpp:283                                           */
    float P_mul_C_BM_transpose[3]; /* SPB.cpp:282                                         */
    float B_r_BS_skew[9];        /* SPB.cpp:284                                           */
    double rel_lower, rel_upper; /* height window, double compare (gpu.cu:397)            */
    gem_sensor_model sensor;
} gem_frame;

typedef struct gem_stats {
    long long points_in;      /* points offered by the last add/process call              */
    long long points_binned;  /* accepted by the filters AND inside the grid              */
    long long cells_touched;  /* distinct cells updated by the last add/fuse call         */
    int max_points_per_cell;  /* longest per-cell list of the last call (exact above 8)       */
} gem_stats;

/* layer ids for gem_get_layer / gem_set_layer */
enum {
    GEM_LAYER_ELEVATION = 0, GEM_LAYER_VARIANCE = 1, GEM_LAYER_INTENSITY = 2,
    GEM_LAYER_COLOR_R = 3, GEM_LAYER_COLOR_G = 4, GEM_LAYER_COLOR_B = 5,
    GEM_LAYER_TRAVER = 6, GEM_LAYER_LOWEST = 7, GEM_LAYER_ROUGH = 8, GEM_LAYER_SLOPE = 9
};

int gem_version(void);
const char *gem_last_error(const gem_map *m); /* m may be NULL: last create error */

/* Init_GPU_elevationmap (gpu.cu:940-994): allocate layers + scratch, init sentinels. */
int gem_create(const gem_config *cfg, gem_map **out);
int gem_destroy(gem_map *m);
int gem_sync(gem_map *m); /* wait for the handle's stream */
/* the cudaStream_t all work of this handle is ordered on (record your own events there) */
void *gem_get_stream(gem_map *m);
/* enqueue everything the pipelined add calls have deferred (the fold of the last gem_add_points_stream /
 * _multi / _host_async call) on the handle's stream without waiting for it; gem_sync and every call that
 * reads or changes the map do this implicitly */
int gem_flush(gem_map *m);
/* debug: %globaltimer marks (ns) of the add kernels' phases, accumulated since the last call (min of the starts,
 * max of the marks): [0] k_bin start, [1] ranks drawn, [2] slots reserved, [3] pointers published, [4] records
 * stored; [8] k_fold start, [9] long + large lists done, [10] short lists done, [11] longest lists loaded,
 * [12] longest lists folded.  enable != 0 (re)arms the marks, 0 disarms them; out may be NULL. */
int gem_debug_stamps(gem_map *m, int enable, unsigned long long out[16]);

/* Move (gpu.cu:1004-1083): scroll the circular buffer to follow pos[0..1], record
 * pos[2] as sensorZatLowestScan.  Outputs may be NULL. */
int gem_move(gem_map *m, const float pos[3], float centre_out[2], int start_out[2],
             float aligned_shift_out[2]);

/* ---- fused hot path: Process_points + Fuse with device-resident intermediates --------
 * xyzi: n x float4 {x, y, z, intensity} in the sensor frame; rgba: n x uchar4 {r,g,b,-}
 * or NULL (colour path off).  NOTE (reference behaviour, gpu.cu:488): a cell takes a point's
 * intensity AND colour only when R, G, B and intensity are ALL non-zero, so with rgba == NULL
 * (or for points whose colour has a zero channel) the intensity layer is not written either --
 * LiDAR-only clouds that want the intensity layer must pass a non-zero dummy colour.  Equivalent to SensorProcessorBase::process +
 * ElevationMapping::processpoints (ElevationMapping.cpp:254-283). */
int gem_add_points(gem_map *m, const void *xyzi_device, const void *rgba_device, int n,
                   const gem_frame *frame);
int gem_add_points_host(gem_map *m, const void *xyzi_host, const void *rgba_host, int n,
                        const gem_frame *frame);
/* Stream mode: same result as gem_add_points, but consecutive calls are software-pipelined: call
 * i+1 issues ONE two-node CUDA graph {fold of frame i || bin of frame i+1} on the handle's
 * stream (the fold is mostly a serial tail, the bin kernel is throughput work; per-cell scratch
 * is double-buffered inside the 32-byte cell record).  The fold of the last frame is issued by
 * the next call of any kind that reads or changes the map, by gem_flush or by gem_sync.
 * Contract: the device inputs are read by the bin kernel of this call AND (intensities) by the
 * deferred fold: they must stay valid until two further stream calls have COMPLETED on the
 * stream, or until gem_sync.  n <= max_points.  GEM_B200_PIPE=stream selects two streams +
 * events instead of the graph, GEM_B200_PIPE=off makes this call identical to gem_add_points. */
int gem_add_points_stream(gem_map *m, const void *xyzi_device, const void *rgba_device, int n,
                          const gem_frame *frame);
/* Several clouds in one launch (multi-sensor rigs, BASELINE config 5): the device buffers hold
 * n_segments clouds back to back, cloud s = points [offsets[s], offsets[s+1]) with its own
 * per-frame constants frames[s] (both host arrays, offsets has n_segments+1 entries,
 * n_segments <= 64).  Equivalent to n_segments gem_add_points calls in order (the per-cell
 * order is the global point index), except that `lowest` is updated once for the whole call. */
int gem_add_points_multi(gem_map *m, const void *xyzi_device, const void *rgba_device, int n_segments,
                         const int *offsets, const gem_frame *frames);
/* Pipelined host ingest: like gem_add_points_host but returns without waiting.  The copy runs on
 * a second stream into one of three staging buffers, so frame i+1's H2D overlaps frame i's kernels
 * (which run pipelined like gem_add_points_stream); every call also reads back the counters of the
 * newest frame whose fold has been issued (gem_get_stats gives the last frame's after a drain).  The
 * host buffers must be pinned (gem_host_alloc / cudaHostRegister) and stay untouched until the call
 * after next on this handle, or gem_sync().  n must not exceed max_points. */
int gem_add_points_host_async(gem_map *m, const void *xyzi_pinned, const void *rgba_pinned, int n,
                              const gem_frame *frame);
/* PCL record ingest: n x 32-byte PointXYZRGBICT {x,y,z,pad, b,g,r,a, covariance, intensity,
 * travers} (PointXYZRGBICT.hpp:26-48), host memory, e.g. cloud->points.data(). */
int gem_add_cloud_pcl_host(gem_map *m, const void *points32_host, int n, const gem_frame *frame);

/* ---- unfused reference calls (host arrays, exactly the reference argument meaning) ----
 * Process_points (gpu.cu:1085-1144): outputs key (storage index or -1), var, x_ts, y_ts,
 * z_ts; rejected points give -1 in every output (gpu.cu:443-450).  Also updates `lowest`. */
int gem_process_points(gem_map *m, int *map_index, const float *x, const float *y,
                       const float *z, float *var, float *x_ts, float *y_ts, float *z_ts,
                       int n, const gem_frame *frame);
/* Fuse (gpu.cu:1154-1193) */
int gem_fuse(gem_map *m, int n, const int *index, const int *R, const int *G, const int *B,
             const float *intensity, const float *height, const float *var);

/* Mapvar_update (gpu.cu:1146-1152) */
int gem_var_update(gem_map *m, float var_update);

/* Map_feature (gpu.cu:1256-1302): computes traversability into the map and copies 9
 * row-major storage-indexed layers to host arrays (any may be NULL). */
int gem_map_feature(gem_map *m, float *elevation, float *var, int *R, int *G, int *B,
                    float *rough, float *slope, float *traver, float *intensity);
/* same computation, no host copies (results stay in the device layers) */
int gem_compute_features(gem_map *m);

/* Raytracing (gpu.cu:1304-1318): visibility clean-up + reset of `lowest` */
int gem_raytracing(gem_map *m);

/* Map_optmove (gpu.cu:1215-1233), Map_closeloop (gpu.cu:1235-1254) */
int gem_opt_move(gem_map *m, const float opt_p[2], float height_update, float aligned_out[2]);
int gem_closeloop(gem_map *m, const float update_position[2], float height_update);

/* ---- colourisation of the cloud from the camera image (ElevationMapping.cpp:331-381), the step
 * right before the fusion path.  T_camera: row-major 3x4 "T.camera", T_lidar: row-major 4x4 "T.lidar"
 * (kitti_intrinsic.yaml / yq_intrinsic.yaml), bgr: device BGR8 image.  Writes rgba_out (r,g,b,255 or
 * 0,0,0,0) and zeroes the intensity of points that do not project into the image, exactly like the
 * reference loop; the reference's debug circle drawing into the image (:372) is not reproduced. */
int gem_colourise_points(gem_map *m, void *xyzi_device, int n, const double T_camera[12], const double T_lidar[16],
                         const unsigned char *bgr_device, int width, int height, int row_stride_bytes,
                         void *rgba_out_device);

/* ---- write-back replacing ElevationMap::show's L*L CPU loop (ElevationMap.cpp:85-149) --
 * Emits 9 float32 layers {elevation, variance, rough, slope, traver, color_r, color_g,
 * color_b, intensity} (ElevationMap.cpp:44) in grid_map::Matrix layout: COLUMN-major,
 * storage indexed, NaN where the reference leaves the cell cleared (elevation == -10 or
 * traver == -10 or traver is NaN, ElevationMap.cpp:101).  host_layers[k] may be NULL. */
int gem_export_layers(gem_map *m, float *host_layers[9]);
/* the same in two halves: _begin returns once the copies are under way (pinned host memory!), _end waits for them.
 * Calls that do not change the exported state may be made in between -- the node's next call after show() is
 * Raytracing (ElevationMapping.cpp:404-421) -- so the 36 * L^2 bytes cross PCIe under the ray clean-up. */
int gem_export_layers_begin(gem_map *m, float *host_layers[9]);
int gem_export_layers_end(gem_map *m);

/* The other two products of ElevationMap::show, from the same pass's state (call after gem_compute_features):
 * gem_export_orthomosaic: the bgr8 image of ElevationMap.cpp:87,123-125, L x L x 3 bytes row-major; a shown cell
 *   (ix, iy) is drawn at pixel ((ix + L - start_x) % L, (iy + L - start_y) % L), everything else is black.
 * gem_export_visual_points: the pcl::PointXYZRGB cloud of ElevationMap.cpp:112-121, one point per shown cell in
 *   GridMapIterator order (linear index ix + iy*L): xyz (3 floats/point: grid_map cell-centre position, elevation)
 *   and rgb (3 bytes/point).  *count_out = number of shown cells; min(count, capacity) points are written. */
int gem_export_orthomosaic(gem_map *m, unsigned char *host_bgr);
int gem_export_visual_points(gem_map *m, float *host_xyz, unsigned char *host_rgb, int capacity, int *count_out);

/* ---- scroll-out capture into the submap store (ElevationMapping.cpp:609-765, SURVEY 8f row 3) ----
 * gem_snapshot_shown: prevMap_ = map_.visualMap_ (:422) on the device: the shown state of this frame (after
 *   gem_compute_features, before gem_raytracing) with its geometry; ~20 B/cell device-to-device, no host copy.
 * gem_harvest_scrolled_out: the "L-shape" loop of :716-765 over that snapshot: every cell with traver >= 0 whose
 *   centre lies outside the window current_xy +- length*resolution/2 on the side(s) selected by the signs of
 *   shift_xy (both as returned by the gem_move that followed the snapshot) becomes one 32-byte PointXYZRGBICT
 *   record {x, y, elevation, 1 | bgra, variance, intensity, traver} (:748-759; the same values GridPointData
 *   stores, :736-737), in GridMapIterator order.  *count_out = number of such cells; min(count, capacity) written.
 *   The host-side gate of :716 (|shift| >= resolution, init / jump flags) stays with the caller. */
int gem_snapshot_shown(gem_map *m);
int gem_harvest_scrolled_out(gem_map *m, const float current_xy[2], const float shift_xy[2], void *host_points32,
                             int capacity, int *count_out);

/* ---- local submaps on the device (ElevationMapping.cpp:609-767, :1124-1140, :1198-1226) ----
 * gem_export_grid_cloud: gridMaptoPointCloud (:1198-1226).  source GEM_GRID_SHOWN reads the state show() publishes
 *   (visualMap_: the current map after gem_compute_features), GEM_GRID_SNAPSHOT what gem_snapshot_shown kept (prevMap_),
 *   with that snapshot's geometry; an error without a snapshot.  A cell is taken when elevation != -10 && traver != -10
 *   && traver is not NaN (:1208) -- on show()'s output these are exactly the shown cells; unlike the harvest, cells
 *   with a negative traversability other than -10 are taken.  One 32-byte PointXYZRGBICT record per cell, GridMapIterator
 *   order, the layout of gem_harvest_scrolled_out (w = 1, a = 0xff), into caller-owned device memory.
 *   *count_out = number of cells taken; min(count, capacity) records are written.  Host-synchronous.
 * gem_harvest_to_local_map: the harvest of gem_harvest_scrolled_out (same cells, records and order), upserted into a
 *   store owned by the handle, keyed by the bit patterns of the record's float (x, y) (GridPointEqual): a key already
 *   present is replaced, across calls and within one call (the later cell in GridMapIterator order wins), as the
 *   find / erase / insert of :740-747 does.  host_points32 may be NULL; when given, min(count, capacity) harvested
 *   records are also copied there (for visualCloud_, :750-760).  *count_out = records harvested by this call.
 * gem_local_map_take: localHashtoPointCloud (:1124-1140): the store's records into device memory, then the store is
 *   empty.  Order DEFINED: all harvests since the last take / clear concatenated, only the last occurrence of each key
 *   kept (an insertion-ordered map with erase-then-insert).  Fields DEFINED: intensity = the harvested value, w = 1,
 *   a = 0xff.  If capacity < count nothing is written and the store is unchanged; *count_out is the size needed
 *   (capacity 0 = size query).
 * gem_local_map_clear: empty the store (the init branch, :697-698).
 * gem_local_map_reserve: make room for `records` log records now.  The store is otherwise allocated on first use and
 *   grows by doubling (from 1024 records) when a harvest needs more; once large enough, no call allocates.  A failed
 *   growth returns GEM_ERR_NOMEM and leaves the store as it was.  Freed by gem_destroy.
 * Tiled handles refuse all of these.  The store keeps every harvested record until the next take / clear (an append
 * log, 32 B per record, plus an index of 24-48 B per record of capacity). */
enum { GEM_GRID_SHOWN = 0, GEM_GRID_SNAPSHOT = 1 };
int gem_export_grid_cloud(gem_map *m, int source, void *points32_device, int capacity, int *count_out);
int gem_harvest_to_local_map(gem_map *m, const float current_xy[2], const float shift_xy[2], void *host_points32,
                             int capacity, int *count_out);
int gem_local_map_take(gem_map *m, void *points32_device, int capacity, int *count_out);
int gem_local_map_clear(gem_map *m);
int gem_local_map_reserve(gem_map *m, int records);

/* ---- the global-map filter of composingGlobalMap (ElevationMapping.cpp:482-514, :1146-1174; DESIGN.md f6) ----
 * gem_grid_cloud_split: PCL's StatisticalOutlierRemoval (setMeanK(mean_k), setStddevMulThresh(stddev_mul); :1152-1156)
 *   over the grid cloud gem_export_grid_cloud(source) defines (same points, records and order), then the survivors
 *   split by (double)travers > travers_threshold into the road cloud and the rest into the obstacle cloud (:1161-1170).
 *   Unpinned: restated from PCL 1.8 applyFilterIndices with an exact FLANN search.  Per point with finite x, y, z the
 *   mean distance to its mean_k nearest other points (float d2 in FLANN's order, double sqrt and sum); 0 otherwise.
 *   mean / stddev / threshold and the removal test (distance > threshold) are PCL's, the sums sequential in point order.
 *   With at most mean_k finite points every point is kept, the distances and statistics are NaN and valid = 0.
 *   road / obstacle receive min(count, capacity) 32-byte PointXYZRGBICT records each, in grid-cloud order; the counts
 *   are reported in *out.  mean_distance_device (may be NULL with distance_capacity 0) receives min(points, capacity)
 *   per-point distances in grid-cloud order.  mean_k in [1, 64].  Host-synchronous; the map is not modified.  Tiled
 *   handles and a missing snapshot are errors.  The two octrees are built from road and obstacle with
 *   gem_color_octree. */
typedef struct gem_grid_split {
    int points, valid;            /* grid-cloud points; points with a computed mean distance */
    int road, obstacle;           /* records each output needs (min(count, capacity) are written) */
    double mean, stddev, threshold;
} gem_grid_split;
int gem_grid_cloud_split(gem_map *m, int source, int mean_k, double stddev_mul, double travers_threshold,
                         void *road_points32_device, int road_capacity,
                         void *obstacle_points32_device, int obstacle_capacity,
                         float *mean_distance_device, int distance_capacity,
                         gem_grid_split *out);

/* ---- the global-map octrees of composingGlobalMap (ElevationMapping.cpp:1146-1174; DESIGN.md f7) ----
 * gem_color_octree: the octomap::ColorOcTree pointCloudtoOctomap builds at `resolution` from n 32-byte PointXYZRGBICT
 *   records in device memory (updateNode(point, true) then integrateNodeColor(x, y, z, r, g, b) per point in cloud
 *   order, r, g, b = bytes 2, 1, 0 of the bgra word; then updateInnerOccupancy), from an empty tree.  The result is the
 *   byte stream ColorOcTree::writeData produces, i.e. octomap_msgs::Octomap::data as fullMapToMsg fills it (the caller
 *   sets id "ColorOcTree", binary false and the resolution); 8 bytes per node, 0 for an empty tree.  Unpinned:
 *   restated from octomap 1.9 with default parameters (items O1-O6 of DESIGN.md f7).  The stream stays in the
 *   handle until the next build; *info receives its size and counts.  Host-synchronous; the map is not modified.
 *   n < 0, NULL points with n > 0, a non-finite or non-positive resolution and tiled handles are errors, which leave
 *   the last stream as it was.
 * gem_color_octree_read: copies the last built stream to `out` (host or device memory).  An error, writing nothing,
 *   before any build or when capacity < bytes. */
typedef struct gem_octree {
    long long bytes;              /* stream size: 8 * nodes */
    int nodes, leaves;            /* leaves: childless nodes, pruned ones included */
    int inserted, skipped;        /* points inserted / skipped because a key is out of range or non-finite */
} gem_octree;
int gem_color_octree(gem_map *m, const void *points32_device, int n, double resolution, gem_octree *info);
int gem_color_octree_read(gem_map *m, void *out, long long capacity);

/* ---- navigation costmaps: the costmap_2d layers of GEM's layers/ package (DESIGN.md f8) ----
 * ElevationMapLayer (layers/src/elevationMap_layer.cpp:42-87) and PointMapLayer (layers/src/pointMap_layer.cpp:45-100), with
 * the costmap_2d functions they use restated from navigation 1.14 (unpinned):
 *   - costs: FREE_SPACE 0, LETHAL_OBSTACLE 254, NO_INFORMATION 255;
 *   - a grid is caller-owned device memory uint8[size_y][size_x], cell (mx, my) at my * size_x + mx (getIndex);
 *   - worldToMap(wx, wy), in double: false if wx < origin_x || wy < origin_y, else mx = (int)((wx - origin_x) / resolution)
 *     (same for my), accepted iff mx < size_x && my < size_y.  DEFINED: a non-finite coordinate is rejected, and so is a
 *     quotient >= 2^31;
 *   - touch: min_x = min(min_x, wx) etc. over every element written, not only over the cells that keep its value.  A zero
 *     bound is reported as +0.
 * gem_costmap_mark_map: ElevationMapLayer::updateBounds (:56-84) over the grid_map show() publishes, source GEM_GRID_SHOWN
 *   (the live map after gem_compute_features) or GEM_GRID_SNAPSHOT.  Per cell in GridMapIterator order (ix + iy * L): the
 *   value is show()'s traver (the feature output where the cell is shown, NaN elsewhere), the position the grid_map cell
 *   centre in double (grid_resolution), the cost LETHAL if (double)value < travers_thresh, else FREE.  mark_unknown = 1 is
 *   the reference (NaN compares false: a cleared cell is FREE); mark_unknown = 0 writes nothing for cleared cells.  Tiled
 *   handles and a missing snapshot are errors.
 * gem_costmap_mark_points: PointMapLayer::updateBounds (:54-81) over n 32-byte PointXYZRGBICT records in device memory, in
 *   order: (double)x, (double)y through worldToMap, cost FREE if (double)travers > travers_thresh, else LETHAL (NaN and
 *   equality give LETHAL).  n = 0 is valid.
 *   In both mark calls the LAST element in order wins a costmap cell several elements fall into; cells nothing writes
 *   keep their value (the layer grid persists).  *out receives the elements written and the touch bounds (+inf / -inf
 *   when none was).  Host-synchronous.  They use a handle-owned scratch of 4 bytes per costmap cell, grown on demand (a
 *   failed growth is GEM_ERR_NOMEM and writes nothing).
 * gem_costmap_update_origin: Costmap2D::updateOrigin in place: cell_ox = (int)((new_origin_x - origin_x) / resolution)
 *   (truncating toward zero; same for y); nothing happens when both are 0; else new cell n holds old cell n + cell_ox (and
 *   n + cell_oy) when that is inside the grid, else `fill`, and the origin becomes origin_x + cell_ox * resolution, written
 *   to *w.  A rolling layer calls it with robot - getSizeInMetersX() / 2, getSizeInMetersX() = (size_x - 1 + 0.5) *
 *   resolution.  fill is the layer's default_value_: FREE_SPACE for the elevation layer; NO_INFORMATION for the point
 *   layer (DEFINED: the reference never sets it).  DEFINED: a shift that is not finite or does not fit an int is an error.
 * gem_costmap_combine: over the rect [min_i, max_i) x [min_j, max_j), clamped to the grid (an empty rect does nothing),
 *   GEM_COSTMAP_MAX = CostmapLayer::updateWithMax (a NO_INFORMATION layer cell is skipped; otherwise written when the
 *   master is NO_INFORMATION or less than the layer), GEM_COSTMAP_OVERWRITE = PointMapLayer::updateCosts (:86-100; every
 *   layer cell that is not NO_INFORMATION is copied).  layer and master are grids of size_x * size_y.
 * update_origin and combine are asynchronous on the handle's stream and, like mark_points, work on any handle.  No call
 * modifies the map.  Every call rejects a bad window (size <= 0, size_x * size_y >= 2^31, a resolution that is <= 0 or not
 * finite); a rejected call writes nothing.  Out of scope: footprint clearing (footprint_clearing_enabled false),
 * InflationLayer (inflation_radius 0 in GEM's configs), publishing, and the elevation_map_available_ subscription gate. */
enum { GEM_COST_FREE = 0, GEM_COST_LETHAL = 254, GEM_COST_UNKNOWN = 255 };
enum { GEM_COSTMAP_MAX = 0, GEM_COSTMAP_OVERWRITE = 1 };
typedef struct gem_costmap_window {
    double origin_x, origin_y, resolution;
    int size_x, size_y;
} gem_costmap_window;
typedef struct gem_costmap_marks {
    long long marked, lethal;          /* elements written (touch calls), of which LETHAL */
    double min_x, min_y, max_x, max_y; /* touch bounds; +inf / -inf when marked == 0 */
} gem_costmap_marks;
int gem_costmap_mark_map(gem_map *m, int source, const gem_costmap_window *w, double travers_thresh, int mark_unknown,
                         unsigned char *cost_device, gem_costmap_marks *out);
int gem_costmap_mark_points(gem_map *m, const void *points32_device, int n, const gem_costmap_window *w, double travers_thresh,
                            unsigned char *cost_device, gem_costmap_marks *out);
int gem_costmap_update_origin(gem_map *m, gem_costmap_window *w, double new_origin_x, double new_origin_y, unsigned char fill,
                              unsigned char *cost_device);
int gem_costmap_combine(gem_map *m, int mode, const unsigned char *layer_device, unsigned char *master_device, int size_x, int size_y,
                        int min_i, int min_j, int max_i, int max_j);

/* ---- the VoxelGrid pre-filter of GEM's demo launches (filter.launch, filter_kitti.launch; DESIGN.md f9) ----
 * gem_voxel_grid: pcl_ros's VoxelGrid nodelet, i.e. pcl::VoxelGrid<pcl::PCLPointCloud2> of PCL 1.8 with downsample_all_data_
 *   true, over n x float4 {x, y, z, intensity} in device memory (the layout the add calls take).  Unpinned: restated, PCL
 *   is not available.
 *   V1 leaf: float leaf_size[3], inv[a] = 1.0f / leaf_size[a] in float; a leaf that is not finite or is <= 0 is an error.
 *   V2 used points: with a field selected (x, y, z or intensity), its float value v is cut when (double)v > limit_max ||
 *      (double)v < limit_min (limit_negative = 0), or when (double)v < limit_max && (double)v > limit_min (limit_negative = 1);
 *      a NaN v passes.  A point that passes (every point without a field) is then cut when x, y or z is not finite; is_dense
 *      is not read.
 *   V3 bounds (getMinMax3D): the same two tests against (float)limit_min, (float)limit_max compared in float; min_p / max_p
 *      are the per-axis float min / max over the survivors, from FLT_MAX / -FLT_MAX.  Every V2 survivor survives V3.
 *   V4 overflow: d[a] = (int64)((max_p[a] - min_p[a]) * inv[a]) + 1, the product in float; if d[0] d[1] d[2] > INT32_MAX the
 *      output is the input unchanged (all n points in order, bit for bit) and passthrough = 1.  DEFINED: a product that is
 *      not finite, or a quotient >= 2^62, also counts as overflow (PCL's cast is undefined there).
 *   V5 no V3 survivor (n = 0 included): count 0.  DEFINED: PCL casts -inf to int64 there.
 *   V6 min_b[a] = floor(min_p[a] * inv[a]), max_b[a] likewise, ijk[a] = floor(p[a] * inv[a]) - min_b[a], idx = ijk0 + ijk1 div0
 *      + ijk2 div0 div1 with div[a] = max_b[a] - min_b[a] + 1; output in ascending idx, i.e. lexicographic in (ijk2, ijk1,
 *      ijk0).  The float and the double floor are both exact, so the overload changes nothing.  DEFINED: where div0 div1
 *      div2 exceeds 2^31 although V4 passed (PCL's int idx overflows) the order is still lexicographic in (ijk2, ijk1, ijk0).
 *   V7 DEFINED: inside a voxel, ascending input index (PCL's std::sort is not stable).
 *   V8 centroid: the four components start at +0.0f, c += p in float in V7 order, then c /= (float)count, one IEEE division
 *      per component.  Intensity is averaged like x, y, z (a lone -0.0 comes out +0.0); no other field is carried.
 *   V9 min(count, capacity) float4 go to out_xyzi_device; *info always receives count (output points), used (V2 survivors)
 *      and passthrough.  capacity = 0 is a size query.
 *   Host-synchronous; works on any handle, tiled ones included; neither reads nor modifies the map and does not issue the
 *   deferred fold.  A bad leaf, n < 0, NULL points with n > 0, capacity < 0, NULL out with capacity > 0, a bad field id
 *   and overlapping input and output ranges are GEM_ERR_INVALID (chain calls, as the KITTI launch does, through two
 *   buffers).  Uses a handle-owned scratch of about 32 bytes per input point, grown on demand: a failed growth is
 *   GEM_ERR_NOMEM.  A rejected call writes nothing.  min_points_per_voxel (0 in GEM's launches) is not exposed. */
enum { GEM_VOXEL_FIELD_NONE = -1, GEM_VOXEL_FIELD_X = 0, GEM_VOXEL_FIELD_Y = 1, GEM_VOXEL_FIELD_Z = 2, GEM_VOXEL_FIELD_INTENSITY = 3 };
typedef struct gem_voxel_grid_params {
    float leaf_size[3];
    int field;                    /* GEM_VOXEL_FIELD_*                                       */
    double limit_min, limit_max;  /* the nodelet's filter_limit_min / _max                   */
    int limit_negative;           /* the nodelet's filter_limit_negative                     */
} gem_voxel_grid_params;
typedef struct gem_voxel_grid_info {
    int count, used, passthrough; /* output points, V2 survivors, V4 taken                   */
} gem_voxel_grid_info;
int gem_voxel_grid(gem_map *m, const void *xyzi_device, int n, const gem_voxel_grid_params *p,
                   void *out_xyzi_device, int capacity, gem_voxel_grid_info *info);

/* ---- the MLS densification of GEM's dense_mapping signal (pointcloudinterpolation, ElevationMapping.cpp:1072-1118;
 *      DESIGN.md f10) ----
 * gem_mls_upsample: pcl::MovingLeastSquares<PointXYZRGB, PointXYZRGB>::process of PCL 1.7.2 (performProcessing /
 *   computeMLSPointNormal, KdTreeFLANN radius search, single-threaded) over n 32-byte PointXYZRGBICT records in device
 *   memory (the layout of gem_local_map_take).  The output holds only the points MLS produces (mls.process's cloud); the
 *   node appends them to the submap (*input += dense).  Unpinned: restated, PCL is not available.  DEFINED: fixed here
 *   where the reference leaves it open.
 *   M1 only x, y, z and the bgra word of a record are read.  DEFINED: a record whose x, y or z is not finite is nobody's
 *      neighbour and produces nothing; it counts in skipped.
 *   M2 neighbours: d2 = ((dx dx) + dy dy) + dz dz in float; j is a neighbour iff d2 <= (float)(r r) (DEFINED inclusive),
 *      the query included, sorted by ascending d2, ties by ascending index (DEFINED), no cap; with fewer than 3
 *      neighbours the point produces nothing.
 *   M3 plane, in double and neighbour order: centroid (sequential sums, then / n), the non-normalised covariance in PCL's
 *      update order, eigen33's smallest eigenvector (scaling, computeRoots with the computeRoots2 fallback, three row
 *      cross products, the largest squared norm in PCL's if-chain order), d = -(n . centroid) with the dot
 *      (a0b0 + a2b2) + (a1b1 + a3b3), point = q - (q . n + d) n.  3-vector dots left to right (DEFINED).  atan2, sin, cos
 *      and exp are the library's own double functions (gem_mathd.h), within 2 ulp of glibc's.
 *   M4 fit when polynomial_fit and n >= nr_coeff = (order + 1)(order + 2) / 2: de = p_j - point, d2f = (float)(de . de),
 *      w = exp(-d2f / sqr_gauss_param), v_axis = n.unitOrthogonal(), u_axis = n x v_axis, (u, v, f) = de . (u_axis, v_axis,
 *      n), monomials u^a v^b with the u power outer; A(a,b) = sum ((P(a) w) P(b)) (a >= b), rhs(a) = sum ((P(a) w) f),
 *      sequential in neighbour order (DEFINED); left-looking Cholesky, forward and back substitution (DEFINED orders,
 *      DESIGN.md f10).  DEFINED: a pivot that is not finite or not > 0, or a non-finite c0, fails the fit.  The Darboux
 *      axes are set only when the fit is attempted (as in 1.7.2); otherwise they are zero.
 *   M5 GEM_MLS_NONE: one output per processed point, point + c0 n when fitted, else point.
 *   M6 GEM_MLS_RANDOM_UNIFORM_DENSITY: k = (int)floor(point_density / 2.0 / n); k <= 0: M5's output; else k samples, u
 *      then v drawn as floats in [-r/2, r/2), again while u u + v v > r r / 4 (double); sample = point + u u_axis +
 *      v v_axis (+ height(u, v) n when fitted).  DEFINED generator: draw j of input point i is splitmix64(seed ^ (i << 32)
 *      ^ j), the float lo + (float)(x >> 40) 2^-24 (hi - lo) in float, hi = (float)(r / 2), lo = -hi; a rejected pair
 *      consumes its two draws.  (The reference seeds boost::mt19937 with time(0), so it differs from run to run.)
 *   M7 records {(float)x, (float)y, (float)z, 1, the query's b g r with a = 0xff, the query's covariance, intensity and
 *      travers} (DEFINED: the alpha and the last three, uninitialised in the reference), in input order, samples in
 *      draw order.
 *   M8 info: count (output records; min(count, capacity) are written), processed (n >= 3), fitted, skipped (n < 3 or
 *      non-finite), max_neighbours (the longest list).
 *   capacity = 0 is a size query: it stops before the fits and reports fitted = -1, the other fields as a full call.
 *   Host-synchronous (two synchronisations); works on any handle; neither reads nor modifies the map.  Errors, which
 *   return GEM_ERR_INVALID and write nothing: overlapping input and output, n < 0, capacity < 0, NULL pointers with a
 *   non-zero size, a radius or Gauss parameter that is not finite or not > 0, an order outside 1..5, an unknown upsampling
 *   id, point_density < 0.  Scratch (about 90 bytes per input point, plus the sort slices of lists longer than 512) is
 *   handle-owned and grown on demand before anything is written: a failed growth is GEM_ERR_NOMEM.  sqr_gauss_param and
 *   search_radius are separate, as in PCL (GEM sets sqr_gauss_param = search_radius^2). */
enum { GEM_MLS_NONE = 0, GEM_MLS_RANDOM_UNIFORM_DENSITY = 1 };
typedef struct gem_mls_params {
    double search_radius;        /* 0.5 in GEM                                   */
    double sqr_gauss_param;      /* 0.25 = search_radius^2                        */
    int polynomial_fit;          /* 1                                             */
    int order;                   /* 5; 1..5 accepted                              */
    int upsampling;              /* GEM_MLS_*                                     */
    int point_density;           /* desired_num_points_in_radius, 1000 in GEM     */
    unsigned long long seed;     /* the random draws, item M6                     */
} gem_mls_params;
typedef struct gem_mls_info {
    long long count;             /* output records (min(count, capacity) written) */
    int processed, fitted, skipped, max_neighbours;
} gem_mls_info;
int gem_mls_upsample(gem_map *m, const void *points32_device, int n, const gem_mls_params *p,
                     void *out_points32_device, long long capacity, gem_mls_info *info);

/* raw layer access (row-major L*L, float or int32 for the colour ids) for tests and
 * checkpoint/restore (the dead G_get_mapinfo/G_set_mapinfo of gpu.cu:457-475). */
int gem_get_layer(gem_map *m, int layer, void *host_out);
int gem_set_layer(gem_map *m, int layer, const void *host_in);
int gem_get_state(gem_map *m, float centre[2], int start[2], float *sensor_z);
int gem_get_stats(gem_map *m, gem_stats *out);

/* ---- launch accounting and per-kernel device timing ------------------------------------
 * The library counts every kernel it launches.  With profiling enabled each launch is also
 * bracketed by CUDA events on the handle's stream (costs ~2 us per launch: use a separate
 * pass, not the timed one) and the pipelined add calls fall back to the serial schedule
 * (bin, then fold, nothing overlapped), so the per-kernel durations are uncontended.
 * gem_profile_read synchronises the stream. */
enum {
    GEM_PROF_BIN = 0,       /* k_bin: transform + bin + record store */
    GEM_PROF_FOLD_LONG = 1, /* k_fold_long: the cells with more than 40 records of the call */
    GEM_PROF_UNUSED = 2,
    GEM_PROF_FOLD = 3,      /* k_fold: all other cells */
    GEM_PROF_CLEAR = 4, GEM_PROF_FEATURES = 5, GEM_PROF_RAYTRACE = 6, GEM_PROF_OTHER = 7,
    GEM_PROF_ROUTE = 8, /* tiled maps: the routing kernel */
    GEM_PROF_CLASSES = 9
};
typedef struct gem_profile {
    long long launches;                  /* kernels launched since the last reset          */
    double ms[GEM_PROF_CLASSES];         /* summed device time per kernel class            */
    long long count[GEM_PROF_CLASSES];   /* timed launches per class                       */
} gem_profile;
int gem_profile_enable(gem_map *m, int on);
int gem_profile_read(gem_map *m, gem_profile *out, int reset);

/* self-test: compares the fold's shared-reciprocal division (div2_rn) with the IEEE `/` operator
 * on n pseudo-random operand triples; mismatches must come back 0.  fast_out = how many triples
 * took the fast path. */
int gem_selftest_division(gem_map *m, unsigned long long seed, unsigned long long n,
                          unsigned long long *mismatches_out, unsigned long long *fast_out);

/* pinned host memory helpers for callers that want async-capable staging */
int gem_host_alloc(void **out, unsigned long long bytes);
int gem_host_free(void *p);

/* ---- multi-GPU tiling helpers (SURVEY 8e) ---------------------------------------------
 * gem_route_points: transform n device points like gem_add_points but do not fuse; emit
 * routed records {key(global geographic linear index), h, var, rgba, intensity} = 20 B
 * stably bucketed by owning tile (owner = (gx / tile_rows) * tiles_per_row + gy / tile_cols)
 * into rec_out_device, and the per-owner counts into counts_out_device[n_owners].
 * bucket_stride == 0: buckets are packed back to back (split sizes come from the counts);
 * bucket_stride  > 0: bucket o starts at record o*bucket_stride and unused slots hold gkey = -1,
 * so a fixed-size all-to-all needs no host-side split sizes (no stream synchronisation).
 * gem_fuse_records: fold received records (any owner order, already in global order)
 * into this handle's tile. */
int gem_route_points(gem_map *m, const void *xyzi_device, const void *rgba_device, int n,
                     const gem_frame *frame, int tiles_r, int tiles_c, void *rec_out_device,
                     int *counts_out_device, int bucket_stride);
int gem_fuse_records(gem_map *m, const void *rec_device, int n);
/* ---- features / ray clean-up on tiled handles (SURVEY 8e: halo + replicated lowest) ---------------
 * gem_get_layer_device: dense rows*cols copy of one layer into device memory (float, or int32 for the
 *   colour ids; id 10 = the traversability output of the last feature pass), e.g. to cut halo strips.
 * gem_compute_features_tiled: Map_feature's kernel on a tile; padded_elevation_device is the tile's
 *   elevation with a 2-cell halo from the neighbouring tiles, (tile_rows+4) x (tile_cols+4) row-major,
 *   -10 outside the map.  Results equal the untiled map's, cell for cell.
 * gem_raytracing_tiled: Raytracing on a tile; global_lowest_device is the map-wide L x L lowest layer
 *   (every rank's tile of it gathered); resets the OWN tile's lowest to 10 afterwards. */
int gem_get_layer_device(gem_map *m, int layer, void *out_device);
int gem_compute_features_tiled(gem_map *m, const float *padded_elevation_device);
int gem_raytracing_tiled(gem_map *m, const float *global_lowest_device);

/* Peer-memory routing (no collective library on the data path): like gem_route_points with a bucket
 * stride, but every record is stored directly into the OWNING rank's receive buffer through a peer
 * mapping (NVLink/NVSwitch): rank r's records for owner o go to peer_recv[o] + r*bucket_stride, its
 * bucket size to ((int*)peer_counts[o])[r].  peer_recv / peer_counts: n_owners device addresses
 * valid on this handle's device (host arrays).  The caller synchronises the ranks (one barrier)
 * before folding with gem_fuse_records_counted. */
int gem_route_points_peer(gem_map *m, const void *xyzi_device, const void *rgba_device, int n,
                          const gem_frame *frame, int tiles_r, int tiles_c,
                          const unsigned long long *peer_recv, const unsigned long long *peer_counts,
                          int my_rank, int bucket_stride);
/* fold a receive buffer of n_sources buckets of bucket_stride slots, bucket s filled up to
 * src_counts_device[s] */
int gem_fuse_records_counted(gem_map *m, const void *rec_device, const int *src_counts_device, int n_sources,
                             int bucket_stride);

/* ---- loop-closure re-fusion of submaps (ElevationMapping::updateGlobalMap, ElevationMapping.cpp:773-905; SURVEY 8f row 4) ----
 * Submaps are arrays of 32-byte PointXYZRGBICT records in device memory (what gem_harvest_scrolled_out produces).
 * gem_transform_cloud: the rigid re-transform of :805 (pcl::transformPointCloud with T = optimised pose * old pose^-1,
 *   row-major 4 x 4; x' = t00 x + t01 y + t02 z + t03 evaluated left to right in float), in place.
 * gem_refuse_submaps: one pass of the pairwise loop :847-883 for the pair (new = the neighbour, old = submap i): both clouds
 *   are reduced to one point per cell (pointCloudtoHash :1180-1192: cell = (ceil(x / res) * res - res / 2, same for y) in
 *   double -> float, the FIRST point of a cell wins), every cell present in both whose OLD variance lies in (0, 1) gets the
 *   fused elevation / variance in both clouds together with the new cloud's colour, intensity and traversability, and both
 *   clouds come back compacted in place (x, y = the cell's position, w = 1; *n_new / *n_old updated; first-occurrence order).
 *   compat != 0 evaluates the fused values exactly as the reference's expression parses (:862-863: var_n^2 e_o + (var_o^2 e_n) /
 *   var_o^2 + var_n^2, and var_o^2 var_n^2 / var_o^2 + var_n^2), compat == 0 the weighting it was written for
 *   ((var_n^2 e_o + var_o^2 e_n) / (var_o^2 + var_n^2), var_o^2 var_n^2 / (var_o^2 + var_n^2)), all in double like pow().
 *   Definitions where the reference is implementation-defined (unordered_map iteration while erasing / inserting, uninitialised
 *   point fields): DESIGN.md "f4".  Host-synchronous.  The kd-tree neighbour selection of :821-838 stays with the caller
 *   (a handful of submap centres). */
int gem_transform_cloud(gem_map *m, void *points32_device, int n, const float T[16]);
int gem_refuse_submaps(gem_map *m, void *new_points32_device, int *n_new, void *old_points32_device, int *n_old, double resolution,
                       int compat, int *fused_out);

/* ---- tiled maps, peer path: one kernel routes AND exchanges (no collective library, no barrier kernel) ----------
 * The caller allocates, on every rank, four peer-accessible buffers (e.g. CUDA IPC / torch symmetric memory; the
 * library does no inter-process plumbing) and passes the addresses under which THIS device sees every rank's copy:
 *   recv_records   uint4 [5][world * cap]   {global geographic key, height, variance, rgb}
 *   recv_intensity float [5][world * cap]
 *   recv_counts    int   [5][world * cap / 256]
 *   flags          int   [world], zero-initialised before the first step
 * with cap = bucket_capacity rounded up to a multiple of 256 (>= the largest cloud any rank adds per step; world * cap
 * <= max_points).  gem_tiled_step(r) = transform rank r's cloud, store every in-grid point into the OWNING rank's
 * buffer over NVLink (slot = (r * cap / 256 + source block) * 256 + position in the block: deterministic, source
 * order), raise rank r's flag on every peer; then, once every peer's flag of this step is up, bin and fold what
 * arrived.  The result equals the single-GPU map of the rank-by-rank concatenated clouds bit for bit.  Steps are
 * pipelined like gem_add_points_stream: call j issues ONE graph {folds of step j-1 || route -> bin of step j}; the cloud
 * of a call is consumed by that call's graph, and the map contains a step one call later or after gem_flush / gem_sync /
 * any reading call (which issue what is outstanding).  Every rank must make the same sequence of gem_tiled_step calls (a
 * bin waits on the device for every peer's flag of its step).  GEM_B200_TILED_DEPTH=3 selects a three-deep schedule
 * {folds of step j-2 || bin of step j-1 || route of step j} (bit-identical, measured slower; it is what the five
 * buffers are sized for). */
typedef struct gem_tiled_peers {
    int tiles_r, tiles_c, my_rank, bucket_capacity;
    unsigned long long recv_records[64], recv_intensity[64], recv_counts[64], flags[64];
} gem_tiled_peers;
int gem_tiled_attach(gem_map *m, const gem_tiled_peers *peers);
int gem_tiled_step(gem_map *m, const void *xyzi_device, const void *rgba_device, int n, const gem_frame *frame);

#ifdef __cplusplus
}
#endif
#endif /* GEM_B200_H */
