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

enum { GEM_SENSOR_LASER = 0, GEM_SENSOR_STRUCTURED_LIGHT = 1, GEM_SENSOR_STEREO = 2, GEM_SENSOR_PERFECT = 3 };

/* Sensor noise model: laser = gpu.cu:410-411 (C_min_r, C_beam_a, C_beam_c);
 * structured light = StructuredLightSensorProcessor.cpp:129-139 (doubles), plus the depth
 * pass-through of its cleanPointCloud (:51-66);
 * stereo = StereoSensorProcessor.cpp:78-90 (doubles; PARITY UNPINNED, restated: the reference's CPU code needs
 * kindr and PCL).  With (x, y, z) the sensor-frame point, idx its index in the cloud the caller passes and
 * w = cloud_width (0: unorganised, one row), row = w ? idx / w : 0 and col = w ? idx % w : idx (getI / getJ,
 * :109-117; the library removes no points, so idx is the position removeNaNFromPointCloud records), and
 *     disp = dtd / (double)z                       dtd = depth_to_disparity_factor
 *     a    = dtd / (disp * disp)
 *     s    = ((p3 * disp) + p4) - (double)col      p1..p5 = stereo_p[0..4]
 *     r    = (double)(240 - row)                   the reference's hard-coded principal row
 *     vN   = (float)((a * a) * ((((p5 * disp) + p2) * sqrt(s * s + r * r)) + p1))
 *     vL   = (float)(l * l),  l = lateral_factor * (double)sqrtf((x * x + y * y) + z * z)
 * pow(v, 2) is DEFINED as v * v, rounded once.  vN and vL are variances (not deviations), fed to the same
 * height-variance expression as every model; z = +-0, subnormal or negative give what the expression gives
 * (inf, NaN, negative values), unclamped.  Its cleanPointCloud only removes non-finite points (:37-48);
 * perfect = PerfectSensorProcessor.cpp:84-101: vN = vL = 0.  Its readParameters skips the base class (:36-39),
 * so its height window is always +-inf: the helpers in gem_b200/elevation_map.hpp ignore ignore_points_* for it.
 * A type outside 0..3 or cloud_width < 0 makes every call that takes a frame return GEM_ERR_INVALID. */
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
    /* stereo only: p_1..p_5, depth_to_disparity_factor (StereoSensorProcessor.cpp:26-32; the node's defaults
     * are 0) and pointCloud->width of the organised cloud, 0 = unorganised (the stereo model reads
     * lateral_factor too) */
    double stereo_p[5];
    double depth_to_disparity_factor;
    int cloud_width;
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
 * stream, or until gem_sync.  n <= max_points. */
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
 * reference loop.  The bgr image is never written.  Which pixel a point's colour comes from is the handle's
 * colour lookup mode (gem_set_colour_lookup):
 *   GEM_COLOUR_LOOKUP_IMAGE (the default): every point reads its own pixel of the unmodified image.
 *   GEM_COLOUR_LOOKUP_NODE: the node's loop (DESIGN.md f19).  It takes the points in array order against a working copy
 *     of the image; an in-image point reads its working pixel (mx, my), then cv::circle(img, midPoint, 1, colour) (:370)
 *     paints that colour into whichever of (mx +- 1, my) and (mx, my +- 1) lie inside the image (no diagonals).  So a
 *     point's colour is the image pixel of the root of its chain of parents, parent(i) being the largest j < i in the
 *     image whose pixel is a 4-neighbour of i's.  Unpinned (restated: OpenCV is not available).  Runs on the handle's
 *     stream with device scratch that grows on demand (GEM_ERR_NOMEM, nothing written, when it cannot).
 * gem_set_colour_lookup: the mode of one handle, used by gem_colourise_points and the image path of
 *   gem_add_pointcloud2_host_async from the next call on.  Another value is GEM_ERR_INVALID and leaves the mode as it
 *   was.  Tiled handles are accepted (the lookup reads no map). */
enum { GEM_COLOUR_LOOKUP_IMAGE = 0, GEM_COLOUR_LOOKUP_NODE = 1 };
int gem_set_colour_lookup(gem_map *m, int mode);
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
 * finite); a rejected call writes nothing.  The plugins fed from their messages, with the elevation_map_available_
 * gate, are gem_grid_map_msg_parse / gem_costmap_mark_grid / gem_decode_pointcloud2_records (DESIGN.md f18).  InflationLayer
 * is gem_costmap_inflate (DESIGN.md f14); footprint clearing and publishing are gem_costmap_footprint and
 * gem_ros_costmap / gem_ros_footprint (DESIGN.md f17). */
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

/* ---- costmap_2d's InflationLayer::updateCosts on a master grid (GEM's global costmap; DESIGN.md f14) ----
 * Restated from navigation 1.14 (unpinned):
 *   I1 r = cellDistance(inflation_radius) = (unsigned)max(0.0, ceil(inflation_radius / resolution)); weight =
 *      cost_scaling_factor; r == 0 writes nothing.  DEFINED: r is capped at ceil(hypot(size_x, size_y)) + 1, beyond which
 *      every in-grid distance is within the radius and the result cannot change.  DEFINED: an r above GEM_INFLATE_MAX_CELLS
 *      (after the cap) is GEM_ERR_INVALID, because the host tables grow with r^2.
 *   I2 for 0 <= i, j <= r + 1: dist[i][j] = hypot(i, j); cost[i][j] = 254 when dist == 0, 253 when dist * resolution <=
 *      inscribed_radius, else (unsigned char)(252 * exp(-weight * (dist * resolution - inscribed_radius))).  DEFINED: both
 *      tables are computed on the host with its libm, as costmap_2d does, and uploaded.
 *   I3 the rect [min_i, max_i) x [min_j, max_j) is widened by r on every side and clamped to the grid; its LETHAL cells are
 *      the seeds of bin 0.0 in row-major order (j outer, i inner), each its own source.
 *   I4 bins (std::map<double, std::vector<CellData>>) in increasing distance value, each in push order.  An entry whose cell
 *      is seen is skipped; otherwise the cell is marked seen, c = cost[|mx - sx|][|my - sy|], and the master's old value o
 *      becomes c if o == NO_INFORMATION && (inflate_unknown ? c > FREE : c >= 253), else max(o, c).  It then pushes
 *      mx - 1, my - 1, mx + 1, my + 1 (inside the grid, unseen, same source) into bin dist[|nx - sx|][|ny - sy|] unless that
 *      is > r.  Bins are keyed by the double values of the table; a push into a passed bin is never processed.  Any grid
 *      cell within r of a seed can be written, inside the rect or not.  A table that would push a cell into its own bin
 *      (a libm whose hypot is not monotone) is refused: GEM_ERR_INVALID.
 * gem_costmap_inflate runs I3-I4 on master_device (size_x * size_y of the window; origin unused), asynchronously on the
 * handle's stream; it works on any handle and does not read or modify the map.  The order-dependent brushfire is reproduced
 * byte for byte.  Scratch on the handle: 16 bytes per cell plus the tables, grown on demand (a failed growth is GEM_ERR_NOMEM
 * and writes nothing; the handle stays usable, and a later call computes the right bytes).  GEM_ERR_INVALID, with nothing
 * written: NULL pointers, a bad window, a radius, weight or inscribed radius that is negative or not finite (DEFINED: a
 * negative weight is refused), inflate_unknown other than 0 or 1, r above GEM_INFLATE_MAX_CELLS.
 * The bounds (I5) and the inscribed radius of the footprint (I7) are host arithmetic: gem_b200/costmap.py. */
enum { GEM_INFLATE_MAX_CELLS = 4094 };
typedef struct gem_costmap_inflation {
    double inflation_radius, cost_scaling_factor, inscribed_radius; /* metres, 1/metres, metres */
    int inflate_unknown;                                            /* 0 or 1 */
} gem_costmap_inflation;
int gem_costmap_inflate(gem_map *m, const gem_costmap_window *w, const gem_costmap_inflation *p, unsigned char *master_device,
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
 *   Host-synchronous (one synchronisation: the steps of gem_add_pointcloud2_filtered_host_async enqueued, then the info
 *   read back); works on any handle, tiled ones included; neither reads nor modifies the map and does not issue the
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

/* ---- raw sensor messages: the first lines of ElevationMapping::Callback (ElevationMapping.cpp:311-317; DESIGN.md f12) ----
 * gem_pointcloud2 mirrors sensor_msgs/PointCloud2 without a ROS dependency (fields points at nfields gem_pointfield,
 * datatype = sensor_msgs/PointField's codes 1..8).  The node turns the message into pcl::PointCloud<PointXYZRGBICT>
 * with pcl::fromPCLPointCloud2; these calls restate PCL 1.8's createMapping<PointXYZRGBICT> and fromPCLPointCloud2
 * (the PCL of ROS Kinetic).  Unpinned: restated, PCL is not available.
 *   M1 match: the struct fields x 0, y 4, z 8, rgb 16, intensity 24, covariance 20, travers 28 (bytes into the 32-byte
 *      record), in this registration order, each take the FIRST message field in list order whose name is equal, whose
 *      datatype is FLOAT32 and whose count is 1 or 0.  No rgb / rgba aliasing.  An unmatched struct field is left alone
 *      (PCL only warns): matched bit k of gem_pc2_mapping says whether field k of that order was found.
 *   M2 coalesce: the mappings sorted by message offset; one is merged into its predecessor when the two differences of
 *      message and struct offsets are equal, the predecessor growing to the end of the later one, so a merged span also
 *      copies the message bytes between the two fields into struct bytes no mapping of their own names.
 *   M3 copy: with exactly one span left, at message and struct offset 0, and point_step == 32, each whole 32-byte
 *      point is copied (the unmapped bytes too; PCL's memcpy fast path); otherwise every span of every point, in span
 *      order (a later span overwrites what an earlier one wrote), from the point at row * row_step + col * point_step.
 *      is_bigendian (and is_dense) are not read.
 *   DEFINED: struct bytes nothing writes are 0 (the reference's constructor is empty: stale heap bytes).  So a cloud
 *      without a FLOAT32 intensity (an Ouster's uint16 one) gets intensity 0, and the colour gate of gpu.cu:488 then
 *      never passes: such a cloud writes no intensity or colour into the map.
 *   DEFINED: GEM_ERR_INVALID, nothing written, where PCL reads out of bounds or wraps a size_t: a datatype outside 1..8,
 *      width * height > INT_MAX, and with width * height > 0: row_step < width * point_step, data_bytes <
 *      (height - 1) * row_step + width * point_step, a matched field ending past point_step, two matched fields
 *      overlapping in the message.  Names longer than 31 bytes never match.
 * gem_pointcloud2_mapping: host code, no handle, no GPU: validates the layout against data_bytes and fills *out.
 * gem_decode_pointcloud2: width * height float4 {x, y, z, intensity} = struct bytes 0-11 and 24-27 of the records
 *   M1-M3 define, row-major, into xyzi_out_device (16-byte aligned).  Bytes are copied, never computed on: NaN payloads
 *   and -0 survive.  No point is removed (the sensor processors' cleanPointCloud and gem_voxel_grid cut non-finite
 *   ones).  data_device may have any alignment; input and output may not overlap.  Asynchronous on the handle's stream.
 * gem_image_to_bgr8: cv_bridge::toCvCopy(image, "bgr8") for the encodings where it is a byte permutation: "bgr8"
 *   copied, "rgb8" channels swapped, "bgra8" / "rgba8" alpha dropped, "mono8" replicated into three channels.  Any other
 *   encoding (cv_bridge scales or demosaics those) is GEM_ERR_INVALID.  step / dst_step: row strides in bytes (at least
 *   channels * width / 3 * width); src and dst may not overlap.  Asynchronous on the handle's stream.
 * gem_add_pointcloud2_host_async: Callback's lines 311-381 plus processpoints in one call: the message bytes (and the
 *   image, when img != NULL) go to the device on the copy stream, are decoded into the staging set of
 *   gem_add_points_host_async, colourised there as gem_colourise_points does by the handle's colour lookup mode (img !=
 *   NULL: intensities of points that do not project are zeroed before the add reads them; img == NULL: no colour, like
 *   rgba NULL) and added pipelined.
 *   It shares the three-slot ring of gem_add_points_host_async (staging sets, events, counters): the two calls may be
 *   interleaved on one handle.  Its own message and image staging buffers, and the NODE lookup's scratch, grow on demand,
 *   after synchronising the handle's streams and before anything is enqueued (a failed growth is GEM_ERR_NOMEM and
 *   changes nothing).  Host
 *   buffers: pinned memory must stay untouched until the call after next (or gem_sync); pageable memory is accepted and
 *   may be reused as soon as the call returns (CUDA stages it before the copy call returns), so a ROS message's data can
 *   be passed as it is.  width * height > max_points is refused; width * height == 0 flushes. */
enum { GEM_PF_INT8 = 1, GEM_PF_UINT8 = 2, GEM_PF_INT16 = 3, GEM_PF_UINT16 = 4, GEM_PF_INT32 = 5, GEM_PF_UINT32 = 6,
       GEM_PF_FLOAT32 = 7, GEM_PF_FLOAT64 = 8 };
enum { GEM_PC2_X = 0, GEM_PC2_Y = 1, GEM_PC2_Z = 2, GEM_PC2_RGB = 3, GEM_PC2_INTENSITY = 4, GEM_PC2_COVARIANCE = 5,
       GEM_PC2_TRAVERS = 6, GEM_PC2_FIELDS = 7 };
typedef struct gem_pointfield {
    char name[32];
    unsigned offset;
    unsigned char datatype;       /* GEM_PF_*                                                 */
    unsigned count;
} gem_pointfield;
typedef struct gem_pointcloud2 {
    unsigned width, height, point_step, row_step;
    unsigned char is_bigendian;   /* not read (as in PCL)                                     */
    int nfields;
    const gem_pointfield *fields; /* host memory                                              */
} gem_pointcloud2;
typedef struct gem_pc2_span {
    unsigned serialized_offset, struct_offset, size;
} gem_pc2_span;
typedef struct gem_pc2_mapping {
    int nspans;                   /* spans after M2, sorted by message offset                 */
    gem_pc2_span spans[GEM_PC2_FIELDS];
    int fast_path;                /* M3's whole-point copy                                    */
    unsigned matched;             /* bit GEM_PC2_*: that struct field found a message field   */
    long long points;             /* width * height                                           */
    unsigned long long bytes;     /* message bytes the copy reads (from the first)            */
} gem_pc2_mapping;
typedef struct gem_camera_image {
    double T_camera[12], T_lidar[16]; /* as gem_colourise_points                              */
    char encoding[32];            /* sensor_msgs/Image encoding                               */
    int width, height, step;
    const void *data;             /* host memory, pinned or pageable                          */
} gem_camera_image;
int gem_pointcloud2_mapping(const gem_pointcloud2 *layout, unsigned long long data_bytes, gem_pc2_mapping *out);
int gem_decode_pointcloud2(gem_map *m, const gem_pointcloud2 *layout, const void *data_device, unsigned long long data_bytes,
                           void *xyzi_out_device);
int gem_image_to_bgr8(gem_map *m, const char *encoding, const void *src_device, int width, int height, int step,
                      void *dst_device, int dst_step);
int gem_add_pointcloud2_host_async(gem_map *m, const gem_pointcloud2 *layout, const void *data_host, unsigned long long data_bytes,
                                   const gem_camera_image *img, const gem_frame *frame);

/* ---- the demos' VoxelGrid pre-filter inside the asynchronous add (DESIGN.md f20) ----
 * gem_prefilter: the VoxelGrid nodelets in front of the node, in launch order (filter.launch: one step; filter_kitti.launch:
 *   three); nsteps == 0 is no filter.  Each step is gem_voxel_grid with these parameters.
 * gem_add_pointcloud2_filtered_host_async: gem_add_pointcloud2_host_async with the pre-filter between the decode and the
 *   colour lookup.  All on the handle's stream, with no host synchronisation and no read-back of any count: H2D copy
 *   (copy stream), decode into a handle buffer, the steps alternating between two handle buffers, the last one into the
 *   ring's staging set, the colour lookup by the handle's mode, the pipelined add.  The map, gem_stats and the steps'
 *   infos equal those of decode -> gem_voxel_grid per step -> gem_colourise_points -> gem_add_points_stream, bit for bit.
 *   Kernels and sorts run at the raw width * height; the filtered count stays on the device, and gem_stats.points_in
 *   reports it (fetched with the other counters).  A raw cloud of 0 points flushes, as gem_add_pointcloud2_host_async;
 *   a filtered count of 0 is an add of nothing.  Same ring, host-buffer rules and growth as
 *   gem_add_pointcloud2_host_async (the two, and gem_add_points_host_async, may be interleaved); the step scratch (about
 *   64 bytes per raw point) grows in the same way.  DEFINED: the composition is decode -> filter -> colour.  The reference
 *   filters the message and decodes the result; the two are equal wherever x, y, z and intensity are FLOAT32 (the only
 *   layouts where the node maps them: the decode keeps those four fields, and the colour comes after the filter in both).
 *   Elsewhere the result is what decode-first gives.
 *   DEFINED: a step whose voxel grid gem_voxel_grid refuses (bounds whose products with 1 / leaf are not finite, a span of
 *   few voxels near FLT_MAX) passes its input through, with passthrough = 1.
 * gem_add_points_filtered_stream: the same from n float4 {x, y, z, intensity} in device memory; bgr_device (BGR8,
 *   projection's size and row stride) may be NULL for no colour, and projection is read only when it is not.  The input
 *   is read until two further add calls have completed (gem_add_points_stream's rule); it is never written.
 * Both return GEM_ERR_INVALID with nothing enqueued for: a step gem_voxel_grid refuses (bad leaf or field id), nsteps
 *   outside 0..GEM_PREFILTER_MAX_STEPS, n (raw width * height) > max_points, a sensor with cloud_width != 0 (the nodelet
 *   publishes an unorganised cloud, so the pixel index of the stereo model is the index in the filtered cloud), and
 *   whatever gem_add_pointcloud2_host_async / gem_add_points_stream refuse.
 * gem_prefilter_info: host-synchronous; out[s] = count, used and passthrough of step s of the newest filtered call (steps
 *   that call did not run, and every step before the first filtered call, read 0); nsteps in 0..GEM_PREFILTER_MAX_STEPS. */
enum { GEM_PREFILTER_MAX_STEPS = 4 };
typedef struct gem_prefilter {
    int nsteps;
    gem_voxel_grid_params step[GEM_PREFILTER_MAX_STEPS];
} gem_prefilter;
typedef struct gem_projection {
    double T_camera[12], T_lidar[16]; /* as gem_colourise_points                              */
    int width, height, row_stride;    /* the BGR8 image; row_stride in bytes >= 3 * width     */
} gem_projection;
int gem_add_pointcloud2_filtered_host_async(gem_map *m, const gem_pointcloud2 *layout, const void *data_host,
                                            unsigned long long data_bytes, const gem_camera_image *img,
                                            const gem_prefilter *prefilter, const gem_frame *frame);
int gem_add_points_filtered_stream(gem_map *m, const void *xyzi_device, int n, const gem_prefilter *prefilter,
                                   const void *bgr_device, const gem_projection *projection, const gem_frame *frame);
int gem_prefilter_info(gem_map *m, gem_voxel_grid_info *out, int nsteps);

/* ---- saving point clouds as PCD files (savingMap / savingSubMap / pointcloudinterpolation's pcl::io::savePCDFile,
 * ElevationMapping.cpp:430-476, :1117; DESIGN.md f13) ----
 * PCL's PCDWriter::generateHeader / writeASCII (savePCDFile's default) / writeBinary for pcl::PointCloud<PointXYZRGBICT>
 * with width n, height 1 (what push_back and operator+ leave), restated; PCL itself is an unpinned dependency.
 * gem_pcd_header: host code, no handle or GPU.  The header, 11 lines: "# .PCD v0.7 - Point Cloud Data file format",
 *   "VERSION 0.7", "FIELDS x y z rgb intensity covariance travers" (registration order, PointXYZRGBICT.hpp:50-58),
 *   "SIZE 4 4 4 4 4 4 4", "TYPE F F F F F F F", "COUNT 1 1 1 1 1 1 1", "WIDTH n", "HEIGHT 1", "VIEWPOINT 0 0 0 1 0 0 0",
 *   "POINTS n", "DATA ascii" or "DATA binary", each ending in '\n'.  *len_out = its length (0 on an error); the bytes and
 *   a terminating NUL are written only when capacity > length (capacity 0 is a size query).
 * gem_pcd_format: the data section of n 32-byte PointXYZRGBICT records in device memory (16-byte aligned) into
 *   out_device (any alignment, must not overlap the records):
 *     ASCII: one line per record, x y z rgb intensity covariance travers separated by one space, '\n' after; a value is
 *       "nan" for any NaN, else exactly glibc's printf("%.8g") of it ("-0", "inf", "-inf" included); with
 *       GEM_PCD_RGB_UINT32 rgb is the unsigned decimal of its 32 bits (newer PCL; which release switched is not pinned).
 *       A line is at most GEM_PCD_LINE_MAX bytes, so n * GEM_PCD_LINE_MAX bytes always suffice.
 *     GEM_PCD_BINARY: 28 bytes per record, the same seven fields' bytes as they are in memory.
 *   The record's w word (bytes 12-15) is never written.  *bytes_out is always set (0 on an error); all bytes are written
 *   when they fit in capacity, none otherwise (out_device NULL with capacity 0 is a size query).  Host-synchronous.
 * DEFINED where PCL throws (IOException, no file): an empty cloud (n == 0) is GEM_ERR_INVALID for both calls, and nothing
 * is written.  n < 0, unknown flags and a record pointer that is NULL or not 16-byte aligned are GEM_ERR_INVALID. */
enum { GEM_PCD_BINARY = 1, GEM_PCD_RGB_UINT32 = 2 };
#define GEM_PCD_LINE_MAX 105    /* 7 values of at most 14 characters ("-1.2345678e-38"), 6 spaces, '\n' */
#define GEM_PCD_HEADER_MAX 512  /* more than the longest header (n with 19 digits), NUL included */
int gem_pcd_header(long long n, int flags, char *out, int capacity, int *len_out);
int gem_pcd_format(gem_map *m, const void *points32_device, int n, int flags, void *out_device, long long capacity,
                   long long *bytes_out);

/* ---- the node's map topics as serialised ROS1 messages (show()'s publishes, ElevationMap.cpp:123-147, and the clouds
 * and octomaps of ElevationMapping.cpp:491-531, :662-681; DESIGN.md f15) ----
 * The bytes roscpp would put on the wire for visual_map (grid_map_msgs/GridMap), orthomosaic (sensor_msgs/Image),
 * visualpoints (PointCloud2 of pcl::PointXYZRGB), history_point / global_point / the SubMap's cloud (PointCloud2 of
 * PointXYZRGBICT) and road_octomap / obs_octomap (octomap_msgs/Octomap), restated (W1-W8 in gem_b200/csrc/gem_rosfmt.h;
 * ROS, grid_map, PCL and cv_bridge are unpinned).  A node can publish them as they are (e.g. topic_tools::ShapeShifter).
 *   header: {seq, stamp, frame_id} written as given (W1).
 *   gem_ros_grid_map: the 9 layers of gem_export_layers bit for bit (column-major, storage order), resolution = the
 *     handle's grid_resolution (or its float resolution), length_x = length_y = L * resolution (double), pose position =
 *     the handle's centre (cx, cy, 0) -- DEFINED as the centre gem_export_visual_points and gem_export_grid_cloud compute
 *     positions from, which after gem_opt_move is the aligned optimised centre (the reference's visualMap_ keeps the last
 *     ElevationMap::move's) -- orientation (0, 0, 0, 1), start index (sx, sy) as uint16.  737 + |frame_id| + 36 L^2 bytes.
 *   gem_ros_orthomosaic: gem_export_orthomosaic's image, "bgr8", step 3L.  41 + |frame_id| + 3 L^2 bytes.
 *   gem_ros_visual_points: one record {x, y, z, 1.0f, b, g, r, 0xff, 12 zero bytes} per point of gem_export_visual_points,
 *     in its order (the bytes the reference leaves uninitialised DEFINED as 0); is_dense 1.  100 + |frame_id| + 32n bytes.
 *     Host-synchronous (the size needs the shown-cell count).
 *   gem_ros_cloud: the nparts parts' n 32-byte PointXYZRGBICT records each, back to back (byte copies; device, pinned or
 *     pageable host memory).  165 + |frame_id| + 32 * sum(n) bytes; a sum with 32 * sum >= 2^32 is GEM_ERR_INVALID.
 *   gem_ros_octomap: the last gem_color_octree stream (gem_color_octree_read's bytes), id "ColorOcTree", binary 0, that
 *     build's resolution.  44 + |frame_id| + bytes.  GEM_ERR_INVALID when no octree has been built.
 * Common to all five: out is device or pinned host memory at any alignment; pageable host memory is GEM_ERR_INVALID.
 *   The map messages are written by the kernels in place into device memory, and for pinned memory into a device staging
 *   buffer on the handle (grown on demand) that one DMA copy moves to out; clouds and the octree stream are byte copies.
 * *bytes_out is always set (0 on an error); the message is written whole when it fits in capacity, and nothing
 * otherwise (out NULL with capacity 0 is a size query).  No byte outside [out, out + size) is written.  GEM_ERR_INVALID,
 * writing nothing: a NULL header or frame_id, capacity < 0, out NULL with capacity > 0, nparts < 0, a part with n < 0 or
 * NULL records with n > 0, an output overlapping a part, a tiled handle (as for the other post-processing calls).
 * The calls read what gem_export_layers reads and change nothing; asynchronous on the handle's stream except
 * gem_ros_visual_points.  No allocation per call beyond the framing and staging buffers on the handle, which grow on
 * demand. */
typedef struct gem_ros_header {
    unsigned seq, stamp_sec, stamp_nsec;
    const char *frame_id;
} gem_ros_header;
typedef struct gem_ros_part {
    const void *points32;         /* n 32-byte records                                        */
    long long n;
} gem_ros_part;
int gem_ros_grid_map(gem_map *m, const gem_ros_header *h, void *out, long long capacity, long long *bytes_out);
int gem_ros_orthomosaic(gem_map *m, const gem_ros_header *h, void *out, long long capacity, long long *bytes_out);
int gem_ros_visual_points(gem_map *m, const gem_ros_header *h, void *out, long long capacity, long long *bytes_out);
int gem_ros_cloud(gem_map *m, const gem_ros_header *h, const gem_ros_part *parts, int nparts, int is_dense, void *out,
                  long long capacity, long long *bytes_out);
int gem_ros_octomap(gem_map *m, const gem_ros_header *h, void *out, long long capacity, long long *bytes_out);

/* ---- what Costmap2DROS publishes, and ObstacleLayer's footprint clearing (DESIGN.md f17) ----
 * Restated from costmap_2d of navigation 1.14 (unpinned); the wire format follows W1 (gem_b200/csrc/gem_rosfmt.h).
 *   T  the cost translation table: T[0] = 0, T[253] = 99, T[254] = 100, T[255] = -1, T[i] = (char)(1 + (97 (i - 1)) / 251)
 *      in integer arithmetic for 1 <= i <= 252.
 *   W9 nav_msgs/OccupancyGrid (Costmap2DPublisher::prepareGrid): header, map_load_time (0, 0), resolution (float),
 *      width = size_x, height = size_y, origin position (wx - res / 2, wy - res / 2, 0) with (wx, wy) = mapToWorld(0, 0) =
 *      origin + 0.5 res, all in double (so not always bit-equal to the origin), orientation (0, 0, 0, 1), int8[] data =
 *      T[cost] in index order my * size_x + mx.  96 + |frame_id| + size_x size_y bytes; the data field at 92 + |frame_id| (its
 *      uint32 count, then the bytes from 96 + |frame_id|).
 *   W10 map_msgs/OccupancyGridUpdate: header, int32 x = x0, int32 y = y0, uint32 width = xn - x0, uint32 height = yn - y0,
 *      int8[] data = T[master(x, y)], y outer from y0, x inner from x0.  36 + |frame_id| + width height bytes.
 *   W11 geometry_msgs/PolygonStamped (Costmap2DROS::updateMap): header, Point32[] with x = (float)(rx + (fx cos t - fy sin
 *      t)), y = (float)(ry + (fx sin t + fy cos t)), z = 0; cos and sin in double, DEFINED as the host libm's.
 *      20 + |frame_id| + 12 n bytes.
 * The publisher (Costmap2DPublisher::updateBounds / publishCostmap), one gem_costmap_publisher per costmap:
 *   P1 gem_costmap_publisher_init: nothing saved, bounds empty.  DEFINED: empty initial bounds are x0 = y0 = INT_MAX,
 *      xn = yn = 0 (the reference starts at the grid's size, unknown here; the first message is full either way and
 *      min(size, b) = min(INT_MAX, b) for every bound b inside the grid).
 *   P2 gem_costmap_publisher_bounds: x0 = min(x0, b), xn = max(xn, b), likewise y (LayeredCostmap::getBounds' rect).
 *   P3 gem_ros_costmap decides: FULL (W9) when force_full, always_send_full, nothing saved, or the saved (float
 *      resolution, size_x, size_y, double origin_x, origin_y) differ from the window; else UPDATE (W10) of the bounds when
 *      x0 < xn (y is not checked: a height of 0 is sent); else NONE (nothing is written, bytes 0).
 *   P4 a FULL message saves the window.  Then the bounds are reset to empty, x0 = size_x, y0 = size_y, xn = yn = 0
 *      (DEFINED: y0 = size_y; for square grids size_x gives the same bytes) -- except after force_full
 *      (onNewSubscription), which leaves them.
 *   The subscriber gate and the publish timer stay with the caller: not calling gem_ros_costmap is what the reference
 *   does without subscribers, and the bounds keep accumulating.
 * gem_ros_costmap: kind_out receives GEM_COSTMAP_PUB_NONE / _FULL / _UPDATE.  The state of *p changes only when the
 *   call writes its message (a NONE message is written by any call that is not a size query); a size query (out NULL,
 *   capacity 0) or a too-small capacity leaves *p as it was.  GEM_ERR_INVALID, with nothing written and *p unchanged: a
 *   NULL p or master, a bad window (f8), an UPDATE whose bounds are not 0 <= x0 < xn <= size_x, 0 <= y0 <= yn <= size_y,
 *   an output overlapping the master grid, force_full other than 0 or 1.
 * gem_ros_footprint: W11 of the n (x, y) pairs spec_xy (the padded footprint) at the robot's pose.
 * Common to both (f15's rules): out is device or pinned host memory at any alignment (pageable memory is GEM_ERR_INVALID);
 *   the message is written whole or not at all; *bytes_out is always set (out NULL with capacity 0 is a size query);
 *   a NULL header or frame_id, n < 0, a NULL spec_xy with n > 0 and a non-finite pose or spec value are GEM_ERR_INVALID.
 *   Asynchronous on the handle's stream; the map is not read, so tiled handles are accepted.  The master grid is read
 *   once, on the device; pinned outputs are staged on the device and copied in one DMA transfer.
 * gem_costmap_footprint: ObstacleLayer::updateFootprint and the footprint clearing of ObstacleLayer::updateCosts
 *   (setConvexPolygonCost(transformed footprint, FREE_SPACE)) on a layer grid of window w, on the host and one small
 *   kernel.  The footprint is W11's transform kept in double; *out gets marked = the cells written (convexFillCells'
 *   list, duplicates included), lethal = 0 and the touch bounds of the n vertices (+inf / -inf for n = 0).
 *   F1 every vertex goes through worldToMap (f8); one outside the window fills nothing.
 *   F2 fewer than 3 vertices fill nothing (convexFillCells).
 *   F3 polygonOutlineCells: raytraceLine (bresenham2D, both end cells included) from each vertex to the next and from the
 *      last to the first, as indexToCells of the walked offsets.
 *   F4 the adjacent-swap sort by x (after a swap, i steps back), then the column walk: for x from the first cell's x to
 *      the last's, cells i and i + 1 give min and max by y, i += 2, cells of the same x widen them, and the cells (x, y)
 *      for min.y <= y < max.y are appended to the list being walked.  Literal: a column of one cell would pair it with the
 *      next column's first, though F3's closed outline gives every column two cells or more.
 *   Asynchronous on the handle's stream; any handle.  GEM_ERR_INVALID, writing nothing: a NULL layer or out, a bad
 *   window, n < 0, a NULL spec_xy with n > 0, a non-finite pose or spec value. */
enum { GEM_COSTMAP_PUB_NONE = 0, GEM_COSTMAP_PUB_FULL = 1, GEM_COSTMAP_PUB_UPDATE = 2 };
typedef struct gem_costmap_publisher {
    int always_send_full;              /* always_send_full_costmap                                             */
    int saved;                         /* 0 until the first full message                                       */
    float resolution;                  /* the saved window: grid_.info's resolution, width, height and         */
    int size_x, size_y;                /*   saved_origin_x_ / _y_                                              */
    double origin_x, origin_y;
    int x0, xn, y0, yn;                /* the accumulated bounds                                               */
} gem_costmap_publisher;
int gem_costmap_publisher_init(gem_costmap_publisher *p, int always_send_full);
int gem_costmap_publisher_bounds(gem_costmap_publisher *p, int x0, int xn, int y0, int yn);
int gem_ros_costmap(gem_map *m, const gem_ros_header *h, const gem_costmap_window *w, const unsigned char *master_device,
                    gem_costmap_publisher *p, int force_full, void *out, long long capacity, long long *bytes_out, int *kind_out);
int gem_ros_footprint(gem_map *m, const gem_ros_header *h, const double *spec_xy, int n, double robot_x, double robot_y,
                      double robot_yaw, void *out, long long capacity, long long *bytes_out);
int gem_costmap_footprint(gem_map *m, const gem_costmap_window *w, const double *spec_xy, int n, double robot_x, double robot_y,
                          double robot_yaw, unsigned char *layer_device, gem_costmap_marks *out);

/* ---- the costmap plugins fed from their subscribed messages (DESIGN.md f18) ----
 * In GEM's deployment the two layers/ plugins run in move_base and subscribe: ElevationMapLayer::elevationMapCB
 * (layers/src/elevationMap_layer.cpp:31-38) runs grid_map::GridMapRosConverter::fromMessage on a grid_map_msgs/GridMap,
 * PointMapLayer::pointMapCB (layers/src/pointMap_layer.cpp:33-41) pcl::fromPCLPointCloud2 on a PointCloud2 of
 * PointXYZRGBICT.  grid_map 1.6 is unpinned; restated (gem_b200/csrc/gem_gridmsg.h):
 *   G1 setGeometry: size = (int)round(length / resolution) per axis (round half away from zero), length = size *
 *      resolution, position = info.pose.position.{x, y} (orientation and z ignored), start index = (outer_start_index,
 *      inner_start_index).
 *   G2 layer i of `layers` goes with data[i]; gridMap.add replaces an existing layer, so the LAST layer of a repeated
 *      name wins.
 *   G3 Float32MultiArray: dim[0].label "column_index" (column-major) is the only order accepted; rows = dim[1].size,
 *      cols = dim[0].size; data_offset is ignored; floats beyond rows * cols are ignored.
 *   G4 GridMapIterator order is the float order of the layer: element k has buffer index (k % size_x, k / size_x) and
 *      position (position + (0.5 length - 0.5 resolution)) + resolution * (-unwrapped index), in double, per axis; the
 *      unwrapped index is (index - start) wrapped into [0, size) for any start value.
 * gem_grid_map_msg_parse: host code, no handle, no GPU.  Walks the serialised GridMap msg[0, bytes) (ROS1 wire format,
 *   W1 / W2 of gem_rosfmt.h read instead of written) and fills *out with G1's geometry and where `layer`'s floats are:
 *   offset = the byte offset of its first float in the message, floats = size_x * size_y (G3's rows * cols).  Bytes after
 *   the message's last field are ignored.  GEM_ERR_INVALID, *out untouched, where fromMessage throws, asserts (compiled
 *   out) or reads out of bounds: a NULL argument, a truncated message (any string or array count running past `bytes`),
 *   layers.size() != data.size(), the layer missing, fewer than two dims or dim[0] not "column_index", (rows, cols) not
 *   (size_x, size_y), fewer floats than rows * cols, a resolution or length that is <= 0 or not finite, a size above
 *   INT_MAX or size_x * size_y above INT_MAX.
 * gem_costmap_mark_grid: ElevationMapLayer::updateBounds (:56-84) over the layer a descriptor locates: layer_device points
 *   at its first float (device memory, any alignment; e.g. msg_device + g->offset of a message copied whole), read in G4
 *   order with G4's positions; the cost rule, mark_unknown, the last writer and the marks are gem_costmap_mark_map's.
 *   It reads no map, so it works on any handle (a costmap-only process creates the smallest handle gem_create accepts).
 *   Host-synchronous; the scratch of the other mark calls.  GEM_ERR_INVALID, nothing written: NULL pointers, a bad
 *   window, a descriptor that fails G1 / G3's checks.
 * gem_decode_pointcloud2_records: M1-M3 (f12) into width * height whole 32-byte PointXYZRGBICT records at
 *   points32_out_device (16-byte aligned): the seven struct fields at their struct offsets, bytes nothing writes 0, M3's
 *   fast path copying whole points (bytes 12-15 included).  Bytes are copied, never computed on.  The records feed
 *   gem_costmap_mark_points, gem_ros_cloud, gem_pcd_format, gem_color_octree and the global map as they are.
 *   Otherwise as gem_decode_pointcloud2. */
typedef struct gem_grid_map_layer {
    double resolution;                 /* info.resolution                                                       */
    double position_x, position_y;     /* info.pose.position                                                    */
    double length_x, length_y;         /* size * resolution (G1)                                                */
    int size_x, size_y;                /* (int)round(length / resolution) of the message's lengths (G1)         */
    int start_x, start_y;              /* outer_start_index, inner_start_index as sent (any value; G4 wraps)     */
    unsigned long long offset;         /* message byte offset of the layer's first float                        */
    long long floats;                  /* size_x * size_y                                                       */
    int column_major;                  /* 1: the only storage order accepted (G3)                               */
} gem_grid_map_layer;
int gem_grid_map_msg_parse(const void *msg, unsigned long long bytes, const char *layer, gem_grid_map_layer *out);
int gem_costmap_mark_grid(gem_map *m, const gem_grid_map_layer *g, const void *layer_device, const gem_costmap_window *w,
                          double travers_thresh, int mark_unknown, unsigned char *cost_device, gem_costmap_marks *out);
int gem_decode_pointcloud2_records(gem_map *m, const gem_pointcloud2 *layout, const void *data_device, unsigned long long data_bytes,
                                   void *points32_out_device);

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

/* ---- the global map: globalMap_, trajectory_, localMapLoc_ and updateGlobalMap (ElevationMapping.cpp:633-662, :688-707,
 * :773-905, :491-498; DESIGN.md f16) ----
 * A stack of keyframe submaps on the handle, in one device arena of 32-byte PointXYZRGBICT records, with the keyframe poses
 * (trajectory_, row-major 4 x 4 floats, row 3 ignored) and centres (localMapLoc_, x, y).  The stack has its own stream and
 * lock: reset, reserve, update, info, submap, records, pose and stream never take the handle's lock nor wait on its stream,
 * so a loop closure does not hold up the add path.  After every call that changes it the submaps lie back to back in push
 * order: the whole stack is one run of records, composingGlobalMap's cloudpt (:491-493) and the visualCloud_ updateGlobalMap
 * rebuilds (:893-897), ready for gem_ros_cloud or gem_pcd_format as it is.
 * gem_global_map_reset: the init branch (:688-707): no submap, trajectory_ = {identity}, centres = {(0, 0)}.  A new handle
 *   starts in this state.
 * gem_global_map_reserve: room for `records` records and `submaps` submaps, and the update scratch for a pair of submaps of
 *   up to `records` records each, so that later pushes and updates do not allocate.  Otherwise capacity doubles on demand;
 *   a growth that fails returns GEM_ERR_NOMEM and leaves the stack as it was.
 * gem_global_map_push: the keyframe branch (:633-662): trajectory_.push_back(pose), centre = (pose[3], pose[7]), then
 *   globalMap_.push_back of the n records (device memory, e.g. the output of cutSubmap), which are copied.  Submap k thus
 *   belongs to keyframe k, where its accumulation started, and there is always one keyframe more than submaps.  The copy
 *   waits for the work already enqueued on the handle's stream; the call returns when the copy is done.
 * gem_global_map_update: updateGlobalMap (:773-905) in one call: K' = min(k, submaps); submap i of 1 <= i < K' is re-posed
 *   with T = opt_poses[i] * trajectory_[i]^-1 (Eigen's Isometry3f arithmetic in float, DESIGN.md f16) and trajectory_[i] =
 *   opt_poses[i]; then every pair (j, i) of :812-891 (kd-tree of the first K' centres within `radius`, nearest first,
 *   ties by index; only when more than two results; the first result and i itself skipped) is re-fused as by
 *   gem_refuse_submaps, with the counts on the device and no host round trip between pairs; the stack is packed again.
 *   Centres are not updated (the reference never does), nor are trajectory_[0] and submap 0.  *fused_out = the cells
 *   fused over all pairs.  One synchronisation, at the end.  opt_poses: k row-major 4 x 4 floats (Eigen's
 *   Isometry3f::matrix().data() is column-major: transpose it).
 * gem_global_map_info: submaps, keyframes (submaps + 1) and records in the stack; any pointer may be NULL.
 * gem_global_map_submap / gem_global_map_records: device pointer and count of submap i / of the whole packed stack, valid
 *   until the next push, update, reserve or reset.
 * gem_global_map_pose: keyframe i's pose (16 floats) and centre (2 floats); either may be NULL.
 * gem_global_map_stream: the stack's stream (NULL on failure).
 * GEM_ERR_INVALID, with nothing changed, for: k < 0 or NULL opt_poses with k > 0; resolution <= 0 or not finite; radius
 * negative or NaN; n < 0, NULL pose, or NULL or non-device records with n > 0 on a push; an index out of range. */
int gem_global_map_reset(gem_map *m);
int gem_global_map_reserve(gem_map *m, long long records, int submaps);
int gem_global_map_push(gem_map *m, const void *records_device, int n, const float pose[16]);
int gem_global_map_update(gem_map *m, const float *opt_poses, int k, double resolution, double radius, int compat, int *fused_out);
int gem_global_map_info(gem_map *m, int *submaps, int *keyframes, long long *records);
int gem_global_map_submap(gem_map *m, int i, void **records_device_out, int *count_out);
int gem_global_map_records(gem_map *m, void **records_device_out, long long *count_out);
int gem_global_map_pose(gem_map *m, int i, float pose_out[16], float centre_out[2]);
void *gem_global_map_stream(gem_map *m);

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
