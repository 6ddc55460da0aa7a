// gem_b200/elevation_map.hpp -- C++ host facade over the C ABI (include/gem_b200.h).
//
// Header-only, C++14.  Mirrors the reference's map object and sensor-processor interface so
// that a maintainer of the ROS node can swap the nine ad hoc `libgpu.so` declarations for it:
//   - elevation_mapping::ElevationMap  (ElevationMap.hpp:46-210; upstream add()/fuse()/clean()
//     vocabulary, which BASELINE.json uses and which GEM replaced by free CUDA functions)
//   - SensorProcessorBase::process / GPUPointCloudprocess (SensorProcessorBase.cpp:66-211)
//   - the free functions of gpu_process.cu: Move :1004, Process_points :1085, Fuse :1154,
//     Mapvar_update :1146, Map_feature :1256, Raytracing :1304, Map_optmove :1215,
//     Map_closeloop :1235.
// All arithmetic happens in libgem_b200.so (sm_90a CUDA); errors become std::runtime_error
// (the reference prints to stderr and continues, gpu_process.cu:987-992).
#pragma once

#include <cmath>
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <limits>
#include <stdexcept>
#include <string>
#include <vector>

#include "../gem_b200.h"

namespace gem_b200 {

// PointXYZRGBICT (PointXYZRGBICT.hpp:26-48): the 32-byte PCL record the node's clouds hold.
struct PointXYZRGBICT {
    float x, y, z, pad;
    unsigned char b, g, r, a;
    float covariance, intensity, travers;
};
static_assert(sizeof(PointXYZRGBICT) == 32, "PCL record layout");

// sensor_processor/* parameters (config/sensor_processors/*.yaml)
struct LaserSensorProcessor { // LaserSensorProcessor.cpp:38-47
    float min_radius = 0.018f, beam_angle = 0.0006f, beam_constant = 0.0015f;
    double ignore_points_above = 0.8, ignore_points_below = -5.0;
    gem_sensor_model model() const
    {
        gem_sensor_model m{};
        m.type = GEM_SENSOR_LASER;
        m.min_radius = min_radius; m.beam_angle = beam_angle; m.beam_constant = beam_constant;
        m.normal_factor_e = 1.0;
        return m;
    }
};
struct StructuredLightSensorProcessor { // StructuredLightSensorProcessor.cpp:36-48
    double normal_factor_a = 0.000611, normal_factor_b = 0.003587, normal_factor_c = 0.3515;
    double normal_factor_d = 0.0, normal_factor_e = 1.0, lateral_factor = 0.01576;
    double cutoff_min_depth = 0.2, cutoff_max_depth = 3.25; // cleanPointCloud pass-through, :51-66
    double ignore_points_above = std::numeric_limits<double>::infinity();
    double ignore_points_below = -std::numeric_limits<double>::infinity();
    gem_sensor_model model() const
    {
        gem_sensor_model m{};
        m.type = GEM_SENSOR_STRUCTURED_LIGHT;
        m.normal_factor_a = normal_factor_a; m.normal_factor_b = normal_factor_b; m.normal_factor_c = normal_factor_c;
        m.normal_factor_d = normal_factor_d; m.normal_factor_e = normal_factor_e; m.lateral_factor = lateral_factor;
        m.cutoff_min_depth = cutoff_min_depth; m.cutoff_max_depth = cutoff_max_depth;
        return m;
    }
};

// Per-frame constants exactly as GPUPointCloudprocess / readcomputerparam derive them
// (SensorProcessorBase.cpp:171-206, 270-290).  T: row-major 4x4 map<-sensor in double
// (the tf lookup), cast to float like the reference does.
template <typename Sensor>
inline gem_frame makeFrame(const double T_map_sensor[16], const Sensor &sensor, double base_z_in_map = 0.0)
{
    gem_frame f;
    std::memset(&f, 0, sizeof f);
    for (int i = 0; i < 16; i++) f.T[i] = (float)T_map_sensor[i];
    for (int j = 0; j < 3; j++) f.sensor_jacobian[j] = (float)T_map_sensor[8 + j]; // e_z^T * R_map<-sensor
    f.C_SB_transpose[0] = f.C_SB_transpose[4] = f.C_SB_transpose[8] = 1.0f;
    f.P_mul_C_BM_transpose[2] = 1.0f;
    f.rel_lower = base_z_in_map + sensor.ignore_points_below; // SPB.cpp:183
    f.rel_upper = base_z_in_map + sensor.ignore_points_above; // SPB.cpp:184
    f.sensor = sensor.model();
    return f;
}

// The 9 layers ElevationMap::show writes into visualMap_ (ElevationMap.cpp:44,97-110),
// column-major (grid_map::Matrix == Eigen::MatrixXf), NaN = empty.
struct Layers {
    int length = 0;
    std::vector<float> elevation, variance, rough, slope, traver, color_r, color_g, color_b, intensity;
    void resize(int L)
    {
        length = L;
        const size_t n = (size_t)L * L;
        for (auto *v : {&elevation, &variance, &rough, &slope, &traver, &color_r, &color_g, &color_b, &intensity}) v->resize(n);
    }
};

// The outputs of ElevationMap::globalOctrees: the two ColorOcTree streams (octomap_msgs::Octomap::data) and the counts.
struct GlobalOctrees {
    std::vector<int8_t> road, obstacle;
    gem_octree roadInfo, obstacleInfo;
    gem_grid_split split;
};

class ElevationMap {
  public:
    ElevationMap(int length, float resolution, float mahalanobis_threshold = 2.5f, float obstacle_threshold = 0.7f,
                 bool compat_box_filter = true, int device = -1, int max_points = 0, double grid_resolution = 0.0)
    {
        gem_config c;
        std::memset(&c, 0, sizeof c);
        c.grid_resolution = grid_resolution; // the node's double resolution_ (ElevationMapping.hpp:314); 0 = the float
        c.length = length; c.resolution = resolution; c.mahalanobis_threshold = mahalanobis_threshold;
        c.obstacle_threshold = obstacle_threshold; c.compat_box_filter = compat_box_filter ? 1 : 0;
        c.device = device; c.max_points = max_points;
        const int rc = gem_create(&c, &h_);
        if (rc != GEM_OK) throw std::runtime_error(std::string("gem_create: ") + gem_last_error(nullptr));
        length_ = length;
    }
    ~ElevationMap() { gem_destroy(h_); }
    ElevationMap(const ElevationMap &) = delete;
    ElevationMap &operator=(const ElevationMap &) = delete;

    int length() const { return length_; }
    gem_map *handle() { return h_; }

    // ElevationMap::move (ElevationMap.cpp:172-177) + Move (gpu_process.cu:1004)
    void move(const float position[3], float centre[2] = nullptr, int start_index[2] = nullptr, float shift[2] = nullptr)
    {
        check(gem_move(h_, position, centre, start_index, shift), "gem_move");
    }
    // upstream ElevationMap::add == SensorProcessorBase::process + Fuse
    // (ElevationMapping::processpoints, ElevationMapping.cpp:254-283), host PCL records
    void add(const PointXYZRGBICT *cloud, size_t n, const gem_frame &frame)
    {
        check(gem_add_cloud_pcl_host(h_, cloud, (int)n, &frame), "gem_add_cloud_pcl_host");
    }
    // device-resident float4 {x,y,z,intensity} + uchar4 rgba (asynchronous)
    void addDevice(const void *xyzi_device, const void *rgba_device, size_t n, const gem_frame &frame)
    {
        check(gem_add_points(h_, xyzi_device, rgba_device, (int)n, &frame), "gem_add_points");
    }
    // The same, frame-pipelined: the per-cell fold of this call is issued together with the NEXT call's binning (one CUDA
    // graph per call); whatever reads the map next -- or flush() -- issues the last fold.  `xyzi_device` must stay valid
    // until then (the fold reads the intensities from it).
    void addStream(const void *xyzi_device, const void *rgba_device, size_t n, const gem_frame &frame)
    {
        check(gem_add_points_stream(h_, xyzi_device, rgba_device, (int)n, &frame), "gem_add_points_stream");
    }
    // several sensors' clouds in ONE launch (offsets[0] = 0 ... offsets[n_segments] = total points, one gem_frame each):
    // equal to adding them one after the other
    void addMulti(const void *xyzi_device, const void *rgba_device, int n_segments, const int *offsets, const gem_frame *frames)
    {
        check(gem_add_points_multi(h_, xyzi_device, rgba_device, n_segments, offsets, frames), "gem_add_points_multi");
    }
    // pinned host float4 / uchar4 buffers: the copy runs on a copy stream under the previous frame's kernels, no host
    // synchronisation (three staging sets rotate)
    void addHostAsync(const void *xyzi_pinned, const void *rgba_pinned, size_t n, const gem_frame &frame)
    {
        check(gem_add_points_host_async(h_, xyzi_pinned, rgba_pinned, (int)n, &frame), "gem_add_points_host_async");
    }
    void flush() { check(gem_flush(h_), "gem_flush"); }
    // ElevationMapping::Callback's image branch (ElevationMapping.cpp:331-381): colours for a device cloud from a device
    // BGR8 image; T_camera 3x4, T_lidar 4x4, row-major doubles as the node's yaml files hold them
    void colourise(void *xyzi_device, size_t n, const double T_camera[12], const double T_lidar[16], const unsigned char *bgr_device,
                   int width, int height, int row_stride_bytes, void *rgba_out_device)
    {
        check(gem_colourise_points(h_, xyzi_device, (int)n, T_camera, T_lidar, bgr_device, width, height, row_stride_bytes,
                                   rgba_out_device), "gem_colourise_points");
    }
    // RobotMotionMapUpdater::update -> Mapvar_update (RobotMotionMapUpdater.cpp:81)
    void update(float variance_increment) { check(gem_var_update(h_, variance_increment), "gem_var_update"); }
    // upstream ElevationMap::fuse: Map_feature + show's write-back into grid_map layers
    void fuse(Layers &out)
    {
        check(gem_compute_features(h_), "gem_compute_features");
        if (out.length != length_) out.resize(length_);
        float *ptr[9] = {out.elevation.data(), out.variance.data(), out.rough.data(), out.slope.data(), out.traver.data(),
                         out.color_r.data(), out.color_g.data(), out.color_b.data(), out.intensity.data()};
        check(gem_export_layers(h_, ptr), "gem_export_layers");
    }
    // fuse() in two halves: fuseBegin starts the write-back on a copy stream and returns, fuseEnd waits for it.  Work
    // that does not change what was exported may be issued in between -- the node calls Raytracing right after show()
    // (ElevationMapping.cpp:404-421): fuseBegin(out); clean(); fuseEnd();  `out` must be page-locked for the copy to
    // overlap (gem_host_alloc) and must not be touched before fuseEnd.
    void fuseBegin(float *layers_pinned[9])
    {
        check(gem_compute_features(h_), "gem_compute_features");
        check(gem_export_layers_begin(h_, layers_pinned), "gem_export_layers_begin");
    }
    void fuseEnd() { check(gem_export_layers_end(h_), "gem_export_layers_end"); }
    // the rest of ElevationMap::show (ElevationMap.cpp:87,112-125), valid after fuse(): the bgr8 orthomosaic
    // (length x length x 3, cv::Mat CV_8UC3 layout) and the pcl::PointXYZRGB visual cloud (xyz + rgb per shown cell)
    void orthomosaic(std::vector<unsigned char> &bgr)
    {
        bgr.resize((size_t)length_ * length_ * 3);
        check(gem_export_orthomosaic(h_, bgr.data()), "gem_export_orthomosaic");
    }
    int visualPoints(std::vector<float> &xyz, std::vector<unsigned char> &rgb)
    {
        const size_t cap = (size_t)length_ * length_;
        xyz.resize(cap * 3);
        rgb.resize(cap * 3);
        int n = 0;
        check(gem_export_visual_points(h_, xyz.data(), rgb.data(), (int)cap, &n), "gem_export_visual_points");
        xyz.resize((size_t)n * 3);
        rgb.resize((size_t)n * 3);
        return n;
    }
    // prevMap_ = map_.visualMap_ (ElevationMapping.cpp:422) kept on the device, and the "L-shape" harvest of the
    // cells that scrolled out of the window into the submap store (ElevationMapping.cpp:716-765).  `current` and
    // `shift` are what move() returned for this frame; the records are PointXYZRGBICT, ready for localMap_ /
    // visualCloud_.  The |shift| >= resolution and init/jump-flag gate of :716 stays with the caller.
    void snapshot() { check(gem_snapshot_shown(h_), "gem_snapshot_shown"); }
    int harvest(const float current[2], const float shift[2], std::vector<PointXYZRGBICT> &out)
    {
        int n = 0;
        check(gem_harvest_scrolled_out(h_, current, shift, nullptr, 0, &n), "gem_harvest_scrolled_out");
        out.resize((size_t)n);
        if (n) check(gem_harvest_scrolled_out(h_, current, shift, out.data(), n, &n), "gem_harvest_scrolled_out");
        return n;
    }
    // The local submap on the device (ElevationMapping.cpp:609-767).  gridCloud: gridMaptoPointCloud (:1198-1226) of the
    // shown map (GEM_GRID_SHOWN, visualMap_) or of the snapshot (GEM_GRID_SNAPSHOT, prevMap_) into device memory; returns
    // the number of cells, min(that, capacity) records are written.  harvestToLocalMap: harvest() upserted into the
    // handle's localMap_ (:740-747); `visual` (may be null) also receives the records, for visualCloud_.  localMapTake:
    // localHashtoPointCloud (:1124-1140) into device memory, the store empties; with capacity < size nothing is written
    // and the size is returned (capacity 0 = size query).  cutSubmap: the keyframe cut of :653-661, local map then grid
    // cloud of the shown map, into one device buffer of `capacity` records; returns the size, writes only if it fits.
    int gridCloud(int source, void *points32_device, size_t capacity)
    {
        int n = 0;
        check(gem_export_grid_cloud(h_, source, points32_device, (int)capacity, &n), "gem_export_grid_cloud");
        return n;
    }
    // The filter of composingGlobalMap (ElevationMapping.cpp:1152-1170): statistical outlier removal over gridCloud(source)
    // and the split of the survivors into road (travers > traversThreshold) and obstacle records, written into device
    // memory (min(count, capacity) each; capacity 0 = size query).  meanDistance (may be null) receives the per-point mean
    // distances in grid-cloud order.  Returns the counts and statistics; colorOctree builds the octrees of the two
    // outputs, globalOctrees does both steps.
    gem_grid_split gridCloudSplit(int source, int meanK, double stddevMul, double traversThreshold, void *road_device,
                                  size_t roadCapacity, void *obstacle_device, size_t obstacleCapacity,
                                  float *meanDistance_device = nullptr, size_t distanceCapacity = 0)
    {
        gem_grid_split s{};
        check(gem_grid_cloud_split(h_, source, meanK, stddevMul, traversThreshold, road_device, (int)roadCapacity, obstacle_device,
                                   (int)obstacleCapacity, meanDistance_device, (int)distanceCapacity, &s),
              "gem_grid_cloud_split");
        return s;
    }
    // pointCloudtoOctomap's octomap::ColorOcTree (ElevationMapping.cpp:1157-1174) of n PointXYZRGBICT records in device
    // memory at `resolution`, as the ColorOcTree::writeData stream: the octomap_msgs::Octomap::data of fullMapToMsg (set
    // id = "ColorOcTree", binary = false, resolution).  info (may be null) receives the counts.
    std::vector<int8_t> colorOctree(const void *points32_device, size_t n, double resolution, gem_octree *info = nullptr)
    {
        if (n > (size_t)std::numeric_limits<int>::max()) throw std::runtime_error("colorOctree: more than INT_MAX points");
        gem_octree o{};
        check(gem_color_octree(h_, points32_device, (int)n, resolution, &o), "gem_color_octree");
        std::vector<int8_t> data((size_t)o.bytes);
        check(gem_color_octree_read(h_, data.data(), o.bytes), "gem_color_octree_read");
        if (info) *info = o;
        return data;
    }
    // composingGlobalMap's numeric work (ElevationMapping.cpp:482-514, :1146-1174): gridCloudSplit into the caller's
    // device buffers (each must hold the whole split output, gridCloud(source) records always do), then the road and the
    // obstacle trees of the node (0.2 m and 0.1 m, :146-147).
    GlobalOctrees globalOctrees(void *road_device, size_t roadCapacity, void *obstacle_device, size_t obstacleCapacity,
                                int source = GEM_GRID_SNAPSHOT, int meanK = 20, double stddevMul = 1.0,
                                double traversThreshold = 0.0, double roadResolution = 0.2, double obstacleResolution = 0.1)
    {
        GlobalOctrees g{};
        g.split = gridCloudSplit(source, meanK, stddevMul, traversThreshold, road_device, roadCapacity, obstacle_device,
                                 obstacleCapacity);
        if ((size_t)g.split.road > roadCapacity || (size_t)g.split.obstacle > obstacleCapacity)
            throw std::runtime_error("globalOctrees: the road or obstacle buffer is smaller than the split output");
        g.road = colorOctree(road_device, (size_t)g.split.road, roadResolution, &g.roadInfo);
        g.obstacle = colorOctree(obstacle_device, (size_t)g.split.obstacle, obstacleResolution, &g.obstacleInfo);
        return g;
    }
    // The costmap_2d layers of GEM's layers/ package (DESIGN.md f8) on caller-owned device grids uint8[size_y][size_x]:
    // ElevationMapLayer::updateBounds over show()'s grid_map, PointMapLayer::updateBounds over PointXYZRGBICT records,
    // Costmap2D::updateOrigin (writes the grid-aligned origin back into w) and updateWithMax / PointMapLayer's overwrite.
    gem_costmap_marks costmapMarkMap(const gem_costmap_window &w, unsigned char *cost_device, double traversThresh = 0.7,
                                     int source = GEM_GRID_SHOWN, bool markUnknown = true)
    {
        gem_costmap_marks mk{};
        check(gem_costmap_mark_map(h_, source, &w, traversThresh, markUnknown ? 1 : 0, cost_device, &mk), "gem_costmap_mark_map");
        return mk;
    }
    gem_costmap_marks costmapMarkPoints(const void *points32_device, size_t n, const gem_costmap_window &w, unsigned char *cost_device,
                                        double traversThresh = 0.7)
    {
        if (n > (size_t)std::numeric_limits<int>::max()) throw std::runtime_error("costmapMarkPoints: more than INT_MAX points");
        gem_costmap_marks mk{};
        check(gem_costmap_mark_points(h_, points32_device, (int)n, &w, traversThresh, cost_device, &mk), "gem_costmap_mark_points");
        return mk;
    }
    void costmapUpdateOrigin(gem_costmap_window &w, double newOriginX, double newOriginY, unsigned char fill, unsigned char *cost_device)
    {
        check(gem_costmap_update_origin(h_, &w, newOriginX, newOriginY, fill, cost_device), "gem_costmap_update_origin");
    }
    void costmapCombine(int mode, const unsigned char *layer_device, unsigned char *master_device, int sizeX, int sizeY, int minI,
                        int minJ, int maxI, int maxJ)
    {
        check(gem_costmap_combine(h_, mode, layer_device, master_device, sizeX, sizeY, minI, minJ, maxI, maxJ), "gem_costmap_combine");
    }
    // pcl_ros's VoxelGrid nodelet (GEM's filter.launch / filter_kitti.launch; DESIGN.md f9) over n float4 {x, y, z, intensity}
    // in device memory: min(count, capacity) centroids go to out_device, which must not overlap the input (capacity 0 is
    // a size query).  Chain calls through two buffers.
    gem_voxel_grid_info voxelGrid(const void *xyzi_device, size_t n, const gem_voxel_grid_params &p, void *out_device, size_t capacity)
    {
        if (n > (size_t)std::numeric_limits<int>::max() || capacity > (size_t)std::numeric_limits<int>::max())
            throw std::runtime_error("voxelGrid: more than INT_MAX points");
        gem_voxel_grid_info info{};
        check(gem_voxel_grid(h_, xyzi_device, (int)n, &p, out_device, (int)capacity, &info), "gem_voxel_grid");
        return info;
    }
    // pointcloudinterpolation's MovingLeastSquares (GEM's dense_mapping signal, ElevationMapping.cpp:1072-1118; DESIGN.md
    // f10) over n PointXYZRGBICT records in device memory: min(count, capacity) new records go to out_device, which must
    // not overlap the input (capacity 0 is a size query).  gemMlsParams() is GEM's setting.
    static gem_mls_params gemMlsParams(unsigned long long seed = 0)
    {
        gem_mls_params p{};
        p.search_radius = 0.5;
        p.sqr_gauss_param = 0.25;
        p.polynomial_fit = 1;
        p.order = 5;
        p.upsampling = GEM_MLS_RANDOM_UNIFORM_DENSITY;
        p.point_density = 1000;
        p.seed = seed;
        return p;
    }
    gem_mls_info mlsUpsample(const void *points32_device, size_t n, const gem_mls_params &p, void *out_device, size_t capacity)
    {
        if (n > (size_t)std::numeric_limits<int>::max() || capacity > (size_t)std::numeric_limits<long long>::max())
            throw std::runtime_error("mlsUpsample: more than INT_MAX points");
        gem_mls_info info{};
        check(gem_mls_upsample(h_, points32_device, (int)n, &p, out_device, (long long)capacity, &info), "gem_mls_upsample");
        return info;
    }
    int harvestToLocalMap(const float current[2], const float shift[2], std::vector<PointXYZRGBICT> *visual = nullptr)
    {
        int n = 0;
        if (visual) visual->resize((size_t)length_ * length_);
        check(gem_harvest_to_local_map(h_, current, shift, visual ? visual->data() : nullptr, visual ? (int)visual->size() : 0, &n),
              "gem_harvest_to_local_map");
        if (visual) visual->resize((size_t)n);
        return n;
    }
    int localMapTake(void *points32_device, size_t capacity)
    {
        int n = 0;
        check(gem_local_map_take(h_, points32_device, (int)capacity, &n), "gem_local_map_take");
        return n;
    }
    void localMapClear() { check(gem_local_map_clear(h_), "gem_local_map_clear"); }
    int cutSubmap(void *points32_device, size_t capacity)
    {
        const int nl = localMapTake(nullptr, 0), ng = gridCloud(GEM_GRID_SHOWN, nullptr, 0);
        if ((size_t)nl + (size_t)ng > capacity) return nl + ng;
        localMapTake(points32_device, (size_t)nl);
        gridCloud(GEM_GRID_SHOWN, (char *)points32_device + (size_t)nl * sizeof(PointXYZRGBICT), (size_t)ng);
        return nl + ng;
    }
    // cutSubmap with the dense_mapping signal (:656-661): [local map, its MLS points (mlsUpsample with p), grid cloud] in
    // one device buffer.  The local map is taken into the front of the buffer and densified from there, so `capacity` must
    // hold the result: when it does not, nothing more is written, the local map stays taken (it is at the front of the
    // buffer) and the size the buffer needs is returned.
    long long cutSubmap(void *points32_device, size_t capacity, bool dense, const gem_mls_params &p = gemMlsParams())
    {
        if (!dense) return cutSubmap(points32_device, capacity);
        const int nl = localMapTake(nullptr, 0), ng = gridCloud(GEM_GRID_SHOWN, nullptr, 0);
        if ((size_t)nl > capacity) return (long long)nl + ng; // nothing taken
        localMapTake(points32_device, (size_t)nl);
        char *base = (char *)points32_device;
        const size_t rest = capacity - (size_t)nl;
        const gem_mls_info info = mlsUpsample(base, (size_t)nl, p, base + (size_t)nl * sizeof(PointXYZRGBICT), rest);
        const long long total = (long long)nl + info.count + ng;
        if ((unsigned long long)total > capacity) return total;
        gridCloud(GEM_GRID_SHOWN, base + ((size_t)nl + (size_t)info.count) * sizeof(PointXYZRGBICT), (size_t)ng);
        return total;
    }
    // Loop closure (ElevationMapping::updateGlobalMap, ElevationMapping.cpp:773-905), on device-resident submaps of
    // PointXYZRGBICT records: re-pose a submap (:805), and one pass of the pairwise fuse loop (:847-883) -- both clouds
    // come back reduced to one point per cell and compacted, *n_new / *n_old updated.  compat_precedence = true evaluates
    // :862-863 exactly as C parses them.  The kd-tree loop around them stays with the caller.
    void transformCloud(void *points32_device, size_t n, const float T_rowmajor[16])
    {
        check(gem_transform_cloud(h_, points32_device, (int)n, T_rowmajor), "gem_transform_cloud");
    }
    int refuseSubmaps(void *new_points32_device, int *n_new, void *old_points32_device, int *n_old, double resolution,
                      bool compat_precedence = true)
    {
        int fused = 0;
        check(gem_refuse_submaps(h_, new_points32_device, n_new, old_points32_device, n_old, resolution, compat_precedence ? 1 : 0, &fused),
              "gem_refuse_submaps");
        return fused;
    }
    // upstream visibilityCleanup / GEM Raytracing (gpu_process.cu:1304)
    void clean() { check(gem_raytracing(h_), "gem_raytracing"); }
    void optMove(const float p[2], float dz, float aligned[2]) { check(gem_opt_move(h_, p, dz, aligned), "gem_opt_move"); }
    void closeLoop(const float p[2], float dz) { check(gem_closeloop(h_, p, dz), "gem_closeloop"); }
    gem_stats stats()
    {
        gem_stats s;
        check(gem_get_stats(h_, &s), "gem_get_stats");
        return s;
    }
    void sync() { check(gem_sync(h_), "gem_sync"); }

  private:
    void check(int rc, const char *what)
    {
        if (rc != GEM_OK) throw std::runtime_error(std::string(what) + ": " + gem_last_error(h_));
    }
    gem_map *h_ = nullptr;
    int length_ = 0;
};

} // namespace gem_b200
