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

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <limits>
#include <new>
#include <stdexcept>
#include <string>
#include <utility>
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

// An allocator of pinned host memory (gem_host_alloc), for buffers the device writes directly, e.g. the rosX messages:
//     std::vector<uint8_t, gem_b200::PinnedAllocator<uint8_t>> msg;
template <class T> struct PinnedAllocator {
    using value_type = T;
    PinnedAllocator() = default;
    template <class U> PinnedAllocator(const PinnedAllocator<U> &) {}
    T *allocate(size_t n)
    {
        void *p = nullptr;
        if (gem_host_alloc(&p, n * sizeof(T)) != GEM_OK) throw std::bad_alloc();
        return static_cast<T *>(p);
    }
    void deallocate(T *p, size_t) { gem_host_free(p); }
    template <class U> bool operator==(const PinnedAllocator<U> &) const { return true; }
    template <class U> bool operator!=(const PinnedAllocator<U> &) const { return false; }
};
using PinnedBytes = std::vector<uint8_t, PinnedAllocator<uint8_t>>;

// sensor_msgs/PointCloud2's layout without ROS (DESIGN.md f12): add the message's fields in order, then pass layout().
// From a sensor_msgs::PointCloud2ConstPtr msg:
//     gem_b200::PointCloud2Layout lay(msg->width, msg->height, msg->point_step, msg->row_step, msg->is_bigendian);
//     for (const auto &f : msg->fields) lay.addField(f.name, f.offset, f.datatype, f.count);
class PointCloud2Layout {
public:
    PointCloud2Layout(unsigned width, unsigned height, unsigned point_step, unsigned row_step, bool is_bigendian = false)
    {
        c_ = gem_pointcloud2{};
        c_.width = width; c_.height = height; c_.point_step = point_step; c_.row_step = row_step;
        c_.is_bigendian = is_bigendian ? 1 : 0;
    }
    // a name of 32 bytes or more is stored without its terminator and matches no struct field (none is that long)
    void addField(const std::string &name, unsigned offset, unsigned char datatype, unsigned count)
    {
        gem_pointfield f{};
        std::memcpy(f.name, name.data(), name.size() < sizeof f.name ? name.size() : sizeof f.name);
        f.offset = offset; f.datatype = datatype; f.count = count;
        fields_.push_back(f);
    }
    const gem_pointcloud2 *layout() const
    {
        c_.nfields = (int)fields_.size();
        c_.fields = fields_.empty() ? nullptr : fields_.data();
        return &c_;
    }
    // createMapping<PointXYZRGBICT>: the spans, the whole-point copy flag and the matched struct fields; throws on the
    // layouts PCL would read out of bounds on (host code, no GPU)
    gem_pc2_mapping mapping(unsigned long long data_bytes) const
    {
        gem_pc2_mapping m{};
        if (gem_pointcloud2_mapping(layout(), data_bytes, &m) != GEM_OK)
            throw std::runtime_error(std::string("gem_pointcloud2_mapping: ") + gem_last_error(nullptr));
        return m;
    }

private:
    std::vector<gem_pointfield> fields_;
    mutable gem_pointcloud2 c_;
};

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

struct StereoSensorProcessor { // StereoSensorProcessor.cpp:23-34: every parameter defaults to 0
    double p_1 = 0.0, p_2 = 0.0, p_3 = 0.0, p_4 = 0.0, p_5 = 0.0, lateral_factor = 0.0, depth_to_disparity_factor = 0.0;
    int cloud_width = 0; // pointCloud->width of the organised cloud the calls receive, 0 = unorganised (getI / getJ, :109-117)
    double ignore_points_above = std::numeric_limits<double>::infinity();
    double ignore_points_below = -std::numeric_limits<double>::infinity();
    gem_sensor_model model() const
    {
        gem_sensor_model m{};
        m.type = GEM_SENSOR_STEREO;
        m.stereo_p[0] = p_1; m.stereo_p[1] = p_2; m.stereo_p[2] = p_3; m.stereo_p[3] = p_4; m.stereo_p[4] = p_5;
        m.lateral_factor = lateral_factor; m.depth_to_disparity_factor = depth_to_disparity_factor;
        m.cloud_width = cloud_width;
        return m;
    }
};
// PerfectSensorProcessor.cpp: zero sensor variance.  Its readParameters does not call the base class (:36-39), so its
// height window is always the constructor's +-inf (SensorProcessorBase.cpp:39-40): it has no ignore_points_*.
struct PerfectSensorProcessor {
    gem_sensor_model model() const
    {
        gem_sensor_model m{};
        m.type = GEM_SENSOR_PERFECT;
        return m;
    }
};

// ignore_points_{below,above} of a sensor processor (SensorProcessorBase.cpp:61-62)
template <typename Sensor> inline void heightWindow(const Sensor &s, double &below, double &above)
{
    below = s.ignore_points_below;
    above = s.ignore_points_above;
}
inline void heightWindow(const PerfectSensorProcessor &, double &below, double &above)
{
    below = -std::numeric_limits<double>::infinity();
    above = std::numeric_limits<double>::infinity();
}

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
    double below, above;
    heightWindow(sensor, below, above);
    f.rel_lower = base_z_in_map + below; // SPB.cpp:183
    f.rel_upper = base_z_in_map + above; // SPB.cpp:184
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
    // which pixel colourise and addPointCloud2HostAsync's image give a point: GEM_COLOUR_LOOKUP_IMAGE (the default, its
    // own pixel of the unmodified image) or GEM_COLOUR_LOOKUP_NODE (the node's loop with its circle painting; DESIGN.md f19)
    void setColourLookup(int mode) { check(gem_set_colour_lookup(h_, mode), "gem_set_colour_lookup"); }
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
    // InflationLayer::updateCosts (DESIGN.md f14) of a master grid over [minI, maxI) x [minJ, maxJ), asynchronous on the
    // handle's stream
    void costmapInflate(const gem_costmap_window &w, const gem_costmap_inflation &p, unsigned char *master_device, int minI, int minJ,
                        int maxI, int maxJ)
    {
        check(gem_costmap_inflate(h_, &w, &p, master_device, minI, minJ, maxI, maxJ), "gem_costmap_inflate");
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
    // raw sensor messages (DESIGN.md f12).  decodePointCloud2: fromPCLPointCloud2's x, y, z, intensity of every point into
    // width * height float4 in device memory (asynchronous).  imageToBgr8: cv_bridge::toCvCopy(image, "bgr8") for bgr8,
    // rgb8, bgra8, rgba8 and mono8 in device memory (asynchronous).  addPointCloud2HostAsync: the message bytes as they
    // arrive (host memory, pinned or pageable) and optionally the camera image, decoded, colourised and added pipelined
    // (Callback's first lines plus processpoints in one call).
    void decodePointCloud2(const PointCloud2Layout &lay, const void *data_device, unsigned long long data_bytes, void *xyzi_out_device)
    {
        check(gem_decode_pointcloud2(h_, lay.layout(), data_device, data_bytes, xyzi_out_device), "gem_decode_pointcloud2");
    }
    void imageToBgr8(const std::string &encoding, const void *src_device, int width, int height, int step, void *dst_device,
                     int dst_step)
    {
        check(gem_image_to_bgr8(h_, encoding.c_str(), src_device, width, height, step, dst_device, dst_step), "gem_image_to_bgr8");
    }
    void addPointCloud2HostAsync(const PointCloud2Layout &lay, const void *data_host, unsigned long long data_bytes,
                                 const gem_camera_image *img, const gem_frame &frame)
    {
        check(gem_add_pointcloud2_host_async(h_, lay.layout(), data_host, data_bytes, img, &frame), "gem_add_pointcloud2_host_async");
    }
    // the demos' VoxelGrid nodelets inside the asynchronous add (DESIGN.md f20): the steps in launch order, then the
    // colour lookup and the pipelined add, with no host synchronisation.  Prefilter::filterLaunch() / filterKittiLaunch()
    // are GEM's two launches.  addPointsFilteredStream reads xyzi_device until two further add calls have completed;
    // bgr_device may be null (no colour).  prefilterInfo synchronises and returns the newest filtered call's steps.
    struct Prefilter {
        gem_prefilter c{};
        Prefilter &add(float leaf, int field, double lo, double hi, bool negative = false)
        {
            if (c.nsteps >= GEM_PREFILTER_MAX_STEPS) throw std::runtime_error("Prefilter: at most GEM_PREFILTER_MAX_STEPS steps");
            gem_voxel_grid_params &p = c.step[c.nsteps++];
            p.leaf_size[0] = p.leaf_size[1] = p.leaf_size[2] = leaf;
            p.field = field;
            p.limit_min = lo;
            p.limit_max = hi;
            p.limit_negative = negative ? 1 : 0;
            return *this;
        }
        static Prefilter filterLaunch() { return Prefilter().add(0.1f, GEM_VOXEL_FIELD_X, -10.0, 10.0); }
        static Prefilter filterKittiLaunch()
        {
            return Prefilter().add(0.2f, GEM_VOXEL_FIELD_X, -40.0, 40.0).add(0.2f, GEM_VOXEL_FIELD_Z, -25.0, 25.0).add(0.2f, GEM_VOXEL_FIELD_Y, -40.0, 40.0);
        }
    };
    void addPointCloud2HostAsync(const PointCloud2Layout &lay, const void *data_host, unsigned long long data_bytes,
                                 const gem_camera_image *img, const Prefilter &pf, const gem_frame &frame)
    {
        check(gem_add_pointcloud2_filtered_host_async(h_, lay.layout(), data_host, data_bytes, img, &pf.c, &frame),
              "gem_add_pointcloud2_filtered_host_async");
    }
    void addPointsFilteredStream(const void *xyzi_device, size_t n, const Prefilter &pf, const void *bgr_device,
                                 const gem_projection *projection, const gem_frame &frame)
    {
        if (n > (size_t)std::numeric_limits<int>::max()) throw std::runtime_error("addPointsFilteredStream: more than INT_MAX points");
        check(gem_add_points_filtered_stream(h_, xyzi_device, (int)n, &pf.c, bgr_device, projection, &frame),
              "gem_add_points_filtered_stream");
    }
    std::vector<gem_voxel_grid_info> prefilterInfo(int nsteps)
    {
        std::vector<gem_voxel_grid_info> out((size_t)std::max(nsteps, 0));
        check(gem_prefilter_info(h_, out.data(), nsteps), "gem_prefilter_info");
        return out;
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
    // Point clouds as PCD files (savingMap / savingSubMap's pcl::io::savePCDFile, ElevationMapping.cpp:430-476; DESIGN.md
    // f13).  pcdHeader: PCL's header for n records (host only).  formatPcd: the data section of n records in device memory
    // into out_device when all of it fits in capacity (nothing otherwise; capacity 0 is a size query); returns its bytes.
    // savePcd: header and data to `path`, the records in device memory (onDevice) or host memory, streamed through pinned
    // buffers in chunks of `chunk` records (the device reads and writes them directly), so the file is the same whatever
    // the chunk.  An empty cloud throws, as PCL does, and writes no file.
    static std::string pcdHeader(long long n, bool binary = false, bool rgbUint32 = false)
    {
        char h[GEM_PCD_HEADER_MAX];
        int len = 0;
        if (gem_pcd_header(n, pcdFlags(binary, rgbUint32), h, (int)sizeof h, &len) != GEM_OK)
            throw std::runtime_error(std::string("gem_pcd_header: ") + gem_last_error(nullptr));
        return std::string(h, (size_t)len);
    }
    long long formatPcd(const void *points32_device, size_t n, bool binary, bool rgbUint32, void *out_device, size_t capacity)
    {
        if (n > (size_t)std::numeric_limits<int>::max()) throw std::runtime_error("formatPcd: more than INT_MAX records");
        long long bytes = 0;
        check(gem_pcd_format(h_, points32_device, (int)n, pcdFlags(binary, rgbUint32), out_device, (long long)capacity, &bytes),
              "gem_pcd_format");
        return bytes;
    }
    void savePcd(const std::string &path, const void *records, size_t n, bool onDevice, bool binary = false, bool rgbUint32 = false,
                 size_t chunk = (size_t)1 << 20)
    {
        const std::string head = pcdHeader((long long)n, binary, rgbUint32);
        const size_t step = std::max<size_t>(1, std::min(chunk, n)), per = binary ? 28 : GEM_PCD_LINE_MAX;
        void *in = nullptr, *out = nullptr;
        if ((!onDevice && gem_host_alloc(&in, step * sizeof(PointXYZRGBICT)) != GEM_OK) || gem_host_alloc(&out, step * per) != GEM_OK) {
            if (in) gem_host_free(in);
            throw std::runtime_error("savePcd: gem_host_alloc failed");
        }
        FILE *f = std::fopen(path.c_str(), "wb");
        bool ok = f && std::fwrite(head.data(), 1, head.size(), f) == head.size();
        try {
            for (size_t i = 0; ok && i < n; i += step) {
                const size_t k = std::min(step, n - i);
                const char *src = static_cast<const char *>(records) + i * sizeof(PointXYZRGBICT);
                if (!onDevice) std::memcpy(in, src, k * sizeof(PointXYZRGBICT));
                const long long bytes = formatPcd(onDevice ? src : in, k, binary, rgbUint32, out, step * per);
                ok = std::fwrite(out, 1, (size_t)bytes, f) == (size_t)bytes;
            }
        } catch (...) {
            ok = false;
        }
        if (f && std::fclose(f) != 0) ok = false;
        if (in) gem_host_free(in);
        gem_host_free(out);
        if (!ok) {
            if (f) std::remove(path.c_str());
            throw std::runtime_error("savePcd: writing " + path + " failed");
        }
    }
    // The node's map topics as serialised ROS1 messages (DESIGN.md f15, W1-W8), into a pinned byte buffer (PinnedBytes or
    // any std::vector-like buffer of bytes in pinned or device-visible memory; the library refuses pageable memory with
    // GEM_ERR_INVALID, so a plain std::vector throws) that a node can publish as it is, e.g. through
    // topic_tools::ShapeShifter.  Each call resizes `out` to the message and returns when the bytes are there.
    // rosGridMap: visual_map; rosOrthomosaic: orthomosaic; rosVisualPoints: visualpoints; rosCloud: history_point /
    // global_point of device or host record parts; rosOctomap: the last colorOctree; rosSubmap: dislam_msgs/SubMap of the
    // records, the received keyframe cloud's serialised bytes, this map's orthomosaic and the pose (xyz, then xyzw).
    template <class Buffer> size_t rosGridMap(const gem_ros_header &h, Buffer &out)
    {
        return rosInto(out, 0, "gem_ros_grid_map", [&](void *p, long long c, long long *nb) { return gem_ros_grid_map(h_, &h, p, c, nb); });
    }
    template <class Buffer> size_t rosOrthomosaic(const gem_ros_header &h, Buffer &out)
    {
        return rosInto(out, 0, "gem_ros_orthomosaic", [&](void *p, long long c, long long *nb) { return gem_ros_orthomosaic(h_, &h, p, c, nb); });
    }
    template <class Buffer> size_t rosVisualPoints(const gem_ros_header &h, Buffer &out)
    {
        return rosInto(out, 0, "gem_ros_visual_points", [&](void *p, long long c, long long *nb) { return gem_ros_visual_points(h_, &h, p, c, nb); });
    }
    template <class Buffer> size_t rosCloud(const gem_ros_header &h, const std::vector<gem_ros_part> &parts, Buffer &out, bool isDense = true)
    {
        return rosInto(out, 0, "gem_ros_cloud", [&](void *p, long long c, long long *nb) {
            return gem_ros_cloud(h_, &h, parts.data(), (int)parts.size(), isDense ? 1 : 0, p, c, nb);
        });
    }
    template <class Buffer> size_t rosOctomap(const gem_ros_header &h, Buffer &out)
    {
        return rosInto(out, 0, "gem_ros_octomap", [&](void *p, long long c, long long *nb) { return gem_ros_octomap(h_, &h, p, c, nb); });
    }
    template <class Buffer>
    size_t rosSubmap(const gem_ros_header &h, const void *records, size_t n, const void *keyframe, size_t keyframeBytes,
                     const double pose[7], Buffer &out, const gem_ros_header &imageHeader = gem_ros_header{0, 0, 0, ""},
                     bool isDense = true)
    {
        const gem_ros_part part{records, (long long)n};
        auto cloud = [&](void *p, long long c, long long *nb) { return gem_ros_cloud(h_, &h, &part, 1, isDense ? 1 : 0, p, c, nb); };
        auto image = [&](void *p, long long c, long long *nb) { return gem_ros_orthomosaic(h_, &imageHeader, p, c, nb); };
        long long nc = 0, ni = 0;
        check(cloud(nullptr, 0, &nc), "gem_ros_cloud");
        check(image(nullptr, 0, &ni), "gem_ros_orthomosaic");
        out.resize((size_t)nc + keyframeBytes + (size_t)ni + 7 * sizeof(double));
        rosInto(out, 0, "gem_ros_cloud", cloud, false);
        rosInto(out, (size_t)nc + keyframeBytes, "gem_ros_orthomosaic", image, false);
        sync();
        if (keyframeBytes) std::memcpy(&out[(size_t)nc], keyframe, keyframeBytes);
        std::memcpy(&out[out.size() - 7 * sizeof(double)], pose, 7 * sizeof(double));
        return out.size();
    }
    // What Costmap2DROS publishes (DESIGN.md f17): rosCostmap is one publishCostmap of a master grid (forceFull:
    // onNewSubscription's full grid) through a CostmapPublisher's state -- kind GEM_COSTMAP_PUB_FULL (OccupancyGrid),
    // _UPDATE (OccupancyGridUpdate) or _NONE (an empty message); rosFootprint is the PolygonStamped of the padded
    // footprint (x, y pairs) at the pose.  costmapFootprint clears the footprint in an ElevationMapLayer's grid as
    // ObstacleLayer does and returns the vertices' touch bounds.
    template <class Buffer>
    size_t rosCostmap(const gem_ros_header &h, const gem_costmap_window &w, const unsigned char *master_device, gem_costmap_publisher &p,
                      Buffer &out, int *kind, bool forceFull = false)
    {
        return rosInto(out, 0, "gem_ros_costmap", [&](void *q, long long c, long long *nb) {
            return gem_ros_costmap(h_, &h, &w, master_device, &p, forceFull ? 1 : 0, q, c, nb, kind);
        });
    }
    template <class Buffer>
    size_t rosFootprint(const gem_ros_header &h, const std::vector<double> &spec_xy, double x, double y, double yaw, Buffer &out)
    {
        return rosInto(out, 0, "gem_ros_footprint", [&](void *q, long long c, long long *nb) {
            return gem_ros_footprint(h_, &h, spec_xy.data(), (int)(spec_xy.size() / 2), x, y, yaw, q, c, nb);
        });
    }
    gem_costmap_marks costmapFootprint(const gem_costmap_window &w, const std::vector<double> &spec_xy, double x, double y, double yaw,
                                       unsigned char *layer_device)
    {
        gem_costmap_marks mk;
        check(gem_costmap_footprint(h_, &w, spec_xy.data(), (int)(spec_xy.size() / 2), x, y, yaw, layer_device, &mk), "gem_costmap_footprint");
        return mk;
    }
    // The costmap plugins fed from their subscribed messages (DESIGN.md f18).  gridMapMsgParse: fromMessage's geometry and
    // where `layer`'s floats are in a serialised grid_map_msgs/GridMap (host code, throws on a refused message);
    // costmapMarkGrid: ElevationMapLayer::updateBounds over such a layer's floats (device or pinned memory, any alignment,
    // e.g. msg_device + g.offset); decodePointCloud2Records: fromPCLPointCloud2 into whole 32-byte PointXYZRGBICT records.
    static gem_grid_map_layer gridMapMsgParse(const void *msg, size_t bytes, const std::string &layer = "traver")
    {
        gem_grid_map_layer g;
        if (gem_grid_map_msg_parse(msg, bytes, layer.c_str(), &g) != GEM_OK)
            throw std::runtime_error(std::string("gem_grid_map_msg_parse: ") + gem_last_error(nullptr));
        return g;
    }
    gem_costmap_marks costmapMarkGrid(const gem_grid_map_layer &g, const void *layer_device, const gem_costmap_window &w,
                                      unsigned char *cost_device, double traversThresh = 0.7, bool markUnknown = true)
    {
        gem_costmap_marks mk{};
        check(gem_costmap_mark_grid(h_, &g, layer_device, &w, traversThresh, markUnknown ? 1 : 0, cost_device, &mk), "gem_costmap_mark_grid");
        return mk;
    }
    void decodePointCloud2Records(const PointCloud2Layout &lay, const void *data_device, unsigned long long data_bytes,
                                  void *points32_out_device)
    {
        check(gem_decode_pointcloud2_records(h_, lay.layout(), data_device, data_bytes, points32_out_device),
              "gem_decode_pointcloud2_records");
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
    // The global map (DESIGN.md f16): globalMap_, trajectory_ and localMapLoc_ on the device, with updateGlobalMap in one
    // call.  Poses are row-major 4 x 4 floats (row 3 ignored); Eigen's Isometry3f::matrix().data() is column-major, so
    // transpose it first.  globalMapPush = the keyframe branch (:633-662), globalMapUpdate = updateGlobalMap (:773-905),
    // globalMapRecords = composingGlobalMap's cloudpt (:491-493), saveSubmaps = savingSubMap (:461-476).  Device pointers
    // from globalMapSubmap / globalMapRecords are valid until the next push, update, reserve or reset.
    void globalMapReset() { check(gem_global_map_reset(h_), "gem_global_map_reset"); }
    void globalMapReserve(long long records, int submaps = 0) { check(gem_global_map_reserve(h_, records, submaps), "gem_global_map_reserve"); }
    void globalMapPush(const void *records_device, size_t n, const float pose_rowmajor[16])
    {
        check(gem_global_map_push(h_, records_device, (int)n, pose_rowmajor), "gem_global_map_push");
    }
    int globalMapUpdate(const float *opt_poses_rowmajor, int k, double resolution, double radius = 25.0, bool compat_precedence = true)
    {
        int fused = 0;
        check(gem_global_map_update(h_, opt_poses_rowmajor, k, resolution, radius, compat_precedence ? 1 : 0, &fused), "gem_global_map_update");
        return fused;
    }
    int globalMapSubmaps()
    {
        int n = 0;
        check(gem_global_map_info(h_, &n, nullptr, nullptr), "gem_global_map_info");
        return n;
    }
    const void *globalMapSubmap(int i, int *count)
    {
        void *p = nullptr;
        check(gem_global_map_submap(h_, i, &p, count), "gem_global_map_submap");
        return p;
    }
    const void *globalMapRecords(long long *count)
    {
        void *p = nullptr;
        check(gem_global_map_records(h_, &p, count), "gem_global_map_records");
        return p;
    }
    void globalMapPose(int i, float pose_rowmajor[16], float centre[2]) { check(gem_global_map_pose(h_, i, pose_rowmajor, centre), "gem_global_map_pose"); }
    // every non-empty submap to directory + i + ".pcd" (directory ends with '/', like GEM's submap_saving_dir)
    void saveSubmaps(const std::string &directory, bool binary = false, bool rgbUint32 = false)
    {
        for (int i = 0, k = globalMapSubmaps(); i < k; i++) {
            int n = 0;
            const void *p = globalMapSubmap(i, &n);
            if (n > 0) savePcd(directory + std::to_string(i) + ".pcd", p, (size_t)n, true, binary, rgbUint32);
        }
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
    // one gem_ros_* call into out at byte `at`: with resize, out becomes the message (size query first) and the call is
    // waited for; without, out must already hold it
    template <class Buffer, class Call> size_t rosInto(Buffer &out, size_t at, const char *what, Call call, bool resize = true)
    {
        long long bytes = 0;
        if (resize) {
            check(call(nullptr, 0, &bytes), what);
            out.resize((size_t)bytes > 0 ? (size_t)bytes : 1); // an empty message (rosCostmap's NONE) still has a buffer to write to
        }
        check(call(&out[0] + at, (long long)(out.size() - at), &bytes), what);
        if ((size_t)bytes > out.size() - at) throw std::runtime_error(std::string(what) + ": the buffer is too small");
        if (resize) {
            out.resize((size_t)bytes);
            sync();
        }
        return (size_t)bytes;
    }
    static int pcdFlags(bool binary, bool rgbUint32) { return (binary ? GEM_PCD_BINARY : 0) | (rgbUint32 ? GEM_PCD_RGB_UINT32 : 0); }
    void check(int rc, const char *what)
    {
        if (rc != GEM_OK) throw std::runtime_error(std::string(what) + ": " + gem_last_error(h_));
    }
    gem_map *h_ = nullptr;
    int length_ = 0;
};

// Costmap2DPublisher's state for one costmap (DESIGN.md f17): feed LayeredCostmap::getBounds after each update once the
// costmap is initialised, then ElevationMap::rosCostmap(..., publisher.state, ...) at the publish rate
struct CostmapPublisher {
    gem_costmap_publisher state;
    explicit CostmapPublisher(bool alwaysSendFull = false) { gem_costmap_publisher_init(&state, alwaysSendFull ? 1 : 0); }
    void updateBounds(int x0, int xn, int y0, int yn) { gem_costmap_publisher_bounds(&state, x0, xn, y0, yn); }
};


// The descriptor of gem_grid_map_msg_parse from an already deserialised grid_map_msgs::GridMap (or any type with its
// field names), without ROS headers: G1-G3 of DESIGN.md f18 on the message's fields.  Returns false where
// gem_grid_map_msg_parse refuses (msg.layers.size() != msg.data.size(), the layer missing, a layout that is not
// column-major, sizes that do not match, too few floats, a bad resolution or length); else fills g (offset 0) and
// *floats with the layer's host floats, which the caller copies to the device for costmapMarkGrid.
template <class GridMapMsg>
bool gridMapLayerFromFields(const GridMapMsg &msg, const std::string &layer, gem_grid_map_layer &g, const float **floats)
{
    const double res = msg.info.resolution, lx = msg.info.length_x, ly = msg.info.length_y;
    if (msg.layers.size() != msg.data.size() || !(std::isfinite(res) && res > 0.0)) return false;
    long long found = -1;
    for (size_t i = 0; i < msg.layers.size(); i++)
        if (msg.layers[i] == layer) found = (long long)i; // G2: the last of a repeated name
    if (found < 0) return false;
    const auto &a = msg.data[(size_t)found];
    if (a.layout.dim.size() < 2 || a.layout.dim[0].label != "column_index") return false;
    int size[2];
    const double len[2] = {lx, ly};
    for (int k = 0; k < 2; k++) {
        if (!(std::isfinite(len[k]) && len[k] > 0.0)) return false;
        const double q = std::round(len[k] / res);
        if (!(q <= 2147483647.0)) return false;
        size[k] = (int)q;
    }
    const unsigned long long rows = a.layout.dim[1].size, cols = a.layout.dim[0].size;
    if ((long long)size[0] * size[1] > 2147483647ll || rows != (unsigned long long)size[0] || cols != (unsigned long long)size[1] ||
        (unsigned long long)a.data.size() < rows * cols)
        return false;
    std::memset(&g, 0, sizeof g);
    g.resolution = res;
    g.position_x = msg.info.pose.position.x;
    g.position_y = msg.info.pose.position.y;
    g.size_x = size[0];
    g.size_y = size[1];
    g.length_x = (double)size[0] * res;
    g.length_y = (double)size[1] * res;
    g.start_x = (int)msg.outer_start_index;
    g.start_y = (int)msg.inner_start_index;
    g.floats = (long long)size[0] * size[1];
    g.column_major = 1;
    if (floats) *floats = a.data.data();
    return true;
}

// layers/src/elevationMap_layer.cpp's ElevationMapLayer fed from serialised visual_map bytes (e.g. a
// topic_tools::ShapeShifter's): onMessage is elevationMapCB with its elevation_map_available_ gate (a message is kept only
// when none is pending; keeping it copies the layer's floats alone into a pinned buffer the device reads); updateBounds
// marks the layer grid from the pending message and consumes it, or marks nothing.  A refused message throws and leaves
// the layer as it was.  travers_thresh: the plugin's default 0.5; GEM's yaml sets 0.7.
class ElevationMapLayer {
  public:
    explicit ElevationMapLayer(ElevationMap &map, double traversThresh = 0.5, bool markUnknown = true, std::string layer = "traver")
        : map_(map), thresh_(traversThresh), markUnknown_(markUnknown), layer_(std::move(layer)) {}
    bool available() const { return pending_; }
    bool onMessage(const void *msg, size_t bytes)
    {
        if (pending_) return false;
        g_ = ElevationMap::gridMapMsgParse(msg, bytes, layer_);
        floats_.resize((size_t)g_.floats * 4 + 4);
        std::memcpy(&floats_[0], static_cast<const uint8_t *>(msg) + g_.offset, (size_t)g_.floats * 4);
        pending_ = true;
        return true;
    }
    gem_costmap_marks updateBounds(const gem_costmap_window &w, unsigned char *layer_grid_device)
    {
        if (!pending_) return noMarks();
        pending_ = false;
        return map_.costmapMarkGrid(g_, &floats_[0], w, layer_grid_device, thresh_, markUnknown_);
    }
    static gem_costmap_marks noMarks()
    {
        const double inf = std::numeric_limits<double>::infinity();
        return gem_costmap_marks{0, 0, inf, inf, -inf, -inf};
    }

  private:
    ElevationMap &map_;
    double thresh_;
    bool markUnknown_;
    std::string layer_;
    bool pending_ = false;
    gem_grid_map_layer g_{};
    PinnedBytes floats_;
};

// layers/src/pointMap_layer.cpp's PointMapLayer fed from history_point: onMessage is pointMapCB (the cloud, given by its
// layout and bytes in device or pinned memory, replaces the stored one, decoded into whole PointXYZRGBICT records in a
// pinned buffer); updateBounds re-marks the stored cloud every time, nothing before the first message.  Calls take effect
// in call order.  The records stay in pinned host memory, so each re-mark reads them across PCIe (32 bytes per point);
// for clouds of millions of points keep the records in device memory and call costmapMarkPoints on them instead.
class PointMapLayer {
  public:
    explicit PointMapLayer(ElevationMap &map, double traversThresh = 0.5) : map_(map), thresh_(traversThresh) {}
    void onMessage(const PointCloud2Layout &lay, const void *data, unsigned long long bytes)
    {
        gem_pc2_mapping mp;
        if (gem_pointcloud2_mapping(lay.layout(), bytes, &mp) != GEM_OK)
            throw std::runtime_error(std::string("gem_pointcloud2_mapping: ") + gem_last_error(nullptr));
        map_.sync(); // the stored records may still be read
        records_.resize((size_t)mp.points > 0 ? (size_t)mp.points : 1);
        map_.decodePointCloud2Records(lay, data, bytes, records_.data());
        n_ = (long long)mp.points;
    }
    gem_costmap_marks updateBounds(const gem_costmap_window &w, unsigned char *layer_grid_device)
    {
        if (n_ < 0) return ElevationMapLayer::noMarks();
        return map_.costmapMarkPoints(records_.data(), (size_t)n_, w, layer_grid_device, thresh_);
    }
    long long points() const { return n_; }
    const PointXYZRGBICT *records() const { return records_.data(); }

  private:
    ElevationMap &map_;
    double thresh_;
    long long n_ = -1;
    std::vector<PointXYZRGBICT, PinnedAllocator<PointXYZRGBICT>> records_;
};

} // namespace gem_b200
