"""ctypes binding of include/gem_b200.h.  Loads gem_b200/lib/libgem_b200.so and fails loudly if
it is missing: there is no Python/CPU fallback for the product path."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libgem_b200.so")

GEM_OK = 0
ERR_NAMES = {0: "GEM_OK", 1: "GEM_ERR_INVALID", 2: "GEM_ERR_CUDA", 3: "GEM_ERR_NO_DEVICE", 4: "GEM_ERR_NOMEM"}

SENSOR_LASER = 0
SENSOR_STRUCTURED_LIGHT = 1
SENSOR_STEREO = 2
SENSOR_PERFECT = 3

GRID_SOURCES = {"shown": 0, "snapshot": 1}   # GEM_GRID_SHOWN / GEM_GRID_SNAPSHOT

LAYERS = {"elevation": 0, "variance": 1, "intensity": 2, "color_r": 3, "color_g": 4, "color_b": 5,
          "traver": 6, "lowest": 7, "rough": 8, "slope": 9}
INT_LAYERS = {3, 4, 5}
# order of gem_export_layers / ElevationMap.cpp:44 visualMap_ layers
EXPORT_LAYERS = ["elevation", "variance", "rough", "slope", "traver", "color_r", "color_g", "color_b", "intensity"]


class GemConfig(C.Structure):
    _fields_ = [
        ("length", C.c_int), ("resolution", C.c_float), ("mahalanobis_threshold", C.c_float),
        ("obstacle_threshold", C.c_float), ("compat_box_filter", C.c_int), ("max_points", C.c_int),
        ("device", C.c_int), ("stream", C.c_void_p),
        ("tile_row0", C.c_int), ("tile_rows", C.c_int), ("tile_col0", C.c_int), ("tile_cols", C.c_int),
        ("grid_resolution", C.c_double),
    ]


class GemSensorModel(C.Structure):
    _fields_ = [
        ("type", C.c_int), ("min_radius", C.c_float), ("beam_angle", C.c_float), ("beam_constant", C.c_float),
        ("normal_factor_a", C.c_double), ("normal_factor_b", C.c_double), ("normal_factor_c", C.c_double),
        ("normal_factor_d", C.c_double), ("normal_factor_e", C.c_double), ("lateral_factor", C.c_double),
        ("cutoff_min_depth", C.c_double), ("cutoff_max_depth", C.c_double),
        ("stereo_p", C.c_double * 5), ("depth_to_disparity_factor", C.c_double), ("cloud_width", C.c_int),
    ]


class GemFrame(C.Structure):
    _fields_ = [
        ("T", C.c_float * 16), ("sensor_jacobian", C.c_float * 3), ("rotation_variance", C.c_float * 9),
        ("C_SB_transpose", C.c_float * 9), ("P_mul_C_BM_transpose", C.c_float * 3), ("B_r_BS_skew", C.c_float * 9),
        ("rel_lower", C.c_double), ("rel_upper", C.c_double), ("sensor", GemSensorModel),
    ]


class GemStats(C.Structure):
    _fields_ = [("points_in", C.c_longlong), ("points_binned", C.c_longlong), ("cells_touched", C.c_longlong),
                ("max_points_per_cell", C.c_int)]


class GemTiledPeers(C.Structure):
    _fields_ = [("tiles_r", C.c_int), ("tiles_c", C.c_int), ("my_rank", C.c_int), ("bucket_capacity", C.c_int),
                ("recv_records", C.c_ulonglong * 64), ("recv_intensity", C.c_ulonglong * 64),
                ("recv_counts", C.c_ulonglong * 64), ("flags", C.c_ulonglong * 64)]


class GemProfile(C.Structure):
    _fields_ = [("launches", C.c_longlong), ("ms", C.c_double * 9), ("count", C.c_longlong * 9)]


class GemGridSplit(C.Structure):
    _fields_ = [("points", C.c_int), ("valid", C.c_int), ("road", C.c_int), ("obstacle", C.c_int),
                ("mean", C.c_double), ("stddev", C.c_double), ("threshold", C.c_double)]


class GemOctree(C.Structure):
    _fields_ = [("bytes", C.c_longlong), ("nodes", C.c_int), ("leaves", C.c_int), ("inserted", C.c_int), ("skipped", C.c_int)]


class GemCostmapWindow(C.Structure):
    _fields_ = [("origin_x", C.c_double), ("origin_y", C.c_double), ("resolution", C.c_double), ("size_x", C.c_int),
                ("size_y", C.c_int)]


class GemCostmapMarks(C.Structure):
    _fields_ = [("marked", C.c_longlong), ("lethal", C.c_longlong), ("min_x", C.c_double), ("min_y", C.c_double),
                ("max_x", C.c_double), ("max_y", C.c_double)]


class GemCostmapInflation(C.Structure):
    _fields_ = [("inflation_radius", C.c_double), ("cost_scaling_factor", C.c_double), ("inscribed_radius", C.c_double),
                ("inflate_unknown", C.c_int)]


class GemVoxelGridParams(C.Structure):
    _fields_ = [("leaf_size", C.c_float * 3), ("field", C.c_int), ("limit_min", C.c_double), ("limit_max", C.c_double),
                ("limit_negative", C.c_int)]


class GemVoxelGridInfo(C.Structure):
    _fields_ = [("count", C.c_int), ("used", C.c_int), ("passthrough", C.c_int)]


PREFILTER_MAX_STEPS = 4


class GemPrefilter(C.Structure):
    _fields_ = [("nsteps", C.c_int), ("step", GemVoxelGridParams * PREFILTER_MAX_STEPS)]


class GemProjection(C.Structure):
    _fields_ = [("T_camera", C.c_double * 12), ("T_lidar", C.c_double * 16), ("width", C.c_int), ("height", C.c_int),
                ("row_stride", C.c_int)]


class GemMlsParams(C.Structure):
    _fields_ = [("search_radius", C.c_double), ("sqr_gauss_param", C.c_double), ("polynomial_fit", C.c_int), ("order", C.c_int),
                ("upsampling", C.c_int), ("point_density", C.c_int), ("seed", C.c_ulonglong)]


class GemMlsInfo(C.Structure):
    _fields_ = [("count", C.c_longlong), ("processed", C.c_int), ("fitted", C.c_int), ("skipped", C.c_int),
                ("max_neighbours", C.c_int)]


class GemPointField(C.Structure):
    _fields_ = [("name", C.c_char * 32), ("offset", C.c_uint), ("datatype", C.c_ubyte), ("count", C.c_uint)]


class GemPointCloud2(C.Structure):
    _fields_ = [("width", C.c_uint), ("height", C.c_uint), ("point_step", C.c_uint), ("row_step", C.c_uint),
                ("is_bigendian", C.c_ubyte), ("nfields", C.c_int), ("fields", C.POINTER(GemPointField))]


class GemPc2Span(C.Structure):
    _fields_ = [("serialized_offset", C.c_uint), ("struct_offset", C.c_uint), ("size", C.c_uint)]


class GemPc2Mapping(C.Structure):
    _fields_ = [("nspans", C.c_int), ("spans", GemPc2Span * 7), ("fast_path", C.c_int), ("matched", C.c_uint),
                ("points", C.c_longlong), ("bytes", C.c_ulonglong)]


class GemCameraImage(C.Structure):
    _fields_ = [("T_camera", C.c_double * 12), ("T_lidar", C.c_double * 16), ("encoding", C.c_char * 32), ("width", C.c_int),
                ("height", C.c_int), ("step", C.c_int), ("data", C.c_void_p)]


class GemRosHeader(C.Structure):
    _fields_ = [("seq", C.c_uint), ("stamp_sec", C.c_uint), ("stamp_nsec", C.c_uint), ("frame_id", C.c_char_p)]


class GemRosPart(C.Structure):
    _fields_ = [("points32", C.c_void_p), ("n", C.c_longlong)]


class GemCostmapPublisher(C.Structure):
    _fields_ = [("always_send_full", C.c_int), ("saved", C.c_int), ("resolution", C.c_float), ("size_x", C.c_int),
                ("size_y", C.c_int), ("origin_x", C.c_double), ("origin_y", C.c_double), ("x0", C.c_int), ("xn", C.c_int),
                ("y0", C.c_int), ("yn", C.c_int)]


class GemGridMapLayer(C.Structure):
    _fields_ = [("resolution", C.c_double), ("position_x", C.c_double), ("position_y", C.c_double), ("length_x", C.c_double),
                ("length_y", C.c_double), ("size_x", C.c_int), ("size_y", C.c_int), ("start_x", C.c_int), ("start_y", C.c_int),
                ("offset", C.c_ulonglong), ("floats", C.c_longlong), ("column_major", C.c_int)]


COST_FREE, COST_LETHAL, COST_UNKNOWN = 0, 254, 255           # GEM_COST_*
INFLATE_MAX_CELLS = 4094                                     # GEM_INFLATE_MAX_CELLS
COSTMAP_MODES = {"max": 0, "overwrite": 1}                  # GEM_COSTMAP_MAX / GEM_COSTMAP_OVERWRITE
VOXEL_FIELDS = {None: -1, "x": 0, "y": 1, "z": 2, "intensity": 3}  # GEM_VOXEL_FIELD_*
MLS_UPSAMPLING = {"none": 0, "random_uniform_density": 1}  # GEM_MLS_*
# sensor_msgs/PointField datatypes (GEM_PF_*) and the PointXYZRGBICT fields in registration order (GEM_PC2_*)
POINTFIELD_TYPES = {"int8": 1, "uint8": 2, "int16": 3, "uint16": 4, "int32": 5, "uint32": 6, "float32": 7, "float64": 8}
PC2_FIELDS = ["x", "y", "z", "rgb", "intensity", "covariance", "travers"]
PCD_BINARY, PCD_RGB_UINT32 = 1, 2   # GEM_PCD_*
COSTMAP_PUB_KINDS = {0: "none", 1: "full", 2: "update"}   # GEM_COSTMAP_PUB_*
PCD_LINE_MAX, PCD_HEADER_MAX = 105, 512   # GEM_PCD_LINE_MAX, GEM_PCD_HEADER_MAX
COLOUR_LOOKUPS = {"image": 0, "node": 1}   # GEM_COLOUR_LOOKUP_IMAGE / _NODE (gem_set_colour_lookup)
IMAGE_ENCODINGS = {"bgr8": 3, "rgb8": 3, "bgra8": 4, "rgba8": 4, "mono8": 1}   # the byte-permutation encodings: channels

PROF_CLASSES = ["bin", "fold_long", "unused", "fold", "clear_floor", "features", "raytrace", "other", "route"]

# every symbol include/gem_b200.h declares: name -> (restype, argtypes)
_P = C.c_void_p
_FP = C.POINTER(C.c_float)
_IP = C.POINTER(C.c_int)
SYMBOLS = {
    "gem_version": (C.c_int, []),
    "gem_last_error": (C.c_char_p, [_P]),
    "gem_create": (C.c_int, [C.POINTER(GemConfig), C.POINTER(_P)]),
    "gem_destroy": (C.c_int, [_P]),
    "gem_sync": (C.c_int, [_P]),
    "gem_get_stream": (C.c_void_p, [_P]),
    "gem_flush": (C.c_int, [_P]),
    "gem_debug_stamps": (C.c_int, [_P, C.c_int, C.POINTER(C.c_ulonglong)]),
    "gem_move": (C.c_int, [_P, _FP, _FP, _IP, _FP]),
    "gem_add_points": (C.c_int, [_P, _P, _P, C.c_int, C.POINTER(GemFrame)]),
    "gem_add_points_host": (C.c_int, [_P, _P, _P, C.c_int, C.POINTER(GemFrame)]),
    "gem_add_points_stream": (C.c_int, [_P, _P, _P, C.c_int, C.POINTER(GemFrame)]),
    "gem_add_points_multi": (C.c_int, [_P, _P, _P, C.c_int, _IP, C.POINTER(GemFrame)]),
    "gem_add_points_host_async": (C.c_int, [_P, _P, _P, C.c_int, C.POINTER(GemFrame)]),
    "gem_add_cloud_pcl_host": (C.c_int, [_P, _P, C.c_int, C.POINTER(GemFrame)]),
    "gem_process_points": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.POINTER(GemFrame)]),
    "gem_fuse": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, _P, _P, _P]),
    "gem_var_update": (C.c_int, [_P, C.c_float]),
    "gem_map_feature": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "gem_compute_features": (C.c_int, [_P]),
    "gem_raytracing": (C.c_int, [_P]),
    "gem_opt_move": (C.c_int, [_P, _FP, C.c_float, _FP]),
    "gem_closeloop": (C.c_int, [_P, _FP, C.c_float]),
    "gem_colourise_points": (C.c_int, [_P, _P, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), _P, C.c_int, C.c_int, C.c_int, _P]),
    "gem_set_colour_lookup": (C.c_int, [_P, C.c_int]),
    "gem_export_layers": (C.c_int, [_P, C.POINTER(_P)]),
    "gem_export_layers_begin": (C.c_int, [_P, C.POINTER(_P)]),
    "gem_export_layers_end": (C.c_int, [_P]),
    "gem_get_layer": (C.c_int, [_P, C.c_int, _P]),
    "gem_set_layer": (C.c_int, [_P, C.c_int, _P]),
    "gem_get_state": (C.c_int, [_P, _FP, _IP, _FP]),
    "gem_get_stats": (C.c_int, [_P, C.POINTER(GemStats)]),
    "gem_profile_enable": (C.c_int, [_P, C.c_int]),
    "gem_profile_read": (C.c_int, [_P, C.POINTER(GemProfile), C.c_int]),
    "gem_selftest_division": (C.c_int, [_P, C.c_ulonglong, C.c_ulonglong, C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong)]),
    "gem_host_alloc": (C.c_int, [C.POINTER(_P), C.c_ulonglong]),
    "gem_host_free": (C.c_int, [_P]),
    "gem_route_points": (C.c_int, [_P, _P, _P, C.c_int, C.POINTER(GemFrame), C.c_int, C.c_int, _P, _P, C.c_int]),
    "gem_fuse_records": (C.c_int, [_P, _P, C.c_int]),
    "gem_export_orthomosaic": (C.c_int, [_P, _P]),
    "gem_export_visual_points": (C.c_int, [_P, _P, _P, C.c_int, C.POINTER(C.c_int)]),
    "gem_snapshot_shown": (C.c_int, [_P]),
    "gem_harvest_scrolled_out": (C.c_int, [_P, C.POINTER(C.c_float), C.POINTER(C.c_float), _P, C.c_int, C.POINTER(C.c_int)]),
    "gem_export_grid_cloud": (C.c_int, [_P, C.c_int, _P, C.c_int, C.POINTER(C.c_int)]),
    "gem_harvest_to_local_map": (C.c_int, [_P, C.POINTER(C.c_float), C.POINTER(C.c_float), _P, C.c_int, C.POINTER(C.c_int)]),
    "gem_local_map_take": (C.c_int, [_P, _P, C.c_int, C.POINTER(C.c_int)]),
    "gem_local_map_clear": (C.c_int, [_P]),
    "gem_local_map_reserve": (C.c_int, [_P, C.c_int]),
    "gem_grid_cloud_split": (C.c_int, [_P, C.c_int, C.c_int, C.c_double, C.c_double, _P, C.c_int, _P, C.c_int, _P, C.c_int,
                                       C.POINTER(GemGridSplit)]),
    "gem_color_octree": (C.c_int, [_P, _P, C.c_int, C.c_double, C.POINTER(GemOctree)]),
    "gem_color_octree_read": (C.c_int, [_P, _P, C.c_longlong]),
    "gem_costmap_mark_map": (C.c_int, [_P, C.c_int, C.POINTER(GemCostmapWindow), C.c_double, C.c_int, _P,
                                       C.POINTER(GemCostmapMarks)]),
    "gem_costmap_mark_points": (C.c_int, [_P, _P, C.c_int, C.POINTER(GemCostmapWindow), C.c_double, _P,
                                          C.POINTER(GemCostmapMarks)]),
    "gem_costmap_update_origin": (C.c_int, [_P, C.POINTER(GemCostmapWindow), C.c_double, C.c_double, C.c_ubyte, _P]),
    "gem_costmap_combine": (C.c_int, [_P, C.c_int, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "gem_costmap_inflate": (C.c_int, [_P, C.POINTER(GemCostmapWindow), C.POINTER(GemCostmapInflation), _P, C.c_int, C.c_int,
                                      C.c_int, C.c_int]),
    "gem_voxel_grid": (C.c_int, [_P, _P, C.c_int, C.POINTER(GemVoxelGridParams), _P, C.c_int, C.POINTER(GemVoxelGridInfo)]),
    "gem_mls_upsample": (C.c_int, [_P, _P, C.c_int, C.POINTER(GemMlsParams), _P, C.c_longlong, C.POINTER(GemMlsInfo)]),
    "gem_get_layer_device": (C.c_int, [_P, C.c_int, _P]),
    "gem_compute_features_tiled": (C.c_int, [_P, _P]),
    "gem_raytracing_tiled": (C.c_int, [_P, _P]),
    "gem_transform_cloud": (C.c_int, [_P, _P, C.c_int, _FP]),
    "gem_refuse_submaps": (C.c_int, [_P, _P, _IP, _P, _IP, C.c_double, C.c_int, _IP]),
    "gem_global_map_reset": (C.c_int, [_P]),
    "gem_global_map_reserve": (C.c_int, [_P, C.c_longlong, C.c_int]),
    "gem_global_map_push": (C.c_int, [_P, _P, C.c_int, _FP]),
    "gem_global_map_update": (C.c_int, [_P, _FP, C.c_int, C.c_double, C.c_double, C.c_int, _IP]),
    "gem_global_map_info": (C.c_int, [_P, _IP, _IP, C.POINTER(C.c_longlong)]),
    "gem_global_map_submap": (C.c_int, [_P, C.c_int, C.POINTER(_P), _IP]),
    "gem_global_map_records": (C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_longlong)]),
    "gem_global_map_pose": (C.c_int, [_P, C.c_int, _FP, _FP]),
    "gem_global_map_stream": (_P, [_P]),
    "gem_tiled_attach": (C.c_int, [_P, C.POINTER(GemTiledPeers)]),
    "gem_tiled_step": (C.c_int, [_P, _P, _P, C.c_int, C.POINTER(GemFrame)]),
    "gem_pointcloud2_mapping": (C.c_int, [C.POINTER(GemPointCloud2), C.c_ulonglong, C.POINTER(GemPc2Mapping)]),
    "gem_decode_pointcloud2": (C.c_int, [_P, C.POINTER(GemPointCloud2), _P, C.c_ulonglong, _P]),
    "gem_image_to_bgr8": (C.c_int, [_P, C.c_char_p, _P, C.c_int, C.c_int, C.c_int, _P, C.c_int]),
    "gem_add_pointcloud2_host_async": (C.c_int, [_P, C.POINTER(GemPointCloud2), _P, C.c_ulonglong, C.POINTER(GemCameraImage),
                                                 C.POINTER(GemFrame)]),
    "gem_add_pointcloud2_filtered_host_async": (C.c_int, [_P, C.POINTER(GemPointCloud2), _P, C.c_ulonglong,
                                                          C.POINTER(GemCameraImage), C.POINTER(GemPrefilter), C.POINTER(GemFrame)]),
    "gem_add_points_filtered_stream": (C.c_int, [_P, _P, C.c_int, C.POINTER(GemPrefilter), _P, C.POINTER(GemProjection),
                                                 C.POINTER(GemFrame)]),
    "gem_prefilter_info": (C.c_int, [_P, C.POINTER(GemVoxelGridInfo), C.c_int]),
    "gem_pcd_header": (C.c_int, [C.c_longlong, C.c_int, C.c_char_p, C.c_int, _IP]),
    "gem_pcd_format": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, C.c_longlong, C.POINTER(C.c_longlong)]),
    "gem_ros_grid_map": (C.c_int, [_P, C.POINTER(GemRosHeader), _P, C.c_longlong, C.POINTER(C.c_longlong)]),
    "gem_ros_orthomosaic": (C.c_int, [_P, C.POINTER(GemRosHeader), _P, C.c_longlong, C.POINTER(C.c_longlong)]),
    "gem_ros_visual_points": (C.c_int, [_P, C.POINTER(GemRosHeader), _P, C.c_longlong, C.POINTER(C.c_longlong)]),
    "gem_ros_cloud": (C.c_int, [_P, C.POINTER(GemRosHeader), C.POINTER(GemRosPart), C.c_int, C.c_int, _P, C.c_longlong,
                                C.POINTER(C.c_longlong)]),
    "gem_ros_octomap": (C.c_int, [_P, C.POINTER(GemRosHeader), _P, C.c_longlong, C.POINTER(C.c_longlong)]),
    "gem_costmap_publisher_init": (C.c_int, [C.POINTER(GemCostmapPublisher), C.c_int]),
    "gem_costmap_publisher_bounds": (C.c_int, [C.POINTER(GemCostmapPublisher), C.c_int, C.c_int, C.c_int, C.c_int]),
    "gem_ros_costmap": (C.c_int, [_P, C.POINTER(GemRosHeader), C.POINTER(GemCostmapWindow), _P, C.POINTER(GemCostmapPublisher),
                                  C.c_int, _P, C.c_longlong, C.POINTER(C.c_longlong), _IP]),
    "gem_ros_footprint": (C.c_int, [_P, C.POINTER(GemRosHeader), C.POINTER(C.c_double), C.c_int, C.c_double, C.c_double,
                                    C.c_double, _P, C.c_longlong, C.POINTER(C.c_longlong)]),
    "gem_costmap_footprint": (C.c_int, [_P, C.POINTER(GemCostmapWindow), C.POINTER(C.c_double), C.c_int, C.c_double, C.c_double,
                                        C.c_double, _P, C.POINTER(GemCostmapMarks)]),
    "gem_grid_map_msg_parse": (C.c_int, [_P, C.c_ulonglong, C.c_char_p, C.POINTER(GemGridMapLayer)]),
    "gem_costmap_mark_grid": (C.c_int, [_P, C.POINTER(GemGridMapLayer), _P, C.POINTER(GemCostmapWindow), C.c_double, C.c_int, _P,
                                        C.POINTER(GemCostmapMarks)]),
    "gem_decode_pointcloud2_records": (C.c_int, [_P, C.POINTER(GemPointCloud2), _P, C.c_ulonglong, _P]),
}

_lib = None


def load() -> C.CDLL:
    """dlopen the library and bind every prototype.  Raises if the extension is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m gem_b200.build` "
            "(or __graft_entry__.build()).  gem_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class GemError(RuntimeError):
    pass


def check(rc: int, handle=None, what: str = "") -> None:
    if rc != GEM_OK:
        lib = load()
        msg = lib.gem_last_error(handle)
        raise GemError(f"{what}: {ERR_NAMES.get(rc, rc)}: {msg.decode() if msg else ''}")
