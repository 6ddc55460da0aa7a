"""Python mirror of the reference's map / sensor-processor interface on top of the C ABI.

Names follow the reference: ``ElevationMap`` (ElevationMap.hpp) with the upstream
``add`` / ``fuse`` / ``clean`` vocabulary BASELINE.json uses, the nine free functions of
gpu_process.cu (``move``, ``process_points``, ``fuse_points``, ``var_update``, ``map_feature``,
``raytracing``, ``opt_move``, ``closeloop``) and the sensor processors of
sensor_processors/*.cpp reduced to what reaches the GPU (SPB.cpp:171-206, 270-290).

This is test/bench plumbing over libgem_b200.so; all arithmetic happens in the CUDA library.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field

import numpy as np

from . import _lib
from ._lib import GemConfig, GemFrame, GemSensorModel, GemStats, check


# ------------------------------------------------------------------------------------------
# sensor processors (parameter holders; config/sensor_processors/*.yaml)
# ------------------------------------------------------------------------------------------
@dataclass
class LaserSensorProcessor:
    """sensor_processor/type: laser (LaserSensorProcessor.cpp:38-47, velodyne.yaml)."""
    min_radius: float = 0.018
    beam_angle: float = 0.0006
    beam_constant: float = 0.0015
    ignore_points_above: float = 0.8
    ignore_points_below: float = -5.0

    def model(self) -> GemSensorModel:
        return GemSensorModel(_lib.SENSOR_LASER, self.min_radius, self.beam_angle, self.beam_constant,
                              0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0)


@dataclass
class StructuredLightSensorProcessor:
    """sensor_processor/type: structured_light (StructuredLightSensorProcessor.cpp:36-48,
    realsense_d435.yaml)."""
    normal_factor_a: float = 0.000611
    normal_factor_b: float = 0.003587
    normal_factor_c: float = 0.3515
    normal_factor_d: float = 0.0
    normal_factor_e: float = 1.0
    lateral_factor: float = 0.01576
    cutoff_min_depth: float = 0.2
    cutoff_max_depth: float = 3.25
    ignore_points_above: float = float("inf")
    ignore_points_below: float = float("-inf")

    def model(self) -> GemSensorModel:
        return GemSensorModel(_lib.SENSOR_STRUCTURED_LIGHT, 0.0, 0.0, 0.0, self.normal_factor_a,
                              self.normal_factor_b, self.normal_factor_c, self.normal_factor_d,
                              self.normal_factor_e, self.lateral_factor, self.cutoff_min_depth, self.cutoff_max_depth)


@dataclass
class StereoSensorProcessor:
    """sensor_processor/type: stereo (StereoSensorProcessor.cpp:23-34, aslam.yaml).  Every parameter defaults to the
    node's 0.0.  cloud_width: pointCloud->width of the organised cloud the calls receive (0 = unorganised); the
    model reads each point's pixel row and column from its index in that cloud."""
    p_1: float = 0.0
    p_2: float = 0.0
    p_3: float = 0.0
    p_4: float = 0.0
    p_5: float = 0.0
    lateral_factor: float = 0.0
    depth_to_disparity_factor: float = 0.0
    cloud_width: int = 0
    ignore_points_above: float = float("inf")
    ignore_points_below: float = float("-inf")

    def model(self) -> GemSensorModel:
        m = GemSensorModel(_lib.SENSOR_STEREO)
        m.lateral_factor = self.lateral_factor
        m.stereo_p[:] = [self.p_1, self.p_2, self.p_3, self.p_4, self.p_5]
        m.depth_to_disparity_factor = self.depth_to_disparity_factor
        m.cloud_width = int(self.cloud_width)
        return m


@dataclass
class PerfectSensorProcessor:
    """sensor_processor/type: perfect (PerfectSensorProcessor.cpp, perfect.yaml): zero sensor variance.  Its
    readParameters does not call the base class (:36-39), so the height window is always the constructor's +-inf
    (SensorProcessorBase.cpp:39-40): there are no ignore_points_* to set."""

    @property
    def ignore_points_above(self) -> float:
        return float("inf")

    @property
    def ignore_points_below(self) -> float:
        return float("-inf")

    def model(self) -> GemSensorModel:
        return GemSensorModel(_lib.SENSOR_PERFECT)


def make_frame(T, sensor, base_z: float = 0.0, rotation_variance=None, C_SB_transpose=None,
               P_mul_C_BM_transpose=None, B_r_BS_skew=None, sensor_jacobian=None) -> GemFrame:
    """Per-frame constants as SensorProcessorBase::GPUPointCloudprocess derives them.

    T: 4x4 map<-sensor (SPB.cpp:171-179, double->float cast).  sensor_jacobian defaults to
    row 3 of its rotation (SPB.cpp:275).  rel thresholds = base_z + ignore_points_{below,above}
    in double (SPB.cpp:183-184).  rotation_variance defaults to zero (SPB.cpp:202-204).
    """
    T = np.asarray(T, dtype=np.float64).reshape(4, 4).astype(np.float32)
    f = GemFrame()
    f.T[:] = T.reshape(-1).tolist()
    sj = T[2, :3] if sensor_jacobian is None else np.asarray(sensor_jacobian, np.float32)
    f.sensor_jacobian[:] = [float(v) for v in sj]
    rv = np.zeros(9, np.float32) if rotation_variance is None else np.asarray(rotation_variance, np.float32).reshape(-1)
    f.rotation_variance[:] = rv.tolist()
    cs = np.eye(3, dtype=np.float32).reshape(-1) if C_SB_transpose is None else np.asarray(C_SB_transpose, np.float32).reshape(-1)
    f.C_SB_transpose[:] = cs.tolist()
    pm = np.array([0, 0, 1], np.float32) if P_mul_C_BM_transpose is None else np.asarray(P_mul_C_BM_transpose, np.float32)
    f.P_mul_C_BM_transpose[:] = pm.tolist()
    bs = np.zeros(9, np.float32) if B_r_BS_skew is None else np.asarray(B_r_BS_skew, np.float32).reshape(-1)
    f.B_r_BS_skew[:] = bs.tolist()
    f.rel_lower = float(base_z) + float(sensor.ignore_points_below)
    f.rel_upper = float(base_z) + float(sensor.ignore_points_above)
    f.sensor = sensor.model()
    return f


def _ptr(a):
    """pointer of a numpy array, a torch tensor (host or device) or a raw int address"""
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    if isinstance(a, np.ndarray):
        return C.c_void_p(a.ctypes.data)
    if hasattr(a, "data_ptr"):
        return C.c_void_p(a.data_ptr())
    raise TypeError(type(a))


def _is_device(a) -> bool:
    return hasattr(a, "is_cuda") and bool(a.is_cuda)


# ------------------------------------------------------------------------------------------
# raw sensor messages (DESIGN.md f12)
# ------------------------------------------------------------------------------------------
_NP_POINTFIELD = {("i", 1): 1, ("u", 1): 2, ("i", 2): 3, ("u", 2): 4, ("i", 4): 5, ("u", 4): 6, ("f", 4): 7, ("f", 8): 8}


class PointCloud2Layout:
    """sensor_msgs/PointCloud2's layout as gem_pointcloud2: `c` is the C struct, `fields` the (name, offset, datatype, count)
    list it was built from (kept alive with the C array)."""

    def __init__(self, fields, width: int, height: int = 1, point_step: int | None = None, row_step: int | None = None,
                 is_bigendian: int = 0):
        if isinstance(fields, np.dtype):
            dt = fields
            point_step = dt.itemsize if point_step is None else point_step
            fields = []
            for name in dt.names:
                ft, off = dt.fields[name][:2]
                base, shape = (ft.subdtype if ft.subdtype else (ft, ()))
                key = (base.kind, base.itemsize)
                if key not in _NP_POINTFIELD:
                    raise ValueError(f"PointCloud2Layout: field {name!r} has no PointField datatype ({base})")
                fields.append((name, off, _NP_POINTFIELD[key], int(np.prod(shape)) if shape else 1))
        self.fields = [(str(n), int(o), _lib.POINTFIELD_TYPES[d] if isinstance(d, str) else int(d), int(c))
                       for n, o, d, c in fields]
        if point_step is None:
            raise ValueError("PointCloud2Layout: point_step is needed with a field list")
        self._arr = (_lib.GemPointField * max(len(self.fields), 1))()
        for k, (n, o, d, c) in enumerate(self.fields):
            nb = n.encode()[:32]      # 32 bytes leave no NUL: such a name matches nothing, like any longer than 31 bytes
            C.memmove(C.addressof(self._arr[k]) + _lib.GemPointField.name.offset, nb, len(nb))
            self._arr[k].offset, self._arr[k].datatype, self._arr[k].count = o, d, c
        self.width, self.height, self.point_step = int(width), int(height), int(point_step)
        self.row_step = self.width * self.point_step if row_step is None else int(row_step)
        self.c = _lib.GemPointCloud2(self.width, self.height, self.point_step, self.row_step, int(is_bigendian),
                                     len(self.fields), C.cast(self._arr, C.POINTER(_lib.GemPointField)))

    @property
    def points(self) -> int:
        return self.width * self.height


def _host_bytes(a):
    """(pointer, bytes) of host memory: a numpy array, bytes / bytearray, or a CPU torch tensor (pinned or not)"""
    if isinstance(a, (bytes, bytearray, memoryview)):
        a = np.frombuffer(a, np.uint8)
    if isinstance(a, np.ndarray):
        if not a.flags.c_contiguous:
            raise ValueError("host buffer must be contiguous")
        return C.c_void_p(a.ctypes.data), int(a.nbytes)
    if hasattr(a, "data_ptr") and not _is_device(a):
        return C.c_void_p(a.data_ptr()), int(a.numel() * a.element_size())
    raise TypeError(f"not a host buffer: {type(a)}")


class CameraImage:
    """gem_camera_image: an 8-bit image in host memory (numpy array or CPU tensor, pinned or pageable) with the
    camera-lidar calibration of gem_colourise_points; `c` is the C struct"""

    def __init__(self, T_camera, T_lidar, encoding: str, data, width: int, height: int, step: int | None = None):
        if encoding not in _lib.IMAGE_ENCODINGS:
            raise ValueError(f"CameraImage: encoding {encoding!r} is not one of {list(_lib.IMAGE_ENCODINGS)}")
        self.data = data
        ptr, _ = _host_bytes(data)
        step = _lib.IMAGE_ENCODINGS[encoding] * int(width) if step is None else int(step)
        self.c = _lib.GemCameraImage()
        self.c.T_camera[:] = [float(v) for v in np.asarray(T_camera, np.float64).reshape(-1)]
        self.c.T_lidar[:] = [float(v) for v in np.asarray(T_lidar, np.float64).reshape(-1)]
        self.c.encoding = encoding.encode()
        self.c.width, self.c.height, self.c.step, self.c.data = int(width), int(height), step, ptr


# ------------------------------------------------------------------------------------------
@dataclass
class RosHeader:
    """std_msgs/Header as the gem_ros_* calls write it (DESIGN.md f15 W1): seq, stamp (sec, nsec) and frame_id, as given"""
    seq: int = 0
    stamp_sec: int = 0
    stamp_nsec: int = 0
    frame_id: str = ""

    def c(self) -> _lib.GemRosHeader:
        return _lib.GemRosHeader(int(self.seq), int(self.stamp_sec), int(self.stamp_nsec), self.frame_id.encode())


class ElevationMap:
    """One robot-centric elevation grid resident on one H100.

    Replaces the process-global state of gpu_process.cu:20-56 and the nine free functions that
    act on it; layer layout as in the reference (row-major L*L, storage indexed)."""

    def __init__(self, length: int, resolution: float, mahalanobis_threshold: float = 2.5,
                 obstacle_threshold: float = 0.7, compat_box_filter: bool = True, max_points: int = 0,
                 device: int = -1, stream=None, tile=None, grid_resolution: float = 0.0):
        self._lib = _lib.load()
        cfg = GemConfig()
        cfg.length = int(length)
        cfg.resolution = float(resolution)
        cfg.mahalanobis_threshold = float(mahalanobis_threshold)
        cfg.obstacle_threshold = float(obstacle_threshold)
        cfg.compat_box_filter = 1 if compat_box_filter else 0
        cfg.max_points = int(max_points)
        cfg.device = int(device)
        cfg.stream = stream
        cfg.grid_resolution = float(grid_resolution)   # the node's double resolution_ (grid_map positions); 0 = float one
        if tile is not None:
            cfg.tile_row0, cfg.tile_rows, cfg.tile_col0, cfg.tile_cols = [int(v) for v in tile]
        self._h = C.c_void_p()
        rc = self._lib.gem_create(C.byref(cfg), C.byref(self._h))
        if rc != 0:
            msg = self._lib.gem_last_error(None)
            raise _lib.GemError(f"gem_create: {_lib.ERR_NAMES.get(rc, rc)}: {msg.decode() if msg else ''}")
        self.length = int(length)
        self.resolution = float(resolution)
        self._cfg_device = int(device)
        self.tile = tile
        self.ncells = (tile[1] * tile[3]) if tile is not None else self.length * self.length
        self.shape = (tile[1], tile[3]) if tile is not None else (self.length, self.length)

    # -- lifetime -------------------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.gem_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        check(self._lib.gem_sync(self._h), self._h, "gem_sync")

    @property
    def handle(self):
        return self._h

    @property
    def cuda_stream(self) -> int:
        """cudaStream_t (as int) that all work of this map is ordered on"""
        return int(self._lib.gem_get_stream(self._h) or 0)

    def torch_stream(self):
        import torch
        return torch.cuda.ExternalStream(self.cuda_stream)

    def debug_stamps(self, enable=True):
        out = (C.c_ulonglong * 16)()
        check(self._lib.gem_debug_stamps(self._h, 1 if enable else 0, out), self._h, "gem_debug_stamps")
        return [int(v) for v in out]

    def flush(self):
        """enqueue the work the pipelined add calls deferred (no host wait)"""
        check(self._lib.gem_flush(self._h), self._h, "gem_flush")

    # -- Move (gpu.cu:1004) -----------------------------------------------------------------
    def move(self, position):
        pos = (C.c_float * 3)(*[float(v) for v in position])
        centre = (C.c_float * 2)()
        start = (C.c_int * 2)()
        shift = (C.c_float * 2)()
        check(self._lib.gem_move(self._h, pos, centre, start, shift), self._h, "gem_move")
        return np.array(centre[:], np.float32), np.array(start[:], np.int32), np.array(shift[:], np.float32)

    def move_fast(self, pos_c):
        """gem_move with a prebuilt (c_float*3) and no outputs: minimal host overhead per frame"""
        rc = self._lib.gem_move(self._h, pos_c, None, None, None)
        if rc:
            check(rc, self._h, "gem_move")

    def add_fast(self, xyzi_ptr, rgba_ptr, n: int, frame_ref):
        """gem_add_points with raw device addresses (c_void_p) and a byref'd gem_frame"""
        rc = self._lib.gem_add_points(self._h, xyzi_ptr, rgba_ptr, n, frame_ref)
        if rc:
            check(rc, self._h, "gem_add_points")

    def add_stream_fast(self, xyzi_ptr, rgba_ptr, n: int, frame_ref):
        """gem_add_points_stream: frame-pipelined add of a device-resident cloud"""
        rc = self._lib.gem_add_points_stream(self._h, xyzi_ptr, rgba_ptr, n, frame_ref)
        if rc:
            check(rc, self._h, "gem_add_points_stream")

    def add_host_async_fast(self, xyzi_ptr, rgba_ptr, n: int, frame_ref):
        """gem_add_points_host_async: pinned host buffers, H2D on a copy stream overlapped with the
        previous frame's kernels, no host synchronisation"""
        rc = self._lib.gem_add_points_host_async(self._h, xyzi_ptr, rgba_ptr, n, frame_ref)
        if rc:
            check(rc, self._h, "gem_add_points_host_async")

    def add_host_fast(self, xyzi_ptr, rgba_ptr, n: int, frame_ref):
        rc = self._lib.gem_add_points_host(self._h, xyzi_ptr, rgba_ptr, n, frame_ref)
        if rc:
            check(rc, self._h, "gem_add_points_host")

    # -- fused hot path: SensorProcessorBase::process + Fuse ------------------------------------
    def add(self, xyzi, rgba, frame: GemFrame, n: int | None = None):
        """ElevationMap::add of the upstream API.  xyzi: (n,4) float32 {x,y,z,intensity};
        rgba: (n,4) uint8 or None.  Device tensors run asynchronously on the map's stream;
        host arrays are copied inside the call."""
        if n is None:
            n = int(xyzi.shape[0])
        if _is_device(xyzi):
            rc = self._lib.gem_add_points(self._h, _ptr(xyzi), _ptr(rgba), n, C.byref(frame))
            check(rc, self._h, "gem_add_points")
        else:
            rc = self._lib.gem_add_points_host(self._h, _ptr(xyzi), _ptr(rgba), n, C.byref(frame))
            check(rc, self._h, "gem_add_points_host")

    def add_multi(self, xyzi, rgba, offsets, frames):
        """gem_add_points_multi: several device-resident clouds (own transforms) in one launch.
        offsets: n_segments+1 ints; frames: list of GemFrame."""
        nseg = len(frames)
        off = (C.c_int * (nseg + 1))(*[int(v) for v in offsets])
        fr = (GemFrame * nseg)(*frames)
        rc = self._lib.gem_add_points_multi(self._h, _ptr(xyzi), _ptr(rgba), nseg, off, fr)
        check(rc, self._h, "gem_add_points_multi")

    def add_pcl(self, points32: np.ndarray, frame: GemFrame):
        """PointXYZRGBICT records, (n, 32) uint8 or (n, 8) float32 host array."""
        n = int(points32.shape[0])
        check(self._lib.gem_add_cloud_pcl_host(self._h, _ptr(points32), n, C.byref(frame)), self._h,
              "gem_add_cloud_pcl_host")

    # -- unfused reference calls ------------------------------------------------------------
    def process_points(self, x, y, z, frame: GemFrame):
        """Process_points (gpu.cu:1085): returns map_index, var, x_ts, y_ts, z_ts."""
        x = np.ascontiguousarray(x, np.float32)
        y = np.ascontiguousarray(y, np.float32)
        z = np.ascontiguousarray(z, np.float32)
        n = x.shape[0]
        key = np.empty(n, np.int32)
        var = np.empty(n, np.float32)
        xt = np.empty(n, np.float32)
        yt = np.empty(n, np.float32)
        zt = np.empty(n, np.float32)
        rc = self._lib.gem_process_points(self._h, _ptr(key), _ptr(x), _ptr(y), _ptr(z), _ptr(var), _ptr(xt),
                                          _ptr(yt), _ptr(zt), n, C.byref(frame))
        check(rc, self._h, "gem_process_points")
        return key, var, xt, yt, zt

    def fuse_points(self, index, R, G, B, intensity, height, var):
        """Fuse (gpu.cu:1154)."""
        index = np.ascontiguousarray(index, np.int32)
        n = index.shape[0]
        conv_i = lambda a: None if a is None else np.ascontiguousarray(a, np.int32)
        conv_f = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)
        R, G, B = conv_i(R), conv_i(G), conv_i(B)
        intensity, height, var = conv_f(intensity), conv_f(height), conv_f(var)
        rc = self._lib.gem_fuse(self._h, n, _ptr(index), _ptr(R), _ptr(G), _ptr(B), _ptr(intensity), _ptr(height),
                                _ptr(var))
        check(rc, self._h, "gem_fuse")

    def var_update(self, dv: float):
        check(self._lib.gem_var_update(self._h, float(dv)), self._h, "gem_var_update")

    def compute_features(self):
        check(self._lib.gem_compute_features(self._h), self._h, "gem_compute_features")

    def map_feature(self):
        """Map_feature (gpu.cu:1256): dict of the 9 row-major storage-indexed host arrays."""
        n = self.ncells
        out = {
            "elevation": np.empty(n, np.float32), "variance": np.empty(n, np.float32),
            "color_r": np.empty(n, np.int32), "color_g": np.empty(n, np.int32), "color_b": np.empty(n, np.int32),
            "rough": np.empty(n, np.float32), "slope": np.empty(n, np.float32), "traver": np.empty(n, np.float32),
            "intensity": np.empty(n, np.float32),
        }
        rc = self._lib.gem_map_feature(self._h, _ptr(out["elevation"]), _ptr(out["variance"]), _ptr(out["color_r"]),
                                       _ptr(out["color_g"]), _ptr(out["color_b"]), _ptr(out["rough"]),
                                       _ptr(out["slope"]), _ptr(out["traver"]), _ptr(out["intensity"]))
        check(rc, self._h, "gem_map_feature")
        return out

    def fuse(self):
        """Upstream ElevationMap::fuse naming: produce the read-out layers (Map_feature + show)."""
        return self.export_layers()

    def raytracing(self):
        check(self._lib.gem_raytracing(self._h), self._h, "gem_raytracing")

    clean = raytracing  # upstream visibilityCleanup naming

    def opt_move(self, opt_p, height_update: float):
        p = (C.c_float * 2)(*[float(v) for v in opt_p])
        out = (C.c_float * 2)()
        check(self._lib.gem_opt_move(self._h, p, float(height_update), out), self._h, "gem_opt_move")
        return np.array(out[:], np.float32)

    def closeloop(self, update_position, height_update: float):
        p = (C.c_float * 2)(*[float(v) for v in update_position])
        check(self._lib.gem_closeloop(self._h, p, float(height_update)), self._h, "gem_closeloop")

    def set_colour_lookup(self, mode: str):
        """gem_set_colour_lookup: "image" (the default) reads every point's own pixel of the unmodified image; "node"
        reproduces the node's loop, where each in-image point paints its colour into its four neighbour pixels for the
        points after it (DESIGN.md f19).  Applies to colourise and to add_pointcloud2_host_async's image."""
        if mode not in _lib.COLOUR_LOOKUPS:
            raise ValueError(f"set_colour_lookup: mode {mode!r} is not one of {sorted(_lib.COLOUR_LOOKUPS)}")
        check(self._lib.gem_set_colour_lookup(self._h, _lib.COLOUR_LOOKUPS[mode]), self._h, "gem_set_colour_lookup")

    def colourise(self, xyzi, T_camera, T_lidar, bgr, rgba_out):
        """ElevationMapping.cpp:331-381 on the device: xyzi (n,4) float32 device tensor (intensity zeroed for
        points outside the image), bgr (H,W,3) uint8 device tensor, rgba_out (n,4) uint8 device tensor"""
        n = int(xyzi.shape[0])
        tc = (C.c_double * 12)(*[float(v) for v in np.asarray(T_camera, np.float64).reshape(-1)])
        tl = (C.c_double * 16)(*[float(v) for v in np.asarray(T_lidar, np.float64).reshape(-1)])
        h, w = int(bgr.shape[0]), int(bgr.shape[1])
        rc = self._lib.gem_colourise_points(self._h, _ptr(xyzi), n, tc, tl, _ptr(bgr), w, h, 3 * w, _ptr(rgba_out))
        check(rc, self._h, "gem_colourise_points")

    # -- read-out ---------------------------------------------------------------------------
    def export_layers(self, out: dict | None = None):
        """grid_map write-back: dict of 9 (L, L) float32 Fortran-ordered arrays, NaN = empty."""
        L = self.length
        if out is None:
            out = {name: np.empty((L, L), np.float32, order="F") for name in _lib.EXPORT_LAYERS}
        ptrs = (C.c_void_p * 9)(*[out[name].ctypes.data for name in _lib.EXPORT_LAYERS])
        check(self._lib.gem_export_layers(self._h, ptrs), self._h, "gem_export_layers")
        return out

    def export_layers_begin(self, out: dict, names=None):
        """asynchronous write-back into PINNED Fortran-ordered arrays (names: subset of the 9 layers, default all);
        finish with export_layers_end()"""
        names = _lib.EXPORT_LAYERS if names is None else names
        ptrs = (C.c_void_p * 9)(*[(out[n].ctypes.data if n in names else None) for n in _lib.EXPORT_LAYERS])
        check(self._lib.gem_export_layers_begin(self._h, ptrs), self._h, "gem_export_layers_begin")

    def export_layers_end(self):
        check(self._lib.gem_export_layers_end(self._h), self._h, "gem_export_layers_end")

    def get_layer(self, name: str) -> np.ndarray:
        lid = _lib.LAYERS[name]
        arr = np.empty(self.ncells, np.int32 if lid in _lib.INT_LAYERS else np.float32)
        check(self._lib.gem_get_layer(self._h, lid, _ptr(arr)), self._h, "gem_get_layer")
        return arr.reshape(self.shape)

    def set_layer(self, name: str, arr):
        lid = _lib.LAYERS[name]
        a = np.ascontiguousarray(arr, np.int32 if lid in _lib.INT_LAYERS else np.float32).reshape(-1)
        assert a.size == self.ncells
        check(self._lib.gem_set_layer(self._h, lid, _ptr(a)), self._h, "gem_set_layer")

    def state(self):
        centre = (C.c_float * 2)()
        start = (C.c_int * 2)()
        sz = C.c_float()
        check(self._lib.gem_get_state(self._h, centre, start, C.byref(sz)), self._h, "gem_get_state")
        return np.array(centre[:], np.float32), np.array(start[:], np.int32), float(sz.value)

    def stats(self) -> dict:
        st = GemStats()
        check(self._lib.gem_get_stats(self._h, C.byref(st)), self._h, "gem_get_stats")
        return {"points_in": st.points_in, "points_binned": st.points_binned, "cells_touched": st.cells_touched,
                "max_points_per_cell": st.max_points_per_cell}

    def selftest_division(self, n: int = 1 << 26, seed: int = 1):
        bad, fast = C.c_ulonglong(), C.c_ulonglong()
        check(self._lib.gem_selftest_division(self._h, seed, n, C.byref(bad), C.byref(fast)), self._h, "gem_selftest_division")
        return int(bad.value), int(fast.value)

    def profile_enable(self, on: bool = True):
        check(self._lib.gem_profile_enable(self._h, 1 if on else 0), self._h, "gem_profile_enable")

    def profile_read(self, reset: bool = True) -> dict:
        """launch count and summed per-kernel-class device milliseconds (synchronises)"""
        pr = _lib.GemProfile()
        check(self._lib.gem_profile_read(self._h, C.byref(pr), 1 if reset else 0), self._h, "gem_profile_read")
        return {"launches": int(pr.launches),
                "ms": {n: float(pr.ms[i]) for i, n in enumerate(_lib.PROF_CLASSES)},
                "count": {n: int(pr.count[i]) for i, n in enumerate(_lib.PROF_CLASSES)}}

    # -- multi-GPU tiling ---------------------------------------------------------------------
    def route_points(self, xyzi, rgba, frame: GemFrame, tiles_r: int, tiles_c: int, rec_out, counts_out,
                     bucket_stride: int = 0):
        n = int(xyzi.shape[0])
        rc = self._lib.gem_route_points(self._h, _ptr(xyzi), _ptr(rgba), n, C.byref(frame), int(tiles_r), int(tiles_c),
                                        _ptr(rec_out), _ptr(counts_out), int(bucket_stride))
        check(rc, self._h, "gem_route_points")

    def export_orthomosaic(self) -> np.ndarray:
        """bgr8 orthomosaic of ElevationMap::show (ElevationMap.cpp:87,123-125), (L, L, 3) uint8"""
        img = np.empty((self.length, self.length, 3), np.uint8)
        check(self._lib.gem_export_orthomosaic(self._h, _ptr(img)), self._h, "gem_export_orthomosaic")
        return img

    def export_visual_points(self, capacity: int = -1):
        """visual cloud of ElevationMap::show (ElevationMap.cpp:112-121): (xyz float32 (n,3), rgb uint8 (n,3))"""
        cap = self.ncells if capacity < 0 else int(capacity)
        xyz = np.empty((max(cap, 1), 3), np.float32)
        rgb = np.empty((max(cap, 1), 3), np.uint8)
        cnt = C.c_int()
        check(self._lib.gem_export_visual_points(self._h, _ptr(xyz), _ptr(rgb), cap, C.byref(cnt)), self._h,
              "gem_export_visual_points")
        n = min(cnt.value, cap)
        return xyz[:n], rgb[:n], cnt.value

    def snapshot_shown(self):
        """prevMap_ = map_.visualMap_ (ElevationMapping.cpp:422), kept on the device"""
        check(self._lib.gem_snapshot_shown(self._h), self._h, "gem_snapshot_shown")

    def harvest_scrolled_out(self, current_xy, shift_xy, capacity: int = -1):
        """ElevationMapping.cpp:716-765: (n, 8) float32 PointXYZRGBICT records of the snapshot's cells that left the
        window, plus the total count"""
        cap = self.ncells if capacity < 0 else int(capacity)
        out = np.empty((max(cap, 1), 8), np.float32)
        cur = (C.c_float * 2)(*[float(v) for v in current_xy])
        sh = (C.c_float * 2)(*[float(v) for v in shift_xy])
        cnt = C.c_int()
        check(self._lib.gem_harvest_scrolled_out(self._h, cur, sh, _ptr(out), cap, C.byref(cnt)), self._h,
              "gem_harvest_scrolled_out")
        return out[:min(cnt.value, cap)], cnt.value

    # -- local submaps on the device (ElevationMapping.cpp:609-767, :1124-1140, :1198-1226) ----------------------------
    def _records_out(self, n: int, out, what: str):
        """an (n, 8) float32 tensor on the map's device for n records: `out`'s first n rows, or a new tensor"""
        import torch
        if out is None:
            dev = torch.device("cuda", self._device_index())
            torch.cuda.current_stream(dev).synchronize()   # the library writes on its own stream
            return torch.empty((n, 8), dtype=torch.float32, device=dev)
        if not (_is_device(out) and out.dtype == torch.float32 and out.dim() == 2 and out.shape[1] == 8 and out.is_contiguous()):
            raise ValueError(f"{what}: out must be a contiguous (k, 8) float32 CUDA tensor")
        if out.shape[0] < n:
            raise ValueError(f"{what}: out holds {out.shape[0]} records, {n} are needed")
        return out[:n]

    def _device_index(self) -> int:
        import torch
        if not hasattr(self, "_dev"):
            self._dev = self._cfg_device if self._cfg_device >= 0 else torch.cuda.current_device()
        return self._dev

    def grid_cloud_count(self, source: str = "shown") -> int:
        """number of cells export_grid_cloud(source) takes"""
        cnt = C.c_int()
        check(self._lib.gem_export_grid_cloud(self._h, _lib.GRID_SOURCES[source], None, 0, C.byref(cnt)), self._h,
              "gem_export_grid_cloud")
        return cnt.value

    def export_grid_cloud(self, source: str = "shown", out=None):
        """gridMaptoPointCloud (ElevationMapping.cpp:1198-1226) of the shown map ("shown", visualMap_) or of the snapshot
        ("snapshot", prevMap_): (n, 8) float32 CUDA tensor of PointXYZRGBICT records in GridMapIterator order"""
        n = self.grid_cloud_count(source)
        rec = self._records_out(n, out, "export_grid_cloud")
        cnt = C.c_int()
        check(self._lib.gem_export_grid_cloud(self._h, _lib.GRID_SOURCES[source], _ptr(rec), n, C.byref(cnt)), self._h,
              "gem_export_grid_cloud")
        return rec

    def grid_cloud_split(self, source: str = "snapshot", mean_k: int = 20, stddev_mul: float = 1.0,
                         travers_threshold: float = 0.0, distances: bool = False):
        """composingGlobalMap's filter (ElevationMapping.cpp:1152-1170): PCL's statistical outlier removal over
        export_grid_cloud(source), then the survivors split by travers > travers_threshold.  Returns (road, obstacle,
        stats) with road / obstacle (n, 8) float32 CUDA tensors of PointXYZRGBICT records in grid-cloud order and stats a
        dict {points, valid, road, obstacle, mean, stddev, threshold}; with distances=True also the per-point mean
        distances (float32 CUDA tensor, grid-cloud order) as a fourth item"""
        import torch
        # one filter pass: every output is sized for the whole grid cloud (the cheap count of export_grid_cloud), which
        # road and obstacle together never exceed
        n = self.grid_cloud_count(source)
        road = self._records_out(n, None, "grid_cloud_split")
        obstacle = self._records_out(n, None, "grid_cloud_split")
        dist = torch.empty(n if distances else 0, dtype=torch.float32, device=road.device)
        st = _lib.GemGridSplit()
        check(self._lib.gem_grid_cloud_split(self._h, _lib.GRID_SOURCES[source], int(mean_k), float(stddev_mul),
                                             float(travers_threshold), _ptr(road), n, _ptr(obstacle), n, _ptr(dist), dist.shape[0],
                                             C.byref(st)), self._h, "gem_grid_cloud_split")
        stats = {k: getattr(st, k) for k, _ in _lib.GemGridSplit._fields_}
        road, obstacle = road[:st.road], obstacle[:st.obstacle]
        return (road, obstacle, stats, dist[:st.points]) if distances else (road, obstacle, stats)

    def color_octree(self, points, resolution: float):
        """pointCloudtoOctomap's octomap::ColorOcTree (ElevationMapping.cpp:1157-1174) of `points`, a contiguous (n, 8)
        float32 CUDA tensor of PointXYZRGBICT records, inserted in order at `resolution`.  Returns (stream, info): the
        ColorOcTree::writeData bytes as a uint8 CUDA tensor (octomap_msgs::Octomap::data with id "ColorOcTree",
        binary false) and a dict {bytes, nodes, leaves, inserted, skipped}"""
        import torch
        if not (_is_device(points) and points.dtype == torch.float32 and points.dim() == 2 and points.shape[1] == 8
                and points.is_contiguous()):
            raise ValueError("color_octree: points must be a contiguous (n, 8) float32 CUDA tensor")
        dev = torch.device("cuda", self._device_index())
        torch.cuda.current_stream(dev).synchronize()   # the library reads the points on its own stream
        info = _lib.GemOctree()
        n = points.shape[0]
        check(self._lib.gem_color_octree(self._h, _ptr(points) if n else None, n, float(resolution), C.byref(info)), self._h,
              "gem_color_octree")
        out = torch.empty(info.bytes, dtype=torch.uint8, device=dev)
        check(self._lib.gem_color_octree_read(self._h, _ptr(out), out.numel()), self._h, "gem_color_octree_read")
        return out, {k: getattr(info, k) for k, _ in _lib.GemOctree._fields_}

    def global_octrees(self, source: str = "snapshot", mean_k: int = 20, stddev_mul: float = 1.0,
                       travers_threshold: float = 0.0, road_resolution: float = 0.2, obstacle_resolution: float = 0.1):
        """the numeric work of composingGlobalMap (ElevationMapping.cpp:482-514, :1146-1174): grid_cloud_split, then the
        road and obstacle ColorOcTrees of its device outputs (the node's 0.2 m and 0.1 m trees, :146-147).  Returns
        (road stream, obstacle stream, split stats), the streams as color_octree returns them"""
        road, obstacle, stats = self.grid_cloud_split(source, mean_k, stddev_mul, travers_threshold)
        road_stream, _ = self.color_octree(road, road_resolution)
        obstacle_stream, _ = self.color_octree(obstacle, obstacle_resolution)
        return road_stream, obstacle_stream, stats

    # -- navigation costmaps (GEM's layers/ package, DESIGN.md f8) -------------------------------------------------------
    # A window is (origin_x, origin_y, resolution, size_x, size_y); a grid is a contiguous uint8 CUDA tensor of
    # size_x * size_y cells, cell (mx, my) at my * size_x + mx.  The library works on its own stream: each call first waits
    # for the current torch stream, and update_origin / combine leave their writes on the library's stream (torch_stream()).
    @staticmethod
    def _cost_window(window):
        ox, oy, res, sx, sy = window
        return _lib.GemCostmapWindow(float(ox), float(oy), float(res), int(sx), int(sy))

    def _cost_grid(self, grid, size_x: int, size_y: int, what: str):
        """the device address of a costmap grid after checking it against the size the call is given: the library only
        sees a pointer, so a tensor smaller than size_x * size_y cells would be read and written past its end"""
        import torch
        if not (_is_device(grid) and grid.dtype == torch.uint8 and grid.is_contiguous()):
            raise ValueError(f"{what}: the grid must be a contiguous uint8 CUDA tensor")
        if grid.device.index != self._device_index():
            raise ValueError(f"{what}: the grid is on {grid.device}, the map on cuda:{self._device_index()}")
        if grid.numel() != int(size_x) * int(size_y):
            raise ValueError(f"{what}: the grid holds {grid.numel()} cells, the window {int(size_x)} x {int(size_y)}")
        torch.cuda.current_stream(grid.device).synchronize()
        return _ptr(grid)

    @staticmethod
    def _cost_marks(mk) -> dict:
        return {k: getattr(mk, k) for k, _ in _lib.GemCostmapMarks._fields_}

    def costmap_mark_map(self, window, cost, travers_thresh: float = 0.7, source: str = "shown", mark_unknown: bool = True) -> dict:
        """ElevationMapLayer::updateBounds over show()'s grid_map ("shown": the live map after compute_features, or
        "snapshot") into the layer grid `cost`; returns the marks {marked, lethal, min_x, min_y, max_x, max_y}"""
        w = self._cost_window(window)
        p = self._cost_grid(cost, w.size_x, w.size_y, "costmap_mark_map")
        mk = _lib.GemCostmapMarks()
        check(self._lib.gem_costmap_mark_map(self._h, _lib.GRID_SOURCES[source], C.byref(w),
                                             float(travers_thresh), 1 if mark_unknown else 0, p, C.byref(mk)), self._h,
              "gem_costmap_mark_map")
        return self._cost_marks(mk)

    def costmap_mark_points(self, points, window, cost, travers_thresh: float = 0.7) -> dict:
        """PointMapLayer::updateBounds over `points`, an (n, 8) float32 CUDA tensor of PointXYZRGBICT records, into the
        layer grid `cost`; returns the marks as costmap_mark_map does"""
        import torch
        if not (_is_device(points) and points.dtype == torch.float32 and points.dim() == 2 and points.shape[1] == 8
                and points.is_contiguous()):
            raise ValueError("costmap_mark_points: points must be a contiguous (n, 8) float32 CUDA tensor")
        if points.device.index != self._device_index():
            raise ValueError(f"costmap_mark_points: the points are on {points.device}, the map on cuda:{self._device_index()}")
        w = self._cost_window(window)
        p = self._cost_grid(cost, w.size_x, w.size_y, "costmap_mark_points")
        mk = _lib.GemCostmapMarks()
        n = int(points.shape[0])
        check(self._lib.gem_costmap_mark_points(self._h, _ptr(points) if n else None, n, C.byref(w),
                                                float(travers_thresh), p, C.byref(mk)), self._h, "gem_costmap_mark_points")
        return self._cost_marks(mk)

    # -- the plugins fed from their subscribed messages (DESIGN.md f18) -----------------------------------------------------
    @staticmethod
    def grid_map_msg_parse(msg, layer: str = "traver") -> _lib.GemGridMapLayer:
        """fromMessage's geometry (G1-G3) and where `layer`'s floats are in the serialised grid_map_msgs/GridMap `msg`
        (host bytes: bytes, numpy or a CPU tensor; host code, no GPU).  A refused message raises GemError."""
        lib = _lib.load()
        p, nb = _host_bytes(msg)
        g = _lib.GemGridMapLayer()
        rc = lib.gem_grid_map_msg_parse(p, nb, layer.encode(), C.byref(g))
        if rc:
            err = lib.gem_last_error(None)
            raise _lib.GemError(f"gem_grid_map_msg_parse: {_lib.ERR_NAMES.get(rc, rc)}: {err.decode() if err else ''}")
        return g

    def costmap_mark_grid(self, g: _lib.GemGridMapLayer, data, window, cost, travers_thresh: float = 0.7,
                          mark_unknown: bool = True, offset: int = 0) -> dict:
        """ElevationMapLayer::updateBounds over a message layer: `data` is a CUDA tensor whose bytes from `offset` hold
        the g.floats floats the descriptor `g` describes (any alignment: e.g. the whole message copied to the device,
        offset = g.offset); returns the marks as costmap_mark_map does"""
        if not _is_device(data):
            raise ValueError("costmap_mark_grid: data must be a CUDA tensor")
        if data.device.index != self._device_index():
            raise ValueError(f"costmap_mark_grid: the data are on {data.device}, the map on cuda:{self._device_index()}")
        nb = int(data.numel() * data.element_size())
        if offset < 0 or offset + 4 * max(int(g.floats), 0) > nb:
            raise ValueError(f"costmap_mark_grid: {nb} bytes from offset {offset} do not hold {int(g.floats)} floats")
        w = self._cost_window(window)
        p = self._cost_grid(cost, w.size_x, w.size_y, "costmap_mark_grid")
        mk = _lib.GemCostmapMarks()
        check(self._lib.gem_costmap_mark_grid(self._h, C.byref(g), C.c_void_p(data.data_ptr() + int(offset)), C.byref(w),
                                              float(travers_thresh), 1 if mark_unknown else 0, p, C.byref(mk)), self._h,
              "gem_costmap_mark_grid")
        return self._cost_marks(mk)

    def costmap_update_origin(self, window, new_origin_x: float, new_origin_y: float, fill: int, cost):
        """Costmap2D::updateOrigin of the grid `cost` in place; returns the new window (the grid-aligned origin)"""
        w = self._cost_window(window)
        check(self._lib.gem_costmap_update_origin(self._h, C.byref(w), float(new_origin_x), float(new_origin_y), int(fill),
                                                  self._cost_grid(cost, w.size_x, w.size_y, "costmap_update_origin")), self._h,
              "gem_costmap_update_origin")
        return (w.origin_x, w.origin_y, w.resolution, w.size_x, w.size_y)

    def costmap_combine(self, mode: str, layer, master, size_x: int, size_y: int, rect):
        """updateWithMax (mode "max") or PointMapLayer's overwrite ("overwrite") of `layer` into `master` over
        rect = (min_i, min_j, max_i, max_j), clamped to the grid"""
        i0, j0, i1, j1 = (int(v) for v in rect)
        pl = self._cost_grid(layer, size_x, size_y, "costmap_combine")
        pm = self._cost_grid(master, size_x, size_y, "costmap_combine")
        check(self._lib.gem_costmap_combine(self._h, _lib.COSTMAP_MODES[mode], pl, pm, int(size_x), int(size_y), i0, j0, i1, j1),
              self._h, "gem_costmap_combine")

    def costmap_inflate(self, window, params, master, rect):
        """InflationLayer::updateCosts (DESIGN.md f14) of the master grid over rect = (min_i, min_j, max_i, max_j);
        params: a dict {inflation_radius, cost_scaling_factor, inscribed_radius, inflate_unknown}.  Asynchronous on
        the library's stream (torch_stream())."""
        w = self._cost_window(window)
        p = _lib.GemCostmapInflation(float(params["inflation_radius"]), float(params["cost_scaling_factor"]),
                                     float(params["inscribed_radius"]), 1 if params.get("inflate_unknown", False) else 0)
        i0, j0, i1, j1 = (int(v) for v in rect)
        check(self._lib.gem_costmap_inflate(self._h, C.byref(w), C.byref(p), self._cost_grid(master, w.size_x, w.size_y,
                                                                                           "costmap_inflate"), i0, j0, i1, j1),
              self._h, "gem_costmap_inflate")

    # -- what Costmap2DROS publishes, and ObstacleLayer's footprint clearing (DESIGN.md f17) ---------------------------------
    # A footprint is a sequence of (x, y) vertices in metres (the padded footprint); the pose is the robot's x, y, yaw.
    @staticmethod
    def _footprint(footprint):
        a = np.ascontiguousarray(np.asarray(footprint, np.float64).reshape(-1, 2))
        return a, a.shape[0], (a.ctypes.data_as(C.POINTER(C.c_double)) if a.shape[0] else None)

    def costmap_footprint(self, window, footprint, robot_x: float, robot_y: float, robot_yaw: float, layer) -> dict:
        """ObstacleLayer::updateFootprint and its updateCosts' setConvexPolygonCost(FREE_SPACE) on the layer grid: the
        footprint at the pose is written FREE (nothing when a vertex lies outside the window or there are fewer than 3);
        returns {marked: cells written, lethal: 0, min_x, min_y, max_x, max_y: the vertices' touch bounds}.
        Asynchronous on the library's stream (torch_stream())."""
        w = self._cost_window(window)
        fp, n, ptr = self._footprint(footprint)
        mk = _lib.GemCostmapMarks()
        check(self._lib.gem_costmap_footprint(self._h, C.byref(w), ptr, n, float(robot_x), float(robot_y), float(robot_yaw),
                                              self._cost_grid(layer, w.size_x, w.size_y, "costmap_footprint"), C.byref(mk)),
              self._h, "gem_costmap_footprint")
        return self._cost_marks(mk)

    def ros_footprint(self, header: RosHeader, footprint, robot_x: float, robot_y: float, robot_yaw: float, out=None):
        """<costmap>/footprint (geometry_msgs/PolygonStamped, W11) of the footprint at the pose"""
        h = header.c()
        fp, n, ptr = self._footprint(footprint)
        return self._ros_message("gem_ros_footprint", lambda p, c, nb: self._lib.gem_ros_footprint(
            self._h, C.byref(h), ptr, n, float(robot_x), float(robot_y), float(robot_yaw), p, c, nb), out)

    def ros_costmap(self, header: RosHeader, window, master, publisher, force_full: bool = False, out=None):
        """one Costmap2DPublisher::publishCostmap (or, with force_full, onNewSubscription's message) of the master grid:
        `publisher` is a gem_costmap_publisher (gem_b200.costmap.CostmapPublisher holds one).  Returns (kind, message) with
        kind "full" (nav_msgs/OccupancyGrid, W9), "update" (map_msgs/OccupancyGridUpdate, W10) or "none" (an empty
        message).  A size query or an `out` too small leaves the publisher as it was."""
        import torch
        w = self._cost_window(window)
        grid = self._cost_grid(master, w.size_x, w.size_y, "ros_costmap")
        h = header.c()
        kind = C.c_int()
        what = "gem_ros_costmap"

        def call(p, c, nb):
            return self._lib.gem_ros_costmap(self._h, C.byref(h), C.byref(w), grid, C.byref(publisher), 1 if force_full else 0,
                                             p, c, nb, C.byref(kind))
        if out is None:
            out = torch.empty(max(self._ros_size(what, call), 1), dtype=torch.uint8,
                              device=torch.device("cuda", self._device_index()))
        else:
            out = self._ros_buffer(out, what)
        n = self._ros_write(what, call, out)
        self.sync()
        return _lib.COSTMAP_PUB_KINDS[kind.value], out[:n]

    # -- the VoxelGrid pre-filter of GEM's demo launches (DESIGN.md f9) ---------------------------------------------------
    def voxel_grid(self, xyzi, leaf_size, field=None, limits=(-3.4028234663852886e38, 3.4028234663852886e38), negative=False,
                   out=None):
        """pcl_ros's VoxelGrid nodelet over `xyzi`, a contiguous (n, 4) float32 CUDA tensor {x, y, z, intensity}: leaf_size
        is a number or three; field None, "x", "y", "z" or "intensity" with the double limits (lo, hi) and the negative
        flag.  The centroids go to `out` (a contiguous (k, 4) float32 CUDA tensor, k = 0 being a size query) or to a new
        (n, 4) tensor.  Returns (out[:min(count, k)], {count, used, passthrough}); the two may not overlap"""
        import torch

        def cloud(t, what):
            if not (_is_device(t) and t.dtype == torch.float32 and t.dim() == 2 and t.shape[1] == 4 and t.is_contiguous()):
                raise ValueError(f"voxel_grid: {what} must be a contiguous (n, 4) float32 CUDA tensor")
            if t.device.index != self._device_index():
                raise ValueError(f"voxel_grid: {what} is on {t.device}, the map on cuda:{self._device_index()}")

        cloud(xyzi, "xyzi")
        n = int(xyzi.shape[0])
        if out is None:
            out = torch.empty((n, 4), dtype=torch.float32, device=xyzi.device)
        cloud(out, "out")
        leaf = [float(leaf_size)] * 3 if np.ndim(leaf_size) == 0 else [float(v) for v in leaf_size]
        if len(leaf) != 3:
            raise ValueError("voxel_grid: leaf_size is one number or three")
        if field not in _lib.VOXEL_FIELDS:
            raise ValueError(f"voxel_grid: field must be one of {list(_lib.VOXEL_FIELDS)}")
        lo, hi = (float(v) for v in limits)
        p = _lib.GemVoxelGridParams((C.c_float * 3)(*leaf), _lib.VOXEL_FIELDS[field], lo, hi, 1 if negative else 0)
        info = _lib.GemVoxelGridInfo()
        cap = int(out.shape[0])
        torch.cuda.current_stream(xyzi.device).synchronize()   # the library reads and writes on its own stream
        check(self._lib.gem_voxel_grid(self._h, _ptr(xyzi) if n else None, n, C.byref(p), _ptr(out) if cap else None, cap,
                                       C.byref(info)), self._h, "gem_voxel_grid")
        return out[:min(info.count, cap)], {k: getattr(info, k) for k, _ in _lib.GemVoxelGridInfo._fields_}

    @staticmethod
    def prefilter(steps) -> _lib.GemPrefilter:
        """gem_prefilter from VoxelGrid steps as voxel_oracle.FILTER_LAUNCH writes them, (leaf, field, (lo, hi), negative)
        in launch order; leaf is a number or three, field None, "x", "y", "z" or "intensity".  None or [] is no filter"""
        steps = list(steps or [])
        if len(steps) > _lib.PREFILTER_MAX_STEPS:
            raise ValueError(f"prefilter: at most {_lib.PREFILTER_MAX_STEPS} steps")
        pf = _lib.GemPrefilter()
        pf.nsteps = len(steps)
        for j, (leaf_size, field, limits, negative) in enumerate(steps):
            leaf = [float(leaf_size)] * 3 if np.ndim(leaf_size) == 0 else [float(v) for v in leaf_size]
            if len(leaf) != 3:
                raise ValueError("prefilter: leaf is one number or three")
            if field not in _lib.VOXEL_FIELDS:
                raise ValueError(f"prefilter: field must be one of {list(_lib.VOXEL_FIELDS)}")
            lo, hi = (float(v) for v in limits)
            pf.step[j] = _lib.GemVoxelGridParams((C.c_float * 3)(*leaf), _lib.VOXEL_FIELDS[field], lo, hi, 1 if negative else 0)
        return pf

    def add_points_filtered_stream(self, xyzi, prefilter, frame: GemFrame, bgr=None, T_camera=None, T_lidar=None):
        """gem_add_points_filtered_stream (DESIGN.md f20): the VoxelGrid steps `prefilter` (see prefilter()) over `xyzi`, a
        contiguous (n, 4) float32 CUDA tensor, the colour lookup from `bgr` (an (H, W, 3) uint8 CUDA tensor with the
        calibration T_camera / T_lidar, or None) and the pipelined add, with no host synchronisation.  xyzi must stay
        untouched until two further add calls have completed"""
        import torch
        if not (_is_device(xyzi) and xyzi.dtype == torch.float32 and xyzi.dim() == 2 and xyzi.shape[1] == 4
                and xyzi.is_contiguous()):
            raise ValueError("add_points_filtered_stream: xyzi must be a contiguous (n, 4) float32 CUDA tensor")
        pf = prefilter if isinstance(prefilter, _lib.GemPrefilter) else self.prefilter(prefilter)
        n = int(xyzi.shape[0])
        proj = None
        if bgr is not None:
            if not (_is_device(bgr) and bgr.dtype == torch.uint8 and bgr.dim() == 3 and bgr.shape[2] == 3 and bgr.is_contiguous()):
                raise ValueError("add_points_filtered_stream: bgr must be a contiguous (H, W, 3) uint8 CUDA tensor")
            proj = _lib.GemProjection()
            proj.T_camera[:] = [float(v) for v in np.asarray(T_camera, np.float64).reshape(-1)]
            proj.T_lidar[:] = [float(v) for v in np.asarray(T_lidar, np.float64).reshape(-1)]
            proj.height, proj.width = int(bgr.shape[0]), int(bgr.shape[1])
            proj.row_stride = 3 * proj.width
        torch.cuda.current_stream(xyzi.device).synchronize()   # the library reads on its own stream
        check(self._lib.gem_add_points_filtered_stream(self._h, _ptr(xyzi) if n else None, n, C.byref(pf),
                                                       _ptr(bgr) if bgr is not None else None,
                                                       C.byref(proj) if proj is not None else None, C.byref(frame)),
              self._h, "gem_add_points_filtered_stream")

    def prefilter_info(self, nsteps: int = _lib.PREFILTER_MAX_STEPS) -> list:
        """gem_prefilter_info: [{count, used, passthrough}] of the newest pre-filtered add's steps (synchronises)"""
        out = (_lib.GemVoxelGridInfo * max(int(nsteps), 1))()
        check(self._lib.gem_prefilter_info(self._h, out, int(nsteps)), self._h, "gem_prefilter_info")
        return [{k: getattr(out[j], k) for k, _ in _lib.GemVoxelGridInfo._fields_} for j in range(int(nsteps))]

    # -- raw sensor messages: PointCloud2 and cv_bridge's 8-bit images (DESIGN.md f12) -------------------------------------
    @staticmethod
    def pointcloud2_mapping(layout: PointCloud2Layout, data_bytes: int | None = None) -> dict:
        """createMapping<PointXYZRGBICT> of PCL 1.8 for `layout` (host code, no GPU): {spans: [(serialized_offset,
        struct_offset, size), ...], fast_path, matched: [struct field names], points, bytes}.  data_bytes defaults to
        the bytes the layout needs.  A refused layout raises GemError."""
        lib = _lib.load()
        mp = _lib.GemPc2Mapping()
        nb = (1 << 64) - 1 if data_bytes is None else int(data_bytes)
        rc = lib.gem_pointcloud2_mapping(C.byref(layout.c), nb, C.byref(mp))
        if rc:
            msg = lib.gem_last_error(None)
            raise _lib.GemError(f"gem_pointcloud2_mapping: {_lib.ERR_NAMES.get(rc, rc)}: {msg.decode() if msg else ''}")
        return {"spans": [(mp.spans[k].serialized_offset, mp.spans[k].struct_offset, mp.spans[k].size) for k in range(mp.nspans)],
                "fast_path": bool(mp.fast_path), "matched": [n for k, n in enumerate(_lib.PC2_FIELDS) if mp.matched >> k & 1],
                "points": int(mp.points), "bytes": int(mp.bytes)}

    def decode_pointcloud2(self, layout: PointCloud2Layout, data, out=None, data_bytes: int | None = None):
        """gem_decode_pointcloud2: the message bytes `data` (a CUDA tensor, any dtype and offset) into `out`, a contiguous
        (width * height, 4) float32 CUDA tensor (new if None), {x, y, z, intensity} as fromPCLPointCloud2 gives them.
        Asynchronous on the map's stream (the current torch stream is synchronised first): sync() before reading out."""
        import torch
        if not _is_device(data):
            raise ValueError("decode_pointcloud2: data must be a CUDA tensor")
        n = layout.points
        if out is None:
            out = torch.empty((n, 4), dtype=torch.float32, device=data.device)
        nb = int(data.numel() * data.element_size()) if data_bytes is None else int(data_bytes)
        torch.cuda.current_stream(data.device).synchronize()
        check(self._lib.gem_decode_pointcloud2(self._h, C.byref(layout.c), _ptr(data), nb, _ptr(out)), self._h,
              "gem_decode_pointcloud2")
        return out

    def decode_pointcloud2_records(self, layout: PointCloud2Layout, data, out=None, data_bytes: int | None = None):
        """gem_decode_pointcloud2_records (DESIGN.md f18): the message bytes `data` (a CUDA tensor, any dtype and offset)
        into `out`, a contiguous (width * height, 8) float32 CUDA tensor (new if None) of whole PointXYZRGBICT records as
        fromPCLPointCloud2 fills them.  Asynchronous on the map's stream, as decode_pointcloud2."""
        import torch
        if not _is_device(data):
            raise ValueError("decode_pointcloud2_records: data must be a CUDA tensor")
        n = layout.points
        if out is None:
            out = torch.empty((n, 8), dtype=torch.float32, device=data.device)
        elif not (_is_device(out) and out.element_size() == 4 and out.is_contiguous() and out.numel() >= 8 * n):
            raise ValueError("decode_pointcloud2_records: out must be a contiguous CUDA tensor of 32-bit words holding "
                             "8 * width * height of them")
        nb = int(data.numel() * data.element_size()) if data_bytes is None else int(data_bytes)
        torch.cuda.current_stream(data.device).synchronize()
        check(self._lib.gem_decode_pointcloud2_records(self._h, C.byref(layout.c), _ptr(data), nb, _ptr(out)), self._h,
              "gem_decode_pointcloud2_records")
        return out

    def image_to_bgr8(self, encoding: str, src, width: int, height: int, step: int | None = None, out=None,
                      dst_step: int | None = None):
        """gem_image_to_bgr8: cv_bridge::toCvCopy(image, "bgr8") for bgr8 / rgb8 / bgra8 / rgba8 / mono8 on CUDA uint8
        tensors.  out defaults to a new (height, width, 3) tensor.  Asynchronous on the map's stream."""
        import torch
        ch = _lib.IMAGE_ENCODINGS.get(encoding, 3)
        step = ch * int(width) if step is None else int(step)
        if out is None:
            out = torch.empty((int(height), int(width), 3), dtype=torch.uint8, device=src.device)
        dst_step = 3 * int(width) if dst_step is None else int(dst_step)
        torch.cuda.current_stream(src.device).synchronize()
        check(self._lib.gem_image_to_bgr8(self._h, encoding.encode(), _ptr(src), int(width), int(height), step, _ptr(out),
                                          dst_step), self._h, "gem_image_to_bgr8")
        return out

    def add_pointcloud2_host_async(self, layout: PointCloud2Layout, data, frame: GemFrame, image: CameraImage | None = None,
                                   data_bytes: int | None = None, prefilter=None):
        """gem_add_pointcloud2_host_async: one sensor_msgs/PointCloud2 (host bytes: numpy, bytes or a CPU tensor, pinned
        or pageable) and optionally its camera image, decoded, colourised and added pipelined.  Pinned buffers must stay
        untouched until the call after next or sync(); pageable ones may be reused at once.  prefilter (VoxelGrid steps,
        see prefilter(), or a GemPrefilter): gem_add_pointcloud2_filtered_host_async, the steps between the decode and
        the colour (DESIGN.md f20)"""
        ptr, nb = _host_bytes(data) if layout.points else (None, 0)
        nb = nb if data_bytes is None else int(data_bytes)
        img = C.byref(image.c) if image is not None else None
        if prefilter is None:
            check(self._lib.gem_add_pointcloud2_host_async(self._h, C.byref(layout.c), ptr, nb, img, C.byref(frame)),
                  self._h, "gem_add_pointcloud2_host_async")
            return
        pf = prefilter if isinstance(prefilter, _lib.GemPrefilter) else self.prefilter(prefilter)
        check(self._lib.gem_add_pointcloud2_filtered_host_async(self._h, C.byref(layout.c), ptr, nb, img, C.byref(pf),
                                                                C.byref(frame)),
              self._h, "gem_add_pointcloud2_filtered_host_async")

    # -- the MLS densification of the dense_mapping signal (DESIGN.md f10) ------------------------------------------------
    GEM_MLS = {"search_radius": 0.5, "sqr_gauss_param": 0.25, "polynomial_fit": True, "order": 5,
               "upsampling": "random_uniform_density", "point_density": 1000, "seed": 0}   # pointcloudinterpolation's settings

    def mls_upsample(self, points, params=None, out=None, info: bool = False):
        """pointcloudinterpolation's pcl::MovingLeastSquares (ElevationMapping.cpp:1072-1118) over `points`, a contiguous
        (n, 8) float32 CUDA tensor of PointXYZRGBICT records: the points MLS produces, which the node appends to the
        submap.  params: a dict overriding GEM_MLS's entries (upsampling "none" or "random_uniform_density").  The records
        go to `out` (a contiguous (k, 8) float32 CUDA tensor that must hold them all) or to a new tensor.  Returns the
        (m, 8) tensor, or (tensor, {count, processed, fitted, skipped, max_neighbours}) with info=True"""
        import torch
        if not (_is_device(points) and points.dtype == torch.float32 and points.dim() == 2 and points.shape[1] == 8
                and points.is_contiguous()):
            raise ValueError("mls_upsample: points must be a contiguous (n, 8) float32 CUDA tensor")
        if points.device.index != self._device_index():
            raise ValueError(f"mls_upsample: the points are on {points.device}, the map on cuda:{self._device_index()}")
        q = dict(self.GEM_MLS)
        for k, v in (params or {}).items():
            if k not in q:
                raise ValueError(f"mls_upsample: unknown parameter {k!r}")
            q[k] = v
        if q["upsampling"] not in _lib.MLS_UPSAMPLING:
            raise ValueError(f"mls_upsample: upsampling must be one of {list(_lib.MLS_UPSAMPLING)}")
        p = _lib.GemMlsParams(float(q["search_radius"]), float(q["sqr_gauss_param"]), 1 if q["polynomial_fit"] else 0,
                              int(q["order"]), _lib.MLS_UPSAMPLING[q["upsampling"]], int(q["point_density"]),
                              int(q["seed"]) & 0xFFFFFFFFFFFFFFFF)
        n = int(points.shape[0])
        pin = _ptr(points) if n else None
        torch.cuda.current_stream(points.device).synchronize()   # the library reads and writes on its own stream
        st = _lib.GemMlsInfo()
        check(self._lib.gem_mls_upsample(self._h, pin, n, C.byref(p), None, 0, C.byref(st)), self._h, "gem_mls_upsample")
        rec = self._records_out(st.count, out, "mls_upsample")
        if st.count:
            check(self._lib.gem_mls_upsample(self._h, pin, n, C.byref(p), _ptr(rec), st.count, C.byref(st)), self._h,
                  "gem_mls_upsample")
        return (rec, {k: getattr(st, k) for k, _ in _lib.GemMlsInfo._fields_}) if info else rec

    def harvest_to_local_map(self, current_xy, shift_xy, records: bool = False):
        """the harvest of harvest_scrolled_out, upserted into the device-resident localMap_ (ElevationMapping.cpp:740-747).
        Returns the number of harvested records, or (records (n, 8) float32 host array, n) with records=True"""
        cur = (C.c_float * 2)(*[float(v) for v in current_xy])
        sh = (C.c_float * 2)(*[float(v) for v in shift_xy])
        cnt = C.c_int()
        out = np.empty((self.ncells, 8), np.float32) if records else None
        check(self._lib.gem_harvest_to_local_map(self._h, cur, sh, _ptr(out), self.ncells if records else 0, C.byref(cnt)),
              self._h, "gem_harvest_to_local_map")
        return (out[:cnt.value], cnt.value) if records else cnt.value

    def local_map_size(self) -> int:
        """records local_map_take would return now (distinct cells harvested since the last take / clear)"""
        cnt = C.c_int()
        check(self._lib.gem_local_map_take(self._h, None, 0, C.byref(cnt)), self._h, "gem_local_map_take")
        return cnt.value

    def local_map_take(self, out=None):
        """localHashtoPointCloud (ElevationMapping.cpp:1124-1140): the local map as an (n, 8) float32 CUDA tensor (last
        occurrence of each cell, in the order of those occurrences); the local map is empty afterwards"""
        n = self.local_map_size()
        rec = self._records_out(n, out, "local_map_take")
        cnt = C.c_int()
        check(self._lib.gem_local_map_take(self._h, _ptr(rec), n, C.byref(cnt)), self._h, "gem_local_map_take")
        return rec

    def local_map_clear(self):
        check(self._lib.gem_local_map_clear(self._h), self._h, "gem_local_map_clear")

    def local_map_reserve(self, records: int):
        """room for `records` harvested records now, so that later harvests do not allocate"""
        check(self._lib.gem_local_map_reserve(self._h, int(records)), self._h, "gem_local_map_reserve")

    def cut_submap(self, out=None, dense: bool = False, seed: int = 0):
        """the submap of a keyframe cut (ElevationMapping.cpp:653-661): local_map_take() followed by
        export_grid_cloud("shown"), in one (n, 8) float32 CUDA tensor; the local map is empty afterwards.  With dense=True
        (the dense_mapping signal, :656-657) the MLS points of the taken local map (mls_upsample with GEM's settings and
        `seed`) come between the two: [local map, its MLS points, grid cloud], i.e. *out_pc + *grid_pc after
        *input += dense; `out` is then not accepted (the size is known only after the fit)"""
        if dense:
            import torch
            if out is not None:
                raise ValueError("cut_submap: out is not accepted with dense=True")
            local = self.local_map_take()
            extra = self.mls_upsample(local, {"seed": seed})
            grid = self.export_grid_cloud("shown")
            return torch.cat([local, extra, grid])
        nl, ng = self.local_map_size(), self.grid_cloud_count("shown")
        rec = self._records_out(nl + ng, out, "cut_submap")
        self.local_map_take(out=rec[:nl])
        self.export_grid_cloud("shown", out=rec[nl:])
        return rec

    # -- point clouds as PCD files: savingMap / savingSubMap's pcl::io::savePCDFile (DESIGN.md f13) -----------------------
    PCD_CHUNK = 1 << 20   # records per save_pcd round trip: 32 MiB in, at most 105 MiB of text out

    @staticmethod
    def _pcd_flags(binary: bool, rgb_uint32: bool) -> int:
        return (_lib.PCD_BINARY if binary else 0) | (_lib.PCD_RGB_UINT32 if rgb_uint32 else 0)

    @staticmethod
    def pcd_header(n: int, binary: bool = False, rgb_uint32: bool = False) -> bytes:
        """the PCD header PCL's generateHeader writes for a PointXYZRGBICT cloud of n records (host code, no GPU); an empty
        cloud raises GemError, as PCL throws"""
        lib = _lib.load()
        buf = C.create_string_buffer(_lib.PCD_HEADER_MAX)
        k = C.c_int()
        rc = lib.gem_pcd_header(int(n), ElevationMap._pcd_flags(binary, rgb_uint32), buf, _lib.PCD_HEADER_MAX, C.byref(k))
        if rc:
            msg = lib.gem_last_error(None)
            raise _lib.GemError(f"gem_pcd_header: {_lib.ERR_NAMES.get(rc, rc)}: {msg.decode() if msg else ''}")
        return buf.raw[:k.value]

    def _pcd_points(self, points, what: str):
        import torch
        if not (_is_device(points) and points.dtype == torch.float32 and points.dim() == 2 and points.shape[1] == 8
                and points.is_contiguous()):
            raise ValueError(f"{what}: points must be a contiguous (n, 8) float32 CUDA tensor")
        if points.device.index != self._device_index():
            raise ValueError(f"{what}: the points are on {points.device}, the map on cuda:{self._device_index()}")

    def format_pcd(self, points, binary: bool = False, rgb_uint32: bool = False, out=None):
        """gem_pcd_format: the data section savePCDFile writes for `points`, a contiguous (n, 8) float32 CUDA tensor of
        PointXYZRGBICT records -- ASCII lines of %.8g values, or 28-byte binary records.  Returns a uint8 CUDA tensor of
        the bytes (a view of `out`, a uint8 CUDA tensor, when given: it must hold them all)"""
        import torch
        self._pcd_points(points, "format_pcd")
        flags, n = self._pcd_flags(binary, rgb_uint32), int(points.shape[0])
        torch.cuda.current_stream(points.device).synchronize()   # the library reads the points on its own stream
        nb = C.c_longlong()
        if out is None:
            check(self._lib.gem_pcd_format(self._h, _ptr(points), n, flags, None, 0, C.byref(nb)), self._h, "gem_pcd_format")
            out = torch.empty(nb.value, dtype=torch.uint8, device=points.device)
        elif not (_is_device(out) and out.dtype == torch.uint8 and out.is_contiguous()):
            raise ValueError("format_pcd: out must be a contiguous uint8 CUDA tensor")
        check(self._lib.gem_pcd_format(self._h, _ptr(points), n, flags, _ptr(out), out.numel(), C.byref(nb)), self._h,
              "gem_pcd_format")
        if nb.value > out.numel():
            raise ValueError(f"format_pcd: out holds {out.numel()} bytes, {nb.value} are needed")
        return out.view(-1)[:nb.value]

    def save_pcd(self, path, points, binary: bool = False, rgb_uint32: bool = False, chunk: int | None = None) -> int:
        """pcl::io::savePCDFile(path, cloud) (ASCII) or savePCDFileBinary for `points`, (n, 8) float32 PointXYZRGBICT
        records: a CUDA tensor, or a host array / CPU tensor (e.g. visualCloud_ gathered from harvest_*(records=True)).
        The header goes first, then the records in chunks of `chunk` (default PCD_CHUNK) through fixed device and pinned
        buffers, so a host cloud larger than free device memory still saves.  The file equals the one-shot
        pcd_header(n) + format_pcd(points).  An empty cloud raises GemError and writes no file.  Returns the file's size"""
        import torch
        dev = torch.device("cuda", self._device_index())
        if _is_device(points):
            self._pcd_points(points, "save_pcd")
            src = points
        else:
            src = torch.as_tensor(np.ascontiguousarray(points, np.float32) if isinstance(points, np.ndarray) else points)
            if not (src.dtype == torch.float32 and src.dim() == 2 and src.shape[1] == 8):
                raise ValueError("save_pcd: points must be (n, 8) float32 records")
            src = src.contiguous()
        n, flags = int(src.shape[0]), self._pcd_flags(binary, rgb_uint32)
        head = self.pcd_header(n, binary, rgb_uint32)           # refuses an empty cloud before the file is opened
        step = max(1, min(int(chunk or self.PCD_CHUNK), n))
        per = 28 if binary else _lib.PCD_LINE_MAX
        dout = torch.empty(step * per, dtype=torch.uint8, device=dev)
        hout = torch.empty(step * per, dtype=torch.uint8, pin_memory=True)
        din = hin = None
        if not _is_device(src):
            din = torch.empty((step, 8), dtype=torch.float32, device=dev)
            hin = torch.empty((step, 8), dtype=torch.float32, pin_memory=True)
        torch.cuda.current_stream(dev).synchronize()
        size = len(head)
        nb = C.c_longlong()
        try:
            with open(path, "wb") as f:
                f.write(head)
                for i in range(0, n, step):
                    k = min(step, n - i)
                    if din is None:
                        part = src[i:i + k]
                    else:
                        hin[:k].copy_(src[i:i + k])
                        part = din[:k]
                        part.copy_(hin[:k], non_blocking=True)
                        torch.cuda.current_stream(dev).synchronize()
                    check(self._lib.gem_pcd_format(self._h, _ptr(part), k, flags, _ptr(dout), dout.numel(), C.byref(nb)),
                          self._h, "gem_pcd_format")
                    hout[:nb.value].copy_(dout[:nb.value])
                    f.write(memoryview(hout.numpy())[:nb.value])
                    size += nb.value
        except BaseException:
            try:
                os.remove(path)
            except OSError:
                pass
            raise
        return size

    # -- the node's map topics as serialised ROS1 messages (DESIGN.md f15) ---------------------------------------------------
    # Each returns the message's bytes as a uint8 tensor: a new CUDA tensor, or a view of `out`, a contiguous uint8 CUDA
    # tensor or pinned CPU tensor that must hold them all (the device writes pinned memory directly).  The call is
    # complete when it returns.
    def _ros_buffer(self, out, what: str):
        import torch
        if not (isinstance(out, torch.Tensor) and out.dtype == torch.uint8 and out.is_contiguous()
                and (out.is_cuda or out.is_pinned())):
            raise ValueError(f"{what}: out must be a contiguous uint8 CUDA tensor or pinned CPU tensor")
        return out.view(-1)

    def _ros_write(self, what: str, call, out, offset: int = 0) -> int:
        """call(ptr, capacity, bytes_out) into out[offset:]; returns the bytes written (raises when they do not fit)"""
        nb = C.c_longlong()
        cap = out.numel() - offset
        check(call(C.c_void_p(out.data_ptr() + offset) if cap > 0 else None, cap, C.byref(nb)), self._h, what)
        if nb.value > cap:
            raise ValueError(f"{what}: out holds {cap} bytes, {nb.value} are needed")
        return nb.value

    def _ros_size(self, what: str, call) -> int:
        nb = C.c_longlong()
        check(call(None, 0, C.byref(nb)), self._h, what)
        return nb.value

    def _ros_message(self, what: str, call, out):
        import torch
        dev = torch.device("cuda", self._device_index())
        out = (torch.empty(self._ros_size(what, call), dtype=torch.uint8, device=dev) if out is None
               else self._ros_buffer(out, what))
        torch.cuda.current_stream(dev).synchronize()   # the library writes on its own stream
        n = self._ros_write(what, call, out)
        self.sync()
        return out[:n]

    def ros_grid_map(self, header: RosHeader, out=None):
        """visual_map (grid_map_msgs/GridMap, W2): export_layers' 9 layers bit for bit, with the map's geometry"""
        h = header.c()
        return self._ros_message("gem_ros_grid_map", lambda p, c, nb: self._lib.gem_ros_grid_map(self._h, C.byref(h), p, c, nb), out)

    def ros_orthomosaic(self, header: RosHeader | None = None, out=None):
        """orthomosaic (sensor_msgs/Image "bgr8", W3) of export_orthomosaic's image; show() publishes it with an empty header
        (the default)"""
        h = (header or RosHeader()).c()
        return self._ros_message("gem_ros_orthomosaic",
                                 lambda p, c, nb: self._lib.gem_ros_orthomosaic(self._h, C.byref(h), p, c, nb), out)

    def ros_visual_points(self, header: RosHeader, out=None):
        """visualpoints (PointCloud2 of pcl::PointXYZRGB, W6) of export_visual_points' points, in its order"""
        h = header.c()
        return self._ros_message("gem_ros_visual_points",
                                 lambda p, c, nb: self._lib.gem_ros_visual_points(self._h, C.byref(h), p, c, nb), out)

    def _ros_parts(self, parts):
        """gem_ros_part array of (n, 8) float32 record arrays (CUDA tensors, CPU tensors or numpy arrays), kept alive"""
        keep, arr = [], (_lib.GemRosPart * max(len(parts), 1))()
        for i, p in enumerate(parts):
            if isinstance(p, np.ndarray):
                p = np.ascontiguousarray(p)
                ok = p.dtype in (np.float32, np.uint32) and p.ndim == 2 and p.shape[1] == 8
            else:
                ok = p.element_size() == 4 and p.dim() == 2 and p.shape[1] == 8 and p.is_contiguous()
            if not ok:
                raise ValueError("ros_cloud: every part must be a contiguous (n, 8) array of 32-bit words")
            keep.append(p)
            arr[i].points32 = _ptr(p).value if p.shape[0] else None
            arr[i].n = int(p.shape[0])
        return arr, keep

    def ros_cloud(self, header: RosHeader, parts, is_dense: bool = True, out=None):
        """history_point / global_point (PointCloud2 of PointXYZRGBICT, W5): the parts' records back to back (device,
        pinned or pageable host memory); is_dense as pcl::PointCloud's flag (push_back and operator+ leave it true)"""
        h = header.c()
        arr, keep = self._ros_parts(list(parts))
        n = len(keep)
        return self._ros_message("gem_ros_cloud", lambda p, c, nb: self._lib.gem_ros_cloud(
            self._h, C.byref(h), arr, n, 1 if is_dense else 0, p, c, nb), out)

    def ros_octomap(self, header: RosHeader, out=None):
        """road_octomap / obs_octomap (octomap_msgs/Octomap, W7) of the last color_octree's stream and resolution"""
        h = header.c()
        return self._ros_message("gem_ros_octomap", lambda p, c, nb: self._lib.gem_ros_octomap(self._h, C.byref(h), p, c, nb), out)

    def ros_submap(self, records, keyframe_pc: bytes, pose, header: RosHeader, image_header: RosHeader | None = None,
                   is_dense: bool = True, out=None):
        """submap (dislam_msgs/SubMap, W8): the cloud of `records` (W5), the received keyframe cloud's serialised bytes as
        they are, this map's orthomosaic (W3) and the pose (position xyz, orientation xyzw) as 7 float64, each part
        written at its offset in one buffer"""
        import torch
        import struct
        h, ih = header.c(), (image_header or RosHeader()).c()
        arr, keep = self._ros_parts([records])
        cloud = lambda p, c, nb: self._lib.gem_ros_cloud(self._h, C.byref(h), arr, 1, 1 if is_dense else 0, p, c, nb)
        image = lambda p, c, nb: self._lib.gem_ros_orthomosaic(self._h, C.byref(ih), p, c, nb)
        kf = np.frombuffer(bytes(keyframe_pc), np.uint8)
        tail = np.frombuffer(struct.pack("<7d", *[float(v) for v in pose]), np.uint8)
        n_cloud, n_image = self._ros_size("gem_ros_cloud", cloud), self._ros_size("gem_ros_orthomosaic", image)
        size = n_cloud + kf.size + n_image + tail.size
        dev = torch.device("cuda", self._device_index())
        out = torch.empty(size, dtype=torch.uint8, device=dev) if out is None else self._ros_buffer(out, "ros_submap")
        if out.numel() < size:
            raise ValueError(f"ros_submap: out holds {out.numel()} bytes, {size} are needed")
        torch.cuda.current_stream(dev).synchronize()
        self._ros_write("gem_ros_cloud", cloud, out, 0)
        self._ros_write("gem_ros_orthomosaic", image, out, n_cloud + kf.size)
        self.sync()
        out[n_cloud:n_cloud + kf.size].copy_(torch.from_numpy(kf.copy()))
        out[size - tail.size:size].copy_(torch.from_numpy(tail.copy()))
        if out.is_cuda:
            torch.cuda.current_stream(dev).synchronize()
        return out[:size]

    def get_layer_device(self, name: str, out):
        """dense (rows, cols) copy of a layer into a device tensor (float32, int32 for colours)"""
        lid = 10 if name == "traver_out" else _lib.LAYERS[name]
        check(self._lib.gem_get_layer_device(self._h, lid, _ptr(out)), self._h, "gem_get_layer_device")

    def compute_features_tiled(self, padded_elevation):
        check(self._lib.gem_compute_features_tiled(self._h, _ptr(padded_elevation)), self._h, "gem_compute_features_tiled")

    def raytracing_tiled(self, global_lowest):
        check(self._lib.gem_raytracing_tiled(self._h, _ptr(global_lowest)), self._h, "gem_raytracing_tiled")

    def transform_cloud(self, points32, T):
        """gem_transform_cloud: (n, 8) float32 device tensor of PointXYZRGBICT records, rigidly transformed in place"""
        t = (C.c_float * 16)(*[float(v) for v in np.asarray(T, np.float32).reshape(-1)])
        check(self._lib.gem_transform_cloud(self._h, _ptr(points32), int(points32.shape[0]), t), self._h, "gem_transform_cloud")

    def refuse_submaps(self, new_points32, old_points32, resolution: float, compat: bool = True):
        """gem_refuse_submaps on two (n, 8) float32 device tensors; returns (n_new, n_old, fused): the tensors' first n rows hold the result"""
        nn, no, fused = C.c_int(int(new_points32.shape[0])), C.c_int(int(old_points32.shape[0])), C.c_int(0)
        check(self._lib.gem_refuse_submaps(self._h, _ptr(new_points32), C.byref(nn), _ptr(old_points32), C.byref(no), float(resolution),
                                           1 if compat else 0, C.byref(fused)), self._h, "gem_refuse_submaps")
        return nn.value, no.value, fused.value

    # -- the global map: globalMap_, trajectory_, localMapLoc_ and updateGlobalMap on the device (DESIGN.md f16) -----------
    def global_map_reset(self):
        """the init branch (ElevationMapping.cpp:688-707): no submap, trajectory_ = [identity], centres = [(0, 0)]"""
        check(self._lib.gem_global_map_reset(self._h), self._h, "gem_global_map_reset")

    def global_map_reserve(self, records: int, submaps: int = 0):
        """room for `records` records and `submaps` submaps (and the update's scratch), so that pushes and updates do not
        allocate"""
        check(self._lib.gem_global_map_reserve(self._h, int(records), int(submaps)), self._h, "gem_global_map_reserve")

    def global_map_push(self, records, pose):
        """the keyframe branch (:633-662): trajectory_.push_back(pose) (4 x 4, row 3 ignored), its centre = the pose's x, y,
        then globalMap_.push_back(records), a contiguous (n, 8) float32 CUDA tensor (e.g. cut_submap()), copied"""
        import torch
        if not (_is_device(records) and records.dtype == torch.float32 and records.dim() == 2 and records.shape[1] == 8
                and records.is_contiguous()):
            raise ValueError("global_map_push: records must be a contiguous (n, 8) float32 CUDA tensor")
        torch.cuda.current_stream(records.device).synchronize()   # the library reads the records on its own stream
        p = (C.c_float * 16)(*[float(v) for v in np.asarray(pose, np.float32).reshape(16)])
        check(self._lib.gem_global_map_push(self._h, _ptr(records), int(records.shape[0]), p), self._h, "gem_global_map_push")

    def global_map_update(self, opt_poses, resolution: float, radius: float = 25.0, compat: bool = True) -> int:
        """updateGlobalMap (:773-905) in one call: re-pose submaps 1 .. K'-1 with opt_poses (k x 4 x 4, K' = min(k,
        submaps)), re-fuse every neighbour pair within `radius` of the pushed centres, pack the stack.  Returns the fused
        cell count"""
        poses = np.ascontiguousarray(np.asarray(opt_poses, np.float32).reshape(-1, 16))
        fused = C.c_int(0)
        check(self._lib.gem_global_map_update(self._h, poses.ctypes.data_as(_lib._FP), int(poses.shape[0]), float(resolution),
                                              float(radius), 1 if compat else 0, C.byref(fused)), self._h, "gem_global_map_update")
        return fused.value

    def global_map_info(self):
        """(submaps, keyframes, records)"""
        s, k, r = C.c_int(), C.c_int(), C.c_longlong()
        check(self._lib.gem_global_map_info(self._h, C.byref(s), C.byref(k), C.byref(r)), self._h, "gem_global_map_info")
        return s.value, k.value, r.value

    def _device_view(self, ptr: int, n: int):
        """an (n, 8) float32 CUDA tensor over library memory, without a copy"""
        import torch

        class _View:
            __cuda_array_interface__ = {"shape": (n, 8), "typestr": "<f4", "data": (ptr, False), "version": 2, "strides": None,
                                        "stream": None}
        dev = torch.device("cuda", self._device_index())
        return torch.empty((0, 8), dtype=torch.float32, device=dev) if n == 0 else torch.as_tensor(_View(), device=dev)

    def global_map_submaps(self):
        """views of every submap as (n, 8) float32 CUDA tensors, valid until the next push, update, reserve or reset"""
        out = []
        p, n = C.c_void_p(), C.c_int()
        for i in range(self.global_map_info()[0]):
            check(self._lib.gem_global_map_submap(self._h, i, C.byref(p), C.byref(n)), self._h, "gem_global_map_submap")
            out.append(self._device_view(p.value or 0, n.value))
        return out

    def global_map_records(self):
        """the whole stack, submaps back to back in push order (composingGlobalMap's cloudpt, updateGlobalMap's
        visualCloud_), as a view like global_map_submaps'"""
        p, n = C.c_void_p(), C.c_longlong()
        check(self._lib.gem_global_map_records(self._h, C.byref(p), C.byref(n)), self._h, "gem_global_map_records")
        return self._device_view(p.value or 0, n.value)

    def global_map_poses(self):
        """(trajectory_ as (keyframes, 4, 4) float32, centres as (keyframes, 2) float32)"""
        k = self.global_map_info()[1]
        poses, centres = np.zeros((k, 16), np.float32), np.zeros((k, 2), np.float32)
        for i in range(k):
            check(self._lib.gem_global_map_pose(self._h, i, poses[i].ctypes.data_as(_lib._FP), centres[i].ctypes.data_as(_lib._FP)),
                  self._h, "gem_global_map_pose")
        return poses.reshape(k, 4, 4), centres

    def save_submaps(self, directory, binary: bool = False, rgb_uint32: bool = False):
        """savingSubMap (:461-476): every submap to `directory`/<i>.pcd through save_pcd.  An empty submap writes no file
        (PCL throws there).  Returns the paths written"""
        paths = []
        for i, sub in enumerate(self.global_map_submaps()):
            if sub.shape[0] == 0:
                continue
            path = os.path.join(str(directory), f"{i}.pcd")
            self.save_pcd(path, sub, binary, rgb_uint32)
            paths.append(path)
        return paths

    def tiled_attach(self, tiles_r, tiles_c, my_rank, bucket_capacity, recv_records, recv_intensity, recv_counts, flags):
        """gem_tiled_attach: lists of device addresses (ints), one per rank, of the four peer-accessible buffers"""
        p = _lib.GemTiledPeers()
        p.tiles_r, p.tiles_c, p.my_rank, p.bucket_capacity = int(tiles_r), int(tiles_c), int(my_rank), int(bucket_capacity)
        for o in range(len(recv_records)):
            p.recv_records[o], p.recv_intensity[o] = int(recv_records[o]), int(recv_intensity[o])
            p.recv_counts[o], p.flags[o] = int(recv_counts[o]), int(flags[o])
        check(self._lib.gem_tiled_attach(self._h, C.byref(p)), self._h, "gem_tiled_attach")

    def tiled_step(self, xyzi, rgba, frame: GemFrame, n: int | None = None):
        n = int(xyzi.shape[0]) if n is None else int(n)
        rc = self._lib.gem_tiled_step(self._h, _ptr(xyzi), _ptr(rgba), n, C.byref(frame))
        if rc:
            check(rc, self._h, "gem_tiled_step")

    def tiled_step_fast(self, xyzi_ptr, rgba_ptr, n: int, frame_ref):
        """gem_tiled_step with raw device addresses (c_void_p) and a byref'd gem_frame: minimal host time per step"""
        rc = self._lib.gem_tiled_step(self._h, xyzi_ptr, rgba_ptr, n, frame_ref)
        if rc:
            check(rc, self._h, "gem_tiled_step")

    def fuse_records(self, rec, n: int):
        check(self._lib.gem_fuse_records(self._h, _ptr(rec), int(n)), self._h, "gem_fuse_records")
