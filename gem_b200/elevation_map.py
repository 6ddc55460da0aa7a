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

    def get_layer_device(self, name: str, out):
        """dense (rows, cols) copy of a layer into a device tensor (float32, int32 for colours)"""
        lid = 10 if name == "traver_out" else _lib.LAYERS[name]
        check(self._lib.gem_get_layer_device(self._h, lid, _ptr(out)), self._h, "gem_get_layer_device")

    def compute_features_tiled(self, padded_elevation):
        check(self._lib.gem_compute_features_tiled(self._h, _ptr(padded_elevation)), self._h, "gem_compute_features_tiled")

    def raytracing_tiled(self, global_lowest):
        check(self._lib.gem_raytracing_tiled(self._h, _ptr(global_lowest)), self._h, "gem_raytracing_tiled")

    def route_points_peer(self, xyzi, rgba, frame: GemFrame, tiles_r: int, tiles_c: int, peer_recv, peer_counts,
                          my_rank: int, bucket_stride: int):
        """peer_recv / peer_counts: lists of device addresses (ints), one per rank"""
        n = int(xyzi.shape[0])
        no = len(peer_recv)
        pr = (C.c_ulonglong * no)(*[int(v) for v in peer_recv])
        pc = (C.c_ulonglong * no)(*[int(v) for v in peer_counts])
        rc = self._lib.gem_route_points_peer(self._h, _ptr(xyzi), _ptr(rgba), n, C.byref(frame), int(tiles_r), int(tiles_c),
                                             pr, pc, int(my_rank), int(bucket_stride))
        check(rc, self._h, "gem_route_points_peer")

    def fuse_records_counted(self, rec, src_counts, n_sources: int, bucket_stride: int):
        rc = self._lib.gem_fuse_records_counted(self._h, _ptr(rec), _ptr(src_counts), int(n_sources), int(bucket_stride))
        check(rc, self._h, "gem_fuse_records_counted")

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
