"""Oracle of the stereo and perfect sensor models.  TEST INFRASTRUCTURE ONLY.

ctypes binding of tests/orc_sensor_models.c, compiled with the oracle's flags into a temporary directory (the checkout
may be read-only) and linked against oracle/libgem_oracle.so, whose index function and fold it shares.  `add` is what
the fused add calls compute for a stereo or perfect frame: the per-point step of orc_sm_process_points, then orc_fuse
through OracleMap.fuse_points.  Laser and structured-light frames go to OracleMap.add unchanged.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import native
import oracle_lib

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orc_sensor_models.c")
NEW_MODELS = (2, 3)  # GEM_SENSOR_STEREO, GEM_SENSOR_PERFECT
_lib = None


class OrcSmSensor(C.Structure):
    _fields_ = [("type", C.c_int), ("p", C.c_double * 5), ("lateral", C.c_double), ("dtd", C.c_double),
                ("width", C.c_int)]


def load():
    global _lib
    if _lib is None:
        oracle_lib.load()  # builds oracle/libgem_oracle.so
        odir = oracle_lib.ODIR
        lib = native.shared_library("orc_sensor_models", [SRC], native.ORACLE_C + ["-I", odir],
                                    ["-L", odir, "-lgem_oracle", "-Wl,-rpath," + odir, "-lm"])
        P = C.c_void_p
        lib.orc_sm_variances.restype = C.c_float
        lib.orc_sm_variances.argtypes = [C.POINTER(OrcSmSensor), C.c_float, C.c_float, C.c_float, C.c_int,
                                         C.POINTER(C.c_float)]
        lib.orc_sm_process_points.argtypes = [C.POINTER(oracle_lib.OrcMap), C.c_int, P, P, P, P, C.c_double, C.c_double,
                                              C.POINTER(OrcSmSensor), P, P, P, P, P, C.c_int, P, P, P, P, P]
        _lib = lib
    return _lib


def sensor_of(frame) -> OrcSmSensor:
    s = frame.sensor
    return OrcSmSensor(s.type, (C.c_double * 5)(*s.stereo_p), s.lateral_factor, s.depth_to_disparity_factor,
                       s.cloud_width)


def variances(sensor: OrcSmSensor, x, y, z, idx):
    """(varianceNormal, varianceLateral) of one point"""
    vn = C.c_float()
    vl = load().orc_sm_variances(C.byref(sensor), float(x), float(y), float(z), int(idx), C.byref(vn))
    return np.float32(vn.value), np.float32(vl)


def _p(a):
    return C.c_void_p(a.ctypes.data)


def process_points(omap, x, y, z, frame, idx0=0):
    """orc_sm_process_points on an OracleMap (updates its lowest layer): key, var, x_ts, y_ts, z_ts"""
    lib = load()
    x, y, z = (np.ascontiguousarray(a, np.float32) for a in (x, y, z))
    n = x.shape[0]
    key = np.empty(n, np.int32)
    out = [np.empty(n, np.float32) for _ in range(4)]
    f32 = lambda v: np.array(v[:], np.float32)
    arrs = [f32(frame.T), f32(frame.sensor_jacobian), f32(frame.rotation_variance), f32(frame.C_SB_transpose),
            f32(frame.P_mul_C_BM_transpose), f32(frame.B_r_BS_skew)]
    sensor = sensor_of(frame)
    lib.orc_sm_process_points(omap.m, n, _p(x), _p(y), _p(z), _p(arrs[0]), frame.rel_lower, frame.rel_upper,
                              C.byref(sensor), *[_p(a) for a in arrs[1:]], int(idx0), _p(key), *[_p(a) for a in out])
    return (key, *out)


def add(omap, xyzi, rgba, frame, idx0=0):
    """what a fused add call computes for one frame of any of the four models"""
    if frame.sensor.type not in NEW_MODELS:
        omap.add(xyzi, rgba, frame)
        return
    xyzi = np.asarray(xyzi, np.float32)
    key, var, _, _, zt = process_points(omap, xyzi[:, 0], xyzi[:, 1], xyzi[:, 2], frame, idx0)
    if rgba is None:
        R = G = B = np.zeros(xyzi.shape[0], np.int32)
    else:
        R, G, B = (np.asarray(rgba)[:, k].astype(np.int32) for k in range(3))
    omap.fuse_points(key, R, G, B, xyzi[:, 3], zt, var)
