"""Oracle of gem_voxel_grid: ctypes binding of tests/orc_voxel_grid.c, compiled with the oracle's flags into a temporary
directory (the checkout may be read-only).  TEST INFRASTRUCTURE ONLY.

A call takes an (n, 4) float32 array {x, y, z, intensity} and returns (out, info): out the min(count, capacity) written
float4 rows, info a dict {count, used, passthrough}; None where the library reports an error."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import native

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orc_voxel_grid.c")
FIELDS = {None: -1, "x": 0, "y": 1, "z": 2, "intensity": 3}
FLT_MAX = 3.4028234663852886e38
_lib = None


class Params(C.Structure):
    _fields_ = [("leaf_size", C.c_float * 3), ("field", C.c_int), ("limit_min", C.c_double), ("limit_max", C.c_double),
                ("limit_negative", C.c_int)]


class Info(C.Structure):
    _fields_ = [("count", C.c_int), ("used", C.c_int), ("passthrough", C.c_int)]


def load():
    global _lib
    if _lib is None:
        lib = native.shared_library("orc_voxel_grid", [SRC], native.ORACLE_C, ["-lm"])
        lib.orc_voxel_grid.argtypes = [C.c_void_p, C.c_int, C.POINTER(Params), C.c_void_p, C.c_int, C.POINTER(Info)]
        lib.orc_voxel_grid.restype = C.c_int
        _lib = lib
    return _lib


def params(leaf, field=None, limits=(-FLT_MAX, FLT_MAX), negative=False):
    leaf = [float(leaf)] * 3 if np.ndim(leaf) == 0 else [float(v) for v in leaf]
    f = FIELDS[field] if field in FIELDS else int(field)
    return Params((C.c_float * 3)(*leaf), f, float(limits[0]), float(limits[1]), 1 if negative else 0)


def voxel_grid(xyzi, leaf, field=None, limits=(-FLT_MAX, FLT_MAX), negative=False, capacity=None):
    pts = np.ascontiguousarray(xyzi, np.float32).reshape(-1, 4)
    n = pts.shape[0]
    cap = n if capacity is None else int(capacity)
    out = np.zeros((max(cap, 1), 4), np.float32)
    info = Info()
    p = params(leaf, field, limits, negative)
    if load().orc_voxel_grid(C.c_void_p(pts.ctypes.data), n, C.byref(p), C.c_void_p(out.ctypes.data), cap, C.byref(info)) != 0:
        return None
    return out[:min(info.count, cap)].copy(), {"count": info.count, "used": info.used, "passthrough": info.passthrough}


def chain(xyzi, steps):
    """calls in sequence, each on the previous output: steps = [(leaf, field, limits, negative), ...]"""
    out, info = np.ascontiguousarray(xyzi, np.float32), None
    infos = []
    for leaf, field, limits, negative in steps:
        out, info = voxel_grid(out, leaf, field, limits, negative)
        infos.append(info)
    return out, infos


# GEM's launches: filter.launch (one nodelet) and filter_kitti.launch (three in a chain)
FILTER_LAUNCH = [(0.1, "x", (-10.0, 10.0), False)]
FILTER_KITTI_LAUNCH = [(0.2, "x", (-40.0, 40.0), False), (0.2, "z", (-25.0, 25.0), False), (0.2, "y", (-40.0, 40.0), False)]
