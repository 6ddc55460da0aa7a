"""Oracles of the local-submap calls (gem_export_grid_cloud, gem_harvest_to_local_map, gem_local_map_take).
TEST INFRASTRUCTURE ONLY.

grid_cloud: ctypes binding of tests/orc_grid_cloud.c, compiled with the oracle's flags into a temporary directory (the
checkout may be read-only).  LocalMapDict: ElevationMapping::updateLocalMap's unordered_map run literally as a Python
dict (find, erase, insert, :740-747); a dict iterates in insertion order, which is the order gem_local_map_take defines.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import native

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orc_grid_cloud.c")
_lib = None


def load():
    global _lib
    if _lib is None:
        lib = native.shared_library("orc_grid_cloud", [SRC], native.ORACLE_C, ["-lm"])
        P = C.c_void_p
        lib.orc_grid_cloud.argtypes = [C.c_int, C.c_double, P, P, P, P, P, P, P, P, P, P, C.POINTER(C.c_int)]
        _lib = lib
    return _lib


def _p(a):
    return C.c_void_p(a.ctypes.data)


def grid_cloud(feature, L, centre, start, grid_res):
    """orc_grid_cloud over Map_feature outputs (the dict OracleMap.map_feature returns) with that frame's geometry:
    (n, 8) float32 PointXYZRGBICT records"""
    lib = load()
    f = {k: np.ascontiguousarray(v) for k, v in feature.items()}
    centre = np.ascontiguousarray(centre, np.float32)
    start = np.ascontiguousarray(start, np.int32)
    out = np.empty((L * L, 8), np.float32)
    cnt = C.c_int()
    lib.orc_grid_cloud(int(L), float(grid_res), _p(centre), _p(start), _p(f["elevation"]), _p(f["variance"]), _p(f["traver"]),
                       _p(f["color_r"]), _p(f["color_g"]), _p(f["color_b"]), _p(f["intensity"]), _p(out), C.byref(cnt))
    return out[:cnt.value].copy()


class LocalMapDict:
    """localMap_ of the node: key = the float (x, y) of a record (GridPointEqual), value = the record"""

    def __init__(self):
        self.d = {}

    def insert_all(self, records):
        for r in np.asarray(records, np.float32):
            key = (r[0].tobytes(), r[1].tobytes())
            if key in self.d:          # :740-747: find, erase, insert
                del self.d[key]
            self.d[key] = r.copy()

    def __len__(self):
        return len(self.d)

    def records(self):
        """localHashtoPointCloud (:1124-1140) in the dict's iteration order"""
        return np.array(list(self.d.values()), np.float32).reshape(-1, 8)

    def clear(self):
        self.d = {}
