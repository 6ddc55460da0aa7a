"""Oracle of gem_color_octree: ctypes binding of tests/orc_color_octree.c, compiled with the oracle's flags into a
temporary directory (the checkout may be read-only).  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import native

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orc_color_octree.c")
_lib = None


def load():
    global _lib
    if _lib is None:
        lib = native.shared_library("orc_color_octree", [SRC], native.ORACLE_C, ["-lm"])
        P = C.c_void_p
        lib.orc_octree_build.argtypes = [C.c_int, P, C.c_double, P]
        lib.orc_octree_build.restype = P
        lib.orc_octree_write.argtypes = [P, P]
        lib.orc_octree_write.restype = None
        lib.orc_octree_free.argtypes = [P]
        lib.orc_octree_free.restype = None
        _lib = lib
    return _lib


def color_octree(records, resolution):
    """orc_color_octree over (n, 8) float32 PointXYZRGBICT records: (stream as a uint8 array, info dict with bytes,
    nodes, leaves, inserted, skipped)"""
    lib = load()
    rec = np.ascontiguousarray(records, np.float32).reshape(-1, 8)
    info = np.zeros(4, np.int64)
    t = lib.orc_octree_build(int(rec.shape[0]), C.c_void_p(rec.ctypes.data), float(resolution), C.c_void_p(info.ctypes.data))
    try:
        out = np.zeros(max(int(info[0]) * 8, 1), np.uint8)
        lib.orc_octree_write(t, C.c_void_p(out.ctypes.data))
    finally:
        lib.orc_octree_free(t)
    nodes, leaves, inserted, skipped = (int(v) for v in info)
    return out[:nodes * 8].copy(), {"bytes": nodes * 8, "nodes": nodes, "leaves": leaves, "inserted": inserted,
                                    "skipped": skipped}
