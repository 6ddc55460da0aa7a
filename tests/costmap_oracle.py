"""Oracle of the gem_costmap_* calls: ctypes binding of tests/orc_costmap.c, compiled with the oracle's flags into a
temporary directory (the checkout may be read-only).  TEST INFRASTRUCTURE ONLY.

A window is (origin_x, origin_y, resolution, size_x, size_y); a grid a (size_y, size_x) uint8 array; marks a dict
{marked, lethal, min_x, min_y, max_x, max_y}."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import native

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orc_costmap.c")
_lib = None


class Window(C.Structure):
    _fields_ = [("origin_x", C.c_double), ("origin_y", C.c_double), ("resolution", C.c_double), ("size_x", C.c_int),
                ("size_y", C.c_int)]


class Marks(C.Structure):
    _fields_ = [("marked", C.c_longlong), ("lethal", C.c_longlong), ("min_x", C.c_double), ("min_y", C.c_double),
                ("max_x", C.c_double), ("max_y", C.c_double)]


def load():
    global _lib
    if _lib is None:
        lib = native.shared_library("orc_costmap", [SRC], native.ORACLE_C, ["-lm"])
        P = C.c_void_p
        lib.orc_mark_map.argtypes = [C.c_int, C.c_double, P, P, P, C.POINTER(Window), C.c_double, C.c_int, P, C.POINTER(Marks)]
        lib.orc_mark_map.restype = None
        lib.orc_mark_points.argtypes = [P, C.c_int, C.POINTER(Window), C.c_double, P, C.POINTER(Marks)]
        lib.orc_mark_points.restype = None
        lib.orc_update_origin.argtypes = [C.POINTER(Window), C.c_double, C.c_double, C.c_ubyte, P]
        lib.orc_update_origin.restype = C.c_int
        lib.orc_combine.argtypes = [C.c_int, P, P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        lib.orc_combine.restype = None
        _lib = lib
    return _lib


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _grid(grid, window):
    g = np.ascontiguousarray(grid, np.uint8).copy()
    assert g.size == window[3] * window[4]
    return g


def _marks(m):
    return {k: getattr(m, k) for k, _ in Marks._fields_}


def mark_map(traver, L, grid_res, centre, start, window, grid, travers_thresh, mark_unknown=True):
    """orc_mark_map; traver: (L, L) array indexed [ix, iy] or its column-major flattening.  Returns (grid, marks)"""
    t = np.ascontiguousarray(np.asarray(traver, np.float32).reshape(L, L).T)   # [iy, ix]: column-major of [ix, iy]
    c = np.ascontiguousarray(centre, np.float32)
    s = np.ascontiguousarray(start, np.int32)
    g = _grid(grid, window)
    m = Marks()
    load().orc_mark_map(int(L), float(grid_res), _p(c), _p(s), _p(t), C.byref(Window(*window)), float(travers_thresh),
                        1 if mark_unknown else 0, _p(g), C.byref(m))
    return g, _marks(m)


def mark_points(records, window, grid, travers_thresh):
    rec = np.ascontiguousarray(records, np.float32).reshape(-1, 8)
    g = _grid(grid, window)
    m = Marks()
    load().orc_mark_points(_p(rec), int(rec.shape[0]), C.byref(Window(*window)), float(travers_thresh), _p(g), C.byref(m))
    return g, _marks(m)


def update_origin(window, new_origin_x, new_origin_y, fill, grid):
    """returns (new window, grid), or None where the library reports an error"""
    g = _grid(grid, window)
    w = Window(*window)
    if load().orc_update_origin(C.byref(w), float(new_origin_x), float(new_origin_y), int(fill), _p(g)) != 0:
        return None
    return (w.origin_x, w.origin_y, w.resolution, w.size_x, w.size_y), g


def combine(mode, layer, master, size_x, size_y, rect):
    lay = np.ascontiguousarray(layer, np.uint8)
    g = np.ascontiguousarray(master, np.uint8).copy()
    i0, j0, i1, j1 = rect
    load().orc_combine(int(mode), _p(lay), _p(g), int(size_x), int(size_y), int(i0), int(j0), int(i1), int(j1))
    return g
