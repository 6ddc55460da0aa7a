"""Oracle of what Costmap2DROS publishes and of ObstacleLayer's footprint clearing (DESIGN.md f17).  TEST INFRASTRUCTURE
ONLY.

- T, and the struct encoder of W9 (OccupancyGrid), W10 (OccupancyGridUpdate) and W11 (PolygonStamped), reusing
  tests/rosmsg_oracle.py's header; an independent decoder (a cursor over the bytes, as a subscriber reads them); a
  subscriber's replica that a full message replaces and an update patches.
- Publisher: a Python restatement of Costmap2DPublisher's updateBounds / publishCostmap / onNewSubscription (P1-P4).
- Footprint: an independent Python restatement of F1-F4 (the outline walked in map coordinates, the adjacent-swap sort
  as the stable sort it is) and the true convex fill for comparison; orc(): tests/orc_footprint.c, the literal loops.
- host(): the library's host code (gem_rosfmt.h, gem_footprint.h) through tests/costmap_pub_host.cpp, built with g++.
All compiled into temporary directories (the checkout may be read-only).
"""
from __future__ import annotations

import ctypes as C
import math
import os
import struct

import numpy as np

import native
import rosmsg_oracle as ro

HERE = os.path.dirname(os.path.abspath(__file__))
INT_MAX = 2**31 - 1
GEM_FOOTPRINT = ((-0.64, -0.40), (-0.64, 0.40), (0.64, 0.40), (0.64, -0.40))


# ---- T and the encoder ------------------------------------------------------------------------------------------------
def translate(c: int) -> int:
    """cost_translation_table_[c]"""
    return {0: 0, 253: 99, 254: 100, 255: -1}.get(c, 1 + (97 * (c - 1)) // 251 if 1 <= c <= 252 else None)


TABLE = np.array([translate(c) for c in range(256)], np.int8)


def occupancy_grid(hdr: bytes, window, grid) -> bytes:
    """W9 of a (size_y, size_x) uint8 grid"""
    ox, oy, res, sx, sy = window
    wx, wy = ox + (0 + 0.5) * res, oy + (0 + 0.5) * res
    data = TABLE[np.asarray(grid, np.uint8).reshape(-1)].tobytes()
    assert len(data) == sx * sy
    return (hdr + struct.pack("<IIfII", 0, 0, res, sx, sy) + struct.pack("<7d", wx - res / 2, wy - res / 2, 0.0, 0.0, 0.0, 0.0, 1.0)
            + struct.pack("<I", len(data)) + data)


def grid_update(hdr: bytes, x: int, y: int, w: int, h: int, grid) -> bytes:
    """W10 of the rectangle [x, x + w) x [y, y + h) of a (size_y, size_x) grid"""
    data = TABLE[np.asarray(grid, np.uint8)[y:y + h, x:x + w]].tobytes()
    return hdr + struct.pack("<iiIII", x, y, w, h, len(data)) + data


def polygon_stamped(hdr: bytes, pts) -> bytes:
    """W11 of (x, y) points, stored as float32 with z = 0"""
    return hdr + struct.pack("<I", len(pts)) + b"".join(struct.pack("<fff", x, y, 0.0) for x, y in pts)


def size_grid(f, sx, sy):
    return 96 + f + sx * sy


def size_update(f, w, h):
    return 36 + f + w * h


def size_polygon(f, n):
    return 20 + f + 12 * n


# ---- the decoder ------------------------------------------------------------------------------------------------------
def decode_occupancy_grid(b: bytes) -> dict:
    r = ro.Reader(b)
    d = {"header": r.header(), "map_load_time": (r.num("I"), r.num("I")), "resolution": r.num("f"), "width": r.num("I"),
         "height": r.num("I"), "position": tuple(r.num("d") for _ in range(3)), "orientation": tuple(r.num("d") for _ in range(4))}
    d["data"] = np.frombuffer(r.take(r.num("I")), np.int8)
    r.end()
    return d


def decode_grid_update(b: bytes) -> dict:
    r = ro.Reader(b)
    d = {"header": r.header(), "x": r.num("i"), "y": r.num("i"), "width": r.num("I"), "height": r.num("I")}
    d["data"] = np.frombuffer(r.take(r.num("I")), np.int8)
    r.end()
    return d


def decode_polygon_stamped(b: bytes) -> dict:
    r = ro.Reader(b)
    d = {"header": r.header()}
    d["points"] = [(r.num("f"), r.num("f"), r.num("f")) for _ in range(r.num("I"))]
    r.end()
    return d


class Replica:
    """a subscriber's copy of the costmap: a full message replaces it, an update patches it"""

    def __init__(self):
        self.grid = None

    def apply(self, kind: str, msg: bytes):
        if kind == "full":
            d = decode_occupancy_grid(msg)
            self.grid = d["data"].reshape(d["height"], d["width"]).copy()
        elif kind == "update":
            d = decode_grid_update(msg)
            assert d["data"].size == d["width"] * d["height"]
            self.grid[d["y"]:d["y"] + d["height"], d["x"]:d["x"] + d["width"]] = d["data"].reshape(d["height"], d["width"])
        else:
            assert len(msg) == 0


# ---- the publisher ----------------------------------------------------------------------------------------------------
class Publisher:
    """Costmap2DPublisher: the saved window (None until a full message) and the accumulated bounds"""

    def __init__(self, always_send_full: bool = False):
        self.always = bool(always_send_full)
        self.saved = None
        self.x0 = self.y0 = INT_MAX
        self.xn = self.yn = 0

    def bounds(self, x0, xn, y0, yn):
        self.x0, self.xn, self.y0, self.yn = min(x0, self.x0), max(xn, self.xn), min(y0, self.y0), max(yn, self.yn)

    def state(self):
        return (self.saved, self.x0, self.xn, self.y0, self.yn)

    def publish(self, window, force_full: bool = False):
        """(kind, (x0, y0, width, height)); the state moves on as after a written message"""
        ox, oy, res, sx, sy = window
        now = (np.float32(res), sx, sy, ox, oy)
        if force_full or self.always or self.saved is None or self.saved != now:
            kind, rect = "full", (0, 0, sx, sy)
            self.saved = now
        elif self.x0 < self.xn:
            kind, rect = "update", (self.x0, self.y0, self.xn - self.x0, self.yn - self.y0)
        else:
            kind, rect = "none", (0, 0, 0, 0)
        if not force_full:
            self.x0, self.y0, self.xn, self.yn = sx, sy, 0, 0
        return kind, rect


# ---- the footprint, restated ------------------------------------------------------------------------------------------
def transform(footprint, rx, ry, yaw):
    c, s = math.cos(yaw), math.sin(yaw)
    return [(rx + (fx * c - fy * s), ry + (fx * s + fy * c)) for fx, fy in footprint]


def to_map(window, x, y):
    ox, oy, res, sx, sy = window
    if not (x >= ox and y >= oy):
        return None
    qx, qy = (x - ox) / res, (y - oy) / res
    if not (qx < 2.0**31 and qy < 2.0**31):
        return None
    mx, my = int(qx), int(qy)
    return (mx, my) if mx < sx and my < sy else None


def _line(a, b):
    """bresenham2D in map coordinates: the dominant axis steps every cell, the other when the error reaches the span;
    the end cell last"""
    (x, y), (x1, y1) = a, b
    dx, dy = x1 - x, y1 - y
    major_x = abs(dx) >= abs(dy)
    span, minor = (abs(dx), abs(dy)) if major_x else (abs(dy), abs(dx))
    sgx, sgy = (1 if dx > 0 else -1), (1 if dy > 0 else -1)
    err, out = span // 2, []
    for _ in range(span):
        out.append((x, y))
        if major_x:
            x += sgx
        else:
            y += sgy
        err += minor
        if err >= span:
            if major_x:
                y += sgy
            else:
                x += sgx
            err -= span
    out.append((x, y))
    return out


def footprint_cells(window, footprint, rx, ry, yaw):
    """(vertices, cells): the cells setConvexPolygonCost writes in list order, None when a vertex lies outside"""
    verts = transform(footprint, rx, ry, yaw)
    poly = [to_map(window, x, y) for x, y in verts]
    if any(p is None for p in poly):
        return verts, None
    if len(poly) < 3:
        return verts, []
    outline = []
    for k in range(len(poly)):
        outline += _line(poly[k], poly[(k + 1) % len(poly)])
    return verts, column_walk(outline)


def column_walk(cells):
    """F4 on a list of (x, y) cells: the adjacent-swap sort that steps back is a stable sort by x; then the walk, which
    pairs cells i, i + 1 whatever their columns and appends to the list it walks"""
    cells = sorted(cells, key=lambda c: c[0])
    if not cells:
        return cells
    i, first, last = 0, cells[0][0], cells[-1][0]
    for x in range(first, last + 1):
        if i >= len(cells) - 1:
            break
        lo, hi = (cells[i], cells[i + 1]) if cells[i][1] < cells[i + 1][1] else (cells[i + 1], cells[i])
        i += 2
        while i < len(cells) and cells[i][0] == x:
            if cells[i][1] < lo[1]:
                lo = cells[i]
            elif cells[i][1] > hi[1]:
                hi = cells[i]
            i += 1
        cells.extend((x, y) for y in range(lo[1], hi[1]))
    return cells


def true_fill(outline_cells):
    """every cell between the lowest and the highest outline cell of each column"""
    cols = {}
    for x, y in outline_cells:
        lo, hi = cols.get(x, (y, y))
        cols[x] = (min(lo, y), max(hi, y))
    return {(x, y) for x, (lo, hi) in cols.items() for y in range(lo, hi + 1)}


def outline(window, footprint, rx, ry, yaw):
    poly = [to_map(window, x, y) for x, y in transform(footprint, rx, ry, yaw)]
    out = []
    for k in range(len(poly)):
        out += _line(poly[k], poly[(k + 1) % len(poly)])
    return out


def touch_bounds(verts):
    if not verts:
        return (math.inf, math.inf, -math.inf, -math.inf)
    return (min(v[0] for v in verts) + 0.0, min(v[1] for v in verts) + 0.0, max(v[0] for v in verts) + 0.0,
            max(v[1] for v in verts) + 0.0)


# ---- the compiled ones ------------------------------------------------------------------------------------------------
class Window(C.Structure):
    _fields_ = [("origin_x", C.c_double), ("origin_y", C.c_double), ("resolution", C.c_double), ("size_x", C.c_int),
                ("size_y", C.c_int)]


class PublisherState(C.Structure):   # gem_costmap_publisher
    _fields_ = [("always_send_full", C.c_int), ("saved", C.c_int), ("resolution", C.c_float), ("size_x", C.c_int),
                ("size_y", C.c_int), ("origin_x", C.c_double), ("origin_y", C.c_double), ("x0", C.c_int), ("xn", C.c_int),
                ("y0", C.c_int), ("yn", C.c_int)]


_orc = _host = None


def orc():
    global _orc
    if _orc is None:
        lib = native.shared_library("orc_footprint", [os.path.join(HERE, "orc_footprint.c")], native.ORACLE_C, ["-lm"])
        P = C.c_void_p
        lib.orc_footprint.argtypes = [P, P, P, C.c_int, C.c_double, C.c_double, C.c_double, P, P, C.c_long]
        lib.orc_footprint.restype = C.c_long
        lib.orc_column_walk.argtypes = [P, C.c_long, P, C.c_long]
        lib.orc_column_walk.restype = C.c_long
        _orc = lib
    return _orc


def host():
    global _host
    if _host is None:
        lib = native.shared_library("costmap_pub_host", [os.path.join(HERE, "costmap_pub_host.cpp")], native.HOST_CXX)
        P, ll = C.c_void_p, C.c_longlong
        hdr = [C.c_uint, C.c_uint, C.c_uint, C.c_char_p]
        lib.cp_translate.argtypes, lib.cp_translate.restype = [C.c_uint], C.c_int
        lib.cp_publisher_init.argtypes, lib.cp_publisher_init.restype = [C.POINTER(PublisherState), C.c_int], None
        lib.cp_publisher_bounds.argtypes = [C.POINTER(PublisherState), C.c_int, C.c_int, C.c_int, C.c_int]
        lib.cp_publisher_bounds.restype = None
        lib.cp_publish.argtypes = hdr + [C.POINTER(Window), P, C.POINTER(PublisherState), C.c_int, P, ll, C.POINTER(C.c_int),
                                         C.POINTER(C.c_int)]
        lib.cp_publish.restype = ll
        lib.cp_footprint_msg.argtypes = hdr + [P, C.c_int, C.c_double, C.c_double, C.c_double, P, ll]
        lib.cp_footprint_msg.restype = ll
        lib.cp_footprint_cells.argtypes = [C.POINTER(Window), P, C.c_int, C.c_double, C.c_double, C.c_double, P, P, ll]
        lib.cp_footprint_cells.restype = ll
        lib.cp_column_walk.argtypes = [P, ll, P, ll]
        lib.cp_column_walk.restype = ll
        _host = lib
    return _host


def _spec(footprint):
    a = np.ascontiguousarray(np.asarray(footprint, np.float64).reshape(-1, 2))
    return a, a.shape[0]


def orc_footprint_cells(window, footprint, rx, ry, yaw):
    """the C oracle's (vertices, cells), cells None when a vertex lies outside"""
    spec, n = _spec(footprint)
    w = np.array(window[:3], np.float64)
    size = np.array(window[3:], np.int32)
    verts = np.zeros(max(2 * n, 2), np.float64)
    cap = 1 << 20
    cells = np.zeros(2 * cap, np.uint32)
    k = orc().orc_footprint(w.ctypes.data, size.ctypes.data, spec.ctypes.data, n, rx, ry, yaw, verts.ctypes.data, cells.ctypes.data, cap)
    assert k != -2
    vs = [(float(verts[2 * i]), float(verts[2 * i + 1])) for i in range(n)]
    return vs, (None if k == -1 else [tuple(int(v) for v in cells[2 * i:2 * i + 2]) for i in range(k)])


def host_footprint_cells(window, footprint, rx, ry, yaw):
    spec, n = _spec(footprint)
    verts = np.zeros(max(2 * n, 2), np.float64)
    cap = 1 << 20
    cells = np.zeros(2 * cap, np.uint32)
    k = host().cp_footprint_cells(C.byref(Window(*window)), spec.ctypes.data, n, rx, ry, yaw, verts.ctypes.data, cells.ctypes.data, cap)
    assert k != -2
    vs = [(float(verts[2 * i]), float(verts[2 * i + 1])) for i in range(n)]
    return vs, (None if k == -1 else [tuple(int(v) for v in cells[2 * i:2 * i + 2]) for i in range(k)])


def walk_both(cells):
    """F4 on a crafted list through the C oracle and the library's header: (orc result, host result)"""
    a = np.ascontiguousarray(np.asarray(cells, np.uint32).reshape(-1, 2))
    res = []
    for fn in (orc().orc_column_walk, host().cp_column_walk):
        out = np.zeros(2 * 65536, np.uint32)
        k = fn(a.ctypes.data, a.shape[0], out.ctypes.data, 65536)
        assert k >= 0
        res.append([tuple(int(v) for v in out[2 * i:2 * i + 2]) for i in range(k)])
    return res


def host_footprint_msg(hdr: tuple, footprint, rx, ry, yaw) -> bytes:
    seq, sec, nsec, fid = hdr
    spec, n = _spec(footprint)
    out = np.zeros(4096 + 12 * n + len(fid), np.uint8)
    k = host().cp_footprint_msg(seq, sec, nsec, fid, spec.ctypes.data, n, rx, ry, yaw, out.ctypes.data, out.size)
    assert k >= 0, k
    return out[:k].tobytes()


class HostPublisher:
    """the library's publisher (gem_rosfmt.h P1-P4) on the host, the data translated from a host grid"""

    def __init__(self, always_send_full: bool = False):
        self.s = PublisherState()
        host().cp_publisher_init(C.byref(self.s), 1 if always_send_full else 0)

    def bounds(self, x0, xn, y0, yn):
        host().cp_publisher_bounds(C.byref(self.s), x0, xn, y0, yn)

    def state(self):
        return bytes(self.s)

    def publish(self, hdr: tuple, window, grid, force_full=False, capacity=None, query=False):
        """(kind, rect, message bytes or the size when nothing was written, or -1 when refused)"""
        seq, sec, nsec, fid = hdr
        g = np.ascontiguousarray(grid, np.uint8)
        cap = (1 << 21) + len(fid) if capacity is None else capacity
        out = np.full(max(cap, 1), 0xA5, np.uint8)
        kind, rect = C.c_int(), (C.c_int * 4)()
        n = host().cp_publish(seq, sec, nsec, fid, C.byref(Window(*window)), g.ctypes.data, C.byref(self.s), 1 if force_full else 0,
                              None if query else out.ctypes.data, 0 if query else cap, C.byref(kind), rect)
        k = {0: "none", 1: "full", 2: "update"}[kind.value]
        if n < 0 or query or n > cap:
            return k, tuple(rect), n
        return k, tuple(rect), out[:n].tobytes()
