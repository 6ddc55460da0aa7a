"""Oracle of gem_costmap_inflate: ctypes binding of tests/orc_inflate.c, compiled with the flags of the costmap oracle into
a temporary directory (the checkout may be read-only), and an independent Python restatement of the brushfire.  TEST
INFRASTRUCTURE ONLY.

A grid is a (size_y, size_x) uint8 array; params a dict {inflation_radius, cost_scaling_factor, inscribed_radius,
inflate_unknown}; a rect (min_i, min_j, max_i, max_j)."""
from __future__ import annotations

import ctypes as C
import math
import os

import numpy as np

import native

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orc_inflate.c")
_lib = None

FREE, INSCRIBED, LETHAL, UNKNOWN = 0, 253, 254, 255


def load():
    global _lib
    if _lib is None:
        lib = native.shared_library("orc_inflate", [SRC], native.ORACLE_C, ["-lm"])
        lib.orc_inflate.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int,
                                    C.c_int, C.c_int, C.c_int, C.c_int]
        lib.orc_inflate.restype = C.c_longlong
        _lib = lib
    return _lib


def params(radius, weight=10.0, inscribed=0.40, unknown=False) -> dict:
    return {"inflation_radius": float(radius), "cost_scaling_factor": float(weight), "inscribed_radius": float(inscribed),
            "inflate_unknown": bool(unknown)}


def inflate(grid, resolution, p, rect):
    """orc_inflate on a copy of `grid`; returns the new grid"""
    g = np.ascontiguousarray(grid, np.uint8).copy()
    sy, sx = g.shape
    i0, j0, i1, j1 = (int(v) for v in rect)
    load().orc_inflate(C.c_void_p(g.ctypes.data), sx, sy, float(resolution), p["inflation_radius"], p["cost_scaling_factor"],
                       p["inscribed_radius"], 1 if p["inflate_unknown"] else 0, i0, j0, i1, j1)
    return g


# ---- independent restatements --------------------------------------------------------------------------------------------
def cell_radius(grid_shape, resolution, radius) -> int:
    sy, sx = grid_shape
    r = max(0.0, math.ceil(radius / resolution))
    return int(min(r, math.ceil(float(np.hypot(float(sx), float(sy)))) + 1.0))


def tables(r, resolution, weight, inscribed):
    """computeCaches with libm's hypot (numpy's) and exp (math's)"""
    n = r + 2
    ii, jj = np.meshgrid(np.arange(n, dtype=np.float64), np.arange(n, dtype=np.float64), indexing="ij")
    dist = np.hypot(ii, jj)
    cost = np.zeros((n, n), np.uint8)
    for i in range(n):
        for j in range(n):
            d = float(dist[i, j])
            if d == 0:
                c = LETHAL
            elif d * resolution <= inscribed:
                c = INSCRIBED
            else:
                c = int(252 * math.exp(-1.0 * weight * (d * resolution - inscribed)))
            cost[i, j] = c
    return dist, cost


def _write(master, idx, c, unknown):
    o = int(master.flat[idx])
    if o == UNKNOWN and (c > FREE if unknown else c >= INSCRIBED):
        master.flat[idx] = c
    else:
        master.flat[idx] = max(o, c)


def brushfire(grid, resolution, p, rect, reverse=False):
    """InflationLayer::updateCosts restated as a dict of lists walked in key order (reverse=True walks each bin backwards:
    the order witnesses must then differ)"""
    m = np.ascontiguousarray(grid, np.uint8).copy()
    sy, sx = m.shape
    r = cell_radius(m.shape, resolution, p["inflation_radius"])
    if r == 0:
        return m
    dist, cost = tables(r, resolution, p["cost_scaling_factor"], p["inscribed_radius"])
    i0, j0, i1, j1 = (int(v) for v in rect)
    i0, j0, i1, j1 = max(0, i0 - r), max(0, j0 - r), min(sx, i1 + r), min(sy, j1 + r)
    seen = np.zeros(sx * sy, bool)
    bins = {0.0: [(j * sx + i, i, j, i, j) for j in range(j0, j1) for i in range(i0, i1) if m[j, i] == LETHAL]}
    cur = -1.0
    while True:
        later = [k for k in bins if k > cur]
        if not later:
            break
        cur = min(later)
        lst = bins[cur]
        k = 0
        while k < len(lst):
            idx, mx, my, ssx, ssy = lst[len(lst) - 1 - k] if reverse else lst[k]
            k += 1
            if seen[idx]:
                continue
            seen[idx] = True
            _write(m, idx, int(cost[abs(mx - ssx), abs(my - ssy)]), p["inflate_unknown"])
            for ok, nx, ny in ((mx > 0, mx - 1, my), (my > 0, mx, my - 1), (mx < sx - 1, mx + 1, my), (my < sy - 1, mx, my + 1)):
                ni = ny * sx + nx
                if not ok or seen[ni]:
                    continue
                d = float(dist[abs(nx - ssx), abs(ny - ssy)])
                if d > r:
                    continue
                assert d != cur, "a push into the bin being walked"
                bins.setdefault(d, []).append((ni, nx, ny, ssx, ssy))
    return m


def nearest_obstacle(grid, resolution, p, rect):
    """the exact nearest-seed cost: every cell within r of a seed gets the cost of its nearest seed, with I4's write
    rule (what a Euclidean distance transform would give; the EDT witnesses must differ from it)"""
    m = np.ascontiguousarray(grid, np.uint8).copy()
    sy, sx = m.shape
    r = cell_radius(m.shape, resolution, p["inflation_radius"])
    if r == 0:
        return m
    dist, cost = tables(r, resolution, p["cost_scaling_factor"], p["inscribed_radius"])
    i0, j0, i1, j1 = (int(v) for v in rect)
    i0, j0, i1, j1 = max(0, i0 - r), max(0, j0 - r), min(sx, i1 + r), min(sy, j1 + r)
    seeds = [(i, j) for j in range(j0, j1) for i in range(i0, i1) if m[j, i] == LETHAL]
    if not seeds:
        return m
    s = np.array(seeds)
    out = m.copy()
    for y in range(sy):
        for x in range(sx):
            dx, dy = np.abs(s[:, 0] - x), np.abs(s[:, 1] - y)
            d = dist[np.minimum(dx, r + 1), np.minimum(dy, r + 1)]
            k = int(np.argmin(d))
            if float(d[k]) <= r:
                _write(out, y * sx + x, int(cost[dx[k], dy[k]]), p["inflate_unknown"])
    return out
