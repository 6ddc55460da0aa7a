"""The node's colour lookup (GEM_COLOUR_LOOKUP_NODE, DESIGN.md f19) without a GPU.  TEST INFRASTRUCTURE ONLY.

- node(): tests/orc_colour_lookup.c, the literal loop with OpenCV's Circle() written out, compiled into a temporary
  directory (the checkout may be read-only).
- literal(): an independent Python restatement of the loop: a working copy, four neighbour pixels painted when inside.
- closed_form(): C5 in numpy: parent(i) by a sorted search per neighbour pixel, roots by pointer jumping.
All three take xyzi (n, 4) float32, the two transforms and a BGR8 image of shape (height, row_stride) uint8 with the
pixels in the first 3 * width bytes of each row, and return (xyzi with intensities zeroed outside the image, rgba)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import native

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orc_colour_lookup.c")
_lib = None


def load():
    global _lib
    if _lib is None:
        lib = native.shared_library("orc_colour_lookup", [SRC], native.ORACLE_C)
        P = C.c_void_p
        lib.orc_colourise_node.restype = C.c_int
        lib.orc_colourise_node.argtypes = [P, C.c_int, P, P, P, C.c_int, C.c_int, C.c_int, P]
        _lib = lib
    return _lib


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _args(xyzi, T_camera, T_lidar, img):
    xyzi = np.array(xyzi, np.float32, copy=True, order="C").reshape(-1, 4)
    tc = np.ascontiguousarray(T_camera, np.float64).reshape(-1)
    tl = np.ascontiguousarray(T_lidar, np.float64).reshape(-1)
    img = np.ascontiguousarray(img, np.uint8)
    return xyzi, tc, tl, img


def node(xyzi, T_camera, T_lidar, img, width: int):
    xyzi, tc, tl, img = _args(xyzi, T_camera, T_lidar, img)
    rgba = np.zeros((xyzi.shape[0], 4), np.uint8)
    before = img.copy()
    rc = load().orc_colourise_node(_p(xyzi), xyzi.shape[0], _p(tc), _p(tl), _p(img), int(width), img.shape[0], img.shape[1],
                                   _p(rgba))
    assert rc == 0 and np.array_equal(img, before)
    return xyzi, rgba


def project(xyzi, T_camera, T_lidar, width: int, height: int):
    """(mx, my, inside) per point: P = Tc Tl with left-to-right sums, the projection in float64 without contraction,
    X / Z rounded to float32 and truncated toward zero (NaN to 0)"""
    tc = np.asarray(T_camera, np.float64).reshape(3, 4)
    tl = np.asarray(T_lidar, np.float64).reshape(4, 4)
    P = np.empty((3, 4))
    for i in range(3):
        for j in range(4):
            a = tc[i, 0] * tl[0, j]
            for k in range(1, 4):
                a = a + tc[i, k] * tl[k, j]
            P[i, j] = a
    x, y, z = (np.asarray(xyzi, np.float32)[:, k].astype(np.float64) for k in range(3))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        X, Y, Z = (((P[r, 0] * x + P[r, 1] * y) + P[r, 2] * z) + P[r, 3] * 1.0 for r in range(3))
        px, py = (X / Z).astype(np.float32), (Y / Z).astype(np.float32)

    def trunc(f):
        g = np.where(np.isnan(f), 0.0, np.clip(np.trunc(f.astype(np.float64)), -2.0**31, 2.0**31 - 1))
        return g.astype(np.int64)

    mx, my = trunc(px), trunc(py)
    return mx, my, (mx > 0) & (mx < width) & (my > 0) & (my < height) & (Z > 0)


def literal(xyzi, T_camera, T_lidar, img, width: int):
    xyzi, _, _, img = _args(xyzi, T_camera, T_lidar, img)
    H = img.shape[0]
    mx, my, inside = project(xyzi, T_camera, T_lidar, width, H)
    work = img[:, :3 * width].reshape(H, width, 3).copy()
    rgba = np.zeros((xyzi.shape[0], 4), np.uint8)
    for i in range(xyzi.shape[0]):
        if not inside[i]:
            xyzi[i, 3] = 0.0
            continue
        x, y = int(mx[i]), int(my[i])
        b, g, r = (int(v) for v in work[y, x])
        rgba[i] = (r, g, b, 255)
        for nx, ny in ((x - 1, y), (x + 1, y), (x, y - 1), (x, y + 1)):
            if 0 <= nx < width and 0 <= ny < H:
                work[ny, nx] = (b, g, r)
    return xyzi, rgba


def parents(key, inside, width: int, height: int):
    """parent(i) of C5 (-1: none) from pixel keys my * width + mx"""
    n = key.shape[0]
    idx = np.flatnonzero(inside)
    k = key[idx]
    order = np.lexsort((idx, k))
    sk, si = k[order], idx[order]
    comb = sk * (n + 1) + si                          # (key, index) in lexicographic order
    mx, my = k % width, k // width
    best = np.full(idx.shape[0], -1, np.int64)
    for dx, dy in ((-1, 0), (1, 0), (0, -1), (0, 1)):
        ok = (mx + dx >= 1) & (mx + dx < width) & (my + dy >= 1) & (my + dy < height)
        nk = k + dy * width + dx
        pos = np.searchsorted(comb, nk * (n + 1) + idx) - 1   # the last (key, index) below (nk, i)
        hit = ok & (pos >= 0) & (sk[np.maximum(pos, 0)] == nk)
        best = np.where(hit, np.maximum(best, si[np.maximum(pos, 0)]), best)
    out = np.full(n, -1, np.int64)
    out[idx] = best
    return out


def closed_form(xyzi, T_camera, T_lidar, img, width: int):
    xyzi, _, _, img = _args(xyzi, T_camera, T_lidar, img)
    H = img.shape[0]
    mx, my, inside = project(xyzi, T_camera, T_lidar, width, H)
    key = np.where(inside, my * width + mx, 0)
    par = parents(key, inside, width, H)
    up = np.where(par >= 0, par, np.arange(xyzi.shape[0]))
    while True:
        nxt = up[up]
        if np.array_equal(nxt, up):
            break
        up = nxt
    rk = key[up]
    px = img[(rk // width)[:, None], 3 * (rk % width)[:, None] + np.arange(3)]
    rgba = np.zeros((xyzi.shape[0], 4), np.uint8)
    rgba[inside, 0], rgba[inside, 1], rgba[inside, 2] = px[inside, 2], px[inside, 1], px[inside, 0]
    rgba[inside, 3] = 255
    xyzi[~inside, 3] = 0.0
    return xyzi, rgba


def chain_depth(xyzi, T_camera, T_lidar, width: int, height: int) -> int:
    """the longest parent chain (links) of a cloud"""
    mx, my, inside = project(xyzi, T_camera, T_lidar, width, height)
    par = parents(np.where(inside, my * width + mx, 0), inside, width, height)
    depth = np.zeros(par.shape[0], np.int64)
    for i in np.flatnonzero(par >= 0):   # parents come first
        depth[i] = depth[par[i]] + 1
    return int(depth.max(initial=0))
