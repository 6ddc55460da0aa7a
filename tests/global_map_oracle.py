"""Oracles of the gem_global_map_* calls (DESIGN.md f16).  TEST INFRASTRUCTURE ONLY.

`OracleStack` binds tests/orc_global_map.c, compiled with the oracle's flags into a temporary directory (the checkout may
be read-only) and linked against oracle/libgem_oracle.so, whose orc_transform_cloud and orc_refuse_submaps it calls.
`PyStack` is the independent restatement: numpy float32 pose arithmetic in the stated order, submaps.neighbours, the
dict re-fusion refuse_cases.refuse and oracle_lib.transform_cloud.  Both have the methods of the stack on
gem_b200.ElevationMap (reset, push, update) and report their state as `state()`: (list of (n, 8) float32 submaps,
(keyframes, 4, 4) poses, (keyframes, 2) centres)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import native
import oracle_lib
import refuse_cases as rc
from gem_b200 import submaps as sm

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orc_global_map.c")
F = np.float32
_lib = None


def load():
    global _lib
    if _lib is None:
        oracle_lib.load()  # builds oracle/libgem_oracle.so
        odir = oracle_lib.ODIR
        lib = native.shared_library("orc_global_map", [SRC], native.ORACLE_C + ["-I", odir],
                                    ["-L", odir, "-lgem_oracle", "-Wl,-rpath," + odir, "-lm"])
        P = C.c_void_p
        lib.orc_gmap_create.restype = P
        lib.orc_gmap_destroy.argtypes = [P]
        lib.orc_gmap_reset.argtypes = [P]
        lib.orc_gmap_push.argtypes = [P, P, C.c_int, P]
        lib.orc_gmap_update.restype = C.c_int
        lib.orc_gmap_update.argtypes = [P, P, C.c_int, C.c_double, C.c_double, C.c_int]
        lib.orc_gmap_relative_pose.argtypes = [P, P, P]
        for fn in ("orc_gmap_submaps", "orc_gmap_keyframes"):
            getattr(lib, fn).restype = C.c_int
            getattr(lib, fn).argtypes = [P]
        lib.orc_gmap_count.restype = C.c_int
        lib.orc_gmap_count.argtypes = [P, C.c_int]
        lib.orc_gmap_read.argtypes = [P, C.c_int, P]
        lib.orc_gmap_pose.argtypes = [P, C.c_int, P, P]
        _lib = lib
    return _lib


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _f32(a, shape):
    return np.ascontiguousarray(np.asarray(a, np.float32).reshape(shape))


class OracleStack:
    def __init__(self):
        self.lib = load()
        self.g = self.lib.orc_gmap_create()

    def __del__(self):
        if getattr(self, "g", None):
            self.lib.orc_gmap_destroy(self.g)
            self.g = None

    def reset(self):
        self.lib.orc_gmap_reset(self.g)

    def push(self, records, pose):
        r, p = _f32(records, (-1, 8)), _f32(pose, 16)
        self.lib.orc_gmap_push(self.g, _p(r), r.shape[0], _p(p))

    def update(self, opt_poses, resolution, radius=25.0, compat=True):
        o = _f32(opt_poses, (-1, 16))
        return self.lib.orc_gmap_update(self.g, _p(o), o.shape[0], float(resolution), float(radius), 1 if compat else 0)

    def state(self):
        subs = []
        for k in range(self.lib.orc_gmap_submaps(self.g)):
            a = np.empty((self.lib.orc_gmap_count(self.g, k), 8), np.float32)
            self.lib.orc_gmap_read(self.g, k, _p(a))
            subs.append(a)
        kf = self.lib.orc_gmap_keyframes(self.g)
        poses, centres = np.empty((kf, 16), np.float32), np.empty((kf, 2), np.float32)
        for i in range(kf):
            self.lib.orc_gmap_pose(self.g, i, _p(poses[i]), _p(centres[i]))
        return subs, poses.reshape(kf, 4, 4), centres


def oracle_relative_pose(pn, po):
    T = np.empty(16, np.float32)
    load().orc_gmap_relative_pose(_p(_f32(pn, 16)), _p(_f32(po, 16)), _p(T))
    return T.reshape(4, 4)


def relative_pose(pn, po):
    """optGlobalMapLoc_[i] * trajectory_[i].inverse() in numpy float32: inverse = (R^T, -(R^T t)), product = (Rn Ri,
    Rn ti + tn), every 3-term dot product (a0 b0 + a1 b1) + a2 b2"""
    pn, po = _f32(pn, (4, 4)), _f32(po, (4, 4))
    ri = po[:3, :3].T.copy()
    with np.errstate(invalid="ignore", over="ignore"):
        ti = -((ri[:, 0] * po[0, 3] + ri[:, 1] * po[1, 3]) + ri[:, 2] * po[2, 3])
        T = np.zeros((4, 4), np.float32)
        T[:3, :3] = (pn[:3, 0:1] * ri[0:1, :] + pn[:3, 1:2] * ri[1:2, :]) + pn[:3, 2:3] * ri[2:3, :]
        T[:3, 3] = ((pn[:3, 0] * ti[0] + pn[:3, 1] * ti[1]) + pn[:3, 2] * ti[2]) + pn[:3, 3]
    T[3, 3] = 1
    return T


class PyStack:
    def __init__(self):
        self.reset()

    def reset(self):
        self.subs, self.poses, self.centres = [], [np.eye(4, dtype=np.float32)], [np.zeros(2, np.float32)]

    def push(self, records, pose):
        p = _f32(pose, (4, 4)).copy()
        self.poses.append(p)
        self.centres.append(np.array([p[0, 3], p[1, 3]], np.float32))
        self.subs.append(_f32(records, (-1, 8)).copy())

    def update(self, opt_poses, resolution, radius=25.0, compat=True):
        opt = _f32(opt_poses, (-1, 4, 4))
        K = min(opt.shape[0], len(self.subs))
        for i in range(1, K):
            self.subs[i] = oracle_lib.transform_cloud(self.subs[i], relative_pose(opt[i], self.poses[i]))
            self.poses[i] = opt[i].copy()
        total = 0
        cen = np.array(self.centres[:K], np.float32).reshape(-1, 2)
        for i in range(K):
            with np.errstate(invalid="ignore"):
                nb = sm.neighbours(cen, i, radius)
            if len(nb) > 2:
                for j in nb[1:]:
                    if j == i:
                        continue
                    self.subs[j], self.subs[i], fused = rc.refuse(self.subs[j], self.subs[i], resolution, compat)[:3]
                    total += fused
        return total

    def state(self):
        return [s.copy() for s in self.subs], np.array(self.poses, np.float32), np.array(self.centres, np.float32)


def stack_difference(got, want):
    """None, or a description of the first difference of two stack states.  Bits are compared, except that a NaN equals
    any NaN in x, y, z and covariance (computed values; NaN payloads differ between the x86 oracle and the GPU)"""
    (gs, gp, gc), (ws, wp, wc) = got, want
    if len(gs) != len(ws):
        return ("submaps", len(gs), len(ws))
    for k, (a, b) in enumerate(zip(gs, ws)):
        a, b = np.ascontiguousarray(a, np.float32).reshape(-1, 8), np.ascontiguousarray(b, np.float32).reshape(-1, 8)
        if a.shape != b.shape:
            return ("count", k, a.shape[0], b.shape[0])
        diff = a.view(np.uint32) != b.view(np.uint32)
        loose = np.zeros(8, bool)
        loose[[0, 1, 2, 5]] = True
        diff &= ~(loose[None, :] & np.isnan(a) & np.isnan(b))
        if diff.any():
            r, f = np.argwhere(diff)[0]
            return ("record", k, int(r), rc.FIELDS[int(f)], hex(int(a.view(np.uint32)[r, f])), hex(int(b.view(np.uint32)[r, f])))
    for what, a, b in (("poses", gp, wp), ("centres", gc, wc)):
        a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
        if a.shape != b.shape or (a.view(np.uint32) != b.view(np.uint32)).any():
            return (what, a.tolist(), b.tolist())
    return None
