"""Oracle of gem_mls_upsample: ctypes binding of tests/orc_mls.c, compiled with the oracle's flags (and the library's
gem_mathd.h, the exp / atan2 / sincos both sides share) into a temporary directory (the checkout may be read-only).
TEST INFRASTRUCTURE ONLY.

upsample() takes an (n, 8) float32 array of PointXYZRGBICT records and returns (out, info): out the min(count, capacity)
written records, info a dict {count, processed, fitted, skipped, max_neighbours}; None where the library reports an
error.  detail() returns what M2-M4 give one point."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import native

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orc_mls.c")
UPSAMPLING = {"none": 0, "random_uniform_density": 1}
GEM = {"search_radius": 0.5, "sqr_gauss_param": 0.25, "polynomial_fit": True, "order": 5,
       "upsampling": "random_uniform_density", "point_density": 1000, "seed": 0}
_lib = None


class Params(C.Structure):
    _fields_ = [("search_radius", C.c_double), ("sqr_gauss_param", C.c_double), ("polynomial_fit", C.c_int), ("order", C.c_int),
                ("upsampling", C.c_int), ("point_density", C.c_int), ("seed", C.c_ulonglong)]


class Info(C.Structure):
    _fields_ = [("count", C.c_longlong), ("processed", C.c_int), ("fitted", C.c_int), ("skipped", C.c_int),
                ("max_neighbours", C.c_int)]


class Detail(C.Structure):
    _fields_ = [("nb", C.c_int), ("fitted", C.c_int), ("attempted", C.c_int), ("normal", C.c_double * 3), ("point", C.c_double * 3),
                ("u_axis", C.c_double * 3), ("v_axis", C.c_double * 3), ("c", C.c_double * 21)]


def load():
    global _lib
    if _lib is None:
        lib = native.shared_library("orc_mls", [SRC], native.ORACLE_C + ["-I", native.CSRC], ["-lm"])
        lib.orc_mls_upsample.argtypes = [C.c_void_p, C.c_int, C.POINTER(Params), C.c_void_p, C.c_longlong, C.POINTER(Info)]
        lib.orc_mls_upsample.restype = C.c_int
        lib.orc_mls_detail.argtypes = [C.c_void_p, C.c_int, C.POINTER(Params), C.c_int, C.POINTER(Detail), C.c_void_p]
        lib.orc_mls_detail.restype = C.c_int
        for f in ("orc_mls_exp_d", "orc_mls_atan2_d"):
            getattr(lib, f).restype = C.c_double
        lib.orc_mls_exp_d.argtypes = [C.c_double]
        lib.orc_mls_atan2_d.argtypes = [C.c_double, C.c_double]
        lib.orc_mls_sincos_d.argtypes = [C.c_double, C.POINTER(C.c_double), C.POINTER(C.c_double)]
        _lib = lib
    return _lib


def params(overrides=None):
    q = dict(GEM)
    q.update(overrides or {})
    up = UPSAMPLING[q["upsampling"]] if isinstance(q["upsampling"], str) else int(q["upsampling"])
    return Params(float(q["search_radius"]), float(q["sqr_gauss_param"]), 1 if q["polynomial_fit"] else 0, int(q["order"]), up,
                  int(q["point_density"]), int(q["seed"]) & 0xFFFFFFFFFFFFFFFF)


def upsample(recs, overrides=None, capacity=None):
    pts = np.ascontiguousarray(recs, np.float32).reshape(-1, 8)
    n = pts.shape[0]
    p = params(overrides)
    info = Info()
    if capacity is None:   # size query first, then the whole output
        if load().orc_mls_upsample(C.c_void_p(pts.ctypes.data), n, C.byref(p), None, 0, C.byref(info)) != 0:
            return None
        capacity = info.count
    cap = int(capacity)
    out = np.zeros((max(cap, 1), 8), np.float32)
    if load().orc_mls_upsample(C.c_void_p(pts.ctypes.data), n, C.byref(p), C.c_void_p(out.ctypes.data), cap, C.byref(info)) != 0:
        return None
    return out[:min(info.count, cap)].copy(), {k: getattr(info, k) for k, _ in Info._fields_}


def detail(recs, i, overrides=None):
    pts = np.ascontiguousarray(recs, np.float32).reshape(-1, 8)
    d = Detail()
    nb = np.zeros(max(pts.shape[0], 1), np.int32)
    assert load().orc_mls_detail(C.c_void_p(pts.ctypes.data), pts.shape[0], C.byref(params(overrides)), int(i), C.byref(d),
                                 C.c_void_p(nb.ctypes.data)) == 0
    return {"nb": nb[:d.nb].copy(), "fitted": d.fitted, "attempted": d.attempted, "normal": np.array(d.normal[:]),
            "point": np.array(d.point[:]), "u_axis": np.array(d.u_axis[:]), "v_axis": np.array(d.v_axis[:]), "c": np.array(d.c[:])}


def exp_d(x):
    f = load().orc_mls_exp_d
    return np.array([f(float(v)) for v in np.ravel(x)])


def atan2_d(y, x):
    f = load().orc_mls_atan2_d
    return np.array([f(float(a), float(b)) for a, b in zip(np.ravel(y), np.ravel(x))])


def sincos_d(x):
    s, c = C.c_double(), C.c_double()
    out = []
    for v in np.ravel(x):
        load().orc_mls_sincos_d(float(v), C.byref(s), C.byref(c))
        out.append((s.value, c.value))
    return np.array(out)
