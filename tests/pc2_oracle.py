"""Oracle of gem_pointcloud2_mapping / gem_decode_pointcloud2: ctypes binding of tests/orc_pointcloud2.c, compiled into a
temporary directory (the checkout may be read-only).  TEST INFRASTRUCTURE ONLY.

decode(case) returns (records, mapping): records an (n, 32) uint8 array of PointXYZRGBICT records as fromPCLPointCloud2
fills them (stale bytes DEFINED as 0), mapping a dict {spans, fast_path, matched, points, bytes}; None for a refused
layout.  xyzi(records) is what the device decode writes: struct bytes 0-11 and 24-27 as an (n, 4) float32 array."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import native

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orc_pointcloud2.c")
_lib = None


class Field(C.Structure):
    _fields_ = [("name", C.c_char * 32), ("offset", C.c_uint), ("datatype", C.c_ubyte), ("count", C.c_uint)]


class Cloud(C.Structure):
    _fields_ = [("width", C.c_uint), ("height", C.c_uint), ("point_step", C.c_uint), ("row_step", C.c_uint),
                ("is_bigendian", C.c_ubyte), ("nfields", C.c_int), ("fields", C.POINTER(Field))]


class Span(C.Structure):
    _fields_ = [("serialized_offset", C.c_uint), ("struct_offset", C.c_uint), ("size", C.c_uint)]


class Mapping(C.Structure):
    _fields_ = [("nspans", C.c_int), ("spans", Span * 7), ("fast_path", C.c_int), ("matched", C.c_uint),
                ("points", C.c_longlong), ("bytes", C.c_ulonglong)]


def load():
    global _lib
    if _lib is None:
        lib = native.shared_library("orc_pointcloud2", [SRC], native.FORMAT_C)
        lib.orc_pc2_decode.argtypes = [C.POINTER(Cloud), C.c_void_p, C.c_ulonglong, C.c_void_p, C.POINTER(Mapping)]
        lib.orc_pc2_decode.restype = C.c_int
        _lib = lib
    return _lib


def _cloud(case):
    arr = (Field * max(len(case["fields"]), 1))()
    for k, (name, off, dt, cnt) in enumerate(case["fields"]):
        nb = name.encode()[:32]
        C.memmove(C.addressof(arr[k]) + Field.name.offset, nb, len(nb))
        arr[k].offset, arr[k].datatype, arr[k].count = off, dt, cnt
    c = Cloud(case["width"], case["height"], case["point_step"], case["row_step"], case.get("is_bigendian", 0),
              len(case["fields"]), C.cast(arr, C.POINTER(Field)))
    return c, arr


def mapping_dict(mp):
    names = ["x", "y", "z", "rgb", "intensity", "covariance", "travers"]
    return {"spans": [(mp.spans[k].serialized_offset, mp.spans[k].struct_offset, mp.spans[k].size) for k in range(mp.nspans)],
            "fast_path": bool(mp.fast_path), "matched": [n for k, n in enumerate(names) if mp.matched >> k & 1],
            "points": int(mp.points), "bytes": int(mp.bytes)}


def decode(case):
    c, keep = _cloud(case)
    data = np.ascontiguousarray(case["data"], np.uint8)
    n = case["width"] * case["height"]
    rec = np.zeros((max(n, 1), 32), np.uint8)
    mp = Mapping()
    if load().orc_pc2_decode(C.byref(c), C.c_void_p(data.ctypes.data), int(case.get("data_bytes", data.nbytes)),
                             C.c_void_p(rec.ctypes.data), C.byref(mp)) != 0:
        return None
    del keep
    return rec[:n].copy(), mapping_dict(mp)


def xyzi(records):
    r = np.ascontiguousarray(records, np.uint8).reshape(-1, 32)
    return np.ascontiguousarray(np.concatenate([r[:, 0:12], r[:, 24:28]], axis=1)).view(np.float32).reshape(-1, 4)
