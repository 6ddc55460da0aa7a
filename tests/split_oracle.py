"""Oracle of gem_grid_cloud_split: ctypes binding of tests/orc_grid_split.c, compiled with the oracle's flags into a
temporary directory (the checkout may be read-only).  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import native

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orc_grid_split.c")
_lib = None


def load():
    global _lib
    if _lib is None:
        lib = native.shared_library("orc_grid_split", [SRC], native.ORACLE_C, ["-lm"])
        P = C.c_void_p
        lib.orc_grid_split.argtypes = [C.c_int, P, C.c_int, C.c_double, C.c_double, P, P, P, P, P]
        lib.orc_grid_split.restype = None
        _lib = lib
    return _lib


def _p(a):
    return C.c_void_p(a.ctypes.data)


def grid_split(records, mean_k=20, stddev_mul=1.0, travers_threshold=0.0):
    """orc_grid_split over (n, 8) float32 grid-cloud records: dict with road / obstacle records, dist (float32 per
    point), valid, mean, stddev, threshold"""
    lib = load()
    rec = np.ascontiguousarray(records, np.float32).reshape(-1, 8)
    n = rec.shape[0]
    dist = np.empty(max(n, 1), np.float32)
    road = np.empty(max(n, 1), np.int32)
    obst = np.empty(max(n, 1), np.int32)
    counts = np.zeros(3, np.int32)
    stats = np.zeros(3, np.float64)
    lib.orc_grid_split(int(n), _p(rec), int(mean_k), float(stddev_mul), float(travers_threshold), _p(dist), _p(road),
                       _p(obst), _p(counts), _p(stats))
    return {"dist": dist[:n].copy(), "road": rec[road[:counts[1]]], "obstacle": rec[obst[:counts[2]]],
            "valid": int(counts[0]), "mean": float(stats[0]), "stddev": float(stats[1]), "threshold": float(stats[2])}
