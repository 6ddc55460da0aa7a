"""ShimMap: RefMap's interface over the drop-in shim (compat/gpu_process_shim.cpp, built with tests/cxx/shim_harness.cpp
into a shared library by test_cxx_facade.compile_with_shim).  So tests drive exactly the nine functions GEM's node
calls.  TEST INFRASTRUCTURE, needs a GPU to run.

The node observes the map only through Map_feature's outputs, and so does get_layer: elevation, variance, intensity
and the colours.  That is harmless to the other layers: Map_feature writes only `traver` (gpu_process.cu:660-667), and
the node's next Map_feature recomputes it before the next Raytracing reads it.  `lowest` and `traver` are refused.
Like the reference, the shim keeps one map per process: each ShimMap re-initialises it."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import ref_lib
from test_cxx_facade import compile_with_shim

FEATURE_LAYERS = ("elevation", "variance", "intensity", "color_r", "color_g", "color_b")
_lib = None


def load(out_dir):
    """the harness library, built into out_dir the first time a process asks for it"""
    global _lib
    if _lib is None:
        _lib = C.CDLL(compile_with_shim(out_dir, "shim_harness", shared=True))
    return _lib


class ShimMap(ref_lib.RefMap):
    def __init__(self, lib, length, resolution, mahalanobis=2.5, obstacle_threshold=0.7):
        self.lib = lib
        self.L, self.res = int(length), float(resolution)
        self.lib.ref_init(self.L, C.c_float(self.res), C.c_float(mahalanobis), C.c_float(obstacle_threshold))

    def get_layer(self, name):
        if name not in FEATURE_LAYERS:
            raise ValueError(f"the shim serves {FEATURE_LAYERS} through Map_feature, not {name!r}")
        return self.map_feature()[name].reshape(self.L, self.L)

    def layers(self, names):
        f = self.map_feature()
        for n in names:
            if n not in FEATURE_LAYERS:
                raise ValueError(f"the shim serves {FEATURE_LAYERS} through Map_feature, not {n!r}")
        return {n: f[n].reshape(self.L, self.L) for n in names}

    def set_layer(self, name, arr):
        raise ValueError("the nine functions cannot set a layer")

    def state(self):
        raise ValueError("the nine functions do not expose the scroll state")

    def close(self):
        pass


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    """shim(L, res, **kw) -> a freshly initialised ShimMap (the one map of the process)"""
    lib = load(tmp_path_factory.mktemp("shim"))
    return lambda L, res, **kw: ShimMap(lib, L, res, **kw)
