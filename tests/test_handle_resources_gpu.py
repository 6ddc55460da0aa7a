"""A handle's CUDA resources: a refused pinned allocation leaves no error behind for the next call, and a handle destroyed
with work queued on its own stream, its copy stream and the global map's stream releases cleanly."""
import ctypes as C

import numpy as np
import pytest
import torch

import gem_b200
import global_map_cases as gc
from gem_b200 import _lib, synth
from helpers import assert_layers_equal
from oracle_lib import OracleMap

pytestmark = pytest.mark.gpu
GEM_ERR_NOMEM = 4


def laser_frame(T):
    return gem_b200.make_frame(T, gem_b200.LaserSensorProcessor())


def add_matches_oracle(g, fr, what):
    o = OracleMap(200, 0.1, compat_box_filter=False)
    f = laser_frame(fr["T"])
    for m in (g, o):
        m.move(fr["position"])
        m.add(fr["xyzi"], fr["rgba"], f)
    assert_layers_equal(g, o, what=what)


def test_refused_pinned_allocation_leaves_no_error_behind():
    """more bytes than any virtual address space: refused before anything is reserved; the next call on this thread must
    not see the refusal as a failed launch"""
    fr = synth.hdl64_frame(0)
    g = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False)
    p = C.c_void_p()
    assert _lib.load().gem_host_alloc(C.byref(p), 1 << 62) == GEM_ERR_NOMEM
    add_matches_oracle(g, fr, "add after a refused gem_host_alloc")   # no torch CUDA call in between
    g.close()


def test_destroy_with_work_queued_on_every_stream():
    frames = [synth.hdl64_frame(k) for k in range(2)]
    g = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False)
    pinned = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
    out = {k: pinned(np.zeros((200, 200), np.float32)).numpy().T for k in _lib.EXPORT_LAYERS}   # Fortran order
    g.export_layers_begin(out)                                                                  # copy stream, no _end
    host = [(pinned(fr["xyzi"]), pinned(fr["rgba"])) for fr in frames]
    fobj = [laser_frame(fr["T"]) for fr in frames]
    for fr, (x, c), f in zip(frames, host, fobj):
        g.move(fr["position"])
        g.add_host_async_fast(C.c_void_p(x.data_ptr()), C.c_void_p(c.data_ptr()), fr["xyzi"].shape[0], C.byref(f))
    cen = gc._line(2, 1.0)
    for _, recs, pose in gc.chain("destroy", cen, [2000, 2000]):
        g.global_map_push(torch.from_numpy(np.array(recs, np.float32).reshape(-1, 8)).cuda(), pose)
    g.global_map_update(gc.perturbed(gc._kf(cen), 3), 0.1)
    g.close()                                                                                   # no sync()
    add_matches_oracle(gem_b200.ElevationMap(200, 0.1, compat_box_filter=False), frames[0], "fresh map after destroy")
