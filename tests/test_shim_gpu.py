"""The drop-in shim (compat/gpu_process_shim.cpp, driven through its nine entry points by tests/shim_lib.py) and the
device against the oracle where only the shim's own code can go wrong: the frame constants it copies from Eigen into
gem_frame (tests/frame_cases.py, pinned to the reference by tests/test_reference_pin_frames.py), a cloud longer than
the 2^20 points one launch takes (the shim creates its map with max_points = 0), and Init_GPU_elevationmap called
again with another size.  Every comparison is bit for bit, NaN as a class."""
import numpy as np
import pytest

import frame_cases as fc
import gem_b200
from gem_b200 import synth
from oracle_lib import OracleMap
from pin_cases import assert_bits
from shim_lib import FEATURE_LAYERS, shim  # noqa: F401  (shim is a fixture)
from test_reference_pin_frames import OUTPUTS

pytestmark = pytest.mark.gpu
f32 = np.float32
LAUNCH = 1 << 20                 # points per launch of a map created with max_points = 0


def _compare_feature(m, o, what):
    fo = o.map_feature()
    fm = m.map_feature()
    for name in FEATURE_LAYERS:
        assert_bits(fm[name], fo[name], f"{what} {name}")
    return fo


@pytest.mark.parametrize("c", fc.frame_cases(), ids=lambda c: c.name)
def test_frame_constants_match_oracle(c, shim):  # noqa: F811
    """Move, Process_points (all five outputs) and Fuse with non-trivial frame constants, through the shim and through
    the C ABI; `lowest` through the C ABI (the shim cannot observe it)"""
    for kind in ("device", "shim"):
        m = gem_b200.ElevationMap(c.L, c.res, compat_box_filter=True) if kind == "device" else shim(c.L, c.res)
        o = OracleMap(c.L, c.res, compat_box_filter=True)
        try:
            for a, b, name in zip(m.move(c.position), o.move(c.position), ("centre", "start", "shift")):
                assert_bits(a, b, f"{kind} {c.name} move {name}")
            km = m.process_points(c.x, c.y, c.z, c.frame)
            ko = o.process_points(c.x, c.y, c.z, c.frame)
            for a, b, name in zip(km, ko, OUTPUTS):
                assert_bits(a, b, f"{kind} {c.name} {name}")
            if kind == "device":
                assert_bits(m.get_layer("lowest"), o.get_layer("lowest"), f"{c.name} lowest")
            for mm in (m, o):
                mm.fuse_points(ko[0], c.R, c.G, c.B, c.I, ko[4], ko[1])
            _compare_feature(m, o, f"{kind} {c.name}")
            if c.name == "overflow":
                assert np.isnan(ko[1][c.overflow & (ko[0] >= 0)]).sum() > 50
        finally:
            m.close()
            o.close()


def test_shim_cloud_longer_than_one_launch(shim):  # noqa: F811
    """2^20 + 77 points into a 40 x 40 map: every cell the second launch reaches also has records from the first, and
    the points either side of the launch boundary share one cell.  The oracle runs each launch as its own call, the
    definition of a long call."""
    L, res = 40, 0.1
    n = LAUNCH + 77
    rng = np.random.default_rng(77)
    # the gem_golden sensor axes: every point keeps y <= -1.6 in the sensor frame, so the box filter passes it
    x = rng.uniform(-1.95, 1.95, n).astype(f32)
    y = rng.uniform(-5.95, -2.05, n).astype(f32)
    z = rng.normal(0.4, 0.3, n).astype(f32)
    x[LAUNCH - 40:LAUNCH + 40] = f32(0.53)             # one cell on both sides of the boundary
    y[LAUNCH - 40:LAUNCH + 40] = f32(-3.27)
    z[LAUNCH - 40:LAUNCH + 40] = np.linspace(1.5, -1.5, 80).astype(f32)   # lowest moves in the second launch
    R, G, B = (rng.integers(0, 256, n).astype(np.int32) for _ in range(3))
    inten = rng.uniform(0.0, 40.0, n).astype(f32)
    T = np.eye(4)
    T[:3, 3] = (0.0, 4.0, 0.0)
    f = gem_b200.make_frame(T, gem_b200.LaserSensorProcessor(ignore_points_above=3.0, ignore_points_below=-3.0))
    s = shim(L, res)
    o = OracleMap(L, res, compat_box_filter=True)
    try:
        for a, b in zip(s.move([0.0, 0.0, 0.5]), o.move([0.0, 0.0, 0.5])):
            assert_bits(a, b, "move")
        ks = s.process_points(x, y, z, f)
        outs = [o.process_points(x[a:a + LAUNCH], y[a:a + LAUNCH], z[a:a + LAUNCH], f) for a in range(0, n, LAUNCH)]
        ko = [np.concatenate(v) for v in zip(*outs)]
        for a, b, name in zip(ks, ko, OUTPUTS):
            assert_bits(a, b, name)
        key = ko[0]
        second = key[LAUNCH:][key[LAUNCH:] >= 0]
        assert np.isin(second, key[:LAUNCH]).all() and np.unique(second).size > 20 and (key >= 0).sum() > 0.9 * n
        s.fuse_points(key, R, G, B, inten, ko[4], ko[1])
        for a in range(0, n, LAUNCH):
            o.fuse_points(key[a:a + LAUNCH], R[a:a + LAUNCH], G[a:a + LAUNCH], B[a:a + LAUNCH], inten[a:a + LAUNCH],
                          ko[4][a:a + LAUNCH], ko[1][a:a + LAUNCH])
        fo = _compare_feature(s, o, "after Fuse")
        for m in (s, o):
            m.raytracing()
        _compare_feature(s, o, "after Raytracing")
        assert (fo["elevation"] != f32(-10)).sum() > 0.9 * L * L
    finally:
        o.close()


def test_shim_reinit_with_another_odd_length(shim):  # noqa: F811
    """Init_GPU_elevationmap again with a different, odd L, then a fresh stream: the same as a fresh oracle map.  The
    stream starts with a Move (the reference keeps the sensor height of the previous map until one)."""
    scene = synth.make_scene()
    frames = []
    for k in range(2):
        fr = synth.hdl64_frame(k, scene=scene, compat_axes=True, speed=8.0)
        frames.append((fr, np.ascontiguousarray(fr["xyzi"][k::9]), np.ascontiguousarray(fr["rgba"][k::9])))
    s = shim(96, 0.2)
    for fr, xyzi, rgba in frames[:1]:
        f = gem_b200.make_frame(fr["T"], gem_b200.LaserSensorProcessor())
        s.move(fr["position"])
        key, var, _, _, zt = s.process_points(xyzi[:, 0], xyzi[:, 1], xyzi[:, 2], f)
        s.fuse_points(key, rgba[:, 0], rgba[:, 1], rgba[:, 2], xyzi[:, 3], zt, var)
        s.raytracing()
    L, res = 77, 0.15
    s = shim(L, res)
    o = OracleMap(L, res, compat_box_filter=True)
    try:
        for k, (fr, xyzi, rgba) in enumerate(frames):
            f = gem_b200.make_frame(fr["T"], gem_b200.LaserSensorProcessor())
            for a, b in zip(s.move(fr["position"]), o.move(fr["position"])):
                assert_bits(a, b, f"frame {k} move")
            ks = s.process_points(xyzi[:, 0], xyzi[:, 1], xyzi[:, 2], f)
            ko = o.process_points(xyzi[:, 0], xyzi[:, 1], xyzi[:, 2], f)
            for a, b, name in zip(ks, ko, OUTPUTS):
                assert_bits(a, b, f"frame {k} {name}")
            for m in (s, o):
                m.fuse_points(ko[0], rgba[:, 0], rgba[:, 1], rgba[:, 2], xyzi[:, 3], ko[4], ko[1])
            fo = _compare_feature(s, o, f"frame {k}")
            for m in (s, o):
                m.raytracing()
            _compare_feature(s, o, f"frame {k} after Raytracing")
        assert (fo["elevation"] != f32(-10)).sum() > 300
    finally:
        o.close()
