"""The VoxelGrid pre-filter (pcl_ros's VoxelGrid nodelet of GEM's demo launches, DESIGN.md f9) byte for byte against the
oracle, tests/orc_voxel_grid.c: output bytes and every info field on the crafted cases of tests/voxel_cases.py, raw
HDL-64 frames under filter.launch and the three-call filter_kitti.launch chain, a raw D435 frame, random clouds of 1 M and
4 M points, a capacity below the count and the size query, scratch growth, every error path, the map left unchanged, a
tiled handle, the C++ facade program, and raw frames filtered into gem_add_points_stream over a scrolling sequence
against the oracle's filter and map."""
import ctypes as C
import subprocess

import numpy as np
import pytest
import torch

import gem_b200
import native
import voxel_cases as vc
import voxel_oracle
from gem_b200 import _lib, synth
from helpers import assert_layers_equal
from oracle_lib import OracleMap

pytestmark = pytest.mark.gpu
LAYERS = ("elevation", "variance", "intensity", "color_r", "color_g", "color_b", "traver", "lowest")
SENTINEL = -12345.5


@pytest.fixture(scope="module")
def emap():
    return gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1, 4)).to("cuda:0")


def same(got, want, what):
    (go, gi), (wo, wi) = got, want
    assert gi == wi, (what, gi, wi)
    g = go.cpu().numpy()
    assert g.shape == wo.shape, (what, g.shape, wo.shape)
    if g.tobytes() != wo.tobytes():
        bad = np.flatnonzero((g.view(np.uint32) != wo.view(np.uint32)).any(axis=1))
        raise AssertionError((what, "rows differ", int(bad.size), "first", int(bad[0]), g[bad[0]], wo[bad[0]]))


def check(g, p, leaf, field=None, limits=vc.ALL, negative=False, what=""):
    got = g.voxel_grid(dev(p), leaf, field, limits, negative)
    same(got, voxel_oracle.voxel_grid(p, leaf, field, limits, negative), what)
    return got


@pytest.mark.parametrize("name", vc.case_names())
def test_crafted(emap, name):
    _, p, leaf, field, limits, neg = vc.case_by_name(name)
    check(emap, p, leaf, field, limits, neg, name)


@pytest.mark.parametrize("frame", [0, 5, 11])
def test_hdl64_filter_launch_and_kitti_chain(emap, frame):
    """raw HDL-64 frames: filter.launch (one call), and filter_kitti.launch's three calls alternating between two
    buffers, every intermediate compared"""
    raw = synth.hdl64_frame(frame)["xyzi"]
    leaf, field, limits, neg = voxel_oracle.FILTER_LAUNCH[0]
    _, info = check(emap, raw, leaf, field, limits, neg, ("filter.launch", frame))
    assert 0 < info["count"] < info["used"] < raw.shape[0]
    bufs = [torch.empty((raw.shape[0], 4), dtype=torch.float32, device="cuda:0") for _ in range(2)]
    cur, want = dev(raw), raw
    for k, (leaf, field, limits, neg) in enumerate(voxel_oracle.FILTER_KITTI_LAUNCH):
        got = emap.voxel_grid(cur, leaf, field, limits, neg, out=bufs[k % 2])
        ref = voxel_oracle.voxel_grid(want, leaf, field, limits, neg)
        same(got, ref, ("kitti", frame, k))
        cur, want = got[0], ref[0]
    assert want.shape[0] > 1000


def test_d435_raw_frame(emap):
    fr = synth.d435_frame(0)
    raw = fr["xyzi"]
    assert np.isnan(raw[:, 2]).sum() > 100
    for leaf, field, limits in ((0.05, None, vc.ALL), (0.02, "z", (0.2, 3.25)), (0.1, "x", (-10.0, 10.0))):
        _, info = check(emap, raw, leaf, field, limits, False, ("d435", leaf))
        assert 0 < info["count"] < info["used"] < raw.shape[0]


@pytest.mark.parametrize("n,leaf,extent", [(1 << 20, 0.5, 50.0), (4 << 20, 0.1, 50.0), (4 << 20, 2.0, 50.0)])
def test_random_clouds(emap, n, leaf, extent):
    rng = np.random.default_rng(n + int(leaf * 10))
    p = vc._cloud(rng, n, -extent, extent)
    _, info = check(emap, p, leaf, what=(n, leaf))
    assert info["passthrough"] == 0 and info["count"] > 0


def test_capacity_below_count_and_size_query(emap):
    rng = np.random.default_rng(4)
    p = vc._cloud(rng, 50000, -3.0, 3.0)
    full, info = voxel_oracle.voxel_grid(p, 0.2)
    for cap in (0, 1, 10, info["count"] - 1, info["count"]):
        out = torch.full((cap + 7, 4), SENTINEL, dtype=torch.float32, device="cuda:0")
        view, ginfo = emap.voxel_grid(dev(p), 0.2, out=out[:cap])
        assert ginfo == info, (cap, ginfo, info)
        assert view.shape[0] == min(cap, info["count"])
        host = out.cpu().numpy()
        assert host[:cap].tobytes() == full[:cap].tobytes(), cap
        assert (host[cap:] == SENTINEL).all(), cap
    # the pass-through copies min(n, capacity) input points
    _, t, leaf, field, limits, neg = vc.case_by_name("passthrough_tiny_leaf")
    out = torch.full((20, 4), SENTINEL, dtype=torch.float32, device="cuda:0")
    _, ginfo = emap.voxel_grid(dev(t), leaf, field, limits, neg, out=out[:13])
    host = out.cpu().numpy()
    assert ginfo["passthrough"] == 1 and ginfo["count"] == t.shape[0]
    assert host[:13].tobytes() == t[:13].tobytes() and (host[13:] == SENTINEL).all()


def test_scratch_growth_small_large_small():
    g = gem_b200.ElevationMap(32, 0.1, compat_box_filter=False)
    rng = np.random.default_rng(8)
    for n in (1000, 3 << 20, 1000, 200000):
        check(g, vc._cloud(rng, n, -20.0, 20.0), 0.25, what=("growth", n))
    g.close()


def test_errors_write_nothing(emap):
    lib, h = emap._lib, emap.handle
    rng = np.random.default_rng(5)
    buf = dev(np.concatenate([vc._cloud(rng, 100, -1.0, 1.0), np.full((60, 4), SENTINEL, np.float32)]))
    inp, out = buf[:100], buf[100:]
    base = buf.clone()
    pin, pout = C.c_void_p(inp.data_ptr()), C.c_void_p(out.data_ptr())
    P = _lib.GemVoxelGridParams

    def params(leaf=(0.1, 0.1, 0.1), field=-1):
        return P((C.c_float * 3)(*leaf), field, -1.0, 1.0, 0)

    good = params()
    calls = []
    for bad_leaf in ((0.0, 0.1, 0.1), (0.1, -0.1, 0.1), (0.1, 0.1, float("nan")), (float("inf"), 0.1, 0.1), (-0.0, 0.1, 0.1)):
        calls.append(("leaf", bad_leaf, lambda q=params(bad_leaf): (inp, 100, q, pout, 60)))
    for f in (-2, 4, 100):
        calls.append(("field", f, lambda q=params(field=f): (pin, 100, q, pout, 60)))
    calls += [("n < 0", None, lambda: (pin, -1, good, pout, 60)),
              ("NULL points", None, lambda: (None, 100, good, pout, 60)),
              ("capacity < 0", None, lambda: (pin, 100, good, pout, -1)),
              ("NULL out", None, lambda: (pin, 100, good, None, 60)),
              ("overlap: same", None, lambda: (pin, 100, good, pin, 60)),
              ("overlap: tail", None, lambda: (pin, 100, good, C.c_void_p(inp.data_ptr() + 99 * 16), 60)),
              ("overlap: head", None, lambda: (C.c_void_p(inp.data_ptr() + 16 * 5), 95, good, C.c_void_p(inp.data_ptr()), 6))]
    for what, arg, make in calls:
        a = make()
        args = (C.c_void_p(a[0].data_ptr()) if isinstance(a[0], torch.Tensor) else a[0],) + a[1:]
        info = _lib.GemVoxelGridInfo(-7, -7, -7)
        assert lib.gem_voxel_grid(h, args[0], args[1], C.byref(args[2]), args[3], args[4], C.byref(info)) == 1, (what, arg)
        assert (info.count, info.used, info.passthrough) == (-7, -7, -7), (what, arg)
        emap.sync()
        assert torch.equal(buf, base), (what, arg)
    assert lib.gem_voxel_grid(h, pin, 100, None, pout, 60, C.byref(_lib.GemVoxelGridInfo())) == 1
    assert lib.gem_voxel_grid(h, pin, 100, C.byref(good), pout, 60, None) == 1
    emap.sync()
    assert torch.equal(buf, base)
    # adjacent ranges do not overlap; n = 0 is valid and writes nothing
    info = _lib.GemVoxelGridInfo(-7, -7, -7)
    assert lib.gem_voxel_grid(h, pin, 100, C.byref(good), pout, 60, C.byref(info)) == 0
    assert lib.gem_voxel_grid(h, None, 0, C.byref(good), pout, 60, C.byref(info)) == 0
    assert (info.count, info.used, info.passthrough) == (0, 0, 0)
    with pytest.raises(ValueError):
        emap.voxel_grid(inp.double(), 0.1)
    with pytest.raises(ValueError):
        emap.voxel_grid(inp, 0.1, field="w")


def test_map_unchanged():
    """a map with a deferred fold outstanding: the filter reads and writes only its own buffers"""
    g = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False)
    fr = synth.hdl64_frame(2)
    f = gem_b200.make_frame(fr["T"], gem_b200.LaserSensorProcessor())
    g.move(fr["position"])
    g.add(fr["xyzi"], fr["rgba"], f)
    x, r = dev(fr["xyzi"]), torch.from_numpy(fr["rgba"]).cuda()
    torch.cuda.synchronize()
    g.add_stream_fast(C.c_void_p(x.data_ptr()), C.c_void_p(r.data_ptr()), x.shape[0], C.byref(f))
    o = OracleMap(200, 0.1, compat_box_filter=False)
    o.move(fr["position"])
    o.add(fr["xyzi"], fr["rgba"], f)
    o.add(fr["xyzi"], fr["rgba"], f)
    check(g, fr["xyzi"], 0.1, "x", (-10.0, 10.0), False, "with a fold pending")
    assert_layers_equal(g, o, what="after the filter")        # the deferred fold lands once, as without the filter
    g2 = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False)
    g2.move(fr["position"])
    g2.add(fr["xyzi"], fr["rgba"], f)
    g2.compute_features()
    before = {k: g2.get_layer(k) for k in LAYERS}
    exported = g2.export_layers()
    check(g2, fr["xyzi"], 0.2, what="after features")
    for k in LAYERS:
        assert before[k].tobytes() == g2.get_layer(k).tobytes(), k
    again = g2.export_layers()
    for k, v in exported.items():
        assert np.asarray(v).tobytes() == np.asarray(again[k]).tobytes(), k


def test_tiled_handle():
    t = gem_b200.ElevationMap(64, 0.1, tile=(0, 32, 0, 64))
    raw = synth.hdl64_frame(1)["xyzi"]
    check(t, raw, 0.1, "x", (-10.0, 10.0), False, "tiled")
    check(t, raw, (0.2, 0.3, 0.1), None, vc.ALL, False, "tiled anisotropic")


def test_filtered_stream_composition():
    """filter.launch in front of the node: raw frames through voxel_grid into gem_add_points_stream over a scrolling
    sequence, a constant non-zero colour so that the intensity layer takes the centroids' intensities; three output
    buffers in rotation, so that each stays untouched until two further add calls are complete.  Every layer equals the
    oracle's filter followed by OracleMap.add"""
    L, res = 300, 0.1
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False)
    o = OracleMap(L, res, compat_box_filter=False)
    leaf, field, limits, neg = voxel_oracle.FILTER_LAUNCH[0]
    frames = [synth.hdl64_frame(k, scene=scene) for k in range(10)]
    nmax = max(fr["xyzi"].shape[0] for fr in frames)
    bufs = [torch.empty((nmax, 4), dtype=torch.float32, device="cuda:0") for _ in range(3)]
    colour = np.tile(np.array([[90, 140, 200, 255]], np.uint8), (nmax, 1))
    rgba = torch.from_numpy(colour).cuda()
    keep = []
    for k, fr in enumerate(frames):
        f = gem_b200.make_frame(fr["T"], gem_b200.LaserSensorProcessor())
        keep.append(f)
        g.move(fr["position"])
        o.move(fr["position"])
        raw = dev(fr["xyzi"])
        out, info = g.voxel_grid(raw, leaf, field, limits, neg, out=bufs[k % 3])
        want, winfo = voxel_oracle.voxel_grid(fr["xyzi"], leaf, field, limits, neg)
        assert info == winfo and info["count"] > 1000, (k, info, winfo)
        g.add_stream_fast(C.c_void_p(out.data_ptr()), C.c_void_p(rgba.data_ptr()), info["count"], C.byref(f))
        o.add(want, colour[:winfo["count"]], f)
        if k % 4 == 3:
            g.raytracing()
            o.raytracing()
    g.flush()
    g.sync()
    assert_layers_equal(g, o, what="filtered stream")
    assert (o.get_layer("intensity") != 0).sum() > 1000


def test_facade_voxel_grid_program_runs():
    exe = native.facade_program("voxel_grid_smoke")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "voxel grid ok" in r.stdout, r.stdout + r.stderr
