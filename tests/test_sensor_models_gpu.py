"""Stereo and perfect sensor models on the device against the CPU oracle (tests/orc_sensor_models.c + orc_fuse), bit for
bit: gem_process_points on the raw organised 640x480 D435 frame (NaNs left in) and on crafted points, every add path
(device, pipelined stream with scrolls, pinned host_async, PCL records, a call chunked past max_points, one multi-cloud
call mixing all four models, the tiled step at world 1), features and ray clean-up after them, fused against unfused,
one frame of each of the twelve shipped sensor configs, the C++ smoke program and the argument checks."""
import ctypes as C
import math
import subprocess
import tempfile

import numpy as np
import pytest

import gem_b200
import oracle_lib
import sensor_models_oracle as smo
import test_sensor_models_cpu as cpu
import test_tiled_step_gpu as tts
from gem_b200 import synth
from gem_b200._lib import GemError, GemFrame, check

pytestmark = pytest.mark.gpu

LAYERS = ["elevation", "variance", "intensity", "color_r", "color_g", "color_b", "lowest"]
L, RES = 512, 0.02  # the c3 shape (a D435 frame into 512^2 at 0.02 m)
_D435 = {}


def stereo(width=640):
    return gem_b200.StereoSensorProcessor(**cpu.ASLAM, cloud_width=width)


MODELS = {"stereo": stereo, "perfect": gem_b200.PerfectSensorProcessor}


def d435(k):
    if k not in _D435:
        _D435[k] = synth.d435_frame(k)  # raw: 640 x 480, NaN where there is no return
    return _D435[k]


def frame(T, sensor, **kw):
    return gem_b200.make_frame(T, sensor, **kw)


def rot_kw():
    return dict(rotation_variance=np.diag([1e-4, 2e-4, 3e-4]), B_r_BS_skew=np.array([[0, -0.3, 0.1], [0.3, 0, -0.2], [-0.1, 0.2, 0]]))


def assert_layers(g, o, where):
    for name in LAYERS:
        d = tts._diff(g.get_layer(name), o.get_layer(name))
        assert d is None, f"{where}: layer {name}: {d}"


def assert_bits(a, b, where):
    d = tts._diff(a, b)
    assert d is None, f"{where}: {d}"


def pair(compat_box_filter=False, max_points=0, length=L, res=RES):
    return (gem_b200.ElevationMap(length, res, compat_box_filter=compat_box_filter, max_points=max_points),
            oracle_lib.OracleMap(length, res, compat_box_filter=compat_box_filter))


@pytest.mark.parametrize("rot", [False, True])
@pytest.mark.parametrize("model", ["stereo", "perfect"])
@pytest.mark.parametrize("cloud", ["d435", "crafted"])
def test_process_points_bit_exact(cloud, model, rot):
    if cloud == "d435":
        fr = d435(0)
        pts, T, sensor = fr["xyzi"][:, :3], fr["T"], MODELS[model]()
    else:
        pts, T, sensor = cpu.crafted_points(), np.eye(4), MODELS[model]()
        T[2, 3] = 0.5
    f = frame(T, sensor, **(rot_kw() if rot else {}))
    P = 200_000  # the D435 frame runs in two chunks, the crafted cloud (640k points) in four
    g, o = pair(max_points=P)
    dev = g.process_points(pts[:, 0], pts[:, 1], pts[:, 2], f)
    ref = oracle_process_chunked(o, pts, f, P)
    for name, a, b in zip(("key", "var", "x_ts", "y_ts", "z_ts"), dev, ref):
        assert_bits(a, b, f"{cloud}/{model}/rot={rot}: {name}")
    assert (dev[0] >= 0).sum() > 1000
    assert_bits(g.get_layer("lowest"), o.get_layer("lowest"), "lowest")


def oracle_process_chunked(o, pts, f, P):
    """a call longer than max_points P runs as one call per chunk (own `lowest` update), the stereo index counting on
    across chunks"""
    outs = [smo.process_points(o, pts[a:a + P, 0], pts[a:a + P, 1], pts[a:a + P, 2], f, idx0=a)
            for a in range(0, pts.shape[0], P)]
    return [np.concatenate(v) for v in zip(*outs)]


def oracle_add_chunked(o, xyzi, rgba, f, P):
    for a in range(0, xyzi.shape[0], P):
        smo.add(o, xyzi[a:a + P], rgba[a:a + P], f, idx0=a)


def _dev(xyzi, rgba, keep):
    import torch
    x = torch.from_numpy(np.ascontiguousarray(xyzi, np.float32)).cuda()
    r = None if rgba is None else torch.from_numpy(np.ascontiguousarray(rgba, np.uint8)).cuda()
    keep.append((x, r))
    return x, r


def _move_both(g, o, pos):
    g.move(pos)
    o.move(pos)


@pytest.mark.parametrize("model", ["stereo", "perfect"])
@pytest.mark.parametrize("path", ["add", "stream", "host_async", "pcl", "chunked"])
def test_add_paths_match_oracle(path, model):
    import torch
    P = 70_000
    g, o = pair(max_points=P if path == "chunked" else 0)
    keep = []
    for k in range(3):
        fr = d435(k)
        xyzi, rgba, T, pos = fr["xyzi"], fr["rgba"], fr["T"], fr["position"]
        f = frame(T, MODELS[model](), base_z=float(pos[2]))
        _move_both(g, o, [pos[0] + 0.3 * k, pos[1] - 0.2 * k, pos[2]])  # scrolls between frames
        if path in ("add", "chunked"):
            x, r = _dev(xyzi, rgba, keep)
            g.add(x, r, f)
        elif path == "stream":
            x, r = _dev(xyzi, rgba, keep)
            check(g._lib.gem_add_points_stream(g.handle, C.c_void_p(x.data_ptr()), C.c_void_p(r.data_ptr()), xyzi.shape[0],
                                               C.byref(f)), g.handle, "gem_add_points_stream")
        elif path == "host_async":
            x = torch.from_numpy(np.ascontiguousarray(xyzi)).pin_memory()
            r = torch.from_numpy(np.ascontiguousarray(rgba)).pin_memory()
            keep.append((x, r))
            check(g._lib.gem_add_points_host_async(g.handle, C.c_void_p(x.data_ptr()), C.c_void_p(r.data_ptr()), xyzi.shape[0],
                                                   C.byref(f)), g.handle, "gem_add_points_host_async")
        else:
            rec = np.zeros((xyzi.shape[0], 8), np.float32)
            rec[:, :3] = xyzi[:, :3]
            bgra = np.stack([rgba[:, 2], rgba[:, 1], rgba[:, 0], rgba[:, 3]], 1).astype(np.uint8)
            rec[:, 4] = np.ascontiguousarray(bgra).view(np.float32)[:, 0]
            rec[:, 6] = xyzi[:, 3]
            g.add_pcl(rec, f)
        if path == "chunked":
            oracle_add_chunked(o, xyzi, rgba, f, P)
        else:
            smo.add(o, xyzi, rgba, f)
    g.sync()
    assert_layers(g, o, f"{path}/{model}")
    g.compute_features()
    o.compute_features()
    g.raytracing()
    o.raytracing()
    assert_layers(g, o, f"{path}/{model} after features + ray clean-up")
    assert_bits(g.get_layer("traver"), o.get_layer("traver"), f"{path}/{model}: traver")


def test_multi_mixes_all_four_models():
    """laser, structured light, stereo and perfect segments in one gem_add_points_multi call.  The segments' clouds land
    in disjoint cells (sensor poses 8 m apart, depths cut to 3 m by NaN so that indices are kept), so the oracle's
    sequence of single-cloud adds equals the call, whose `lowest` is one update over all segments."""
    import torch
    g, o = pair(length=512, res=0.05)
    sensors = [gem_b200.LaserSensorProcessor(ignore_points_above=math.inf, ignore_points_below=-math.inf),
               gem_b200.StructuredLightSensorProcessor(), stereo(), gem_b200.PerfectSensorProcessor()]
    fr = d435(1)
    clouds, frames_, rgbas = [], [], []
    for s, sensor in enumerate(sensors):
        xyzi = fr["xyzi"][s::2].copy()  # every other pixel: indices within each segment's own cloud
        xyzi[~(xyzi[:, 2] <= 3.0), :3] = np.nan
        T = fr["T"].copy()
        T[1, 3] = -12.0 + 8.0 * s
        clouds.append(xyzi)
        rgbas.append(fr["rgba"][s::2])
        frames_.append(frame(T, sensor))
    offsets = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])])
    x = torch.from_numpy(np.concatenate(clouds)).cuda()
    r = torch.from_numpy(np.concatenate(rgbas)).cuda()
    g.add_multi(x, r, offsets, frames_)
    for c, rg, f in zip(clouds, rgbas, frames_):
        smo.add(o, c, rg, f)
    g.sync()
    assert_layers(g, o, "multi")


def test_tiled_step_world1_alternating_models():
    """gem_tiled_step at world 1 (k_route_peer_any and k_route_peer in turn: the step graph is rebuilt when the kind of
    model changes) against the oracle's sequence of adds"""
    cap = tts.CAP
    bufs = tts.PeerBuffers(1, cap)
    g = tts._tile_map(256, 0, 1, cap)
    o = oracle_lib.OracleMap(256, tts.RES, compat_box_filter=False)
    keep = []
    sensors = [stereo(320), gem_b200.LaserSensorProcessor(), gem_b200.PerfectSensorProcessor(), stereo(320), stereo(0)]
    bufs.attach(g, 0)
    for k, sensor in enumerate(sensors):
        fr = d435(k)
        xyzi, rgba = fr["xyzi"][::2], fr["rgba"][::2]  # 153600 > cap: the first cap points
        xyzi, rgba = xyzi[:cap], rgba[:cap]
        if isinstance(sensor, gem_b200.LaserSensorProcessor):
            xyzi = xyzi[np.isfinite(xyzi).all(1)]  # the laser oracle removes non-finite points: keep the indices equal
            rgba = fr["rgba"][::2][:cap][np.isfinite(fr["xyzi"][::2][:cap]).all(1)]
        f = frame(fr["T"], sensor)
        x, r = _dev(xyzi, rgba, keep)
        g.tiled_step(x, r, f)
        smo.add(o, xyzi, rgba, f)
    g.flush()
    g.sync()
    tts._assert_tile(g, o, 0, 1, "tiled world 1")


@pytest.mark.parametrize("model", ["stereo", "perfect"])
def test_fused_equals_unfused(model):
    fr = d435(2)
    xyzi, rgba = fr["xyzi"], fr["rgba"]
    f = frame(fr["T"], MODELS[model](), **rot_kw())
    a = gem_b200.ElevationMap(L, RES, compat_box_filter=False)
    b = gem_b200.ElevationMap(L, RES, compat_box_filter=False)
    a.add(xyzi, rgba, f)
    key, var, _, _, zt = b.process_points(xyzi[:, 0], xyzi[:, 1], xyzi[:, 2], f)
    b.fuse_points(key, rgba[:, 0], rgba[:, 1], rgba[:, 2], xyzi[:, 3], zt, var)
    for name in LAYERS:
        assert_bits(a.get_layer(name), b.get_layer(name), name)


def test_each_shipped_config_end_to_end():
    fr = d435(0)
    for name, sensor in cpu.shipped_models().items():
        if isinstance(sensor, gem_b200.StereoSensorProcessor):
            sensor.cloud_width = 640
        f = frame(fr["T"], sensor, base_z=float(fr["position"][2]))
        g, o = pair()
        g.add(fr["xyzi"], fr["rgba"], f)
        smo.add(o, fr["xyzi"], fr["rgba"], f)
        assert_layers(g, o, name)
        assert (g.get_layer("elevation") != -10).sum() > 100, name


def test_cxx_smoke_runs():
    with tempfile.TemporaryDirectory() as d:
        exe = cpu.compile_sensor_models_smoke(d)
        r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "sensor models ok" in r.stdout, r.stdout + r.stderr[-2000:]


def test_invalid_models_are_refused_and_write_nothing():
    import torch
    g = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)
    fr = d435(0)
    x = torch.from_numpy(fr["xyzi"][:1000]).cuda()
    before = {n: g.get_layer(n) for n in LAYERS}
    for t, w in ((4, 0), (-1, 0), (2, -1), (3, -5)):
        f = frame(np.eye(4), stereo())
        f.sensor.type, f.sensor.cloud_width = t, w
        calls = [lambda: g.add(x, None, f), lambda: g.add(fr["xyzi"][:1000], None, f),
                 lambda: g.process_points(fr["xyzi"][:10, 0], fr["xyzi"][:10, 1], fr["xyzi"][:10, 2], f),
                 lambda: g.add_multi(x, None, [0, 1000], [f]),
                 lambda: g.add_pcl(np.zeros((10, 8), np.float32), f)]
        for call in calls:
            with pytest.raises(GemError, match="GEM_ERR_INVALID"):
                call()
        for fn in ("gem_add_points_stream", "gem_add_points_host_async"):
            assert getattr(g._lib, fn)(g.handle, C.c_void_p(x.data_ptr()), None, 1000, C.byref(f)) == 1
    g.sync()
    for n in LAYERS:
        assert_bits(g.get_layer(n), before[n], n)
