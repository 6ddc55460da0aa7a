"""The map topics as ROS messages on the device (DESIGN.md f15): every gem_ros_* call's bytes equal the struct oracle
(tests/rosmsg_oracle.py) built from the oracle map (orc_show / export_layers) and from the library's existing exports on
the same state, into device and pinned host memory at every base offset 0-15, for every map size and frame_id length of
tests/rosmsg_cases.py; guard bytes around the output stay untouched by every call and refusal; size queries equal the
written size; a c2-sized map with history_point over scrolled harvests; octrees; the SubMap; the C++ facade."""
import ctypes as C
import subprocess

import numpy as np
import pytest
import torch

import gem_b200
import native
import rosmsg_cases as rc
import rosmsg_oracle as ro
from gem_b200 import GemError, RosHeader, _lib, synth
from oracle_lib import OracleMap

pytestmark = pytest.mark.gpu
f32 = np.float32
GUARD = 64


def _pair(c):
    g = gem_b200.ElevationMap(c.L, c.res, compat_box_filter=False)
    o = OracleMap(c.L, c.res, compat_box_filter=False)
    for m in (g, o):
        c.apply(m)
    g.compute_features()
    return g, o


def _hb(h: RosHeader):
    return ro.header(h.seq, h.stamp_sec, h.stamp_nsec, h.frame_id.encode())


def _buffers(size):
    """(name, guarded buffer, offset) for device and pinned memory at every base offset"""
    for where in ("cuda", "pinned"):
        for off in rc.OFFSETS:
            n = size + off + 2 * GUARD
            buf = (torch.full((n,), 0xA5, dtype=torch.uint8, device="cuda:0") if where == "cuda"
                   else torch.full((n,), 0xA5, dtype=torch.uint8).pin_memory())
            yield where, buf, GUARD + off


def _check_into(call, want, what):
    """call(ptr, capacity, nb) into guarded device and pinned buffers at every offset: the bytes, the guards, the size
    query, and nothing written when the capacity is one short"""
    nb = C.c_longlong(-1)
    assert call(None, 0, C.byref(nb)) == 0 and nb.value == len(want), (what, nb.value, len(want))
    for where, buf, off in _buffers(len(want)):
        ptr = C.c_void_p(buf.data_ptr() + off)
        nb.value = -1
        assert call(ptr, len(want) - 1, C.byref(nb)) == 0 and nb.value == len(want)
        torch.cuda.synchronize()
        assert bool((buf == 0xA5).all()), (what, where, off, "one short")
        assert call(ptr, len(want), C.byref(nb)) == 0 and nb.value == len(want)
        torch.cuda.synchronize()
        got = buf.cpu().numpy().tobytes()
        assert got[:off] == b"\xa5" * off and got[off + len(want):] == b"\xa5" * (len(buf) - off - len(want)), (what, where, off)
        if got[off:off + len(want)] != want:
            k = next(i for i in range(len(want)) if got[off + i] != want[i])
            raise AssertionError((what, where, off, k, got[off + k:off + k + 16], want[k:k + 16]))


def _grid_call(g, h):
    hc = h.c()
    return lambda p, c, nb: g._lib.gem_ros_grid_map(g.handle, C.byref(hc), p, c, nb)


def _ortho_call(g, h):
    hc = h.c()
    return lambda p, c, nb: g._lib.gem_ros_orthomosaic(g.handle, C.byref(hc), p, c, nb)


def _visual_call(g, h):
    hc = h.c()
    return lambda p, c, nb: g._lib.gem_ros_visual_points(g.handle, C.byref(hc), p, c, nb)


@pytest.mark.parametrize("name", [c.name for c in rc.map_cases()])
def test_map_messages_match_oracle_and_exports(name):
    c = rc.case(name)
    g, o = _pair(c)
    res = float(f32(c.res))
    layers_o, layers_g = o.export_layers(), g.export_layers()
    img_o, xyz_o, rgb_o = o.show()
    centre, start, _ = o.state()
    gc, gs, _ = g.state()
    assert np.array_equal(gc.view(np.uint32), centre.view(np.uint32)) and np.array_equal(gs, start)
    fids = rc.FRAME_ID_LENGTHS if c.L <= 64 else [0, 7, 300]
    for fl in fids:
        h = RosHeader(seq=fl, stamp_sec=17, stamp_nsec=999999999, frame_id=rc.frame_id(fl))
        want = ro.grid_map(_hb(h), c.L, res, float(centre[0]), float(centre[1]), start, layers_o)
        assert want == ro.grid_map(_hb(h), c.L, res, float(gc[0]), float(gc[1]), gs, layers_g)   # the existing export
        if fl in (0, 5, 300) or c.L <= 5:
            _check_into(_grid_call(g, h), want, (name, "grid_map", fl))
        else:   # every frame_id length into device memory at offset 0
            assert g.ros_grid_map(h).cpu().numpy().tobytes() == want, (name, fl)
    h = RosHeader(frame_id="")
    want = ro.image(_hb(h), c.L, img_o.tobytes())
    assert want == ro.image(_hb(h), c.L, g.export_orthomosaic().tobytes())
    _check_into(_ortho_call(g, h), want, (name, "orthomosaic"))
    h = RosHeader(seq=3, stamp_sec=5, stamp_nsec=123000, frame_id="map")
    want = ro.visual_points(_hb(h), xyz_o, rgb_o)
    xyz_g, rgb_g, _ = g.export_visual_points()
    assert want == ro.visual_points(_hb(h), xyz_g, rgb_g)
    _check_into(_visual_call(g, h), want, (name, "visual_points"))
    # the calls change nothing
    after = g.export_layers()
    for n in ro.GRID_LAYERS:
        assert after[n].tobytes() == layers_g[n].tobytes()


def _part(p, where):
    if where == "numpy":
        return p
    t = torch.from_numpy(p.view(f32).copy())
    return t.to("cuda:0") if where == "cuda" else (t.pin_memory() if where == "pinned" else t)


@pytest.mark.parametrize("name", sorted(rc.cloud_parts()))
def test_cloud_matches_oracle(name):
    g = gem_b200.ElevationMap(16, 0.1, compat_box_filter=False)
    parts = rc.cloud_parts()[name]
    rec = np.concatenate(parts) if parts else np.zeros((0, 8), np.uint32)
    for where in ("cuda", "pinned", "pageable", "numpy"):
        ps = [_part(p, where) for p in parts]
        for dense in (True, False):
            h = RosHeader(frame_id=rc.frame_id(11))
            want = ro.ict_cloud(_hb(h), rec, dense)
            arr, keep = g._ros_parts(ps)
            hc = h.c()
            call = lambda p, c, nb: g._lib.gem_ros_cloud(g.handle, C.byref(hc), arr, len(keep), int(dense), p, c, nb)
            _check_into(call, want, (name, where, dense))
            assert g.ros_cloud(h, ps, is_dense=dense).cpu().numpy().tobytes() == want


def test_octomap_messages():
    g = gem_b200.ElevationMap(32, 0.1, compat_box_filter=False)
    h = RosHeader(frame_id="map")
    hc = h.c()
    call = lambda p, c, nb: g._lib.gem_ros_octomap(g.handle, C.byref(hc), p, c, nb)
    nb = C.c_longlong(-1)
    assert call(None, 0, C.byref(nb)) == 1 and nb.value == 0      # no octree yet
    with pytest.raises(GemError):
        g.ros_octomap(h)
    empty = torch.zeros((0, 8), dtype=torch.float32, device="cuda:0")
    stream, _ = g.color_octree(empty, 0.2)
    _check_into(call, ro.octomap(_hb(h), 0.2, b""), "empty octree")
    rng = np.random.default_rng(5)
    pts = np.zeros((20000, 8), f32)
    pts[:, :3] = rng.uniform(-30, 30, (20000, 3))
    pts[:, 3] = 1.0
    pts[:, 4] = rng.integers(0, 1 << 24, 20000).astype(np.uint32).view(f32)
    stream, info = g.color_octree(torch.from_numpy(pts).to("cuda:0"), 0.05)
    assert info["bytes"] > 100000
    want = ro.octomap(_hb(h), 0.05, stream.cpu().numpy().tobytes())
    _check_into(call, want, "deep octree")
    assert g.ros_octomap(h).cpu().numpy().tobytes() == want


def test_c2_map_history_point_and_submap():
    res, L = 0.05, 1024
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    pos = np.array((0.3, -0.2, 1.7), np.float32)
    harvested = []
    for k in range(6):
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([1.5, 0.4, 0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        centre, _, shift = g.move(pos)
        if k > 0:
            rec, n = g.harvest_to_local_map(centre, shift, records=True)
            harvested.append(np.ascontiguousarray(rec))
        g.add(fr["xyzi"], fr["rgba"], gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
        g.compute_features()
        g.snapshot_shown()
    grid = g.export_grid_cloud("shown")
    visual = np.concatenate(harvested)
    assert visual.shape[0] > 10 and grid.shape[0] > 1000
    h = RosHeader(frame_id="map")
    want = ro.ict_cloud(_hb(h), np.concatenate([visual.view(np.uint32), grid.cpu().numpy().view(np.uint32)]))
    assert g.ros_cloud(h, [visual, grid]).cpu().numpy().tobytes() == want           # visualCloud_ + grid cloud
    pinned = torch.empty(len(want) + 9, dtype=torch.uint8).pin_memory()
    assert g.ros_cloud(h, [visual, grid], out=pinned[9:]).numpy().tobytes() == want
    layers = g.export_layers()
    c, s, _ = g.state()
    gm = ro.grid_map(_hb(h), L, res, float(c[0]), float(c[1]), s, layers)
    assert len(gm) == ro.size_grid_map(3, L) and g.ros_grid_map(h).cpu().numpy().tobytes() == gm
    # the SubMap of the keyframe cut
    kf = bytes(range(256)) * 3 + b"\x07"
    pose = (1.0, 2.0, 3.0, 0.0, 0.0, 0.0, 1.0)
    sub = g.ros_submap(grid, kf, pose, h)
    want = ro.submap(ro.ict_cloud(_hb(h), grid.cpu().numpy()), kf, ro.image(ro.header(), L, g.export_orthomosaic().tobytes()), pose)
    assert sub.cpu().numpy().tobytes() == want
    d = ro.decode_submap(want, len(kf))
    assert d["pose"] == pose and d["keyframePC"] == kf


def test_refusals_write_nothing():
    g = gem_b200.ElevationMap(8, 0.1, compat_box_filter=False)
    lib, hd = _lib.load(), g.handle
    buf = torch.full((4096,), 0xA5, dtype=torch.uint8, device="cuda:0")
    o = C.c_void_p(buf.data_ptr() + 5)
    h = RosHeader(frame_id="map").c()
    bad = _lib.GemRosHeader(0, 0, 0, None)
    nb = C.c_longlong(-1)
    rec = torch.zeros((4, 8), dtype=torch.float32, device="cuda:0")
    part = (_lib.GemRosPart * 1)(_lib.GemRosPart(rec.data_ptr(), 4))
    neg = (_lib.GemRosPart * 1)(_lib.GemRosPart(rec.data_ptr(), -1))
    null = (_lib.GemRosPart * 1)(_lib.GemRosPart(None, 3))
    big = (_lib.GemRosPart * 2)(_lib.GemRosPart(rec.data_ptr(), 1 << 26), _lib.GemRosPart(rec.data_ptr(), 1 << 26))
    overlap = (_lib.GemRosPart * 1)(_lib.GemRosPart(buf.data_ptr() + 100, 4))
    calls = [
        lambda: lib.gem_ros_grid_map(hd, None, o, 4000, C.byref(nb)),
        lambda: lib.gem_ros_grid_map(hd, C.byref(bad), o, 4000, C.byref(nb)),
        lambda: lib.gem_ros_grid_map(hd, C.byref(h), None, 4000, C.byref(nb)),
        lambda: lib.gem_ros_grid_map(hd, C.byref(h), o, -1, C.byref(nb)),
        lambda: lib.gem_ros_orthomosaic(hd, C.byref(bad), o, 4000, C.byref(nb)),
        lambda: lib.gem_ros_visual_points(hd, None, o, 4000, C.byref(nb)),
        lambda: lib.gem_ros_cloud(hd, C.byref(h), part, -1, 1, o, 4000, C.byref(nb)),
        lambda: lib.gem_ros_cloud(hd, C.byref(h), neg, 1, 1, o, 4000, C.byref(nb)),
        lambda: lib.gem_ros_cloud(hd, C.byref(h), null, 1, 1, o, 4000, C.byref(nb)),
        lambda: lib.gem_ros_cloud(hd, C.byref(h), big, 2, 1, o, 4000, C.byref(nb)),
        lambda: lib.gem_ros_cloud(hd, C.byref(h), overlap, 1, 1, o, 4000, C.byref(nb)),
        lambda: lib.gem_ros_octomap(hd, C.byref(h), o, 4000, C.byref(nb)),
    ]
    for i, call in enumerate(calls):
        nb.value = -1
        assert call() == 1 and nb.value == 0, i
        torch.cuda.synchronize()
        assert bool((buf == 0xA5).all()), i
    # pageable host memory as the output (the device cannot store to it)
    page = np.full(4096, 0xA5, np.uint8)
    po = C.c_void_p(page.ctypes.data + 3)
    for i, call in enumerate([lambda: lib.gem_ros_grid_map(hd, C.byref(h), po, 4000, C.byref(nb)),
                              lambda: lib.gem_ros_orthomosaic(hd, C.byref(h), po, 4000, C.byref(nb)),
                              lambda: lib.gem_ros_visual_points(hd, C.byref(h), po, 4000, C.byref(nb)),
                              lambda: lib.gem_ros_cloud(hd, C.byref(h), part, 1, 1, po, 4000, C.byref(nb))]):
        nb.value = -1
        assert call() == 1 and nb.value == 0, ("pageable", i)
        assert b"pageable" in lib.gem_last_error(hd)
    torch.cuda.synchronize()
    assert (page == 0xA5).all()
    # a tiled handle
    t = gem_b200.ElevationMap(8, 0.1, compat_box_filter=False, tile=(0, 4, 0, 8))
    for fn in (lib.gem_ros_grid_map, lib.gem_ros_orthomosaic, lib.gem_ros_visual_points, lib.gem_ros_octomap):
        nb.value = -1
        assert fn(t.handle, C.byref(h), o, 4000, C.byref(nb)) == 1 and nb.value == 0
    assert lib.gem_ros_cloud(t.handle, C.byref(h), part, 1, 1, o, 4000, C.byref(nb)) == 1 and nb.value == 0
    torch.cuda.synchronize()
    assert bool((buf == 0xA5).all())
    with pytest.raises(ValueError):
        g.ros_grid_map(RosHeader(), out=torch.empty(10, dtype=torch.uint8, device="cuda:0"))


def test_facade_rosmsg_program(tmp_path):
    exe = native.facade_program("rosmsg_smoke", tmp_path)
    c = rc.case("L33_opt_move")

    class Recorder:   # the layers the case sets, for the program
        def move(self, p):
            pass

        def opt_move(self, p, dz):
            pass

        def set_layer(self, name, a):
            (tmp_path / f"layer.{name}.bin").write_bytes(np.ascontiguousarray(a).astype(np.int32 if name.startswith("color") else f32).tobytes())

    c.apply(Recorder())
    rec = rc.records(100, 8)
    (tmp_path / "rec.bin").write_bytes(rec.tobytes())
    r = subprocess.run([exe, str(tmp_path / "rec.bin"), str(tmp_path / "cxx"), str(tmp_path)], capture_output=True, text=True,
                       timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "rosmsg ok" in r.stdout, r.stdout + r.stderr
    # the same calls from Python on the same state (the program builds it with the same moves and layers)
    g = gem_b200.ElevationMap(c.L, c.res, compat_box_filter=False)
    c.apply(g)
    g.compute_features()
    h = RosHeader(seq=1, stamp_sec=2, stamp_nsec=3, frame_id="map")
    cxx = {k: (tmp_path / f"cxx.{k}.bin").read_bytes() for k in ("grid_map", "orthomosaic", "visual_points", "cloud", "submap")}
    assert cxx["grid_map"] == g.ros_grid_map(h).cpu().numpy().tobytes()
    assert cxx["orthomosaic"] == g.ros_orthomosaic(RosHeader()).cpu().numpy().tobytes()
    assert cxx["visual_points"] == g.ros_visual_points(h).cpu().numpy().tobytes()
    assert cxx["cloud"] == g.ros_cloud(h, [rec]).cpu().numpy().tobytes()
    pose = (1.0, 2.0, 3.0, 0.0, 0.0, 0.0, 1.0)
    assert cxx["submap"] == g.ros_submap(rec, b"keyframe", pose, h).cpu().numpy().tobytes()
