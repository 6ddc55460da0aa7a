"""The costmap topics and the footprint clearing on the device (DESIGN.md f17), byte for byte against the encoder of
tests/costmap_pub_oracle.py: W9 / W10 / W11 into device and pinned memory at every 16-byte phase with guard bytes, grids
holding all 256 costs, rectangles of every shape; a subscriber's replica of GEM's local costmap (footprint cleared at
changing yaws) and global costmap (inflated) through 12 moves, against the oracle chain; the refusals, which write
nothing and keep the publisher; and the C++ facade program."""
import ctypes as C
import math
import subprocess

import numpy as np
import pytest
import torch

import costmap_cases as cc
import costmap_oracle
import costmap_pub_oracle as cp
import inflation_oracle as O
import native
import rosmsg_oracle as ro
import gem_b200
from gem_b200 import _lib, costmap, synth
from gem_b200.elevation_map import RosHeader

pytestmark = pytest.mark.gpu
GUARD = 0xA5
SIZES = [(1, 1), (1, 37), (41, 1), (75, 75), (257, 33), (1000, 1000)]


@pytest.fixture(scope="module")
def emap():
    return gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)


def grid_with_all_costs(sx, sy, seed):
    g = np.random.default_rng(seed).integers(0, 256, sx * sy, dtype=np.uint8)
    g[:min(256, g.size)] = np.random.default_rng(seed + 1).permutation(256)[:min(256, g.size)].astype(np.uint8)
    return g.reshape(sy, sx)


def buffer(nbytes, pinned):
    if pinned:
        b = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
        b.fill_(GUARD)
        return b
    return torch.full((nbytes,), GUARD, dtype=torch.uint8, device="cuda:0")


def publish_at(emap, pub, header, window, master, offset, pinned, force_full=False):
    """publish into a buffer at byte `offset` with guard bytes before and after; returns (kind, message bytes)"""
    n = emap._ros_size("q", lambda p, c, nb: emap._lib.gem_ros_costmap(emap._h, C.byref(header.c()), C.byref(emap._cost_window(window)),
                                                                      emap._cost_grid(master, window[3], window[4], "q"),
                                                                      C.byref(pub.state), 1 if force_full else 0, p, c, nb,
                                                                      C.byref(C.c_int())))
    buf = buffer(offset + n + 40, pinned)
    kind, msg = emap.ros_costmap(header, window, master, pub.state, force_full, buf[offset:offset + n + 1])
    host = buf.cpu().numpy()
    assert (host[:offset] == GUARD).all() and (host[offset + n:] == GUARD).all(), "a byte outside the message was written"
    assert msg.numel() == n
    return kind, host[offset:offset + n].tobytes()


@pytest.mark.parametrize("size", SIZES)
def test_full_and_update_bytes(emap, size):
    sx, sy = size
    g = grid_with_all_costs(sx, sy, sx * 3 + sy)
    master = torch.from_numpy(g.copy()).to("cuda:0")
    window = (-3.3 + 0.1 * sx, 1.7, 0.05, sx, sy)
    rects = {(0, 0, sx, sy), (0, 0, 1, 1), (sx - 1, sy - 1, 1, 1), (0, sy // 2, sx, 1), (sx // 3, 0, sx - sx // 3, sy),
             (0, 0, sx, 0), (min(5, sx - 1), min(2, sy), min(17, sx - min(5, sx - 1)), sy - min(2, sy)),
             (min(1, sx - 1), 0, max(1, min(33, sx - 1)), min(3, sy))}
    offsets = range(16) if sx * sy < 10**5 else (0, 1, 7, 15)
    for fl in (0, 3, 20, 300) if sx * sy < 10**5 else (0, 300):
        fid = ("map/" * 80)[:fl]
        h = RosHeader(seq=fl, stamp_sec=11, stamp_nsec=12, frame_id=fid)
        hb = ro.header(fl, 11, 12, fid.encode())
        want_full = cp.occupancy_grid(hb, window, g)
        for pinned in (False, True):
            for off in offsets:
                pub = costmap.CostmapPublisher()
                assert publish_at(emap, pub, h, window, master, off, pinned) == ("full", want_full)
                for x, y, w, hh in sorted(rects):
                    pub.bounds(x, x + w, y, y + hh)
                    kind, got = publish_at(emap, pub, h, window, master, off, pinned)
                    if w == 0:
                        assert (kind, got) == ("none", b"")
                    else:
                        assert kind == "update" and got == cp.grid_update(hb, x, y, w, hh, g), (x, y, w, hh, off, pinned)


@pytest.mark.parametrize("pinned", [False, True])
def test_footprint_message_bytes(emap, pinned):
    for fl in (0, 7, 300):
        fid = ("base/" * 80)[:fl]
        h = RosHeader(seq=2, stamp_sec=3, stamp_nsec=4, frame_id=fid)
        for fp in (cp.GEM_FOOTPRINT, [], [(0.1 * k, math.cos(k)) for k in range(33)]):
            for pose in ((0.0, 0.0, 0.0), (12.5, -3.25, 2.9), (-40.0, 7.0, -1.0)):
                want = cp.polygon_stamped(ro.header(2, 3, 4, fid.encode()), cp.transform(fp, *pose))
                for off in range(16):
                    buf = buffer(off + len(want) + 24, pinned)
                    got = emap.ros_footprint(h, fp, *pose, out=buf[off:])
                    host = buf.cpu().numpy()
                    assert got.numel() == len(want) and host[off:off + len(want)].tobytes() == want
                    assert (host[:off] == GUARD).all() and (host[off + len(want):] == GUARD).all()


def test_footprint_clearing_matches_the_oracles(emap):
    rng = np.random.default_rng(4)
    window = (-7.45, -7.45, 0.2, 75, 75)
    for k in range(48):
        yaw = 2 * math.pi * k / 48
        rx, ry = float(rng.uniform(-0.1, 0.1)), float(rng.uniform(-0.1, 0.1))
        g0 = rng.integers(0, 256, (75, 75), dtype=np.uint8)
        layer = torch.from_numpy(g0.copy()).to("cuda:0")
        mk = emap.costmap_footprint(window, cp.GEM_FOOTPRINT, rx, ry, yaw, layer)
        emap.sync()
        verts, cells = cp.orc_footprint_cells(window, cp.GEM_FOOTPRINT, rx, ry, yaw)
        want = g0.copy()
        for x, y in cells:
            want[y, x] = cc.FREE
        assert np.array_equal(layer.cpu().numpy(), want), k
        assert mk["marked"] == len(cells) and mk["lethal"] == 0
        b = cp.touch_bounds(verts)
        assert np.array([mk["min_x"], mk["min_y"], mk["max_x"], mk["max_y"]]).tobytes() == np.array(b).tobytes()
    # a vertex outside the window fills nothing but still widens the bounds
    g0 = np.full((75, 75), 200, np.uint8)
    layer = torch.from_numpy(g0.copy()).to("cuda:0")
    mk = emap.costmap_footprint(window, cp.GEM_FOOTPRINT, 7.3, 0.0, 0.0, layer)
    emap.sync()
    assert mk["marked"] == 0 and mk["max_x"] > 7.5 and torch.equal(layer.cpu(), torch.from_numpy(g0))


def test_subscriber_replica_follows_the_robot():
    """test_costmap_gpu's 12 moves: the local costmap ("max", the footprint cleared at changing yaws) and the global one
    ("overwrite", inflated), bounds fed and published after every update as Costmap2DROS does; each replica equals T of
    the master, the kinds equal the restatement's, and the grids equal the oracle chain"""
    L, res = 200, 0.05
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    lm = costmap.Costmap(g, 75, 75, 0.2, fill=cc.FREE)
    ll = costmap.Costmap(g, 75, 75, 0.2, fill=cc.FREE)
    gm = costmap.Costmap(g, 1000, 1000, 0.2, -100.0, -100.0, fill=cc.FREE)
    gl = costmap.Costmap(g, 1000, 1000, 0.2, -100.0, -100.0, fill=cc.UNKNOWN)
    ginf = costmap.InflationLayer(0.55, 10.0, costmap.inscribed_radius(costmap.GEM_FOOTPRINT))
    oracle = {id(c): [c.window, c.grid.cpu().numpy()] for c in (lm, ll, gm, gl)}
    inf_state = [True, None]
    pubs = {id(lm): (costmap.CostmapPublisher(), cp.Publisher(), cp.Replica()),
            id(gm): (costmap.CostmapPublisher(), cp.Publisher(), cp.Replica())}
    stale = {id(lm): None, id(gm): None}
    history = np.zeros((0, 8), np.float32)
    pos = np.array([0.1, 0.2, 1.7], np.float32)
    rng = np.random.default_rng(5)
    h = RosHeader(frame_id="odom")
    kinds = []

    def oracle_update(master, layer, robot, yaw, mode, mark, inf):
        for c in (master, layer):
            w, gr = oracle[id(c)]
            sx_m, sy_m = c.size_in_meters()
            oracle[id(c)] = list(costmap_oracle.update_origin(w, robot[0] - sx_m / 2, robot[1] - sy_m / 2, c.fill, gr))
        lw, lg = oracle[id(layer)]
        lg, marks = mark(lw, lg)
        b = [min(1e30, marks["min_x"]), min(1e30, marks["min_y"]), max(-1e30, marks["max_x"]), max(-1e30, marks["max_y"])]
        if yaw is not None:
            verts, cells = cp.orc_footprint_cells(lw, cp.GEM_FOOTPRINT, robot[0], robot[1], yaw)
            for x, y in cells or []:
                lg[y, x] = cc.FREE
            fb = cp.touch_bounds(verts)
            b = [min(b[0], fb[0]), min(b[1], fb[1]), max(b[2], fb[2]), max(b[3], fb[3])]
        oracle[id(layer)][1] = lg
        if inf:
            if inf_state[0]:
                inf_state[0], inf_state[1] = False, tuple(b)
                b = (-costmap.FLT_MAX, -costmap.FLT_MAX, costmap.FLT_MAX, costmap.FLT_MAX)
            else:
                last, inf_state[1] = inf_state[1], tuple(b)
                r = ginf.params["inflation_radius"]
                b = (min(last[0], b[0]) - r, min(last[1], b[1]) - r, max(last[2], b[2]) + r, max(last[3], b[3]) + r)
        mw, mg = oracle[id(master)]
        rect = costmap.update_rect(mw, dict(zip(("min_x", "min_y", "max_x", "max_y"), b)))
        if rect is not None:
            x0, y0, xn, yn = rect
            mg = mg.copy()
            mg[y0:yn, x0:xn] = master.fill
            mg = costmap_oracle.combine(mode, lg, mg, mw[3], mw[4], rect)
            if inf:
                mg = O.inflate(mg, mw[2], ginf.params, rect)
            oracle[id(master)][1] = mg
        return rect

    def feed_and_publish(master, rect, k):
        mine, py, rep = pubs[id(master)]
        if rect is not None:
            stale[id(master)] = (rect[0], rect[2], rect[1], rect[3])
            assert (master.bx0, master.bxn, master.by0, master.byn) == stale[id(master)] and master.initialized
        if stale[id(master)] is not None:                 # getBounds: the last rect, also after an early return
            mine.update_bounds(master)
            py.bounds(*stale[id(master)])
        if k % 5 == 3:                                    # no subscriber at this cycle: nothing is published
            return
        kind, msg = mine.publish(master, h, out=torch.empty(2 << 20, dtype=torch.uint8, pin_memory=True) if k % 2 else None)
        assert (kind, ) == (py.publish(master.window)[0], )
        rep.apply(kind, msg.cpu().numpy().tobytes())
        kinds.append(kind)
        assert np.array_equal(rep.grid, cp.TABLE[master.grid.cpu().numpy()]), (k, kind)

    for k in range(12):
        fr = synth.hdl64_frame(k % 8, scene=scene)
        g.snapshot_shown() if k else None
        step = rng.uniform(0.2, 0.9, 2).astype(np.float32)
        pos = pos + np.array([step[0], step[1], 0.0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        centre, _, shift = g.move(pos)
        if k:
            harvested, n = g.harvest_scrolled_out(centre, shift)
            history = np.concatenate([history, harvested[:n]])
        g.add(fr["xyzi"], fr["rgba"], gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
        g.compute_features()
        robot = (float(pos[0]), float(pos[1]))
        tr = np.array(g.export_layers()["traver"])
        c_now, s_now, _ = g.state()
        cloud = torch.cat([torch.from_numpy(history).to("cuda:0").reshape(-1, 8), g.export_grid_cloud("shown")]).contiguous()
        host_cloud = cloud.cpu().numpy()
        for sub in range(2):       # a move (the windows roll: full grids), then the robot turning in place (updates)
            yaw = 0.37 * k - 1.0 + 0.45 * sub
            rect, _ = lm.update(ll, robot, "max", lambda l: l.mark_map(0.7), robot_yaw=yaw, footprint=costmap.GEM_FOOTPRINT)
            want = oracle_update(lm, ll, robot, yaw, 0,
                                 lambda w, gr: costmap_oracle.mark_map(tr, L, res, c_now, s_now, w, gr, 0.7), False)
            assert rect == want, (k, rect, want)
            rect_g, _ = gm.update(gl, robot, "overwrite", lambda l: l.mark_points(cloud, 0.7), inflation=ginf)
            want = oracle_update(gm, gl, robot, None, 1, lambda w, gr: costmap_oracle.mark_points(host_cloud, w, gr, 0.7), True)
            assert rect_g == want, (k, rect_g, want)
            g.sync()
            for c in (lm, ll, gm, gl):
                assert np.array_equal(c.grid.cpu().numpy(), oracle[id(c)][1]), ("grid", k, sub)
            feed_and_publish(lm, rect, 2 * k + sub)
            feed_and_publish(gm, rect_g, 2 * k + sub)
        g.raytracing()
    assert kinds.count("full") >= 10 and kinds.count("update") >= 5, kinds
    with pytest.raises(ValueError):
        gm.update(gl, (0.0, 0.0), "overwrite", lambda l: l.mark_points(cloud, 0.7), robot_yaw=0.0, footprint=costmap.GEM_FOOTPRINT)


def test_without_footprint_the_update_is_unchanged():
    g = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)
    pts = torch.from_numpy(cc.records(np.array([[0.5, 0.5], [1.5, -0.3], [-2.0, 1.0]]), np.array([0.1, 0.9, 0.2]))).to("cuda:0")
    a = [costmap.Costmap(g, 75, 75, 0.2, fill=cc.FREE) for _ in range(2)]
    b = [costmap.Costmap(g, 75, 75, 0.2, fill=cc.FREE) for _ in range(2)]
    ra = a[0].update(a[1], (0.3, 0.2), "max", lambda l: l.mark_points(pts.reshape(-1, 8), 0.7))
    rb = b[0].update(b[1], (0.3, 0.2), "max", lambda l: l.mark_points(pts.reshape(-1, 8), 0.7), robot_yaw=None, footprint=None)
    g.sync()
    assert ra == rb and torch.equal(a[0].grid, b[0].grid) and torch.equal(a[1].grid, b[1].grid)


def test_refusals_write_nothing_and_keep_the_publisher(emap):
    lib = emap._lib
    window = (0.0, 0.0, 0.2, 75, 75)
    master = torch.from_numpy(grid_with_all_costs(75, 75, 9)).to("cuda:0")
    pub = costmap.CostmapPublisher()
    assert emap.ros_costmap(RosHeader(), window, master, pub.state)[0] == "full"
    pub.bounds(2, 9, 3, 7)
    before = bytes(pub.state)
    out = torch.full((4096,), GUARD, dtype=torch.uint8, device="cuda:0")
    w = emap._cost_window(window)
    h = RosHeader(frame_id="map").c()
    nb, kind = C.c_longlong(-5), C.c_int(-5)
    P = C.c_void_p

    def call(hdr=C.byref(h), win=C.byref(w), m=P(master.data_ptr()), p=C.byref(pub.state), force=0, o=P(out.data_ptr()), cap=4096):
        return lib.gem_ros_costmap(emap._h, hdr, win, m, p, force, o, cap, C.byref(nb), C.byref(kind))

    pageable = np.zeros(4096, np.uint8)
    bad_window = _lib.GemCostmapWindow(0.0, 0.0, 0.0, 75, 75)
    cases = [dict(hdr=None), dict(win=None), dict(win=C.byref(bad_window)), dict(m=None), dict(p=None), dict(force=2),
             dict(o=P(pageable.ctypes.data)), dict(o=P(master.data_ptr() + 100)), dict(o=None, cap=10), dict(cap=-1),
             dict(hdr=C.byref(_lib.GemRosHeader(0, 0, 0, None)))]
    for kw in cases:
        assert call(**kw) == 1, kw
        assert nb.value == 0 and bytes(pub.state) == before, kw
    pub.bounds(0, 76, 0, 1)                                   # bounds outside the grid
    before = bytes(pub.state)
    assert call() == 1 and bytes(pub.state) == before
    torch.cuda.synchronize()
    assert (out.cpu().numpy() == GUARD).all() and (pageable == 0).all()
    # a size query and a too-small capacity change nothing either
    pub2 = costmap.CostmapPublisher()
    before = bytes(pub2.state)
    assert call(p=C.byref(pub2.state), o=None, cap=0) == 0 and nb.value == 96 + 75 * 75 + 0 * 0 + 3 and kind.value == 1
    assert call(p=C.byref(pub2.state), cap=100) == 0 and bytes(pub2.state) == before
    # footprint calls: n < 0, non-finite pose or spec values
    spec = (C.c_double * 8)(*[v for xy in cp.GEM_FOOTPRINT for v in xy])
    nan_spec = (C.c_double * 8)(*([float("nan")] + [0.0] * 7))
    mk = _lib.GemCostmapMarks()
    layer = torch.full((75, 75), 77, dtype=torch.uint8, device="cuda:0")
    for args in ((spec, -1, 0.0, 0.0, 0.0), (spec, 4, float("inf"), 0.0, 0.0), (spec, 4, 0.0, 0.0, float("nan")), (nan_spec, 4, 0.0, 0.0, 0.0),
                 (None, 4, 0.0, 0.0, 0.0)):
        assert lib.gem_costmap_footprint(emap._h, C.byref(w), *args, P(layer.data_ptr()), C.byref(mk)) == 1
        assert lib.gem_ros_footprint(emap._h, C.byref(h), *args, P(out.data_ptr()), 4096, C.byref(nb)) == 1 and nb.value == 0
    torch.cuda.synchronize()
    assert (layer.cpu().numpy() == 77).all() and (out.cpu().numpy() == GUARD).all()


def test_cxx_facade_program(emap, tmp_path):
    exe = native.facade_program("costmap_publish_smoke", tmp_path)
    r = subprocess.run([exe, str(tmp_path / "cxx")], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "costmap publish ok kinds=1,2,0,1" in r.stdout, r.stdout + r.stderr
    S = 75
    g = ((7 * np.arange(S * S) + 3) % 256).astype(np.uint8).reshape(S, S)
    master = torch.from_numpy(g).to("cuda:0")
    window = (-7.45, -7.45, 0.2, S, S)
    h = RosHeader(5, 6, 7, "odom")
    pub = costmap.CostmapPublisher()
    py = [emap.ros_costmap(h, window, master, pub.state)[1]]
    pub.bounds(3, 20, 4, 9)
    py.append(emap.ros_costmap(h, window, master, pub.state)[1])
    py.append(emap.ros_costmap(h, window, master, pub.state)[1])
    pub.bounds(0, 1, 0, 1)
    py.append(emap.ros_costmap(h, window, master, pub.state, force_full=True)[1])
    for k in range(4):
        assert (tmp_path / f"cxx.{k}.bin").read_bytes() == py[k].cpu().numpy().tobytes(), k
    assert (tmp_path / "cxx.footprint.bin").read_bytes() == emap.ros_footprint(h, cp.GEM_FOOTPRINT, 0.03, -0.02, 0.7).cpu().numpy().tobytes()
    layer = torch.zeros((S, S), dtype=torch.uint8, device="cuda:0")
    emap.costmap_footprint(window, cp.GEM_FOOTPRINT, 0.03, -0.02, 0.7, layer)
    emap.sync()
    assert (tmp_path / "cxx.layer.bin").read_bytes() == layer.cpu().numpy().tobytes()
