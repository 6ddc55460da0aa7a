"""The costmap plugins fed from their messages on the H100 (DESIGN.md f18): gem_costmap_mark_grid against the oracle
(tests/orc_gridmsg.c) on the crafted messages with the layer at all 16 byte phases and guard bytes around the layer and
the costmap; the visual_map round trip (gem_ros_grid_map -> parse -> mark_grid equals gem_costmap_mark_map of the shown
map, scrolled and after gem_opt_move); the history_point round trip (gem_ros_cloud -> decode_pointcloud2_records gives
the records back) and the f12 crafted layouts against orc_pc2_decode; the two layer classes through Costmap.update with
inflation and a CostmapPublisher against a host model of the plugins over the oracle; refusals; the C++ facade."""
import ctypes as C
import subprocess

import numpy as np
import pytest
import torch

import costmap_cases as cc
import costmap_oracle
import gridmsg_oracle as gm
import native
import pc2_cases as pc
import pc2_oracle
import rosmsg_cases as rc
import gem_b200
from gem_b200 import GemError, PointCloud2Layout, _lib, costmap, synth
from gem_b200.elevation_map import RosHeader

pytestmark = pytest.mark.gpu
GUARD = 0xA5
ICT = [("x", 0, 7, 1), ("y", 4, 7, 1), ("z", 8, 7, 1), ("rgb", 16, 7, 1), ("intensity", 24, 7, 1), ("covariance", 20, 7, 1),
       ("travers", 28, 7, 1)]


@pytest.fixture(scope="module")
def emap():
    """the smallest handle: the mark and decode calls read no map"""
    return gem_b200.ElevationMap(1, 0.1, compat_box_filter=False)


def guarded(nbytes, phase, fill=GUARD):
    """(big, view): view is nbytes at `phase` past a 256-byte aligned allocation, with 64 guard bytes on either side"""
    big = torch.full((nbytes + phase + 128,), fill, dtype=torch.uint8, device="cuda:0")
    return big, big[64 + phase:64 + phase + nbytes]


def lib_layer(d):
    """a descriptor dict as the library's gem_grid_map_layer"""
    return _lib.GemGridMapLayer.from_buffer_copy(gm.layer_struct(d))


def same_marks(got, want, what):
    assert got["marked"] == want["marked"] and got["lethal"] == want["lethal"], (what, got, want)
    for k in ("min_x", "min_y", "max_x", "max_y"):
        assert np.float64(got[k]).tobytes() == np.float64(want[k]).tobytes(), (what, k, got[k], want[k])


def windows(d):
    lx, ly = d["length_x"], d["length_y"]
    cx, cy = d["position_x"], d["position_y"]
    return [(cx - 0.5 * lx - 0.3, cy - 0.5 * ly - 0.3, 0.2, int(lx / 0.2) + 4, int(ly / 0.2) + 4),
            (cx - 0.5 * lx + 0.77 * d["resolution"], cy - 0.5 * ly + 0.31 * d["resolution"], 0.5 * d["resolution"],
             2 * d["size_x"] + 1, d["size_y"] + 3)]


@pytest.mark.parametrize("name", sorted(c[0] for c in gm.cases()))
def test_mark_grid_crafted_at_every_phase(emap, name):
    _, msg, layer = next(c for c in gm.cases() if c[0] == name)
    d = gm.parse(msg, layer)
    g = lib_layer(d)
    v = gm.layer_floats(msg, d)
    rng = np.random.default_rng(len(msg))
    arr = np.frombuffer(msg, np.uint8)
    for phase in range(16):
        mbig, mview = guarded(len(msg), (phase - d["offset"]) % 16)      # the layer's first float at `phase` mod 16
        mview.copy_(torch.from_numpy(arr.copy()))
        assert (mview.data_ptr() + d["offset"]) % 16 == phase
        for w in windows(d):
            g0 = cc.random_grid(rng, w)
            want, wm = gm.orc_mark_grid(d, v, w, g0, 0.7, phase % 2 == 0)
            cbig, grid = guarded(w[3] * w[4], 3)
            grid.copy_(torch.from_numpy(g0.reshape(-1)))
            m = emap.costmap_mark_grid(g, mview, w, grid, 0.7, phase % 2 == 0, offset=d["offset"])
            assert np.array_equal(grid.cpu().numpy(), want.reshape(-1)), (name, phase, w)
            same_marks(m, wm, (name, phase))
            c = cbig.cpu().numpy()
            assert (c[:67] == GUARD).all() and (c[67 + grid.numel():] == GUARD).all()
        mb = mbig.cpu().numpy()
        assert (mb[:64 + (mview.data_ptr() - mbig.data_ptr() - 64)] == GUARD).all()
        assert (mb[mview.data_ptr() - mbig.data_ptr() + len(msg):] == GUARD).all()


@pytest.fixture(scope="module")
def moving_map():
    """a 256^2 map at 0.05 m driven over six frames so that its start index is far from 0"""
    L, res = 256, 0.05
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    pos = np.array([0.3, -0.2, 1.7], np.float32)
    for k in range(6):
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([0.9, 0.7, 0.0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        g.move(pos)
        g.add(fr["xyzi"], fr["rgba"], gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
        g.compute_features()
        g.raytracing()
    g.compute_features()
    return g, pos


def round_trip(g, what, need_marks=True):
    centre, start, _ = g.state()
    c = (float(centre[0]), float(centre[1]))
    pinned = torch.empty(g.length ** 2 * 36 + 4096, dtype=torch.uint8).pin_memory()
    msg = g.ros_grid_map(RosHeader(3, 4, 5, "odom"), out=pinned)
    d = g.grid_map_msg_parse(msg, "traver")
    dev_msg = msg.to("cuda:0")
    assert (d.start_x, d.start_y) == (int(start[0]), int(start[1])), what
    for w in [(c[0] - 7.45, c[1] - 7.45, 0.2, 75, 75), (c[0] - 100.0, c[1] - 100.0, 0.2, 1000, 1000),
              (c[0] - 3.0, c[1] - 2.0, 0.05, 101, 77)]:
        for mu in (False, True):
            g0 = cc.random_grid(np.random.default_rng(5), w)
            a, b = torch.from_numpy(g0).cuda(), torch.from_numpy(g0).cuda()
            ma = g.costmap_mark_map(w, a, 0.7, "shown", mu)
            mb = g.costmap_mark_grid(d, dev_msg, w, b, 0.7, mu, offset=d.offset)
            assert torch.equal(a, b), (what, w, mu)
            same_marks(mb, ma, (what, w, mu))
            assert ma["marked"] > 0 or not need_marks


@pytest.mark.parametrize("name", [c.name for c in rc.map_cases()])
def test_visual_map_round_trip_map_cases(name):
    """the map cases of the f15 message tests: sizes 1-257, scrolled starts, the frame after opt_move, crafted -10 / NaN /
    -0 elevations"""
    c = rc.case(name)
    g = gem_b200.ElevationMap(c.L, c.res, compat_box_filter=False)
    c.apply(g)
    g.compute_features()
    round_trip(g, name, need_marks=False)


@pytest.mark.parametrize("shape", [(200, 0.1), (1024, 0.05), (512, 0.02)], ids=["c1", "c2", "c3"])
def test_visual_map_round_trip_config_shapes(shape):
    L, res = shape
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    scene = synth.make_scene()
    pos = np.array((0.3, -0.2, 1.7), np.float32)
    for k in range(4):
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([0.4, 0.1, 0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        g.move(pos)
        g.add(fr["xyzi"], fr["rgba"], gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
        g.compute_features()
    round_trip(g, f"L{L}")


def test_visual_map_round_trip(moving_map):
    g, pos = moving_map
    assert all(int(s) != 0 for s in g.state()[1])
    round_trip(g, "scrolled")
    g.opt_move((float(pos[0]) + 0.37, float(pos[1]) - 0.21), 0.05)
    g.compute_features()
    round_trip(g, "after opt_move")


def cloud_data(msg, n, fl):
    """the data field of a W5 message: its uint32 count, then 32 n bytes, then is_dense"""
    at = 164 + fl
    assert int(np.frombuffer(msg[at - 4:at].cpu().numpy().tobytes(), np.uint32)[0]) == 32 * n
    return msg[at:at + 32 * n]


def test_history_point_round_trip(emap, moving_map):
    g, _ = moving_map
    recs = g.export_grid_cloud("shown")
    n = int(recs.shape[0])
    assert n > 1000
    special = recs[:5].clone()
    words = lambda *v: torch.from_numpy(np.array(v, np.uint32).view(np.int32)).cuda()   # noqa: E731
    special.view(torch.int32)[:, 3] = words(0x7fc00001, 0x80000000, 0x7f800000, 0xff800000, 0x12345678)  # NaN payloads, -0
    special.view(torch.int32)[:, 7] = words(0x7fa00000, 0x80000000, 1, 2, 3)
    for parts in ([recs], [special, recs[:777]]):
        want = torch.cat(parts)
        msg = g.ros_cloud(RosHeader(1, 2, 3, "map"), parts)
        data = cloud_data(msg, want.shape[0], 3)
        lay = PointCloud2Layout(ICT, want.shape[0], 1, 32)
        for shift in (0, 5):
            big, view = guarded(data.numel(), shift)
            view.copy_(data)
            out = emap.decode_pointcloud2_records(lay, view)
            emap.sync()
            assert torch.equal(out.view(torch.int32), want.view(torch.int32)), shift


def records_round_trip(emap, g, parts, what):
    want = torch.cat([p if isinstance(p, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in parts])
    msg = g.ros_cloud(RosHeader(1, 2, 3, "map"), parts)
    data = cloud_data(msg, want.shape[0], 3)
    out = emap.decode_pointcloud2_records(PointCloud2Layout(ICT, want.shape[0], 1, 32), data)
    emap.sync()
    assert torch.equal(out.view(torch.int32), want.view(torch.int32)), what


def test_history_point_round_trip_harvests_and_global_map(emap):
    """visualCloud_ (the harvested records of every scrolled frame) and the global map's submap stack, as the node
    publishes them in history_point / global_point"""
    L, res = 256, 0.05
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    g.global_map_reset()
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
        if k % 2 == 1:
            g.global_map_push(g.export_grid_cloud("shown"), T.astype(np.float32))
    visual = np.concatenate(harvested)
    assert visual.shape[0] > 10
    records_round_trip(emap, g, [visual], "harvests")
    records_round_trip(emap, g, [visual, g.export_grid_cloud("shown")], "visualCloud_ + grid cloud")
    torch.cuda.synchronize()                     # the stack's copies run on its own stream
    stack = g.global_map_records()
    assert stack.shape[0] > 1000
    records_round_trip(emap, g, [stack.contiguous()], "global map stack")


@pytest.mark.parametrize("name", pc.case_names())
def test_records_match_the_oracle_on_crafted_layouts(emap, name):
    case = pc.case_by_name(name)
    lay = PointCloud2Layout(case["fields"], case["width"], case["height"], case["point_step"], case["row_step"], case["is_bigendian"])
    n = case["width"] * case["height"]
    want = pc2_oracle.decode(case)
    nb = case.get("data_bytes", case["data"].nbytes)
    for shift in (0, 1, 6, 13):
        big, data = guarded(case["data"].nbytes, shift)
        data.copy_(torch.from_numpy(np.ascontiguousarray(case["data"]).reshape(-1).view(np.uint8)))
        obig = torch.full((max(n, 1) * 32 + 64,), GUARD, dtype=torch.uint8, device="cuda:0")
        out = obig[16:16 + max(n, 1) * 32].view(torch.float32).view(-1, 8)
        if case["refused"]:
            assert want is None
            with pytest.raises(GemError):
                emap.decode_pointcloud2_records(lay, data, out, data_bytes=nb)
            assert (obig.cpu().numpy() == GUARD).all()
            continue
        emap.decode_pointcloud2_records(lay, data, out, data_bytes=nb)
        emap.sync()
        o = obig.cpu().numpy()
        assert np.array_equal(o[16:16 + 32 * n].reshape(-1, 32), want[0]), (name, shift)
        assert (o[:16] == GUARD).all() and (o[16 + 32 * n:] == GUARD).all()


def test_refusals_write_nothing(emap):
    msg = gm.cases()[0][1]
    with pytest.raises(GemError):
        emap.grid_map_msg_parse(msg[:-1])
    with pytest.raises(GemError):
        emap.grid_map_msg_parse(msg, "missing")
    d = gm.parse(msg)
    w = (0.0, 0.0, 0.1, 10, 10)
    grid = torch.full((10, 10), 77, dtype=torch.uint8, device="cuda:0")
    data = torch.from_numpy(np.frombuffer(msg, np.uint8).copy()).cuda()
    lib, P = _lib.load(), C.c_void_p
    mk = _lib.GemCostmapMarks()
    cw = _lib.GemCostmapWindow(*w)
    for bad in (dict(d, resolution=0.0), dict(d, floats=d["floats"] + 1), dict(d, column_major=0), dict(d, size_x=-1)):
        g = lib_layer(bad)
        assert lib.gem_costmap_mark_grid(emap._h, C.byref(g), P(data.data_ptr() + d["offset"]), C.byref(cw), 0.7, 1,
                                         P(grid.data_ptr()), C.byref(mk)) == 1
    g = lib_layer(d)
    bad_w = _lib.GemCostmapWindow(0.0, 0.0, -0.1, 10, 10)
    assert lib.gem_costmap_mark_grid(emap._h, C.byref(g), P(data.data_ptr()), C.byref(bad_w), 0.7, 1, P(grid.data_ptr()), C.byref(mk)) == 1
    assert lib.gem_costmap_mark_grid(emap._h, C.byref(g), None, C.byref(cw), 0.7, 1, P(grid.data_ptr()), C.byref(mk)) == 1
    case = pc.case_by_name(pc.case_names()[0])
    lay = PointCloud2Layout(case["fields"], case["width"], case["height"], case["point_step"], case["row_step"])
    dd = torch.from_numpy(np.ascontiguousarray(case["data"]).reshape(-1).view(np.uint8)).cuda()
    out = torch.zeros(lay.points * 8 + 8, dtype=torch.float32, device="cuda:0")
    assert lib.gem_decode_pointcloud2_records(emap._h, C.byref(lay.c), P(dd.data_ptr()), dd.numel(), P(out.data_ptr() + 4)) == 1
    torch.cuda.synchronize()
    assert (grid.cpu().numpy() == 77).all() and (out.cpu().numpy() == 0).all()


def test_point_layer_refusal_keeps_the_stored_cloud(emap):
    """a refused history_point (short data, a field past point_step) after a valid one, larger than the stored cloud:
    the layer keeps the valid cloud and re-marks the same grid and marks"""
    rng = np.random.default_rng(3)
    rec = np.zeros((300, 8), np.float32)
    rec[:, 0:2] = rng.uniform(-2.0, 2.0, (300, 2))
    rec[:, 7] = rng.uniform(0.0, 1.0, 300)
    pl = costmap.PointMapLayer(emap, 0.5)
    layer = costmap.Costmap(emap, 50, 50, 0.1, -2.5, -2.5, fill=cc.UNKNOWN)
    pl.on_message(PointCloud2Layout(ICT, 300, 1, 32), rec.tobytes())
    m0 = pl(layer)
    g0 = layer.grid.clone()
    big = np.zeros((100000, 8), np.float32).tobytes()
    bad_field = [("x", 0, 7, 1), ("y", 4, 7, 1), ("travers", 30, 7, 1)]
    for lay, data, nb in ((PointCloud2Layout(ICT, 100000, 1, 32), big, len(big) - 1),
                          (PointCloud2Layout(bad_field, 100000, 1, 32), big, None),
                          (PointCloud2Layout(ICT, 100000, 1, 32), torch.from_numpy(np.frombuffer(big, np.uint8).copy()).cuda(),
                           len(big) - 32)):
        with pytest.raises(GemError):
            pl.on_message(lay, data, data_bytes=nb)
        assert pl.n == 300
        layer.grid.fill_(cc.UNKNOWN)
        same_marks(pl(layer), m0, "after a refusal")
        assert torch.equal(layer.grid, g0)


def test_layers_on_another_handle_and_host_staging():
    """the layer objects on one handle and the costmaps on another, host clouds staged by the layer while other
    allocations churn: the same grids as the oracle"""
    a = gem_b200.ElevationMap(1, 0.1, compat_box_filter=False)
    b = gem_b200.ElevationMap(1, 0.1, compat_box_filter=False)
    rng = np.random.default_rng(9)
    pl = costmap.PointMapLayer(a, 0.5)
    el = costmap.ElevationMapLayer(a, 0.5)
    layer = costmap.Costmap(b, 200, 150, 0.05, -5.0, -4.0, fill=cc.UNKNOWN)
    msg = next(c for c in gm.cases() if c[0] == "rect_tall")[1]
    d = gm.parse(msg)
    for k in range(6):
        n = 200000 + 1000 * k
        rec = np.zeros((n, 8), np.float32)
        rec[:, 0] = rng.uniform(-5.0, 5.0, n)
        rec[:, 1] = rng.uniform(-4.0, 3.5, n)
        rec[:, 7] = rng.uniform(0.0, 1.0, n)
        pl.on_message(PointCloud2Layout(ICT, n, 1, 32), rec.tobytes())
        junk = [torch.full((n * 8,), float(j), device="cuda:0") for j in range(4)]   # reuse of freed blocks
        g0 = layer.grid.cpu().numpy()
        m = pl(layer)
        want, wm = costmap_oracle.mark_points(rec, layer.window, g0, 0.5)
        assert np.array_equal(layer.grid.cpu().numpy().reshape(-1), np.asarray(want, np.uint8).reshape(-1)), k
        same_marks(m, wm, k)
        del junk
        pinned = torch.from_numpy(np.frombuffer(msg, np.uint8).copy()).pin_memory()
        assert el.on_message(pinned)
        g0 = layer.grid.cpu().numpy()
        m = el(layer)
        want, wm = gm.orc_mark_grid(d, gm.layer_floats(msg, d), layer.window, g0, 0.5, True)
        assert np.array_equal(layer.grid.cpu().numpy(), want), k
        same_marks(m, wm, ("elev", k))


def test_layer_classes_follow_the_robot():
    """GEM's two move_base costmaps fed from the mapping side's bytes through 10 moves: the local one (ElevationMapLayer
    on visual_map, max) and the global one (PointMapLayer on history_point, overwrite, inflated, published), against the
    same costmaps whose marks come from a host model of the two plugins over the oracle"""
    L, res = 200, 0.05
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    nav = gem_b200.ElevationMap(1, 0.1, compat_box_filter=False)           # move_base's own handle
    el, pl = costmap.ElevationMapLayer(nav, 0.7), costmap.PointMapLayer(nav, 0.7)
    stacks = {}
    for kind in ("dev", "model"):
        stacks[kind] = dict(lm=costmap.Costmap(nav, 75, 75, 0.2, fill=cc.FREE), ll=costmap.Costmap(nav, 75, 75, 0.2, fill=cc.FREE),
                            gm=costmap.Costmap(nav, 500, 500, 0.2, -50.0, -50.0, fill=cc.FREE),
                            gl=costmap.Costmap(nav, 500, 500, 0.2, -50.0, -50.0, fill=cc.UNKNOWN),
                            inf=costmap.InflationLayer(0.55, 10.0, costmap.inscribed_radius(costmap.GEM_FOOTPRINT)),
                            pub=costmap.CostmapPublisher())
    model = {"pending": None, "cloud": None}
    hdr = RosHeader(0, 0, 0, "odom")

    def model_elev(layer):
        if model["pending"] is None:
            return dict(costmap.NO_MARKS)
        d, v = model["pending"]
        model["pending"] = None
        grid, marks = gm.orc_mark_grid(d, v, layer.window, layer.grid.cpu().numpy(), 0.7, True)
        layer.grid.copy_(torch.from_numpy(grid.reshape(layer.grid.shape)))
        return marks

    def model_points(layer):
        if model["cloud"] is None:
            return dict(costmap.NO_MARKS)
        grid, marks = costmap_oracle.mark_points(model["cloud"], layer.window, layer.grid.cpu().numpy(), 0.7)
        layer.grid.copy_(torch.from_numpy(np.asarray(grid, np.uint8).reshape(layer.grid.shape)))
        return marks

    pos = np.array([0.1, 0.2, 1.7], np.float32)
    rng = np.random.default_rng(11)
    history = []
    kept = 0
    for k in range(10):
        fr = synth.hdl64_frame(k % 8, scene=scene)
        step = rng.uniform(0.2, 0.9, 2).astype(np.float32)
        pos = pos + np.array([step[0], step[1], 0.0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        g.move(pos)
        g.add(fr["xyzi"], fr["rgba"], gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
        g.compute_features()
        # the mapping side publishes; move_base receives visual_map every frame (pinned or pageable), history_point on
        # even frames
        vm = g.ros_grid_map(hdr)
        vm_host = vm.cpu().pin_memory() if k % 2 else vm.cpu().numpy().tobytes()
        got = el.on_message(vm_host)
        vm_bytes = vm.cpu().numpy().tobytes()
        if model["pending"] is None:
            d = gm.parse(vm_bytes)
            model["pending"] = (d, gm.layer_floats(vm_bytes, d).copy())
            assert got
            kept += 1
        else:
            assert not got
        if k % 2 == 0:
            history.append(g.export_grid_cloud("shown")[::7].contiguous())
            recs = torch.cat(history)
            hp = g.ros_cloud(hdr, [recs])
            pl.on_message(PointCloud2Layout(ICT, recs.shape[0], 1, 32), cloud_data(hp, recs.shape[0], len(hdr.frame_id)))
            model["cloud"] = recs.cpu().numpy()
        robot = (float(pos[0]), float(pos[1]))
        yaw = 0.3 * k
        out = {}
        for kind, elev, points in (("dev", el, pl), ("model", model_elev, model_points)):
            s = stacks[kind]
            if k % 3 != 2:                                                    # the local costmap misses some updates
                s["lm"].update(s["ll"], robot, "max", elev, robot_yaw=yaw, footprint=costmap.GEM_FOOTPRINT)
            s["gm"].update(s["gl"], robot, "overwrite", points, inflation=s["inf"])
            s["pub"].update_bounds(s["gm"])
            kind_, msg = s["pub"].publish(s["gm"], hdr)
            out[kind] = (kind_, msg.cpu().numpy().tobytes())
        nav.sync()
        for name in ("lm", "ll", "gm", "gl"):
            assert torch.equal(stacks["dev"][name].grid, stacks["model"][name].grid), (k, name)
            assert stacks["dev"][name].window == stacks["model"][name].window
        assert out["dev"] == out["model"], k
    assert kept >= 6 and int((stacks["dev"]["gm"].grid == cc.LETHAL).sum()) > 0


def test_cxx_facade_program(tmp_path):
    exe = native.facade_program("costmap_ingest_smoke", tmp_path)
    prefix = str(tmp_path / "cxx")
    r = subprocess.run([exe, prefix], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "costmap ingest ok" in r.stdout, r.stdout + r.stderr
    msg = open(prefix + ".msg.bin", "rb").read()
    d = gm.parse(msg)
    w = (-1.5, -1.5, 0.1, 40, 30)
    want, wm = gm.orc_mark_grid(d, gm.layer_floats(msg, d), w, np.zeros((30, 40), np.uint8), 0.5, True)
    assert open(prefix + ".elev.bin", "rb").read() == want.tobytes() and wm["marked"] > 0
    rec = np.frombuffer(open(prefix + ".cloud.bin", "rb").read(), np.float32).reshape(-1, 8)
    pw, pm = costmap_oracle.mark_points(rec, w, np.full((30, 40), 255, np.uint8), 0.5)
    assert open(prefix + ".point.bin", "rb").read() == np.asarray(pw, np.uint8).tobytes() and pm["marked"] > 0
