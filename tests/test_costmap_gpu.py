"""The navigation costmaps (GEM's ElevationMapLayer / PointMapLayer, DESIGN.md f8) byte for byte against the oracle,
tests/orc_costmap.c: the grids and every field of gem_costmap_marks on the crafted cases of tests/costmap_cases.py, show()'s
grid_map of natural maps (both sources, scrolled so that the wrap seam runs through a costmap cell), the local and the
global costmap driven through a moving robot with gem_b200.costmap, the c2 geometry, the map left unchanged, every error
path, and the C++ facade program run against the library."""
import ctypes as C
import subprocess

import numpy as np
import pytest
import torch

import costmap_cases as cc
import costmap_oracle
import gem_b200
import native
from gem_b200 import _lib, costmap, synth

pytestmark = pytest.mark.gpu
LAYERS = ("elevation", "variance", "intensity", "color_r", "color_g", "color_b", "traver", "lowest")


@pytest.fixture(scope="module")
def emap():
    return gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def same_marks(got, want, what):
    for k in ("marked", "lethal"):
        assert got[k] == want[k], (what, k, got[k], want[k])
    for k in ("min_x", "min_y", "max_x", "max_y"):
        assert np.float64(got[k]).tobytes() == np.float64(want[k]).tobytes(), (what, k, got[k], want[k])


def same_grid(got, want, what):
    g = got.cpu().numpy().reshape(-1)
    w = np.asarray(want, np.uint8).reshape(-1)
    if not np.array_equal(g, w):
        bad = np.flatnonzero(g != w)
        raise AssertionError((what, "cells differ", int(bad.size), "first", int(bad[0]), int(g[bad[0]]), int(w[bad[0]])))


@pytest.mark.parametrize("name", [c[0] for c in cc.point_cases()])
def test_mark_points_crafted(emap, name):
    _, rec, w, th, g0 = next(c for c in cc.point_cases() if c[0] == name)
    grid = dev(g0)
    m = emap.costmap_mark_points(dev(rec.reshape(-1, 8)), w, grid, th)
    want, wm = costmap_oracle.mark_points(rec, w, g0, th)
    same_grid(grid, want, name)
    same_marks(m, wm, name)


@pytest.mark.parametrize("name", [c[0] for c in cc.roll_cases()])
def test_update_origin_crafted(emap, name):
    _, w, seq, fill, g0 = next(c for c in cc.roll_cases() if c[0] == name)
    grid, wd, wo, go = dev(g0), w, w, g0
    for k, (nx, ny) in enumerate(seq):
        wd = emap.costmap_update_origin(wd, nx, ny, fill, grid)
        wo, go = costmap_oracle.update_origin(wo, nx, ny, fill, go)
        assert np.float64(wd[:3]).tobytes() == np.float64(wo[:3]).tobytes(), (name, k, wd, wo)
        same_grid(grid, go, (name, k))


@pytest.mark.parametrize("name", [c[0] for c in cc.combine_cases()])
@pytest.mark.parametrize("offset", [0, 3])
def test_combine_crafted(emap, name, offset):
    """offset 3 puts the layer at another 16-byte alignment than the master: the byte path"""
    _, mode, lay, mas, sx, sy, rect = next(c for c in cc.combine_cases() if c[0] == name)
    big = torch.zeros(lay.size + 16, dtype=torch.uint8, device="cuda:0")
    layer = big[offset:offset + lay.size]
    layer.copy_(dev(lay.reshape(-1)))
    master = dev(mas)
    emap.costmap_combine("max" if mode == 0 else "overwrite", layer, master, sx, sy, rect)
    emap.sync()
    same_grid(master, costmap_oracle.combine(mode, lay, mas, sx, sy, rect), (name, offset))
    assert torch.equal(big[offset:offset + lay.size].cpu(), torch.from_numpy(lay.reshape(-1)))


def shown_state(g):
    """show()'s traver ([ix, iy], NaN where cleared) and the geometry of the map as it is now"""
    tr = np.array(g.export_layers()["traver"])
    centre, start, _ = g.state()
    return tr, centre, start


def seam_window(L, res, centre, start, size, cres=0.2):
    """a window whose costmap cell holds the two neighbouring grid cells on either side of the storage wrap line (the last
    and the first in GridMapIterator order of a row)"""
    half = 0.5 * (L * res) - 0.5 * res
    gx, gy = L - int(start[0]), L - int(start[1])            # geographic index of storage cell 0
    px = float(np.float32(centre[0])) + half - res * gx
    py = float(np.float32(centre[1])) + half - res * gy
    k = size // 2
    return (px - 0.07 - k * cres, py - 0.07 - k * cres, cres, size, size)


@pytest.fixture(scope="module")
def scrolled():
    """a 256^2 map at 0.05 m after six frames on a track, so that the storage start index is far from 0, with its shown
    state and a snapshot taken one frame earlier"""
    L, res = 256, 0.05
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    pos = np.array([0.3, -0.2, 1.7], np.float32)
    snap = None
    for k in range(6):
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([0.9, 0.7, 0.0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        g.move(pos)
        g.add(fr["xyzi"], fr["rgba"], gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
        g.compute_features()
        if k == 4:
            g.snapshot_shown()
            snap = shown_state(g)
        g.raytracing()
    g.compute_features()
    return g, L, res, shown_state(g), snap


def map_windows(L, res, centre, start):
    c = (float(centre[0]), float(centre[1]))
    return {"local": (c[0] - 7.45, c[1] - 7.45, 0.2, 75, 75), "global": (c[0] - 100.0, c[1] - 100.0, 0.2, 1000, 1000),
            "seam": seam_window(L, res, centre, start, 9), "fine": (c[0] - 3.0, c[1] - 2.0, 0.05, 101, 77)}


@pytest.mark.parametrize("source", ["shown", "snapshot"])
@pytest.mark.parametrize("mark_unknown", [True, False])
@pytest.mark.parametrize("win", ["local", "global", "seam", "fine"])
def test_mark_map_natural(scrolled, source, mark_unknown, win):
    g, L, res, shown, snap = scrolled
    tr, centre, start = shown if source == "shown" else snap
    assert int(start[0]) != 0 and int(start[1]) != 0
    w = map_windows(L, res, centre, start)[win]
    vals = tr[np.isfinite(tr)]
    for th in (0.7, cc.F32_07, float(vals[len(vals) // 3])):     # the last one equals a cell's traversability
        rng = np.random.default_rng(7)
        g0 = cc.random_grid(rng, w)
        grid = dev(g0)
        m = g.costmap_mark_map(w, grid, th, source, mark_unknown)
        want, wm = costmap_oracle.mark_map(tr, L, res, centre, start, w, g0, th, mark_unknown)
        same_grid(grid, want, (source, win, th))
        same_marks(m, wm, (source, win, th))
        assert m["marked"] > 0


def test_mark_map_unknown_option_differs(scrolled):
    g, L, res, (tr, centre, start), _ = scrolled
    w = map_windows(L, res, centre, start)["local"]
    a, b = torch.full((75, 75), 255, dtype=torch.uint8, device="cuda:0"), torch.full((75, 75), 255, dtype=torch.uint8, device="cuda:0")
    ma, mb = g.costmap_mark_map(w, a, 0.7, "shown", True), g.costmap_mark_map(w, b, 0.7, "shown", False)
    assert ma["marked"] > mb["marked"] > 0
    assert int((b == 255).sum()) > int((a == 255).sum())


def test_local_and_global_costmaps_follow_the_robot():
    """GEM's two configs through 12 moves: the local costmap (ElevationMapLayer on the shown map, updateWithMax) and the
    global one (PointMapLayer on the history cloud = every harvested record so far + the grid cloud, overwrite), each
    compared after every update with the oracle run through the same LayeredCostmap::updateMap steps"""
    L, res = 200, 0.05
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    lm = costmap.Costmap(g, 75, 75, 0.2, fill=cc.FREE)
    ll = costmap.Costmap(g, 75, 75, 0.2, fill=cc.FREE)
    gm = costmap.Costmap(g, 1000, 1000, 0.2, -100.0, -100.0, fill=cc.FREE)
    gl = costmap.Costmap(g, 1000, 1000, 0.2, -100.0, -100.0, fill=cc.UNKNOWN)
    oracle = {id(c): [c.window, c.grid.cpu().numpy()] for c in (lm, ll, gm, gl)}
    history = np.zeros((0, 8), np.float32)
    pos = np.array([0.1, 0.2, 1.7], np.float32)
    rng = np.random.default_rng(5)

    def oracle_update(master, layer, robot, mode, mark):
        for c in (master, layer):
            w, gr = oracle[id(c)]
            sx_m, sy_m = c.size_in_meters()
            oracle[id(c)] = list(costmap_oracle.update_origin(w, robot[0] - sx_m / 2, robot[1] - sy_m / 2, c.fill, gr))
        lw, lg = oracle[id(layer)]
        lg, marks = mark(lw, lg)
        oracle[id(layer)][1] = lg
        mw, mg = oracle[id(master)]
        rect = costmap.update_rect(mw, marks)
        if rect is not None:
            x0, y0, xn, yn = rect
            mg = mg.copy()
            mg[y0:yn, x0:xn] = master.fill
            mg = costmap_oracle.combine(mode, lg, mg, mw[3], mw[4], rect)
            oracle[id(master)][1] = mg
        return rect, marks

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
        tr, c_now, s_now = shown_state(g)
        rect, marks = lm.update(ll, robot, "max", lambda l: l.mark_map(0.7))
        want = oracle_update(lm, ll, robot, 0, lambda w, gr: costmap_oracle.mark_map(tr, L, res, c_now, s_now, w, gr, 0.7))
        assert rect == want[0], (k, rect, want[0])
        same_marks(marks, want[1], ("local", k))
        cloud = torch.cat([dev(history).reshape(-1, 8), g.export_grid_cloud("shown")]).contiguous()
        host_cloud = cloud.cpu().numpy()
        rect, marks = gm.update(gl, robot, "overwrite", lambda l: l.mark_points(cloud, 0.7))
        want = oracle_update(gm, gl, robot, 1, lambda w, gr: costmap_oracle.mark_points(host_cloud, w, gr, 0.7))
        assert rect == want[0], (k, rect, want[0])
        same_marks(marks, want[1], ("global", k))
        g.sync()
        for c in (lm, ll, gm, gl):
            w, gr = oracle[id(c)]
            assert np.float64(c.window[:3]).tobytes() == np.float64(w[:3]).tobytes(), (k, c.window, w)
            same_grid(c.grid, gr, ("step", k))
        g.raytracing()
    assert history.shape[0] > 1000 and int((gm.grid == cc.LETHAL).sum()) > 0 and int((lm.grid == cc.LETHAL).sum()) > 0


@pytest.fixture(scope="module")
def c2_map():
    """the c2 geometry (1024^2 at 0.05 m) after 40 synthetic HDL-64 frames on a 0.3 m-per-frame track"""
    L, res = 1024, 0.05
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    for k in range(40):
        fr = synth.hdl64_frame(k % 16, scene=scene)
        pos = np.array([0.3 * k, 0.1 * k, 1.7], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        g.move(pos)
        g.add(torch.from_numpy(fr["xyzi"]).cuda(), torch.from_numpy(fr["rgba"]).cuda(),
              gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
    g.compute_features()
    g.snapshot_shown()
    return g, L, res, shown_state(g)


@pytest.mark.parametrize("size", [75, 1000])
@pytest.mark.parametrize("source", ["shown", "snapshot"])
def test_c2_geometry(c2_map, size, source):
    g, L, res, (tr, centre, start) = c2_map
    w = (float(centre[0]) - size * 0.1 + 0.03, float(centre[1]) - size * 0.1 - 0.01, 0.2, size, size)
    for mu in (True, False):
        g0 = np.full((size, size), 255, np.uint8)
        grid = dev(g0)
        m = g.costmap_mark_map(w, grid, 0.7, source, mu)
        want, wm = costmap_oracle.mark_map(tr, L, res, centre, start, w, g0, 0.7, mu)
        same_grid(grid, want, (size, source, mu))
        same_marks(m, wm, (size, source, mu))
    if size == 1000:
        assert m["marked"] > 100_000


def test_mark_map_compares_the_float_value_in_double(scrolled):
    """is_obstacle = (double)value < travers_thresh: a threshold a quarter float ulp above a cell's value makes that cell
    LETHAL, where a float comparison (the threshold rounded to the value) would leave it FREE.  One grid cell per
    costmap cell ("fine" window), so every such cell decides its costmap cell."""
    g, L, res, (tr, centre, start), _ = scrolled
    w = map_windows(L, res, centre, start)["fine"]
    ok, _, _ = cc.np_world_to_map(w, *cc.np_grid_positions(L, res, centre, start))
    inside = tr.reshape(-1, order="F")[ok]
    vals = np.unique(inside[np.isfinite(inside) & (inside > 0.0) & (inside < 1.0)])
    assert vals.size > 10
    for v in (vals[vals.size // 2], vals[vals.size // 5]):
        up = float(np.nextafter(v, np.float32(np.inf)))
        th = float(v) + (up - float(v)) / 4
        assert np.float32(th) == v
        g0 = np.full((w[4], w[3]), 255, np.uint8)
        grid = dev(g0)
        m = g.costmap_mark_map(w, grid, th, "shown", True)
        want, wm = costmap_oracle.mark_map(tr, L, res, centre, start, w, g0, th, True)
        as_float, _ = cc.np_mark_map(tr, L, res, centre, start, w, g0, float(v), True)
        assert not np.array_equal(want, as_float)          # the case tells double from float comparison apart
        same_grid(grid, want, ("double threshold", float(v)))
        same_marks(m, wm, ("double threshold", float(v)))


@pytest.mark.parametrize("source", ["shown", "snapshot"])
def test_mark_map_seam_cells_follow_iterator_order(scrolled, source):
    """costmap cells that straddle the storage wrap line get grid cells from both of its sides; the winner is the last in
    GridMapIterator order, which differs from the last in geographic order.  The case is checked to tell them apart."""
    g, L, res, shown, snap = scrolled
    tr, centre, start = shown if source == "shown" else snap
    w = seam_window(L, res, centre, start, 41)
    vals = tr[np.isfinite(tr)]
    told_apart = 0
    for th in [0.7] + [float(q) for q in np.quantile(vals, [0.2, 0.4, 0.6, 0.8])]:
        g0 = np.full((w[4], w[3]), 255, np.uint8)
        want, wm = costmap_oracle.mark_map(tr, L, res, centre, start, w, g0, th, True)
        geo, _ = cc.np_mark_map(tr, L, res, centre, start, w, g0, th, True, geographic=True)
        told_apart += int(np.count_nonzero(want != geo))
        grid = dev(g0)
        m = g.costmap_mark_map(w, grid, th, source, True)
        same_grid(grid, want, ("seam", source, th))
        same_marks(m, wm, ("seam", source, th))
    assert told_apart > 0


def test_grid_size_and_device_are_checked_against_the_tensor(scrolled):
    """the library sees only a pointer: the Python layer refuses a grid whose size is not the window's, before any call"""
    g, L, res, (tr, centre, start), _ = scrolled
    w = (float(centre[0]) - 100.0, float(centre[1]) - 100.0, 0.2, 1000, 1000)
    small = torch.full((75, 75), 7, dtype=torch.uint8, device="cuda:0")
    big = torch.full((1000, 1000), 7, dtype=torch.uint8, device="cuda:0")
    pts = g.export_grid_cloud("shown")
    calls = {"mark_map": lambda: g.costmap_mark_map(w, small, 0.7),
             "mark_points": lambda: g.costmap_mark_points(pts, w, small, 0.7),
             "update_origin": lambda: g.costmap_update_origin(w, w[0] + 3.0, w[1], 0, small),
             "combine_layer": lambda: g.costmap_combine("max", small, big, 1000, 1000, (0, 0, 1000, 1000)),
             "combine_master": lambda: g.costmap_combine("overwrite", big, small, 1000, 1000, (0, 0, 1000, 1000)),
             "wrong_dtype": lambda: g.costmap_mark_map(w, big.to(torch.int32), 0.7),
             "host_tensor": lambda: g.costmap_mark_map(w, big.cpu(), 0.7)}
    for what, call in calls.items():
        with pytest.raises(ValueError):
            call()
        g.sync()
        assert int((small != 7).sum()) == 0 and int((big != 7).sum()) == 0, what
    g.costmap_mark_map(w, big.view(1000, 1000), 0.7)   # any shape with size_x * size_y cells is accepted


def test_map_unchanged(scrolled):
    g, L, res, (tr, centre, start), _ = scrolled
    before = {k: g.get_layer(k) for k in LAYERS}
    exported = g.export_layers()
    w = map_windows(L, res, centre, start)["local"]
    grid = torch.zeros((75, 75), dtype=torch.uint8, device="cuda:0")
    g.costmap_mark_map(w, grid, 0.7, "shown")
    g.costmap_mark_map(w, grid, 0.7, "snapshot", False)
    g.costmap_mark_points(g.export_grid_cloud("shown"), w, grid, 0.7)
    w2 = g.costmap_update_origin(w, w[0] + 1.0, w[1] - 1.0, 0, grid)
    g.costmap_combine("max", grid, grid.clone(), 75, 75, (0, 0, 75, 75))
    g.sync()
    assert w2 != w
    for k in LAYERS:
        assert before[k].tobytes() == g.get_layer(k).tobytes(), k
    again = g.export_layers()
    for k, v in exported.items():
        assert np.asarray(v).tobytes() == np.asarray(again[k]).tobytes(), k


def test_errors_leave_the_grid_unchanged():
    g = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)
    lib, h = g._lib, g.handle
    g0 = np.arange(20 * 20, dtype=np.uint8).reshape(20, 20)
    grid = dev(g0)
    pg = C.c_void_p(grid.data_ptr())
    rec = dev(cc.records([(0.1, 0.1), (0.3, 0.3)], [0.1, 0.9]))
    pr = C.c_void_p(rec.data_ptr())
    mk = _lib.GemCostmapMarks()
    W = _lib.GemCostmapWindow
    good = W(-1.0, -1.0, 0.2, 20, 20)
    bad_windows = [W(-1.0, -1.0, 0.2, 0, 20), W(-1.0, -1.0, 0.2, 20, -1), W(-1.0, -1.0, 0.2, 65536, 32768),
                   W(-1.0, -1.0, 0.0, 20, 20), W(-1.0, -1.0, -0.2, 20, 20), W(-1.0, -1.0, float("nan"), 20, 20),
                   W(-1.0, -1.0, float("inf"), 20, 20)]
    calls = []
    for w in bad_windows:
        calls += [lambda w=w: lib.gem_costmap_mark_map(h, 0, C.byref(w), 0.7, 1, pg, C.byref(mk)),
                  lambda w=w: lib.gem_costmap_mark_points(h, pr, 2, C.byref(w), 0.7, pg, C.byref(mk)),
                  lambda w=w: lib.gem_costmap_update_origin(h, C.byref(w), 3.0, 3.0, 0, pg)]
        if w.resolution == 0.2:   # combine takes only the sizes
            calls.append(lambda w=w: lib.gem_costmap_combine(h, 0, pg, pg, w.size_x, w.size_y, 0, 0, 5, 5))
    calls += [lambda: lib.gem_costmap_mark_map(h, 0, None, 0.7, 1, pg, C.byref(mk)),
              lambda: lib.gem_costmap_mark_map(h, 0, C.byref(good), 0.7, 1, None, C.byref(mk)),
              lambda: lib.gem_costmap_mark_map(h, 0, C.byref(good), 0.7, 1, pg, None),
              lambda: lib.gem_costmap_mark_map(h, 2, C.byref(good), 0.7, 1, pg, C.byref(mk)),
              lambda: lib.gem_costmap_mark_map(h, 1, C.byref(good), 0.7, 1, pg, C.byref(mk)),       # no snapshot yet
              lambda: lib.gem_costmap_mark_points(h, None, 2, C.byref(good), 0.7, pg, C.byref(mk)),
              lambda: lib.gem_costmap_mark_points(h, pr, -1, C.byref(good), 0.7, pg, C.byref(mk)),
              lambda: lib.gem_costmap_mark_points(h, pr, 2, C.byref(good), 0.7, None, C.byref(mk)),
              lambda: lib.gem_costmap_update_origin(h, C.byref(good), float("nan"), 0.0, 0, pg),
              lambda: lib.gem_costmap_update_origin(h, C.byref(good), 0.0, float("inf"), 0, pg),
              lambda: lib.gem_costmap_update_origin(h, C.byref(good), 0.2 * 2.0 ** 31, 0.0, 0, pg),
              lambda: lib.gem_costmap_update_origin(h, C.byref(good), 3.0, 3.0, 0, None),
              lambda: lib.gem_costmap_combine(h, 2, pg, pg, 20, 20, 0, 0, 5, 5),
              lambda: lib.gem_costmap_combine(h, 0, None, pg, 20, 20, 0, 0, 5, 5),
              lambda: lib.gem_costmap_combine(h, 0, pg, None, 20, 20, 0, 0, 5, 5)]
    for k, call in enumerate(calls):
        assert call() != 0, k
        g.sync()
        assert np.array_equal(grid.cpu().numpy(), g0), k
    assert (good.origin_x, good.origin_y) == (-1.0, -1.0)
    # n = 0 is valid and writes nothing
    assert lib.gem_costmap_mark_points(h, None, 0, C.byref(good), 0.7, pg, C.byref(mk)) == 0
    assert mk.marked == 0 and mk.min_x == float("inf") and mk.max_y == float("-inf")
    assert np.array_equal(grid.cpu().numpy(), g0)


def test_tiled_handle():
    """mark_map reads the map and refuses a tiled handle; the other three calls work on any handle"""
    t = gem_b200.ElevationMap(64, 0.1, tile=(0, 32, 0, 64))
    w = (-1.0, -1.0, 0.2, 20, 20)
    g0 = np.full((20, 20), 255, np.uint8)
    grid = dev(g0)
    with pytest.raises(gem_b200.GemError, match="tiled"):
        t.costmap_mark_map(w, grid, 0.7)
    t.sync()
    assert np.array_equal(grid.cpu().numpy(), g0)
    rec = cc.records([(0.1, 0.1), (0.3, 0.3), (0.31, 0.32)], [0.1, 0.9, 0.2])
    m = t.costmap_mark_points(dev(rec), w, grid, 0.7)
    want, wm = costmap_oracle.mark_points(rec, w, g0, 0.7)
    same_grid(grid, want, "tiled points")
    same_marks(m, wm, "tiled points")
    w2 = t.costmap_update_origin(w, 0.0, -2.0, 255, grid)
    w2o, want = costmap_oracle.update_origin(w, 0.0, -2.0, 255, want)
    master = dev(np.zeros((20, 20), np.uint8))
    t.costmap_combine("overwrite", grid, master, 20, 20, (2, 2, 18, 18))
    t.sync()
    assert w2 == w2o
    same_grid(master, costmap_oracle.combine(1, want, np.zeros((20, 20), np.uint8), 20, 20, (2, 2, 18, 18)), "tiled combine")


def test_facade_costmap_program_runs():
    exe = native.facade_program("costmap_smoke")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "costmap ok" in r.stdout, r.stdout + r.stderr
