"""InflationLayer on the device (gem_costmap_inflate, DESIGN.md f14) byte for byte against the oracle tests/orc_inflate.c:
every crafted case and witness of tests/inflation_cases.py, seeded random grids at r = 1 ... 40, the 1000 x 1000 global
geometry with the c2 grid cloud marked, rolling global and local costmaps through a moving robot, back-to-back calls on one
stream, the map left unchanged, every error path, scratch growth, and the C++ facade program."""
import ctypes as C
import subprocess

import numpy as np
import pytest
import torch

import costmap_oracle
import inflation_cases as ic
import inflation_oracle as O
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


def same_grid(got, want, what):
    g = got.cpu().numpy().reshape(-1)
    w = np.asarray(want, np.uint8).reshape(-1)
    if not np.array_equal(g, w):
        bad = np.flatnonzero(g != w)
        raise AssertionError((what, "cells differ", int(bad.size), "first", int(bad[0]), int(g[bad[0]]), int(w[bad[0]])))


def window(g, res):
    return (0.0, 0.0, float(res), int(g.shape[1]), int(g.shape[0]))


def run(emap, g, res, p, rect):
    grid = dev(g)
    emap.costmap_inflate(window(g, res), p, grid, rect)
    emap.sync()
    return grid


@pytest.mark.parametrize("name", [c[0] for c in ic.all_cases()])
def test_crafted(emap, name):
    _, g, res, p, rect = {c[0]: c for c in ic.all_cases()}[name]
    same_grid(run(emap, g, res, p, rect), O.inflate(g, res, p, rect), name)


@pytest.mark.parametrize("r", [1, 2, 3, 5, 8, 13, 21, 40])
def test_random_grids(emap, r):
    for k, density in enumerate((0.002, 0.02, 0.1, 0.3, 0.5)):
        seed = 100 * r + k
        rng = np.random.default_rng(seed)
        sy, sx = int(rng.integers(60, 200)), int(rng.integers(60, 200))
        g = ic.random_grid(seed, sy, sx, density, unknown=float(rng.choice([0.0, 0.1])))
        p = O.params(0.1 * r - 0.001, float(rng.uniform(0.5, 12.0)), float(rng.uniform(0.0, 0.4)), bool(k & 1))
        rect = (int(rng.integers(0, sx // 2)), int(rng.integers(0, sy // 2)), int(rng.integers(sx // 2, sx + 1)),
                int(rng.integers(sy // 2, sy + 1)))
        same_grid(run(emap, g, 0.1, p, rect), O.inflate(g, 0.1, p, rect), (r, density))


def test_back_to_back_calls_share_the_scratch(emap):
    """calls issued without synchronising in between, on grids of different sizes and radii"""
    cases, grids = [], []
    for k in range(12):
        rng = np.random.default_rng(700 + k)
        sy, sx = int(rng.integers(10, 300)), int(rng.integers(10, 300))
        g = ic.random_grid(700 + k, sy, sx, float(rng.choice([0.01, 0.05, 0.2])))
        p = O.params(float(rng.uniform(0.05, 2.5)), 3.0, 0.2, bool(k & 1))
        cases.append((g, p))
        grids.append(dev(g))
    for (g, p), grid in zip(cases, grids):
        emap.costmap_inflate(window(g, 0.1), p, grid, (0, 0, g.shape[1], g.shape[0]))
    # one grid inflated twice in a row: the second call sees the first one's output
    g, p = cases[0]
    emap.costmap_inflate(window(g, 0.1), p, grids[0], (3, 3, 9, 9))
    emap.sync()
    for k, ((g, p), grid) in enumerate(zip(cases, grids)):
        want = O.inflate(g, 0.1, p, (0, 0, g.shape[1], g.shape[0]))
        if k == 0:
            want = O.inflate(want, 0.1, p, (3, 3, 9, 9))
        same_grid(grid, want, ("back to back", k))


def test_scratch_growth(emap):
    for n in (8, 120, 700, 1500):
        g = ic.random_grid(n, n, n + 3, 0.01)
        p = O.params(0.4, 5.0, 0.1)
        same_grid(run(emap, g, 0.1, p, (0, 0, n + 3, n)), O.inflate(g, 0.1, p, (0, 0, n + 3, n)), n)


def c2_grid_cloud():
    """the c2 geometry (1024^2 at 0.05 m) after 40 synthetic HDL-64 frames: its shown grid cloud"""
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
    return g, g.export_grid_cloud("shown"), pos


def test_global_costmap_c2_geometry():
    """GEM's global costmap (1000 x 1000 at 0.2 m): PointMapLayer's overwrite of the c2 grid cloud, then the inflation at
    costmap_2d's defaults, at 2 m, over the update rect and over the whole grid"""
    g, cloud, pos = c2_grid_cloud()
    w = (float(pos[0]) - 100.0, float(pos[1]) - 100.0, 0.2, 1000, 1000)
    layer = dev(np.full((1000, 1000), 255, np.uint8))
    marks = g.costmap_mark_points(cloud, w, layer, 0.7)
    rect = costmap.update_rect(w, marks)
    master0 = np.zeros((1000, 1000), np.uint8)
    master0 = costmap_oracle.combine(1, layer.cpu().numpy(), master0, 1000, 1000, rect)
    assert int((master0 == 254).sum()) > 100
    ins = costmap.inscribed_radius(costmap.GEM_FOOTPRINT)
    for radius, r in ((0.55, rect), (2.0, rect), (0.55, (0, 0, 1000, 1000))):
        p = O.params(radius, 10.0, ins)
        grid = dev(master0)
        g.costmap_inflate(w, p, grid, r)
        g.sync()
        want = O.inflate(master0, 0.2, p, r)
        assert int((want != master0).sum()) > 100
        same_grid(grid, want, (radius, r))


def test_rolling_global_and_local_costmaps():
    """a moving robot: the global costmap (PointMapLayer + InflationLayer) and a local one (ElevationMapLayer +
    InflationLayer) through Costmap.update(..., inflation=...), grid and rect compared with the oracle every update"""
    L, res = 200, 0.05
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    gm = costmap.Costmap(g, 300, 300, 0.2, -30.0, -30.0, fill=O.FREE)
    gl = costmap.Costmap(g, 300, 300, 0.2, -30.0, -30.0, fill=O.UNKNOWN)
    lm = costmap.Costmap(g, 75, 75, 0.2, fill=O.FREE)
    ll = costmap.Costmap(g, 75, 75, 0.2, fill=O.FREE)
    ins = costmap.inscribed_radius(costmap.GEM_FOOTPRINT)
    ginf = costmap.InflationLayer(0.55, 10.0, ins)
    linf = costmap.InflationLayer(0.5, 3.0, ins, inflate_unknown=True)
    oracle = {id(c): [c.window, c.grid.cpu().numpy()] for c in (gm, gl, lm, ll)}
    state = {id(ginf): [True, None], id(linf): [True, None]}
    pos = np.array([0.1, 0.2, 1.7], np.float32)
    rng = np.random.default_rng(9)

    def oracle_update(master, layer, inf, robot, mode, mark):
        for c in (master, layer):
            w, gr = oracle[id(c)]
            sx_m, sy_m = c.size_in_meters()
            oracle[id(c)] = list(costmap_oracle.update_origin(w, robot[0] - sx_m / 2, robot[1] - sy_m / 2, c.fill, gr))
        lw, lg = oracle[id(layer)]
        lg, marks = mark(lw, lg)
        oracle[id(layer)][1] = lg
        b = (min(1e30, marks["min_x"]), min(1e30, marks["min_y"]), max(-1e30, marks["max_x"]), max(-1e30, marks["max_y"]))
        st = state[id(inf)]
        rad = inf.params["inflation_radius"]
        if st[0]:
            st[0], st[1] = False, b
            b = (-costmap.FLT_MAX, -costmap.FLT_MAX, costmap.FLT_MAX, costmap.FLT_MAX)
        else:
            last, st[1] = st[1], b
            b = (min(last[0], b[0]) - rad, min(last[1], b[1]) - rad, max(last[2], b[2]) + rad, max(last[3], b[3]) + rad)
        mw, mg = oracle[id(master)]
        rect = costmap.update_rect(mw, dict(zip(("min_x", "min_y", "max_x", "max_y"), b)))
        if rect is not None:
            x0, y0, xn, yn = rect
            mg = mg.copy()
            mg[y0:yn, x0:xn] = master.fill
            mg = costmap_oracle.combine(mode, lg, mg, mw[3], mw[4], rect)
            mg = O.inflate(mg, mw[2], inf.params, rect)
            oracle[id(master)][1] = mg
        return rect

    for k in range(10):
        fr = synth.hdl64_frame(k % 8, scene=scene)
        step = rng.uniform(0.2, 0.9, 2).astype(np.float32)
        pos = pos + np.array([step[0], step[1], 0.0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        g.move(pos)
        g.add(fr["xyzi"], fr["rgba"], gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
        g.compute_features()
        robot = (float(pos[0]), float(pos[1]))
        if k == 6:
            ginf.set_parameters(1.0, 5.0, ins)   # a parameter change re-inflates the whole grid
            state[id(ginf)][0] = True
        cloud = g.export_grid_cloud("shown").contiguous()
        host_cloud = cloud.cpu().numpy()
        rect, _ = gm.update(gl, robot, "overwrite", lambda l: l.mark_points(cloud, 0.7), inflation=ginf)
        want = oracle_update(gm, gl, ginf, robot, 1, lambda w, gr: costmap_oracle.mark_points(host_cloud, w, gr, 0.7))
        assert rect == want, (k, rect, want)
        # the local costmap: ElevationMapLayer on the shown map (its marking is checked against the oracle by the f8
        # suite; here the device's layer grid and marks feed the oracle's updateMap)
        seen = {}

        def mark_map(l):
            seen["marks"] = l.mark_map(0.7)
            seen["grid"] = l.grid.cpu().numpy()
            return seen["marks"]
        rect, _ = lm.update(ll, robot, "max", mark_map, inflation=linf)
        want = oracle_update(lm, ll, linf, robot, 0, lambda w, gr: (seen["grid"], seen["marks"]))
        assert rect == want, (k, rect, want)
        g.sync()
        for c in (gm, gl, lm, ll):
            w, gr = oracle[id(c)]
            assert np.float64(c.window[:3]).tobytes() == np.float64(w[:3]).tobytes(), (k, c.window, w)
            same_grid(c.grid, gr, ("step", k))
    assert int((gm.grid == 254).sum()) > 0 and int((gm.grid == 253).sum()) > 0


def test_map_unchanged():
    g, cloud, pos = c2_grid_cloud()
    before = {k: g.get_layer(k) for k in LAYERS}
    gr = ic.random_grid(5, 200, 200, 0.05)
    grid = dev(gr)
    g.costmap_inflate(window(gr, 0.1), O.params(1.0, 3.0, 0.2), grid, (0, 0, 200, 200))
    g.sync()
    same_grid(grid, O.inflate(gr, 0.1, O.params(1.0, 3.0, 0.2), (0, 0, 200, 200)), "map unchanged")
    for k in LAYERS:
        assert before[k].tobytes() == g.get_layer(k).tobytes(), k


def test_errors_leave_the_grid_unchanged():
    g = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)
    lib, h = g._lib, g.handle
    g0 = ic.random_grid(2, 20, 20, 0.2)
    grid = dev(g0)
    pg = C.c_void_p(grid.data_ptr())
    W, P = _lib.GemCostmapWindow, _lib.GemCostmapInflation
    good, gp = W(0.0, 0.0, 0.1, 20, 20), P(0.5, 3.0, 0.1, 0)
    nan, inf = float("nan"), float("inf")
    bad_windows = [W(0.0, 0.0, 0.1, 0, 20), W(0.0, 0.0, 0.1, 20, -1), W(0.0, 0.0, 0.1, 65536, 32768), W(0.0, 0.0, 0.0, 20, 20),
                   W(0.0, 0.0, -0.1, 20, 20), W(0.0, 0.0, nan, 20, 20), W(0.0, 0.0, inf, 20, 20)]
    bad_params = [P(-0.5, 3.0, 0.1, 0), P(nan, 3.0, 0.1, 0), P(inf, 3.0, 0.1, 0), P(0.5, -1.0, 0.1, 0), P(0.5, nan, 0.1, 0),
                  P(0.5, inf, 0.1, 0), P(0.5, 3.0, -0.1, 0), P(0.5, 3.0, nan, 0), P(0.5, 3.0, inf, 0), P(0.5, 3.0, 0.1, 2),
                  P(0.5, 3.0, 0.1, -1)]
    calls = [lambda w=w: lib.gem_costmap_inflate(h, C.byref(w), C.byref(gp), pg, 0, 0, 20, 20) for w in bad_windows]
    calls += [lambda p=p: lib.gem_costmap_inflate(h, C.byref(good), C.byref(p), pg, 0, 0, 20, 20) for p in bad_params]
    calls += [lambda: lib.gem_costmap_inflate(h, None, C.byref(gp), pg, 0, 0, 20, 20),
              lambda: lib.gem_costmap_inflate(h, C.byref(good), None, pg, 0, 0, 20, 20),
              lambda: lib.gem_costmap_inflate(h, C.byref(good), C.byref(gp), None, 0, 0, 20, 20)]
    for k, call in enumerate(calls):
        assert call() == 1, k   # GEM_ERR_INVALID
        assert b"gem_costmap_inflate" in C.string_at(lib.gem_last_error(h)), k
        g.sync()
        assert np.array_equal(grid.cpu().numpy(), g0), k
    with pytest.raises(gem_b200.GemError, match="gem_costmap_inflate"):
        g.costmap_inflate(window(g0, 0.1), O.params(-1.0), grid, (0, 0, 20, 20))
    # radius 0 and an empty widened rect are valid and write nothing
    assert lib.gem_costmap_inflate(h, C.byref(good), C.byref(P(0.0, 3.0, 0.1, 0)), pg, 0, 0, 20, 20) == 0
    assert lib.gem_costmap_inflate(h, C.byref(good), C.byref(gp), pg, 40, 40, 50, 50) == 0
    g.sync()
    assert np.array_equal(grid.cpu().numpy(), g0)


def test_tiled_handle():
    t = gem_b200.ElevationMap(64, 0.1, tile=(0, 32, 0, 64))
    g0 = ic.random_grid(8, 30, 30, 0.05)
    p = O.params(0.6, 4.0, 0.1)
    same_grid(run(t, g0, 0.1, p, (0, 0, 30, 30)), O.inflate(g0, 0.1, p, (0, 0, 30, 30)), "tiled")


def test_facade_inflation_program_runs():
    exe = native.facade_program("inflation_smoke")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "inflation ok" in r.stdout, r.stdout + r.stderr
