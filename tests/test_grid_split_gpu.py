"""gem_grid_cloud_split (composingGlobalMap's statistical outlier removal and road / obstacle split, ElevationMapping.cpp
:1146-1174) bit for bit against the oracle, tests/orc_grid_split.c.  The oracle's input is the grid cloud
gem_export_grid_cloud returns for the same source and state (itself checked against its oracle in
test_local_submap_gpu.py), so every case here only has to put points where the filter decides.

Crafted maps are built without the fusion path: a tilted rough surface gets the feature pass (every cell then has a
traversability), then the elevation layer is overwritten with the crafted point set (-10 = no point).  The grid cloud
is then exactly the crafted cells, with the traversabilities of the surface."""
import ctypes as C

import numpy as np
import pytest
import torch

import gem_b200
import native
import split_oracle
from gem_b200 import synth

pytestmark = pytest.mark.gpu
f32 = np.float32
PARAMS = [(20, 1.0), (1, 0.0), (2, -1.0), (64, 1.0), (20, -1.0), (20, 0.0)]


def bits32(a):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return np.ascontiguousarray(a, f32).view(np.uint32)


def same_f64(a, b):
    return np.float64(a).view(np.uint64) == np.float64(b).view(np.uint64) or (np.isnan(a) and np.isnan(b))


def check_split(g, source, mean_k, mul, tt=0.0, what=""):
    cloud = g.export_grid_cloud(source).cpu().numpy()
    road, obst, st, dist = g.grid_cloud_split(source, mean_k, mul, tt, distances=True)
    want = split_oracle.grid_split(cloud, mean_k, mul, tt)
    tag = (what, source, mean_k, mul, tt)
    assert st["points"] == cloud.shape[0], tag
    d, w = bits32(dist), bits32(want["dist"])
    nan_d, nan_w = np.isnan(dist.cpu().numpy()), np.isnan(want["dist"])
    assert d.shape == w.shape and np.array_equal(nan_d, nan_w) and np.array_equal(d[~nan_d], w[~nan_w]), \
        (tag, int(np.sum(d != w)))
    assert st["valid"] == want["valid"], (tag, st["valid"], want["valid"])
    for k in ("mean", "stddev", "threshold"):
        assert same_f64(st[k], want[k]), (tag, k, st[k], want[k])
    assert st["road"] == want["road"].shape[0] and st["obstacle"] == want["obstacle"].shape[0], (tag, st)
    assert np.array_equal(bits32(road), bits32(want["road"])) and np.array_equal(bits32(obst), bits32(want["obstacle"])), tag
    return st, want


def surface(rng, L, res, noise=0.05):
    g = np.arange(L)
    return (0.1 * g[:, None] * res - 0.15 * g[None, :] * res + rng.normal(0, noise, (L, L))).astype(f32)


def crafted(L, res, z_geo, start=(0, 0), pos=None, seed=1):
    """an ElevationMap whose shown map and snapshot hold exactly the points z_geo != -10 (geographic-indexed), with
    storage start index `start` (the wrap line runs through the map unless start is 0)"""
    rng = np.random.default_rng(seed)
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    if pos is None:
        k = [-(s % L) for s in start]
        pos = np.array([f32(k[0] * f32(res)), f32(k[1] * f32(res)), 0.0], f32)
    g.move(pos)
    cs = np.zeros(2, np.int32)
    centre = np.zeros(2, np.float32)
    sz = (C.c_float * 1)()
    assert g._lib.gem_get_state(g.handle, centre.ctypes.data_as(C.POINTER(C.c_float)), cs.ctypes.data_as(C.POINTER(C.c_int)), sz) == 0
    roll = lambda a: np.ascontiguousarray(np.roll(a, shift=(int(cs[0]), int(cs[1])), axis=(0, 1)))
    g.set_layer("elevation", roll(surface(rng, L, res)))
    g.set_layer("variance", np.full((L, L), f32(0.01)))
    g.compute_features()
    g.set_layer("elevation", roll(np.asarray(z_geo, f32)))
    g.snapshot_shown()
    return g


@pytest.mark.parametrize("L,res", [(256, 0.1), (200, 0.05), (201, 0.2)])
def test_natural_clouds_both_sources_after_scrolls(L, res):
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    pos = np.array([0.3, -0.2, 1.7], np.float32)
    steps = [(0.0, 0.0), (0.9, 0.5), (1.0, -0.3), (-0.7, 0.6)]
    for k, (dx, dy) in enumerate(steps):
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([dx, dy, 0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        g.move(pos)
        if k > 1:   # the snapshot of the previous frame, seen after the Move (its own geometry, wrap line inside)
            check_split(g, "snapshot", *PARAMS[k % len(PARAMS)], what=k)
        g.add(fr["xyzi"], fr["rgba"], gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
        g.compute_features()
        g.snapshot_shown()
        g.raytracing()
    for mk, mul in PARAMS:
        st, _ = check_split(g, "shown", mk, mul, what="final")
    assert st["points"] > 1000 and st["valid"] == st["points"]
    check_split(g, "snapshot", 20, 1.0, 0.3, what="final")


@pytest.mark.parametrize("start", [(0, 0), (5, 250), (131, 17)])
def test_dense_map_with_wrap_line_and_holes(start):
    L, res = 256, 0.1
    rng = np.random.default_rng(3)
    z = surface(rng, L, res, 0.08)
    z[rng.random((L, L)) < 0.3] = f32(-10.0)
    g = crafted(L, res, z, start)
    for mk, mul in PARAMS:
        for src in ("shown", "snapshot"):
            st, _ = check_split(g, src, mk, mul, what=start)
    assert st["points"] > 30000


@pytest.mark.parametrize("spacing", [3, 5, 17, 60])
def test_sparse_maps_and_isolated_cells(spacing):
    L, res = 200, 0.1
    rng = np.random.default_rng(spacing)
    z = np.full((L, L), f32(-10.0))
    for a in range(1, L, spacing):
        for b in range(2, L, spacing + 1):
            z[a, b] = f32(rng.normal(0, 0.3))
    z[0, L - 1] = f32(0.7)      # a corner cell far from the rest
    g = crafted(L, res, z, (37, 113))
    for mk, mul in PARAMS:
        check_split(g, "shown", mk, mul, what=spacing)


def test_far_corners_only():
    """a handful of points at the map's extremes: rings grow to the whole map"""
    L, res = 256, 0.1
    z = np.full((L, L), f32(-10.0))
    for (a, b) in [(0, 0), (0, L - 1), (L - 1, 0), (L - 1, L - 1), (128, 128), (0, 128), (200, 3)]:
        z[a, b] = f32(0.1 * a - 0.05 * b)
    g = crafted(L, res, z, (9, 200))
    for mk in (1, 2, 5, 6):
        check_split(g, "shown", mk, 1.0, what=mk)


@pytest.mark.parametrize("extra", [0, 1, 2])
def test_exactly_mean_k_and_a_few_more_points(extra):
    L, res = 64, 0.1
    rng = np.random.default_rng(20 + extra)
    for mk in (1, 2, 20, 64):
        z = np.full((L, L), f32(-10.0))
        z.ravel()[rng.choice(L * L, mk + extra, replace=False)] = rng.normal(0, 0.3, mk + extra).astype(f32)
        z.ravel()[rng.choice(np.flatnonzero(z.ravel() == f32(-10.0)), 3, replace=False)] = np.nan   # non-finite beside them
        g = crafted(L, res, z, (3, 60))
        st, _ = check_split(g, "shown", mk, 1.0, what=extra)
        assert st["valid"] == (0 if extra == 0 else mk + extra) and st["points"] == mk + extra + 3


def test_steps_of_several_metres():
    L, res = 128, 0.05
    rng = np.random.default_rng(8)
    z = surface(rng, L, res, 0.02)
    z[:, 64:] += f32(5.0)
    z[40:46, 10:90] -= f32(8.0)
    z[90:, :30] += f32(2.5)
    g = crafted(L, res, z, (100, 7))
    for mk, mul in PARAMS:
        check_split(g, "snapshot", mk, mul, what="steps")


def test_non_finite_and_huge_elevations():
    L, res = 128, 0.1
    rng = np.random.default_rng(11)
    z = surface(rng, L, res)
    for v, cnt in ((np.nan, 200), (np.inf, 50), (-np.inf, 50), (1e18, 100), (-1e18, 100), (3e38, 10), (-3e38, 10)):
        z.ravel()[rng.choice(L * L, cnt, replace=False)] = f32(v)
    g = crafted(L, res, z, (64, 1))
    for mk, mul in PARAMS:
        st, _ = check_split(g, "shown", mk, mul, what="magnitudes")
    assert st["valid"] < st["points"]


def test_far_from_origin_centres_round_together():
    """about 2e5 m from the origin at 0.01 m neighbouring cell centres round to the same float (float spacing 1/64 m):
    a ring bound from q * res instead of the rounded positions would stop too early"""
    L, res = 128, 0.01
    rng = np.random.default_rng(9)
    z = (0.5 + 0.0005 * np.arange(L)[:, None] + rng.normal(0, 0.002, (L, L))).astype(f32)
    z[rng.random((L, L)) < 0.2] = f32(-10.0)
    g = crafted(L, res, z, pos=np.array([2.0e5 + 0.37, 2.0e5 - 0.41, 0.0], f32))
    cloud = g.export_grid_cloud("shown").cpu().numpy()
    assert np.unique(cloud[:, 0]).size < 0.9 * L
    for mk, mul in PARAMS:
        check_split(g, "shown", mk, mul, what="far")


def test_pairs_at_a_quarter_metre_nothing_removed():
    L, res = 64, 0.25
    z = np.full((L, L), f32(-10.0))
    for a in range(4, L - 8, 9):
        for b in range(4, L - 8, 9):
            z[a, b] = z[a, b + 1] = f32(0.0)
    g = crafted(L, res, z, (10, 20))
    for mul in (1.0, 0.0, -1.0):
        st, want = check_split(g, "shown", 1, mul, what="pairs")
        assert st["mean"] == 0.25 and st["stddev"] == 0.0 and st["threshold"] == 0.25
        assert st["road"] + st["obstacle"] == st["points"] > 50


def test_traversability_at_the_threshold_and_one_ulp_either_side():
    L, res = 96, 0.1
    rng = np.random.default_rng(4)
    z = surface(rng, L, res)
    g = crafted(L, res, z, (50, 50))
    cloud = g.export_grid_cloud("shown").cpu().numpy()
    t = np.sort(cloud[:, 7])[cloud.shape[0] // 2]
    assert np.sum(cloud[:, 7] == t) >= 1
    for thr in (t, np.nextafter(t, f32(-np.inf)), np.nextafter(t, f32(np.inf))):
        check_split(g, "shown", 20, 1.0, float(thr), what="trav")
    st_at, _ = check_split(g, "shown", 20, 10.0, float(t))
    st_below, _ = check_split(g, "shown", 20, 10.0, float(np.nextafter(t, f32(-np.inf))))
    assert st_below["road"] > st_at["road"]     # the cells at t go to the obstacle cloud at equality


def test_capacity_prefix_size_query_and_map_unchanged():
    L, res = 128, 0.1
    rng = np.random.default_rng(6)
    z = surface(rng, L, res)
    z[rng.random((L, L)) < 0.2] = f32(-10.0)
    g = crafted(L, res, z, (11, 99))
    lib = g._lib
    layers = {n: g.get_layer(n) for n in gem_b200._lib.LAYERS}
    before = {s: g.export_grid_cloud(s).cpu().numpy() for s in ("shown", "snapshot")}
    _, want = check_split(g, "snapshot", 20, 0.5, 0.4)
    st = gem_b200._lib.GemGridSplit()
    assert lib.gem_grid_cloud_split(g.handle, 1, 20, 0.5, 0.4, None, 0, None, 0, None, 0, C.byref(st)) == 0
    nr, no, n = want["road"].shape[0], want["obstacle"].shape[0], st.points
    assert st.road == nr and st.obstacle == no and nr > 10 and no > 10
    cr, co, cd = nr // 3, no // 2, n // 4
    road = torch.full((cr + 1, 8), -7.0, device="cuda")
    obst = torch.full((co + 1, 8), -7.0, device="cuda")
    dist = torch.full((cd + 1,), -7.0, device="cuda")
    assert lib.gem_grid_cloud_split(g.handle, 1, 20, 0.5, 0.4, C.c_void_p(road.data_ptr()), cr, C.c_void_p(obst.data_ptr()), co,
                                    C.c_void_p(dist.data_ptr()), cd, C.byref(st)) == 0
    assert st.road == nr and st.obstacle == no and st.points == n
    assert np.array_equal(bits32(road[:cr]), bits32(want["road"][:cr])) and bool((road[cr] == -7.0).all())
    assert np.array_equal(bits32(obst[:co]), bits32(want["obstacle"][:co])) and bool((obst[co] == -7.0).all())
    assert np.array_equal(bits32(dist[:cd]), bits32(want["dist"][:cd])) and float(dist[cd]) == -7.0
    for name, a in layers.items():
        assert np.array_equal(np.asarray(g.get_layer(name)).view(np.uint32), np.asarray(a).view(np.uint32)), name
    for s in ("shown", "snapshot"):
        assert np.array_equal(bits32(g.export_grid_cloud(s)), bits32(before[s])), s


def test_errors():
    lib = gem_b200._lib.load()
    st = gem_b200._lib.GemGridSplit()
    t = gem_b200.ElevationMap(64, 0.1, tile=(0, 32, 0, 64))
    with pytest.raises(gem_b200.GemError, match="tiled"):
        t.grid_cloud_split("shown")
    g = gem_b200.ElevationMap(64, 0.1)
    with pytest.raises(gem_b200.GemError, match="snapshot"):
        g.grid_cloud_split("snapshot")
    h = g.handle
    buf = torch.empty((4, 8), dtype=torch.float32, device="cuda")
    p = C.c_void_p(buf.data_ptr())
    ok = lambda *a: lib.gem_grid_cloud_split(*a, C.byref(st))
    assert ok(h, 0, 20, 1.0, 0.0, p, 4, p, 4, None, 0) == 0 and st.points == 0 and st.valid == 0   # empty map
    for mk in (0, -1, 65):
        assert ok(h, 0, mk, 1.0, 0.0, p, 4, p, 4, None, 0) == 1
    assert ok(h, 2, 20, 1.0, 0.0, p, 4, p, 4, None, 0) == 1                  # unknown source
    assert ok(h, 0, 20, 1.0, 0.0, None, 4, p, 4, None, 0) == 1               # capacity without a buffer
    assert ok(h, 0, 20, 1.0, 0.0, p, 4, None, 4, None, 0) == 1
    assert ok(h, 0, 20, 1.0, 0.0, p, 4, p, 4, None, 3) == 1
    assert ok(h, 0, 20, 1.0, 0.0, p, -1, p, 4, None, 0) == 1                 # negative capacities
    assert ok(h, 0, 20, 1.0, 0.0, p, 4, p, -1, None, 0) == 1
    assert ok(h, 0, 20, 1.0, 0.0, p, 4, p, 4, p, -1) == 1
    assert lib.gem_grid_cloud_split(h, 0, 20, 1.0, 0.0, p, 4, p, 4, None, 0, None) == 1
    assert lib.gem_grid_cloud_split(None, 0, 20, 1.0, 0.0, p, 4, p, 4, None, 0, C.byref(st)) == 1


def test_facade_grid_split_program_runs():
    import subprocess
    exe = native.facade_program("grid_split_smoke")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "grid_split ok" in r.stdout, r.stdout + r.stderr
