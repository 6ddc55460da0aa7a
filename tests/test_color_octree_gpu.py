"""gem_color_octree (composingGlobalMap's road / obstacle ColorOcTrees, ElevationMapping.cpp:1146-1174) byte for byte
against the oracle, tests/orc_color_octree.c: the stream and every count of gem_octree, on the crafted families of
tests/octree_cases.py, large random clouds, natural split clouds through global_octrees (a small map and the c2
snapshot), the API's behaviour, and the C++ facade program run against the library."""
import ctypes as C
import subprocess

import numpy as np
import pytest
import torch

import gem_b200
import native
import octree_cases as oc
import octree_oracle
from gem_b200 import synth

pytestmark = pytest.mark.gpu
CASES = oc.crafted_cases()
LAYERS = ("elevation", "variance", "intensity", "color_r", "color_g", "color_b", "traver", "lowest")


@pytest.fixture(scope="module")
def emap():
    return gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)


def device_records(rec):
    return torch.from_numpy(np.ascontiguousarray(rec, np.float32).reshape(-1, 8)).to("cuda:0")


def check_tree(g, rec, res, what):
    s, info = g.color_octree(device_records(rec), res)
    want, winfo = octree_oracle.color_octree(rec, res)
    got = s.cpu().numpy()
    assert info == winfo, (what, info, winfo)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if not np.array_equal(got, want):
        bad = np.flatnonzero(got != want)
        raise AssertionError((what, "first differing byte", int(bad[0]), "node", int(bad[0]) // 8, int(bad.size)))
    return info


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_crafted_clouds(emap, name):
    _, rec, res = next(c for c in CASES if c[0] == name)
    check_tree(emap, rec, res, name)


@pytest.mark.parametrize("n,box,voxels,res,seed", [(100_000, 64, 20_000, 0.1, 1), (1_000_000, 256, 150_000, 0.1, 2),
                                                   (300_000, 12, 9_000, 0.1, 3), (200_000, 6, 1_500, 0.05, 4),
                                                   (500_000, 40, 60_000, 0.2, 5)])
def test_random_clouds(emap, n, box, voxels, res, seed):
    rng = np.random.default_rng(seed)
    rec = oc.random_cloud(rng, n, box, voxels, res)
    info = check_tree(emap, rec, res, (n, box, voxels))
    assert info["inserted"] == n


def test_random_cloud_with_full_cubes_beside_leaves(emap):
    rng = np.random.default_rng(9)
    parts = [oc.block_keys((8 * i, 0, 8), 8, ("morton", "reverse", "random")[i % 3], rng) for i in range(6)]
    parts += [oc.block_keys((4 * i, 16, 0), 4, "random", rng) for i in range(20)]
    keys = np.concatenate(parts + [rng.integers(-40, 40, (30_000, 3))])
    keys = np.concatenate([keys, keys[rng.integers(0, keys.shape[0], 200_000)]])
    rec = oc.cloud(keys, 0.1, rng.integers(0, 256, (keys.shape[0], 3)))
    check_tree(emap, rec, 0.1, "cubes")
    check_tree(emap, rec[rng.permutation(rec.shape[0])], 0.1, "cubes permuted")


def test_full_cubes_beyond_the_shared_memory_subtree(emap):
    """a 64^3 cube is a level-6 group, simulated in the global scratch; the 32^3 cube beside it (level 5) and the small
    ones in shared memory"""
    rng = np.random.default_rng(11)
    big = oc.block_keys((0, 0, 0), 64, "random", rng)
    mid = oc.block_keys((64, 0, 0), 32, "random", rng)
    keys = np.concatenate([big, mid, oc.block_keys((0, 64, 0), 4, "random", rng), rng.integers(-20, 0, (5000, 3))])
    keys = np.concatenate([keys, keys[rng.integers(0, keys.shape[0], 100_000)]])
    keys = keys[rng.permutation(keys.shape[0])]
    check_tree(emap, oc.cloud(keys, 0.1, rng.integers(0, 256, (keys.shape[0], 3))), 0.1, "level 6")


@pytest.fixture(scope="module")
def natural():
    L, res = 256, 0.1
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    pos = np.array([0.3, -0.2, 1.7], np.float32)
    for k, (dx, dy) in enumerate([(0.0, 0.0), (0.9, 0.5), (1.0, -0.3)]):
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([dx, dy, 0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        g.move(pos)
        g.add(fr["xyzi"], fr["rgba"], gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
        g.compute_features()
        g.snapshot_shown()
        g.raytracing()
    return g


@pytest.mark.parametrize("road_res,obstacle_res", [(0.2, 0.1), (0.1, 0.1), (0.05, 0.3)])
def test_natural_global_octrees(natural, road_res, obstacle_res):
    g = natural
    road, obstacle, st = g.grid_cloud_split("snapshot", 20, 1.0, 0.0)
    assert st["road"] > 1000 and st["obstacle"] > 100
    rs, os_, st2 = g.global_octrees("snapshot", 20, 1.0, 0.0, road_res, obstacle_res)
    assert st2 == st
    for part, s, res in (("road", rs, road_res), ("obstacle", os_, obstacle_res)):
        want, winfo = octree_oracle.color_octree((road if part == "road" else obstacle).cpu().numpy(), res)
        assert np.array_equal(s.cpu().numpy(), want), (part, res)
        assert oc.decode(want)[0] == winfo["nodes"]


@pytest.fixture(scope="module")
def c2_snapshot():
    """the c2 geometry (1024^2 at 0.05 m) after 40 synthetic HDL-64 frames on a 0.3 m-per-frame track, snapshotted"""
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
    return g


@pytest.mark.parametrize("road_res,obstacle_res", [(0.2, 0.1), (0.05, 0.05)])
def test_c2_snapshot_global_octrees(c2_snapshot, road_res, obstacle_res):
    g = c2_snapshot
    road, obstacle, st = g.grid_cloud_split("snapshot", 20, 1.0, 0.0)
    assert st["points"] > 400_000 and st["road"] > 100_000
    rs, os_, st2 = g.global_octrees("snapshot", 20, 1.0, 0.0, road_res, obstacle_res)
    assert st2 == st
    for part, s, cloud, res in (("road", rs, road, road_res), ("obstacle", os_, obstacle, obstacle_res)):
        want, _ = octree_oracle.color_octree(cloud.cpu().numpy(), res)
        assert s.shape[0] == want.shape[0] and np.array_equal(s.cpu().numpy(), want), (part, res)


def test_repeated_builds_and_map_unchanged(natural):
    g = natural
    before = {k: g.get_layer(k) for k in LAYERS}
    road, _, _ = g.grid_cloud_split("snapshot")
    first, info = g.color_octree(road, 0.2)
    for res in (0.1, 0.2):
        g.color_octree(road, res)
    again, info2 = g.color_octree(road, 0.2)
    assert info == info2 and torch.equal(first, again)
    for k in LAYERS:
        a, b = before[k], g.get_layer(k)
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), k


def read_raw(g, nbytes):
    out = np.zeros(max(nbytes, 1), np.uint8)
    rc = g._lib.gem_color_octree_read(g.handle, C.c_void_p(out.ctypes.data), nbytes)
    return rc, out[:nbytes]


def test_errors_leave_the_last_stream():
    g = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)
    lib, h = g._lib, g.handle
    info = gem_b200._lib.GemOctree()
    rc, _ = read_raw(g, 1 << 20)
    assert rc != 0, "read before any build"
    rec = device_records(oc.random_cloud(np.random.default_rng(3), 5000, 20, 2000))
    s, inf = g.color_octree(rec, 0.1)
    want = s.cpu().numpy()
    p = C.c_void_p(rec.data_ptr())
    bad = [(p, -1, 0.1), (None, 10, 0.1), (p, 10, float("nan")), (p, 10, float("inf")), (p, 10, 0.0), (p, 10, -0.1),
           (p, 10, float("-inf"))]
    for args in bad:
        assert lib.gem_color_octree(h, *args, C.byref(info)) != 0, args
        rc, got = read_raw(g, inf["bytes"])
        assert rc == 0 and np.array_equal(got, want), args
    rc, _ = read_raw(g, inf["bytes"] - 1)
    assert rc != 0, "capacity < bytes"
    rc, got = read_raw(g, inf["bytes"])
    assert rc == 0 and np.array_equal(got, want)
    dev = torch.zeros(inf["bytes"], dtype=torch.uint8, device="cuda:0")
    assert lib.gem_color_octree_read(h, C.c_void_p(dev.data_ptr()), dev.numel()) == 0
    assert np.array_equal(dev.cpu().numpy(), want)
    e, einf = g.color_octree(rec[:0], 0.1)
    assert e.numel() == 0 and einf["bytes"] == 0 and einf["nodes"] == 0
    assert read_raw(g, 0)[0] == 0


def test_tiled_handle_is_refused():
    t = gem_b200.ElevationMap(64, 0.1, tile=(0, 32, 0, 64))
    rec = device_records(oc.random_cloud(np.random.default_rng(4), 100, 10, 50))
    with pytest.raises(gem_b200.GemError, match="tiled"):
        t.color_octree(rec, 0.1)
    info = gem_b200._lib.GemOctree()
    assert t._lib.gem_color_octree(t.handle, C.c_void_p(rec.data_ptr()), 100, 0.1, C.byref(info)) != 0
    assert read_raw(t, 1 << 16)[0] != 0     # nothing was built


def test_facade_color_octree_program_runs():
    exe = native.facade_program("color_octree_smoke")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "color_octree ok" in r.stdout, r.stdout + r.stderr
