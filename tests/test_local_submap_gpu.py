"""Local submaps on the device, bit for bit against the oracles: gem_export_grid_cloud (gridMaptoPointCloud,
ElevationMapping.cpp:1198-1226), the device-resident localMap_ (gem_harvest_to_local_map / gem_local_map_take /
gem_local_map_clear, :740-747 and :1124-1140), the keyframe cut (:653-661) and the f3 -> f4 chain into loop-closure
re-fusion."""
import ctypes as C

import numpy as np
import pytest
import torch

import gem_b200
import native
import oracle_lib
import submap_oracle
from gem_b200 import synth
from oracle_lib import OracleMap
from submap_oracle import LocalMapDict

pytestmark = pytest.mark.gpu

# the driving sequence of test_scroll_out_harvest_matches_node_loop (diagonal, axis-aligned and zero shifts), then a
# back-and-forth leg over the same ground, so that keys repeat across calls
STEPS = [(0.0, 0.0), (0.9, 0.5), (1.0, 0.0), (0.0, -0.8), (-0.7, 0.6), (0.0, 0.0), (-1.1, -0.4), (0.8, -0.9),
         (-1.0, 0.0), (1.0, 0.0), (-1.0, 0.0), (0.0, 1.0), (0.0, -1.0), (1.0, 1.0)]


def bits(a):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same(a, b):
    return bits(a).shape == bits(b).shape and np.array_equal(bits(a), bits(b))


def laser_frame(T):
    return gem_b200.make_frame(T, gem_b200.LaserSensorProcessor())


def oracle_grid(o, res):
    """gridMaptoPointCloud of the oracle's current shown map"""
    centre, start, _ = o.state()
    return submap_oracle.grid_cloud(o.map_feature(), o.length, centre, start, res)


def oracle_snapshot_grid(o, res):
    f, centre, start = o._prev
    return submap_oracle.grid_cloud(f, o.length, centre, start, res)


def drive(L, res, steps, on_frame, scene, maps=None, pos0=(0.3, -0.2, 1.7)):
    """the node's per-frame order: Move, harvest (from the previous frame's snapshot), add, features + show, snapshot,
    ray clean-up; on_frame(k, g, o, centre, shift) runs after the harvest point, on_frame(k, ..., phase="shown") after
    the features"""
    g, o = maps if maps is not None else (gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res),
                                          OracleMap(L, res, compat_box_filter=False))
    pos = np.array(pos0, np.float32)
    for k, (dx, dy) in enumerate(steps):
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([dx, dy, 0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        f = laser_frame(T)
        cg, _, shg = g.move(pos)
        co, _, sho = o.move(pos)
        assert np.array_equal(cg, co) and np.array_equal(shg, sho)
        on_frame(k, g, o, cg, shg, "moved")
        for m in (g, o):
            m.add(fr["xyzi"], fr["rgba"], f)
            m.compute_features()
        on_frame(k, g, o, cg, shg, "shown")
        for m in (g, o):
            m.snapshot_shown()
            m.raytracing()
    return g, o


@pytest.mark.parametrize("L", [256, 200])
def test_grid_cloud_both_sources_over_a_scrolled_run(L):
    res = 0.1
    scene = synth.make_scene()
    seen = {"shown": 0, "snapshot": 0}

    def on_frame(k, g, o, centre, shift, phase):
        if phase == "shown":
            got, want = g.export_grid_cloud("shown"), oracle_grid(o, res)
            assert want.shape[0] > 1000 and same(got, want), (k, got.shape, want.shape)
            seen["shown"] += 1
            # a smaller capacity: the count is still the number of cells, the prefix is written
            cap = want.shape[0] // 3
            buf = torch.full((cap, 8), -7.0, dtype=torch.float32, device="cuda")
            cnt = C.c_int()
            assert g._lib.gem_export_grid_cloud(g.handle, 0, C.c_void_p(buf.data_ptr()), cap, C.byref(cnt)) == 0
            assert cnt.value == want.shape[0] and same(buf, want[:cap])
        elif k > 0:   # after the Move: the snapshot keeps its own geometry
            got, want = g.export_grid_cloud("snapshot"), oracle_snapshot_grid(o, res)
            assert want.shape[0] > 1000 and same(got, want), k
            seen["snapshot"] += 1
    drive(L, res, STEPS[:8], on_frame, scene)
    assert seen == {"shown": 8, "snapshot": 7}


def test_harvest_into_local_map_take_and_cut():
    L, res = 256, 0.1
    scene = synth.make_scene()
    d = LocalMapDict()
    st = {"total": 0, "cuts": 0}

    def on_frame(k, g, o, centre, shift, phase):
        if phase == "moved" and k > 0:
            plain, n_plain = g.harvest_scrolled_out(centre, shift)
            rec, n = g.harvest_to_local_map(centre, shift, records=True)
            want, n_o = o.harvest_scrolled_out(centre, shift, grid_res=res)
            assert n == n_plain == n_o and same(rec, plain) and same(rec, want), k
            d.insert_all(want)
            st["total"] += n
            assert g.local_map_size() == len(d), (k, g.local_map_size(), len(d))
        if phase == "shown" and k in (7, 13):
            nd = len(d)
            assert nd > 300, nd
            # too small: nothing written, the store kept, the size needed reported
            buf = torch.full((nd - 1, 8), -7.0, dtype=torch.float32, device="cuda")
            cnt = C.c_int()
            assert g._lib.gem_local_map_take(g.handle, C.c_void_p(buf.data_ptr()), nd - 1, C.byref(cnt)) == 0
            assert cnt.value == nd and bool((buf == -7.0).all()) and g.local_map_size() == nd
            grid = oracle_grid(o, res)
            cut = g.cut_submap()
            local = d.records()
            assert same(cut[:nd], local), k                    # insertion order of the literal dict
            assert same(cut[nd:], grid), k
            c = cut[:nd].cpu().numpy()                          # DEFINED fields: w = 1, a = 0xff, harvested intensity
            assert np.all(c[:, 3] == 1.0) and np.all((c[:, 4].view(np.uint32) >> 24) == 0xff)
            assert g.local_map_size() == 0
            assert same(g.cut_submap(), grid)                   # a second cut is exactly the grid part
            d.clear()
            st["cuts"] += 1
    drive(L, res, STEPS, on_frame, scene)
    assert st["cuts"] == 2 and st["total"] > 1000


def test_keys_repeat_across_calls_and_clear():
    L, res = 256, 0.1
    scene = synth.make_scene()
    d = LocalMapDict()
    st = {"total": 0}

    def on_frame(k, g, o, centre, shift, phase):
        if phase == "moved" and k > 0:
            rec, n = g.harvest_to_local_map(centre, shift, records=True)
            d.insert_all(rec)
            st["total"] += n
            assert g.local_map_size() == len(d)
    g, o = drive(L, res, [(0.0, 0.0)] + [(1.0, 0.0), (-1.0, 0.0)] * 4, on_frame, scene)
    n = g.local_map_size()
    assert n == len(d) and n > 100, (n, len(d))
    assert n < 0.75 * st["total"], (n, st["total"])   # the same columns went out again and again: keys repeated across calls
    taken = g.local_map_take()
    assert same(taken, d.records())
    g.harvest_to_local_map([0.0, 0.0], [0.0, 0.0])    # zero shift: nothing harvested
    assert g.local_map_size() == 0
    g.local_map_reserve(10)
    g.local_map_clear()
    assert g.local_map_size() == 0 and g.local_map_take().shape == (0, 8)


def test_same_key_twice_in_one_call_far_from_origin():
    """about 2e5 m from the origin at 0.01 m, neighbouring cell centres round to the same float: the later cell in
    GridMapIterator order wins, as in the sequential loop"""
    L, res = 128, 0.01
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    o = OracleMap(L, res, compat_box_filter=False)
    rng = np.random.default_rng(9)
    pos = np.array([2.0e5 + 0.37, 2.0e5 - 0.41, 0.0], np.float32)
    # a gentle slope: traversable cells (a rough 1 cm grid would leave none with traver >= 0 to harvest)
    layers = {"elevation": (0.5 + 0.0005 * np.arange(L)[:, None] + np.zeros((1, L))).astype(np.float32),
              "variance": np.full((L, L), 0.01, np.float32),
              "intensity": rng.uniform(1, 200, (L, L)).astype(np.float32),
              "color_r": rng.integers(1, 256, (L, L)).astype(np.int32),
              "color_g": rng.integers(1, 256, (L, L)).astype(np.int32),
              "color_b": rng.integers(1, 256, (L, L)).astype(np.int32)}
    for m in (g, o):
        m.move(pos)
        for name, a in layers.items():
            m.set_layer(name, a)
        m.compute_features()
        m.snapshot_shown()
    pos2 = pos + np.array([0.3, 0.25, 0.0], np.float32)
    cg, _, shg = g.move(pos2)
    co, _, sho = o.move(pos2)
    assert np.array_equal(cg, co) and np.array_equal(shg, sho)
    rec, n = g.harvest_to_local_map(cg, shg, records=True)
    want, n_o = o.harvest_scrolled_out(co, sho, grid_res=res)
    assert n == n_o and n > 500 and same(rec, want), (n, n_o)
    keys = rec[:, :2].copy().view(np.uint64).ravel()
    assert np.unique(keys).size < 0.9 * keys.size, (np.unique(keys).size, keys.size)   # cells share keys inside this one call
    d = LocalMapDict()
    d.insert_all(want)
    assert g.local_map_size() == len(d)
    assert same(g.local_map_take(), d.records())


def test_store_growth_equals_a_run_that_did_not_grow():
    L, res = 256, 0.1
    scene = synth.make_scene()
    small = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    big = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    small.local_map_reserve(1)          # 1024 records: the run below grows it several times
    big.local_map_reserve(1 << 20)      # never grows
    total = 0
    pos = np.array([0.3, -0.2, 1.7], np.float32)
    for k, (dx, dy) in enumerate(STEPS[:9]):   # two handles fed identically
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([dx, dy, 0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        f = laser_frame(T)
        c1, _, s1 = small.move(pos)
        c2, _, s2 = big.move(pos)
        assert np.array_equal(c1, c2) and np.array_equal(s1, s2)
        if k > 0:
            n1, n2 = small.harvest_to_local_map(c1, s1), big.harvest_to_local_map(c2, s2)
            assert n1 == n2
            total += n1
            assert small.local_map_size() == big.local_map_size()
        for m in (small, big):
            m.add(fr["xyzi"], fr["rgba"], f)
            m.compute_features()
            m.snapshot_shown()
            m.raytracing()
    assert total > 2 * 1024, total     # 1024 -> 2048 -> 4096: at least two growths
    a, b = small.local_map_take(), big.local_map_take()
    assert a.shape == b.shape and a.shape[0] > 500 and same(a, b), (a.shape, b.shape)


def test_f3_to_f4_end_to_end():
    """drive out and cut a submap, drive back over the same ground and cut a second one; loop-closure re-fusion of the
    two device cuts equals the same steps on the oracle's cuts"""
    L, res = 200, 0.1
    scene = synth.make_scene()
    d = LocalMapDict()
    cuts_dev, cuts_orc = [], []

    def on_frame(k, g, o, centre, shift, phase):
        if phase == "moved" and k > 0:
            g.harvest_to_local_map(centre, shift)
            d.insert_all(o.harvest_scrolled_out(centre, shift, grid_res=res)[0])
        if phase == "shown" and k in (5, 11):
            cuts_dev.append(g.cut_submap())
            cuts_orc.append(np.concatenate([d.records(), oracle_grid(o, res)]))
            d.clear()
    steps = [(0.0, 0.0)] + [(1.0, 0.2)] * 5 + [(-1.0, -0.2)] * 6
    drive(L, res, steps, on_frame, scene)
    assert len(cuts_dev) == 2
    for a, b in zip(cuts_dev, cuts_orc):
        assert b.shape[0] > 1000 and same(a, b)
    g = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)
    a = np.float32(0.02)
    T = np.array([[np.cos(a), -np.sin(a), 0, 0.07], [np.sin(a), np.cos(a), 0, -0.04], [0, 0, 1, 0.01], [0, 0, 0, 1]], np.float32)
    dev = [c.clone() for c in cuts_dev]
    orc = [c.copy() for c in cuts_orc]
    g.transform_cloud(dev[1], T)
    orc[1] = oracle_lib.transform_cloud(orc[1], T)
    assert same(dev[1], orc[1])
    for compat in (True, False):
        dn, do = dev[1].clone(), dev[0].clone()
        nn, no, fused = g.refuse_submaps(dn, do, res, compat)
        on, oo, fo = oracle_lib.refuse_submaps(orc[1], orc[0], res, compat)
        assert fused == fo and fused > 100
        assert same(dn[:nn], on) and same(do[:no], oo)


def test_facade_local_submap_program_runs():
    import subprocess
    exe = native.facade_program("local_submap_smoke")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "local_submap ok" in r.stdout, r.stdout + r.stderr


def test_errors():
    lib = gem_b200._lib.load()
    cnt = C.c_int()
    cur = (C.c_float * 2)(0.0, 0.0)
    sh = (C.c_float * 2)(1.0, 0.0)
    t = gem_b200.ElevationMap(64, 0.1, tile=(0, 32, 0, 64))
    for call in (lambda: t.export_grid_cloud("shown"), lambda: t.harvest_to_local_map([0, 0], [1, 0]),
                 lambda: t.local_map_take(), lambda: t.local_map_clear(), lambda: t.local_map_reserve(10)):
        with pytest.raises(gem_b200.GemError, match="tiled"):
            call()
    g = gem_b200.ElevationMap(64, 0.1)
    with pytest.raises(gem_b200.GemError, match="snapshot"):
        g.export_grid_cloud("snapshot")
    with pytest.raises(gem_b200.GemError, match="snapshot"):
        g.harvest_to_local_map([0, 0], [1, 0])
    h = g.handle
    buf = torch.empty((4, 8), dtype=torch.float32, device="cuda")
    p = C.c_void_p(buf.data_ptr())
    assert lib.gem_export_grid_cloud(h, 0, None, 5, C.byref(cnt)) == 1        # capacity without a buffer
    assert lib.gem_export_grid_cloud(h, 0, p, -1, C.byref(cnt)) == 1          # negative capacity
    assert lib.gem_export_grid_cloud(h, 2, p, 4, C.byref(cnt)) == 1           # unknown source
    assert lib.gem_export_grid_cloud(h, 0, p, 4, None) == 1
    assert lib.gem_export_grid_cloud(None, 0, p, 4, C.byref(cnt)) == 1
    assert lib.gem_export_grid_cloud(h, 0, p, 4, C.byref(cnt)) == 0 and cnt.value == 0   # empty map: no cell
    assert lib.gem_harvest_to_local_map(h, None, sh, None, 0, C.byref(cnt)) == 1
    assert lib.gem_harvest_to_local_map(h, cur, None, None, 0, C.byref(cnt)) == 1
    assert lib.gem_harvest_to_local_map(h, cur, sh, None, 3, C.byref(cnt)) == 1
    assert lib.gem_harvest_to_local_map(h, cur, sh, None, -1, C.byref(cnt)) == 1
    assert lib.gem_harvest_to_local_map(h, cur, sh, None, 0, None) == 1
    assert lib.gem_local_map_take(h, None, 3, C.byref(cnt)) == 1
    assert lib.gem_local_map_take(h, p, -1, C.byref(cnt)) == 1
    assert lib.gem_local_map_take(h, p, 4, None) == 1
    assert lib.gem_local_map_take(None, p, 4, C.byref(cnt)) == 1
    assert lib.gem_local_map_take(h, None, 0, C.byref(cnt)) == 0 and cnt.value == 0
    assert lib.gem_local_map_clear(None) == 1
    assert lib.gem_local_map_reserve(h, -1) == 1
    assert lib.gem_local_map_reserve(None, 5) == 1
