"""GPU parity tests: CUDA path (through the C ABI) vs the CPU oracle on identical inputs.

Bar (BASELINE.json north_star): cell indices bit-exact; fused height/variance within 1e-5
relative.  Because the library is compiled without FMA contraction and shares the oracle's
arithmetic definition, the tests assert the stronger property: every layer bit-identical.
"""
import numpy as np
import pytest

import frame_cases as fc
import gem_b200
from gem_b200 import synth
from helpers import assert_layers_equal, split_rgb
from oracle_lib import OracleMap

pytestmark = pytest.mark.gpu


def laser_frame(T, base_z=0.0, **kw):
    return gem_b200.make_frame(T, gem_b200.LaserSensorProcessor(), base_z=base_z, **kw)


def both(L, res, **kw):
    return gem_b200.ElevationMap(L, res, **kw), OracleMap(L, res, **{k: v for k, v in kw.items() if k != "max_points"})


def test_process_points_bit_exact_c1():
    """BASELINE config 1: one 64-beam frame into 200x200 @ 0.1 m; keys/var/height bit-exact."""
    fr = synth.hdl64_frame(0)
    g, o = both(200, 0.1, compat_box_filter=False)
    f = laser_frame(fr["T"], base_z=0.0)
    g.move(fr["position"]); o.move(fr["position"])
    x, y, z = (fr["xyzi"][:, k].copy() for k in range(3))
    kg = g.process_points(x, y, z, f)
    ko = o.process_points(x, y, z, f)
    names = ["map_index", "var", "x_ts", "y_ts", "z_ts"]
    for a, b, nm in zip(kg, ko, names):
        assert a.dtype == b.dtype
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), nm
    assert (kg[0] >= 0).sum() > 10000
    assert_layers_equal(g, o, ["lowest"], what="process_points")


def test_fused_add_c1_all_layers():
    fr = synth.hdl64_frame(0)
    g, o = both(200, 0.1, compat_box_filter=False)
    f = laser_frame(fr["T"])
    g.move(fr["position"]); o.move(fr["position"])
    g.add(fr["xyzi"], fr["rgba"], f)
    o.add(fr["xyzi"], fr["rgba"], f)
    assert_layers_equal(g, o, what="c1 add")
    st = g.stats()
    assert st["points_in"] == fr["xyzi"].shape[0]
    assert 0 < st["points_binned"] <= st["points_in"]
    assert st["cells_touched"] == int((o.get_layer("elevation") != -10).sum())


def test_unfused_equals_fused():
    fr = synth.hdl64_frame(1)
    f = laser_frame(fr["T"])
    g1 = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False)
    g2 = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False)
    g1.move(fr["position"]); g2.move(fr["position"])
    g1.add(fr["xyzi"], fr["rgba"], f)
    x, y, z = (fr["xyzi"][:, k].copy() for k in range(3))
    key, var, xt, yt, zt = g2.process_points(x, y, z, f)
    R, G, B = split_rgb(fr["rgba"])
    g2.fuse_points(key, R, G, B, fr["xyzi"][:, 3], zt, var)
    assert_layers_equal(g1, g2, what="fused vs unfused")


def test_order_dependence_dense_collisions():
    """many points per cell, gate hits, replacements: the per-cell order must be index order"""
    L, res = 64, 0.25
    c = synth.random_cloud(60000, seed=7, extent=7.5, zmin=-1.0, zmax=2.0)
    T = synth.pose_matrix(0.3, -0.2, 0.5, 0.3)
    f = laser_frame(T, base_z=0.5)
    g, o = both(L, res, compat_box_filter=False)
    for m in (g, o):
        m.move([0.3, -0.2, 0.5])
        m.add(c["xyzi"], c["rgba"], f)
    assert_layers_equal(g, o, what="dense")
    assert g.stats()["max_points_per_cell"] > 20


def test_every_cell_carries_a_long_list():
    """small map, every cell gets tens of points: the per-call lists of long cells (work queue of k_fold) are as
    long as the map has cells; their capacity is min(cells, points / (k + 1)), not cells / k"""
    L, res = 96, 0.1
    c = synth.random_cloud(500000, seed=21, extent=4.9, zmin=-0.5, zmax=1.0, dup_frac=0.0)
    f = laser_frame(np.eye(4), base_z=0.0)
    g, o = both(L, res, compat_box_filter=False)
    for m in (g, o):
        m.add(c["xyzi"], c["rgba"], f)
    assert_layers_equal(g, o, what="all cells long")
    st = g.stats()
    assert st["cells_touched"] > 0.9 * L * L and st["max_points_per_cell"] > 60


def test_very_long_cell_lists_fallback_paths():
    """> 1024 points in one cell exercises the global-memory selection path of k_fold"""
    L, res = 32, 0.5
    rng = np.random.default_rng(3)
    n = 5000
    xyz = np.zeros((n, 3), np.float32)
    xyz[:3000, :2] = rng.uniform(0.01, 0.49, (3000, 2))      # one cell, 3000 points
    xyz[3000:, :2] = rng.uniform(-7, 7, (2000, 2))
    xyz[:, 2] = rng.uniform(-0.5, 0.5, n)
    xyzi = np.concatenate([xyz, rng.integers(1, 255, (n, 1)).astype(np.float32)], 1).astype(np.float32)
    rgba = rng.integers(1, 255, (n, 4)).astype(np.uint8)
    f = laser_frame(np.eye(4), base_z=0.0)
    g, o = both(L, res, compat_box_filter=False)
    for m in (g, o):
        m.add(xyzi, rgba, f)
    assert_layers_equal(g, o, what="long lists")
    assert g.stats()["max_points_per_cell"] >= 3000


def test_gate_boundary_is_decided_like_the_literal_expression():
    """the CUDA fold decides the 5-sigma gate with a squared pre-test and falls back to the
    literal |dh|/sqrt(var) > 5 inside a narrow band: sweep heights across the boundary, ulp by ulp"""
    L = 64
    rng = np.random.default_rng(9)
    ncell = L * L
    var0 = rng.uniform(1.2e-4, 0.5, ncell).astype(np.float32)
    e0 = rng.uniform(-1, 1, ncell).astype(np.float32)
    g, o = both(L, 0.1, compat_box_filter=False)
    for m in (g, o):
        m.set_layer("elevation", e0)
        m.set_layer("variance", var0)
    s = np.sqrt(var0.astype(np.float64))
    keys, hs, vs = [], [], []
    for c in range(ncell):
        base = np.float32(e0[c] + (5.0 * s[c]) * (1 if c & 1 else -1))
        k = int(rng.integers(-40, 41))
        h = base
        for _ in range(abs(k)):
            h = np.nextafter(h, np.float32(np.inf if k > 0 else -np.inf), dtype=np.float32)
        keys.append(c); hs.append(h); vs.append(np.float32(rng.uniform(1e-3, 0.1)))
    keys = np.array(keys, np.int32); hs = np.array(hs, np.float32); vs = np.array(vs, np.float32)
    ones = np.ones(ncell, np.int32)
    for m in (g, o):
        m.fuse_points(keys, ones, ones, ones, ones.astype(np.float32), hs, vs)
    assert_layers_equal(g, o, ["elevation", "variance"], what="gate boundary")
    # extreme magnitudes take the literal path
    big = np.array([1e20, -1e20, 3e38, 1e-30, np.inf, np.nan], np.float32)
    kk = np.arange(6, dtype=np.int32)
    for m in (g, o):
        m.set_layer("variance", np.full(ncell, 1e30, np.float32))
        m.fuse_points(kk, ones[:6], ones[:6], ones[:6], ones[:6].astype(np.float32), big, np.full(6, 1e25, np.float32))
    assert_layers_equal(g, o, ["elevation", "variance"], what="extreme magnitudes")


def test_shared_reciprocal_division_is_ieee_exact():
    """div2_rn (the fold's division) must be bit-identical to the `/` operator: 2^28 random triples"""
    g = gem_b200.ElevationMap(64, 0.1)
    bad, fast = g.selftest_division(n=1 << 28, seed=12345)
    assert bad == 0
    assert fast > (1 << 27)      # most samples really exercise the fast path


def test_compat_box_filter_and_thresholds():
    fr = synth.hdl64_frame(2, compat_axes=True)
    g, o = both(200, 0.1, compat_box_filter=True)
    f = laser_frame(fr["T"], base_z=0.0)
    for m in (g, o):
        m.move(fr["position"])
        m.add(fr["xyzi"], fr["rgba"], f)
    assert_layers_equal(g, o, what="box filter")
    n_valid = int((o.get_layer("elevation") != -10).sum())
    assert 0 < n_valid


def test_multi_frame_stream_with_scroll_and_cleanup():
    """10-frame stream: move -> add -> var_update -> features -> raytracing, layers after every frame"""
    L, res = 256, 0.1
    scene = synth.make_scene()
    g, o = both(L, res, compat_box_filter=False)
    for k in range(10):
        fr = synth.hdl64_frame(k, scene=scene, speed=7.0)
        f = laser_frame(fr["T"])
        for m in (g, o):
            m.move(fr["position"])
            m.add(fr["xyzi"], fr["rgba"], f)
            m.var_update(0.0)
        assert_layers_equal(g, o, what=f"frame {k} after add")
        fg = g.map_feature()
        fo = o.map_feature()
        for name in fo:
            a, b = fg[name], fo[name]
            same = (a == b) | (np.isnan(a.astype(np.float64)) & np.isnan(b.astype(np.float64)))
            assert same.all(), f"frame {k} map_feature {name}: {np.count_nonzero(~same)} differ"
        assert_layers_equal(g, o, ["traver"], what=f"frame {k} traver")
        g.raytracing(); o.raytracing()
        assert_layers_equal(g, o, what=f"frame {k} after raytracing")
        sg, so = g.state(), o.state()
        assert np.array_equal(sg[0], so[0]) and np.array_equal(sg[1], so[1]) and sg[2] == so[2]
    assert (o.get_layer("elevation") != -10).sum() > 1000


def test_structured_light_c3_small():
    """config c3: the raw 640x480 D435 image (NaN where there is no return, depths beyond the useful range kept)
    through the fused add; cleanPointCloud's depth pass-through (StructuredLightSensorProcessor.cpp:51-66) is part
    of the path: the oracle really removes the points (orc_clean_point_cloud), the device rejects them in place"""
    fr = synth.d435_frame(0)
    z = fr["xyzi"][:, 2]
    assert fr["xyzi"].shape[0] == 640 * 480
    assert np.isnan(z).sum() > 100 and (z > 3.25).sum() > 1000 and ((z >= 0.2) & (z <= 3.25)).sum() > 50000
    sp = gem_b200.StructuredLightSensorProcessor()
    f = gem_b200.make_frame(fr["T"], sp, base_z=0.0)
    g, o = both(512, 0.02, compat_box_filter=False)
    for m in (g, o):
        m.move(fr["position"])
        m.add(fr["xyzi"], fr["rgba"], f)
    assert_layers_equal(g, o, what="structured light")
    assert (o.get_layer("elevation") != -10).sum() > 5000
    assert g.stats()["points_binned"] <= int(((z >= 0.2) & (z <= 3.25)).sum())
    # the filter bites: with the pass-through wide open more points reach the map
    wide = gem_b200.StructuredLightSensorProcessor(cutoff_min_depth=-1e30, cutoff_max_depth=1e30)
    fw = gem_b200.make_frame(fr["T"], wide, base_z=0.0)
    g2, o2 = both(512, 0.02, compat_box_filter=False)
    for m in (g2, o2):
        m.move(fr["position"])
        m.add(fr["xyzi"], fr["rgba"], fw)
    assert_layers_equal(g2, o2, what="structured light, pass-through wide open")
    assert g2.stats()["points_binned"] > g.stats()["points_binned"]
    # limits are compared as floats and inclusive (pcl::PassThrough): a point exactly on a limit is kept
    edge = np.array([[0.0, 0.0, np.float32(0.2), 9.0], [0.0, 0.0, np.nextafter(np.float32(0.2), np.float32(0)), 9.0],
                     [0.0, 0.0, np.float32(3.25), 9.0], [0.0, 0.0, np.nextafter(np.float32(3.25), np.float32(9)), 9.0]], np.float32)
    g3, o3 = both(64, 0.1, compat_box_filter=False)
    fe = gem_b200.make_frame(np.eye(4), sp, base_z=0.0)
    for m in (g3, o3):
        m.add(edge, None, fe)
    assert_layers_equal(g3, o3, what="pass-through limits")
    assert g3.stats()["points_binned"] == 2


def test_rotation_variance_term():
    """the fused add path on the frames whose rotation term tests/test_reference_pin_frames.py pins the oracle to the
    reference with (device = oracle = reference): every constant non-trivial, the rotation term alone, and a rotation
    Jacobian that overflows under a zero rotation variance (NaN variances, as in the reference)"""
    for c in fc.frame_cases():
        g, o = both(c.L, c.res, compat_box_filter=True)
        for m in (g, o):
            m.move(c.position)
            m.add(c.xyzi, c.rgba, c.frame)
        assert_layers_equal(g, o, what=f"rotation variance, {c.name}")
        if c.name == "overflow":
            assert np.isnan(o.get_layer("variance")).sum() > 20


def test_odd_length_and_edges():
    c = synth.random_cloud(30000, seed=5, extent=8.0)
    f = laser_frame(np.eye(4))
    for L in (75, 120):
        g, o = both(L, 0.2, compat_box_filter=False)
        for m in (g, o):
            m.move([0.37, -1.21, 0.0])
            m.add(c["xyzi"], c["rgba"], f)
        assert_layers_equal(g, o, what=f"L={L}")


def test_empty_and_ragged_inputs():
    g, o = both(64, 0.1, compat_box_filter=False)
    f = laser_frame(np.eye(4))
    empty = np.zeros((0, 4), np.float32)
    g.add(empty, None, f, n=0)
    o.fuse_points(np.zeros(0, np.int32), None, None, None, None, np.zeros(0, np.float32), np.zeros(0, np.float32))
    assert_layers_equal(g, o, what="empty")   # variance floor applied to every cell by the empty fuse
    c = synth.random_cloud(1, seed=1, extent=1.0)
    for m in (g, o):
        m.add(c["xyzi"], None, f)
    assert_layers_equal(g, o, what="single point, no colour")
    nanpts = np.full((5, 4), np.nan, np.float32)
    for m in (g, o):
        m.add(nanpts, None, f)
    assert_layers_equal(g, o, what="NaN points")


def test_chunking_preserves_order():
    c = synth.random_cloud(50000, seed=21, extent=6.0)
    f = laser_frame(np.eye(4))
    g = gem_b200.ElevationMap(64, 0.2, compat_box_filter=False, max_points=4096)
    o = OracleMap(64, 0.2, compat_box_filter=False)
    g.add(c["xyzi"], c["rgba"], f)
    o.add(c["xyzi"], c["rgba"], f)
    assert_layers_equal(g, o, ["elevation", "variance", "intensity", "color_r", "color_g", "color_b"], what="chunked")


def test_device_pointer_path_matches_host_path():
    import torch
    fr = synth.hdl64_frame(3)
    f = laser_frame(fr["T"])
    g1 = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False)
    g2 = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False)
    xyzi = torch.from_numpy(fr["xyzi"]).cuda()
    rgba = torch.from_numpy(fr["rgba"]).cuda()
    torch.cuda.synchronize()
    g1.move(fr["position"]); g2.move(fr["position"])
    g1.add(xyzi, rgba, f)
    g1.sync()
    g2.add(fr["xyzi"], fr["rgba"], f)
    assert_layers_equal(g1, g2, what="device vs host input")
    assert g1.stats() == g2.stats()


def test_stream_mode_overlapping_frames_matches_oracle():
    """gem_add_points_stream overlaps frame i+1's front kernels with frame i's fold: 24 frames issued
    back to back without any synchronisation, with scrolling, must equal the oracle's sequential result"""
    import torch
    import ctypes as C
    scene = synth.make_scene()
    nf = 6
    frames = [synth.hdl64_frame(k, scene=scene) for k in range(nf)]
    fobj = [laser_frame(fr["T"]) for fr in frames]
    xd = [torch.from_numpy(fr["xyzi"]).cuda() for fr in frames]
    rd = [torch.from_numpy(fr["rgba"]).cuda() for fr in frames]
    torch.cuda.synchronize()
    g, o = both(512, 0.1, compat_box_filter=False)
    seq = [0, 1, 2, 3, 4, 5, 4, 3, 2, 1, 0, 1, 2, 3, 4, 5, 4, 3, 2, 1, 0, 1, 2, 3]
    g.add(frames[0]["xyzi"], frames[0]["rgba"], fobj[0])            # mix with the ordinary path
    for k in seq:
        g.move(frames[k]["position"])
        g.add_stream_fast(C.c_void_p(xd[k].data_ptr()), C.c_void_p(rd[k].data_ptr()), frames[k]["xyzi"].shape[0], C.byref(fobj[k]))
    g.add(xd[2], rd[2], fobj[2])                                     # ordinary path after stream mode
    g.sync()
    o.add(frames[0]["xyzi"], frames[0]["rgba"], fobj[0])
    for k in seq:
        o.move(frames[k]["position"])
        o.add(frames[k]["xyzi"], frames[k]["rgba"], fobj[k])
    o.add(frames[2]["xyzi"], frames[2]["rgba"], fobj[2])
    assert_layers_equal(g, o, what="stream mode")


def test_pipelined_host_ingest_matches_sync_path():
    import torch
    import ctypes as C
    scene = synth.make_scene()
    frames = [synth.hdl64_frame(k, scene=scene) for k in range(5)]
    g1 = gem_b200.ElevationMap(512, 0.1, compat_box_filter=False)
    g2 = gem_b200.ElevationMap(512, 0.1, compat_box_filter=False)
    pinned = [(torch.from_numpy(fr["xyzi"]).pin_memory(), torch.from_numpy(fr["rgba"]).pin_memory()) for fr in frames]
    fobj = [laser_frame(fr["T"]) for fr in frames]
    for k, fr in enumerate(frames):
        g1.move(fr["position"]); g2.move(fr["position"])
        g1.add(fr["xyzi"], fr["rgba"], fobj[k])
        g2.add_host_async_fast(C.c_void_p(pinned[k][0].data_ptr()), C.c_void_p(pinned[k][1].data_ptr()),
                               fr["xyzi"].shape[0], C.byref(fobj[k]))
    g2.sync()
    assert_layers_equal(g1, g2, what="pipelined host ingest")
    assert g1.stats() == g2.stats()


def test_multi_segment_batch_equals_sequential_adds():
    """gem_add_points_multi (8 sensors, own transforms, one launch) == 8 sequential adds"""
    import torch
    L, res = 1024, 0.1
    scene = synth.make_scene()
    frs = [synth.hdl64_frame(k, scene=scene) for k in range(8)]
    for k, fr in enumerate(frs):
        fr["T"] = fr["T"].copy()
        fr["T"][:2, 3] = (-30.0 + 9.0 * k, 12.0 * ((k % 3) - 1))
    fobj = [laser_frame(fr["T"]) for fr in frs]
    seq = gem_b200.ElevationMap(L, res, compat_box_filter=False)
    for fr, f in zip(frs, fobj):
        seq.add(fr["xyzi"], fr["rgba"], f)
    multi = gem_b200.ElevationMap(L, res, compat_box_filter=False)
    x = torch.from_numpy(np.concatenate([fr["xyzi"] for fr in frs])).cuda()
    c = torch.from_numpy(np.concatenate([fr["rgba"] for fr in frs])).cuda()
    off = np.concatenate([[0], np.cumsum([fr["xyzi"].shape[0] for fr in frs])])
    torch.cuda.synchronize()
    multi.add_multi(x, c, off, fobj)
    multi.sync()
    assert_layers_equal(seq, multi, ["elevation", "variance", "intensity", "color_r", "color_g", "color_b"], what="multi")
    assert multi.stats()["points_in"] == int(off[-1])


def test_colourise_matches_oracle_and_feeds_the_fold():
    """SURVEY 8f row 2 (ElevationMapping.cpp:331-381): KITTI-shaped projection, random image"""
    import torch
    import oracle_lib
    rng = np.random.default_rng(17)
    W, H = 1241, 376
    bgr = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
    Tc = np.array([[718.856, 0, 607.1928, 0], [0, 718.856, 185.2157, 0], [0, 0, 1, 0]], np.float64)
    Tl = np.array([[0, -1, 0, 0.0], [0, 0, -1, -0.08], [1, 0, 0, -0.27], [0, 0, 0, 1]], np.float64)  # lidar x fwd -> camera z
    fr = synth.hdl64_frame(2)
    xo, co = oracle_lib.colourise(fr["xyzi"], Tc, Tl, bgr)
    x = torch.from_numpy(fr["xyzi"].copy()).cuda()
    c = torch.zeros((x.shape[0], 4), dtype=torch.uint8, device="cuda")
    img = torch.from_numpy(bgr).cuda()
    g = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False)
    torch.cuda.synchronize()
    g.colourise(x, Tc, Tl, img, c)
    g.sync()
    assert np.array_equal(c.cpu().numpy(), co)
    assert np.array_equal(x.cpu().numpy().view(np.uint32), xo.view(np.uint32))
    inside = int((co[:, 3] == 255).sum())
    assert 2000 < inside < x.shape[0] - 2000          # both branches exercised
    f = laser_frame(fr["T"])
    o = OracleMap(200, 0.1, compat_box_filter=False)
    g.add(x, c, f); g.sync()
    o.add(xo, co, f)
    assert_layers_equal(g, o, what="colourised cloud fused")


def test_pcl_record_ingest():
    fr = synth.hdl64_frame(4)
    n = fr["xyzi"].shape[0]
    rec = np.zeros((n, 8), np.float32)
    rec[:, 0:3] = fr["xyzi"][:, :3]
    bgra = (fr["rgba"][:, 2].astype(np.uint32) | (fr["rgba"][:, 1].astype(np.uint32) << 8) |
            (fr["rgba"][:, 0].astype(np.uint32) << 16))
    rec[:, 4] = bgra.view(np.float32)
    rec[:, 6] = fr["xyzi"][:, 3]
    f = laser_frame(fr["T"])
    g1 = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False)
    g2 = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False)
    g1.add_pcl(rec, f)
    g2.add(fr["xyzi"], fr["rgba"], f)
    assert_layers_equal(g1, g2, what="pcl ingest")


def test_export_layers_matches_show_masking():
    fr = synth.hdl64_frame(0)
    f = laser_frame(fr["T"])
    g, o = both(200, 0.1, compat_box_filter=False)
    for m in (g, o):
        m.move(fr["position"])
        m.add(fr["xyzi"], fr["rgba"], f)
    eo = o.export_layers()
    g.compute_features()
    eg = g.export_layers()
    for name in eo:
        a, b = eg[name], eo[name]
        assert a.flags["F_CONTIGUOUS"]
        same = (a == b) | (np.isnan(a) & np.isnan(b))
        assert same.all(), name


def test_orthomosaic_and_visual_cloud_match_show():
    """the other two products of ElevationMap::show (ElevationMap.cpp:112-125) after a scrolled multi-frame run:
    bgr8 orthomosaic byte for byte, visual cloud point for point in GridMapIterator order"""
    scene = synth.make_scene()
    g, o = both(256, 0.1, compat_box_filter=False)
    for k in range(4):
        fr = synth.hdl64_frame(k, scene=scene, speed=9.0)
        f = laser_frame(fr["T"])
        for m in (g, o):
            m.move(fr["position"])
            m.add(fr["xyzi"], fr["rgba"], f)
    assert tuple(o.state()[1]) != (0, 0)            # the window scrolled: start index is not trivial
    img_o, xyz_o, rgb_o = o.show()
    g.compute_features()
    img_g = g.export_orthomosaic()
    xyz_g, rgb_g, n = g.export_visual_points()
    assert n == xyz_o.shape[0] > 5000
    assert np.array_equal(img_g, img_o)
    assert (img_o.reshape(-1, 3).any(axis=1)).sum() > 5000
    assert np.array_equal(xyz_g.view(np.uint32), xyz_o.view(np.uint32))
    assert np.array_equal(rgb_g, rgb_o)
    # bounded capacity: the count is still the number of shown cells, the prefix is written
    xyz_c, rgb_c, n_c = g.export_visual_points(capacity=1000)
    assert n_c == n and xyz_c.shape[0] == 1000 and np.array_equal(xyz_c, xyz_g[:1000]) and np.array_equal(rgb_c, rgb_g[:1000])
    # odd map size (block-edge handling: L not a multiple of 32)
    g2, o2 = both(200, 0.1, compat_box_filter=False)
    fr = synth.hdl64_frame(0, scene=scene)
    for m in (g2, o2):
        m.move(fr["position"])
        m.add(fr["xyzi"], fr["rgba"], laser_frame(fr["T"]))
    img_o, xyz_o, rgb_o = o2.show()
    g2.compute_features()
    assert np.array_equal(g2.export_orthomosaic(), img_o)
    xyz_g, rgb_g, n = g2.export_visual_points()
    assert n == xyz_o.shape[0] and np.array_equal(xyz_g.view(np.uint32), xyz_o.view(np.uint32)) and np.array_equal(rgb_g, rgb_o)


def test_scroll_out_harvest_matches_node_loop():
    """gem_snapshot_shown + gem_harvest_scrolled_out against the L-shape loop of ElevationMapping.cpp:716-765 over a
    driving sequence (diagonal, axis-aligned and zero shifts), with the node's double resolution"""
    scene = synth.make_scene()
    L, res = 256, 0.1
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=0.1)
    o = OracleMap(L, res, compat_box_filter=False)
    steps = [(0.0, 0.0), (0.9, 0.5), (1.0, 0.0), (0.0, -0.8), (-0.7, 0.6), (0.0, 0.0), (-1.1, -0.4), (0.8, -0.9)]
    pos = np.array([0.3, -0.2, 1.7], np.float32)
    total = 0
    for k, (dx, dy) in enumerate(steps):
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([dx, dy, 0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        f = laser_frame(T)
        cg, sg, shg = g.move(pos)
        co, so, sho = o.move(pos)
        assert np.array_equal(cg, co) and np.array_equal(shg, sho)
        if k > 0:
            rec_g, n_g = g.harvest_scrolled_out(cg, shg)
            rec_o, n_o = o.harvest_scrolled_out(co, sho, grid_res=0.1)
            assert n_g == n_o, (k, n_g, n_o)
            assert np.array_equal(rec_g.view(np.uint32), rec_o.view(np.uint32)), k
            if dx == 0 and dy == 0:
                assert n_g == 0
            total += n_g
            rec_c, n_c = g.harvest_scrolled_out(cg, shg, capacity=7)
            assert n_c == n_g and np.array_equal(rec_c.view(np.uint32), rec_g[:7].view(np.uint32))
        for m in (g, o):
            m.add(fr["xyzi"], fr["rgba"], f)
            m.compute_features()
            m.snapshot_shown()          # prevMap_ = visualMap_ (before the ray clean-up, :421-422)
            m.raytracing()
    assert total > 1000
    with pytest.raises(gem_b200.GemError):
        gem_b200.ElevationMap(64, 0.1).harvest_scrolled_out([0, 0], [1, 0])   # no snapshot yet


def test_opt_move_closeloop_var_update():
    c = synth.random_cloud(20000, seed=2, extent=6.0)
    f = laser_frame(np.eye(4))
    g, o = both(128, 0.1, compat_box_filter=False)
    for m in (g, o):
        m.add(c["xyzi"], c["rgba"], f)
        m.var_update(0.002)
        a = m.opt_move([0.33, -0.48], 0.05)
        m.closeloop([1.02, 0.51], -0.02)
        m.add(c["xyzi"][:5000], c["rgba"][:5000], f)
        m.var_update(-0.0015)
        m.add(c["xyzi"][5000:7000], c["rgba"][5000:7000], f)
    assert_layers_equal(g, o, what="optmove/closeloop/var_update")
    assert np.array_equal(g.state()[0], o.state()[0])


def test_headline_config_properties_c2():
    """BASELINE config 2 at full size (1024x1024 @ 0.05 m): oracle comparison on 3 frames plus
    size-independent properties: permutation across cells is invariant, idempotent re-export."""
    scene = synth.make_scene()
    g, o = both(1024, 0.05, compat_box_filter=False)
    for k in range(3):
        fr = synth.hdl64_frame(k, scene=scene)
        f = laser_frame(fr["T"])
        for m in (g, o):
            m.move(fr["position"])
            m.add(fr["xyzi"], fr["rgba"], f)
    assert_layers_equal(g, o, what="c2")
    # permutation that keeps the relative order inside every cell must not change anything
    fr = synth.hdl64_frame(3, scene=scene)
    f = laser_frame(fr["T"])
    g2 = gem_b200.ElevationMap(1024, 0.05, compat_box_filter=False)
    g3 = gem_b200.ElevationMap(1024, 0.05, compat_box_filter=False)
    g2.move(fr["position"]); g3.move(fr["position"])
    x, y, z = (fr["xyzi"][:, k].copy() for k in range(3))
    key = g2.process_points(x, y, z, f)[0]
    g2.raytracing()  # reset lowest, the dry run above touched it
    perm = np.argsort(key, kind="stable")  # groups cells together, stable inside each cell
    g2.add(fr["xyzi"], fr["rgba"], f)
    g3.add(np.ascontiguousarray(fr["xyzi"][perm]), np.ascontiguousarray(fr["rgba"][perm]), f)
    assert_layers_equal(g2, g3, ["elevation", "variance", "intensity", "color_r", "color_g", "color_b"], what="perm")


def test_large_grid_4096_config4_size():
    """BASELINE config 4 map size (4096x4096 @ 0.05 m) on one GPU: oracle parity on a frame, plus
    size-independent properties (empty add is idempotent, export round-trips through set_layer)"""
    L, res = 4096, 0.05
    fr = synth.hdl64_frame(7)
    f = laser_frame(fr["T"])
    g, o = both(L, res, compat_box_filter=False)
    for m in (g, o):
        m.move(fr["position"])
        m.add(fr["xyzi"], fr["rgba"], f)
    assert_layers_equal(g, o, what="4096^2")
    before = {n: g.get_layer(n) for n in ("elevation", "variance", "intensity", "color_r", "lowest")}
    g.add(np.zeros((0, 4), np.float32), None, f, n=0)           # empty cloud: nothing may change
    for n, a in before.items():
        assert np.array_equal(a.view(np.uint32) if a.dtype.kind == "f" else a, (g.get_layer(n).view(np.uint32) if a.dtype.kind == "f" else g.get_layer(n))), n
    # checkpoint / restore (the dead G_get_mapinfo / G_set_mapinfo of gpu.cu:457-475)
    g2 = gem_b200.ElevationMap(L, res, compat_box_filter=False)
    g2.move(fr["position"])
    for n in ("elevation", "variance", "intensity", "color_r", "color_g", "color_b", "traver", "lowest"):
        g2.set_layer(n, g.get_layer(n))
    fr2 = synth.hdl64_frame(8)
    f2 = laser_frame(fr2["T"])
    for m in (g, g2, o):
        m.move(fr2["position"])
        m.add(fr2["xyzi"], fr2["rgba"], f2)
    assert_layers_equal(g, g2, what="restored map continues identically")
    assert_layers_equal(g, o, what="4096^2 second frame")


def test_c5_size_8192_frame_and_multi_sensor_vs_oracle():
    """BASELINE config 5 map size (8192x8192 @ 0.05 m, 2.1 GB of cells) on one GPU: one frame against the oracle, then
    gem_add_points_multi (8 sensors on the SURVEY rig, one launch) against the oracle fed the same eight clouds.  The
    fused layers of the multi call equal eight sequential adds; `lowest` is one call's minimum (ORACLE DEFINITION,
    DESIGN.md section 5) and is checked against a numpy evaluation of that definition from the oracle's per-point outputs."""
    import torch
    from gem_b200 import tiled
    L, res = 8192, 0.05
    fr = synth.hdl64_frame(3)
    f = laser_frame(fr["T"])
    g, o = both(L, res, compat_box_filter=False)
    for m in (g, o):
        m.add(fr["xyzi"], fr["rgba"], f)
    assert_layers_equal(g, o, what="8192^2 one frame")
    scene = synth.make_scene()
    frs = [synth.hdl64_frame(20 + k, scene=scene) for k in range(8)]
    fobj = []
    for k, fr8 in enumerate(frs):
        T = fr8["T"].copy()
        T[0, 3], T[1, 3] = tiled.sensor_offset(k, 8)
        fobj.append(laser_frame(T))
    x = torch.from_numpy(np.concatenate([q["xyzi"] for q in frs])).cuda()
    c = torch.from_numpy(np.concatenate([q["rgba"] for q in frs])).cuda()
    off = np.concatenate([[0], np.cumsum([q["xyzi"].shape[0] for q in frs])])
    torch.cuda.synchronize()
    low0 = o.get_layer("lowest").reshape(-1).copy()
    g.add_multi(x, c, off, fobj)
    keys, hs, hvs = [], [], []
    for q, fq in zip(frs, fobj):   # oracle: the same clouds in order (per-cell order = global point index)
        key, var, _, _, zt = o.process_points(q["xyzi"][:, 0], q["xyzi"][:, 1], q["xyzi"][:, 2], fq)
        R, G, B = (q["rgba"][:, k].astype(np.int32) for k in range(3))
        o.fuse_points(key, R, G, B, q["xyzi"][:, 3], zt, var)
        keys.append(key); hs.append(zt); hvs.append(var)
    assert_layers_equal(g, o, ["elevation", "variance", "intensity", "color_r", "color_g", "color_b"], what="8192^2 multi-sensor")
    assert g.stats()["points_in"] == int(off[-1])
    # lowest of ONE call over all eight clouds (start index is 0: storage key == geographic index)
    key, h, hv = np.concatenate(keys), np.concatenate(hs), np.concatenate(hvs)
    ok = key >= 0
    key, h, hv = key[ok], h[ok], hv[ok]
    order = np.lexsort((np.arange(key.size), h, key))       # per cell: lowest height first, first index among equals
    first = np.ones(key.size, bool)
    first[1:] = key[order][1:] != key[order][:-1]
    ck, cm, cv = key[order][first], h[order][first], hv[order][first]
    expect = low0.copy()
    upd = cm <= low0[ck]
    expect[ck[upd]] = (cm[upd] + np.float32(3.0) * cv[upd]).astype(np.float32)
    got = g.get_layer("lowest").reshape(-1)
    assert np.array_equal(got.view(np.uint32), expect.view(np.uint32)), int((got != expect).sum())


def test_loop_closure_submap_refusion_matches_oracle():
    """SURVEY 8f row 4 (ElevationMapping.cpp:773-905): five overlapping submaps harvested as PointXYZRGBICT records, rigid
    re-transform + pairwise cell-hash re-fusion on the device vs the oracle twin, both precedence modes; plus the
    properties that hold at any size: one point per cell afterwards, positions on cell centres, idempotent second pass
    for cells whose old variance left (0, 1)"""
    import torch
    import oracle_lib
    from gem_b200 import submaps as sm
    rng = np.random.default_rng(5)
    res = 0.1

    class OracleBackend:
        def transform_cloud(self, pts, T):
            pts[:] = oracle_lib.transform_cloud(pts, T)

        def refuse_submaps(self, new, old, resolution, compat):
            n2, o2, fused = oracle_lib.refuse_submaps(new, old, resolution, compat)
            new[:n2.shape[0]] = n2
            old[:o2.shape[0]] = o2
            return n2.shape[0], o2.shape[0], fused

    def make_submap(cx, cy, n):
        p = np.zeros((n, 8), np.float32)
        p[:, 0] = cx + rng.uniform(-6, 6, n); p[:, 1] = cy + rng.uniform(-6, 6, n)
        p[:, 2] = rng.uniform(-1, 1, n); p[:, 3] = 1.0
        p[:, 4] = rng.integers(1, 1 << 24, n).astype(np.uint32).view(np.float32)
        p[:, 5] = rng.choice([0.05, 0.3, 0.9, 1.2, 0.0, -0.1], n).astype(np.float32)
        p[:, 6] = rng.integers(1, 255, n); p[:, 7] = rng.uniform(0, 1, n)
        p[rng.integers(0, n, 5), 0] = np.nan          # a few broken points: they equal nothing and are kept
        return p
    centres = [(0.0, 0.0), (4.0, 1.0), (-3.0, 2.0), (2.0, -5.0), (60.0, 60.0)]   # the last one has no neighbour
    base = [make_submap(cx, cy, 40000) for cx, cy in centres]
    yaw = lambda a, x, y: np.array([[np.cos(a), -np.sin(a), 0, x], [np.sin(a), np.cos(a), 0, y], [0, 0, 1, 0.02], [0, 0, 0, 1]], np.float32)
    old_poses = [yaw(0.1 * k, c[0], c[1]) for k, c in enumerate(centres)]
    new_poses = [yaw(0.1 * k + 0.01, c[0] + 0.07, c[1] - 0.04) for k, c in enumerate(centres)]
    g = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)
    for compat in (True, False):
        ora = [b.copy() for b in base]
        dev = [torch.from_numpy(b.copy()).cuda() for b in base]
        ora, fo = sm.update_global_map(OracleBackend(), ora, old_poses, new_poses, centres, res, 25.0, compat)
        dev, fd = sm.update_global_map(g, dev, old_poses, new_poses, centres, res, 25.0, compat)
        assert fo == fd and fo > 1000
        for k in range(len(base)):
            a, b = dev[k].cpu().numpy(), ora[k]
            assert a.shape == b.shape, (k, a.shape, b.shape)
            same = a.view(np.uint32) == b.view(np.uint32)
            same[:, :3] |= np.isnan(a[:, :3]) & np.isnan(b[:, :3])     # broken points: NaN payload bits differ between x86 and the GPU
            assert same.all(), (compat, k, int((~same).sum()))
        k0 = dev[0].cpu().numpy()
        ok = ~np.isnan(k0[:, 0])
        cells = np.round((k0[ok, :2] + res / 2) / res).astype(np.int64)
        assert np.unique(cells, axis=0).shape[0] == cells.shape[0]                 # one point per cell
        assert np.abs((k0[ok, :2] + res / 2) / res - cells).max() < 1e-3           # on cell centres
        assert base[4].shape[0] == dev[4].shape[0]                                  # no neighbour: untouched (not even hashed)


def test_error_paths_return_codes():
    import ctypes as C
    from gem_b200 import _lib
    lib = _lib.load()
    g = gem_b200.ElevationMap(64, 0.1)
    f = laser_frame(np.eye(4))
    assert lib.gem_add_points(g.handle, None, None, 5, C.byref(f)) == 1            # null cloud
    assert b"bad argument" in lib.gem_last_error(g.handle)
    assert lib.gem_add_points(g.handle, None, None, -1, C.byref(f)) == 1
    assert lib.gem_get_layer(g.handle, 99, None) == 1
    assert lib.gem_add_points_multi(g.handle, None, None, 0, None, None) == 1
    t = gem_b200.ElevationMap(64, 0.1, tile=(0, 64, 0, 32))
    with pytest.raises(gem_b200.GemError):
        t.compute_features()                                                         # tiled handles: not implemented
    with pytest.raises(gem_b200.GemError):
        gem_b200.ElevationMap(64, 0.1, tile=(0, 64, 40, 32))                        # tile outside the map
    big = np.zeros((1000, 4), np.float32)
    g3 = gem_b200.ElevationMap(64, 0.1, max_points=4)          # raised internally to nc/32+1 = 129
    with pytest.raises(gem_b200.GemError):
        import torch
        x = torch.from_numpy(big).cuda()
        g3.add_stream_fast(C.c_void_p(x.data_ptr()), None, 1000, C.byref(f))        # n > max_points in stream mode
    g3.add(big, None, f)                                                             # chunked path copes
