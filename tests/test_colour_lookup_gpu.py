"""The node's colour lookup on the device (GEM_COLOUR_LOOKUP_NODE, DESIGN.md f19): gem_colourise_points byte for byte
against the literal oracle (tests/orc_colour_lookup.c) on every crafted case and on the two measured clouds, IMAGE mode
as before, gem_add_pointcloud2_host_async in NODE mode against the oracle chain decode -> orc_colourise_node -> fuse for
every accepted encoding, refusals, and the C++ facade."""
import ctypes as C
import subprocess

import numpy as np
import pytest
import torch

import colour_lookup_cases as cc
import colour_lookup_oracle as clo
import gem_b200
import native
import oracle_lib
import pc2_cases as pc
import pc2_oracle
import sensor_models_oracle as smo
from gem_b200 import CameraImage, PointCloud2Layout, _lib, synth
from helpers import assert_layers_equal
from oracle_lib import OracleMap

pytestmark = pytest.mark.gpu
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def emap():
    return gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)


def colourise(m, c, mode=None):
    """gem_colourise_points in `mode` (None: the handle's) on the case's cloud and its image with its row stride; checks
    the image is not written.  Returns (xyzi, rgba) on the host."""
    if mode is not None:
        m.set_colour_lookup(mode)
    n = c["xyzi"].shape[0]
    x = torch.from_numpy(c["xyzi"]).cuda()
    img = torch.from_numpy(c["img"]).cuda()
    out = torch.full((max(n, 1), 4), SENTINEL, dtype=torch.uint8, device="cuda:0")
    tc = (C.c_double * 12)(*np.asarray(c["T_camera"], np.float64).reshape(-1))
    tl = (C.c_double * 16)(*np.asarray(c["T_lidar"], np.float64).reshape(-1))
    torch.cuda.synchronize()
    rc = _lib.load().gem_colourise_points(m.handle, C.c_void_p(x.data_ptr()), n, tc, tl, C.c_void_p(img.data_ptr()),
                                          c["width"], c["height"], c["row_stride"], C.c_void_p(out.data_ptr()))
    assert rc == 0, _lib.load().gem_last_error(m.handle)
    m.sync()
    assert np.array_equal(img.cpu().numpy(), c["img"])
    return x.cpu().numpy(), out[:n].cpu().numpy()


def same(got, want, what):
    (xg, cg), (xw, cw) = got, want
    assert xg.tobytes() == xw.tobytes(), what
    if not np.array_equal(cg, cw):
        bad = np.flatnonzero((cg != cw).any(axis=1))
        raise AssertionError((what, int(bad.size), int(bad[0]), cg[bad[0]], cw[bad[0]]))


def image_oracle(c):
    img = np.ascontiguousarray(c["img"][:, :3 * c["width"]]).reshape(c["height"], c["width"], 3)
    return oracle_lib.colourise(c["xyzi"], c["T_camera"], c["T_lidar"], img)


@pytest.mark.parametrize("name", cc.case_names())
def test_node_matches_oracle(emap, name):
    c = cc.case_by_name(name)
    same(colourise(emap, c, "node"), clo.node(c["xyzi"], c["T_camera"], c["T_lidar"], c["img"], c["width"]), name)


@pytest.mark.parametrize("cloud", ["d435", "lidar_008"])
def test_measured_clouds(emap, cloud):
    c = cc.d435() if cloud == "d435" else cc.lidar_008()
    node = colourise(emap, c, "node")
    same(node, clo.node(c["xyzi"], c["T_camera"], c["T_lidar"], c["img"], c["width"]), cloud)
    image = colourise(emap, c, "image")
    same(image, image_oracle(c), (cloud, "image"))
    differs = int((node[1] != image[1]).any(axis=1).sum())
    assert differs > 20_000, differs


@pytest.mark.parametrize("name", ["organised", "alternating", "invalid_interleaved", "padded_stride_5", "tiny_3x3"])
def test_image_mode_unchanged(name):
    """a new handle reads the unmodified image, and so does one switched to NODE and back"""
    c = cc.case_by_name(name)
    m = gem_b200.ElevationMap(32, 0.1, compat_box_filter=False)
    img = np.ascontiguousarray(c["img"][:, :3 * c["width"]]).reshape(c["height"], c["width"], 3)
    x = torch.from_numpy(c["xyzi"]).cuda()
    out = torch.zeros((c["xyzi"].shape[0], 4), dtype=torch.uint8, device="cuda:0")
    m.colourise(x, c["T_camera"], c["T_lidar"], torch.from_numpy(img).cuda(), out)   # the default mode
    m.sync()
    want = image_oracle(c)
    same((x.cpu().numpy(), out.cpu().numpy()), want, (name, "default"))
    colourise(m, c, "node")
    same(colourise(m, c, "image"), want, (name, "back to image"))


def test_mode_refusals_and_bad_arguments(emap):
    lib, h = _lib.load(), emap.handle
    c = cc.case_by_name("alternating")
    want = clo.node(c["xyzi"], c["T_camera"], c["T_lidar"], c["img"], c["width"])
    emap.set_colour_lookup("node")
    for bad in (2, -1, 7, 1 << 30):
        assert lib.gem_set_colour_lookup(h, bad) == 1
    assert lib.gem_set_colour_lookup(None, 1) == 1
    with pytest.raises(ValueError):
        emap.set_colour_lookup("painted")
    same(colourise(emap, c), want, "mode kept")
    # refused colourise calls write nothing, in NODE mode too
    n = c["xyzi"].shape[0]
    x = torch.from_numpy(c["xyzi"]).cuda()
    img = torch.from_numpy(c["img"]).cuda()
    out = torch.full((n, 4), SENTINEL, dtype=torch.uint8, device="cuda:0")
    tc = (C.c_double * 12)(*np.asarray(c["T_camera"], np.float64).reshape(-1))
    tl = (C.c_double * 16)(*np.asarray(c["T_lidar"], np.float64).reshape(-1))
    xp, ip, op = C.c_void_p(x.data_ptr()), C.c_void_p(img.data_ptr()), C.c_void_p(out.data_ptr())
    W, H, S = c["width"], c["height"], c["row_stride"]
    for args in [(xp, -1, tc, tl, ip, W, H, S, op), (None, n, tc, tl, ip, W, H, S, op), (xp, n, tc, tl, ip, W, H, S, None),
                 (xp, n, tc, tl, None, W, H, S, op), (xp, n, tc, tl, ip, 0, H, S, op), (xp, n, tc, tl, ip, W, 0, S, op),
                 (xp, n, tc, tl, ip, W, H, 3 * W - 1, op), (xp, n, None, tl, ip, W, H, S, op)]:
        assert lib.gem_colourise_points(h, *args) == 1
    emap.sync()
    assert (out == SENTINEL).all() and np.array_equal(x.cpu().numpy(), c["xyzi"])


def test_tiled_handle_accepted():
    m = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False, tile=(0, 32, 0, 32))
    c = cc.case_by_name("organised_columns")
    same(colourise(m, c, "node"), clo.node(c["xyzi"], c["T_camera"], c["T_lidar"], c["img"], c["width"]), "tiled")


def test_scratch_grows_and_shrinking_calls_reuse_it(emap):
    """calls alternating between large and small clouds on one handle (the scratch grows once, never shrinks)"""
    for name in ("pair_horizontal", "patch_3x3_1e6", "organised", "tiny_2x2", "patch_3x3_1e6"):
        c = cc.case_by_name(name)
        same(colourise(emap, c, "node"), clo.node(c["xyzi"], c["T_camera"], c["T_lidar"], c["img"], c["width"]), name)


# ---- gem_add_pointcloud2_host_async in NODE mode ------------------------------------------------------------------------
SEQUENCES = {
    # name: (cloud, encoding, pinned, interleave)
    "d435_bgr8_pinned": ("d435", "bgr8", True, False),
    "d435_rgb8_pageable": ("d435", "rgb8", False, False),
    "d435_bgra8_pinned_interleaved": ("d435", "bgra8", True, True),
    "d435_rgba8_pageable_interleaved": ("d435", "rgba8", False, True),
    "d435_mono8_pinned": ("d435", "mono8", True, False),
    "lidar_008_bgr8_pageable": ("lidar", "bgr8", False, False),
    "lidar_008_rgb8_pinned_interleaved": ("lidar", "rgb8", True, True),
}


def np_bgr(img, enc, width):
    """cv_bridge's conversion as a numpy permutation of an (H, step) uint8 image"""
    ch = _lib.IMAGE_ENCODINGS[enc]
    px = img[:, :width * ch].reshape(img.shape[0], width, ch)
    if enc == "mono8":
        return np.repeat(px, 3, axis=2)
    if enc in ("rgb8", "rgba8"):
        return px[..., [2, 1, 0]].copy()
    return px[..., :3].copy()


@pytest.mark.parametrize("name", list(SEQUENCES))
def test_pointcloud2_sequence(name):
    cloud, enc, pinned, interleave = SEQUENCES[name]
    depth = cloud == "d435"
    L_map, res = (120, 0.05) if depth else (200, 0.1)
    g = gem_b200.ElevationMap(L_map, res, compat_box_filter=False)
    ref = gem_b200.ElevationMap(L_map, res, compat_box_filter=False)   # IMAGE mode: the maps must differ
    o = OracleMap(L_map, res, compat_box_filter=False)
    g.set_colour_lookup("node")
    sp = gem_b200.StructuredLightSensorProcessor() if depth else gem_b200.LaserSensorProcessor()
    keep = []
    for k in range(3):
        c = cc.d435(k) if depth else cc.lidar_008(k)
        T, pos = (synth.d435_pose(k) if depth else synth.hdl64_pose(k))
        f = gem_b200.make_frame(T, sp)
        W, H = c["width"], c["height"]
        case = pc.from_xyzi("f", "xyzir32", c["xyzi"], width=640 if depth else None, height=480 if depth else 1,
                            row_pad=32 if k % 2 else 0, seed=300 + k)
        lay = PointCloud2Layout(case["fields"], case["width"], case["height"], case["point_step"], case["row_step"],
                                case["is_bigendian"])
        step = _lib.IMAGE_ENCODINGS[enc] * W + 3 * k
        img = np.random.default_rng(400 + k).integers(0, 256, (H, step)).astype(np.uint8)
        bgr = np_bgr(img, enc, W).reshape(H, 3 * W)
        for m in (g, ref, o):
            m.move(pos)
        x_o, c_o = clo.node(pc2_oracle.xyzi(pc2_oracle.decode(case)[0]), c["T_camera"], c["T_lidar"], bgr, W)
        if interleave and k == 1:
            hx, hc = torch.from_numpy(x_o).pin_memory(), torch.from_numpy(c_o).pin_memory()
            keep.append((hx, hc))
            g.add_host_async_fast(C.c_void_p(hx.data_ptr()), C.c_void_p(hc.data_ptr()), x_o.shape[0], C.byref(f))
        else:
            if pinned:
                data, im = torch.from_numpy(case["data"]).pin_memory(), torch.from_numpy(img).pin_memory()
                keep.append((data, im))
            else:
                data, im = case["data"].copy(), img.copy()
            g.add_pointcloud2_host_async(lay, data, f, CameraImage(c["T_camera"], c["T_lidar"], enc, im, W, H, step))
            if not pinned:   # pageable buffers may be reused as soon as the call returns
                data[:] = 0xAB
                im[:] = 0x5C
        ref.add_pointcloud2_host_async(lay, case["data"], f, CameraImage(c["T_camera"], c["T_lidar"], enc, img, W, H, step))
        smo.add(o, x_o, c_o, f)
    g.sync()
    ref.sync()
    assert_layers_equal(g, o, what=(name, "oracle"))
    assert (g.get_layer("color_r") != 0).sum() > 100
    assert not np.array_equal(g.get_layer("color_r"), ref.get_layer("color_r"))


def test_pointcloud2_refusals_change_nothing():
    g = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False, max_points=2000)
    g.set_colour_lookup("node")
    fr = synth.hdl64_frame(0)
    f = gem_b200.make_frame(fr["T"], gem_b200.LaserSensorProcessor())
    g.move(fr["position"])
    ok = pc.from_xyzi("ok", "xyzir32", fr["xyzi"][:2000], seed=1)
    L = PointCloud2Layout(ok["fields"], ok["width"], ok["height"], ok["point_step"], ok["row_step"], ok["is_bigendian"])
    img = np.random.default_rng(1).integers(0, 256, (376, 3 * 1241)).astype(np.uint8)
    cam = CameraImage(cc.TC_KITTI, cc.TL_KITTI, "bgr8", img, 1241, 376, 3 * 1241)
    g.add_pointcloud2_host_async(L, ok["data"], f, cam)
    g.sync()
    before = {n: g.get_layer(n).copy() for n in ("elevation", "variance", "intensity", "color_r", "lowest")}
    big = pc.from_xyzi("big", "xyzir32", fr["xyzi"][:2001], seed=2)
    Lbig = PointCloud2Layout(big["fields"], big["width"], big["height"], big["point_step"], big["row_step"], big["is_bigendian"])
    bad_cam = CameraImage(cc.TC_KITTI, cc.TL_KITTI, "bgr8", img, 1241, 376, 3 * 1241)
    bad_cam.c.encoding = b"bgr16"
    short_cam = CameraImage(cc.TC_KITTI, cc.TL_KITTI, "bgr8", img, 1241, 376, 3 * 1241)
    short_cam.c.step = 3 * 1241 - 1
    lib, h = _lib.load(), g.handle
    dp, nb = C.c_void_p(ok["data"].ctypes.data), ok["data"].nbytes
    for k, args in enumerate([(C.byref(Lbig.c), C.c_void_p(big["data"].ctypes.data), big["data"].nbytes, C.byref(cam.c), C.byref(f)),
                              (C.byref(L.c), dp, nb - 1, C.byref(cam.c), C.byref(f)),
                              (C.byref(L.c), dp, nb, C.byref(bad_cam.c), C.byref(f)),
                              (C.byref(L.c), dp, nb, C.byref(short_cam.c), C.byref(f))]):
        assert lib.gem_add_pointcloud2_host_async(h, *args) == 1, k
    g.sync()
    for n, a in before.items():
        assert np.array_equal(g.get_layer(n).view(np.uint32), a.view(np.uint32)), n


def test_cxx_facade_program(tmp_path):
    exe = native.facade_program("colour_lookup_smoke", tmp_path)
    c = cc.lidar_008()
    T, pos = synth.hdl64_pose(0)
    W, H = c["width"], c["height"]
    bgr = np.ascontiguousarray(c["img"][:, :3 * W])
    n = c["xyzi"].shape[0]
    blob = (np.asarray(T, np.float64).tobytes() + np.asarray(c["T_camera"], np.float64).tobytes()
            + np.asarray(c["T_lidar"], np.float64).tobytes() + np.asarray(pos, np.float32).tobytes()
            + np.int32(n).tobytes() + c["xyzi"].tobytes() + np.array([W, H], np.int32).tobytes() + bgr.tobytes())
    (tmp_path / "in.bin").write_bytes(blob)
    prefix = str(tmp_path / "cxx")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), prefix], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "colour lookup ok" in r.stdout, (r.returncode, r.stdout, r.stderr)
    got = np.fromfile(prefix + ".layers.bin", np.float32).reshape(9, 200, 200)
    o = OracleMap(200, 0.1, compat_box_filter=False)
    o.move(pos)
    x_o, c_o = clo.node(c["xyzi"], c["T_camera"], c["T_lidar"], c["img"], W)
    f = gem_b200.make_frame(T, gem_b200.LaserSensorProcessor())
    smo.add(o, x_o, c_o, f)
    want = o.export_layers()
    for k, name in enumerate(["elevation", "variance", "rough", "slope", "traver", "color_r", "color_g", "color_b", "intensity"]):
        if name in ("elevation", "color_r", "color_g", "color_b", "intensity"):
            w = np.asarray(want[name], np.float32).reshape(-1, order="F")   # grid_map's column-major layout
            assert np.array_equal(got[k].reshape(-1), w, equal_nan=True), name
    assert np.isfinite(got[5]).sum() > 100
