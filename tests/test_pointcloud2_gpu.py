"""The PointCloud2 ingest on the device (DESIGN.md f12): gem_decode_pointcloud2 bit for bit against the oracle
(tests/orc_pointcloud2.c) on every crafted case of tests/pc2_cases.py, also from misaligned addresses; gem_image_to_bgr8
against a numpy permutation for each encoding with padded rows; sequences of gem_add_pointcloud2_host_async (scrolls,
every sensor model, no image and each encoding, pinned and pageable buffers, interleaved with gem_add_points_host_async)
against the oracle chain decode -> colourise -> fuse and against the device chain decode -> gem_colourise_points ->
gem_add_points_stream; refusals leave the map unchanged."""
import ctypes as C

import numpy as np
import pytest
import torch

import gem_b200
import oracle_lib
import pc2_cases as pc
import pc2_oracle
import sensor_models_oracle as smo
from gem_b200 import CameraImage, GemError, PointCloud2Layout, _lib, synth
from helpers import assert_layers_equal
from oracle_lib import OracleMap

pytestmark = pytest.mark.gpu
SENTINEL = 0x7FBADBAD
TC = np.array([[718.856, 0, 607.1928, 0], [0, 718.856, 185.2157, 0], [0, 0, 1, 0]], np.float64)
TL = np.array([[0, -1, 0, 0.0], [0, 0, -1, -0.08], [1, 0, 0, -0.27], [0, 0, 0, 1]], np.float64)
TL_D435 = np.eye(4)   # the depth camera's optical frame is the colour camera's
TC_D435 = np.array([[385.0, 0, 320.0, 0], [0, 385.0, 240.0, 0], [0, 0, 1, 0]], np.float64)


@pytest.fixture(scope="module")
def emap():
    return gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)


def layout(case):
    return PointCloud2Layout(case["fields"], case["width"], case["height"], case["point_step"], case["row_step"],
                             case["is_bigendian"])


def on_device(data, shift):
    """the message bytes at `shift` bytes past a 256-byte aligned allocation"""
    buf = torch.zeros(data.nbytes + shift + 16, dtype=torch.uint8, device="cuda:0")
    buf[shift:shift + data.nbytes] = torch.from_numpy(np.ascontiguousarray(data))
    return buf[shift:shift + data.nbytes]


@pytest.mark.parametrize("name", pc.case_names())
def test_decode_matches_oracle(emap, name):
    case = pc.case_by_name(name)
    L = layout(case)
    n = case["width"] * case["height"]
    want = pc2_oracle.decode(case)
    for shift in (0, 1, 6, 13):
        data = on_device(case["data"], shift)
        out = torch.full((max(n, 1), 4), 0, dtype=torch.int32, device="cuda:0").fill_(SENTINEL).view(torch.float32)
        nb = case.get("data_bytes", case["data"].nbytes)
        if case["refused"]:
            assert want is None
            with pytest.raises(GemError):
                emap.decode_pointcloud2(L, data, out, data_bytes=nb)
            emap.sync()
            assert (out.view(torch.int32) == SENTINEL).all()
            continue
        emap.decode_pointcloud2(L, data, out[:n], data_bytes=nb)
        emap.sync()
        got = out[:n].cpu().numpy()
        exp = pc2_oracle.xyzi(want[0])
        if got.tobytes() != exp.tobytes():
            bad = np.flatnonzero((got.view(np.uint32) != exp.view(np.uint32)).any(axis=1))
            raise AssertionError((name, shift, int(bad.size), int(bad[0]), got[bad[0]].view(np.uint32), exp[bad[0]].view(np.uint32)))
        if n == 0:
            assert (out.view(torch.int32) == SENTINEL).all()


def test_decode_argument_errors(emap):
    case = pc.case_by_name("kitti16")
    L, data = layout(case), on_device(case["data"], 0)
    lib, h = _lib.load(), emap.handle
    out = torch.empty((case["width"] + 1, 4), dtype=torch.float32, device="cuda:0")
    nb = case["data"].nbytes
    assert lib.gem_decode_pointcloud2(h, C.byref(L.c), None, nb, C.c_void_p(out.data_ptr())) == 1
    assert lib.gem_decode_pointcloud2(h, C.byref(L.c), C.c_void_p(data.data_ptr()), nb, None) == 1
    assert lib.gem_decode_pointcloud2(h, None, C.c_void_p(data.data_ptr()), nb, C.c_void_p(out.data_ptr())) == 1
    assert lib.gem_decode_pointcloud2(h, C.byref(L.c), C.c_void_p(data.data_ptr()), nb, C.c_void_p(out.data_ptr() + 4)) == 1
    assert lib.gem_decode_pointcloud2(h, C.byref(L.c), C.c_void_p(data.data_ptr()), nb, C.c_void_p(data.data_ptr())) == 1


def np_bgr(img, enc, width):
    """cv_bridge's conversion as a numpy permutation of an (H, step) uint8 image"""
    ch = _lib.IMAGE_ENCODINGS[enc]
    px = img[:, :width * ch].reshape(img.shape[0], width, ch)
    if enc == "mono8":
        return np.repeat(px, 3, axis=2)
    if enc in ("rgb8", "rgba8"):
        return px[..., [2, 1, 0]].copy()
    return px[..., :3].copy()


def make_image(enc, W, H, pad, seed):
    step = _lib.IMAGE_ENCODINGS[enc] * W + pad
    return np.random.default_rng(seed).integers(0, 256, (H, step)).astype(np.uint8), step


@pytest.mark.parametrize("enc", list(_lib.IMAGE_ENCODINGS))
def test_image_to_bgr8(emap, enc):
    W, H = 641, 37
    img, step = make_image(enc, W, H, 7, 3)
    src = torch.from_numpy(img).cuda()
    out = torch.full((H, 3 * W + 5), 77, dtype=torch.uint8, device="cuda:0")
    emap.image_to_bgr8(enc, src, W, H, step, out, dst_step=3 * W + 5)
    emap.sync()
    o = out.cpu().numpy()
    assert np.array_equal(o[:, :3 * W].reshape(H, W, 3), np_bgr(img, enc, W))
    assert (o[:, 3 * W:] == 77).all()


@pytest.mark.parametrize("enc", ["bgr16", "bayer_rggb8", "16UC1", "BGR8", "8UC3", ""])
def test_image_other_encodings_refused(emap, enc):
    src = torch.zeros((4, 12), dtype=torch.uint8, device="cuda:0")
    out = torch.full((4, 12), 9, dtype=torch.uint8, device="cuda:0")
    with pytest.raises(GemError):
        emap.image_to_bgr8(enc, src, 4, 4, 12, out)
    emap.sync()
    assert (out == 9).all()


# ---- sequences of gem_add_pointcloud2_host_async ----------------------------------------------------------------------
SEQUENCES = {
    # name: (layout, sensor, encoding or None, pinned, interleave)
    "laser_xyzir32_bgr8_pinned": ("xyzir32", "laser", "bgr8", True, False),
    "laser_xyzir22_rgb8_pageable": ("xyzir22", "laser", "rgb8", False, False),
    "laser_pandarqt_bgra8_pinned": ("pandarqt", "laser", "bgra8", True, False),
    "laser_kitti16_rgba8_pageable": ("kitti16", "laser", "rgba8", False, False),
    "laser_kitti16_mono8_pinned": ("kitti16", "laser", "mono8", True, False),
    "laser_xyzrgbict_no_image_pageable": ("xyzrgbict", "laser", None, False, False),
    "laser_ouster_bgr8_pageable": ("ouster", "laser", "bgr8", False, False),
    "laser_xyzir32_rgb8_interleaved": ("xyzir32", "laser", "rgb8", True, True),
    "structured_d435_no_image_pinned": ("d435", "structured", None, True, False),
    "structured_d435_bgr8_pageable": ("d435", "structured", "bgr8", False, False),
    "stereo_d435_mono8_pinned": ("d435", "stereo", "mono8", True, False),
    "perfect_kitti16_rgb8_pageable": ("kitti16", "perfect", "rgb8", False, False),
}


def sensor(kind):
    if kind == "laser":
        return gem_b200.LaserSensorProcessor()
    if kind == "structured":
        return gem_b200.StructuredLightSensorProcessor()
    if kind == "stereo":
        return gem_b200.StereoSensorProcessor(p_1=0.01, p_2=0.002, p_3=0.001, p_4=0.3, p_5=0.0001, lateral_factor=0.01,
                                              depth_to_disparity_factor=40.0, cloud_width=640)
    return gem_b200.PerfectSensorProcessor()


@pytest.mark.parametrize("name", list(SEQUENCES))
def test_sequence(name):
    lay, kind, enc, pinned, interleave = SEQUENCES[name]
    depth = lay == "d435"
    L_map, res = (120, 0.05) if depth else (200, 0.1)
    g = gem_b200.ElevationMap(L_map, res, compat_box_filter=False)
    d = gem_b200.ElevationMap(L_map, res, compat_box_filter=False)
    o = OracleMap(L_map, res, compat_box_filter=False)
    sp = sensor(kind)
    keep, pinned_ring = [], []
    W, H = (640, 480) if depth else (1241, 376)
    Tc, Tl = (TC_D435, TL_D435) if depth else (TC, TL)
    for k in range(4):
        fr = synth.d435_frame(k) if depth else synth.hdl64_frame(k)
        f = gem_b200.make_frame(fr["T"], sp)
        if depth:
            case = pc.from_xyzi("f", lay, fr["xyzi"], width=640, height=480, row_pad=32 if k % 2 else 0, seed=100 + k,
                                rgb=fr["rgba"])
        else:
            case = pc.from_xyzi("f", lay, fr["xyzi"], seed=100 + k)
        L = layout(case)
        img, step = make_image(enc, W, H, 3 * k, 200 + k) if enc else (None, 0)
        for m in (g, d, o):
            m.move(fr["position"])
        # oracle chain
        x_o = pc2_oracle.xyzi(pc2_oracle.decode(case)[0])
        c_o = None
        if enc:
            x_o, c_o = oracle_lib.colourise(x_o, Tc, Tl, np_bgr(img, enc, W))
        # device chain: decode -> image_to_bgr8 -> gem_colourise_points -> gem_add_points_stream
        dd = torch.from_numpy(case["data"]).cuda()
        xd = d.decode_pointcloud2(L, dd)
        cd = bgr = di = None
        if enc:
            di = torch.from_numpy(img).cuda()
            bgr = d.image_to_bgr8(enc, di, W, H, step)
            cd = torch.zeros((xd.shape[0], 4), dtype=torch.uint8, device="cuda:0")
            torch.cuda.synchronize()
            d.colourise(xd, Tc, Tl, bgr, cd)
        keep.append((dd, xd, di, bgr, cd))   # the map's stream may still read them
        d.add_stream_fast(C.c_void_p(xd.data_ptr()), C.c_void_p(cd.data_ptr()) if enc else None, int(xd.shape[0]), C.byref(f))
        # the one call
        if interleave and k % 2:
            xyzi = np.ascontiguousarray(x_o)
            rgba = np.ascontiguousarray(c_o)
            hx, hc = torch.from_numpy(xyzi).pin_memory(), torch.from_numpy(rgba).pin_memory()
            pinned_ring.append((hx, hc))
            g.add_host_async_fast(C.c_void_p(hx.data_ptr()), C.c_void_p(hc.data_ptr()), xyzi.shape[0], C.byref(f))
        else:
            if pinned:
                data = torch.from_numpy(case["data"]).pin_memory()
                im = torch.from_numpy(img).pin_memory() if enc else None
                pinned_ring.append((data, im))
            else:
                data, im = case["data"].copy(), (img.copy() if enc else None)
            cam = CameraImage(Tc, Tl, enc, im, W, H, step) if enc else None
            g.add_pointcloud2_host_async(L, data, f, cam)
            if not pinned:   # pageable buffers may be reused as soon as the call returns
                data[:] = 0xAB
                if enc:
                    im[:] = 0x5C
        smo.add(o, x_o, c_o, f)   # every model (stereo reads each point's index in the cloud)
    g.sync()
    d.sync()
    assert_layers_equal(g, o, what=(name, "oracle"))
    assert_layers_equal(g, d, what=(name, "device chain"))
    sg, sd = g.stats(), d.stats()
    assert sg == sd, (sg, sd)
    assert sg["points_binned"] > 1000, sg
    if enc and lay not in ("ouster", "d435"):   # (no FLOAT32 intensity: 0, and the colour gate never passes)
        assert (g.get_layer("color_r") != 0).sum() > 100


def test_refusals_leave_the_map_unchanged():
    g = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False, max_points=2000)
    fr = synth.hdl64_frame(0)
    f = gem_b200.make_frame(fr["T"], gem_b200.LaserSensorProcessor())
    g.move(fr["position"])
    ok = pc.from_xyzi("ok", "xyzir32", fr["xyzi"][:2000], seed=1)
    g.add_pointcloud2_host_async(layout(ok), ok["data"], f)
    g.sync()
    before = {n: g.get_layer(n).copy() for n in ("elevation", "variance", "intensity", "lowest")}
    big = pc.from_xyzi("big", "xyzir32", fr["xyzi"][:2001], seed=2)
    img, step = make_image("bgr8", 1241, 376, 0, 1)
    lib, h = _lib.load(), g.handle
    L = layout(ok)
    cam = CameraImage(TC, TL, "bgr8", img, 1241, 376, step)
    bad_cam = CameraImage(TC, TL, "bgr8", img, 1241, 376, step)
    bad_cam.c.encoding = b"bgr16"
    short_cam = CameraImage(TC, TL, "bgr8", img, 1241, 376, step)
    short_cam.c.step = 3 * 1241 - 1
    dp = C.c_void_p(ok["data"].ctypes.data)
    nb = ok["data"].nbytes
    Lbig = layout(big)
    refused = {name: pc.case_by_name(name) for name in ("short_data", "short_row_step", "field_past_point_step",
                                                        "overlapping_fields", "bad_datatype")}
    Lref = {name: layout(case) for name, case in refused.items()}   # alive for the calls
    calls = [
        (C.byref(Lbig.c), C.c_void_p(big["data"].ctypes.data), big["data"].nbytes, None, C.byref(f)),   # n > max_points
        (None, dp, nb, None, C.byref(f)),
        (C.byref(L.c), None, nb, None, C.byref(f)),
        (C.byref(L.c), dp, nb, None, None),
        (C.byref(L.c), dp, nb - 1, None, C.byref(f)),
        (C.byref(L.c), dp, nb, C.byref(bad_cam.c), C.byref(f)),
        (C.byref(L.c), dp, nb, C.byref(short_cam.c), C.byref(f)),
    ]
    for name, case in refused.items():
        calls.append((C.byref(Lref[name].c), C.c_void_p(case["data"].ctypes.data), case.get("data_bytes", case["data"].nbytes),
                      None, C.byref(f)))
    for k, args in enumerate(calls):
        assert lib.gem_add_pointcloud2_host_async(h, *args) == 1, k
    g.sync()
    for n, a in before.items():
        assert np.array_equal(g.get_layer(n).view(np.uint32), a.view(np.uint32)), n
    g.add_pointcloud2_host_async(L, ok["data"], f, cam)   # the handle still works
    g.sync()
    assert g.stats()["points_in"] == 2000
