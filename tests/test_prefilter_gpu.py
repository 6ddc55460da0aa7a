"""The pre-filtered asynchronous add (DESIGN.md f20) on the device, bit for bit on every layer, gem_stats and the steps'
infos against the oracle chain (tests/orc_pointcloud2.c -> tests/orc_voxel_grid.c per step -> the colour oracle ->
OracleMap) and against the synchronous device chain (decode -> gem_voxel_grid per step -> gem_colourise_points ->
gem_add_points_stream): every crafted voxel case, raw HDL-64 frames under filter.launch and filter_kitti.launch with no
image, bgr8 and rgb8 images in both colour lookup modes and through both entry points, the PointCloud2 layouts,
sequences with a filtered count of 0, a raw frame of exactly max_points, staging growth and interleaved unfiltered calls,
the call returning while the handle's stream is still busy, and the C++ facade against the C ABI."""
import ctypes as C
import subprocess

import numpy as np
import pytest
import torch

import colour_lookup_oracle as clo
import gem_b200
import native
import oracle_lib
import pc2_cases as pc
import pc2_oracle
import voxel_cases as vc
import voxel_oracle
from gem_b200 import CameraImage, PointCloud2Layout, _lib, synth
from helpers import assert_layers_equal
from oracle_lib import OracleMap

pytestmark = pytest.mark.gpu
TC = np.array([[718.856, 0, 607.1928, 0], [0, 718.856, 185.2157, 0], [0, 0, 1, 0]], np.float64)
TL = np.array([[0, -1, 0, 0.0], [0, 0, -1, -0.08], [1, 0, 0, -0.27], [0, 0, 0, 1]], np.float64)
TC_D435 = np.array([[385.0, 0, 320.0, 0], [0, 385.0, 240.0, 0], [0, 0, 1, 0]], np.float64)
LAUNCHES = {"filter": voxel_oracle.FILTER_LAUNCH, "kitti": voxel_oracle.FILTER_KITTI_LAUNCH}


def layout(case):
    return PointCloud2Layout(case["fields"], case["width"], case["height"], case["point_step"], case["row_step"],
                             case["is_bigendian"])


def make_image(enc, W, H, seed):
    step = _lib.IMAGE_ENCODINGS[enc] * W
    return np.random.default_rng(seed).integers(0, 256, (H, step)).astype(np.uint8), step


def np_bgr(img, enc, W):
    px = img[:, :W * 3].reshape(img.shape[0], W, 3)
    return px[..., [2, 1, 0]].copy() if enc == "rgb8" else px.copy()


class Chains:
    """one map per path: g takes the new calls, d the synchronous device chain, o the oracle chain"""

    def __init__(self, L, res, mode="image", max_points=0):
        self.g = gem_b200.ElevationMap(L, res, compat_box_filter=False, max_points=max_points)
        self.d = gem_b200.ElevationMap(L, res, compat_box_filter=False, max_points=max_points)
        self.o = OracleMap(L, res, compat_box_filter=False)
        self.mode = mode
        for m in (self.g, self.d):
            m.set_colour_lookup(mode)
        self.keep = []
        self.last_count = 0

    def move(self, pos):
        for m in (self.g, self.d, self.o):
            m.move(pos)

    def reference(self, xyzi, steps, f, bgr=None, Tc=TC, Tl=TL):
        """the device chain on d and the oracle chain on o; returns the oracle's step infos"""
        x = np.ascontiguousarray(xyzi, np.float32)
        cur = torch.from_numpy(x).cuda()
        infos = []
        for leaf, field, limits, neg in steps:
            out = torch.empty_like(cur)
            cur, info = self.d.voxel_grid(cur, leaf, field, limits, neg, out=out)
            infos.append(info)
            self.keep.append(out)
        x_o, winfos = voxel_oracle.chain(x, steps) if steps else (x, [])
        assert infos == winfos, (infos, winfos)
        n = int(cur.shape[0])
        c_d = c_o = None
        if bgr is not None and n:
            W = bgr.shape[1]
            bgr_d = torch.from_numpy(np.ascontiguousarray(bgr)).cuda()
            c_d = torch.zeros((n, 4), dtype=torch.uint8, device="cuda:0")
            torch.cuda.synchronize()
            self.d.colourise(cur, Tc, Tl, bgr_d, c_d)
            self.keep += [bgr_d, c_d]
            if self.mode == "image":
                x_o, c_o = oracle_lib.colourise(x_o, Tc, Tl, bgr)
            else:
                x_o, c_o = clo.node(x_o, Tc, Tl, bgr.reshape(bgr.shape[0], 3 * W), W)
        self.keep.append(cur)
        self.d.add_stream_fast(C.c_void_p(cur.data_ptr()) if n else None, C.c_void_p(c_d.data_ptr()) if c_d is not None else None,
                               n, C.byref(f))
        self.o.add(np.asarray(x_o, np.float32).reshape(-1, 4), c_o, f)   # an empty cloud still runs the fuse (its floor)
        self.last_count = n
        return winfos

    def check(self, what, infos=None, nsteps=0):
        self.g.sync()
        self.d.sync()
        assert_layers_equal(self.g, self.o, what=(what, "oracle"))
        assert_layers_equal(self.g, self.d, what=(what, "device chain"))
        if infos is not None:
            got = self.g.prefilter_info(nsteps)
            assert got[:len(infos)] == infos, (what, got, infos)
        if self.last_count:
            assert self.g.stats() == self.d.stats(), (what, self.g.stats(), self.d.stats())


@pytest.mark.parametrize("name", vc.case_names())
def test_voxel_cases(name):
    _, p, leaf, field, limits, neg = vc.case_by_name(name)
    ch = Chains(64, 0.1, max_points=max(p.shape[0], 1))
    f = gem_b200.make_frame(np.eye(4), gem_b200.LaserSensorProcessor())
    steps = [(leaf, field, limits, neg)]
    x = torch.from_numpy(np.ascontiguousarray(p, np.float32)).cuda()
    ch.g.add_points_filtered_stream(x, steps, f)
    infos = ch.reference(p, steps, f)
    ch.check(name, infos, 1)
    if p.shape[0] and infos[0]["count"]:
        assert ch.g.stats()["points_in"] == infos[0]["count"]


VARIANTS = {"none": (None, "host"), "bgr8": ("bgr8", "host"), "rgb8": ("rgb8", "host"), "bgr8_stream": ("bgr8", "stream")}


@pytest.mark.parametrize("launch", list(LAUNCHES))
@pytest.mark.parametrize("mode", ["image", "node"])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_hdl64_frames(launch, mode, variant):
    """raw c2 frames as 32-byte XYZIR messages, scrolling, with an unfiltered call interleaved on the same handle"""
    enc, entry = VARIANTS[variant]
    steps = LAUNCHES[launch]
    ch = Chains(200, 0.1, mode)
    W, H = 1241, 376
    pinned = []
    for k in range(4):
        fr = synth.hdl64_frame(k)
        f = gem_b200.make_frame(fr["T"], gem_b200.LaserSensorProcessor())
        ch.keep.append(f)
        ch.move(fr["position"])
        case = pc.from_xyzi("f", "xyzir32", fr["xyzi"], seed=10 + k)
        raw = pc2_oracle.xyzi(pc2_oracle.decode(case)[0])
        img, step = make_image(enc, W, H, 40 + k) if enc else (None, 0)
        bgr = np_bgr(img, enc, W) if enc else None
        s = steps if k != 2 else []     # frame 2: the unfiltered call of the same ring
        if entry == "stream":
            x = torch.from_numpy(raw).cuda()
            bd = torch.from_numpy(bgr).cuda()
            ch.keep += [x, bd]
            ch.g.add_points_filtered_stream(x, s, f, bd, TC, TL)
        else:
            data = torch.from_numpy(case["data"]).pin_memory()
            im = torch.from_numpy(img).pin_memory() if enc else None
            pinned.append((data, im))
            cam = CameraImage(TC, TL, enc, im, W, H, step) if enc else None
            ch.g.add_pointcloud2_host_async(layout(case), data, f, cam, prefilter=s if k != 2 else None)
        infos = ch.reference(raw, s, f, bgr)
        if k == 1:
            ch.check((launch, mode, variant, k), infos, len(steps))
    ch.check((launch, mode, variant), infos, len(steps))
    if enc:
        assert (ch.g.get_layer("color_r") != 0).sum() > 100


@pytest.mark.parametrize("lay", ["xyzir22", "xyzir32_padded", "ouster", "d435"])
def test_layouts(lay):
    depth = lay == "d435"
    ch = Chains(120, 0.05) if depth else Chains(200, 0.1)
    sp = gem_b200.StructuredLightSensorProcessor() if depth else gem_b200.LaserSensorProcessor()
    W, H = (640, 480) if depth else (1241, 376)
    Tc, Tl = (TC_D435, np.eye(4)) if depth else (TC, TL)
    steps = [(0.02, "z", (0.2, 3.25), False)] if depth else voxel_oracle.FILTER_LAUNCH
    for k in range(3):
        fr = synth.d435_frame(k) if depth else synth.hdl64_frame(k)
        f = gem_b200.make_frame(fr["T"], sp)
        ch.keep.append(f)
        ch.move(fr["position"])
        if depth:
            case = pc.from_xyzi("f", "d435", fr["xyzi"], width=640, height=480, row_pad=32, seed=k, rgb=fr["rgba"])
        elif lay == "xyzir32_padded":
            rows = fr["xyzi"][:fr["xyzi"].shape[0] // 4 * 4]
            case = pc.from_xyzi("f", "xyzir32", rows, width=rows.shape[0] // 4, height=4, row_pad=24, seed=k)
            case_n = case["width"] * case["height"]
            assert case_n > 1000
        else:
            case = pc.from_xyzi("f", lay, fr["xyzi"], seed=k)
        raw = pc2_oracle.xyzi(pc2_oracle.decode(case)[0])
        img, step = make_image("bgr8", W, H, k)
        ch.g.add_pointcloud2_host_async(layout(case), case["data"].copy(), f, CameraImage(Tc, Tl, "bgr8", img.copy(), W, H, step),
                                        prefilter=steps)
        infos = ch.reference(raw, steps, f, np_bgr(img, "bgr8", W), Tc, Tl)
    ch.check(lay, infos, len(steps))


def test_sequence_edges():
    """staging growth in the middle, a filtered count of 0, a raw frame of exactly max_points, interleaved plain calls"""
    frames = [synth.hdl64_frame(k) for k in range(6)]
    full = min(fr["xyzi"].shape[0] for fr in frames)
    ch = Chains(200, 0.1, max_points=full)
    plan = [(5000, voxel_oracle.FILTER_LAUNCH), (8000, voxel_oracle.FILTER_KITTI_LAUNCH),
            (full, [(0.1, "x", (1000.0, 2000.0), False)]),      # nothing survives: an add of nothing
            (full, voxel_oracle.FILTER_KITTI_LAUNCH),           # exactly max_points, and the scratch grows
            (None, None),                                       # gem_add_points_host_async of the filtered cloud
            (30000, voxel_oracle.FILTER_LAUNCH)]
    pinned = []
    for k, (n, steps) in enumerate(plan):
        fr = frames[k]
        f = gem_b200.make_frame(fr["T"], gem_b200.LaserSensorProcessor())
        ch.keep.append(f)
        ch.move(fr["position"])
        if steps is None:
            x, _ = voxel_oracle.chain(fr["xyzi"], voxel_oracle.FILTER_LAUNCH)
            hx = torch.from_numpy(np.ascontiguousarray(x)).pin_memory()
            pinned.append(hx)
            ch.g.add_host_async_fast(C.c_void_p(hx.data_ptr()), None, x.shape[0], C.byref(f))
            ch.reference(x, [], f)
            continue
        case = pc.from_xyzi("f", "xyzir32", fr["xyzi"][:n], seed=k)
        data = torch.from_numpy(case["data"]).pin_memory()
        pinned.append(data)
        ch.g.add_pointcloud2_host_async(layout(case), data, f, prefilter=steps)
        infos = ch.reference(pc2_oracle.xyzi(pc2_oracle.decode(case)[0]), steps, f)
        if k == 2:
            assert infos[0]["count"] == 0
            assert ch.g.stats()["points_in"] == 0
    ch.check("edges", infos, len(plan[-1][1]))


def test_returns_while_the_stream_is_busy():
    s = torch.cuda.Stream()
    g = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False, stream=s.cuda_stream)
    d = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False)
    fr = synth.hdl64_frame(0)
    steps = voxel_oracle.FILTER_KITTI_LAUNCH
    keep = []
    for k in range(4):
        f = gem_b200.make_frame(fr["T"], gem_b200.LaserSensorProcessor())
        case = pc.from_xyzi("f", "xyzir32", fr["xyzi"], seed=k)
        data = torch.from_numpy(case["data"]).pin_memory()
        keep += [f, data]
        for m in (g, d):
            m.move(fr["position"])
        if k == 3:   # the first three calls sized every ring slot's buffers; now one bounded sleep ahead of the call
            g.sync()
            with torch.cuda.stream(s):
                torch.cuda._sleep(1_000_000_000)
            g.add_pointcloud2_host_async(layout(case), data, f, prefilter=steps)
            assert not s.query(), "the call waited for the handle's stream"
        else:
            g.add_pointcloud2_host_async(layout(case), data, f, prefilter=steps)
        x, _ = voxel_oracle.chain(pc2_oracle.xyzi(pc2_oracle.decode(case)[0]), steps)
        xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
        keep.append(xd)
        d.add_stream_fast(C.c_void_p(xd.data_ptr()), None, x.shape[0], C.byref(f))
    g.sync()
    d.sync()
    assert_layers_equal(g, d, what="after the sleep")
    assert g.stats() == d.stats()


def test_facade_matches_the_c_abi():
    exe = native.facade_program("prefilter_smoke")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "prefilter ok" in r.stdout, r.stdout + r.stderr
