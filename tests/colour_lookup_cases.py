"""Crafted clouds for the node's colour lookup (GEM_COLOUR_LOOKUP_NODE, DESIGN.md f19).  TEST INFRASTRUCTURE ONLY.

A case is a dict: name, width, height, row_stride (bytes), img (height, row_stride) uint8 BGR8 with padding bytes,
xyzi (n, 4) float32, T_camera (3, 4), T_lidar (4, 4).  Crafted cases use the pinhole P = [I | 0], so a point
(x + 0.5, y + 0.5, 1) lands on pixel (x, y).  Also the two measured clouds: the organised D435 frame into its 640 x 480
image, and a 64-beam cloud at 0.08 degrees of azimuth (the HDL-64E's step at 10 Hz) into the KITTI camera's 1241 x 376."""
from __future__ import annotations

import numpy as np

from gem_b200 import synth

T_PIN = np.array([[1.0, 0, 0, 0], [0, 1.0, 0, 0], [0, 0, 1.0, 0]])
EYE = np.eye(4)
TC_KITTI = np.array([[718.856, 0, 607.1928, 0], [0, 718.856, 185.2157, 0], [0, 0, 1, 0]], np.float64)
TL_KITTI = np.array([[0, -1, 0, 0.0], [0, 0, -1, -0.08], [1, 0, 0, -0.27], [0, 0, 0, 1]], np.float64)
TC_D435 = np.array([[385.0, 0, 320.0, 0], [0, 385.0, 240.0, 0], [0, 0, 1, 0]], np.float64)
NAN = float("nan")


def image(width: int, height: int, seed: int, pad: int = 0):
    return np.random.default_rng(seed).integers(0, 256, (height, 3 * width + pad)).astype(np.uint8)


def at(pixels, seed: int = 0):
    """points on the given pixels (x, y), in order, with nonzero intensities"""
    p = np.asarray(pixels, np.float64).reshape(-1, 2)
    inten = np.random.default_rng(seed).integers(1, 256, p.shape[0]).astype(np.float32)
    return np.stack([p[:, 0] + 0.5, p[:, 1] + 0.5, np.ones(p.shape[0]), inten], 1).astype(np.float32)


def case(name, width, height, xyzi, seed=1, pad=0, T_camera=T_PIN, T_lidar=EYE):
    return {"name": name, "width": width, "height": height, "row_stride": 3 * width + pad,
            "img": image(width, height, seed, pad), "xyzi": np.ascontiguousarray(xyzi, np.float32),
            "T_camera": T_camera, "T_lidar": T_lidar}


def _crafted():
    rng = np.random.default_rng(7)
    out = [
        case("pair_horizontal", 12, 10, at([(5, 5), (6, 5)])),
        case("pair_horizontal_left", 12, 10, at([(6, 5), (5, 5)])),
        case("pair_vertical", 12, 10, at([(5, 5), (5, 6)])),
        case("pair_vertical_up", 12, 10, at([(5, 6), (5, 5)])),
        case("pair_diagonal", 12, 10, at([(5, 5), (6, 6), (4, 4), (6, 4), (4, 6)])),
        case("one_pixel_twice", 12, 10, at([(5, 5), (5, 5), (6, 5), (5, 5), (4, 5)])),
        # (5, 5) reads what the later of its two painters left
        case("later_writer", 12, 10, at([(4, 5), (6, 5), (5, 5), (5, 4), (5, 5), (5, 6)])),
        case("alternating", 12, 10, at([(5, 5), (6, 5)] * 40 + [(7, 5), (6, 6)])),
        case("alternating_vertical", 12, 10, at([(3, 8), (3, 7)] * 25)),
        case("row_run", 30, 6, at([(x, 3) for x in range(1, 30)])),
        case("row_run_backwards", 30, 6, at([(x, 3) for x in range(29, 0, -1)])),
        case("column_run", 6, 30, at([(2, y) for y in range(1, 30)])),
        case("organised", 64, 48, at([(x, y) for y in range(1, 48) for x in range(1, 64)])),
        case("organised_columns", 40, 30, at([(x, y) for x in range(1, 40) for y in range(1, 30)])),
        case("organised_twice", 33, 17, at([(x, y) for _ in range(2) for y in range(1, 17) for x in range(1, 33)])),
        # clipped painting: points on the first and last readable rows and columns, corners included
        case("edges", 9, 7, at([(1, 1), (8, 1), (1, 6), (8, 6), (2, 1), (1, 2), (7, 6), (8, 5), (4, 1), (4, 6), (1, 3),
                                (8, 3), (4, 2), (4, 5), (2, 3), (7, 3), (1, 1), (8, 6)])),
        case("edges_all", 8, 6, at([(x, y) for y in (1, 5) for x in range(1, 8)] + [(x, y) for x in (1, 7) for y in range(1, 6)]
                                   + [(x, y) for y in (5, 1) for x in range(7, 0, -1)])),
    ]
    for w, h in ((2, 2), (2, 3), (3, 2), (3, 3), (2, 9), (9, 2), (3, 11), (11, 3)):
        pts = [(x, y) for _ in range(3) for y in range(h) for x in range(w)]   # x or y = 0: never read
        rng.shuffle(pts)
        out.append(case(f"tiny_{w}x{h}", w, h, at(pts, seed=w * 16 + h), seed=w * 16 + h))
    for pad in (1, 2, 5, 13):
        pts = rng.integers(1, 11, (300, 2))
        out.append(case(f"padded_stride_{pad}", 11, 11, at(pts, seed=pad), seed=pad, pad=pad))
    # out-of-image, behind-camera and NaN points between in-image ones: none reads or paints
    pts = at(rng.integers(1, 8, (400, 2)), seed=3)
    bad = np.array([[-3.0, 2.5, 1.0, 9], [0.5, 2.5, 1.0, 9], [2.5, 0.5, 1.0, 9], [8.5, 2.5, 1.0, 9], [2.5, 8.5, 1.0, 9],
                    [100.0, 2.5, 1.0, 9], [-2.5, -2.5, -1.0, 9], [2.5, 2.5, -1.0, 9], [2.5, 2.5, 0.0, 9], [2.5, 2.5, -0.0, 9],
                    [NAN, 2.5, 1.0, 9], [2.5, NAN, 1.0, 9], [2.5, 2.5, NAN, 9], [float("inf"), 2.5, 1.0, 9],
                    [2.5, 2.5, float("inf"), 9], [1e30, 1e30, 1e-30, 9]], np.float32)
    mixed = np.empty((pts.shape[0] + 40 * bad.shape[0], 4), np.float32)
    slot = np.zeros(mixed.shape[0], bool)
    slot[rng.choice(mixed.shape[0], 40 * bad.shape[0], replace=False)] = True
    mixed[slot] = np.tile(bad, (40, 1))[rng.permutation(40 * bad.shape[0])]
    mixed[~slot] = pts
    out.append(case("invalid_interleaved", 8, 8, mixed))
    # a perspective camera with a pose: pixels from real projections
    pts = np.stack([rng.uniform(-2, 2, 5000), rng.uniform(-1.5, 1.5, 5000), rng.uniform(0.5, 4, 5000),
                    rng.integers(1, 256, 5000)], 1).astype(np.float32)
    out.append(case("pinhole_random", 40, 30, pts, T_camera=np.array([[10.0, 0, 20, 0], [0, 10.0, 15, 0], [0, 0, 1, 0]]),
                    T_lidar=synth.pose_matrix(0.1, -0.05, 0.2, 0.02)))
    return out


def large_patch(n: int = 1_000_000):
    """n points in a 3 x 3 pixel patch in random order: chains as long as the cloud"""
    rng = np.random.default_rng(11)
    return case("patch_3x3_1e6", 16, 12, at(np.stack([rng.integers(6, 9, n), rng.integers(4, 7, n)], 1), seed=11))


_CASES = None


def cases():
    global _CASES
    if _CASES is None:
        _CASES = _crafted()
    return _CASES


def case_names():
    return [c["name"] for c in cases()] + ["patch_3x3_1e6"]


def case_by_name(name):
    if name == "patch_3x3_1e6":
        return large_patch()
    return next(c for c in cases() if c["name"] == name)


def d435(frame: int = 0):
    """the organised D435 frame (640 x 480 points, NaN where no return) into its 640 x 480 image"""
    fr = synth.d435_frame(frame)
    return case("d435", 640, 480, fr["xyzi"], seed=500 + frame, T_camera=TC_D435, T_lidar=EYE)


def lidar_008(frame: int = 0, n_az: int = 4500, step_deg: float = 0.08):
    """synth.hdl64_frame's scene and pose with 4,500 azimuth steps of 0.08 degrees, into the KITTI camera"""
    scene = synth.make_scene()
    rng = np.random.Generator(np.random.PCG64(synth.FRAME_SEED0 + 50000 + frame))
    elev = np.deg2rad(np.linspace(2.0, -24.8, 64))
    AZ, EL = np.meshgrid(np.arange(n_az) * np.deg2rad(step_deg), elev, indexing="ij")   # azimuth-major
    AZ, EL = AZ.reshape(-1), EL.reshape(-1)
    d_s = np.stack([np.cos(EL) * np.cos(AZ), np.cos(EL) * np.sin(AZ), np.sin(EL)], 1)
    T, _ = synth.hdl64_pose(frame)
    t, _ = synth._cast(T[:3, 3], d_s @ T[:3, :3].T, scene, 0.9, 120.0)
    ok = np.isfinite(t)
    p = d_s[ok] * t[ok, None]
    xyzi = np.concatenate([p, rng.integers(1, 256, (p.shape[0], 1))], 1).astype(np.float32)
    return case("lidar_008", 1241, 376, xyzi, seed=600 + frame, T_camera=TC_KITTI, T_lidar=TL_KITTI)
