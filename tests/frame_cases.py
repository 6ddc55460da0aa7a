"""Frames whose per-frame constants are not make_frame's defaults, for tests/test_reference_pin_frames.py (the oracle
against the reference's own kernels), tests/test_shim_gpu.py (the device and the drop-in shim against the oracle) and
tests/test_gpu_parity.py::test_rotation_variance_term.  CPU only, no GPU imports.

Every recording of the reference made before these used zero rotation variance, C_SB_transpose = I, P = (0, 0, 1) and
a zero skew, where the rotation-Jacobian term of G_pointsprocess (gpu_process.cu:417-422) is zero.  Here:

  full      T with roll, pitch and yaw, a sensor Jacobian that is not row 2 of T, an asymmetric rotation variance (only
            an asymmetric one exposes a transpose), C_SB_transpose a rotation about all three axes, all three components
            of P_mul_C_BM_transpose non-zero and an antisymmetric B_r_BS_skew with all three components non-zero;
  rot_only  the same kinds of constants with min_r = beam_a = beam_c = 0: the variance is the rotation term alone;
  overflow  zero rotation variance, height window +-inf, and points so far along the map's z axis that the rotation
            Jacobian overflows: the reference computes 0 * inf = NaN there.

Each cloud holds a point at the sensor origin (the hard-coded box filter of gpu_process.cu:393 drops it), points near
the sensor, long-range points (most outside the map) and random R, G, B and intensity values.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from gem_b200 import LaserSensorProcessor, make_frame

f32 = np.float32


def rpy(roll, pitch, yaw):
    """R = Rz(yaw) Ry(pitch) Rx(roll) in float64"""
    cr, sr, cp, sp, cy, sy = np.cos(roll), np.sin(roll), np.cos(pitch), np.sin(pitch), np.cos(yaw), np.sin(yaw)
    Rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
    Ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]])
    Rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


@dataclass
class FrameCase:
    name: str
    L: int
    res: float
    position: np.ndarray        # move() target before the cloud
    frame: object               # gem_b200 GemFrame
    consts: dict                # the frame's matrices as float32 arrays (T 4x4, sJ 3, rv / csb / bskew 3x3, P 3)
    x: np.ndarray               # sensor-frame cloud, float32
    y: np.ndarray
    z: np.ndarray
    R: np.ndarray               # int32 colours and float32 intensity for Fuse
    G: np.ndarray
    B: np.ndarray
    I: np.ndarray
    overflow: np.ndarray        # bool per point: placed where the rotation Jacobian overflows

    @property
    def xyzi(self):
        return np.ascontiguousarray(np.stack([self.x, self.y, self.z, self.I], axis=1), f32)

    @property
    def rgba(self):
        a = np.stack([self.R, self.G, self.B, np.full_like(self.R, 255)], axis=1)
        return np.ascontiguousarray(a, np.uint8)


def _T(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def _cloud(rng, n_near, n_far):
    """sensor-frame points that the box filter keeps (y <= -1.5 or |x| >= 1.5 with y <= -1), plus the origin"""
    near = np.stack([rng.uniform(-9.0, 9.0, n_near), rng.uniform(-9.0, -1.6, n_near), rng.uniform(-2.0, 2.0, n_near)], 1)
    r = rng.uniform(40.0, 160.0, n_far)
    a = rng.uniform(np.pi * 1.05, np.pi * 1.95, n_far)              # sin(a) < 0: y < 0, far from the filter band
    far = np.stack([r * np.cos(a), r * np.sin(a), rng.uniform(-3.0, 3.0, n_far)], 1)
    return np.concatenate([np.zeros((1, 3)), near, far]).astype(f32)


def _case(name, L, res, T, consts, sensor, pts, rng, overflow=None, base_z=0.0):
    T32 = np.asarray(T, np.float64).astype(f32)
    frame = make_frame(T, sensor, base_z=base_z, rotation_variance=consts["rv"], C_SB_transpose=consts["csb"],
                       P_mul_C_BM_transpose=consts["P"], B_r_BS_skew=consts["bskew"], sensor_jacobian=consts["sJ"])
    n = pts.shape[0]
    col = rng.integers(1, 256, (n, 3)).astype(np.int32)
    col[rng.random(n) < 0.1, rng.integers(0, 3)] = 0
    inten = rng.uniform(0.5, 60.0, n).astype(f32)
    inten[rng.random(n) < 0.1] = 0
    c = {k: np.asarray(v, f32) for k, v in consts.items()}
    c["T"] = T32
    pos = np.array([T32[0, 3], T32[1, 3], T32[2, 3]], f32)
    return FrameCase(name, L, res, pos, frame, c, *(np.ascontiguousarray(pts[:, k]) for k in range(3)),
                     col[:, 0].copy(), col[:, 1].copy(), col[:, 2].copy(), inten,
                     np.zeros(n, bool) if overflow is None else overflow)


def frame_cases():
    out = []
    rng = np.random.default_rng(20261018)
    # full: every constant non-trivial, the laser's own variances
    rv = np.array([[2.0e-4, 7.0e-5, -3.0e-5], [-4.0e-5, 3.0e-4, 6.0e-5], [9.0e-5, -2.0e-5, 1.5e-4]])
    consts = dict(sJ=[0.12, -0.27, 0.93], rv=rv, csb=rpy(0.21, -0.33, 0.47).T, P=[0.31, -0.44, 0.84],
                  bskew=skew([0.12, -0.31, 0.07]))
    T = _T(rpy(0.08, -0.11, 0.6), [3.7, -2.4, 0.9])
    out.append(_case("full", 101, 0.2, T, consts, LaserSensorProcessor(ignore_points_above=30.0,
                                                                       ignore_points_below=-30.0),
                     _cloud(rng, 3000, 400), rng))
    # rot_only: the variance is the rotation term alone; an even L
    rv2 = np.array([[1.0e-3, -2.0e-4, 5.0e-4], [3.0e-4, 4.0e-4, -1.0e-4], [-6.0e-4, 2.0e-4, 8.0e-4]])
    consts2 = dict(sJ=[-0.2, 0.35, 0.9], rv=rv2, csb=rpy(-0.4, 0.25, -0.9).T, P=[-0.52, 0.23, 0.77],
                   bskew=skew([-0.25, 0.18, 0.33]))
    T2 = _T(rpy(-0.15, 0.07, -1.3), [-5.3, 8.1, 1.4])
    out.append(_case("rot_only", 96, 0.25, T2, consts2,
                     LaserSensorProcessor(min_radius=0.0, beam_angle=0.0, beam_constant=0.0, ignore_points_above=30.0,
                                          ignore_points_below=-30.0),
                     _cloud(rng, 2500, 300), rng))
    # overflow: a yaw-only T so that z goes to the height alone (row 2 = (0, 0, 1)), zero rotation variance, +-inf
    # thresholds; points at |z| of 1e38 .. 3e38 keep a finite height and land inside the map.  With |P| about 2.7 the
    # rotation Jacobian (P times the skew of C_SB_transpose * p, sums of terms near 1e38) overflows for about half
    consts3 = dict(sJ=[0.3, -0.4, 0.86], rv=np.zeros((3, 3)), csb=rpy(0.5, -0.6, 0.7).T, P=[1.6, -1.5, 1.55],
                   bskew=skew([0.2, -0.1, 0.3]))
    T3 = _T(rpy(0.0, 0.0, 0.4), [1.5, -0.5, 0.25])
    base = _cloud(rng, 1500, 200)
    m = 400
    huge = np.stack([rng.uniform(-6.0, 6.0, m), rng.uniform(-6.0, -1.6, m), rng.uniform(1.0e38, 3.0e38, m)], 1)
    huge[m // 2:, 2] *= -1
    pts = np.concatenate([base, huge.astype(f32)])
    over = np.zeros(pts.shape[0], bool)
    over[base.shape[0]:] = True
    out.append(_case("overflow", 75, 0.2, T3, consts3,
                     LaserSensorProcessor(ignore_points_above=float("inf"), ignore_points_below=float("-inf")),
                     pts, rng, overflow=over))
    return out


def rotation_jacobian_f32(c, x, y, z, csb=None, bskew=None, P=None):
    """rotJ of gpu_process.cu:417-418 in float32, the reference's sums left to right"""
    csb = c.consts["csb"] if csb is None else csb
    bskew = c.consts["bskew"] if bskew is None else bskew
    P = c.consts["P"] if P is None else P
    x, y, z = (np.asarray(a, f32) for a in (x, y, z))
    with np.errstate(all="ignore"):
        q = [(csb[j, 0] * x + csb[j, 1] * y) + csb[j, 2] * z for j in range(3)]
        S = [[f32(0) + bskew[0, 0], -q[2] + bskew[0, 1], q[1] + bskew[0, 2]],
             [q[2] + bskew[1, 0], f32(0) + bskew[1, 1], -q[0] + bskew[1, 2]],
             [-q[1] + bskew[2, 0], q[0] + bskew[2, 1], f32(0) + bskew[2, 2]]]
        return [(P[0] * S[0][j] + P[1] * S[1][j]) + P[2] * S[2][j] for j in range(3)]


def variance_f64(c, x, y, z, rv=None, csb=None, bskew=None, sJ=None):
    """the height variance of gpu_process.cu:403-425 in float64 (error propagation law), with any of the frame's
    matrices replaced: what a copy that transposes one of them or flips the skew's sign would compute"""
    k = {n: np.asarray(c.consts[n], np.float64) for n in ("rv", "csb", "bskew", "sJ", "P")}
    for n, v in (("rv", rv), ("csb", csb), ("bskew", bskew), ("sJ", sJ)):
        if v is not None:
            k[n] = np.asarray(v, np.float64)
    p = np.stack([x, y, z], 1).astype(np.float64)
    q = p @ k["csb"].T
    Sk = np.zeros((p.shape[0], 3, 3))
    Sk[:, 0, 1], Sk[:, 0, 2], Sk[:, 1, 0] = -q[:, 2], q[:, 1], q[:, 2]
    Sk[:, 1, 2], Sk[:, 2, 0], Sk[:, 2, 1] = -q[:, 0], -q[:, 1], q[:, 0]
    J = np.einsum("i,nij->nj", k["P"], Sk + k["bskew"])
    term1 = np.einsum("ni,ij,nj->n", J, k["rv"], J)
    s = c.frame.sensor
    d = np.linalg.norm(p, axis=1)
    vL = (s.beam_constant + s.beam_angle * d) ** 2
    vN = np.full_like(d, s.min_radius ** 2)
    sJ = k["sJ"]
    term2 = sJ[0] ** 2 * vL + sJ[1] ** 2 * vL + sJ[2] ** 2 * vN
    return term1 + term2


def variance_f32(c, x, y, z, rv=None):
    """the laser height variance of gpu_process.cu:403-425 in float32 with the reference's left-to-right sums (the
    stand-in Eigen header's products), with the rotation variance optionally replaced"""
    rv = c.consts["rv"] if rv is None else np.asarray(rv, f32)
    sJ, s = c.consts["sJ"], c.frame.sensor
    x, y, z = (np.asarray(a, f32) for a in (x, y, z))
    J = rotation_jacobian_f32(c, x, y, z)
    with np.errstate(all="ignore"):
        A1 = [(J[0] * rv[0, j] + J[1] * rv[1, j]) + J[2] * rv[2, j] for j in range(3)]
        term1 = (A1[0] * J[0] + A1[1] * J[1]) + A1[2] * J[2]
        d = np.sqrt((x * x + y * y) + z * z)
        b = f32(s.beam_constant) + f32(s.beam_angle) * d
        vL, vN = b * b, np.full_like(x, f32(s.min_radius) * f32(s.min_radius))
        zero = np.zeros_like(x)
        B = [(sJ[0] * vL + sJ[1] * zero) + sJ[2] * zero, (sJ[0] * zero + sJ[1] * vL) + sJ[2] * zero,
             (sJ[0] * zero + sJ[1] * zero) + sJ[2] * vN]
        return term1 + ((B[0] * sJ[0] + B[1] * sJ[1]) + B[2] * sJ[2])
