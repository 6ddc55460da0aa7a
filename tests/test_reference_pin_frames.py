"""Pins the CPU oracle against the REFERENCE ITSELF on frames whose per-frame constants are not make_frame's defaults
(tests/frame_cases.py): T with roll, pitch and yaw, an explicit sensor Jacobian, an asymmetric rotation variance,
C_SB_transpose a rotation about all three axes, P and B_r_BS_skew with every component non-zero, a laser whose
variance is the rotation term alone, and points whose rotation Jacobian overflows.  Every earlier recording used the
default constants, where the rotation-Jacobian term of G_pointsprocess (gpu_process.cu:417-422) is zero.

Each scenario runs Move, Process_points (all five outputs) and Fuse and compares elevation, variance, intensity and
colour; `lowest` only in cells that received a single point (the reference's update of it is racy,
gpu_process.cu:434-438).  Every comparison is bit for bit, NaN as a class.

The reference's outputs are stored in tests/golden/reference_pin_frames_v1.npz, recorded on an H100 by
`tests/golden/make_reference_pin.py test_reference_pin_frames tests/golden/reference_pin_frames_v1.npz` from the
reference's gpu_process.cu compiled unmodified with -fmad=false against oracle/mini_eigen (oracle/build_ref.py), and
replayed through ref_lib.PinnedRef.  The stand-in Eigen header's products sum left to right, which fixes the order of
the rotation term's sums; real Eigen's order depends on its version, so a node built against real Eigen may differ from
this pin in the last bits of the variance."""
import os

import numpy as np
import pytest

import frame_cases as fc
import ref_lib
from oracle_lib import OracleMap
from pin_cases import assert_bits

PIN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pin_frames_v1.npz")
f32 = np.float32
PACKED = True               # the recording is stored in ref_lib.pack's form
LAYERS = ("elevation", "variance", "intensity", "color_r", "color_g", "color_b")
OUTPUTS = ("map_index", "var", "x_ts", "y_ts", "z_ts")


@pytest.fixture(scope="module")
def reference():
    """reference(tag, L, res, nofma) -> the reference's map for one scenario, replayed from the stored outputs"""
    g = ref_lib.Packed(np.load(PIN, allow_pickle=False))
    assert "reference gpu_process.cu" in str(g["generated_by"])
    return lambda tag, L, res, nofma: ref_lib.PinnedRef(g, tag)


def single_point_cells(o, ko):
    """geographic cells that received exactly one accepted point"""
    acc = ko[1] != f32(-1)
    geo = np.array([o.points_to_index(a, b)[0] for a, b in zip(ko[2][acc], ko[3][acc])], np.int64)
    geo = geo[geo >= 0]
    u, cnt = np.unique(geo, return_counts=True)
    return u[cnt == 1]


def run_scenario(r, o, c):
    """Move, Process_points and Fuse on the map under test `r` and the oracle `o`; every output compared bit for bit.
    Returns the oracle's Process_points outputs."""
    co = o.move(c.position)
    for a, b, name in zip(r.move(c.position, like=co), co, ("centre", "start", "shift")):
        assert_bits(a, b, f"{c.name} move {name}")
    ko = o.process_points(c.x, c.y, c.z, c.frame)
    kr = r.process_points(c.x, c.y, c.z, c.frame, like=ko)
    for a, b, name in zip(kr, ko, OUTPUTS):
        assert_bits(a, b, f"{c.name} {name}")
    single = single_point_cells(o, ko)
    assert single.size > 100, c.name
    lo = o.get_layer("lowest").reshape(-1)
    pick = lambda a: np.ascontiguousarray(np.asarray(a).reshape(-1)[single])
    assert_bits(r.get_layer("lowest", like=pick(lo), derive=pick), pick(lo), f"{c.name} lowest")
    for m in (r, o):
        m.fuse_points(ko[0], c.R, c.G, c.B, c.I, ko[4], ko[1])
    lo = {n: o.get_layer(n) for n in LAYERS}
    for name, a in r.layers(LAYERS, like=lo).items():
        assert_bits(a, lo[name], f"{c.name} {name} after Fuse")
    return ko


def assert_discriminates(c, ko):
    """the decisions the scenario exists for: the oracle's variance is the float64 error propagation law to float32
    precision, and each likely wrong copy of the frame constants (C_SB_transpose transposed, the skew's sign flipped,
    the sensor Jacobian taken from T) changes it materially on most accepted points.  A transposed rotation variance
    leaves the quadratic form J Sigma J^T unchanged in exact arithmetic; it changes the float32 result's last bits
    (the products pair other entries before they are summed), on a good share of the points"""
    acc = ko[1] != f32(-1)
    assert ko[1][0] == f32(-1) and c.x[0] == 0 and c.y[0] == 0 and c.z[0] == 0, "the sensor origin is filtered out"
    assert (np.sqrt(c.x[acc].astype(float) ** 2 + c.y[acc] ** 2) > 40).sum() > 100, "long-range points"
    assert ((ko[0] >= 0) & acc).sum() > 1000
    x, y, z = c.x[acc], c.y[acc], c.z[acc]
    want = fc.variance_f64(c, x, y, z)
    assert np.allclose(ko[1][acc], want, rtol=2e-4, atol=0), c.name
    k = c.consts
    assert_bits(fc.variance_f32(c, x, y, z), ko[1][acc], f"{c.name} float32 restatement")
    flipped = fc.variance_f32(c, x, y, z, rv=k["rv"].T).view(np.uint32) != ko[1][acc].view(np.uint32)
    assert flipped.mean() > 0.2, (c.name, float(flipped.mean()))
    wrong = {"C_SB_transpose^T": dict(csb=k["csb"].T),
             "-B_r_BS_skew": dict(bskew=-k["bskew"])}
    if c.frame.sensor.beam_constant != 0:
        wrong["sensor_jacobian from T"] = dict(sJ=k["T"][2, :3])
    for name, kw in wrong.items():
        v = fc.variance_f64(c, x, y, z, **kw)
        changed = np.abs(v - want) > 1e-3 * np.abs(want)
        assert changed.mean() > 0.75, (c.name, name, float(changed.mean()))
    return wrong


CASES = {c.name: c for c in fc.frame_cases()}


def test_full_frame_constants_vs_reference(reference):
    c = CASES["full"]
    ko = run_scenario(reference("frames_full", c.L, c.res, True), OracleMap(c.L, c.res, compat_box_filter=True), c)
    assert "sensor_jacobian from T" in assert_discriminates(c, ko)
    assert not np.allclose(c.consts["sJ"], c.consts["T"][2, :3], atol=0.05)


def test_rotation_term_alone_vs_reference(reference):
    c = CASES["rot_only"]
    ko = run_scenario(reference("frames_rot_only", c.L, c.res, True), OracleMap(c.L, c.res, compat_box_filter=True), c)
    assert_discriminates(c, ko)
    s = c.frame.sensor
    assert s.min_radius == 0 and s.beam_angle == 0 and s.beam_constant == 0


def test_rotation_jacobian_overflow_vs_reference(reference):
    """zero rotation variance, a rotation Jacobian that overflows: the reference's 0 * inf makes the variance NaN,
    and the NaN variance is fused into the cells"""
    c = CASES["overflow"]
    ko = run_scenario(reference("frames_overflow", c.L, c.res, True), OracleMap(c.L, c.res, compat_box_filter=True), c)
    acc = ko[1] != f32(-1)
    J = fc.rotation_jacobian_f32(c, c.x, c.y, c.z)
    inf = acc & ~(np.isfinite(J[0]) & np.isfinite(J[1]) & np.isfinite(J[2]))
    assert not c.consts["rv"].any() and np.isinf(c.frame.rel_lower) and np.isinf(c.frame.rel_upper)
    assert (inf & (ko[0] >= 0)).sum() > 50, "overflowing points inside the map"
    assert np.isnan(ko[1][inf]).all()
    assert np.isfinite(ko[1][acc & ~c.overflow]).all()
