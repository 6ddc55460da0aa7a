"""The device against the oracle on the inputs tests/test_reference_pin_cases.py pins the oracle to the reference with
that no other device test runs: the point front end at odd and even L with scrolled starts (cell boundaries one ulp
apart, box-filter limits), the scroll script (wrapping bands, shifts of +-(L-1), L and L + 5, var_update of both
signs, Map_optmove / Map_closeloop at their rounding boundaries and far from the origin) and the 5-sigma gate at
equality.  So device = oracle = reference holds on each of them.  Every comparison is bit for bit."""
import numpy as np
import pytest

import gem_b200
import pin_cases as pc
from oracle_lib import OracleMap
from pin_cases import assert_bits, front_end_frame
from shim_lib import FEATURE_LAYERS, shim  # noqa: F401  (shim is a fixture)

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.mark.parametrize("c", pc.front_end_cases(), ids=lambda c: c.name)
def test_front_end_cases_match_oracle(c, shim):
    """through the C ABI and through the drop-in shim's nine entry points (which cannot observe `lowest`)"""
    f = front_end_frame()
    for kind in ("device", "shim"):
        g = gem_b200.ElevationMap(c.L, c.res, compat_box_filter=True) if kind == "device" else shim(c.L, c.res)
        o = OracleMap(c.L, c.res, compat_box_filter=True)
        try:
            for a, b in zip(g.move(c.position), o.move(c.position)):
                assert_bits(a, b, f"{kind} {c.name} move")
            kg = g.process_points(c.x, c.y, c.z, f)
            ko = o.process_points(c.x, c.y, c.z, f)
            for a, b, name in zip(kg, ko, ("map_index", "var", "x_ts", "y_ts", "z_ts")):
                assert_bits(a, b, f"{kind} {c.name} {name}")
            if kind == "device":
                assert_bits(g.get_layer("lowest"), o.get_layer("lowest"), f"{c.name} lowest")
            assert (ko[0] >= 0).any()
        finally:
            g.close()
            o.close()


def test_scroll_script_matches_oracle(shim):
    """through the C ABI (every step, the scroll state and every layer) and through the drop-in shim: its `traver`
    steps left out (only Raytracing reads traver, gpu_process.cu:712, and the script never calls it), Move's and
    Map_optmove's outputs and the layers Map_feature returns compared after every step"""
    s = pc.scroll_script()
    g = gem_b200.ElevationMap(s.L, s.res, compat_box_filter=False)
    o = OracleMap(s.L, s.res, compat_box_filter=False)
    try:
        for k, (op, args) in enumerate(s.steps):
            rg, ro = pc.apply_step(g, op, args), pc.apply_step(o, op, args)
            if ro is not None:
                for a, b in zip(rg if isinstance(rg, tuple) else (rg,), ro if isinstance(ro, tuple) else (ro,)):
                    assert_bits(a, b, f"step {k} {op} result")
            (cg, sg, zg), (co, so, zo) = g.state(), o.state()
            assert_bits(cg, co, f"step {k} {op} centre")
            assert np.array_equal(sg, so) and f32(zg) == f32(zo), (k, op, sg, so, zg, zo)
            for name in pc.SCROLL_LAYERS:
                assert_bits(g.get_layer(name), o.get_layer(name), f"step {k} {op} {name}")
    finally:
        g.close()
        o.close()
    # the shim's map has the reference's hard-coded box filter, which Fuse, the scrolls and the map-wide calls never
    # consult, so the oracle keeps it too
    m = shim(s.L, s.res)
    o = OracleMap(s.L, s.res, compat_box_filter=True)
    try:
        n = 0
        for k, (op, args) in enumerate(s.steps):
            if op == "traver":
                continue
            rm, ro = pc.apply_step(m, op, args), pc.apply_step(o, op, args)
            if ro is not None:
                for a, b in zip(rm if isinstance(rm, tuple) else (rm,), ro if isinstance(ro, tuple) else (ro,)):
                    assert_bits(a, b, f"shim step {k} {op} result")
            fm, fo = m.map_feature(), o.map_feature()
            for name in FEATURE_LAYERS:
                assert_bits(fm[name], fo[name], f"shim step {k} {op} {name}")
            n += 1
        assert n > 50
    finally:
        o.close()


def test_gate_at_equality_matches_oracle():
    s = pc.gate_records()
    g = gem_b200.ElevationMap(s.L, 0.1, compat_box_filter=False)
    o = OracleMap(s.L, 0.1, compat_box_filter=False)
    try:
        for m in (g, o):
            s.apply_init(m)
            m.fuse_points(*s.fuse_args())
        for name in ("elevation", "variance", "intensity", "color_r", "color_g", "color_b"):
            assert_bits(g.get_layer(name), o.get_layer(name), f"gate {name}")
    finally:
        g.close()
        o.close()
