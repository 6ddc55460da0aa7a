"""The node's colour lookup without a GPU (DESIGN.md f19): the literal C oracle (tests/orc_colour_lookup.c) equals an
independent Python restatement of the loop and the closed form C5 that the device computes, on every crafted case and on
the two measured clouds; where nothing paints, the lookup is the IMAGE one (the oracle's orc_colourise)."""
import numpy as np
import pytest

import colour_lookup_cases as cc
import colour_lookup_oracle as clo
import oracle_lib

LITERAL_MAX = 200_000   # the Python loop runs a few microseconds per point


def run(c, fn):
    return fn(c["xyzi"], c["T_camera"], c["T_lidar"], c["img"], c["width"])


def same(a, b, what):
    (xa, ca), (xb, cb) = a, b
    assert xa.tobytes() == xb.tobytes(), what
    if not np.array_equal(ca, cb):
        bad = np.flatnonzero((ca != cb).any(axis=1))
        raise AssertionError((what, int(bad.size), int(bad[0]), ca[bad[0]], cb[bad[0]]))


@pytest.mark.parametrize("name", cc.case_names())
def test_oracle_equals_literal_loop_and_closed_form(name):
    c = cc.case_by_name(name)
    want = run(c, clo.node)
    if c["xyzi"].shape[0] <= LITERAL_MAX:
        same(want, run(c, clo.literal), (name, "literal"))
    same(want, run(c, clo.closed_form), (name, "closed form"))


@pytest.mark.parametrize("cloud", ["d435", "lidar_008"])
def test_measured_clouds(cloud):
    c = cc.d435() if cloud == "d435" else cc.lidar_008()
    want = run(c, clo.node)
    same(want, run(c, clo.closed_form), (cloud, "closed form"))
    if cloud == "lidar_008":
        same(want, run(c, clo.literal), (cloud, "literal"))
    img = c["img"][:, :3 * c["width"]].reshape(c["height"], c["width"], 3)
    x_i, c_i = oracle_lib.colourise(c["xyzi"], c["T_camera"], c["T_lidar"], img)
    assert x_i.tobytes() == want[0].tobytes()
    inside = c_i[:, 3] == 255
    assert np.array_equal(inside, want[1][:, 3] == 255)
    differs = int((c_i != want[1]).any(axis=1).sum())
    assert inside.sum() > 10_000 and differs > inside.sum() // 2, (int(inside.sum()), differs)


@pytest.mark.parametrize("name", ["pair_diagonal", "edges", "invalid_interleaved", "pinhole_random"])
def test_image_mode_is_orc_colourise(name):
    """a cloud whose points never share a 4-neighbour reads the unmodified image in both modes"""
    c = cc.case_by_name(name)
    mx, my, inside = clo.project(c["xyzi"], c["T_camera"], c["T_lidar"], c["width"], c["height"])
    par = clo.parents(np.where(inside, my * c["width"] + mx, 0), inside, c["width"], c["height"])
    img = np.ascontiguousarray(c["img"][:, :3 * c["width"]]).reshape(c["height"], c["width"], 3)
    x_i, c_i = oracle_lib.colourise(c["xyzi"], c["T_camera"], c["T_lidar"], img)
    x_n, c_n = run(c, clo.node)
    assert x_i.tobytes() == x_n.tobytes()
    root = par < 0
    assert np.array_equal(c_i[root], c_n[root])
    if name == "pair_diagonal":
        assert root.all() and np.array_equal(c_i, c_n)


def test_chains():
    """the cases reach what they are named for: long chains, clipped painting, the patch's chain across the cloud"""
    depth = {c["name"]: clo.chain_depth(c["xyzi"], c["T_camera"], c["T_lidar"], c["width"], c["height"]) for c in cc.cases()}
    assert depth["pair_horizontal"] == 1 and depth["pair_diagonal"] == 0 and depth["organised"] == 62 + 46
    assert depth["row_run"] == 28 and depth["alternating"] >= 80
    c = cc.large_patch(20_000)
    assert clo.chain_depth(c["xyzi"], c["T_camera"], c["T_lidar"], c["width"], c["height"]) > 4_000
