"""The global-map octrees, CPU side: the oracle (tests/orc_color_octree.c) against the independent Python restatement of
tests/octree_cases.py, bit for bit, on every crafted family and on natural split clouds; the stream decoder's structure
and O5 checks on the oracle's streams; the ctypes mirror of gem_octree; the C++ facade program compiles."""

import numpy as np
import pytest

import native
import octree_cases as oc
import octree_oracle
import split_oracle
import submap_oracle
from gem_b200 import synth
from oracle_lib import OracleMap

CASES = oc.crafted_cases()


def check_against_restatement(rec, res, what):
    got, info = octree_oracle.color_octree(rec, res)
    want, ins, skip = oc.py_color_octree(rec, res)
    assert got.shape == want.shape and np.array_equal(got, want), (what, got.shape, want.shape)
    assert (info["inserted"], info["skipped"]) == (ins, skip), what
    nodes, leaves = oc.decode(got)
    assert (info["nodes"], info["leaves"], info["bytes"]) == (nodes, leaves, 8 * nodes), what
    return info


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_oracle_matches_restatement_on_crafted_clouds(name):
    _, rec, res = next(c for c in CASES if c[0] == name)
    info = check_against_restatement(rec, res, name)
    if name in ("empty", "all_skipped"):
        assert info["bytes"] == 0 and info["inserted"] == 0
    if name == "block_equal_hits":    # the block is pruned: its parent holds one childless node there
        assert info["leaves"] == 1 and info["nodes"] == 16
    if name == "block_unequal_hits":
        assert info["leaves"] == 8 and info["nodes"] == 16 + 8
    if name == "cube4_twice_saturating_order":   # every voxel saturated: the whole cube ends as one pruned node
        assert info["leaves"] == 1 and info["nodes"] == 15


def test_saturation_sequence():
    """one voxel hit h times: the leaf value walks the O2 states and stops at max; the colour of a white-only voxel
    stays unset"""
    for h in range(1, 9):
        s, info = octree_oracle.color_octree(oc.cloud([[3, 4, 5]] * h, 0.1, [oc.WHITE] * h), 0.1)
        assert info["nodes"] == 17
        v = np.frombuffer(s[-8:-4].tobytes(), np.float32)[0]
        want = oc.HIT
        for _ in range(h - 1):
            want = min(np.float32(want + oc.HIT), oc.MAX)
        assert v == want and tuple(s[-4:-1]) == oc.WHITE, h


@pytest.mark.parametrize("res", [0.2, 0.1])
def test_oracle_matches_restatement_on_split_clouds(res):
    L, gres = 96, 0.1
    o = OracleMap(L, gres, compat_box_filter=False)
    scene = synth.make_scene()
    pos = np.array([0.3, -0.2, 1.7], np.float32)
    import gem_b200
    for k in range(2):
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([0.4, 0.3, 0.0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        o.move(pos)
        o.add(fr["xyzi"], fr["rgba"], gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
        o.compute_features()
        o.snapshot_shown()
    f, centre, start = o._prev
    rec = submap_oracle.grid_cloud(f, L, centre, start, gres)
    sp = split_oracle.grid_split(rec, 20, 1.0, 0.0)
    assert sp["road"].shape[0] + sp["obstacle"].shape[0] > 300
    for part in ("road", "obstacle"):
        check_against_restatement(sp[part], res, (part, res))


def test_gem_octree_struct_matches_the_header():
    import gem_b200._lib as L
    assert {"nodes", "leaves", "inserted", "skipped"} <= {f for f, _ in L.GemOctree._fields_}
    native.assert_struct_layouts({"gem_octree": L.GemOctree}, std=None)


def test_facade_program_with_color_octree_compiles():
    native.facade_compiles("color_octree_smoke")
