"""The global-map octrees, CPU side: the oracle (tests/orc_color_octree.c) against the independent Python restatement of
tests/octree_cases.py, bit for bit, on every crafted family and on natural split clouds; the stream decoder's structure
and O5 checks on the oracle's streams; the ctypes mirror of gem_octree; the C++ facade program compiles."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import octree_cases as oc
import octree_oracle
import split_oracle
import submap_oracle
from gem_b200 import synth
from oracle_lib import OracleMap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
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


def test_gem_octree_struct_matches_the_header(tmp_path):
    import gem_b200._lib as L
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gem_b200.h"\nint main(void){gem_octree s;'
                   'printf("%zu %zu %zu %zu %zu\\n", sizeof s, offsetof(gem_octree, nodes), offsetof(gem_octree, leaves),'
                   ' offsetof(gem_octree, inserted), offsetof(gem_octree, skipped));return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    S = L.GemOctree
    assert got == [C.sizeof(S), S.nodes.offset, S.leaves.offset, S.inserted.offset, S.skipped.offset]


def test_facade_program_with_color_octree_compiles():
    tmp = tempfile.mkdtemp(prefix="gem_color_octree_cxx_")
    obj = os.path.join(tmp, "color_octree_smoke.o")
    subprocess.run(["g++", "-O2", "-std=c++14", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", "-o", obj,
                    os.path.join(ROOT, "tests", "cxx", "color_octree_smoke.cpp")], check=True)
    os.remove(obj)
    os.rmdir(tmp)
