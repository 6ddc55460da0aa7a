"""The global-map filter, CPU side: the oracle (tests/orc_grid_split.c) against the independent cKDTree restatement of
tests/split_cases.py, bit for bit, on natural snapshot clouds and on every crafted family; the ctypes mirror of
gem_grid_split; the C++ facade program compiles."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import split_cases
import split_oracle
import submap_oracle
from gem_b200 import synth
from oracle_lib import OracleMap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def f64bits(v):
    return np.float64(v).view(np.uint64)


def assert_same_split(got, want, what):
    assert np.array_equal(got["dist"].view(np.uint32), want["dist"].view(np.uint32)) or (
        np.array_equal(np.isnan(got["dist"]), np.isnan(want["dist"])) and np.isnan(got["dist"]).all()), what
    assert got["valid"] == want["valid"], (what, got["valid"], want["valid"])
    for k in ("mean", "stddev", "threshold"):
        a, b = got[k], want[k]
        assert f64bits(a) == f64bits(b) or (np.isnan(a) and np.isnan(b)), (what, k, a, b)
    for k in ("road", "obstacle"):
        assert got[k].shape == want[k].shape and np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), (what, k)


@pytest.mark.parametrize("name", [c[0] for c in split_cases.cloud_cases()])
def test_oracle_matches_restatement_on_crafted_clouds(name):
    _, rec, params = next(c for c in split_cases.cloud_cases() if c[0] == name)
    for mean_k, mul, tt in params:
        got = split_oracle.grid_split(rec, mean_k, mul, tt)
        want = split_cases.np_grid_split(rec, mean_k, mul, tt)
        assert_same_split(got, want, (name, mean_k, mul, tt))
    if name == "pairs":   # every distance is 0.25 = the threshold: nothing removed
        got = split_oracle.grid_split(rec, 1, 1.0, 0.0)
        assert got["mean"] == 0.25 and got["stddev"] == 0.0
        assert got["road"].shape[0] + got["obstacle"].shape[0] == rec.shape[0]
    if name == "count_20":
        assert split_oracle.grid_split(rec, 20)["valid"] == 0
    if name == "count_21":
        assert split_oracle.grid_split(rec, 20)["valid"] == 21


@pytest.mark.parametrize("L", [128, 101])
def test_oracle_matches_restatement_on_snapshot_clouds(L):
    res = 0.1
    o = OracleMap(L, res, compat_box_filter=False)
    scene = synth.make_scene()
    pos = np.array([0.3, -0.2, 1.7], np.float32)
    for k in range(3):
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([0.4, 0.3, 0.0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        o.move(pos)
        import gem_b200
        o.add(fr["xyzi"], fr["rgba"], gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
        o.compute_features()
        o.snapshot_shown()
    f, centre, start = o._prev
    rec = submap_oracle.grid_cloud(f, L, centre, start, res)
    assert rec.shape[0] > 300
    for mean_k, mul, tt in ((20, 1.0, 0.0), (2, -1.0, 0.5), (64, 0.0, 0.0)):
        got = split_oracle.grid_split(rec, mean_k, mul, tt)
        want = split_cases.np_grid_split(rec, mean_k, mul, tt)
        assert_same_split(got, want, (L, mean_k))
        assert got["valid"] == rec.shape[0]


def test_grid_split_struct_matches_the_header(tmp_path):
    import gem_b200._lib as L
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gem_b200.h"\nint main(void){gem_grid_split s;'
                   'printf("%zu %zu %zu %zu\\n", sizeof s, offsetof(gem_grid_split, obstacle), offsetof(gem_grid_split, mean),'
                   ' offsetof(gem_grid_split, threshold));return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    S = L.GemGridSplit
    assert got == [C.sizeof(S), S.obstacle.offset, S.mean.offset, S.threshold.offset]


def test_facade_program_with_grid_cloud_split_compiles():
    tmp = tempfile.mkdtemp(prefix="gem_grid_split_cxx_")
    obj = os.path.join(tmp, "grid_split_smoke.o")
    subprocess.run(["g++", "-O2", "-std=c++14", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", "-o", obj,
                    os.path.join(ROOT, "tests", "cxx", "grid_split_smoke.cpp")], check=True)
    os.remove(obj)
    os.rmdir(tmp)
