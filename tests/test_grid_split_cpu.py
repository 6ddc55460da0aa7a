"""The global-map filter, CPU side: the oracle (tests/orc_grid_split.c) against the independent cKDTree restatement of
tests/split_cases.py, bit for bit, on natural snapshot clouds and on every crafted family; the ctypes mirror of
gem_grid_split; the C++ facade program compiles."""

import numpy as np
import pytest

import native
import split_cases
import split_oracle
import submap_oracle
from gem_b200 import synth
from oracle_lib import OracleMap


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


def test_grid_split_struct_matches_the_header():
    import gem_b200._lib as L
    assert {"obstacle", "mean", "threshold"} <= {f for f, _ in L.GemGridSplit._fields_}
    native.assert_struct_layouts({"gem_grid_split": L.GemGridSplit}, std=None)


def test_facade_program_with_grid_cloud_split_compiles():
    native.facade_compiles("grid_split_smoke")
