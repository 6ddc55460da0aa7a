"""The global map's submap stack without a GPU (DESIGN.md f16): the oracle (tests/orc_global_map.c over orc_transform_cloud
and orc_refuse_submaps) against the independent Python restatement on the crafted call sequences of
tests/global_map_cases.py, and the library's host pose arithmetic and pair schedule (a g++ build of gem_globalmap.h)
against the restatement, bit for bit."""
import ctypes as C
import os

import numpy as np
import pytest

import global_map_cases as gc
import global_map_oracle as go
import native
from gem_b200 import submaps as sm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("compat", [True, False], ids=["compat", "weighted"])
@pytest.mark.parametrize("name", list(gc.CASES))
def test_oracle_equals_restatement(name, compat):
    ops = gc.CASES[name]()
    fo, so = gc.run(go.OracleStack(), ops, compat)
    fp, sp = gc.run(go.PyStack(), ops, compat)
    assert fo == fp, (name, fo, fp)
    for step, (a, b) in enumerate(zip(so, sp)):
        assert go.stack_difference(a, b) is None, (name, step, go.stack_difference(a, b))


def test_cases_reach_their_decisions():
    """the gate cases fuse only from K = 3 on, k = 0 changes nothing, the NaN centre and empty submaps survive"""
    fused = {n: gc.run(go.OracleStack(), gc.CASES[n]())[0] for n in gc.CASES}
    assert fused["gate_K0"] == fused["gate_K1"] == fused["gate_K2"] == [0] and fused["gate_K3"][0] > 0
    assert fused["k_0"] == [0] and fused["k_2"] == [0] and fused["k_4"][0] > 0
    assert all(f > 0 for f in fused["sequence"]) and fused["variance"][0] > 0
    ops = gc.CASES["k_2"]()
    _, states = gc.run(go.OracleStack(), ops)
    before, after = states[-2], states[-1]
    assert go.stack_difference((before[0][2:], before[1][2:], before[2]), (after[0][2:], after[1][2:], after[2])) is None
    assert (after[1][1] != before[1][1]).any()          # keyframe 1 took its optimised pose, the tail kept theirs


@pytest.fixture(scope="module")
def host():
    lib = native.shared_library("gm_host", [os.path.join(ROOT, "tests", "global_map_host.cpp")], native.HOST_CXX + ["-Werror"])
    lib.gm_relative_pose.argtypes = [C.c_void_p] * 3
    lib.gm_pair_schedule.restype = C.c_int
    lib.gm_pair_schedule.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_int]
    return lib


def _poses(seed, n):
    rng = np.random.default_rng(seed)
    out = [gc.pose(x=x, y=y, z=z, q=rng.normal(size=4)) for x, y, z in rng.uniform(-1e3, 1e3, (n, 3))]
    out += [gc.pose(x=448_251.3 + d, y=5_411_937.6 - d, q=rng.normal(size=4)) for d in rng.uniform(-50, 50, n)]
    rough = rng.normal(size=(n, 4, 4)).astype(np.float32)          # any floats: the arithmetic is defined on all of them
    return out + list(rough)


def test_host_pose_arithmetic(host):
    P = _poses(1, 300)
    for pn, po in zip(P, P[1:] + P[:1]):
        want = go.relative_pose(pn, po)
        got = np.empty(16, np.float32)
        a, b = np.ascontiguousarray(pn, np.float32), np.ascontiguousarray(po, np.float32)
        host.gm_relative_pose(a.ctypes.data, b.ctypes.data, got.ctypes.data)
        assert got.view(np.uint32).tolist() == want.reshape(-1).view(np.uint32).tolist()
        assert go.oracle_relative_pose(pn, po).view(np.uint32).tolist() == want.view(np.uint32).tolist()


def _schedule(centres, radius):
    c = np.asarray(centres, np.float32).reshape(-1, 2)
    pairs = []
    with np.errstate(invalid="ignore"):
        for i in range(c.shape[0]):
            nb = sm.neighbours(c, i, radius)
            if len(nb) > 2:
                pairs += [(j, i) for j in nb[1:] if j != i]
    return pairs


@pytest.mark.parametrize("seed", range(6))
def test_host_pair_schedule(host, seed):
    rng = np.random.default_rng(seed)
    K = int(rng.integers(0, 40))
    c = (rng.integers(-6, 6, (K, 2)) * 2.5).astype(np.float32)          # many ties and points at the radius exactly
    if K > 3:
        c[rng.integers(0, K)] = np.nan
    radius = float(rng.choice([0.0, 2.5, 5.0, 7.5, 25.0]))
    out = np.zeros(2 * 40 * 40, np.int32)
    n = host.gm_pair_schedule(np.ascontiguousarray(c).ctypes.data, K, radius, out.ctypes.data, 40 * 40)
    assert [tuple(p) for p in out[:2 * n].reshape(-1, 2).tolist()] == _schedule(c, radius)
