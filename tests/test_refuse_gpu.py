"""Loop-closure re-fusion on the device (DESIGN.md f4) byte for byte against the oracle: gem_refuse_submaps on every
crafted pair of tests/refuse_cases.py in both precedence modes (output records, n_new, n_old, fused, and the same bytes
from a second call), gem_transform_cloud on non-rigid, NaN and large-translation matrices, update_global_map through
the device over a chain of submaps, and the argument checks of both calls."""
import ctypes as C

import numpy as np
import pytest
import torch

import gem_b200
import oracle_lib
import refuse_cases as rc
from gem_b200 import submaps as sm

pytestmark = pytest.mark.gpu
GEM_ERR_INVALID = 1


@pytest.fixture(scope="module")
def emap():
    return gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)


def dev(a):
    return torch.from_numpy(np.array(a, np.float32, copy=True).reshape(-1, 8)).to("cuda:0")


def device_refuse(g, new, old, res, compat):
    dn, do = dev(new), dev(old)
    nn, no, fused = g.refuse_submaps(dn, do, res, compat)
    return dn[:nn].cpu().numpy(), do[:no].cpu().numpy(), fused


def assert_pair(got, want, fused_rows, what):
    (gn, go, gf), (wn, wo, wf) = got, want
    for side, g, w, fused in (("new", gn, wn, fused_rows[0]), ("old", go, wo, fused_rows[1])):
        assert g.shape[0] == w.shape[0], (what, side, "n", g.shape[0], w.shape[0])
        d = rc.first_difference(g, w, fused)
        assert d is None, (what, side, "first difference (row, field, device bits, oracle bits)", d)
    assert gf == wf, (what, "fused", gf, wf)


@pytest.mark.parametrize("compat", [True, False], ids=["compat", "weighted"])
@pytest.mark.parametrize("name", rc.case_names())
def test_crafted(emap, name, compat):
    new, old, res = rc.case_by_name(name)
    want = oracle_lib.refuse_submaps(new, old, res, compat)
    fused_rows = rc.refuse(new, old, res, compat)[3:]
    got = device_refuse(emap, new, old, res, compat)
    assert_pair(got, want, fused_rows, (name, "compat" if compat else "weighted"))
    again = device_refuse(emap, new, old, res, compat)
    for a, b in zip(got[:2], again[:2]):
        assert a.tobytes() == b.tobytes(), (name, "a second call on the same inputs gave other bytes")
    assert got[2] == again[2]


@pytest.mark.parametrize("m", list(rc.MATRICES))
def test_transform_cloud(emap, m):
    p = rc.transform_input()
    d = dev(p)
    emap.transform_cloud(d, rc.MATRICES[m])
    got = d.cpu().numpy()
    want = oracle_lib.transform_cloud(p, rc.MATRICES[m])
    assert rc.transform_difference(got, want) is None, (m, rc.transform_difference(got, want))
    d2 = dev(p)
    emap.transform_cloud(d2, rc.MATRICES[m])
    assert d2.cpu().numpy().tobytes() == got.tobytes()


class OracleBackend:
    def transform_cloud(self, pts, T):
        pts[:] = oracle_lib.transform_cloud(pts, T)

    def refuse_submaps(self, new, old, resolution, compat):
        n2, o2, fused = oracle_lib.refuse_submaps(new, old, resolution, compat)
        new[:n2.shape[0]] = n2
        old[:o2.shape[0]] = o2
        return n2.shape[0], o2.shape[0], fused


def chain_submaps(k_maps=7, res=0.1):
    """overlapping submaps within 25 m of each other: every submap is the new map of some pairs and the old map of later
    ones, and shrinks between calls"""
    rng = rc._rng("chain")
    centres = [(2.0 * k, 1.5 * (k % 3)) for k in range(k_maps)]
    subs = []
    for k, (cx, cy) in enumerate(centres):
        n = [700, 3100, 1025, 2048, 4000, 1500, 2600, 900][k]
        c = rng.integers(0, n // 2, n)
        ix, iy = c % 60 + int(cx / res) - 30, c // 60 + int(cy / res) - 10
        x, y = rc.in_cell(rng, ix, iy, res)
        subs.append(rc.records(rng, x, y, var=rng.choice(np.array([0.2, 0.5, 0.8, 1.0], np.float32), n)))
    yaw = lambda a, x, y: np.array([[np.cos(a), -np.sin(a), 0, x], [np.sin(a), np.cos(a), 0, y], [0, 0, 1, 0.01],
                                    [0, 0, 0, 1]], np.float32)
    old = [yaw(0.05 * k, cx, cy) for k, (cx, cy) in enumerate(centres)]
    new = [yaw(0.05 * k + 0.002, cx + 0.03, cy - 0.02) for k, (cx, cy) in enumerate(centres)]
    return subs, old, new, centres


@pytest.mark.parametrize("compat", [True, False], ids=["compat", "weighted"])
def test_update_global_map_chain(emap, compat):
    subs, old, new, centres = chain_submaps()
    ora, fo = sm.update_global_map(OracleBackend(), [s.copy() for s in subs], old, new, centres, 0.1, 25.0, compat)
    devs, fd = sm.update_global_map(emap, [dev(s) for s in subs], old, new, centres, 0.1, 25.0, compat)
    assert fd == fo and fo > 1000
    for k, (a, b) in enumerate(zip(devs, ora)):
        a = a.cpu().numpy()
        assert a.shape[0] < subs[k].shape[0], k                          # every map shrank
        d = rc.first_difference(a, b, np.ones(b.shape[0], bool))
        assert d is None, ("chain", k, d)


def test_argument_checks(emap):
    """bad arguments are refused with GEM_ERR_INVALID and leave the clouds and counts as they were"""
    lib, h = emap._lib, emap._h
    new, old, _ = rc.case_by_name("sizes_1023_1025")
    dn, do = dev(new), dev(old)
    pn, po = C.c_void_p(dn.data_ptr()), C.c_void_p(do.data_ptr())
    fused = C.c_int(-7)

    def refuse(p_new, n_new, p_old, n_old, res, with_counts=True):
        a, b = C.c_int(n_new), C.c_int(n_old)
        rc_ = lib.gem_refuse_submaps(h, p_new, C.byref(a) if with_counts else None, p_old,
                                     C.byref(b) if with_counts else None, res, 1, C.byref(fused))
        return rc_, a.value, b.value

    bad = [(pn, -1, po, 5, 0.1), (pn, 5, po, -1, 0.1), (None, 5, po, 5, 0.1), (pn, 5, None, 5, 0.1),
           (pn, 5, po, 5, 0.0), (pn, 5, po, 5, -0.1), (pn, 5, po, 5, float("nan")), (pn, 5, po, 5, -float("inf")),
           (pn, 5, po, 5, -0.0)]
    for args in bad:
        assert refuse(*args) == (GEM_ERR_INVALID, args[1], args[3]), args
    assert lib.gem_refuse_submaps(h, pn, None, po, C.byref(C.c_int(5)), 0.1, 1, C.byref(fused)) == GEM_ERR_INVALID
    assert lib.gem_refuse_submaps(h, pn, C.byref(C.c_int(5)), po, None, 0.1, 1, C.byref(fused)) == GEM_ERR_INVALID
    assert fused.value == -7
    assert refuse(None, 0, None, 0, 0.1) == (0, 0, 0) and fused.value == 0   # empty sides need no pointer
    T = (C.c_float * 16)(*np.eye(4, dtype=np.float32).reshape(-1).tolist())
    assert lib.gem_transform_cloud(h, pn, -1, T) == GEM_ERR_INVALID
    assert lib.gem_transform_cloud(h, None, 3, T) == GEM_ERR_INVALID
    assert lib.gem_transform_cloud(h, pn, 3, None) == GEM_ERR_INVALID
    assert lib.gem_transform_cloud(h, None, 0, T) == 0
    torch.cuda.synchronize()
    assert dn.cpu().numpy().tobytes() == new.tobytes() and do.cpu().numpy().tobytes() == old.tobytes()
    got = device_refuse(emap, new, old, 0.1, True)                       # the handle still works
    assert_pair(got, oracle_lib.refuse_submaps(new, old, 0.1, True), rc.refuse(new, old, 0.1, True)[3:], "after errors")
