"""Loop-closure re-fusion (DESIGN.md f4) on the CPU: the oracle's orc_refuse_submaps / orc_transform_cloud bit for bit
against the independent restatement of tests/refuse_cases.py on every crafted submap pair, and the host-side outer
loops of gem_b200/submaps.py (kd-tree neighbours, pair order, pose update) on crafted centre sets."""
import numpy as np
import pytest

import oracle_lib
import refuse_cases as rc
from gem_b200 import submaps as sm

F = np.float32


def check_pair(got, want, what):
    (gn, go, gf), (wn, wo, wf, fn, fo) = got, want
    assert gf == wf, (what, "fused", gf, wf)
    for side, g, w, fused in (("new", gn, wn, fn), ("old", go, wo, fo)):
        d = rc.first_difference(g, w, fused)
        assert d is None, (what, side, "n", g.shape[0], w.shape[0], "first difference (row, field, got, want)", d)


@pytest.mark.parametrize("compat", [True, False], ids=["compat", "weighted"])
@pytest.mark.parametrize("name", rc.case_names())
def test_oracle_matches_restatement(name, compat):
    new, old, res = rc.case_by_name(name)
    check_pair(oracle_lib.refuse_submaps(new, old, res, compat), rc.refuse(new, old, res, compat), (name, compat))


def test_cases_reach_their_edges():
    """what each crafted case is there for actually happens in it"""
    new, old, res = rc.case_by_name("variance_gate")
    _, _, fused, _, fo = rc.refuse(new, old, res)
    assert fused == 6                               # subnormals (3), FLT_MIN, 0.5, nextafter(1, 0); not 0, -0, 1, NaN, inf
    assert fo.sum() == 6
    new, old, res = rc.case_by_name("nan_positions")
    n2, o2, fused, fn, _ = rc.refuse(new, old, res)
    nanpos = np.isnan(new[:, 0]) | np.isnan(new[:, 1])
    assert np.isnan(n2[:, :2]).any(axis=1).sum() == nanpos.sum()            # every NaN-positioned point stays
    assert not fn[np.isnan(n2[:, :2]).any(axis=1)].any()                     # and fuses with nothing
    assert np.isinf(n2[fn, :2]).any()                                        # an infinite position is a cell like any other
    new, old, res = rc.case_by_name("one_cell_200k")
    n2, o2, fused, _, _ = rc.refuse(new, old, res)
    assert (n2.shape[0], o2.shape[0], fused) == (4, 6, 4)                   # the big cell and the three lead cells
    for n in (40, 1000):
        new, old, res = rc.case_by_name(f"hash_wrap_{n}")
        s = rc.hash_slot(rc.cell_centre(new[:, 0], res), rc.cell_centre(new[:, 1], res), rc.table_mask(n))
        assert (s == 0).any()
        keys = set(zip(rc.cell_centre(new[:, 0], res)[s == rc.table_mask(n)].tolist(),
                       rc.cell_centre(new[:, 1], res)[s == rc.table_mask(n)].tolist()))
        assert len(keys) >= 2                                                # the chain from the last slot wraps
    new, old, res = rc.case_by_name("distinct_full_load")
    assert rc.table_mask(new.shape[0]) + 1 == 2 * new.shape[0] + 2
    n2, o2, _, _, _ = rc.refuse(new, old, res)
    assert n2.shape[0] == new.shape[0] and o2.shape[0] == old.shape[0]
    for name in ("utm_scale_res0.25", "utm_scale_res0.5"):
        new, old, res = rc.case_by_name(name)
        for c in (0, 1):
            rx = rc.cell_centre(new[:, c], res)
            big = np.abs(new[:, c]) > 1e5
            assert big.sum() >= 32 and (rc.cell_centre(rx[big], res) != rx[big]).all()
        _, o2, fused, _, fo = rc.refuse(new, old, res)
        assert fused == new.shape[0] and o2.shape[0] == 500_000 + new.shape[0] and fo[-new.shape[0]:].all()
    for r in (0.1, 0.05):                           # no float re-keys at these resolutions, from 2^19 to 2^20 m
        x = np.arange(*np.array([2.0 ** 19 - 512, 2.0 ** 20 + 512], np.float32).view(np.uint32),
                      dtype=np.uint32).view(np.float32)
        rx = rc.cell_centre(x, r)
        assert (rc.cell_centre(rx, r) == rx).all()


def test_fused_values_by_hand():
    """one fused cell, the two expressions written out with numpy float64 scalars"""
    rng = rc._rng("by hand")
    new = rc.records(rng, [0.03], [0.04], var=0.2, z=1.0)
    old = rc.records(rng, [0.09], [0.01], var=0.4, z=4.0)
    vn2, vo2 = np.float64(F(0.2)) ** 2, np.float64(F(0.4)) ** 2
    for compat, e, v in ((True, vn2 * 4.0 + vo2 * 1.0 / vo2 + vn2, vo2 * vn2 / vo2 + vn2),
                         (False, (vn2 * 4.0 + vo2 * 1.0) / (vo2 + vn2), vo2 * vn2 / (vo2 + vn2))):
        n2, o2, fused, _, _ = rc.refuse(new, old, 0.1, compat)
        assert fused == 1
        for p in (n2, o2):
            assert p[0, 2] == F(e) and p[0, 5] == F(v) and p[0, 4].view(np.uint32) == new[0, 4].view(np.uint32)
            assert p[0, 0] == F(0.05) and p[0, 1] == F(0.05) and p[0, 3] == 1


@pytest.mark.parametrize("m", list(rc.MATRICES))
def test_transform_cloud_matches_restatement(m):
    p = rc.transform_input()
    got, want = oracle_lib.transform_cloud(p, rc.MATRICES[m]), rc.transform(p, rc.MATRICES[m])
    assert rc.transform_difference(got, want) is None, (m, rc.transform_difference(got, want))
    assert np.array_equal(got.view(np.uint32)[:, 3:], p.view(np.uint32)[:, 3:])


# ---- the host-side outer loops ---------------------------------------------------------------------------------------
def neighbours_restated(centres, i, radius):
    """radius search in float32 squared distances, nearest first, ties by index"""
    c = [(F(a), F(b)) for a, b in centres]
    r2 = F(radius) * F(radius)
    d2 = [F((x - c[i][0]) * (x - c[i][0]) + (y - c[i][1]) * (y - c[i][1])) for x, y in c]
    return sorted((k for k in range(len(c)) if d2[k] <= r2), key=lambda k: (d2[k], k))


CENTRES = {
    "ties": [(0, 0), (5, 0), (3, -4), (0, 5), (-4, 3), (4, 3), (0, -5)],                       # all at 5 from 0
    "mixed_ties": [(0, 0), (0, 2), (1, 0), (0, -1), (2, 0), (-1, 0), (0, 1)],
    "two_only": [(0, 0), (1, 0), (100, 0), (100, 30)],
    "self_tie": [(5, 5), (5, 5), (5, 6), (5, 7), (5, 5)],
    "radius_edge": [(0, 0), (25, 0), (0, float(np.nextafter(F(25), F(30)))), (-25, 0), (0, -24.999998), (17.5, 17.85)],
}


@pytest.mark.parametrize("name", list(CENTRES))
def test_neighbours(name):
    c = CENTRES[name]
    for i in range(len(c)):
        assert sm.neighbours(c, i, 25.0) == neighbours_restated(c, i, 25.0), (name, i)
    if name == "ties":
        assert sm.neighbours(c, 0) == [0, 1, 2, 3, 4, 5, 6]
    if name == "self_tie":
        assert sm.neighbours(c, 1) == [0, 1, 4, 2, 3] and sm.neighbours(c, 4) == [0, 1, 4, 2, 3]
    if name == "radius_edge":
        assert sm.neighbours(c, 0) == [0, 5, 4, 1, 3]                # 25 m is in, one float step past it is out


def test_neighbours_random_against_restatement():
    rng = rc._rng("centres")
    c = [tuple(v) for v in np.round(rng.uniform(-40, 40, (60, 2)), 1).astype(np.float32).tolist()]
    c += c[:5]                                                         # exact duplicates: self-ties
    for r in (5.0, 25.0, 0.1):
        for i in range(len(c)):
            assert sm.neighbours(c, i, r) == neighbours_restated(c, i, r), (r, i)


class Recorder:
    """a backend that records the calls: submap k is tagged by the value k in every field; each refusion drops the last
    point of both maps and reports k_new * 100 + k_old fused cells"""

    def __init__(self):
        self.calls = []

    def transform_cloud(self, pts, T):
        self.calls.append(("transform", int(pts[0, 0]), np.array(T, np.float32)))

    def refuse_submaps(self, new, old, resolution, compat):
        a, b = int(new[0, 0]), int(old[0, 0])
        self.calls.append(("refuse", a, b, resolution, compat))
        return new.shape[0] - 1, old.shape[0] - 1, 100 * a + b


def run_recorder(centres, compat=True):
    K = len(centres)
    subs = [np.full((20, 8), k, np.float32) for k in range(K)]
    yaw = lambda a, x: np.array([[np.cos(a), -np.sin(a), 0, x], [np.sin(a), np.cos(a), 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    old = [yaw(0.1 * k, k) for k in range(K)]
    newp = [yaw(0.1 * k + 0.02, k + 0.5) for k in range(K)]
    rec = Recorder()
    out, total = sm.update_global_map(rec, subs, old, newp, centres, 0.1, 25.0, compat)
    return rec, out, total, old, newp


@pytest.mark.parametrize("name", list(CENTRES))
def test_update_global_map_pairs(name):
    c = CENTRES[name]
    rec, out, total, old, newp = run_recorder(c, compat=(name != "ties"))
    K = len(c)
    tr = [x for x in rec.calls if x[0] == "transform"]
    assert [x[1] for x in tr] == list(range(1, K))                     # submap 0 keeps its pose
    for _, k, T in tr:
        want = np.asarray(newp[k], np.float32) @ np.linalg.inv(np.asarray(old[k], np.float32))
        assert np.allclose(T, want, atol=1e-5), k
    assert all(x[0] == "transform" for x in rec.calls[:K - 1])          # every re-pose before the first refusion
    want_pairs = []
    for i in range(K):
        nb = neighbours_restated(c, i, 25.0)
        if len(nb) > 2:
            want_pairs += [(j, i) for j in nb[1:] if j != i]
    pairs = [(x[1], x[2]) for x in rec.calls if x[0] == "refuse"]
    assert pairs == want_pairs
    assert all(x[3] == 0.1 and x[4] == (name != "ties") for x in rec.calls if x[0] == "refuse")
    assert total == sum(100 * a + b for a, b in pairs)
    for k in range(K):                                                  # each call shortens both maps by one
        assert out[k].shape[0] == 20 - sum((a == k) + (b == k) for a, b in pairs), k
    if name == "two_only":
        assert pairs == []
    if name == "self_tie":
        assert (1, 1) not in pairs and (0, 1) not in pairs and (2, 1) in pairs and (4, 0) in pairs
