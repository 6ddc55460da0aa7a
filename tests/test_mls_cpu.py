"""The MLS oracle (tests/orc_mls.c, DESIGN.md f10) pinned independently of its operation order: on every crafted case of
tests/mls_cases.py its neighbour lists equal scipy's cKDTree ball query under M2's float rule, its plane normal, Darboux
axes and polynomial coefficients equal a numpy float64 restatement (eigh, unitOrthogonal, a weighted least-squares
solve), its M5 positions lie within 1e-6 m of the restatement's, its sample counts are M6's exactly, every sample lies in
the disc, and the generator is reproducible and seeded.  Also: gem_mathd.h's exp against libm and its atan2 / sincos
against the restatement of gem_math.cuh's, the ABI structs against the header, and that the facade program compiles."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial import cKDTree

import mls_cases as mc
import mls_oracle
from gem_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def full(o):
    q = dict(mls_oracle.GEM)
    q.update(o)
    return q


def neighbours(xyz, i, r):
    """M2 by scipy: the ball query with a margin, then the float rule, sorted by (d2, index)"""
    fin = np.isfinite(xyz).all(1)
    if not fin[i]:
        return np.zeros(0, np.int64)
    idx = np.flatnonzero(fin)
    tree = cKDTree(xyz[idx].astype(np.float64))
    cand = idx[tree.query_ball_point(xyz[i].astype(np.float64), r * (1 + 1e-5))]
    d = (xyz[cand] - xyz[i]).astype(f32)
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    keep = d2 <= f32(r * r)
    cand, d2 = cand[keep], d2[keep]
    return cand[np.lexsort((cand, d2))]


def unit_orthogonal(n):
    if not (abs(n[0]) <= abs(n[2]) * 1e-12) or not (abs(n[1]) <= abs(n[2]) * 1e-12):
        return np.array([-n[1], n[0], 0.0]) / np.hypot(n[0], n[1])
    return np.array([0.0, -n[2], n[1]]) / np.hypot(n[1], n[2])


def monomials(u, v, order):
    return np.stack([u ** a * v ** b for a in range(order + 1) for b in range(order + 1 - a)], -1)


def pinned_points(n):
    return range(n) if n <= 60 else np.linspace(0, n - 1, 60).astype(int)


@pytest.mark.parametrize("name", mc.case_names())
def test_oracle_against_numpy(name):
    _, recs, o = mc.case_by_name(name)
    q = full(o)
    r, order = q["search_radius"], q["order"]
    nc = (order + 1) * (order + 2) // 2
    xyz = recs[:, :3]
    res = mls_oracle.upsample(recs, o)
    assert res is not None
    out, info = res
    counts = []
    for i in range(recs.shape[0]):
        nb = neighbours(xyz, i, r)
        counts.append(nb.size if np.isfinite(xyz[i]).all() else -1)
    counts = np.array(counts)
    # M6 / M8: the counts follow from the neighbour counts alone
    proc = counts >= 3
    k = np.floor(q["point_density"] / 2.0 / np.maximum(counts, 1)).astype(int) if q["upsampling"] != "none" else np.zeros_like(counts)
    per = np.where(proc, np.where(k > 0, k, 1), 0)
    assert info["count"] == per.sum() and info["processed"] == proc.sum() and info["skipped"] == (~proc).sum()
    assert info["max_neighbours"] == max(0, counts.max(initial=0))
    offs = np.concatenate([[0], np.cumsum(per)])
    for i in pinned_points(recs.shape[0]):
        d = mls_oracle.detail(recs, i, o)
        nb = neighbours(xyz, i, r)
        assert np.array_equal(d["nb"], nb), (name, i)
        if nb.size < 3:
            continue
        P = xyz[nb].astype(np.float64)
        cen = P.mean(0)
        w, V = np.linalg.eigh((P - cen).T @ (P - cen))
        n = d["normal"]
        assert abs(np.linalg.norm(n) - 1) < 1e-12
        if w[1] - w[0] > 1e-6 * max(w[2], 1e-300):   # the smallest eigenvector is unique
            assert 1 - abs(n @ V[:, 0]) < 1e-9, (name, i, n, V[:, 0])
        qd = xyz[i].astype(np.float64)
        pt = qd - ((qd - cen) @ n) * n
        assert np.allclose(d["point"], pt, rtol=0, atol=1e-9 * max(1.0, np.abs(qd).max())), (name, i)
        if not d["attempted"]:
            assert not d["fitted"] and not d["u_axis"].any() and not d["v_axis"].any()
            continue
        va = unit_orthogonal(n)
        ua = np.cross(n, va)
        assert np.allclose(d["v_axis"], va, rtol=0, atol=1e-14) and np.allclose(d["u_axis"], ua, rtol=0, atol=1e-14)
        de = P - d["point"]
        wt = np.exp(-(np.sum(de * de, 1).astype(f32).astype(np.float64)) / q["sqr_gauss_param"])
        M = monomials(de @ d["u_axis"], de @ d["v_axis"], order)
        f = de @ n
        A = M.T @ (M * wt[:, None])
        cond = np.linalg.cond(A)
        if cond > 1e13:   # singular to double precision: the oracle's fit must have failed or be meaningless
            continue
        assert d["fitted"], (name, i, cond)
        sw = np.sqrt(wt)
        c = np.linalg.lstsq(M * sw[:, None], f * sw, rcond=None)[0]
        # the normal equations square the condition number: the tolerance scales with it, 1e-9 at cond <= 1e4
        tol = 1e-9 * max(1.0, cond / 1e4)
        assert np.allclose(d["c"][:nc], c, rtol=0, atol=tol * max(1.0, np.abs(c).max())), (name, i, cond)
        if q["upsampling"] == "none" or per[i] == 1:
            want = d["point"] + c[0] * n
            assert np.abs(out[offs[i], :3] - want).max() < 1e-6, (name, i)
    # M7 and the disc: every sample of a processed point carries its attributes and lies inside r / 2 in the plane
    for i in np.flatnonzero(per > 1)[:40]:
        d = mls_oracle.detail(recs, i, o)
        s = out[offs[i]:offs[i + 1]]
        assert np.all(s[:, 3] == 1.0) and np.all(s[:, 5:] == recs[i, 5:])
        bg = recs[i, 4:5].view(np.uint32)[0]
        assert np.all(s[:, 4].view(np.uint32) == (bg | 0xFF000000))
        rel = s[:, :3].astype(np.float64) - d["point"]
        if d["attempted"]:
            uv = np.stack([rel @ d["u_axis"], rel @ d["v_axis"]], 1)
            assert np.all(np.sum(uv * uv, 1) <= r * r / 4 * (1 + 1e-4) + 1e-10), (name, i)
        else:
            assert np.abs(rel).max() < 1e-5 * max(1.0, np.abs(d["point"]).max())


def test_crafted_cases_reach_their_targets():
    got = {name: mls_oracle.upsample(recs, o)[1] for name, recs, o in mc.cases()}
    assert got["two_neighbours"]["processed"] == 0 and got["three_neighbours"]["processed"] == 3
    assert got["cluster_20_neighbours"]["fitted"] == 0 and got["cluster_21_neighbours"]["fitted"] == 21
    assert got["collinear_singular"]["fitted"] == 0 and got["collinear_singular"]["processed"] == 40
    assert got["long_list_over_shared_budget"]["max_neighbours"] > 512
    assert got["density_k_hundreds"]["count"] >= 400 * 3
    assert got["non_finite_records"]["skipped"] == 4
    recs = mc.case_by_name("boundary_exact_radius")[1]
    assert list(mls_oracle.detail(recs, 0, mc.NONE)["nb"]) == [0, 6, 1, 2, 3]   # d2 == (float)(r r) included, the next float out


def test_generator_reproducible_and_seeded():
    _, recs, o = mc.case_by_name("noisy_surface_order3")
    a, ia = mls_oracle.upsample(recs, dict(o, seed=1))
    b, ib = mls_oracle.upsample(recs, dict(o, seed=1))
    c, ic = mls_oracle.upsample(recs, dict(o, seed=2))
    assert a.tobytes() == b.tobytes() and ia == ib
    assert ic == ia and a.shape == c.shape and a.tobytes() != c.tobytes()


def test_invalid_parameters():
    recs = mc.case_by_name("tilted_lattice_plane")[1]
    for kw in ({"search_radius": 0.0}, {"search_radius": float("nan")}, {"sqr_gauss_param": -1.0}, {"sqr_gauss_param": float("inf")},
               {"order": 0}, {"order": 6}, {"upsampling": 2}, {"point_density": -1}):
        assert mls_oracle.upsample(recs, kw) is None, kw


def test_exp_d_against_libm():
    rng = np.random.default_rng(3)
    x = np.concatenate([rng.uniform(-745, 709, 20000), rng.uniform(-5, 0, 20000), [0.0, -0.0, 1.0, -1.0, 709.7, -744.0]])
    got, want = mls_oracle.exp_d(x), np.exp(x)
    ulp = np.abs(got - want) / np.spacing(np.abs(want))
    normal = want >= 2.2250738585072014e-308
    assert ulp[normal].max() <= 2, ulp[normal].max()
    assert np.all(np.abs(got[~normal] - want[~normal]) <= 2 * 5e-324)
    assert mls_oracle.exp_d([np.inf, -np.inf, 800.0, -800.0]).tolist() == [np.inf, 0.0, np.inf, 0.0]
    assert np.isnan(mls_oracle.exp_d([np.nan])[0])


def test_atan2_sincos_equal_gem_math():
    """gem_mathd.h's atan2 / sincos are gem_math.cuh's definitions: equal bit for bit to test_map_cases' restatement of it"""
    from test_map_cases import _atan2_d, _sincos_d
    rng = np.random.default_rng(4)
    y, x = rng.normal(0, 3, 5000), rng.normal(0, 3, 5000)
    assert mls_oracle.atan2_d(y, x).tobytes() == _atan2_d(y, x).tobytes()
    t = rng.uniform(-10, 10, 5000)
    sc = mls_oracle.sincos_d(t)
    s, c = _sincos_d(t)
    assert sc[:, 0].tobytes() == np.asarray(s, np.float64).tobytes() and sc[:, 1].tobytes() == np.asarray(c, np.float64).tobytes()


def test_abi_structs_match_header():
    assert C.sizeof(_lib.GemMlsParams) == 40 and C.sizeof(_lib.GemMlsInfo) == 24
    assert [f for f, _ in _lib.GemMlsParams._fields_] == [f for f, _ in mls_oracle.Params._fields_]
    assert [f for f, _ in _lib.GemMlsInfo._fields_] == [f for f, _ in mls_oracle.Info._fields_]
    src = ("#include <stddef.h>\n#include \"gem_b200.h\"\n"
           "_Static_assert(sizeof(gem_mls_params) == 40, \"p\");\n_Static_assert(sizeof(gem_mls_info) == 24, \"i\");\n"
           "_Static_assert(offsetof(gem_mls_params, seed) == 32, \"s\");\n_Static_assert(offsetof(gem_mls_info, max_neighbours) == 20, \"m\");\n"
           "_Static_assert(GEM_MLS_NONE == 0 && GEM_MLS_RANDOM_UNIFORM_DENSITY == 1, \"e\");\n")
    subprocess.run(["gcc", "-std=c11", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), "-x", "c", "-"], input=src, text=True,
                   check=True)


def test_facade_program_compiles():
    subprocess.run(["g++", "-std=c++14", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cxx", "mls_smoke.cpp")], check=True)
