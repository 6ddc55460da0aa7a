"""The crafted map cases (tests/map_cases.py) on the CPU: an independent numpy restatement of the feature step and the
ray clean-up pins the oracle on every case, and its counters prove that every family reaches what its name says.

The feature restatement is written from G_Mapfeature + computerEigenvalue (gpu_process.cu:549-670, :66-187) with
the deterministic trig of gem_b200/csrc/gem_math.cuh restated in float64: float32 per operation, no contraction,
double where the reference promotes, the pivot search and the rotation with dynamic indices over the full 3 x 3
matrix as the reference spells them.  It runs vectorised over the cells whose elevation is valid."""
import numpy as np
import pytest

import map_cases as mc
import np_reference
from oracle_lib import OracleMap

f32 = np.float32


# ---------------------------------------------------------------------------------------------------------------------
# deterministic trig (gem_math.cuh), float64, vectorised
# ---------------------------------------------------------------------------------------------------------------------
_SIN = (-2.81145725434552076320e-15, 7.64716373181981647590e-13, -1.60590438368216145994e-10,
        2.50521083854417187751e-08, -2.75573192239858906526e-06, 1.98412698412698412698e-04,
        -8.33333333333333333333e-03, 1.66666666666666666667e-01)
_COS = (-1.56192069685862264622e-16, 4.77947733238738529744e-14, -1.14707455977297247139e-11,
        2.08767569878680989792e-09, -2.75573192239858906526e-07, 2.48015873015873015873e-05,
        -1.38888888888888888889e-03, 4.16666666666666666667e-02, -0.5)


def _sincos_d(x):
    x = np.asarray(x, np.float64)
    with np.errstate(all="ignore"):
        bad = ~np.isfinite(x)
        xs = np.where(bad, 0.0, x)
        kd = np.floor(xs * 0.63661977236758134308 + 0.5)
        r = (xs - kd * 1.57079632673412561417e+00) - kd * 6.07710050650619224932e-11
        r2 = r * r
        p = np.full_like(r, _SIN[0])
        for c in _SIN[1:]:
            p = p * r2 + c
        sr = r - (r * r2) * p
        p = np.full_like(r, _COS[0])
        for c in _COS[1:]:
            p = p * r2 + c
        cr = 1.0 + r2 * p
        k = kd.astype(np.int64) & 3
        s = np.choose(k, [sr, cr, -sr, -cr])
        c = np.choose(k, [cr, -sr, -cr, sr])
        nan = x - x
        return np.where(bad, nan, s), np.where(bad, nan, c)


def _atan_poly(t):
    t2 = t * t
    p = np.zeros_like(t)
    for n in range(43, 2, -2):
        coef = 1.0 / n
        if ((n - 1) // 2) & 1:
            coef = -coef
        p = (p + coef) * t2
    return t + t * p


def _atan_core(z):
    with np.errstate(all="ignore"):
        big = z > 0.41421356237309503
        t = (z - 1.0) / (z + 1.0)
        return np.where(big, 0.78539816339744830962 + _atan_poly(t), _atan_poly(z))


def _atan2_d(y, x):
    y = np.asarray(y, np.float64)
    x = np.asarray(x, np.float64)
    with np.errstate(all="ignore"):
        ax, ay = np.abs(x), np.abs(y)
        a = np.where((ax == 0) & (ay == 0), 0.0,
                     np.where(ay <= ax, _atan_core(ay / ax), 1.57079632679489661923 - _atan_core(ax / ay)))
        a = np.where(x < 0, 3.14159265358979323846 - a, a)
        a = np.where(y < 0, -a, a)
        return np.where(np.isnan(y) | np.isnan(x), y + x, a)


def atan2f_det(y, x):
    return _atan2_d(np.asarray(y, f32).astype(np.float64), np.asarray(x, f32).astype(np.float64)).astype(f32)


def sinf_det(a):
    return _sincos_d(np.asarray(a, f32).astype(np.float64))[0].astype(f32)


def cosf_det(a):
    return _sincos_d(np.asarray(a, f32).astype(np.float64))[1].astype(f32)


def acosf_det(v):
    x = np.asarray(v, f32).astype(np.float64)
    with np.errstate(all="ignore"):
        ok = (x >= -1.0) & (x <= 1.0)
        xs = np.where(ok, x, 0.0)
        r = _atan2_d(np.sqrt((1.0 - xs) * (1.0 + xs)), xs)
    return np.where(ok, r, np.nan).astype(f32)


# ---------------------------------------------------------------------------------------------------------------------
# G_Mapfeature + computerEigenvalue
# ---------------------------------------------------------------------------------------------------------------------
def features_np(elev, L, res, start, n_jt=30):
    """slope, rough, traver (d_* outputs, storage-indexed, flat) and the instrumentation of every centre cell"""
    E = np.asarray(elev, f32).reshape(L, L)
    res = f32(res)
    n = L * L
    slope, rough, traver = np.zeros(n, f32), np.zeros(n, f32), np.full(n, f32(-10))
    centre = np.nonzero(E.reshape(-1) != f32(-10))[0]         # :581
    cx, cy = centre // L, centre % L
    ex0, ey0 = (cx + L - start[0]) % L, (cy + L - start[1]) % L
    m = centre.size
    pts = []
    sx, sy, sz = np.zeros(m, f32), np.zeros(m, f32), np.zeros(m, f32)
    cnt = np.zeros(m, np.int64)
    wrap = np.zeros(m, bool)                                   # a valid storage neighbour across the wrap line
    err = np.seterr(all="ignore")
    for i in range(-2, 3):
        for j in range(-2, 3):
            ex, ey = ex0 + i, ey0 + j
            inside = (ex >= 0) & (ex < L) & (ey >= 0) & (ey < L)
            qx, qy = (cx + i + L) % L, (cy + j + L) % L
            z = E[qx, qy]
            ok = inside & (z != f32(-10))
            px, py = qx.astype(f32) * res, qy.astype(f32) * res    # :606-607 int * float
            sx = np.where(ok, sx + px, sx)
            sy = np.where(ok, sy + py, sy)
            sz = np.where(ok, sz + z, sz)
            cnt += ok
            wrap |= ok & ((cx + i < 0) | (cx + i >= L) | (cy + j < 0) | (cy + j >= L))
            pts.append((ok, px, py, z))
    np.seterr(**err)
    info = {"cells": centre, "cnt": cnt, "wrap": wrap}
    go = cnt > 7                                                # :619
    with np.errstate(all="ignore"):
        c = cnt.astype(f32)
        mx, my, mz = sx / c, sy / c, sz / c
        M = np.zeros((m, 9), f32)
        for ok, px, py, z in pts:                               # :626-637, in the order of the neighbour list
            dx, dy, dz = px - mx, py - my, z - mz
            for k, v in ((0, dx * dx), (4, dy * dy), (8, dz * dz), (1, dx * dy), (2, dx * dz), (5, dy * dz)):
                M[:, k] = np.where(ok, M[:, k] + v, M[:, k])
            M[:, 3], M[:, 6], M[:, 7] = M[:, 1], M[:, 2], M[:, 5]
        V, jinfo = _jacobi(M, go, n_jt)
    info.update(jinfo)
    r = np.arange(m)
    minv, mid = M[:, 0].copy(), np.zeros(m, np.int64)           # :165-181
    ties = np.zeros(m, bool)
    for i in (1, 2):
        d = M[:, 4 * i]
        ties |= d == minv
        upd = minv > d
        ties &= ~upd
        minv = np.where(upd, d, minv)
        mid = np.where(upd, i, mid)
    info["eig_tie"] = ties & go
    nz = V[r, mid + 6]                                          # maxvector[2] = V[min_id + 3 * 2]
    with np.errstate(all="ignore"):
        sl = np.where(nz > 0, acosf_det(nz), acosf_det(-nz))    # :649-652
        ro = np.abs(E.reshape(-1)[centre] - mz)                 # :654
        tr = (0.5 * (1.0 - sl.astype(np.float64) / 0.6) + 0.5 * (1.0 - (ro.astype(np.float64) / 0.2))).astype(f32)
    slope[centre] = np.where(go, sl, f32(0))
    rough[centre] = np.where(go, ro, f32(0))
    traver[centre] = np.where(go, tr, f32(-10))
    return slope, rough, traver, info


def _jacobi(M, active, n_jt=30):
    """computerEigenvalue with nDim = 3, dbEps = 0.01, nJt = n_jt on every row of M (in place); returns the eigenvector
    matrices and what the iteration met"""
    m = M.shape[0]
    r = np.arange(m)
    V = np.tile(np.eye(3, dtype=f32).reshape(9), (m, 1))
    act = active.copy()
    count = np.zeros(m, np.int64)
    first = np.full(m, f32(np.nan))
    tie01_02 = np.zeros(m, bool)
    tie02_12 = np.zeros(m, bool)
    neg01 = np.zeros(m, bool)
    eqdiag = np.zeros(m, bool)
    for it in range(40):
        dbmax = M[:, 1].copy()                                  # :85 signed
        row, col = np.zeros(m, np.int64), np.ones(m, np.int64)
        for i in range(3):
            for j in range(3):
                if i == j:
                    continue
                d = np.abs(M[:, 3 * i + j])
                upd = d > dbmax
                dbmax = np.where(upd, d, dbmax)
                row = np.where(upd, i, row)
                col = np.where(upd, j, col)
        if it == 0:
            first = np.where(active, dbmax, first)
            a01, a02, a12 = np.abs(M[:, 1]), np.abs(M[:, 2]), np.abs(M[:, 5])
            big = dbmax >= f32(0.01)
            tie01_02 = active & big & (a01 == a02) & (a01 >= a12)
            tie02_12 = active & big & (a02 == a12) & (a02 >= a01)
            neg01 = active & big & (M[:, 1] < 0) & (a01 > a02) & (a01 > a12)
        act &= ~((dbmax < f32(0.01)) | (count > n_jt))            # :103-107
        if not act.any():
            break
        count += act
        pp, pq, qq = 3 * row + row, 3 * row + col, 3 * col + col
        app, apq, aqq = M[r, pp], M[r, pq], M[r, qq]
        eqdiag |= act & (aqq - app == 0)
        with np.errstate(all="ignore"):
            ang = (0.5 * atan2f_det(f32(-2) * apq, aqq - app).astype(np.float64)).astype(f32)   # :116
            s, c = sinf_det(ang), cosf_det(ang)
            s2, c2 = sinf_det(f32(2) * ang), cosf_det(f32(2) * ang)
            npp = (app * c * c + aqq * s * s) + f32(2) * apq * c * s                      # :122-127
            nqq = (app * s * s + aqq * c * c) - f32(2) * apq * c * s
            npq = (0.5 * (aqq - app).astype(np.float64) * s2.astype(np.float64) + (apq * c2).astype(np.float64)).astype(f32)
        upd = lambda k, v: M.__setitem__((r[act], k[act]), v[act])
        upd(pp, npp)
        upd(qq, nqq)
        upd(pq, npq)
        upd(3 * col + row, npq)
        with np.errstate(all="ignore"):
            for i in range(3):                                  # :129-139
                sel = act & (i != col) & (i != row)
                u, w = 3 * i + row, 3 * i + col
                t, mw = M[r, u], M[r, w]
                nu, nw = mw * s + t * c, mw * c - t * s
                M[r[sel], u[sel]], M[r[sel], w[sel]] = nu[sel], nw[sel]
            for j in range(3):                                  # :141-151
                sel = act & (j != col) & (j != row)
                u, w = 3 * row + j, 3 * col + j
                t, mw = M[r, u], M[r, w]
                nu, nw = mw * s + t * c, mw * c - t * s
                M[r[sel], u[sel]], M[r[sel], w[sel]] = nu[sel], nw[sel]
            for i in range(3):                                  # :154-161
                u, w = 3 * i + row, 3 * i + col
                t, vw = V[r, u], V[r, w]
                nu, nw = vw * s + t * c, vw * c - t * s
                V[r[act], u[act]], V[r[act], w[act]] = nu[act], nw[act]
    return V, {"rotations": count, "first_pivot": first, "tie01_02": tie01_02, "tie02_12": tie02_12, "neg01": neg01,
               "eqdiag": eqdiag}


def _same(a, b):
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _assert_same(a, b, what):
    ok = _same(a, b)
    if not ok.all():
        i = int(np.argmax(~ok))
        raise AssertionError(f"{what}: {int((~ok).sum())} cells differ, first at {i}: numpy={a.reshape(-1)[i]!r} "
                             f"oracle={b.reshape(-1)[i]!r}")


def _oracle(c):
    o = OracleMap(c.L, c.res, obstacle_threshold=c.obstacle_threshold)
    c.apply(o)
    return o


CASES = mc.all_cases()
IDS = [c.name for c in CASES]


_features_cache = {}


def _features(c):
    if c.name not in _features_cache:
        _features_cache[c.name] = features_np(c.elevation, c.L, c.res, c.start)
    return _features_cache[c.name]


# ---------------------------------------------------------------------------------------------------------------------
# the oracle against the restatements
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_case_applies_and_features_match_oracle(c):
    o = _oracle(c)
    centre, start, sz = o.state()
    assert tuple(start) == c.start and sz == f32(c.sensor_z)
    f = o.map_feature()
    slope, rough, traver, _ = _features(c)
    _assert_same(slope, f["slope"], f"{c.name} slope")
    _assert_same(rough, f["rough"], f"{c.name} rough")
    _assert_same(traver, f["traver"], f"{c.name} traver")
    # the traver layer: the new value where the elevation is valid, the stale one elsewhere (gpu.cu:581)
    layer = np.where(c.elevation.reshape(-1) != f32(-10), traver, c.traver.reshape(-1))
    _assert_same(layer, o.get_layer("traver").reshape(-1), f"{c.name} traver layer")


RAY_CASES = [c for c in CASES if c.L <= 64]


@pytest.mark.parametrize("c", RAY_CASES, ids=[c.name for c in RAY_CASES])
def test_rays_match_oracle(c):
    o = _oracle(c)
    o.compute_features()
    c.apply_ray(o)
    traver = o.get_layer("traver")
    r = mc.trace_rays(c.elevation, c.variance, traver, c.lowest, c.L, c.start, c.sensor_z, c.obstacle_threshold)
    o.raytracing()
    _assert_same(r["new_elevation"], o.get_layer("elevation").reshape(-1), f"{c.name} elevation")
    assert (o.get_layer("lowest") == 10).all()


@pytest.mark.parametrize("name", ["ray_ties_L16", "ray_removal_L24", "ray_low_special", "ray_obstacle_test",
                                  "ray_geom_L17_s5_16_all"])
def test_vectorised_dda_matches_scalar_reference(name):
    """trace_rays against the scalar DDA of np_reference (written separately from the same source lines)"""
    c = mc.case(name)
    tr = c.ray_traver if c.ray_traver is not None else c.traver
    r = mc.trace_rays(c.elevation, c.variance, tr, c.lowest, c.L, c.start, c.sensor_z, c.obstacle_threshold)
    ref = np_reference.raytracing(c.elevation, c.variance, tr, c.lowest, c.L, c.start, f32(c.sensor_z),
                                  thr=c.obstacle_threshold)
    _assert_same(r["new_elevation"], ref, name)


# ---------------------------------------------------------------------------------------------------------------------
# reach: every family meets what its name says
# ---------------------------------------------------------------------------------------------------------------------
def _target_info(c):
    _, _, _, info = _features(c)
    pos = {int(q): k for k, q in enumerate(info["cells"])}
    for gx, gy, tag in c.targets:
        sx, sy = (gx + c.start[0]) % c.L, (gy + c.start[1]) % c.L
        yield tag, info, pos[sx * c.L + sy]


def test_reach_neighbour_count():
    seen = set()
    for c in CASES:
        if c.family != "feat_count":
            continue
        for want, info, k in _target_info(c):
            assert info["cnt"][k] == want, (c.name, want, int(info["cnt"][k]))
            seen.add((c.name.split("_")[-1], want))
    assert seen == {(p, n) for p in ("interior", "edge", "corner", "wrap") for n in (7, 8)}
    for n in (7, 8):        # the counted neighbours of a target lie across the storage wrap line
        assert sum(bool(info["wrap"][k]) for _, info, k in _target_info(mc.case(f"feat_count{n}_wrap"))) >= 2


def test_reach_pivot():
    tags = {}
    for c in CASES:
        if not hasattr(c, "targets") or c.family != "feat_pivot":
            continue
        for tag, info, k in _target_info(c):
            hit = {"tie01_02": info["tie01_02"][k], "tie02_12": info["tie02_12"][k], "neg01": info["neg01"][k],
                   "eqdiag": info["eqdiag"][k], "eqeig02": info["eig_tie"][k], "eqeig12": info["eig_tie"][k]}
            if tag in hit:
                assert hit[tag], (c.name, tag)
            else:                                       # first pivot one ulp around 0.01
                fp = info["first_pivot"][k]
                want = {"pivot_below": mc.PRED(0.01), "pivot_on": f32(0.01), "pivot_above": mc.SUCC(0.01)}[tag]
                assert fp == want, (c.name, tag, fp)
                assert (info["rotations"][k] > 0) == (tag != "pivot_below")
            tags[tag] = tags.get(tag, 0) + 1
    assert set(tags) == {"tie01_02", "tie02_12", "neg01", "eqdiag", "eqeig02", "eqeig12", "pivot_below", "pivot_on",
                         "pivot_above"}, tags
    # the rotation cap: finite matrices converge in a few rotations; overflowing squares run into the cap
    _, _, _, info = _features(mc.case("feat_pivot_cap31"))
    assert (info["rotations"] == 31).sum() > 100


def test_reach_geometry_and_empty_tiles():
    # the storage wrap line inside a window: valid neighbours across it, for every scrolled start of every L >= 5
    for c in CASES:
        if c.family == "feat_geom" and c.L >= 5 and c.start != (0, 0):
            _, _, _, info = _features(c)
            assert (info["wrap"] & (info["cnt"] > 7)).any(), c.name
    # an empty tile with valid cells in its halo; a tile whose only valid cell is its corner
    kinds = set()
    for c in CASES:
        if c.family != "feat_empty":
            continue
        e = c.elevation != f32(-10)
        L = c.L
        nt = (L + 15) // 16
        empty_with_halo = corner_only = False
        for ti in range(nt):
            for tj in range(nt):
                rs, cs = slice(16 * ti, min(L, 16 * ti + 16)), slice(16 * tj, min(L, 16 * tj + 16))
                inner = e[rs, cs]
                hal = e[np.arange(16 * ti - 2, 16 * ti + 18)[:, None] % L, np.arange(16 * tj - 2, 16 * tj + 18)[None, :] % L]
                if not inner.any() and hal.any():
                    empty_with_halo = True
                if inner.sum() == 1 and (inner[0, 0] or inner[0, -1] or inner[-1, 0] or inner[-1, -1]):
                    corner_only = True
        assert empty_with_halo or corner_only, c.name
        kinds |= {"empty_with_halo"} if empty_with_halo else set()
        kinds |= {"corner_only"} if corner_only else set()
    assert kinds == {"empty_with_halo", "corner_only"}


def test_reach_rays():
    ties = eq = 0
    removal = {"eq": 0, "above": 0, "below": 0}
    for c in CASES:
        if not c.family.startswith("ray") or c.L > 64:
            continue
        r = mc.trace_rays(c.elevation, c.variance, c.ray_traver, c.lowest, c.L, c.start, c.sensor_z,
                          c.obstacle_threshold)
        if c.family == "ray_ties":
            assert r["tie_steps_nondiag"] > 0 and r["threshold_eq"] > 0, c.name
        ties += r["tie_steps_nondiag"]
        eq += r["threshold_eq"]
        v, rr = r["value"], r["restrict"]
        removal["eq"] += int((v == rr).sum())
        removal["above"] += int((v == mc.SUCC(rr)).sum())
        removal["below"] += int((v == mc.PRED(rr)).sum())
        # robot row and column: never cast
        robot = mc.robot_index(c.L)
        geo = ((r["cells"] // c.L - c.start[0]) % c.L, (r["cells"] % c.L - c.start[1]) % c.L)
        assert not ((geo[0] == robot) | (geo[1] == robot)).any()
    assert ties > 100 and eq > 10 and min(removal.values()) > 100, (ties, eq, removal)


def test_reach_lowest_above_10():
    """valid lowest values above the sentinel decide removals: treating them as invalid changes the map"""
    c = mc.case("ray_low_above_10")
    args = (c.elevation, c.variance, c.ray_traver)
    a = mc.trace_rays(*args, c.lowest, c.L, c.start, c.sensor_z, c.obstacle_threshold)
    low = np.where(c.lowest > 10, f32(10), c.lowest)
    b = mc.trace_rays(*args, low, c.L, c.start, c.sensor_z, c.obstacle_threshold)
    assert (a["removed"] != b["removed"]).sum() > 10


def test_reach_bitmap_tail():
    for c in CASES:
        if c.family == "ray_tail":
            n = c.L * c.L
            assert n % 32 and n % 256
            assert (c.lowest.reshape(-1)[32 * ((n - 1) // 32):] != 10).all()


def test_long_ray_case_reaches_the_ring():
    c = mc.long_ray_case()
    r = mc.trace_rays(c.elevation, c.variance, c.ray_traver, c.lowest, c.L, c.start, c.sensor_z, c.obstacle_threshold)
    assert r["cells"].size > 10000 and 0 < r["removed"].sum() < r["cells"].size
    assert (r["value"] == r["restrict"]).sum() > 1000


# ---------------------------------------------------------------------------------------------------------------------
# plausibility: on planes at coarse resolution the slope is the angle of the plane's normal
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("res", [0.5, 1.0])
def test_slope_agrees_with_float64_pca(res):
    L = 24
    rng = np.random.default_rng(int(res * 10))
    gx, gy = np.meshgrid(np.arange(L), np.arange(L), indexing="ij")
    checked = 0
    for _ in range(6):
        a, b = rng.uniform(-1.5, 1.5, 2)
        if np.hypot(a, b) < 0.25:
            continue
        z = (a * gx * res + b * gy * res + 0.3).astype(f32)
        slope, _, _, info = features_np(z, L, res, (0, 0))
        o = OracleMap(L, res)
        o.set_layer("elevation", z)
        _assert_same(slope, o.map_feature()["slope"], "plane")
        for x in range(2, L - 2):
            for y in range(2, L - 2):
                P = np.stack([(gx[x - 2:x + 3, y - 2:y + 3] * res).ravel(), (gy[x - 2:x + 3, y - 2:y + 3] * res).ravel(),
                              z[x - 2:x + 3, y - 2:y + 3].astype(np.float64).ravel()], 1)
                w, v = np.linalg.eigh(np.cov(P.T))
                ref = np.arccos(abs(v[2, 0]))
                if ref < 0.2:
                    continue
                assert abs(float(slope[x * L + y]) - ref) < 1e-3, (res, a, b, x, y, slope[x * L + y], ref)
                checked += 1
    assert checked > 500
