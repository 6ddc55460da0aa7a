"""Pins the CPU oracle against the REFERENCE ITSELF on the crafted inputs: the fold record lists (tests/fold_cases.py),
the feature and ray maps (tests/map_cases.py), the point front end at odd and even L and the scroll calls
(tests/pin_cases.py).  The crafted suites compare the device with the oracle on the exact float edges where a kernel
decides something; this module checks that the oracle decides them as the reference's own kernels do
(gpu_process.cu compiled unmodified with -fmad=false by oracle/build_ref.py and run on an H100).

Like tests/test_reference_pin.py, the reference's outputs are stored in tests/golden/reference_pin_cases_v1.npz
(recorded by `tests/golden/make_reference_pin.py test_reference_pin_cases tests/golden/reference_pin_cases_v1.npz`,
which runs these same functions against the live reference; in ref_lib.pack's form, a few arrays rather than two per
call) and replayed through ref_lib.PinnedRef, so no GPU and no reference are needed here.  Every comparison is bit for bit, except the feature kernel's rough / slope / traver
values, whose trig goes through CUDA's libm in the reference and through the oracle's deterministic trig.

Parts of the reference that are not defined are left out of the comparisons, each where it occurs: the racy `lowest`
update (gpu_process.cu:434-438) is compared only in cells that received one point, Map_feature's rough / slope /
traver outputs are uninitialised in empty cells (:581-582), the sensor height is uninitialised until the first Move
(:33, :1011-1012), and NaNs are compared as a class (their sign and payload come from the hardware)."""
import os

import numpy as np
import pytest

import fold_cases as fc
import map_cases as mc
import pin_cases as pc
import ref_lib
from oracle_lib import OracleMap
from pin_cases import assert_bits, front_end_frame

PIN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pin_cases_v1.npz")
f32 = np.float32
FOLD_LAYERS = fc.LAYERS
PACKED = True               # the recording is stored in ref_lib.pack's form
TRIG = ("rough", "slope", "traver")
FULL_TRIG_L = 64            # maps up to this size pin the trig-valued outputs of every valid cell


@pytest.fixture(scope="module")
def reference():
    """reference(tag, L, res, nofma) -> the reference's map for one scenario, replayed from the stored outputs"""
    g = ref_lib.Packed(np.load(PIN, allow_pickle=False))
    assert "reference gpu_process.cu" in str(g["generated_by"])
    return lambda tag, L, res, nofma: ref_lib.PinnedRef(g, tag)


def pick(d, names):
    return {n: d[n] for n in names}


def layers(m, names):
    return {n: m.get_layer(n) for n in names}


def oracle_state(o):
    c, s, z = o.state()
    return c, s, np.array([z], f32)


# ---------------------------------------------------------------------------------------------------------------------
# A. fold lists
# ---------------------------------------------------------------------------------------------------------------------
def _fold(reference, tag, s):
    r = reference(tag, s.L, fc.RES, True)
    o = OracleMap(s.L, fc.RES, compat_box_filter=False)
    for m in (r, o):
        s.apply_init(m)
        m.fuse_points(*s.fuse_args())
    fo = o.map_feature()
    fr = r.map_feature(like=pick(fo, FOLD_LAYERS))
    for name in FOLD_LAYERS:
        assert_bits(fr[name], fo[name], f"{tag} {name}")
    return fo


def _gate_ratio(s):
    """|h - e| / sqrt(max(v, 1e-4)) in float32 per record, as G_fuse computes it (gpu_process.cu:500-502)"""
    with np.errstate(all="ignore"):
        return (np.abs(s.h - s.pre_e) / np.sqrt(s.pre_v).astype(f32)).astype(f32)


def test_fold_value_families_vs_reference(reference):
    s = fc.value_families()
    _fold(reference, "fold_values", s)
    # the decisions the families exist for
    finite = np.isfinite(s.pre_e) & (s.pre_e != f32(-10))
    mah = _gate_ratio(s)
    assert ((np.abs(mah - f32(5)) < f32(1e-5)) & finite).sum() > 20, "records within a few ulps of the gate"
    colour_no_intensity = (s.R != 0) & (s.G != 0) & (s.B != 0) & (s.I == 0)
    assert colour_no_intensity.sum() > 0, "records with a colour and no intensity"
    assert (~np.isfinite(s.h)).sum() > 0 and (np.abs(s.pre_e) < f32(1.2e-38)).any()


def test_fold_gate_at_equality_vs_reference(reference):
    s = pc.gate_records()
    _fold(reference, "fold_gate", s)
    mah = s.ratio()
    for ulps in (-1, 0, 1):
        at = mah.view(np.int32) - f32(5).view(np.int32) == ulps
        assert (at & (s.h > s.pre_e)).sum() >= 2 and (at & (s.h < s.pre_e)).sum() >= 2, ulps


def test_fold_length_sweep_vs_reference(reference):
    s = fc.length_sweep()
    _fold(reference, "fold_lengths", s)
    assert set(s.lists().values()) == set(fc.SWEEP)


def test_fold_floor_after_negative_var_update_vs_reference(reference):
    """Mapvar_update(-dv) leaves variances below the floor and negative; an empty Fuse floors every cell, the empty
    ones (-10) included (gpu_process.cu:533-534)"""
    s = fc.value_families()
    r = reference("fold_floor", s.L, fc.RES, True)
    o = OracleMap(s.L, fc.RES, compat_box_filter=False)
    e = np.zeros(0, np.int32), np.zeros(0, f32)
    for m in (r, o):
        s.apply_init(m)
        m.var_update(-0.02)
    vo = o.get_layer("variance")
    assert_bits(r.get_layer("variance", like=vo), vo, "variance after var_update(-0.02)")
    assert (vo == f32(-10)).sum() > 0 and ((vo < 0) & (vo != f32(-10))).sum() > 0
    for m in (r, o):
        m.fuse_points(e[0], e[0], e[0], e[0], e[1], e[1], e[1])
    fo = o.map_feature()
    fr = r.map_feature(like=pick(fo, ("elevation", "variance")))
    for name in ("elevation", "variance"):
        assert_bits(fr[name], fo[name], f"after the empty Fuse: {name}")
    assert (fo["variance"] == f32(1e-4)).sum() >= (vo.reshape(-1) < f32(1e-4)).sum()


# ---------------------------------------------------------------------------------------------------------------------
# B. crafted maps
# ---------------------------------------------------------------------------------------------------------------------
def _apply_case(r, o, c):
    pos = c.position()
    co = o.move(pos)
    cr = r.move(pos, like=co)
    for a, b in zip(cr, co):
        assert_bits(a, b, f"{c.name} move")
    for name in ("elevation", "variance", "traver", "lowest"):
        for m in (r, o):
            m.set_layer(name, getattr(c, name))


def _close(a, b, tol=1e-4):
    """per element: equal as a class for NaN, else |a - b| < tol"""
    a, b = a.astype(np.float64), b.astype(np.float64)
    na, nb = np.isnan(a), np.isnan(b)
    with np.errstate(all="ignore"):
        return np.where(na | nb, na & nb, (a == b) | (np.abs(a - b) < tol)), np.where(na | nb, np.where(na & nb, 0, np.inf),
                                                                                      np.abs(a - b))


def _edge_band(c):
    """storage cells whose 5 x 5 window reaches the storage wrap line or the geographic edge of the map"""
    r = np.arange(c.L)

    def near(start):
        g = (r - start) % c.L                    # the geographic index of storage index r
        return (np.minimum(r, c.L - 1 - r) < 2) | (np.minimum(g, c.L - 1 - g) < 2)
    return (near(c.start[0])[:, None] | near(c.start[1])[None, :]).reshape(-1)


def test_map_feature_cases_vs_reference(reference):
    worst = {}
    for c in mc.all_cases():
        if not c.family.startswith("feat"):
            continue
        # G_Mapfeature stays inside its buffers for every L >= 1: the window is range-checked in geographic
        # coordinates before it is wrapped (gpu_process.cu:589-602), at most 25 points, and the Jacobi loop is
        # bounded by nJt for non-finite entries
        r = reference(c.name, c.L, c.res, True)
        o = OracleMap(c.L, c.res, obstacle_threshold=c.obstacle_threshold, compat_box_filter=False)
        _apply_case(r, o, c)
        fo = o.map_feature()
        exact = ("elevation", "variance", "color_r", "color_g", "color_b", "intensity")
        fr = r.map_feature(like=pick(fo, exact))
        for name in exact:
            assert_bits(fr[name], fo[name], f"{c.name} {name}")
        valid = fo["elevation"] != f32(-10)
        # rough / slope / traver of valid cells only: the reference leaves them uninitialised in empty cells.  Their
        # values differ from the oracle's in the last bits nearly everywhere (libm trig), so maps larger than
        # FULL_TRIG_L keep the values of the cells whose window reaches the wrap line or the geographic edge, what
        # those maps are there for; the -10 pattern (the window count's decision) is kept for every valid cell
        sel = valid & (_edge_band(c) if c.L > FULL_TRIG_L else True)

        def trig(f):
            return {"invalid": (f["traver"][valid] == f32(-10)).astype(np.uint8), **{n: f[n][sel] for n in TRIG}}
        fv = r.map_feature(like=trig(fo), derive=trig)
        ft = trig(fo)
        # the window count decides: traver -10 and rough = slope = 0 for 7 or fewer valid cells (:619, :662-667)
        assert_bits(fv["invalid"], ft["invalid"], f"{c.name} traver -10 pattern")
        both = ft["traver"] != f32(-10)
        tl = c.obstacle_threshold
        for name in TRIG:
            ok, d = _close(fv[name][both], ft[name][both])
            assert ok.mean() > 0.995 if ok.size else True, (c.name, name, float(ok.mean()))
            fam = worst.setdefault(c.family, {})
            fam[name] = max(fam.get(name, 0.0), float(d.max()) if d.size else 0.0)
        # the traver layer: Map_feature writes it in valid cells only, empty cells keep their stale values
        stale = lambda t: t.reshape(-1)[~valid]
        to = stale(o.get_layer("traver"))
        assert_bits(r.get_layer("traver", like=to, derive=stale), to, f"{c.name} stale traver")
        assert tl == 0.7
    print("worst |reference - oracle| in rough / slope / traver per family:", worst)
    assert set(worst) == {"feat_geom", "feat_mag", "feat_count", "feat_pivot", "feat_empty"}


def test_ray_cases_vs_reference(reference):
    removed = {}
    for c in mc.all_cases():
        if not c.family.startswith("ray"):
            continue
        # G_Raytracing stays inside its buffers: every probe is range-checked against [0, L) on both axes before it
        # reads `lowest` (gpu_process.cu:765, 781, 821), for L = 1 the only cell is the robot's and casts no ray
        assert c.obstacle_threshold == 0.7 and c.ray_traver is not None
        r = reference(c.name, c.L, c.res, True)
        o = OracleMap(c.L, c.res, obstacle_threshold=c.obstacle_threshold, compat_box_filter=False)
        _apply_case(r, o, c)
        for m in (r, o):
            c.apply_ray(m)
        lo = layers(o, ("traver", "lowest"))
        for name, a in r.layers(("traver", "lowest"), like=lo).items():
            assert_bits(a, lo[name], f"{c.name} {name} before the ray step")
        e0 = o.get_layer("elevation")
        for m in (r, o):
            m.raytracing()
        lo = layers(o, ("elevation", "lowest"))
        lr = r.layers(("elevation", "lowest"), like=lo)
        for name in lo:
            assert_bits(lr[name], lo[name], f"{c.name} {name} after Raytracing")
        eo, er = lo["elevation"], lr["elevation"]
        gone = lambda e: int(((e == f32(-10)) & (e0 != f32(-10))).sum())
        n = removed.setdefault(c.family, [0, 0])
        n[0] += gone(er)
        n[1] += gone(eo)
    for fam in ("ray_geom", "ray_ties", "ray_low", "ray_removal", "ray_tail"):
        assert removed[fam][0] > 0 and removed[fam][0] == removed[fam][1], (fam, removed[fam])


# ---------------------------------------------------------------------------------------------------------------------
# C. the point front end at odd and even L
# ---------------------------------------------------------------------------------------------------------------------
def test_front_end_odd_and_even_L_vs_reference(reference):
    f = front_end_frame()
    odd_keys_differ = 0
    for c in pc.front_end_cases():
        r = reference(f"front_{c.name}", c.L, c.res, True)
        o = OracleMap(c.L, c.res, compat_box_filter=True)
        co = o.move(c.position)
        for a, b in zip(r.move(c.position, like=co), co):
            assert_bits(a, b, f"{c.name} move")
        ko = o.process_points(c.x, c.y, c.z, f)
        kr = r.process_points(c.x, c.y, c.z, f, like=ko)
        for a, b, name in zip(kr, ko, ("map_index", "var", "x_ts", "y_ts", "z_ts")):
            assert_bits(a, b, f"{c.name} {name}")
        key, xt, yt = ko[0], ko[2], ko[3]
        acc = ko[1] != f32(-1)
        # every boundary point passes the filter and lands on both sides of a cell boundary
        assert acc[c.boundary].all(), c.name
        assert (key[c.boundary] >= 0).sum() > 0 and (key[c.boundary] < 0).sum() > 0
        # the filter-limit points: both decisions, matching the literal filter, one ulp apart
        rej = pc.box_filter_rejects(c.x, c.y)
        assert np.array_equal(~acc[~c.boundary], rej[~c.boundary]), c.name
        assert rej[~c.boundary].any() and (~rej[~c.boundary]).any()
        # lowest: race-free where a cell got exactly one point
        geo = np.array([o.points_to_index(a, b)[0] for a, b in zip(xt[acc], yt[acc])])
        geo = geo[geo >= 0]
        u, cnt = np.unique(geo, return_counts=True)
        single = u[cnt == 1]
        lo = o.get_layer("lowest")
        lr = r.get_layer("lowest", like=lo).reshape(-1)
        assert_bits(lr[single], lo.reshape(-1)[single], f"{c.name} lowest")
        assert single.size > 0 or c.L <= 3, c.name    # a map of 1 or 9 cells gets several points per cell
        if c.L % 2:
            cen, _, _ = o.state()
            trunc = np.array([[pc.axis_index(c.L, c.res, cen[0], a, truncate=True),
                               pc.axis_index(c.L, c.res, cen[1], b, truncate=True)] for a, b in zip(xt[acc], yt[acc])])
            rnd = np.array([[pc.axis_index(c.L, c.res, cen[0], a), pc.axis_index(c.L, c.res, cen[1], b)]
                            for a, b in zip(xt[acc], yt[acc])])
            n = int((trunc != rnd).any(axis=1).sum())
            assert n > 0, c.name
            odd_keys_differ += n
    assert odd_keys_differ > 0


# ---------------------------------------------------------------------------------------------------------------------
# D. scrolls and the map-wide calls
# ---------------------------------------------------------------------------------------------------------------------
def test_scroll_script_vs_reference(reference):
    s = pc.scroll_script()
    for name in ("wrap_rows", "wrap_cols", "shift_+(L-1)_rows", "shift_+(L-1)_cols", "shift_-(L-1)_rows",
                 "shift_-(L-1)_cols", "shift_L_rows", "shift_L_cols", "shift_L+5_rows", "shift_L+5_cols", "clear_all",
                 "boundary_position", "opt_differs_from_closeloop", "closeloop_differs_from_opt"):
        assert s.marks.get(name), name
    r = reference("scroll", s.L, s.res, True)
    o = OracleMap(s.L, s.res, compat_box_filter=False)
    traver_reset, moved = 0, False
    for k, (op, args) in enumerate(s.steps):
        t0 = o.get_layer("traver")
        res_o = pc.apply_step(o, op, args)
        res_r = pc.apply_step(r, op, args, reference=True, like=res_o)
        if res_o is not None:
            for a, b in zip(res_r if isinstance(res_r, tuple) else (res_r,),
                            res_o if isinstance(res_o, tuple) else (res_o,)):
                assert_bits(a, b, f"step {k} {op} result")
        so = oracle_state(o)
        moved = moved or op == "move"
        # sensorZatLowestScan is set by Move only (gpu_process.cu:1011-1012): Init leaves it as the last map of the
        # process had it, so it is compared from the first move on
        for a, b, name in list(zip(r.state(like=so), so, ("centre", "start", "sensorZ")))[:3 if moved else 2]:
            assert_bits(a, b, f"step {k} {op} {name}")
        lo = layers(o, pc.SCROLL_LAYERS)
        for name, a in r.layers(pc.SCROLL_LAYERS, like=lo).items():
            assert_bits(a, lo[name], f"step {k} {op} {name}")
        if op == "move" and k in s.marks["clear_all"]:
            t1 = o.get_layer("traver")
            traver_reset += int((t0 != f32(-10)).any() and (t1 == f32(-10)).all())
    assert traver_reset > 0, "a clear-all that resets a traver layer holding values"
