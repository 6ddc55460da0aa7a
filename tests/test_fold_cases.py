"""CPU checks of the crafted fold cases (tests/fold_cases.py): every crafted record reaches the step tier its family
names, and the oracle's definition of the new cases is pinned three ways (O(N) fuse, the O(C*N) literal G_fuse twin,
the independent numpy restatement).  The GPU side is tests/test_fold_paths_gpu.py."""
import numpy as np
import pytest

import fold_cases as fc
import np_reference
from oracle_lib import OracleMap

f32 = np.float32


# ---- the kernel's predicates (gem_add.cuh), restated in numpy float32 ------------------------------------------------
def mag_ok(x):
    """|x| in [2^-40, 2^20), on the bit pattern (NaN fails)"""
    u = np.asarray(x, f32).view(np.uint32) & np.uint32(0x7fffffff)
    return (u >= np.uint32(0x2b800000)) & (u < np.uint32(0x49800000))


def num_ok(x):
    """{0} U [2^-66, 2^66)"""
    u = np.asarray(x, f32).view(np.uint32) & np.uint32(0x7fffffff)
    return ((u >= np.uint32(0x1e800000)) & (u < np.uint32(0x60800000))) | (u == 0)


def den_ok(x):
    """[2^-50, 2^50)"""
    u = np.asarray(x, f32).view(np.uint32) & np.uint32(0x7fffffff)
    return (u >= np.uint32(0x26800000)) & (u < np.uint32(0x58800000))


def tiers(e, var, h, v):
    """per record: which step decides it -- 'skip', 'first' (state -10), 'plain' (plain_step / fold_chunk's plain
    loop), 'general' (the plain step leaves, fold_step_fast decides), 'literal' (fold_step_fast reports, fold_step
    decides) -- and the literal gate decision RN(|h-e| / RN(sqrt(ov))) > 5"""
    e, var, h, v = (np.asarray(a, f32) for a in (e, var, h, v))
    with np.errstate(all="ignore"):
        ov = np.where(var <= f32(1e-4), f32(1e-4), var).astype(f32)
        d = np.abs(h - e).astype(f32)
        dd = (d * d).astype(f32)
        n0 = ((ov * h).astype(f32) + (v * e).astype(f32)).astype(f32)
        n1 = (v * ov).astype(f32)
        den = (ov + v).astype(f32)
        lo_p = dd < (ov * f32(24.9995)).astype(f32)
        hi_p = dd > (ov * f32(25.0005)).astype(f32)
        plain_in = (h != f32(-1)) & ((h == 0) | mag_ok(h)) & (v >= f32(2.0 ** -40)) & (v < f32(2.0 ** 20))
        plain_st = (e != f32(-10)) & ((e == 0) | mag_ok(e)) & (ov < f32(2.0 ** 20))
        plain = plain_in & plain_st & (lo_p | hi_p) & (~lo_p | num_ok(n0))
        tv = (f32(25) * ov).astype(f32)
        hi = dd > (tv * f32(1.00001)).astype(f32)
        lo = dd < (tv * f32(0.99999)).astype(f32)
        rare_gate = ~((dd < f32(1e30)) & (tv < f32(1e30))) | ~(hi | lo)
        rare_div = ~(den_ok(den) & num_ok(n0) & num_ok(n1))
        literal = rare_gate | (~hi & rare_div)
        gate = (d / np.sqrt(ov).astype(f32)).astype(f32) > f32(5)
    out = np.where(plain, "plain", np.where(literal, "literal", "general")).astype(object)
    out[e == f32(-10)] = "first"
    out[h == f32(-1)] = "skip"
    return out, gate


def _family(s, name):
    cells = [c for c, p in s.plans.items() if p.family == name]
    return np.isin(s.key, cells)


# ---- generator self-check ------------------------------------------------------------------------------------------------
def test_crafted_records_reach_the_tier_their_family_names():
    s = fc.value_families()
    tier, gate = tiers(s.pre_e, s.pre_v, s.h, s.v)
    key = s.role == "key"
    names = sorted({p.family for p in s.plans.values()})
    assert len(names) == len(fc.FAMILIES) + len(fc.START_FAMILIES)
    for name in names:
        want = fc.family_tier(name)
        m = _family(s, name)
        if want is not None:
            got = tier[m & key]
            assert got.size > 0, name
            bad = got != want
            assert not bad.any(), f"{name}: key records in tiers {sorted(set(got[bad]))}, want {want}"
    # the control family is plain from the first record to the last
    ctl = _family(s, "plain")
    assert (tier[ctl] == "plain").all(), sorted(set(tier[ctl]))
    # the ulp sweep crosses the literal gate decision and stays near it (the plain step never decides it)
    sw = _family(s, "ulp_sweep") & key
    assert gate[sw].any() and (~gate[sw]).any()
    assert (tier[sw] != "plain").all() and (tier[sw] == "literal").sum() > sw.sum() // 2
    # the colour families: the key record and the one before it take, the tail is ignored
    for ch in "RGBI":
        m = _family(s, f"colour_zero_{ch}")
        lower = s.h < s.pre_e
        assert not (gate[m & (s.role == "key")]).any() and not (gate[m & (s.role == "setup")]).any()
        assert (gate[m & (s.role == "tail")] & lower[m & (s.role == "tail")]).all()
    # every list length and every key position is there
    for name in fc.FAMILIES:
        got = {(p.k, p.pos) for p in s.plans.values() if p.family == name}
        assert {k for k, _ in got} == set(fc.LENGTHS), name
        # a return to -10 needs one (replacement) or two (Kalman) records before the key record
        need = 2 if name.startswith("sentinel_kalman") else (1 if name.startswith("sentinel") else 0)
        for k in fc.LENGTHS:
            want = {min(max(q, need), k - 1) for q in fc.POSITIONS + (k - 1,) if q < k}
            assert {pos for kk, pos in got if kk == k} == want, (name, k)


def test_length_sweep_is_plain_and_has_every_length():
    s = fc.length_sweep()
    tier, _ = tiers(s.pre_e, s.pre_v, s.h, s.v)
    assert (tier == "plain").all(), sorted(set(tier))
    assert sorted(set(s.lists().values())) == sorted(fc.SWEEP)
    assert max(s.lists().values()) == 10921


def test_sweep_points_bin_into_their_cells():
    import gem_b200
    sp = gem_b200.LaserSensorProcessor(ignore_points_above=100.0, ignore_points_below=-100.0)
    frame = gem_b200.make_frame(np.eye(4), sp)
    ps = fc.sweep_points(frame)
    assert ps.lists == dict(fc.sweep_cells())
    assert ps.binned == ps.xyzi.shape[0] == sum(fc.SWEEP) * 2


# ---- the oracle's definition on the crafted cases, three ways ------------------------------------------------------------
def _same(a, b):
    a, b = np.asarray(a).reshape(-1), np.asarray(b).reshape(-1)
    if a.dtype.kind == "f":
        return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))
    return a == b


@pytest.mark.parametrize("which", ["value_families", "length_sweep"])
def test_oracle_literal_and_numpy_agree_bit_for_bit(which):
    s = getattr(fc, which)()
    maps = []
    for literal in (False, True):
        o = OracleMap(s.L, fc.RES, compat_box_filter=False)
        s.apply_init(o)
        o.fuse_points(*s.fuse_args(), literal=literal)
        maps.append({name: o.get_layer(name).reshape(-1) for name in fc.LAYERS})
        o.close()
    ini = s.init
    ref = np_reference.fuse(ini["elevation"], ini["variance"], ini["intensity"], ini["color_r"], ini["color_g"],
                            ini["color_b"], *s.fuse_args())
    ref = dict(zip(fc.LAYERS, ref))
    for name in fc.LAYERS:
        for what, other in (("literal", maps[1][name]), ("numpy", ref[name]), ("lockstep", s.shadow[name])):
            ok = _same(maps[0][name], other)
            assert ok.all(), (f"{which} {name}: oracle vs {what} differ in {int((~ok).sum())} cells, first "
                              f"{int(np.argmin(ok))}: {maps[0][name][np.argmin(ok)]!r} vs {other[np.argmin(ok)]!r}")
    # the crafted cells really changed (the call is not a no-op on them)
    cells = np.array(sorted(s.plans))
    assert (maps[0]["elevation"][cells] != ini["elevation"][cells]).mean() > 0.9


def test_sentinel_cases_take_the_record_after_a_return_to_minus_10():
    """the two minimal cases: one call into one cell whose state starts plain; the state becomes exactly -10
    (replacement, Kalman) and the next record is taken as it is"""
    for (e0, v0), recs, want in (((-12.0, 1e-4), [(-10.0, 0.01), (-10.05, 0.01)], (-10.05, 0.01)),
                                 ((-10.25, 0.25), [(-9.75, 0.25), (-30.0, 0.01)], (-30.0, 0.01))):
        o = OracleMap(4, 0.1, compat_box_filter=False)
        el = o.get_layer("elevation"); va = o.get_layer("variance")
        el.flat[5], va.flat[5] = e0, v0
        o.set_layer("elevation", el); o.set_layer("variance", va)
        h = np.array([r[0] for r in recs], f32)
        v = np.array([r[1] for r in recs], f32)
        one = np.ones(2, np.int32)
        o.fuse_points(np.full(2, 5, np.int32), one, one, one, one.astype(f32), h, v)
        assert (o.get_layer("elevation").flat[5], o.get_layer("variance").flat[5]) == (f32(want[0]), f32(want[1]))
        o.close()
