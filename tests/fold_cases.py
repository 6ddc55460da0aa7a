"""Crafted per-cell record lists for the fold of the add path (gem_b200/csrc/gem_add.cuh).  CPU only, no GPU imports.

How the fold treats a cell depends on two things:
  * the number of records the cell receives in one call picks the kernel, the ordering method and the record
    addressing (1-8: fold_small_cell; 9-40: k_fold; 41-64: rank counting in k_fold_long; 65-256: register bitonic;
    257-1024: shared-memory bitonic; longer: repeated selection), and
  * the step tier decides each record: the plain step, the general step (fold_step_fast) or the literal fold_step.
Random clouds reach few of these combinations, so this module builds record lists that reach all of them:

  value_families()  for many cells of one small map, lists of k records in which a crafted record sits at a chosen
                    position; each family aims at one tier or edge (gate bands, skip records, magnitude edges,
                    numerator cancellation, non-finite heights, start states, colours, a state that returns to -10
                    in the middle of a list);
  length_sweep()    plain records at list lengths on both sides of every boundary of the fold;
  sweep_points()    the same lengths as a point cloud for the add path (identity frame, points placed in cells).

Every set comes back as ONE gem_fuse-shaped call: the cells are interleaved and the global order is shuffled across
cells, while the order inside each cell is kept, so the device really has to sort and its arrival ranks are
scrambled.

Crafting against the real state.  A record that must sit at a given distance from the gate needs the cell state just
before it.  A shadow OracleMap runs in lockstep: at position t one fuse_points call feeds the t-th record of every
cell, the elevation and variance are read back and record t+1 is crafted from them.  Every fuse_points call also
floors the variance of every cell at 1e-4, which one long call would do only at its end; that changes no decision
and no result, because every step floors the variance before it uses it (gpu.cu:500-501) and the last call floors it
anyway.  (The tests check that the lockstep result equals the single shuffled call.)
"""
from __future__ import annotations

import functools
from dataclasses import dataclass, field

import numpy as np

from oracle_lib import OracleMap

f32 = np.float32
L = 64
RES = 0.1
LENGTHS = (5, 33, 41, 100, 200, 300, 700, 1100)
POSITIONS = (0, 1, 30, 31, 32, 33)                  # and k - 1
SWEEP = (1, 2, 7, 8, 9, 31, 32, 33, 39, 40, 41, 64, 65, 128, 129, 167, 168, 169, 256, 257, 512, 513, 679, 680, 681,
         1024, 1025, 2728, 2729, 10921)            # 10921 = level_base(6) + 1
LAYERS = ("elevation", "variance", "intensity", "color_r", "color_g", "color_b")

TWO20, TWOM40 = f32(2.0 ** 20), f32(2.0 ** -40)
PRED = lambda x: np.nextafter(f32(x), f32(0))
SUBNORMAL = f32(1e-41)


# ---------------------------------------------------------------------------------------------------------------------
# cell plans
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class CellPlan:
    family: str
    k: int                      # list length
    pos: int                    # position of the family's decisive ("key") record, -1: none
    init_e: float
    init_v: float
    base: float                 # filler centre while the state is not finite
    jumps: bool = True          # filler may replace (higher, gated) and ignore (lower, gated) records
    specs: dict = field(default_factory=dict)    # position -> (role, fn(e, ov) -> (h, v))
    colour: dict = field(default_factory=dict)   # position -> (R, G, B, I)
    invalid_colour: bool = False                 # every record of the list has one zero channel


def _sig(ov):
    return float(np.sqrt(np.float64(ov)))


def _at_ratio(ratio, sign, v=f32(0.01)):
    """h with (h - e)^2 = ratio * 25 * ov: ratio 1 is the 5-sigma gate"""
    return lambda e, ov: (f32(float(e) + sign * np.sqrt(25.0 * float(ov) * ratio)), v)


def _ulp_sweep(offset, sign):
    def fn(e, ov):
        h = f32(float(e) + sign * 5.0 * _sig(ov))
        for _ in range(abs(offset)):
            h = np.nextafter(h, f32(np.inf) if offset > 0 else f32(-np.inf))
        return f32(h), f32(0.01)
    return fn


def _fixed(h, v=None):
    return lambda e, ov: (f32(h), f32(0.01) if v is None else f32(v))


def _in_gate(z, v=f32(0.01)):
    return lambda e, ov: (f32(float(e) + z * _sig(ov)), v)


# the families that put one decisive record at a chosen position: name -> (tier of that record, maker)
# tier: what the kernel's predicates make of the key record (tests/test_fold_cases.py restates them): 'plain',
# 'general' (the plain step leaves, fold_step_fast decides), 'literal' (fold_step decides), 'skip', 'first' (the state
# is -10: the record is taken as it is), None (no single tier, see the test)
def _families():
    fam = {}

    def simple(name, tier, fn, base=None, jumps=True, v=None):
        def make(k, p, rng, cell):
            b = base if base is not None else float(rng.uniform(0.5, 2.0))
            v0 = float(rng.uniform(1e-3, 0.05)) if base is None else 1e-3  # near-gate families: keep the state near base
            return CellPlan(name, k, p, b, v0, b, jumps, {p: ("key", fn)})
        fam[name] = (tier, make)

    simple("plain", "plain", None)
    # the plain step decides the gate outside +-2e-5 (relative, on (h-e)^2 against 25 ov), the general step outside
    # +-1e-5, the literal expression inside.  States near 0 keep the spacing of h fine against these bands
    for s in (-1, 1):
        simple(f"band_general_{'hi' if s > 0 else 'lo'}", "general", _at_ratio(1 + s * 1.5e-5, 1 if s > 0 else -1),
               base=0.01, jumps=False)
        simple(f"band_literal_{'hi' if s > 0 else 'lo'}", "literal", _at_ratio(1 + s * 4e-6, -1 if s > 0 else 1),
               base=0.01, jumps=False)

    def sweep(k, p, rng, cell):
        off = (cell * 37 + p * 11) % 81 - 40
        return CellPlan("ulp_sweep", k, p, 0.01, 1e-3, 0.01, False,
                        {p: ("key", _ulp_sweep(off, 1 if cell & 1 else -1))})
    fam["ulp_sweep"] = (None, sweep)
    simple("skip", "skip", _fixed(-1.0))
    for nm, h, tier in (("h_2p20", TWO20, "general"), ("h_pred_2p20", PRED(TWO20), "plain"),
                        ("h_2pm40", TWOM40, "plain"), ("h_pred_2pm40", PRED(TWOM40), "general"),
                        ("h_zero", f32(0.0), "plain"), ("h_negzero", f32(-0.0), "plain"),
                        ("h_subnormal", SUBNORMAL, "general")):
        simple(nm, tier, _fixed(h))
    for nm, v, tier in (("v_2pm40", TWOM40, "plain"), ("v_pred_2pm40", PRED(TWOM40), "general"),
                        ("v_2p20", TWO20, "general"), ("v_pred_2p20", PRED(TWO20), "plain")):
        simple(nm, tier, _in_gate(0.5, v))

    # numerator cancellation: state (3*2^-20, 2^-13) -- set by a gated higher record, or as the start state -- and
    # h = -3*2^-37 + j*2^-59, v = 2^-30: ov*h + v*e = j*2^-72 exactly, nonzero and below 2^-66, in the gate
    def cancel(k, p, rng, cell):
        j = 1 + cell % 8
        key = ("key", _fixed(f32(-3 * 2.0 ** -37 + j * 2.0 ** -59), f32(2.0 ** -30)))
        if p == 0:
            return CellPlan("cancel", k, 0, 3 * 2.0 ** -20, 2.0 ** -13, -1.0, False, {0: key})
        return CellPlan("cancel", k, p, -1.0, 1e-3, -1.0, False,
                        {p - 1: ("setup", _fixed(f32(3 * 2.0 ** -20), f32(2.0 ** -13))), p: key})
    fam["cancel"] = ("literal", cancel)
    for nm, h in (("h_inf", np.inf), ("h_neginf", -np.inf), ("h_nan", np.nan)):
        simple(nm, "literal", _fixed(h))

    # colour: the last taking record of the chunk has a zero R, G, B or intensity; the one before takes a valid colour;
    # the rest of the chunk are lower points the gate ignores (valid colours that must not be taken)
    for ch in range(4):
        def colour(k, p, rng, cell, ch=ch):
            b = float(rng.uniform(0.5, 2.0))
            pl = CellPlan(f"colour_zero_{'RGBI'[ch]}", k, p, b, float(rng.uniform(1e-3, 0.05)), b, False,
                          {p: ("key", _in_gate(0.5))})
            c = [11, 22, 33, 44.0]
            c[ch] = 0
            pl.colour[p] = tuple(c)
            if p > 0:
                pl.specs[p - 1] = ("setup", _in_gate(-0.5))
                pl.colour[p - 1] = (101, 102, 103, 104.0)
            for t in range(p + 1, min(k, (p // 32 + 1) * 32)):
                pl.specs[t] = ("tail", _in_gate(-8.0))
                pl.colour[t] = (201, 202, 203, 204.0)
            return pl
        fam[f"colour_zero_{'RGBI'[ch]}"] = ("plain", colour)

    # return to the sentinel: the state becomes exactly -10 at position p-1, by replacement (a gated higher record
    # at -10) or by a Kalman result of -10 ((-10.25, 0.25) then (-9.75, 0.25)); the record at p is then "first"
    followers = {"lower": (-30.0, 0.01), "ingate": (-10.05, 0.01), "higher": (-8.0, 0.01)}
    for how in ("replace", "kalman"):
        for fol, (fh, fv) in followers.items():
            def sentinel(k, p, rng, cell, how=how, fh=fh, fv=fv, fol=fol):
                need = 1 if how == "replace" else 2
                a = min(max(p, need), k - 1)
                pl = CellPlan(f"sentinel_{how}_{fol}", k, a, -12.0, 1e-3, -12.0, False,
                              {a: ("key", _fixed(fh, fv))})
                if how == "replace":
                    pl.specs[a - 1] = ("setup", _fixed(-10.0, 0.01))
                else:
                    pl.specs[a - 2] = ("setup", _fixed(-10.25, 0.25))
                    pl.specs[a - 1] = ("setup", _fixed(-9.75, 0.25))
                return pl
            fam[f"sentinel_{how}_{fol}"] = ("first", sentinel)
    return fam


# start states and whole-list colour: one cell per list length, key = the first record
def _start_families():
    def start(name, e, v):
        return lambda k, rng: CellPlan(name, k, 0, e, v, 0.7, True, {0: ("key", None)})
    out = {
        "start_empty": ("first", start("start_empty", -10.0, 0.3)),
        "start_var_below_floor": ("plain", start("start_var_below_floor", 0.7, 1e-6)),
        "start_elev_2p20": ("general", start("start_elev_2p20", float(TWO20), 0.01)),
        "start_elev_subnormal": ("general", start("start_elev_subnormal", float(SUBNORMAL), 0.01)),
        "start_elev_negzero": ("plain", start("start_elev_negzero", -0.0, 0.01)),
    }

    def invalid(k, rng):
        pl = CellPlan("colour_all_invalid", k, -1, 0.9, 0.01, 0.9)
        pl.invalid_colour = True
        return pl
    out["colour_all_invalid"] = (None, invalid)
    return out


FAMILIES = _families()
START_FAMILIES = _start_families()


def family_tier(name):
    if name in FAMILIES:
        return FAMILIES[name][0]
    if name in START_FAMILIES:
        return START_FAMILIES[name][0]
    return "plain"


# ---------------------------------------------------------------------------------------------------------------------
# the lockstep crafting run
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class Crafted:
    L: int
    init: dict       # layer -> flat (L*L,) array: the state both maps start from (set_layer)
    key: np.ndarray  # the gem_fuse call, in its (shuffled) order
    R: np.ndarray
    G: np.ndarray
    B: np.ndarray
    I: np.ndarray
    h: np.ndarray
    v: np.ndarray
    pos: np.ndarray      # per record: its position in its cell's list
    role: np.ndarray     # per record: 'fill', 'key', 'setup', 'tail'
    pre_e: np.ndarray    # per record: the cell's elevation and (floored) variance just before the record
    pre_v: np.ndarray
    plans: dict          # cell key -> CellPlan
    shadow: dict         # layer -> flat array the lockstep run ended with

    @property
    def n(self):
        return int(self.key.shape[0])

    def lists(self):
        return {c: p.k for c, p in self.plans.items()}

    def fuse_args(self):
        return self.key, self.R, self.G, self.B, self.I, self.h, self.v

    def apply_init(self, m):
        for name, a in self.init.items():
            m.set_layer(name, a.reshape(self.L, self.L))


def _fill(rng, e, ov, base, jumps):
    n = e.shape[0]
    sig = np.sqrt(ov.astype(np.float64))
    centre = np.where(np.isfinite(e), e.astype(np.float64), base)
    u = rng.random(n)
    z = rng.uniform(-3.0, 3.0, n)
    up = jumps & (u < 0.03)
    dn = jumps & (u >= 0.03) & (u < 0.06)
    z = np.where(up, rng.uniform(7.0, 10.0, n), np.where(dn, -rng.uniform(7.0, 10.0, n), z))
    with np.errstate(all="ignore"):
        h = (centre + z * sig).astype(f32)
    v = rng.uniform(1e-3, 0.05, n).astype(f32)
    col = np.concatenate([rng.integers(1, 256, (n, 3)), rng.integers(1, 256, (n, 1))], 1).astype(np.float64)
    zero = rng.random(n) < 0.1
    col[zero, rng.integers(0, 4, n)[zero]] = 0
    return h, v, col


def _floor(var):
    return np.where(var <= f32(1e-4), f32(1e-4), var).astype(f32)


def _run(plans: dict, seed: int) -> Crafted:
    rng = np.random.default_rng(seed)
    nc = L * L
    cells = np.array(sorted(plans), np.int64)
    pl = [plans[int(c)] for c in cells]
    ks = np.array([p.k for p in pl], np.int64)
    off = np.concatenate([[0], np.cumsum(ks)])
    total = int(off[-1])
    base = np.array([p.base for p in pl])
    jumps = np.array([p.jumps for p in pl])
    invalid = np.array([p.invalid_colour for p in pl])
    o = OracleMap(L, RES, compat_box_filter=False)
    init = {name: o.get_layer(name).reshape(-1).copy() for name in LAYERS}
    init["elevation"][cells] = [p.init_e for p in pl]
    init["variance"][cells] = [p.init_v for p in pl]
    init["intensity"][cells] = f32(3.5)
    init["color_r"][cells] = 1 + cells % 200
    init["color_g"][cells] = 2 + cells % 150
    init["color_b"][cells] = 3 + cells % 100
    for name, a in init.items():
        o.set_layer(name, a)
    events = {}
    for j, p in enumerate(pl):
        for t in set(p.specs) | set(p.colour):
            events.setdefault(t, []).append(j)
    flat = {nm: np.zeros(total, dt) for nm, dt in (("h", f32), ("v", f32), ("pre_e", f32), ("pre_v", f32))}
    flat["col"] = np.zeros((total, 4), np.float64)
    role = np.full(total, "fill", dtype=object)
    e = init["elevation"].copy()
    var = _floor(init["variance"])
    for t in range(int(ks.max())):
        act = np.nonzero(ks > t)[0]
        c = cells[act]
        ec, ov = e[c], _floor(var[c])
        h, v, col = _fill(rng, ec, ov, base[act], jumps[act])
        where = {int(j): i for i, j in enumerate(act)}
        for j in events.get(t, ()):
            i = where[j]
            p = pl[j]
            if t in p.specs:
                r, fn = p.specs[t]
                role[off[j] + t] = r
                if fn is not None:
                    h[i], v[i] = fn(ec[i], ov[i])
            if t in p.colour:
                col[i] = p.colour[t]
        bad = invalid[act]
        col[bad, rng.integers(0, 4, act.shape[0])[bad]] = 0
        rows = off[act] + t
        flat["h"][rows], flat["v"][rows], flat["col"][rows] = h, v, col
        flat["pre_e"][rows], flat["pre_v"][rows] = ec, ov
        ci = col[:, :3].astype(np.int32)
        o.fuse_points(c.astype(np.int32), ci[:, 0], ci[:, 1], ci[:, 2], col[:, 3].astype(f32), h, v)
        e = o.get_layer("elevation").reshape(-1)
        var = o.get_layer("variance").reshape(-1)
    shadow = {name: o.get_layer(name).reshape(-1).copy() for name in LAYERS}
    o.close()
    # one call: cells interleaved, shuffled across cells, in order inside each cell
    labels = rng.permutation(np.repeat(np.arange(cells.shape[0]), ks))
    order = np.argsort(labels, kind="stable")       # global positions of the records of cell 0, then cell 1, ...

    def scatter(a):
        out = np.empty_like(a)
        out[order] = a
        return out
    key = scatter(np.repeat(cells, ks).astype(np.int32))
    pos = scatter(np.concatenate([np.arange(k) for k in ks]).astype(np.int32))
    col = scatter(flat["col"])
    ci = col[:, :3].astype(np.int32)
    return Crafted(L, init, key, ci[:, 0].copy(), ci[:, 1].copy(), ci[:, 2].copy(), col[:, 3].astype(f32),
                   scatter(flat["h"]), scatter(flat["v"]), pos, scatter(role), scatter(flat["pre_e"]),
                   scatter(flat["pre_v"]), {int(c): p for c, p in zip(cells, pl)}, shadow)


def _cell_slots(n, rng):
    """n distinct cells of the map, spread over all rows"""
    return rng.permutation(L * L)[:n]


@functools.lru_cache(maxsize=None)
def value_families(seed: int = 1) -> Crafted:
    rng = np.random.default_rng(seed)
    specs = []
    for name, (_, make) in FAMILIES.items():
        for k in LENGTHS:
            for p in sorted({q for q in POSITIONS if q < k} | {k - 1}):
                specs.append((make, k, p))
    for name, (_, make) in START_FAMILIES.items():
        for k in LENGTHS:
            specs.append((make, k, None))
    slots = _cell_slots(len(specs), rng)
    plans = {}
    for (make, k, p), c in zip(specs, slots):
        plans[int(c)] = make(k, rng) if p is None else make(k, p, rng, int(c))
    return _run(plans, seed)


def sweep_cells(copies: int = 2):
    """cell keys of the length sweep: `copies` cells per length, rows spread from the first to the last row"""
    n = copies * len(SWEEP)
    rows = np.round(np.linspace(0, L - 1, n)).astype(np.int64)
    cols = (np.arange(n) * 17 + 5) % L
    return [(int(r * L + c), SWEEP[i % len(SWEEP)]) for i, (r, c) in enumerate(zip(rows, cols))]


@functools.lru_cache(maxsize=None)
def length_sweep(seed: int = 2) -> Crafted:
    rng = np.random.default_rng(seed)
    plans = {}
    for c, k in sweep_cells():
        b = float(rng.uniform(0.5, 2.0))
        plans[c] = CellPlan("plain", k, -1, b, float(rng.uniform(1e-3, 0.05)), b)
    return _run(plans, seed)


# ---------------------------------------------------------------------------------------------------------------------
# the add path: the same lengths as points
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class PointSet:
    xyzi: np.ndarray     # (n, 4) float32
    rgba: np.ndarray     # (n, 4) uint8
    lists: dict          # cell key -> number of points the oracle bins into it
    binned: int          # points inside the grid and the height window


def cell_centre(c):
    gx, gy = divmod(int(c), L)
    return (L / 2 - gx - 0.5) * RES, (L / 2 - gy - 0.5) * RES


def place_points(lists: dict, rng, z_base=None):
    """points whose cells (identity pose, map centred at the origin, no scroll) are `lists`' keys, as many as the
    values, shuffled across cells"""
    xs, ys, zs = [], [], []
    for c, k in lists.items():
        x0, y0 = cell_centre(c)
        xs.append(x0 + rng.uniform(-0.3, 0.3, k) * RES)
        ys.append(y0 + rng.uniform(-0.3, 0.3, k) * RES)
        zb = rng.uniform(0.5, 2.0) if z_base is None else z_base
        z = zb + rng.normal(0.0, 0.01, k)
        jump = rng.random(k) < 0.05
        z[jump] += rng.choice([-0.5, 0.5], int(jump.sum()))
        zs.append(z)
    xyz = np.stack([np.concatenate(xs), np.concatenate(ys), np.concatenate(zs)], 1).astype(f32)
    n = xyz.shape[0]
    perm = rng.permutation(n)
    xyzi = np.concatenate([xyz[perm], rng.integers(0, 256, (n, 1)).astype(f32)], 1).astype(f32)
    rgba = rng.integers(0, 256, (n, 4)).astype(np.uint8)
    return xyzi, rgba


def count_cells(xyzi, frame):
    """the oracle's process_points: per-cell counts of the binned points (fresh map, identity pose)"""
    o = OracleMap(L, RES, compat_box_filter=False)
    key = o.process_points(xyzi[:, 0], xyzi[:, 1], xyzi[:, 2], frame)[0]
    o.close()
    ok = key >= 0
    cnt = np.bincount(key[ok], minlength=L * L)
    return {int(c): int(cnt[c]) for c in np.nonzero(cnt)[0]}, int(ok.sum())


def sweep_points(frame, seed: int = 3) -> PointSet:
    """the length sweep as a cloud for the add path.  The sensor variance of a point cannot be steered, so the add
    path gets the lengths only, not the value families.  `frame`: identity pose, laser model, height window wide
    enough for every point (built by the caller; this module stays free of the GPU package)"""
    rng = np.random.default_rng(seed)
    want = dict(sweep_cells())
    xyzi, rgba = place_points(want, rng)
    got, binned = count_cells(xyzi, frame)
    assert got == want, "the points of a cell must bin into that cell"
    return PointSet(xyzi, rgba, got, binned)
