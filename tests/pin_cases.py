"""Inputs that pin the point front end and the scroll calls at their edges, for tests/test_reference_pin_cases.py (the
oracle against the reference's own kernels) and tests/test_reference_pin_cases_gpu.py (the device against the oracle).
CPU only, no GPU imports.

  front_end_cases()  Process_points at odd and even L with scrolled starts: points one ulp either side of every cell
                     boundary PointsToIndex / PointsToMapIndex decide (gpu_process.cu:309-358; odd L rounds with
                     +-0.5, even L truncates), on both axes and both signs, and on the hard-coded box-filter limits
                     (:393) and one ulp either side of them;
  scroll_script()    one call script: moves whose cleared bands wrap the storage edge on each axis, shifts of
                     +-(L-1), +L and +L+5 (the clear-all of Move, :1033-1038), positions one ulp either side of a
                     shift's rounding boundary, Mapvar_update of both signs, Map_optmove and Map_closeloop with targets
                     at their rounding boundaries and centres far from the origin, a small Fuse after each call.

Shifts <= -L are left out on purpose: Move then runs its partial clear with more cells than the map has and writes
out of bounds (SURVEY appendix A7); the oracle's clear-all there is a definition, not a restatement.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

import sequence_cases as sc

f32 = np.float32


def assert_bits(a, b, what):
    """a and b identical bit for bit, NaN as a class: the reference's NaNs are the GPU's canonical NaN, the oracle's
    those of the CPU it runs on (sign and payload are not defined by the operations that make them)"""
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, a.dtype, b.shape, b.dtype)
    if a.dtype == np.float32:
        bad = (a.view(np.uint32) != b.view(np.uint32)) & ~(np.isnan(a) & np.isnan(b))
    else:
        bad = a != b
    if bad.any():
        i = np.flatnonzero(bad.reshape(-1))
        raise AssertionError(f"{what}: {i.size} elements differ, first at {i[0]}: {a.reshape(-1)[i[0]]!r} != "
                             f"{b.reshape(-1)[i[0]]!r}")


SUCC = lambda x: np.nextafter(f32(x), f32(np.inf))
PRED = lambda x: np.nextafter(f32(x), f32(-np.inf))


# ---------------------------------------------------------------------------------------------------------------------
# A: the 5-sigma gate at equality
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class GateSet:
    """one record per cell against a cell state where |h - e| / sqrt(v) is exact in float32 (the crafted fold lists
    reach the gate within a few ulps, never at it)"""
    L: int
    init: dict
    key: np.ndarray
    R: np.ndarray
    G: np.ndarray
    B: np.ndarray
    I: np.ndarray
    h: np.ndarray
    v: np.ndarray
    pre_e: np.ndarray
    pre_v: np.ndarray

    def apply_init(self, m):
        for name, a in self.init.items():
            m.set_layer(name, a.reshape(self.L, self.L))

    def fuse_args(self):
        return self.key, self.R, self.G, self.B, self.I, self.h, self.v

    def ratio(self):
        return (np.abs(self.h - self.pre_e) / np.sqrt(np.maximum(self.pre_v, f32(1e-4)))).astype(f32)


def gate_records():
    """the ratio G_fuse compares with 5 (gpu_process.cu:502-504) exactly 5 (in the gate: fused) and one ulp either
    side, above and below the cell, with and without intensity (the colour gate, :488); plus a state below the variance
    floor (:500-501)"""
    L = 16
    init = {"elevation": np.full(L * L, f32(-10)), "variance": np.full(L * L, f32(-10)),
            "intensity": np.zeros(L * L, f32), "color_r": np.zeros(L * L, np.int32),
            "color_g": np.zeros(L * L, np.int32), "color_b": np.zeros(L * L, np.int32)}
    rec = []
    c = 0
    for e0, v0, d in ((1.0, 0.25, 2.5), (-2.0, 0.0625, 1.25), (0.5, 1.0, 5.0), (3.0, 4.0, 10.0), (0.75, 1e-6, 0.05)):
        for sign in (1, -1):
            for off in (-1, 0, 1):
                for inten in (0.0, 7.5):
                    h = f32(f32(e0) + f32(sign * d))
                    for _ in range(abs(off)):
                        h = np.nextafter(h, f32(sign * off * np.inf))
                    init["elevation"][c], init["variance"][c] = f32(e0), f32(v0)
                    init["intensity"][c] = f32(3.5)
                    init["color_r"][c], init["color_g"][c], init["color_b"][c] = 1, 2, 3
                    rec.append((c, 10 + c, 20, 30, inten, h, f32(e0), f32(v0)))
                    c += 1
    a = list(zip(*rec))
    i32 = lambda x: np.array(x, np.int32)
    return GateSet(L, init, i32(a[0]), i32(a[1]), i32(a[2]), i32(a[3]), np.array(a[4], f32), np.array(a[5], f32),
                   np.full(len(rec), f32(0.01)), np.array(a[6], f32), np.array(a[7], f32))


# ---------------------------------------------------------------------------------------------------------------------
# C: the point front end
# ---------------------------------------------------------------------------------------------------------------------
# T = a half turn about z: x_ts = -x and y_ts = -y exactly (1 * a + 0 * b + 0 * c + 0 == a), height = z.  The map is
# scrolled to y > 0, where every transformed point has a sensor y <= -1.5 and so passes the box filter.
HALF_TURN = np.diag([-1.0, -1.0, 1.0, 1.0])
FILTER_LIMITS_X = (-1.5, -1.0, 0.0, 1.0, 1.5)
FILTER_LIMITS_Y = (-1.5, -1.0, 0.0, 1.0, 1.5)


def front_end_frame():
    return sc.frame(HALF_TURN)


def axis_index(L, res, c, p, truncate=None):
    """PointsToIndex along one axis (gpu_process.cu:314-323) in float32, before its range check; truncate=True forces
    the even-L branch"""
    s = f32(f32(p) - f32(c))
    q = f32(s / f32(res))
    if (L % 2 == 0) if truncate is None else truncate:
        return int(np.trunc(f32(f32(L // 2) - q)))
    return L // 2 - int(math.trunc(float(q) + 0.5 * (1 if s > 0 else -1)))


def flip_points(L, res, c, b):
    """the float32 coordinates p, p + 1 ulp, p + 2 ulp where the index along an axis changes between p and p + 1 ulp,
    p nearest c + b * res.  For odd L and b = k + 0.5 with an exact quotient, p + 1 ulp is the boundary itself."""
    p0 = f32(float(c) + b * float(res))
    down, up = [p0], [p0]
    for _ in range(256):
        down.append(PRED(down[-1]))
        up.append(SUCC(up[-1]))
    cand = down[::-1] + up[1:]
    idx = [axis_index(L, res, c, p) for p in cand]
    flips = [i for i in range(len(cand) - 1) if idx[i] != idx[i + 1]]
    assert flips, (L, res, c, b)
    i = min(flips, key=lambda j: abs(j - 256))
    return [cand[i], cand[i + 1], SUCC(cand[i + 1])]


@dataclass
class FrontEndCase:
    name: str
    L: int
    res: float
    position: np.ndarray        # move() target from a new map: scrolls start and centre
    x: np.ndarray               # sensor-frame points (float32)
    y: np.ndarray
    z: np.ndarray
    boundary: np.ndarray        # bool per point: placed on a cell boundary (else on a filter limit)


def _boundaries(L):
    """the index quotients where the index changes, near the centre and at the window edges: +-(k + 0.5) for odd L;
    integers for even L, where the truncation toward zero moves the far edge from h to h + 1 (L/2 - q in (-1, 0]
    still truncates to index 0)"""
    h = L // 2
    ks = sorted({0, 1, 2, max(h - 1, 0), h})
    if L % 2:
        return sorted({s * (k + 0.5) for k in ks for s in (1, -1)})
    return sorted({-k for k in ks} | {k for k in ks if k < h} | {h + 1})


def _front_end_case(name, L, res, shift, seed):
    res32 = f32(res)
    centre = [f32(f32(k) * res32) for k in shift]
    rng = np.random.default_rng(seed)
    # a quarter cell off the cell centre: safely inside one cell for odd and even L
    inside = lambda c: f32(float(c) + 0.25 * float(res32))
    xs, ys = [], []
    bx = [p for b in _boundaries(L) for p in flip_points(L, res32, centre[0], b)]
    by = [p for b in _boundaries(L) for p in flip_points(L, res32, centre[1], b)]
    for p in bx:
        xs.append(p); ys.append(inside(centre[1]))
    for p in by:
        xs.append(inside(centre[0])); ys.append(p)
    for p, q in zip(bx, by[::-1]):          # both axes on a boundary at once
        xs.append(p); ys.append(q)
    nb = len(xs)
    lim = lambda v: (PRED(v), f32(v), SUCC(v))
    for a in FILTER_LIMITS_X:
        for b in FILTER_LIMITS_Y:
            for xa in lim(a):
                for yb in lim(b):
                    xs.append(-xa); ys.append(-yb)   # sensor (xa, yb) after the half turn
    xs, ys = np.array(xs, f32), np.array(ys, f32)
    z = rng.uniform(-0.5, 1.0, xs.shape[0]).astype(f32)
    boundary = np.arange(xs.shape[0]) < nb
    pos = np.array([centre[0], centre[1], f32(0.75)], f32)
    # transformed = (-x, -y): store the sensor-frame coordinates
    return FrontEndCase(name, L, float(res), pos, (-xs).astype(f32), (-ys).astype(f32), z, boundary)


def front_end_cases():
    """(L, res, shift in cells).  The y shift puts the window at y > 1.5 + half the window, so every boundary point
    passes the box filter; shifts are positive (>= L: the clear-all), never <= -L"""
    out = []
    for L, res, shift in ((1, 0.1, (3, 40)), (3, 0.1, (1, 40)), (3, 0.25, (7, 15)), (75, 0.1, (40, 60)),
                          (75, 0.05, (80, 120)), (201, 0.1, (130, 150)), (200, 0.1, (123, 150))):
        out.append(_front_end_case(f"L{L}_r{res}_s{shift[0]}_{shift[1]}", L, res, shift, 10 * L + shift[0]))
    return out


def box_filter_rejects(x, y):
    """the hard-coded filter of gpu_process.cu:393 (True: the point is dropped)"""
    x, y = np.asarray(x, f32).astype(np.float64), np.asarray(y, f32).astype(np.float64)
    return ((x > -1.5) & (x < 1.5) & (y > -1.5) & (y < 1.5)) | ((y > -1) & (y < 1)) | (y > 0)


# ---------------------------------------------------------------------------------------------------------------------
# D: scrolls and the map-wide calls
# ---------------------------------------------------------------------------------------------------------------------
SCROLL_L, SCROLL_RES = 48, 0.1


@dataclass
class Scroll:
    L: int
    res: float
    steps: list          # (op, args): fuse(seed), traver(seed), move(pos3), var(dv), opt(p2, dz), loop(p2, dz)
    marks: dict          # what the script reaches: name -> step indices


def fuse_records(L, seed, n=160):
    """a small Fuse call: heights near 0.5 with some jumps out of the gate, some invalid colours and intensities"""
    rng = np.random.default_rng(seed)
    key = rng.integers(0, L * L, n).astype(np.int32)
    h = (0.5 + rng.normal(0.0, 0.05, n) + np.where(rng.random(n) < 0.1, rng.uniform(-2.0, 2.0, n), 0.0)).astype(f32)
    v = rng.uniform(1e-3, 0.05, n).astype(f32)
    col = rng.integers(1, 256, (n, 3)).astype(np.int32)
    col[rng.random(n) < 0.1, rng.integers(0, 3)] = 0
    inten = rng.uniform(0.5, 50.0, n).astype(f32)
    inten[rng.random(n) < 0.1] = 0
    return key, col[:, 0].copy(), col[:, 1].copy(), col[:, 2].copy(), inten, h, v


def traver_pattern(L, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(-1.0, 1.0, (L, L)).astype(f32)


def scroll_script():
    L, res = SCROLL_L, f32(SCROLL_RES)
    centre, start = [f32(0), f32(0)], [0, 0]
    steps, marks = [], {}
    seed = [100]

    def mark(name):
        marks.setdefault(name, []).append(len(steps) - 1)

    def fuse():
        seed[0] += 1
        steps.append(("fuse", seed[0]))

    def move_to(pos, z=0.6):
        nonlocal centre, start
        c, s, _, ops = sc.move_model(L, res, centre, start, pos)
        shifts = [sc.index_shift(pos[i], centre[i], res) for i in range(2)]
        assert min(shifts) > -L, shifts                  # shifts <= -L write out of bounds in the reference
        steps.append(("move", np.array([pos[0], pos[1], z], f32)))
        for i, kind in enumerate(("rows", "cols")):
            if sum(1 for op in ops if op[0] == kind) == 2:
                mark(f"wrap_{kind}")
            if shifts[i] in (L - 1, -(L - 1)):
                mark(f"shift_{'+' if shifts[i] > 0 else '-'}(L-1)_{kind}")
            if shifts[i] == L:
                mark(f"shift_L_{kind}")
            if shifts[i] == L + 5:
                mark(f"shift_L+5_{kind}")
        if ("all",) in ops:
            mark("clear_all")
        centre, start = c, s
        fuse()

    def move_cells(dx, dy):
        pos = [f32(float(centre[0]) + dx * float(res)), f32(float(centre[1]) + dy * float(res))]
        for i, d in enumerate((dx, dy)):
            assert sc.index_shift(pos[i], centre[i], res) == d
        move_to(pos)

    def opt(p, dz):
        nonlocal centre
        a = sc._opt_move_centre(centre, p, res)
        if a != sc._closeloop_centre(centre, p, res):
            mark("opt_differs_from_closeloop")
        steps.append(("opt", (np.array(p, f32), dz)))
        centre = a
        fuse()

    def loop(p, dz):
        nonlocal centre
        a = sc._closeloop_centre(centre, p, res)
        if a != sc._opt_move_centre(centre, p, res):
            mark("closeloop_differs_from_opt")
        steps.append(("loop", (np.array(p, f32), dz)))
        centre = a
        fuse()

    fuse()
    steps.append(("traver", 1))
    move_cells(5, 7)
    move_cells(-(L - 1), 0)
    move_cells(0, -(L - 1))
    move_cells(L - 1, L - 1)
    move_cells(-20, 31)
    move_cells(33, -26)
    steps.append(("var", 0.003))                         # bands just cleared hold variance -10: left alone
    fuse()
    move_cells(-7, -9)
    steps.append(("var", -0.004))
    steps.append(("traver", 2))
    move_cells(L, 0)                                     # clear-all: traver reset too
    fuse()
    steps.append(("traver", 3))
    move_cells(3, L + 5)
    steps.append(("traver", 4))
    move_cells(L - 1, -(L - 1))
    # far from the origin (positive shifts only: a shift <= -L is not a defined call)
    move_to([f32(1234.5678), f32(987.6543)])
    steps.append(("traver", 5))
    for k, sign in ((2, 1), (2, -1), (L - 2, -1), (L - 2, 1), (L - 1, 1)):
        for before in (True, False):
            move_to([f32(sc.boundary_position(res, centre[0], k, sign, before)),
                     f32(sc.boundary_position(res, centre[1], 1, -sign, not before))])
            mark("boundary_position")
    steps.append(("var", -0.02))
    fuse()
    # Map_optmove / Map_closeloop: targets one ulp either side of their rounding boundaries
    for k, sign, dz in ((3, 1, 0.25), (3, -1, -0.5), (11, 1, 0.125), (0, -1, 1.5)):
        for before in (True, False):
            p = [f32(sc.boundary_position(res, centre[0], k, sign, before)),
                 f32(sc.boundary_position(res, centre[1], k + 1, -sign, before))]
            opt(p, dz) if before else loop(p, dz)
    move_cells(4, -3)                                    # a move from the unaligned centre Map_optmove leaves
    opt([f32(5000.123), f32(7000.987)], 0.0)             # far centres: an unaligned centre far from the origin
    loop([f32(-5000.321), f32(-6000.5)], -0.75)
    opt([f32(-5000.0), f32(-6000.0)], 0.0625)
    steps.append(("traver", 6))
    move_cells(L, L)
    move_cells(L + 5, L - 1)
    steps.append(("var", 0.01))
    fuse()
    return Scroll(L, float(res), steps, marks)


def apply_step(m, op, args, reference=None, like=None):
    """one scroll step on a map with the OracleMap / ElevationMap interface.  For a ref_lib.PinnedRef pass
    reference=True and like=the oracle's result of the same step (move and opt return arrays that are pinned)."""
    if op == "fuse":
        m.fuse_points(*fuse_records(SCROLL_L, args))
    elif op == "traver":
        m.set_layer("traver", traver_pattern(SCROLL_L, args))
    elif op == "move":
        return m.move(args, like=like) if reference else m.move(args)
    elif op == "var":
        m.var_update(args)
    elif op == "opt":
        p, dz = args
        return m.opt_move(p, dz, like=like) if reference else m.opt_move(p, dz)
    elif op == "loop":
        p, dz = args
        m.closeloop(p, dz)
    else:
        raise ValueError(op)
    return None


SCROLL_LAYERS = ("elevation", "variance", "intensity", "color_r", "color_g", "color_b", "traver", "lowest")
