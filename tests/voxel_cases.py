"""Crafted cases of gem_voxel_grid (DESIGN.md f9) and an independent numpy restatement of it.  TEST INFRASTRUCTURE ONLY.

The restatement computes the call with whole-array float32 / float64 expressions: the voxel order by np.lexsort on
(ijk2, ijk1, ijk0, input index), the centroid sums strictly in that order (np.add.accumulate in float32 from a +0.0 row
for long voxels, one vectorised step per position for the others; never np.sum, which sums pairwise).  The oracle
(tests/orc_voxel_grid.c) instead runs PCL's loops with a 64-bit idx and qsort.  A case is
(name, xyzi (n, 4) float32, leaf, field, limits, negative)."""
from __future__ import annotations

import numpy as np

FIELDS = {None: -1, "x": 0, "y": 1, "z": 2, "intensity": 3}
FLT_MAX = 3.4028234663852886e38
ALL = (-FLT_MAX, FLT_MAX)
F = np.float32


# ---- the numpy restatement -------------------------------------------------------------------------------------------
def _masks(pts, field, limits, negative):
    """(V2 used, V3 bounded)"""
    fin = np.isfinite(pts[:, :3]).all(axis=1)
    if field is None:
        return fin, fin
    v = pts[:, FIELDS[field]]
    lo, hi = float(limits[0]), float(limits[1])
    vd = v.astype(np.float64)
    flo, fhi = F(lo), F(hi)
    with np.errstate(invalid="ignore"):
        if negative:
            cut_d, cut_f = (vd < hi) & (vd > lo), (v < fhi) & (v > flo)
        else:
            cut_d, cut_f = (vd > hi) | (vd < lo), (v > fhi) | (v < flo)
    return fin & ~cut_d, fin & ~cut_f


def _nan_bits(partial_nan, p):
    """the bits of the first NaN of a run: x86-64's, the NaN input quieted, or the default NaN of inf - inf"""
    pb = p.view(np.uint32)
    return np.where(np.isnan(p), pb | np.uint32(0x00400000), np.uint32(0xFFC00000)).astype(np.uint32) * partial_nan


def _run_sums(vals, starts, lengths):
    """per run, +0.0f + p0 + p1 + ... in float32, strictly in order, and per component the bits of the first NaN the
    chain produces (0 for none)"""
    out = np.zeros((starts.size, 4), np.float32)
    nan = np.zeros((starts.size, 4), np.uint32)
    long_ = lengths > 2048
    with np.errstate(invalid="ignore", over="ignore"):   # inf + -inf is NaN, as in C
        for r in np.flatnonzero(long_):
            s, n = int(starts[r]), int(lengths[r])
            run = np.concatenate([np.zeros((1, 4), np.float32), vals[s:s + n]])
            acc = np.add.accumulate(run, axis=0, dtype=np.float32)
            out[r] = acc[-1]
            for q in range(4):
                hit = np.flatnonzero(np.isnan(acc[1:, q]))
                if hit.size:
                    nan[r, q] = _nan_bits(True, vals[s + hit[0], q:q + 1])[0]
        short = np.flatnonzero(~long_)
        if short.size:
            for j in range(int(lengths[short].max())):
                k = short[lengths[short] > j]
                p = vals[starts[k] + j]
                out[k] = out[k] + p
                first = np.isnan(out[k]) & (nan[k] == 0)
                nan[k] = np.where(first, _nan_bits(first, p), nan[k])
    return out, nan


def np_voxel_grid(xyzi, leaf, field=None, limits=ALL, negative=False):
    """(out, info) as the oracle returns them with an unlimited capacity"""
    pts = np.ascontiguousarray(xyzi, np.float32).reshape(-1, 4)
    n = pts.shape[0]
    leaf = np.full(3, leaf, np.float32) if np.ndim(leaf) == 0 else np.asarray(leaf, np.float32)
    inv = F(1.0) / leaf
    used, bnd = _masks(pts, field, limits, negative)
    info = {"count": 0, "used": int(used.sum()), "passthrough": 0}
    empty = np.zeros((0, 4), np.float32)
    if not bnd.any():
        return empty, info
    b = pts[bnd, :3]
    mn, mx = b.min(axis=0), b.max(axis=0)
    with np.errstate(over="ignore", invalid="ignore"):
        q = (mx - mn) * inv
    over = not np.isfinite(q).all() or bool((q >= F(2.0 ** 62)).any())
    if not over:
        d = [int(v) + 1 for v in q]
        over = d[0] * d[1] * d[2] > 2 ** 31 - 1
    if over:
        info.update(count=n, passthrough=1)
        return pts.copy(), info
    if not used.any():
        return empty, info
    minb = np.floor(mn * inv).astype(np.float64)
    src = np.flatnonzero(used)
    p = pts[src]
    ijk = (np.floor(p[:, :3] * inv).astype(np.float64) - minb).astype(np.int64)
    assert (ijk >= 0).all()
    order = np.lexsort((src, ijk[:, 0], ijk[:, 1], ijk[:, 2]))
    ijk, vals = ijk[order], p[order]
    new = np.ones(ijk.shape[0], bool)
    new[1:] = (ijk[1:] != ijk[:-1]).any(axis=1)
    starts = np.flatnonzero(new)
    lengths = np.diff(np.append(starts, ijk.shape[0]))
    sums, nan = _run_sums(vals, starts, lengths)
    with np.errstate(invalid="ignore"):
        out = sums / lengths.astype(np.float32)[:, None]
    out = np.where(nan != 0, nan.view(np.float32), out)
    info["count"] = int(starts.size)
    return out.astype(np.float32), info


def div_product(xyzi, leaf, field=None, limits=ALL, negative=False):
    """(d0 d1 d2 of V4, div0 div1 div2 of V6) over the V3 bounds"""
    pts = np.ascontiguousarray(xyzi, np.float32).reshape(-1, 4)
    leaf = np.full(3, leaf, np.float32) if np.ndim(leaf) == 0 else np.asarray(leaf, np.float32)
    inv = F(1.0) / leaf
    _, bnd = _masks(pts, field, limits, negative)
    b = pts[bnd, :3]
    mn, mx = b.min(axis=0), b.max(axis=0)
    d = [int(v) + 1 for v in (mx - mn) * inv]
    div = [int(v) for v in (np.floor(mx * inv).astype(np.float64) - np.floor(mn * inv).astype(np.float64) + 1)]
    return d[0] * d[1] * d[2], div[0] * div[1] * div[2]


# ---- crafted cases ---------------------------------------------------------------------------------------------------
def _cloud(rng, n, lo, hi, intensity=(0.0, 255.0)):
    p = np.empty((n, 4), np.float32)
    p[:, :3] = rng.uniform(lo, hi, (n, 3))
    p[:, 3] = rng.uniform(*intensity, n)
    return p


def _edges(leaf):
    """coordinates on the voxel edges k * leaf and one float below each"""
    e = np.array([F(k * leaf) for k in range(-4, 5)], np.float32)
    below = np.nextafter(e, F(-np.inf))
    return np.concatenate([e, below])


def cases():
    rng = np.random.default_rng(2024)
    out = []

    for leaf in (0.5, 0.1):
        v = _edges(leaf)
        g = np.stack(np.meshgrid(v, v[::3], v[::5], indexing="ij"), -1).reshape(-1, 3)
        p = np.concatenate([g, rng.uniform(0, 255, (g.shape[0], 1))], 1).astype(np.float32)
        out.append((f"edges_{leaf}", p[rng.permutation(p.shape[0])], leaf, None, ALL, False))

    nz = np.array([[-0.0, -0.0, -0.0, -0.0],                      # alone in its voxel: comes out +0.0
                   [-0.25, -0.0, 0.0, 3.0], [-1e-30, 0.0, -0.0, 1.0], [-0.05, -0.1, -0.15, 2.0], [-7.5, -0.0, 0.4, 0.0],
                   [-0.0, 0.0, 0.0, -0.0], [-3.0, -2.0, -1.0, -0.0], [-2.99, -1.99, -0.99, -5.0]], np.float32)
    out.append(("negative_and_negzero", nz, 0.2, None, ALL, False))
    out.append(("negzero_alone", nz[:1].copy(), 0.2, None, ALL, False))

    base = _cloud(rng, 400, -2.0, 2.0)
    for comp in range(4):
        p = base.copy()
        p[0::7, comp] = np.nan
        p[1::11, comp] = np.inf
        p[2::13, comp] = -np.inf
        for field in (None, "x", "y", "z", "intensity"):
            out.append((f"nonfinite_{'xyzi'[comp]}_field_{field}", p, 0.3, field, (-1.0, 1.5), False))

    # NaN bits of the sums: inf - inf then a NaN (the default NaN stays), NaNs with payloads and a signalling NaN
    # (quieted), one NaN after another (the first stays); each row group is one voxel
    nb = np.array([0x7fc12345, 0x7f800001, 0xffc0beef, 0x7fc00000], np.uint32).view(np.float32)
    w = np.array([[1.0, np.inf, -np.inf, nb[0]], [nb[0], nb[2], 1.0, np.inf], [nb[1], 2.0, nb[3], -np.inf],
                  [np.inf, -np.inf, 3.0, 4.0], [5.0, nb[2], nb[1], 6.0]], np.float32)
    pts = np.zeros((w.size, 4), np.float32)
    pts[:, 0] = np.repeat(np.arange(w.shape[0]) * 1.0 + 0.5, w.shape[1])
    pts[:, 1] = 0.25
    pts[:, 3] = w.reshape(-1)
    out.append(("nan_bits_intensity", pts, 1.0, None, ALL, False))

    p = _cloud(rng, 300, -2.0, 2.0)
    for field in ("x", "y", "z", "intensity"):
        f = FIELDS[field]
        vals = np.sort(p[:, f])
        lims = (float(vals[40]), float(vals[250]))        # limits equal to a point's value
        for neg in (False, True):
            out.append((f"limits_equal_{field}_neg{int(neg)}", p, 0.25, field, lims, neg))

    q = _cloud(rng, 500, -2.0, 2.0, intensity=(0.0, 5.0))
    q[::9, 3] = np.nan                                     # NaN intensities pass the field test
    for field in ("x", "y", "z", "intensity"):
        for neg in (False, True):
            out.append((f"field_{field}_neg{int(neg)}", q, 0.2, field, (-0.7, 1.1), neg))

    # limits at float roundings: float32(0.1) lies above the double 0.1, so V2 cuts the point and V3 (float limits)
    # keeps it; its far y then widens the V3 bounds past the overflow check, so the output is the input
    r = _cloud(rng, 200, -1.0, 0.09)
    r[:, 1:3] = rng.uniform(0.0, 0.5, (200, 2))
    r[7] = [F(0.1), 2000.0, 0.2, 1.0]
    out.append(("limit_rounding_passthrough", r, 1e-3, "x", (-1.0, 0.1), False))
    out.append(("limit_rounding_without_point", np.delete(r, 7, axis=0), 1e-3, "x", (-1.0, 0.1), False))
    lim_lo = float(np.nextafter(F(-0.5), F(0)))            # a double limit that is a float
    out.append(("limit_rounding_negative", r, 0.05, "x", (float(F(-0.5)) - 1e-12, 0.1), True))
    out.append(("limit_at_float_lo", r, 0.05, "x", (lim_lo, 0.05), False))

    out.append(("anisotropic", _cloud(rng, 5000, -3.0, 3.0), (0.1, 0.25, 0.7), None, ALL, False))

    t = _cloud(rng, 1000, -50.0, 50.0)
    t[::17, 0] = np.nan
    out.append(("passthrough_tiny_leaf", t, 1e-6, "x", (-10.0, 10.0), False))
    h = _cloud(rng, 64, -1.0, 1.0)
    h[0, :3] = [-1e30, 0.0, 0.0]
    h[1, :3] = [1e30, 0.0, 0.0]
    out.append(("passthrough_huge_coordinates", h, 1.0, None, ALL, False))
    h2 = h.copy()
    h2[0, :3] = [-3e38, 0.0, 0.0]
    h2[1, :3] = [3e38, 0.0, 0.0]
    out.append(("passthrough_infinite_span", h2, 1.0, None, ALL, False))
    far = _cloud(rng, 2000, 0.0, 1.0)
    far[:, :3] = far[:, :3] * 4000.0 + 1e10                # beyond the int range, a span of a few voxels
    out.append(("far_from_origin", far, 1000.0, None, ALL, False))

    # V6 DEFINED: d0 d1 d2 = 1290^3 <= INT32_MAX (V4 passes) but div0 div1 div2 = 1291^3 > 2^31
    c = np.array([[0.9, 0.9, 0.9, 1.0], [1290.4, 1290.4, 1290.4, 2.0]], np.float32)
    c = np.concatenate([c, _cloud(rng, 3000, 0.9, 1290.4)])
    c[2:200, 2] = rng.uniform(1289.0, 1290.4, 198)         # keys that wrap an int idx
    out.append(("defined_order", c[rng.permutation(c.shape[0])], 1.0, None, ALL, False))

    out.append(("empty", np.zeros((0, 4), np.float32), 0.1, None, ALL, False))
    a = _cloud(rng, 100, -1.0, 1.0)
    a[:, 1] = np.nan
    out.append(("all_cut_nonfinite", a, 0.1, None, ALL, False))
    out.append(("all_cut_field", _cloud(rng, 100, -1.0, 1.0), 0.1, "z", (5.0, 6.0), False))

    g = np.stack(np.meshgrid(np.arange(20), np.arange(15), np.arange(8), indexing="ij"), -1).reshape(-1, 3)
    own = np.concatenate([(g * 0.2 + 0.1), rng.uniform(0, 255, (g.shape[0], 1))], 1).astype(np.float32)
    out.append(("own_voxel", own[rng.permutation(own.shape[0])], 0.2, None, ALL, False))

    out.append(("dense_random", _cloud(rng, 20000, -2.0, 2.0), 0.3, None, ALL, False))
    return out


def one_voxel_case(n=1 << 20):
    """one voxel holding n points (the sequential sum of V8 decides every bit)"""
    rng = np.random.default_rng(77)
    p = _cloud(rng, n, 0.01, 0.09, intensity=(0.0, 255.0))
    return ("one_voxel_1m", p, 0.1, None, ALL, False)


def case_by_name(name):
    if name == "one_voxel_1m":
        return one_voxel_case()
    return next(c for c in cases() if c[0] == name)


def case_names():
    return [c[0] for c in cases()] + ["one_voxel_1m"]
