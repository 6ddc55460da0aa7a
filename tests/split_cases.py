"""Crafted grid clouds for the global-map filter (gem_grid_cloud_split, tests/orc_grid_split.c).  CPU only.

np_grid_split() is an independent restatement of the filter: candidates from scipy's cKDTree (double distances over the
float32 positions), every d2 recomputed in float32 in FLANN's order, and the candidate set proven complete before it is
used; then PCL's statistics and the split.  cloud_cases() are record arrays laid out like a grid cloud (cell-centre
positions from grid_map's formula, GridMapIterator order) that put points where the filter makes decisions.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

f32 = np.float32


def grid_records(L, res, centre, start, z_geo, trav_geo):
    """records of the cells whose z is not the -10 sentinel, in GridMapIterator order (storage ix fastest), with the
    positions gridMaptoPointCloud writes (grid_map getPositionFromIndex in double, then float)"""
    half = 0.5 * (L * res) - 0.5 * res
    out = []
    for iy in range(L):
        for ix in range(L):
            gx, gy = (ix - start[0]) % L, (iy - start[1]) % L
            z = z_geo[gx, gy]
            if z == f32(-10.0):
                continue
            x = f32(float(f32(centre[0])) + half - res * gx)
            y = f32(float(f32(centre[1])) + half - res * gy)
            out.append([x, y, z, 1.0, 0.0, 0.01, 10.0, trav_geo[gx, gy]])
    return np.array(out, f32).reshape(-1, 8)


def _d2(a, b):
    """FLANN's L2_Simple in float32: r = 0; r += d*d per dimension"""
    d = (a - b).astype(f32)
    r = f32(0.0)
    r = (r + d[..., 0] * d[..., 0]).astype(f32)
    r = (r + d[..., 1] * d[..., 1]).astype(f32)
    return (r + d[..., 2] * d[..., 2]).astype(f32)


def np_grid_split(records, mean_k=20, stddev_mul=1.0, travers_threshold=0.0):
    rec = np.asarray(records, f32).reshape(-1, 8)
    n = rec.shape[0]
    xyz = rec[:, :3]
    fin = np.isfinite(xyz).all(axis=1)
    idx = np.flatnonzero(fin)
    pts = xyz[idx]
    K = mean_k + 1
    dist = np.zeros(n, f32)
    nf = idx.size
    if nf > mean_k:
        tree = cKDTree(pts.astype(np.float64))
        k = min(nf, K + 8)
        todo = np.arange(nf)
        while todo.size:
            dd, nb = tree.query(pts[todo].astype(np.float64), k=k)
            dd, nb = dd.reshape(todo.size, k), nb.reshape(todo.size, k)
            d2 = _d2(pts[todo][:, None, :], pts[nb])
            d2.sort(axis=1)
            kth = d2[:, K - 1].astype(np.float64)
            # complete when every point outside the candidates is provably no closer: its exact distance is >= the
            # largest candidate distance D, and a float d2 is within a relative 1e-6 of the exact square
            ok = (k == nf) | (kth < (dd[:, -1] ** 2) * (1 - 1e-5))
            s = np.zeros(ok.sum())
            for j in range(1, K):
                s = s + np.sqrt(d2[ok, j].astype(np.float64))
            dist[idx[todo[ok]]] = (s / mean_k).astype(f32)
            todo = todo[~ok]
            k = min(nf, 2 * k)
        valid = nf
        s = 0.0
        sq = 0.0
        for v in dist:
            s += float(v)
            sq += float(f32(v * v))
        mean = s / valid
        with np.errstate(all="ignore"):
            var = (sq - s * s / valid) / (valid - 1.0)
            sd = float(np.sqrt(np.float64(var)))
        thr = mean + stddev_mul * sd
    else:
        dist[:] = np.nan
        valid, mean, sd, thr = 0, np.nan, np.nan, np.nan
    with np.errstate(invalid="ignore"):
        keep = ~(dist.astype(np.float64) > thr)
    road = keep & (rec[:, 7].astype(np.float64) > travers_threshold)
    obst = keep & ~road
    return {"dist": dist, "road": rec[road], "obstacle": rec[obst], "valid": valid, "mean": mean, "stddev": sd,
            "threshold": thr}


def _surface(rng, L, res, empty=0.1):
    g = np.arange(L)
    z = (0.15 * g[:, None] * res - 0.2 * g[None, :] * res + rng.normal(0, 0.04, (L, L))).astype(f32)
    z[rng.random((L, L)) < empty] = f32(-10.0)
    return z


def _trav(rng, L):
    return rng.uniform(-0.6, 1.0, (L, L)).astype(f32)


def cloud_cases():
    """(name, records, [(mean_k, stddev_mul, travers_threshold), ...])"""
    rng = np.random.default_rng(5)
    cases = []
    std = [(20, 1.0, 0.0), (1, 0.0, 0.0), (2, -1.0, 0.3), (64, 1.0, 0.0)]
    for L, res, start in ((24, 0.1, (0, 0)), (25, 0.05, (7, 19)), (32, 0.2, (31, 3))):
        cases.append((f"surface_L{L}", grid_records(L, res, (0.3, -1.2), start, _surface(rng, L, res), _trav(rng, L)), std))
    # sparse: a few points 3..L cells apart, plus an isolated cell in a corner
    L = 48
    z = np.full((L, L), f32(-10.0))
    pick = rng.choice(L * L, 40, replace=False)
    z.ravel()[pick] = rng.normal(0, 0.2, 40).astype(f32)
    z[0, 0] = f32(0.5)
    cases.append(("sparse", grid_records(L, 0.1, (0, 0), (5, 9), z, _trav(rng, L)), [(20, 1.0, 0.0), (2, 0.0, 0.0)]))
    # exactly mean_k, mean_k + 1 and mean_k + 2 finite points, and non-finite ones beside them
    for extra in (0, 1, 2):
        L = 16
        z = np.full((L, L), f32(-10.0))
        z.ravel()[rng.choice(L * L, 20 + extra, replace=False)] = rng.normal(0, 0.3, 20 + extra).astype(f32)
        rec = grid_records(L, 0.1, (0, 0), (3, 3), z, _trav(rng, L))
        rec = np.concatenate([rec, np.array([[0.05, 0.05, np.nan, 1, 0, 0.01, 10, 0.5]], f32)])
        cases.append((f"count_{20 + extra}", rec, [(20, 1.0, 0.0)]))
    # steps of several metres
    L = 32
    z = _surface(rng, L, 0.1, empty=0.0)
    z[:, 16:] += f32(4.0)
    z[10:14, 3:7] += f32(-7.5)
    cases.append(("steps", grid_records(L, 0.1, (0, 0), (0, 11), z, _trav(rng, L)), std))
    # non-finite and +-1e18 elevations
    z = _surface(rng, L, 0.1, empty=0.05)
    z.ravel()[rng.choice(L * L, 30, replace=False)] = np.nan
    z.ravel()[rng.choice(L * L, 20, replace=False)] = np.inf
    z.ravel()[rng.choice(L * L, 20, replace=False)] = f32(1e18)
    z.ravel()[rng.choice(L * L, 20, replace=False)] = f32(-1e18)
    cases.append(("magnitudes", grid_records(L, 0.1, (0, 0), (4, 4), z, _trav(rng, L)), std))
    # about 2e5 m from the origin at 0.01 m: neighbouring centres round to the same float
    L = 40
    cases.append(("far", grid_records(L, 0.01, (2.0e5 + 0.37, 2.0e5 - 0.41), (13, 2), _surface(rng, L, 0.01, 0.05),
                                      _trav(rng, L)), std))
    # pairs 0.25 m apart, far from each other: with mean_k = 1 every distance equals the threshold
    L = 64
    z = np.full((L, L), f32(-10.0))
    for a in range(4, L - 8, 12):
        for b in range(4, L - 8, 12):
            z[a, b] = z[a, b + 1] = f32(0.0)
    cases.append(("pairs", grid_records(L, 0.25, (0, 0), (0, 0), z, _trav(rng, L)), [(1, 1.0, 0.0), (1, 0.0, 0.0), (1, -1.0, 0.0)]))
    # traversabilities at the threshold and one ulp either side
    L = 20
    t = np.full((L, L), f32(0.25))
    t[::3] = np.nextafter(f32(0.25), f32(1))
    t[1::3] = np.nextafter(f32(0.25), f32(-1))
    cases.append(("trav_ties", grid_records(L, 0.1, (0, 0), (0, 0), _surface(rng, L, 0.1, 0.0), t),
                  [(20, 1.0, float(f32(0.25))), (20, 1.0, float(np.nextafter(f32(0.25), f32(1))))]))
    return cases
