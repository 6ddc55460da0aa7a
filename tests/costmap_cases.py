"""Crafted cases of the costmap calls (DESIGN.md f8) and an independent numpy restatement of them.  TEST INFRASTRUCTURE
ONLY.

The restatement computes each call as a whole-array expression (the last writer of a cell is the largest order that
maps there, np.maximum.at), where the oracle (tests/orc_costmap.c) runs the reference's loops.  A window is
(origin_x, origin_y, resolution, size_x, size_y); grids are (size_y, size_x) uint8 arrays; records (n, 8) float32."""
from __future__ import annotations

import numpy as np

FREE, LETHAL, UNKNOWN = 0, 254, 255
F32_07 = float(np.float32(0.7))


# ---- the numpy restatement -------------------------------------------------------------------------------------------
def np_world_to_map(window, wx, wy):
    """(accepted mask, mx, my) of worldToMap over float64 arrays; non-finite coordinates and quotients >= 2^31 are not
    on the map"""
    ox, oy, res, sx, sy = window
    with np.errstate(all="ignore"):
        ok = np.isfinite(wx) & np.isfinite(wy) & ~(wx < ox) & ~(wy < oy)
        qx, qy = (wx - ox) / res, (wy - oy) / res
        ok &= (qx < 2.0 ** 31) & (qy < 2.0 ** 31)
        mx = np.where(ok, qx, 0.0).astype(np.int64)
        my = np.where(ok, qy, 0.0).astype(np.int64)
    ok &= (mx < sx) & (my < sy)
    return ok, mx, my


def np_scatter(window, grid, wx, wy, cost, writes, rank=None):
    """the last element (in array order, or of the largest `rank`) that writes a cell wins it; the marks over every
    written element"""
    _, _, _, sx, sy = window
    g = np.array(grid, np.uint8).reshape(-1).copy()
    ok, mx, my = np_world_to_map(window, wx, wy)
    ok &= writes
    idx = np.flatnonzero(ok)
    cell = my[idx] * sx + mx[idx]
    key = idx if rank is None else np.asarray(rank, np.int64)[idx]
    best = np.full(sx * sy, -1, np.int64)
    np.maximum.at(best, cell, key)
    has = best >= 0
    if rank is None:
        winner = best
    else:   # the element holding each cell's largest rank
        pos = np.full(sx * sy, -1, np.int64)
        mine = key == best[cell]
        pos[cell[mine]] = idx[mine]
        winner = pos
    g[has] = cost[winner[has]]
    if idx.size:
        b = (float(wx[idx].min()) + 0.0, float(wy[idx].min()) + 0.0, float(wx[idx].max()) + 0.0, float(wy[idx].max()) + 0.0)
    else:
        b = (np.inf, np.inf, -np.inf, -np.inf)
    marks = {"marked": int(idx.size), "lethal": int(np.count_nonzero(cost[idx] == LETHAL)),
             "min_x": b[0], "min_y": b[1], "max_x": b[2], "max_y": b[3]}
    return g.reshape(sy, sx), marks


def np_mark_points(records, window, grid, thresh):
    rec = np.asarray(records, np.float32).reshape(-1, 8)
    t = rec[:, 7].astype(np.float64)
    with np.errstate(invalid="ignore"):
        cost = np.where(t > thresh, FREE, LETHAL).astype(np.uint8)
    return np_scatter(window, grid, rec[:, 0].astype(np.float64), rec[:, 1].astype(np.float64), cost,
                      np.ones(rec.shape[0], bool))


def np_grid_positions(L, grid_res, centre, start):
    """grid_map cell-centre positions of every cell in GridMapIterator order (ix + iy * L over storage indices)"""
    k = np.arange(L * L)
    ix, iy = k % L, k // L
    half = 0.5 * (L * grid_res) - 0.5 * grid_res
    px = (np.float64(np.float32(centre[0])) + half) - grid_res * ((ix + L - int(start[0])) % L).astype(np.float64)
    py = (np.float64(np.float32(centre[1])) + half) - grid_res * ((iy + L - int(start[1])) % L).astype(np.float64)
    return px, py


def np_mark_map(traver, L, grid_res, centre, start, window, grid, thresh, mark_unknown=True, geographic=False):
    """traver: (L, L) indexed [ix, iy], NaN where show() cleared the cell.  geographic=True lets the last cell in
    geographic order win instead of the last in GridMapIterator order (what a scatter that ignored the circular buffer's
    start index would do): tests use it to show that a case tells the two apart."""
    v = np.asarray(traver, np.float32).reshape(L, L).reshape(-1, order="F").astype(np.float64)
    px, py = np_grid_positions(L, grid_res, centre, start)
    with np.errstate(invalid="ignore"):
        cost = np.where(v < thresh, LETHAL, FREE).astype(np.uint8)
    writes = np.ones(v.size, bool) if mark_unknown else ~np.isnan(v)
    rank = None
    if geographic:
        k = np.arange(L * L)
        rank = ((k // L + L - int(start[1])) % L) * L + (k % L + L - int(start[0])) % L
    return np_scatter(window, grid, px, py, cost, writes, rank)


def np_update_origin(window, nx, ny, fill, grid):
    ox, oy, res, sx, sy = window
    qx, qy = (nx - ox) / res, (ny - oy) / res
    if not (abs(qx) < 2.0 ** 31 and abs(qy) < 2.0 ** 31):
        return None
    cx, cy = int(qx), int(qy)
    g = np.asarray(grid, np.uint8).reshape(sy, sx)
    if cx == 0 and cy == 0:
        return tuple(window), g.copy()
    out = np.full((sy, sx), fill, np.uint8)
    jj, ii = np.mgrid[0:sy, 0:sx]
    oi, oj = ii + cx, jj + cy
    inside = (oi >= 0) & (oi < sx) & (oj >= 0) & (oj < sy)
    out[inside] = g[oj[inside], oi[inside]]
    return (ox + cx * res, oy + cy * res, res, sx, sy), out


def np_combine(mode, layer, master, sx, sy, rect):
    i0, j0, i1, j1 = rect
    i0, j0, i1, j1 = max(i0, 0), max(j0, 0), min(i1, sx), min(j1, sy)
    m = np.asarray(master, np.uint8).reshape(sy, sx).copy()
    if i0 >= i1 or j0 >= j1:
        return m
    lay = np.asarray(layer, np.uint8).reshape(sy, sx)[j0:j1, i0:i1]
    sub = m[j0:j1, i0:i1]
    if mode == 1:
        w = lay != UNKNOWN
    else:
        w = (lay != UNKNOWN) & ((sub == UNKNOWN) | (sub < lay))
    sub[w] = lay[w]
    return m


# ---- crafted inputs ----------------------------------------------------------------------------------------------------
def records(xy, travers):
    xy = np.asarray(xy, np.float32).reshape(-1, 2)
    r = np.zeros((xy.shape[0], 8), np.float32)
    r[:, :2] = xy
    r[:, 3] = 1.0
    r[:, 7] = np.asarray(travers, np.float32)
    return r


def random_grid(rng, window, unknown_share=0.3):
    g = rng.choice(np.array([FREE, LETHAL, 17, 128], np.uint8), size=(window[4], window[3]))
    g[rng.random(g.shape) < unknown_share] = UNKNOWN
    return g


def _f32_neighbours(v):
    f = np.float32(v)
    return [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]


def point_cases():
    """(name, records, window, thresh, initial grid)"""
    rng = np.random.default_rng(41)
    out = []
    # cell edges, the origin, one ulp below it, and (wx - origin) / res just below and at size
    for w in [(-1.0, 2.0, 0.25, 40, 30), (-3.7, -1.3, 0.2, 37, 23), (0.0, 0.0, 0.05, 64, 64)]:
        ox, oy, res, sx, sy = w
        xs = []
        for k in list(range(0, sx + 1)) + [sx - 1, sx]:
            xs += _f32_neighbours(ox + k * res)
        ys = []
        for k in list(range(0, sy + 1)):
            ys += _f32_neighbours(oy + k * res)
        X, Y = np.meshgrid(np.array(xs, np.float32), np.array(ys, np.float32))
        xy = np.stack([X.ravel(), Y.ravel()], 1)
        t = rng.choice(np.array([0.1, 0.9, F32_07, np.nan], np.float32), xy.shape[0])
        out.append((f"edges_{sx}x{sy}", records(xy, t), w, 0.7, random_grid(rng, w)))
    w = (-2.0, -2.0, 0.2, 20, 20)
    # non-finite coordinates among valid ones; huge quotients
    bad = [np.nan, np.inf, -np.inf, 3.0e9, -3.0e9, np.float32(-2.0 + 0.2 * 2.0 ** 31), 1e38]
    xy = [(a, 0.5) for a in bad] + [(0.5, a) for a in bad] + [(a, b) for a in bad for b in bad] + [(0.1, 0.1), (-1.9, 1.9)]
    out.append(("nonfinite", records(xy, np.linspace(0, 1, len(xy))), w, 0.5, random_grid(rng, w)))
    # travers equal to the threshold, 0.7f against 0.7 and 0.7f against 0.7f, NaN travers, signed zeros
    xy = [(0.1 + 0.2 * i, 0.1) for i in range(8)]
    t = [F32_07, 0.7, np.nextafter(np.float32(0.7), np.float32(1)), np.nan, 0.0, -0.0, 1.0, -np.nan]
    for th in (0.7, F32_07, 0.0):
        out.append((f"thresh_{th!r}", records(xy, t), w, th, random_grid(rng, w)))
    z = np.float32(0.0)
    out.append(("signed_zero", records([(-z, -z), (z, z), (-z, 0.3), (0.3, -z)], [1, 0, 1, 0]), (-1.0, -1.0, 0.5, 8, 8), 0.5,
                random_grid(rng, (-1.0, -1.0, 0.5, 8, 8))))
    out.append(("empty", records(np.zeros((0, 2)), []), w, 0.7, random_grid(rng, w)))
    # many records per cell with alternating travers, early and late in the cloud, in different blocks (> 1 M records)
    w2 = (-5.0, -5.0, 0.5, 20, 20)
    n = 1_200_000
    cells = rng.integers(0, 400, n)
    xy = np.stack([-5.0 + 0.5 * (cells % 20) + rng.random(n) * 0.49, -5.0 + 0.5 * (cells // 20) + rng.random(n) * 0.49], 1)
    t = np.where(np.arange(n) % 2 == 0, 0.9, 0.1)
    xy[n // 2: n // 2 + 300] = xy[:300]                     # the same points early, in the middle and last
    xy[-300:] = xy[:300]
    xy = np.concatenate([xy, rng.uniform(-8, 8, (50_000, 2))])   # and some off the window
    t = np.concatenate([t, rng.random(50_000)])
    out.append(("many_per_cell", records(xy, t), w2, 0.5, random_grid(rng, w2)))
    # a global-costmap-sized window with a cloud spread over it
    w3 = (-100.0, -100.0, 0.2, 1000, 1000)
    xy = rng.uniform(-110, 110, (300_000, 2))
    out.append(("global_window", records(xy, rng.random(300_000)), w3, 0.7, random_grid(rng, w3)))
    return out


def map_cases():
    """synthetic show() traver layers for the map source: (name, traver (L, L) [ix, iy], L, grid_res, centre, start,
    window, thresh, mark_unknown, initial grid)"""
    rng = np.random.default_rng(43)
    out = []
    for L, gres, start in [(64, 0.05, (17, 40)), (96, 0.05, (0, 0)), (50, 0.1, (49, 1))]:
        tr = rng.choice(np.array([0.1, 0.5, 0.9, F32_07, np.nan, -0.3], np.float32), (L, L))
        centre = np.array([0.37, -1.21], np.float32)
        half = L * gres / 2
        for k, w in enumerate([(float(centre[0]) - half, float(centre[1]) - half, 0.2, int(L * gres / 0.2) + 1,
                                int(L * gres / 0.2) + 1),
                               (float(centre[0]) - 0.55, float(centre[1]) - 0.73, 0.2, 5, 7),
                               (-0.1, -1.4, 0.05, L, L)]):
            for mu in (True, False):
                for th in (0.7, F32_07):
                    out.append((f"map_L{L}_w{k}_{'unknown' if mu else 'known'}_{th!r}", tr, L, gres, centre, np.array(start, np.int32),
                                w, th, mu, random_grid(rng, w)))
    return out


def roll_cases():
    """(name, window, [(new_origin_x, new_origin_y), ...], fill, initial grid)"""
    rng = np.random.default_rng(47)
    w = (-3.0, 1.0, 0.2, 30, 20)
    g = random_grid(rng, w)
    out = [("positive", w, [(-3.0 + 0.2 * 3.3, 1.0 + 0.2 * 2.0)], FREE, g),
           ("negative", w, [(-3.0 - 0.2 * 2.7, 1.0 - 0.2 * 5.5)], UNKNOWN, g),
           ("fractional_half_cell", w, [(-3.0 - 0.1, 1.0 + 0.1)], FREE, g),
           ("larger_than_window", w, [(-3.0 + 0.2 * 45, 1.0), (-3.0 - 0.2 * 100, 1.0 - 0.2 * 21)], UNKNOWN, g),
           ("mixed", w, [(-3.0 + 0.2 * 10, 1.0 - 0.2 * 7.9), (-3.0, 1.0)], FREE, g)]
    # 200 consecutive rolls of the rolling-window rule (robot - getSizeInMetersX() / 2): the origin drifts on the grid
    lw = (0.0, 0.0, 0.2, 75, 75)
    mx = (75 - 1 + 0.5) * 0.2
    robot = np.cumsum(rng.uniform(-0.05, 0.45, (200, 2)), 0)
    out.append(("200_rolls", lw, [(float(x) - mx / 2, float(y) - mx / 2) for x, y in robot], FREE, random_grid(rng, lw)))
    return out


def combine_cases():
    """(name, mode, layer, master, size_x, size_y, rect)"""
    rng = np.random.default_rng(53)
    out = []
    for sx, sy in [(37, 23), (75, 75), (1000, 40)]:
        w = (0, 0, 1, sx, sy)
        lay, mas = random_grid(rng, w, 0.4), random_grid(rng, w, 0.2)
        for name, rect in [("full", (0, 0, sx, sy)), ("partial", (3, 5, sx - 7, sy - 2)), ("one_row", (1, 4, sx - 1, 5)),
                           ("empty_i", (9, 0, 9, sy)), ("empty_j", (0, 7, sx, 3)), ("clamped", (-5, -3, sx + 9, sy + 4)),
                           ("narrow", (13, 0, 14, sy))]:
            for mode in (0, 1):
                out.append((f"{name}_{sx}x{sy}_{'max' if mode == 0 else 'overwrite'}", mode, lay, mas, sx, sy, rect))
    return out
