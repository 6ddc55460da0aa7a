"""Crafted map states for the feature kernel and the ray clean-up (gem_b200/csrc/gem_kernels.cuh k_features,
k_lowest_bitmap / k_ray_collect / k_ray_trace).  CPU only, no GPU or torch imports.

Natural LiDAR scenes put valid cells wherever the scene puts them.  The cases here put them where the kernels make
decisions:

  feature families  the storage wrap line and the geographic edge cutting through tiles and halos (L from 1 to 257,
                    scrolled starts), exactly 7 and 8 valid cells in a window, tiles with no valid cell next to
                    valid halos, pivot ties and the signed initial maximum of the Jacobi step, a first pivot one ulp
                    either side of 0.01, equal diagonals and equal eigenvalues, the 31-rotation cap, extreme and
                    non-finite elevations, four resolutions;
  ray families      odd and even L with scrolled starts, obstacles everywhere / in rings / on the robot's row and
                    column, a valid `lowest` on every probed cell (DDA ties and threshold equalities), special
                    `lowest` values, the removal decision at equality and one ulp either side of it, the obstacle
                    test at its threshold, valid `lowest` cells in the last word of the validity bitmap.

A case is applied identically to gem_b200.ElevationMap and oracle_lib.OracleMap with `move` and `set_layer` only
(apply() for the feature inputs, apply_ray() before the ray clean-up).  Elevation, variance and traver are
storage-indexed, `lowest` is geographic-indexed, as in the reference.

trace_rays() is a vectorised float32 restatement of the DDA of G_Raytracing (gpu_process.cu:708-891).  The generator
uses it to place the removal decision exactly at restrict_ele; the CPU suite uses its counters to prove the ray
families reach the decisions they name.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np

f32 = np.float32
SENTINEL = f32(-10.0)
LOW_INVALID = f32(10.0)
SUCC = lambda x: np.nextafter(f32(x), f32(np.inf))
PRED = lambda x: np.nextafter(f32(x), f32(-np.inf))


@dataclass
class MapCase:
    name: str
    family: str                 # "feat_*" or "ray_*"
    L: int
    res: float
    start: tuple                # storage index of geographic cell (0, 0) after move()
    sensor_z: float
    elevation: np.ndarray       # (L, L) float32, storage-indexed
    variance: np.ndarray
    traver: np.ndarray          # the traver layer before Map_feature (empty cells keep it)
    lowest: np.ndarray          # (L, L) float32, geographic-indexed
    obstacle_threshold: float = 0.7
    ray_traver: np.ndarray | None = None  # traver layer set right before the ray clean-up (None: Map_feature's)

    def position(self):
        """a move() target that leaves the map with start index `start` and sensorZ `sensor_z`, from a new map"""
        # from centre 0 / start 0, move() shifts by k = round(pos / res) cells and sets start = (-k) mod L
        k = [-(s % self.L) for s in self.start]
        return np.array([f32(k[0] * f32(self.res)), f32(k[1] * f32(self.res)), f32(self.sensor_z)], f32)

    def apply(self, m):
        m.move(self.position())
        for name in ("elevation", "variance", "traver", "lowest"):
            m.set_layer(name, getattr(self, name))

    def apply_ray(self, m):
        if self.ray_traver is not None:
            m.set_layer("traver", self.ray_traver)

    @property
    def tileable(self):
        """usable on tiled handles: tiled maps do not scroll"""
        return self.start[0] % self.L == 0 and self.start[1] % self.L == 0


def to_storage(geo, start):
    """geographic (L, L) layer -> storage layer: storage cell (g + start) mod L holds geographic cell g"""
    return np.roll(geo, shift=(start[0], start[1]), axis=(0, 1))


def stale_traver(L):
    """a recognisable traver layer: Map_feature must leave it in every empty cell (gpu.cu:581)"""
    return (f32(-1000.0) - np.arange(L * L, dtype=np.float64).reshape(L, L) % 4093).astype(f32)


def _case(name, family, L, res, start, elev_geo, var_geo=None, traver_geo=None, lowest=None, sensor_z=1.0, thr=0.7,
          ray_traver_geo=None):
    start = (start[0] % L, start[1] % L)
    var_geo = np.full((L, L), f32(0.01)) if var_geo is None else var_geo
    traver_geo = stale_traver(L) if traver_geo is None else traver_geo
    lowest = np.full((L, L), LOW_INVALID) if lowest is None else lowest
    st = lambda a: np.ascontiguousarray(to_storage(np.asarray(a, f32), start))
    return MapCase(name, family, L, float(res), start, float(sensor_z), st(elev_geo), st(var_geo), st(traver_geo),
                   np.ascontiguousarray(lowest, f32), float(thr), None if ray_traver_geo is None else st(ray_traver_geo))


def _dense(rng, L, res, empty=0.15, noise=0.05):
    """a tilted, rough surface with random holes (geographic)"""
    gx, gy = np.meshgrid(np.arange(L), np.arange(L), indexing="ij")
    z = 0.2 * gx * res - 0.35 * gy * res + rng.normal(0.0, noise, (L, L)) + 0.3 * np.sin(gx * res * 3.0)
    z = z.astype(f32)
    z[rng.random((L, L)) < empty] = SENTINEL
    return z


def _var(rng, L):
    return rng.uniform(1e-4, 2e-2, (L, L)).astype(f32)


def _lowest(rng, L, density, lo=-1.0, hi=0.6):
    low = rng.uniform(lo, hi, (L, L)).astype(f32)
    low[rng.random((L, L)) >= density] = LOW_INVALID
    return low


# ---------------------------------------------------------------------------------------------------------------------
# feature families
# ---------------------------------------------------------------------------------------------------------------------
GEOMETRY_L = (1, 2, 3, 4, 5, 15, 16, 17, 31, 33, 200, 257)
RESOLUTIONS = (0.05, 0.1, 0.3, 1.0)


def geometry_starts(L):
    out = []
    for s in ((0, 0), (1, L - 1), (L - 2, 3), (L // 2, L // 2)):
        s = (s[0] % L, s[1] % L)
        if s not in out:
            out.append(s)
    return out


def feature_geometry():
    out = []
    for L in GEOMETRY_L:
        for k, s in enumerate(geometry_starts(L)):
            rng = np.random.default_rng(1000 * L + k)
            e = _dense(rng, L, 0.1)
            out.append(_case(f"feat_geom_L{L}_s{s[0]}_{s[1]}", "feat_geom", L, 0.1, s, e, _var(rng, L),
                             lowest=_lowest(rng, L, 0.2)))
    return out


def _window(L, gx, gy):
    return [(gx + i, gy + j) for i in range(-2, 3) for j in range(-2, 3)
            if (i or j) and 0 <= gx + i < L and 0 <= gy + j < L]


def feature_count():
    """exactly 7 and exactly 8 valid cells (centre included) in the window of target cells; `cnt > 7` decides"""
    out = []
    L = 32
    placements = {
        "interior": ((0, 0), [(10, 10), (20, 22)]),
        "edge": ((0, 0), [(0, 12), (31, 20), (14, 0), (22, 31)]),
        "corner": ((0, 0), [(0, 0), (31, 31), (0, 31), (31, 0)]),
        "wrap": ((3, 30), [(28, 3), (20, 1), (28, 18), (10, 2)]),  # storage windows straddle row 31|0 and column 31|0
    }
    for q, (pname, (start, targets)) in enumerate(placements.items()):
        for cnt in (7, 8):
            rng = np.random.default_rng(10 * q + cnt)
            e = np.full((L, L), SENTINEL)
            for gx, gy in targets:
                e[gx, gy] = f32(rng.uniform(-0.2, 0.2))
                nb = _window(L, gx, gy)
                for p in rng.permutation(len(nb))[:cnt - 1]:
                    e[nb[p]] = f32(rng.uniform(-0.2, 0.2))
            c = _case(f"feat_count{cnt}_{pname}", "feat_count", L, 0.1, start, e, lowest=_lowest(rng, L, 0.3))
            c.targets = [(gx, gy, cnt) for gx, gy in targets]
            out.append(c)
    return out


def feature_empty_tiles():
    """tiles (in storage coordinates) without a valid cell but with valid halos, and a tile whose only valid cell is
    its corner; the stale traver layer must survive in the empty cells of both kinds of tile"""
    out = []
    for L, start in ((64, (0, 0)), (40, (7, 35))):
        rng = np.random.default_rng(L)
        s = np.full((L, L), SENTINEL)                 # storage coordinates
        if L == 64:
            s[14:34, 14:34] = f32(0.1)                # the 2-cell halo ring of tile (1, 1) ...
            s[16:32, 16:32] = SENTINEL                # ... around an empty tile
        s += np.where(s != SENTINEL, rng.normal(0, 0.02, (L, L)), 0).astype(f32)
        if L == 64:
            # tile (0, 3) = rows 0-15, cols 48-63: its only valid cell is the corner (15, 48); its window's cells in
            # the tiles (0, 2), (1, 2), (1, 3) are valid
            for i in range(13, 18):
                for j in range(46, 51):
                    if i >= 16 or j < 48 or (i, j) == (15, 48):
                        s[i, j] = f32(0.05 * rng.random())
        else:
            # L = 40: partial tiles; the corner cell (32, 0) of tile (2, 0) with its window wrapping to column 38-39
            for i in range(30, 35):
                for j in range(-2, 3):
                    if i < 32 or j < 0 or (i, j) == (32, 0):
                        s[i, j % L] = f32(0.05 * rng.random())
        geo = np.roll(s, shift=(-start[0], -start[1]), axis=(0, 1))
        out.append(_case(f"feat_empty_tile_L{L}", "feat_empty", L, 0.1, start, geo, lowest=_lowest(rng, L, 0.3)))
    return out


def _put_block(e, gx, gy, block):
    """place a 5 x 5 block (-10 = empty) centred on geographic cell (gx, gy)"""
    e[gx - 2:gx + 3, gy - 2:gy + 3] = block


def _mask_sums(mask):
    """exact (Sxx, Syy, Sxy) in units of res^2 of a 5 x 5 validity mask, or None when a mean is not dyadic"""
    ii, jj = np.nonzero(mask)
    n = ii.size
    if n & (n - 1):
        return None
    dx, dy = ii - ii.mean(), jj - jj.mean()
    return float((dx * dx).sum()), float((dy * dy).sum()), float((dx * dy).sum())


@functools.lru_cache(maxsize=None)
def _tie_masks():
    """5 x 5 masks (centre valid, 8 or 16 cells) with Sxy / Sxx = +-1/2 or +-1/4: with z = a * x, a = Sxy / Sxx, the
    scatter matrix has o02 == o01 exactly and |o12| < |o01|"""
    rng = np.random.default_rng(7)
    found = {}
    for _ in range(20000):
        n = 8 if rng.random() < 0.5 else 16
        m = np.zeros(25, bool)
        m[12] = True
        m[rng.choice([q for q in range(25) if q != 12], n - 1, replace=False)] = True
        m = m.reshape(5, 5)
        sums = _mask_sums(m)
        if sums is None or sums[2] == 0:
            continue
        ratio = sums[2] / sums[0]
        if ratio in (0.5, -0.5, 0.25, -0.25) and ratio not in found:
            found[ratio] = m
        if len(found) == 4:
            break
    return tuple(sorted(found.items()))


def feature_pivot():
    out = []
    # exact arithmetic: power-of-two resolution, integer cells, 8/16/25-cell windows, dyadic elevations
    res = 0.5
    L = 64
    blocks = []                                     # (block, tag)
    for ratio, m in _tie_masks():
        for sign, z0 in ((1.0, 0.25), (-1.0, 0.25), (1.0, -3.0)):   # o02 = +-o01: a tie in magnitude either sign
            xs = (np.arange(5)[:, None] * np.ones((1, 5))) * res
            blocks.append((np.where(m, (ratio * sign) * xs + z0, SENTINEL).astype(f32), "tie01_02"))
    full = np.ones((5, 5), bool)
    xs, ys = np.meshgrid(np.arange(5) * res, np.arange(5) * res, indexing="ij")
    for a in (0.5, -0.25, 0.125):                   # full window, Sxy == 0, z = a (x + y): o02 == o12, o01 == 0
        blocks.append((np.where(full, a * (xs + ys) + 1.0, SENTINEL).astype(f32), "tie02_12"))
        blocks.append((np.where(full, a * (xs - ys) + 1.0, SENTINEL).astype(f32), "tie02_12"))
    anti = np.fliplr(np.eye(5, dtype=bool)) | np.fliplr(np.eye(5, k=1, dtype=bool)) | np.fliplr(np.eye(5, k=-1, dtype=bool))
    anti[0, 4] = anti[4, 0] = False
    anti[1, 1] = anti[3, 3] = True                  # 13 cells, Sxy < 0, flat: o01 negative and the largest
    for zc in (0.0, 0.3):
        blocks.append((np.where(anti, f32(zc), SENTINEL).astype(f32), "neg01"))
    diag = np.zeros((5, 5), bool)                   # 8 cells, symmetric under transpose: d0 == d1 exactly, o01 the pivot
    for q in ((0, 0), (1, 1), (2, 2), (3, 3), (1, 2), (2, 1), (2, 3), (3, 2)):
        diag[q] = True
    for zc in (0.0, 0.75):
        blocks.append((np.where(diag, f32(zc), SENTINEL).astype(f32), "eqdiag"))
    # equal eigenvalues at the final selection: no rotation (every off-diagonal < 0.01), d0 == d2 < d1 or
    # d1 == d2 < d0; res 1/32 keeps the sums small
    eig_blocks = []
    zpat = np.array([[1, -1, 1, -1], [-1, 1, -1, 1]], np.float64)
    b = np.full((5, 5), SENTINEL)
    b[2:4, 0:4] = (0.5 * zpat * (1 / 32)).astype(f32)            # 8 cells, units res^2: Sxx = 2 = Szz < Syy = 10
    eig_blocks.append((b, "eqeig02"))
    b = np.full((5, 5), SENTINEL)
    b[0:4, 2:4] = (0.5 * zpat.T * (1 / 32)).astype(f32)          # Syy = 2 = Szz < Sxx = 10
    eig_blocks.append((b, "eqeig12"))

    def layout(blocks, L, res, start, name):
        e = np.full((L, L), SENTINEL)
        targets = []
        per_row = (L - 2) // 7
        for q, (blk, tag) in enumerate(blocks):
            gx, gy = 3 + 7 * (q // per_row), 3 + 7 * (q % per_row)
            _put_block(e, gx, gy, blk)
            targets.append((gx, gy, tag))
        c = _case(name, "feat_pivot", L, res, start, e, lowest=_lowest(np.random.default_rng(L), L, 0.3))
        c.targets = targets
        return c

    for start in ((0, 0), (5, 9)):                  # scrolled, but no window crosses the wrap line (exact sums)
        out.append(layout(blocks, L, res, start, f"feat_pivot_ties_s{start[0]}_{start[1]}"))
    out.append(layout(eig_blocks * 3, 32, 1 / 32, (0, 0), "feat_pivot_eqeig"))
    out.append(layout(eig_blocks, 32, 1 / 32, (17, 9), "feat_pivot_eqeig_scrolled"))
    out.append(_first_pivot_sweep())
    # the 31-rotation cap: squares that overflow leave inf / NaN entries the stopping rule never accepts
    rng = np.random.default_rng(31)
    e = rng.uniform(-3e19, 3e19, (40, 40)).astype(f32)
    e[rng.random((40, 40)) < 0.1] = SENTINEL
    out.append(_case("feat_pivot_cap31", "feat_pivot", 40, 0.1, (3, 7), e, lowest=_lowest(rng, 40, 0.3)))
    return out


def _plane_o02(slopes, cx, cy, res):
    """float32 |o02| of the full window centred on storage cell (cx, cy) (start 0) of the plane z = s x, for every
    s in `slopes`; also returns the blocks.  Summation order of gpu.cu:610-633."""
    px = (np.arange(cx - 2, cx + 3)[:, None] * np.ones((1, 5), np.int64)).astype(f32) * f32(res)
    blocks = (slopes[:, None, None] * px[None]).astype(f32)
    sx, sz = f32(0), np.zeros(slopes.size, f32)
    for v in range(25):
        sx = f32(sx + px.flat[v])
        sz = sz + blocks[:, v // 5, v % 5]
    mx, mz = f32(sx / f32(25)), sz / f32(25)
    o02 = np.zeros(slopes.size, f32)
    for v in range(25):
        o02 = o02 + (px.flat[v] - mx) * (blocks[:, v // 5, v % 5] - mz)
    return np.abs(o02), blocks


def _first_pivot_sweep():
    """a plane z = s x over full windows, s swept ulp by ulp so that the first pivot |o02| lands one ulp below,
    on and one ulp above 0.01 (the stopping rule `big < 0.01f`); o01 and o12 stay near 0"""
    L, res = 64, 0.1
    eps = f32(0.01)
    wanted = [PRED(eps), eps, SUCC(eps)] * 4
    e = np.full((L, L), SENTINEL)
    targets = []
    s0 = f32(0.01 / (50 * res * res)).view(np.int32)    # o02 ~ s Sxx, Sxx = 50 res^2
    slopes = (s0 + np.arange(-3000, 3001)).astype(np.int32).view(f32)
    per_row = (L - 2) // 7
    for k in range(per_row * per_row):
        if not wanted:
            break
        cx, cy = 3 + 7 * (k // per_row), 3 + 7 * (k % per_row)
        o, blocks = _plane_o02(slopes, cx, cy, res)
        for w in list(wanted):
            hit = np.nonzero(o == w)[0]
            if hit.size:
                _put_block(e, cx, cy, blocks[hit[0]])
                targets.append((cx, cy, "pivot_" + ("below" if w < eps else "on" if w == eps else "above")))
                wanted.remove(w)
                break
    c = _case("feat_pivot_first_eps", "feat_pivot", L, res, (0, 0), e, lowest=_lowest(np.random.default_rng(5), L, 0.3))
    c.targets = targets
    return c


def feature_magnitudes():
    out = []
    L = 40
    for res in RESOLUTIONS:
        rng = np.random.default_rng(int(res * 1000))
        out.append(_case(f"feat_res{res}", "feat_mag", L, res, (11, 29), _dense(rng, L, res, noise=0.1), _var(rng, L),
                         lowest=_lowest(rng, L, 0.3)))
    rng = np.random.default_rng(99)
    e = rng.choice(np.array([SENTINEL, PRED(SENTINEL), SUCC(SENTINEL)], f32), (L, L), p=[0.4, 0.3, 0.3])
    out.append(_case("feat_mag_sentinel_ulp", "feat_mag", L, 0.1, (5, 5), e))
    for name, lo, hi in (("feat_mag_1e18", 1e18, 4e19), ("feat_mag_neg1e18", -4e19, -1e18)):
        e = rng.uniform(lo, hi, (L, L)).astype(f32)
        e[rng.random((L, L)) < 0.15] = SENTINEL
        out.append(_case(name, "feat_mag", L, 0.1, (0, 0), e))
    e = (rng.uniform(-1.0, 1.0, (L, L)) * 1e-20).astype(f32)          # dz^2 subnormal
    out.append(_case("feat_mag_tiny_diff", "feat_mag", L, 0.1, (2, 37), e))
    e = (rng.integers(-40, 40, (L, L)) * f32(1.4e-45)).astype(f32)     # subnormal elevations
    out.append(_case("feat_mag_subnormal", "feat_mag", L, 1.0, (0, 0), e))
    e = (f32(1.0) + rng.integers(-8, 8, (L, L)).astype(f32) * f32(2.0 ** -23)).astype(f32)  # a few ulps around 1
    out.append(_case("feat_mag_ulp_diff", "feat_mag", L, 0.05, (0, 0), e))
    for where in ("centre", "neighbour"):
        e = _dense(np.random.default_rng(3), L, 0.1, empty=0.05)
        spots = [(8, 8), (8, 20), (20, 8), (30, 30)]
        for q, (gx, gy) in enumerate(spots):
            v = (f32(np.inf), f32(-np.inf), f32(np.nan), f32(np.inf))[q]
            if where == "centre":
                e[gx, gy] = v
            else:
                e[gx + 1, gy - 2] = v
        out.append(_case(f"feat_mag_nonfinite_{where}", "feat_mag", L, 0.1, (13, 2), e))
    return out


def feature_cases():
    return feature_geometry() + feature_count() + feature_empty_tiles() + feature_pivot() + feature_magnitudes()


# ---------------------------------------------------------------------------------------------------------------------
# the DDA of G_Raytracing, vectorised over rays
# ---------------------------------------------------------------------------------------------------------------------
def robot_index(L):
    """gpu.cu:731-742"""
    return int(f32(L // 2 - 0.5)) if L % 2 == 0 else L // 2


def trace_rays(elev, var, traver, lowest, L, start, sensor_z, thr):
    """the ray clean-up of one map (storage-indexed elev / var / traver, geographic lowest).  Returns a dict:
    cells (storage index of every casting cell), restrict (its restrict_ele), removed (bool), new_elevation (L*L),
    and counters: tie_steps_nondiag (rays that step both ways at least once while |inc0| != |inc1|),
    threshold_eq (probes of a valid lowest exactly at `mcur - later == threshold` whose max_ele is below the ray's
    final restrict_ele), value (obstacle_ele - 3 sqrt(var) per casting cell)."""
    elev = np.asarray(elev, f32).reshape(-1)
    var = np.asarray(var, f32).reshape(-1)
    traver = np.asarray(traver, f32).reshape(-1)
    lowest = np.asarray(lowest, f32).reshape(-1)
    robot = robot_index(L)
    idx = np.arange(L * L)
    ox = (idx // L + L - start[0]) % L
    oy = (idx % L + L - start[1]) % L
    cast = (traver < f32(thr)) & (elev != SENTINEL) & (ox != robot) & (oy != robot)
    cells = np.nonzero(cast)[0]
    ox, oy = ox[cells], oy[cells]
    obst = elev[cells]
    with np.errstate(all="ignore"):
        inc0, inc1 = (ox - robot).astype(f32), (oy - robot).astype(f32)
        ix = np.where(inc0 > 0, 1, -1)
        iy = np.where(inc1 > 0, 1, -1)
        dis = np.sqrt(inc0 * inc0 + inc1 * inc1)
        d0, d1 = inc0 / dis, inc1 / dis
        a0, a1 = inc0.astype(np.float64), inc1.astype(np.float64)
        t = np.where(np.abs(inc0) > np.abs(inc1), 0.5 / a0 * a1, 0.5 / a1 * a0)
        threshold = np.sqrt(0.5 * 0.5 + t * t).astype(f32)
        bx, by = ix.astype(f32) / f32(2), iy.astype(f32) / f32(2)
        dnx, dny = bx / d0, by / d1
        later = np.zeros(cells.size, f32)
        restrict = obst.copy()
        cx, cy = ox.copy(), oy.copy()
        tie_nd = np.zeros(cells.size, bool)
        eq_min = np.full(cells.size, f32(np.inf))
        nondiag = np.abs(inc0) != np.abs(inc1)
        act = np.ones(cells.size, bool)
        sz = f32(sensor_z)
        fr = f32(robot)
        while True:
            act &= (cx >= 0) & (cx < L) & (cy >= 0) & (cy < L)
            if not act.any():
                break
            a = np.nonzero(act)[0]
            gx, gy, dx_, dy_ = cx[a], cy[a], dnx[a], dny[a]
            gt, lt = dx_ > dy_, dx_ < dy_
            mcur = np.where(gt, dy_, dx_)
            gap = mcur - later[a]
            probe = (gap > threshold[a]) & (gx != ox[a]) & (gy != oy[a])
            eqp = (gap == threshold[a]) & (gx != ox[a]) & (gy != oy[a])
            low = lowest[gx * L + gy]
            valid = low != LOW_INVALID
            x1 = (gx - ox[a]).astype(f32)
            x2 = gx.astype(f32) - fr
            h2 = sz - low
            me = low + h2 / x2 * x1
            upd = probe & valid & (me < restrict[a])
            restrict[a] = np.where(upd, me, restrict[a])
            e = eqp & valid
            eq_min[a] = np.where(e & (me < eq_min[a]), me, eq_min[a])
            tie_nd[a] |= (~gt) & (~lt) & nondiag[a]
            later[a] = mcur
            sx_, sy_ = ~gt, ~lt
            cx[a] = gx + np.where(sx_, ix[a], 0)
            cy[a] = gy + np.where(sy_, iy[a], 0)
            nbx = np.where(sx_, bx[a] + ix[a].astype(f32), bx[a])
            nby = np.where(sy_, by[a] + iy[a].astype(f32), by[a])
            dnx[a] = np.where(sx_, nbx / d0[a], dx_)
            dny[a] = np.where(sy_, nby / d1[a], dy_)
            bx[a], by[a] = nbx, nby
        value = obst - f32(3) * np.sqrt(var[cells])
        removed = value > restrict
    out = elev.copy()
    out[cells[removed]] = SENTINEL
    return {"cells": cells, "restrict": restrict, "value": value, "removed": removed, "new_elevation": out,
            "tie_steps_nondiag": int(tie_nd.sum()), "threshold_eq": int((eq_min < restrict).sum())}


def solve_variance(obst, target):
    """per cell a float32 variance v >= 0 with obst - 3 sqrt(v) == target exactly (float32), or NaN if none is
    found within 300 ulps of the real-valued solution"""
    obst = np.asarray(obst, f32)
    target = np.asarray(target, f32)
    with np.errstate(all="ignore"):
        d = obst.astype(np.float64) - target.astype(np.float64)
        v0 = np.where(d >= 0, (d / 3.0) ** 2, np.nan).astype(f32)
        base = v0.view(np.int32).astype(np.int64)
        off = np.concatenate([[0], np.arange(1, 301), -np.arange(1, 301)])
        cand = np.clip(base[:, None] + off[None, :], 0, 0x7f7fffff).astype(np.int32).view(f32)
        val = obst[:, None] - f32(3) * np.sqrt(cand)
        ok = (val == target[:, None]) & np.isfinite(v0)[:, None]
    first = np.argmax(ok, axis=1)
    got = ok[np.arange(ok.shape[0]), first]
    return np.where(got, cand[np.arange(ok.shape[0]), first], f32(np.nan)).astype(f32)


# ---------------------------------------------------------------------------------------------------------------------
# ray families
# ---------------------------------------------------------------------------------------------------------------------
VAR_TARGETS = ("eq", "above", "below", "zero", "negative")


def _ray_case(name, family, L, start, elev_geo, traver_geo, lowest, sensor_z=1.0, thr=0.7, var_mode="mix", rng=None,
              targets=VAR_TARGETS[:3]):
    """a ray case whose obstacle variances put `obstacle_ele - 3 sqrt(var)` exactly at restrict_ele (eq), one ulp
    above (above: removed) or one ulp below (below: kept), cycling over the casting cells, so that a restrict_ele
    that is off by one ulp in either direction changes the map.  var_mode "random": plain random variances."""
    rng = np.random.default_rng(L) if rng is None else rng
    var_geo = _var(rng, L)
    c = _case(name, family, L, 0.1, start, elev_geo, var_geo, stale_traver(L), lowest, sensor_z, thr, traver_geo)
    if var_mode == "random":
        return c
    r = trace_rays(c.elevation, c.variance, c.ray_traver, c.lowest, L, c.start, sensor_z, thr)
    cells, restrict, obst = r["cells"], r["restrict"], c.elevation.reshape(-1)[r["cells"]]
    kind = np.arange(cells.size) % len(targets)
    want = np.select([kind == k for k in range(len(targets))],
                     [{"eq": restrict, "above": SUCC(restrict), "below": PRED(restrict),
                       "zero": restrict, "negative": restrict}[t] for t in targets])
    v = solve_variance(obst, want.astype(f32))
    for k, t in enumerate(targets):
        if t == "zero":
            v[kind == k] = f32(0.0)
        elif t == "negative":
            v[kind == k] = f32(-1e-3)
    var = c.variance.reshape(-1).copy()
    ok = ~np.isnan(v)
    var[cells[ok]] = v[ok]
    c.variance = var.reshape(L, L)
    return c


def _obstacle_layout(L, kind):
    robot = robot_index(L)
    gx, gy = np.meshgrid(np.arange(L), np.arange(L), indexing="ij")
    t = np.full((L, L), f32(0.9))
    if kind == "all":
        t[:] = f32(0.0)
    elif kind == "rings":
        cheb = np.maximum(np.abs(gx - robot), np.abs(gy - robot))
        t[(cheb % 4 == 1) | (cheb == L // 2 - 1)] = f32(0.0)
    t[robot, :] = f32(0.0)                           # the robot's row and column cast no ray
    t[:, robot] = f32(0.0)
    return t


RAY_GEOMETRY_L = (2, 3, 17, 32, 33, 64, 257)


def ray_geometry():
    out = []
    for L in RAY_GEOMETRY_L:
        for start in ((0, 0), (L // 3, L - 1)):
            for kind in (("all", "rings") if L <= 64 else ("rings",)):
                rng = np.random.default_rng(L * 7 + start[0] + len(kind))
                e = rng.uniform(0.0, 1.5, (L, L)).astype(f32)
                out.append(_ray_case(f"ray_geom_L{L}_s{start[0] % L}_{start[1] % L}_{kind}", "ray_geom", L, start, e,
                                     _obstacle_layout(L, kind), _lowest(rng, L, 0.3), rng=rng))
    return out


def ray_ties():
    """a valid lowest on every cell: every probe counts, so a wrong DDA step or a wrong `>` changes restrict_ele"""
    out = []
    for L, start in ((16, (0, 0)), (17, (5, 11)), (24, (0, 0)), (31, (30, 2))):
        rng = np.random.default_rng(100 + L)
        e = rng.uniform(0.2, 1.5, (L, L)).astype(f32)
        out.append(_ray_case(f"ray_ties_L{L}", "ray_ties", L, start, e, _obstacle_layout(L, "all"),
                             _lowest(rng, L, 1.0, -0.5, 0.4), sensor_z=0.9, rng=rng))
    return out


def ray_lowest_values():
    out = []
    L = 32
    special = np.array([10.0, SUCC(10.0), PRED(10.0), np.nan, np.inf, -np.inf, 100.0, 11.0], f32)
    rng = np.random.default_rng(71)
    e = rng.uniform(0.0, 1.5, (L, L)).astype(f32)
    low = _lowest(rng, L, 0.6)
    pick = rng.random((L, L)) < 0.5
    low[pick] = rng.choice(special, int(pick.sum()))
    out.append(_ray_case("ray_low_special", "ray_low", L, (9, 4), e, _obstacle_layout(L, "all"), low, rng=rng))
    low = np.where(rng.random((L, L)) < 0.7, f32(0.5), LOW_INVALID).astype(f32)
    out.append(_ray_case("ray_low_eq_sensor", "ray_low", L, (0, 0), e, _obstacle_layout(L, "all"), low, sensor_z=0.5,
                         rng=rng))
    low = _lowest(rng, L, 0.7, 0.0, 1.0)
    out.append(_ray_case("ray_low_above_sensor", "ray_low", L, (3, 3), e, _obstacle_layout(L, "all"), low,
                         sensor_z=-1.0, rng=rng))
    # a lowest above 10 only lowers restrict_ele when the sensor is higher still: valid values just above the
    # sentinel (nextafter(10), 11, 15) under a sensor at 20 m
    low = rng.choice(np.array([SUCC(10.0), 11.0, 15.0, 10.0, PRED(10.0), 100.0], f32), (L, L))
    out.append(_ray_case("ray_low_above_10", "ray_low", L, (20, 6), rng.uniform(5.0, 15.0, (L, L)).astype(f32),
                         _obstacle_layout(L, "all"), low, sensor_z=20.0, rng=rng))
    return out


def ray_removal():
    out = []
    for L, start in ((24, (3, 20)), (25, (0, 0))):
        rng = np.random.default_rng(200 + L)
        e = rng.uniform(0.0, 1.5, (L, L)).astype(f32)
        out.append(_ray_case(f"ray_removal_L{L}", "ray_removal", L, start, e, _obstacle_layout(L, "all"),
                             _lowest(rng, L, 0.5), rng=rng, targets=VAR_TARGETS))
    return out


def ray_obstacle_test():
    L, thr = 20, 0.7
    rng = np.random.default_rng(300)
    e = rng.uniform(0.0, 1.5, (L, L)).astype(f32)
    t = rng.choice(np.array([thr, np.nan, -10.0, PRED(thr), SUCC(thr), 0.0], f32), (L, L))
    return [_ray_case("ray_obstacle_test", "ray_obstacle", L, (4, 13), e, t, _lowest(rng, L, 0.8), thr=thr, rng=rng)]


def ray_bitmap_tail():
    out = []
    for L in (17, 23, 33):
        rng = np.random.default_rng(400 + L)
        e = rng.uniform(0.0, 1.5, (L, L)).astype(f32)
        low = np.full(L * L, LOW_INVALID)
        tail = 32 * ((L * L - 1) // 32)             # first cell of the last bitmap word
        low[tail:] = rng.uniform(-1.0, 0.4, L * L - tail).astype(f32)
        low[rng.choice(tail, 5, replace=False)] = f32(-0.3)
        out.append(_ray_case(f"ray_bitmap_tail_L{L}", "ray_tail", L, (0, 0), e, _obstacle_layout(L, "all"),
                             low.reshape(L, L), rng=rng))
    return out


def ray_cases():
    return ray_geometry() + ray_ties() + ray_lowest_values() + ray_removal() + ray_obstacle_test() + ray_bitmap_tail()


def tiled_cases():
    """start-0 maps whose tiles (world 2: L x L/2, world 4: L/2 x L/2) are not multiples of the 16-cell feature tile"""
    out = []
    for L in (66, 34):
        rng = np.random.default_rng(500 + L)
        e = _dense(rng, L, 0.1)
        out.append(_case(f"feat_tiled_L{L}", "feat_geom", L, 0.1, (0, 0), e, _var(rng, L), lowest=_lowest(rng, L, 0.3)))
        e = rng.uniform(0.0, 1.5, (L, L)).astype(f32)
        out.append(_ray_case(f"ray_tiled_L{L}", "ray_geom", L, (0, 0), e, _obstacle_layout(L, "all"),
                             _lowest(rng, L, 0.6), rng=rng))
    return out


@functools.lru_cache(maxsize=None)
def all_cases():
    return tuple(feature_cases() + ray_cases() + tiled_cases())


def case(name):
    return next(c for c in all_cases() if c.name == name)


def long_ray_case():
    """L = 1024: a ring of obstacles about 500 cells from the robot and a valid lowest on every cell: long rays and a
    multi-word bitmap"""
    L = 1024
    rng = np.random.default_rng(1024)
    robot = robot_index(L)
    gx, gy = np.meshgrid(np.arange(L), np.arange(L), indexing="ij")
    rr = np.hypot(gx - robot, gy - robot)
    ring = (rr >= 498) & (rr < 502)
    e = np.where(ring, rng.uniform(0.5, 2.0, (L, L)), SENTINEL).astype(f32)
    t = np.where(ring, f32(0.0), f32(0.9)).astype(f32)
    return _ray_case("ray_long_L1024", "ray_long", L, (300, 700), e, t, _lowest(rng, L, 1.0, -1.0, 0.5), rng=rng)
