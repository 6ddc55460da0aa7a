"""Crafted submap pairs for the loop-closure re-fusion (gem_refuse_submaps / orc_refuse_submaps, DESIGN.md f4) and an
independent restatement of f4 items 2-5.  TEST INFRASTRUCTURE ONLY.

The restatement keys a Python dict by the float32 cell centre (rx, ry) in first-insertion order, which is the point
unordered_map::insert keeps, fuses every cell present in both maps once, in new-map order, and evaluates the fused
values in float64 as C parses the expressions.  The oracle (oracle/gem_oracle.c) instead sorts the cells with qsort and
finds them by binary search; the device probes open-addressing tables.  A case is (name, new (n, 8) float32,
old (m, 8) float32, resolution); a record is PointXYZRGBICT: x, y, z, w, bgra bits, covariance, intensity, travers."""
from __future__ import annotations

import zlib

import numpy as np

F = np.float32
FIELDS = ("x", "y", "z", "w", "bgra", "covariance", "intensity", "travers")


# ---- f4 arithmetic in numpy ------------------------------------------------------------------------------------------
def cell_centre(v, res):
    """pointCloudtoHash (ElevationMapping.cpp:1183-1184): float(ceil(v / res) * res - res / 2) evaluated in double"""
    with np.errstate(invalid="ignore", over="ignore"):
        v = np.asarray(v, np.float32).astype(np.float64)
        return (np.ceil(v / res) * res - res / 2.0).astype(np.float32)


def table_mask(n):
    """gem_refuse_submaps sizes each table to the power of two >= 2 n + 2, at least 64"""
    p = 64
    while p < 2 * n + 2:
        p <<= 1
    return p - 1


def hash_slot(rx, ry, mask):
    """the home slot of a cell: hash_slot (gem_submap.cuh) of the bits of (rx, ry), -0 folded into +0"""
    rx = np.atleast_1d(np.asarray(rx, np.float32))
    ry = np.atleast_1d(np.asarray(ry, np.float32))
    rx = np.where(rx == 0, F(0), rx).astype(np.float32)
    ry = np.where(ry == 0, F(0), ry).astype(np.float32)
    k = (rx.view(np.uint32).astype(np.uint64) << np.uint64(32)) | ry.view(np.uint32).astype(np.uint64)
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xff51afd7ed558ccd)
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xc4ceb9fe1a85ec53)
        k ^= k >> np.uint64(33)
    return (k & np.uint64(mask)).astype(np.int64)


# ---- the restatement -------------------------------------------------------------------------------------------------
def _cells(rx, ry):
    """{(rx, ry): index of the first point} in first-insertion order, and the keep flags (first of a cell, or a NaN
    position, which equals nothing)"""
    first, keep = {}, []
    for i, key in enumerate(zip(rx.tolist(), ry.tolist())):
        if key[0] != key[0] or key[1] != key[1]:
            keep.append(True)
        else:
            keep.append(first.setdefault(key, i) == i)
    return first, np.array(keep, bool)


def refuse(new, old, res, compat=True):
    """f4 items 2-5 for one pair: returns (new', old', fused count, fused rows of new', fused rows of old')"""
    new = np.array(new, np.float32, copy=True, order="C").reshape(-1, 8)
    old = np.array(old, np.float32, copy=True, order="C").reshape(-1, 8)
    rxn, ryn = cell_centre(new[:, 0], res), cell_centre(new[:, 1], res)
    rxo, ryo = cell_centre(old[:, 0], res), cell_centre(old[:, 1], res)
    cn, keep_n = _cells(rxn, ryn)
    co, keep_o = _cells(rxo, ryo)
    fused_n, fused_o = np.zeros(new.shape[0], bool), np.zeros(old.shape[0], bool)
    count = 0
    for key, i in cn.items():                    # every cell of the new map once, in the order of its first point
        j = co.get(key)
        if j is None:
            continue
        vo = float(old[j, 5])
        if not (vo > 0.0 and vo < 1.0):         # :857
            continue
        vn, en, eo = float(new[i, 5]), float(new[i, 2]), float(old[j, 2])
        vn2, vo2 = vn * vn, vo * vo              # pow(float, 2): exact in double
        if compat:                               # :862-863 as C parses them: a*b + (c*d)/e + f
            ef = (vn2 * eo + (vo2 * en) / vo2) + vn2
            vf = (vo2 * vn2) / vo2 + vn2
        else:
            ef = (vn2 * eo + vo2 * en) / (vo2 + vn2)
            vf = (vo2 * vn2) / (vo2 + vn2)
        with np.errstate(over="ignore", invalid="ignore"):
            new[i, 2], new[i, 5] = F(ef), F(vf)
        old.view(np.uint32)[j] = new.view(np.uint32)[i]    # the new map's record lands in both (:856)
        fused_n[i] = fused_o[j] = True
        count += 1
    for p, rx, ry in ((new, rxn, ryn), (old, rxo, ryo)):   # localHashtoPointCloud (:1129-1130): the cell's position
        p[:, 0], p[:, 1], p[:, 3] = rx, ry, F(1)
    return new[keep_n], old[keep_o], count, fused_n[keep_n], fused_o[keep_o]


def transform(pts, T):
    """pcl::transformPointCloud's scalar form (f4 item 1): x' = ((t00 x + t01 y) + t02 z) + t03, each step in float32"""
    p = np.array(pts, np.float32, copy=True).reshape(-1, 8)
    T = np.asarray(T, np.float32).reshape(4, 4)
    x, y, z = p[:, 0].copy(), p[:, 1].copy(), p[:, 2].copy()
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(3):
            p[:, r] = ((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3]
    return p


def transform_difference(got, want):
    """None, or (row, field) of the first difference of two transformed clouds (a NaN coordinate equals any NaN)"""
    same = np.asarray(got, np.float32).view(np.uint32) == np.asarray(want, np.float32).view(np.uint32)
    same[:, :3] |= np.isnan(got[:, :3]) & np.isnan(want[:, :3])
    bad = np.argwhere(~same)
    return None if bad.size == 0 else (int(bad[0, 0]), FIELDS[int(bad[0, 1])])


def first_difference(got, want, fused):
    """None, or (row, field, got bits, want bits) of the first difference.  Bits are compared, except that a NaN equals
    any NaN where the value is computed: the position of every row, elevation and variance of a fused row (NaN payloads
    differ between the x86 oracle and the GPU)"""
    got = np.ascontiguousarray(got, np.float32).reshape(-1, 8)
    want = np.ascontiguousarray(want, np.float32).reshape(-1, 8)
    if got.shape != want.shape:
        return ("shape", got.shape, want.shape)
    diff = got.view(np.uint32) != want.view(np.uint32)
    loose = np.zeros(diff.shape, bool)
    loose[:, :2] = True
    loose[np.asarray(fused, bool), 2] = True
    loose[np.asarray(fused, bool), 5] = True
    diff &= ~(loose & np.isnan(got) & np.isnan(want))
    rows = np.flatnonzero(diff.any(axis=1))
    if rows.size == 0:
        return None
    r = int(rows[0])
    f = int(np.flatnonzero(diff[r])[0])
    return (r, FIELDS[f], hex(int(got.view(np.uint32)[r, f])), hex(int(want.view(np.uint32)[r, f])))


# ---- building records ------------------------------------------------------------------------------------------------
def _rng(name):
    return np.random.default_rng(zlib.crc32(name.encode()))


def records(rng, x, y, var=0.5, z=None):
    """(n, 8) records at (x, y) with a distinct payload per point, so that keeping the wrong point of a cell shows"""
    x = np.atleast_1d(np.asarray(x, np.float32))
    n = x.shape[0]
    p = np.zeros((n, 8), np.float32)
    p[:, 0] = x
    p[:, 1] = np.asarray(y, np.float32)
    p[:, 2] = rng.uniform(-3, 3, n).astype(np.float32) if z is None else np.asarray(z, np.float32)
    p[:, 3] = rng.uniform(0, 2, n).astype(np.float32)                       # w: overwritten with 1 by the call
    p.view(np.uint32)[:, 4] = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    p[:, 5] = np.asarray(var, np.float32)
    p[:, 6] = rng.integers(0, 256, n).astype(np.float32)
    p[:, 7] = rng.uniform(0, 1, n).astype(np.float32)
    return p


def in_cell(rng, cx, cy, res):
    """points strictly inside the cells with ceil(x / res) = cx, ceil(y / res) = cy (clear of the edges)"""
    cx, cy = np.asarray(cx, np.float64), np.asarray(cy, np.float64)
    x = ((cx - 0.9 + 0.8 * rng.uniform(0, 1, cx.shape)) * res).astype(np.float32)
    y = ((cy - 0.9 + 0.8 * rng.uniform(0, 1, cy.shape)) * res).astype(np.float32)
    return x, y


def _bits(u):
    return np.asarray(u, np.uint32).view(np.float32)


VARIANCE_GATE = _bits([0x00000000, 0x80000000, 0x00000001, 0x00400000, 0x007fffff, 0x80000001, 0x00800000,
                       0x3f000000, 0x3f7fffff, 0x3f800000, 0x3f800001, 0x7fc00000, 0xffc00000, 0x7f800001,
                       0x7f800000, 0xff800000])
NAN_WORDS = np.array([0x7f800001, 0x7fbfffff, 0xff800001, 0x7fc00000, 0xffffffff, 0xffc00001, 0x7f800000,
                      0x80000000, 0xff800000, 0x7fffffff], np.uint32)
SIZES = [(0, 0), (0, 1), (1, 0), (1, 1), (1023, 1025), (1025, 1023), (1024, 3079), (3079, 1024), (3079, 0),
         (0, 3079), (1, 3079), (1025, 1), (1024, 1023)]


# ---- the cases -------------------------------------------------------------------------------------------------------
def _cell_edges(name, res):
    rng = _rng(name)
    k = np.arange(-5, 6, dtype=np.float64)
    on = np.concatenate([(k * res).astype(np.float32), k.astype(np.float32) * F(res)])
    xs = np.concatenate([on, np.nextafter(on, F(np.inf)), np.nextafter(on, F(-np.inf)),
                         _bits([0x80000000, 0x00000000, 0x00000001, 0x80000001, 0x0d000000, 0x8d000000])])
    xs = np.unique(xs.view(np.uint32)).view(np.float32)                    # -0 and +0 both stay
    ys = _bits([0x80000000, 0x00000000, 0x80000001]).tolist() + [F(res), np.nextafter(F(res), F(1)), F(-res)]
    ys = np.array(ys, np.float32)
    gx, gy = np.meshgrid(xs, ys, indexing="ij")
    px = np.concatenate([gx.ravel(), gy.ravel()])
    py = np.concatenate([gy.ravel(), gx.ravel()])
    new = records(rng, px, py, var=rng.choice(np.array([0.3, 2.0, 0.0], np.float32), px.size))
    perm = rng.permutation(px.size)[: px.size * 2 // 3]
    old = records(rng, px[perm], py[perm], var=rng.choice(np.array([0.5, 0.25, 1.0, 0.0], np.float32), perm.size))
    return new, old, res


def _nan_positions(name, res):
    rng = _rng(name)
    nan, inf = F(np.nan), F(np.inf)
    q = F(0.03)
    xy = [(nan, q), (q, nan), (nan, nan), (inf, q), (-inf, q), (q, inf), (q, -inf), (inf, inf), (-inf, -inf),
          (inf, nan), (q, q), (F(0.13), q), (q, F(0.13))]
    x = np.array([a for a, _ in xy] * 3, np.float32)
    y = np.array([b for _, b in xy] * 3, np.float32)
    n = x.shape[0]
    for col, w in ((x, 0x7f800001), (y, 0xffc00000)):                       # NaN positions with other payloads
        col.view(np.uint32)[n // 3: 2 * n // 3][np.isnan(col[n // 3: 2 * n // 3])] = w
    new = records(rng, x, y, var=0.2)
    o = rng.permutation(n)
    old = records(rng, x[o], y[o], var=0.5)
    return new, old, res


def _duplicates(name, res):
    """cells repeated inside each map and across warps and blocks; the first point of a cell is rarely lane 0"""
    rng = _rng(name)
    out = []
    for n, ncell in ((5000, 700), (4100, 300)):
        cx = rng.integers(-40, 40, ncell)
        cy = rng.integers(-40, 40, ncell)
        c = rng.integers(0, ncell, n)
        c[32::32] = c[rng.integers(0, 32, c[32::32].size)]                  # lane 0 of every later warp repeats a cell
        x, y = in_cell(rng, cx[c], cy[c], res)
        out.append(records(rng, x, y, var=rng.choice(np.array([0.4, 0.9, 1.5], np.float32), n)))
    return out[0], out[1], res


def _variance_gate(name, res):
    rng = _rng(name)
    g = VARIANCE_GATE.shape[0]
    cx, cy = np.arange(g) - 8, np.full(g, 3)
    x, y = in_cell(rng, cx, cy, res)
    new = records(rng, x, y, var=F(0.3), z=F(5.0))
    x2, y2 = in_cell(rng, np.concatenate([cx, cx]), np.concatenate([cy, cy]), res)
    var = np.concatenate([VARIANCE_GATE, np.full(g, 0.5, np.float32)])     # the second point of each cell is dropped
    old = records(rng, x2, y2, var=var, z=F(2.0))
    old.view(np.uint32)[:g, 5] = VARIANCE_GATE.view(np.uint32)              # the exact bit patterns, NaNs included
    return new, old, res


def _extreme_values(name, res):
    rng = _rng(name)
    vn = np.array([3.4028235e38, -3.4028235e38, 1e-45, 1e-20, 0.0, -0.0, np.inf, np.nan, 1e19, 1.5], np.float32)
    en = np.array([3.4028235e38, -3.4028235e38, 1e-45, 0.0, np.inf, -np.inf, np.nan], np.float32)
    eo = np.array([3.4028235e38, -1e-45, 7.0, -np.inf], np.float32)
    vo = np.array([0.5, 1e-45, np.nextafter(F(1), F(0)), 1e-20], np.float32)
    a, b, c, d = (m.ravel() for m in np.meshgrid(vn, en, eo, vo, indexing="ij"))
    n = a.shape[0]
    x, y = in_cell(rng, np.arange(n) % 50, np.arange(n) // 50, res)
    new = records(rng, x, y, var=a, z=b)
    old = records(rng, x, y, var=d, z=c)
    return new, old, res


def _bgra_nan_bits(name, res):
    rng = _rng(name)
    w = NAN_WORDS.shape[0]
    cx = np.arange(3 * w)
    x, y = in_cell(rng, cx, np.zeros(3 * w), res)
    new = records(rng, x[: 2 * w], y[: 2 * w], var=0.2)                    # w cells fused, w new-only
    old = records(rng, np.concatenate([x[:w], x[2 * w:]]), np.concatenate([y[:w], y[2 * w:]]),
                  var=np.concatenate([np.full(w, 0.5, np.float32), np.full(w, 0.5, np.float32)]))
    for p in (new, old):
        u = p.view(np.uint32)
        u[:, 4] = np.resize(NAN_WORDS, u.shape[0])
        u[:, 6] = np.resize(NAN_WORDS[::-1], u.shape[0])
        u[:, 7] = np.resize(np.roll(NAN_WORDS, 3), u.shape[0])
    old.view(np.uint32)[:, 4] = old.view(np.uint32)[::-1, 4].copy()
    return new, old, res


def hash_wrap_cells(n, res, count=6):
    """cells (cx, cy) whose home slot in a table for n points is the last slot, then slot 0 and slot 1"""
    mask = table_mask(n)
    cx, cy = np.meshgrid(np.arange(-300, 300), np.arange(-300, 300), indexing="ij")
    cx, cy = cx.ravel(), cy.ravel()
    s = hash_slot(cell_centre(((cx - 0.5) * res).astype(np.float32), res),
                  cell_centre(((cy - 0.5) * res).astype(np.float32), res), mask)
    pick = [np.flatnonzero(s == mask)[:count], np.flatnonzero(s == 0)[:2], np.flatnonzero(s == 1)[:2]]
    assert pick[0].size == count
    pick = np.concatenate(pick)
    return cx[pick], cy[pick]


def _hash_wrap(name, res, n):
    rng = _rng(name)
    cx, cy = hash_wrap_cells(n, res)
    c = np.concatenate([np.arange(cx.size), rng.integers(0, cx.size, n - cx.size)])
    c[: cx.size] = rng.permutation(cx.size)
    x, y = in_cell(rng, cx[c], cy[c], res)
    new = records(rng, x, y, var=0.3)
    o = rng.permutation(n)
    old = records(rng, x[o], y[o], var=rng.choice(np.array([0.5, 1.0], np.float32), n))
    assert hash_slot(cell_centre(x, res), cell_centre(y, res), table_mask(n)).max() == table_mask(n)
    return new, old, res


def _one_big_cell(name, res):
    rng = _rng(name)
    big = 200_000
    out = []
    for lead in (3, 5):                                                     # a few other cells come first
        cx = np.concatenate([np.arange(1, lead + 1), np.full(big, 7)])
        x, y = in_cell(rng, cx, np.full(cx.size, -2), res)
        out.append(records(rng, x, y, var=rng.choice(np.array([0.5, 0.7], np.float32), cx.size)))
    return out[0], out[1], res


def _distinct_full_load(name, res):
    """every point its own cell, n = 32767: 2 n + 2 = 2^16, the fullest table the sizing produces"""
    rng = _rng(name)
    n = 32767
    i = np.arange(n)
    x, y = in_cell(rng, i % 181, i // 181, res)
    new = records(rng, x, y, var=0.3)
    j = i + n // 2
    x2, y2 = in_cell(rng, j % 181, j // 181, res)
    old = records(rng, x2, y2, var=0.5)[rng.permutation(n)]
    return new, old, res


def _sizes(name, res, nn, no):
    rng = _rng(name)
    cells = max(1, (nn + no) // 3)
    cx, cy = rng.integers(-30, 30, cells), rng.integers(-30, 30, cells)
    out = []
    for n in (nn, no):
        c = rng.integers(0, cells, n)
        x, y = in_cell(rng, cx[c], cy[c], res)
        out.append(records(rng, x, y, var=rng.choice(np.array([0.2, 0.6, 1.2], np.float32), n)))
    return out[0], out[1], res


def utm_coordinate(res):
    """the float coordinate whose cell centre lies in another cell: with res = 2^m, v = 2^(m+23) + res is the only
    float of its cell, its centre v - res / 2 is a tie that rounds to 2^(m+23), and the centre of THAT is the cell below.
    (For a resolution that is not a power of two, such as 0.1 or 0.05, no float coordinate does this.)"""
    v = F(res * 2.0 ** 23 + res)
    rx = cell_centre(v, res)
    assert float(v) == res * 2.0 ** 23 + res and cell_centre(rx, res) != rx
    return v


def _utm_scale(name, res):
    """UTM-scale coordinates where the cell centre re-keys (utm_coordinate): the re-fused old points sit in the last
    blocks of an old map several resident waves long, the new points that fuse them in the first block"""
    rng = _rng(name)
    u = utm_coordinate(res)
    c = np.arange(96)
    _, other = in_cell(rng, c, c, res)
    ex = np.concatenate([np.full(64, u), other[64:]])                      # 32 with the large coordinate in y instead
    ey = np.concatenate([other[:64], np.full(32, u)])
    fill = 2_000_000                                                        # ~7800 blocks of 256
    i = np.arange(fill)
    fx, fy = in_cell(rng, i % 1000 - 500, (i // 1000) % 500 + 5, res)
    old = records(rng, np.concatenate([fx, ex]), np.concatenate([fy, ey]), var=0.5)
    new = records(rng, ex, ey, var=0.3)
    return new, old, res


CASES = {
    "cell_edges_res0.1": lambda n: _cell_edges(n, 0.1),
    "cell_edges_res0.05": lambda n: _cell_edges(n, 0.05),
    "cell_edges_res0.3": lambda n: _cell_edges(n, 0.3),
    "nan_positions": lambda n: _nan_positions(n, 0.1),
    "duplicates": lambda n: _duplicates(n, 0.1),
    "variance_gate": lambda n: _variance_gate(n, 0.1),
    "extreme_values": lambda n: _extreme_values(n, 0.1),
    "bgra_nan_bits": lambda n: _bgra_nan_bits(n, 0.1),
    "hash_wrap_40": lambda n: _hash_wrap(n, 0.1, 40),
    "hash_wrap_1000": lambda n: _hash_wrap(n, 0.05, 1000),
    "one_cell_200k": lambda n: _one_big_cell(n, 0.1),
    "distinct_full_load": lambda n: _distinct_full_load(n, 0.1),
    "utm_scale_res0.25": lambda n: _utm_scale(n, 0.25),
    "utm_scale_res0.5": lambda n: _utm_scale(n, 0.5),
}
for _nn, _no in SIZES:
    CASES[f"sizes_{_nn}_{_no}"] = (lambda a, b: lambda n: _sizes(n, 0.1, a, b))(_nn, _no)


MATRICES = {   # gem_transform_cloud takes any 4 x 4 matrix, rigid or not
    "non_rigid": np.array([[1.5, 0.3, -0.2, 0.7], [0.1, 0.8, 0.4, -1.1], [-0.6, 0.2, 2.0, 0.05], [0, 0, 0, 1]], np.float32),
    "nan_entry": np.array([[1, 0, 0, 0], [0, np.nan, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], np.float32),
    "large_translation": np.array([[0.6, -0.8, 0, 1048576.3], [0.8, 0.6, 0, -524288.7], [0, 0, 1, 3e4], [0, 0, 0, 1]],
                                  np.float32),
    "inf_translation": np.array([[1, 0, 0, np.inf], [0, 1, 0, 0], [0, 0, 1, -np.inf], [0, 0, 0, 1]], np.float32),
}


def transform_input():
    rng = _rng("transform")
    p = records(rng, rng.uniform(-50, 50, 3000), rng.uniform(-50, 50, 3000))
    p[:5, 0] = [np.nan, np.inf, -np.inf, 3e38, -0.0]
    p[5:10, 2] = [np.nan, 1e-45, -3e38, np.inf, 0.0]
    return p


def case_names():
    return list(CASES)


_cache = {}


def case_by_name(name):
    """(new, old, resolution); the arrays are shared, copy before modifying"""
    if name not in _cache:
        _cache[name] = CASES[name](name)
    return _cache[name]
