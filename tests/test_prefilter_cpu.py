"""The pre-filtered asynchronous add (DESIGN.md f20), CPU side: the device-side decision of a VoxelGrid step
(gem_voxgrid.h, built by the host compiler) against the host arithmetic gem_voxel_grid used before the decision moved to
the device, on every crafted voxel case, limits at float roundings, V4 just under and over INT32_MAX and large-coordinate
clouds where div exceeds d the most, with the fixed 40-bit key width holding on all of them; the oracle chain decode ->
VoxelGrid steps against the independent numpy composition on the PointCloud2 layouts; the ctypes mirrors against the
header; the refusals of the new calls without a device."""
import ctypes as C
import os

import numpy as np
import pytest

import native
import pc2_cases as pc
import pc2_oracle
import voxel_cases as vc
import voxel_oracle

F = np.float32
KEY_BITS = 40
PASS, GRID, WIDE = 1, 2, 3
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        _LIB = native.shared_library("voxgrid_host", [os.path.join(native.HERE, "voxgrid_host.cpp")], native.HOST_CXX)
        _LIB.voxgrid_layout.restype = C.c_int
    return _LIB


def device_layout(mn, mx, inv):
    a = [np.ascontiguousarray(v, np.float32) for v in (mn, mx, inv)]
    minb = np.zeros(3, np.float64)
    radix = np.zeros(3, np.uint64)
    mode = lib().voxgrid_layout(*[C.c_void_p(v.ctypes.data) for v in a], C.c_void_p(minb.ctypes.data),
                                C.c_void_p(radix.ctypes.data))
    return mode, minb, [int(v) for v in radix]


def host_layout(mn, mx, inv):
    """the host arithmetic of gem_voxel_grid before this change (V4, then V6), in numpy float32 / float64"""
    d = []
    with np.errstate(over="ignore", invalid="ignore"):
        for a in range(3):
            q = F(F(mx[a]) - F(mn[a])) * F(inv[a])
            if not np.isfinite(q) or q >= F(2.0 ** 62):
                return PASS, None, None, None
            d.append(int(q) + 1)
        if max(d) > 2 ** 31 - 1 or d[0] * d[1] > 2 ** 31 - 1 or d[0] * d[1] * d[2] > 2 ** 31 - 1:
            return PASS, None, None, d
        lo = [F(mn[a]) * F(inv[a]) for a in range(3)]
        hi = [F(mx[a]) * F(inv[a]) for a in range(3)]
    if not all(np.isfinite(lo) & np.isfinite(hi)):
        return WIDE, None, None, d   # the old host code cast a NaN difference here and refused the call
    minb = np.floor(np.array(lo, np.float64))
    div = [int(np.floor(np.float64(hi[a])) - minb[a]) + 1 for a in range(3)]
    return GRID, minb, [div[0], div[0] * div[1], div[0] * div[1] * div[2]], d


def check(mn, mx, inv, what):
    mode, minb, radix = device_layout(mn, mx, inv)
    hm, hminb, hradix, d = host_layout(mn, mx, inv)
    assert mode == hm, (what, mode, hm)
    if mode == GRID:
        assert minb.tobytes() == hminb.tobytes() and radix == hradix, (what, minb, hminb, radix, hradix)
        assert radix[2] < 2 ** KEY_BITS, (what, radix)     # every key, the cut key included, fits the sort's width
        div = [radix[0], radix[1] // radix[0], radix[2] // radix[1]]
        assert all(div[a] <= 8 * d[a] for a in range(3)), (what, div, d)
        return max(div[a] / d[a] for a in range(3))
    return 0.0


def bounds(p, field, limits, negative):
    _, bnd = vc._masks(np.ascontiguousarray(p, np.float32).reshape(-1, 4), field, limits, negative)
    b = np.ascontiguousarray(p, np.float32).reshape(-1, 4)[bnd, :3]
    return (b.min(axis=0), b.max(axis=0)) if b.shape[0] else None


def inv_of(leaf):
    leaf = np.full(3, leaf, np.float32) if np.ndim(leaf) == 0 else np.asarray(leaf, np.float32)
    return F(1.0) / leaf


@pytest.mark.parametrize("name", vc.case_names())
def test_layout_matches_the_host_arithmetic_on_the_voxel_cases(name):
    _, p, leaf, field, limits, neg = vc.case_by_name(name)
    b = bounds(p, field, limits, neg)
    if b is None:
        pytest.skip("no V3 survivor: V5, decided before the layout")
    check(b[0], b[1], inv_of(leaf), name)


def test_layout_at_float_rounded_limits():
    rng = np.random.default_rng(11)
    p = vc._cloud(rng, 2000, -3.0, 3.0)
    for lo in (0.1, -0.1, 1e-3, float(np.nextafter(F(0.5), F(1))), 2.9999999):
        for neg in (False, True):
            for field in ("x", "y", "z", "intensity"):
                b = bounds(p, field, (lo, lo + 1.0), neg)
                if b is not None:
                    check(b[0], b[1], inv_of(0.05), (lo, neg, field))


def test_v4_just_under_and_over_int32_max():
    one = np.ones(3, F)
    # d = 1290^3 (under), 1291 * 1290^2 (over); and one axis alone at the top of the int range
    assert check(np.zeros(3, F), np.array([1289.5, 1289.5, 1289.5], F), one, "1290^3") > 0
    assert device_layout(np.zeros(3, F), np.array([1290.5, 1289.5, 1289.5], F), one)[0] == PASS
    assert host_layout(np.zeros(3, F), np.array([1290.5, 1289.5, 1289.5], F), one)[0] == PASS
    top = F(2.0 ** 31 - 128)               # the largest float below 2^31: d = 2^31 - 127
    assert check(np.zeros(3, F), np.array([top, 0, 0], F), one, "d0 near INT32_MAX") > 0
    assert device_layout(np.zeros(3, F), np.array([F(2.0 ** 31), 0, 0], F), one)[0] == PASS


def test_large_coordinates_where_div_exceeds_d():
    """clouds far from the origin with spans of a few ulps: the products' rounding, not the span, sets div"""
    rng = np.random.default_rng(5)
    worst = 0.0
    for _ in range(4000):
        e = int(rng.integers(-10, 120))
        base = F(rng.uniform(1.0, 2.0) * 2.0 ** e) * F(rng.choice([-1.0, 1.0]))
        mn = np.full(3, base, F)
        mx = mn.copy()
        for a in range(3):
            for _ in range(int(rng.integers(0, 4))):
                mx[a] = np.nextafter(mx[a], F(np.inf))
        inv = F(1.0) / np.array([F(2.0 ** -rng.uniform(-20, 20)) for _ in range(3)], F)
        worst = max(worst, check(mn, mx, inv, (base, mx - mn, inv)))
    assert 1.0 < worst <= 8.0, worst        # the bound is exercised, and it holds


def test_non_finite_products_are_wide():
    """bounds whose products with 1 / leaf overflow although their span is small: no integer voxel index"""
    mn = np.array([3e38, 0, 0], F)
    assert device_layout(mn, mn, np.array([10, 1, 1], F))[0] == WIDE
    assert host_layout(mn, mn, np.array([10, 1, 1], F))[0] == WIDE


FLOAT_LAYOUTS = ["kitti16", "xyzir32", "xyzir22", "pandarqt", "ouster", "xyzrgbict"]


@pytest.mark.parametrize("lay", FLOAT_LAYOUTS)
@pytest.mark.parametrize("launch", ["filter", "kitti"])
def test_oracle_chain_equals_numpy_composition(lay, launch):
    """pc2_oracle.decode -> voxel_oracle.chain against pc2_cases.np_decode -> voxel_cases.np_voxel_grid per step"""
    steps = voxel_oracle.FILTER_LAUNCH if launch == "filter" else voxel_oracle.FILTER_KITTI_LAUNCH
    rng = np.random.default_rng(hash((lay, launch)) & 0xFFFF)
    cloud = vc._cloud(rng, 20000, -50.0, 50.0)
    cloud[::97, 2] = np.nan
    case = pc.from_xyzi("c", lay, cloud, seed=3, row_pad=8)
    got, ginfos = voxel_oracle.chain(pc2_oracle.xyzi(pc2_oracle.decode(case)[0]), steps)
    want = pc2_oracle.xyzi(pc.np_decode(case)[0])
    winfos = []
    for leaf, field, limits, neg in steps:
        want, info = vc.np_voxel_grid(want, leaf, field, limits, neg)
        winfos.append(info)
    assert ginfos == winfos, (ginfos, winfos)
    assert got.tobytes() == want.tobytes()
    assert ginfos[-1]["count"] > 100


def test_structs_match_the_header():
    import gem_b200._lib as L
    native.assert_struct_layouts({"gem_prefilter": L.GemPrefilter, "gem_projection": L.GemProjection},
                                 {"GEM_PREFILTER_MAX_STEPS": L.PREFILTER_MAX_STEPS})


def test_refusals_without_a_device():
    """every new call refuses a NULL handle and bad arguments before it touches a device"""
    import gem_b200._lib as L
    g = L.load()
    pf = L.GemPrefilter()
    info = (L.GemVoxelGridInfo * 4)()
    frame = L.GemFrame()
    lay = L.GemPointCloud2()
    assert g.gem_add_pointcloud2_filtered_host_async(None, C.byref(lay), None, 0, None, C.byref(pf), C.byref(frame)) == 1
    assert g.gem_add_pointcloud2_filtered_host_async(None, C.byref(lay), None, 0, None, None, C.byref(frame)) == 1
    assert g.gem_add_points_filtered_stream(None, None, 0, C.byref(pf), None, None, C.byref(frame)) == 1
    assert g.gem_prefilter_info(None, info, 1) == 1
    from gem_b200 import ElevationMap
    with pytest.raises(ValueError):
        ElevationMap.prefilter([(0.1, "x", (-1, 1), False)] * 5)
    with pytest.raises(ValueError):
        ElevationMap.prefilter([(0.1, "w", (-1, 1), False)])
    p = ElevationMap.prefilter(voxel_oracle.FILTER_KITTI_LAUNCH)
    assert p.nsteps == 3 and p.step[1].field == 2 and abs(p.step[2].leaf_size[0] - 0.2) < 1e-7


def test_facade_program_with_prefilter_compiles():
    native.facade_compiles("prefilter_smoke")
