"""The VoxelGrid pre-filter, CPU side: the oracle (tests/orc_voxel_grid.c) against the independent numpy restatement of
tests/voxel_cases.py, bit for bit (output bytes and every info field), on every crafted case; the V3-contains-V2 claim
on limits placed at float roundings; the ctypes mirrors of gem_voxel_grid_params / gem_voxel_grid_info against the C
compiler; the C++ facade program compiles."""
import ctypes as C

import numpy as np
import pytest

import native
import voxel_cases as vc
import voxel_oracle


def same(got, want, what):
    (go, gi), (wo, wi) = got, want
    assert gi == wi, (what, gi, wi)
    assert go.shape == wo.shape, (what, go.shape, wo.shape)
    if go.tobytes() != wo.tobytes():
        bad = np.flatnonzero((go.view(np.uint32) != wo.view(np.uint32)).any(axis=1))
        raise AssertionError((what, "rows differ", int(bad.size), "first", int(bad[0]), go[bad[0]], wo[bad[0]]))


@pytest.mark.parametrize("name", vc.case_names())
def test_oracle_matches_restatement(name):
    _, p, leaf, field, limits, neg = vc.case_by_name(name)
    got = voxel_oracle.voxel_grid(p, leaf, field, limits, neg)
    want = vc.np_voxel_grid(p, leaf, field, limits, neg)
    same(got, want, name)
    out, info = got
    if name == "negzero_alone":
        assert out.view(np.uint32).tolist() == [[0, 0, 0, 0]]          # -0.0 comes out +0.0
    if name.startswith("passthrough") or name == "limit_rounding_passthrough":
        assert info["passthrough"] == 1 and out.tobytes() == np.ascontiguousarray(p, np.float32).tobytes()
    if name in ("limit_rounding_without_point", "far_from_origin", "defined_order", "one_voxel_1m", "own_voxel"):
        assert info["passthrough"] == 0 and info["count"] > 0
    if name in ("empty", "all_cut_nonfinite", "all_cut_field"):
        assert info["count"] == 0 and info["used"] == 0
    if name == "own_voxel":
        assert info["count"] == p.shape[0]
    if name == "one_voxel_1m":
        assert info["count"] == 1 and info["used"] == p.shape[0]


def test_defined_order_case_overflows_an_int_idx():
    """V6 DEFINED: the case passes V4 (d0 d1 d2 <= INT32_MAX) while div0 div1 div2 exceeds 2^31"""
    _, p, leaf, field, limits, neg = vc.case_by_name("defined_order")
    dprod, divprod = vc.div_product(p, leaf, field, limits, neg)
    assert dprod <= 2 ** 31 - 1 < 2 ** 31 < divprod


def test_limit_rounding_case_turns_on_the_v3_point():
    """float32(0.1) is cut by the double limit (V2) and kept by the float one (V3): it alone decides the overflow"""
    _, p, leaf, field, limits, neg = vc.case_by_name("limit_rounding_passthrough")
    used, bnd = vc._masks(p, field, limits, neg)
    assert bnd[7] and not used[7] and (used <= bnd).all()


def test_one_voxel_sum_order_matters():
    """the sequential float sum of V8 is not the pairwise one of np.sum: the case tells them apart"""
    _, p, leaf, field, limits, neg = vc.case_by_name("one_voxel_1m")
    out, _ = voxel_oracle.voxel_grid(p, leaf, field, limits, neg)
    cols = np.ascontiguousarray(p.T)                     # contiguous rows: np.sum sums them pairwise
    pairwise = np.sum(cols, axis=1, dtype=np.float32) / np.float32(p.shape[0])
    assert out[0].tobytes() != pairwise.tobytes()


def test_v3_contains_v2_at_float_roundings():
    """no float lies strictly between a double limit and its float rounding, so every point V2 keeps V3 keeps: checked
    with limits drawn as doubles and points placed at their float roundings and the neighbouring floats"""
    rng = np.random.default_rng(3)
    lims = np.concatenate([rng.uniform(-50, 50, 300), rng.uniform(-1e-3, 1e-3, 100), [0.1, -0.1, 1e-40, 3.4e38, -3.4e38]])
    vals = []
    for d in lims:
        f = np.float32(d)
        vals += [f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf))]
    v = np.array(vals, np.float32)
    p = np.zeros((v.size, 4), np.float32)
    for field, col in (("x", 0), ("intensity", 3)):
        p[:, :] = 0.0
        p[:, col] = v
        for lo, hi in zip(lims[::2], lims[1::2]):
            lo, hi = min(lo, hi), max(lo, hi)
            for neg in (False, True):
                used, bnd = vc._masks(p, field, (lo, hi), neg)
                assert (used <= bnd).all(), (field, lo, hi, neg)


def test_capacity_and_errors():
    _, p, leaf, *_ = vc.case_by_name("dense_random")
    full, info = voxel_oracle.voxel_grid(p, leaf)
    part, pinfo = voxel_oracle.voxel_grid(p, leaf, capacity=10)
    assert pinfo == info and part.tobytes() == full[:10].tobytes()
    q, qinfo = voxel_oracle.voxel_grid(p, leaf, capacity=0)
    assert qinfo == info and q.shape[0] == 0
    for bad in ((0.0, None), (-0.1, None), (float("nan"), None), (float("inf"), None), ((0.1, 0.1, 0.0), None), (0.1, 4), (0.1, -2)):
        assert voxel_oracle.voxel_grid(p, bad[0], bad[1]) is None, bad


def test_launch_chains_run():
    """filter.launch and the three-call KITTI chain on a cloud spanning their limits"""
    rng = np.random.default_rng(9)
    p = vc._cloud(rng, 30000, -60.0, 60.0)
    out, infos = voxel_oracle.chain(p, voxel_oracle.FILTER_KITTI_LAUNCH)
    assert len(infos) == 3 and 0 < infos[2]["count"] <= infos[1]["count"] <= infos[0]["count"]
    assert (np.abs(out[:, 0]) <= 40.0).all() and (np.abs(out[:, 1]) <= 40.0).all()
    one, info = voxel_oracle.voxel_grid(p, *voxel_oracle.FILTER_LAUNCH[0])
    assert info["count"] == one.shape[0] > 0 and (np.abs(one[:, 0]) <= 10.0).all()


def test_voxel_structs_match_the_header():
    import gem_b200._lib as L
    consts = {f"GEM_VOXEL_FIELD_{c}": L.VOXEL_FIELDS[k] for c, k in (("NONE", None), ("X", "x"), ("Y", "y"), ("Z", "z"),
                                                                      ("INTENSITY", "intensity"))}
    native.assert_struct_layouts({"gem_voxel_grid_params": L.GemVoxelGridParams, "gem_voxel_grid_info": L.GemVoxelGridInfo},
                                 consts)
    # the oracle's mirror of the parameters has the library's layout too
    assert C.sizeof(voxel_oracle.Params) == C.sizeof(L.GemVoxelGridParams)


def test_facade_program_with_voxel_grid_compiles():
    native.facade_compiles("voxel_grid_smoke")
