"""The MLS densification of the dense_mapping signal (pointcloudinterpolation, DESIGN.md f10) byte for byte against the
oracle, tests/orc_mls.c: output bytes and every info field on the crafted cases of tests/mls_cases.py, on local maps
harvested from the synthetic c2 stream at 0.05 m and at 0.2 m, a capacity below the count and the size query, every
error path, two runs, cut_submap(dense=True) against take + oracle + grid cloud, and the C++ facade program."""
import ctypes as C
import subprocess

import numpy as np
import pytest
import torch

import gem_b200
import mls_cases as mc
import mls_oracle
import native
from gem_b200 import _lib, synth

pytestmark = pytest.mark.gpu
SENTINEL = -12345.5


@pytest.fixture(scope="module")
def emap():
    return gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1, 8)).to("cuda:0")


def same(got, want, what):
    (go, gi), (wo, wi) = got, want
    assert gi == wi, (what, gi, wi)
    g = go.cpu().numpy()
    assert g.shape == wo.shape, (what, g.shape, wo.shape)
    if g.tobytes() != wo.tobytes():
        bad = np.flatnonzero((g.view(np.uint32) != wo.view(np.uint32)).any(axis=1))
        raise AssertionError((what, "rows differ", int(bad.size), "first", int(bad[0]), g[bad[0]], wo[bad[0]]))


def check(g, recs, overrides, what):
    got = g.mls_upsample(dev(recs), overrides, info=True)
    same(got, mls_oracle.upsample(recs, overrides), what)
    return got


@pytest.mark.parametrize("name", mc.case_names())
def test_crafted(emap, name):
    _, recs, o = mc.case_by_name(name)
    check(emap, recs, o, name)


def harvested_local_map(res, L, frames):
    """a local map harvested from the synthetic c2 stream: the node's per-frame order, moving 0.4 m per frame"""
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    pos = np.array((0.3, -0.2, 1.7), np.float32)
    for k in range(frames):
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([0.4, 0.15, 0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        f = gem_b200.make_frame(T, gem_b200.LaserSensorProcessor())
        centre, _, shift = g.move(pos)
        if k > 0:
            g.harvest_to_local_map(centre, shift)
        g.add(fr["xyzi"], fr["rgba"], f)
        g.compute_features()
        g.snapshot_shown()
        g.raytracing()
    return g


@pytest.fixture(scope="module")
def c2_local_005():
    g = harvested_local_map(0.05, 400, 10)
    rec = g.local_map_take().cpu().numpy()
    assert rec.shape[0] > 3000
    return rec


def test_c2_local_map_005(emap, c2_local_005):
    _, info = check(emap, c2_local_005, {}, "c2 0.05 m")
    assert info["fitted"] > 0 and info["max_neighbours"] > 21


def test_c2_local_map_005_none_and_two_runs(emap, c2_local_005):
    a = check(emap, c2_local_005, mc.NONE, "c2 0.05 m, NONE")
    b = emap.mls_upsample(dev(c2_local_005), mc.NONE, info=True)
    assert a[1] == b[1] and a[0].cpu().numpy().tobytes() == b[0].cpu().numpy().tobytes()   # bytes: the records carry NaNs


def test_kitti_like_02(emap):
    g = harvested_local_map(0.2, 150, 10)
    rec = g.local_map_take().cpu().numpy()
    assert rec.shape[0] > 500
    _, info = check(emap, rec, {}, "c2 0.2 m")
    assert info["max_neighbours"] < 40 and info["fitted"] < info["processed"] and info["count"] > 10 * rec.shape[0]
    check(emap, mc.kitti_like(half=8.0), {}, "kitti-like 0.2 m grid")


def test_dense_blob_long_lists(emap):
    recs = mc.blob(3000, 0.15)
    _, info = check(emap, recs, {"order": 3}, "blob")
    assert info["max_neighbours"] > 1000


def test_capacity_below_count_and_size_query(emap):
    _, recs, o = mc.case_by_name("noisy_plane_tilted")
    full, info = mls_oracle.upsample(recs, o)
    lib, h = emap._lib, emap.handle
    inp = dev(recs)
    p = mls_oracle.params(o)
    pp = _lib.GemMlsParams(*[getattr(p, k) for k, _ in _lib.GemMlsParams._fields_])
    for cap in (0, 1, 10, info["count"] - 1, info["count"]):
        out = torch.full((cap + 7, 8), SENTINEL, dtype=torch.float32, device="cuda:0")
        st = _lib.GemMlsInfo()
        assert lib.gem_mls_upsample(h, C.c_void_p(inp.data_ptr()), inp.shape[0], C.byref(pp), C.c_void_p(out.data_ptr()), cap,
                                    C.byref(st)) == 0
        want = dict(info, fitted=-1) if cap == 0 else info
        assert {k: getattr(st, k) for k, _ in _lib.GemMlsInfo._fields_} == want, cap
        host = out.cpu().numpy()
        assert host[:cap].tobytes() == full[:cap].tobytes(), cap
        assert (host[cap:] == SENTINEL).all(), cap


def test_errors_write_nothing(emap):
    lib, h = emap._lib, emap.handle
    _, recs, _ = mc.case_by_name("tilted_lattice_plane")
    buf = dev(np.concatenate([recs[:100], np.full((60, 8), SENTINEL, np.float32)]))
    inp, out = buf[:100], buf[100:]
    base = buf.clone()
    pin, pout = C.c_void_p(inp.data_ptr()), C.c_void_p(out.data_ptr())

    def params(**kw):
        q = dict(mls_oracle.GEM, upsampling=1)
        q.update(kw)
        return _lib.GemMlsParams(q["search_radius"], q["sqr_gauss_param"], int(q["polynomial_fit"]), q["order"], q["upsampling"],
                                 q["point_density"], q["seed"])

    good = params()
    calls = []
    for kw in ({"search_radius": 0.0}, {"search_radius": -0.5}, {"search_radius": float("nan")}, {"search_radius": float("inf")},
               {"sqr_gauss_param": 0.0}, {"sqr_gauss_param": float("nan")}, {"sqr_gauss_param": -1.0}, {"order": 0}, {"order": 6},
               {"upsampling": 2}, {"upsampling": -1}, {"point_density": -1}):
        assert mls_oracle.upsample(recs[:100], {k: v for k, v in kw.items()}) is None, kw
        calls.append((kw, lambda q=params(**kw): (pin, 100, q, pout, 60)))
    calls += [("n < 0", lambda: (pin, -1, good, pout, 60)),
              ("NULL points", lambda: (None, 100, good, pout, 60)),
              ("capacity < 0", lambda: (pin, 100, good, pout, -1)),
              ("NULL out", lambda: (pin, 100, good, None, 60)),
              ("overlap: same", lambda: (pin, 100, good, pin, 60)),
              ("overlap: tail", lambda: (pin, 100, good, C.c_void_p(inp.data_ptr() + 99 * 32), 60)),
              ("overlap: head", lambda: (C.c_void_p(inp.data_ptr() + 32 * 5), 95, good, pin, 6))]
    for what, make in calls:
        a = make()
        st = _lib.GemMlsInfo(-7, -7, -7, -7, -7)
        assert lib.gem_mls_upsample(h, a[0], a[1], C.byref(a[2]), a[3], a[4], C.byref(st)) == 1, what
        assert (st.count, st.processed, st.fitted, st.skipped, st.max_neighbours) == (-7,) * 5, what
        emap.sync()
        assert torch.equal(buf, base), what
    assert lib.gem_mls_upsample(h, pin, 100, None, pout, 60, C.byref(_lib.GemMlsInfo())) == 1
    assert lib.gem_mls_upsample(h, pin, 100, C.byref(good), pout, 60, None) == 1
    emap.sync()
    assert torch.equal(buf, base)
    st = _lib.GemMlsInfo(-7, -7, -7, -7, -7)
    assert lib.gem_mls_upsample(h, None, 0, C.byref(good), pout, 60, C.byref(st)) == 0
    assert (st.count, st.processed, st.fitted, st.skipped, st.max_neighbours) == (0, 0, 0, 0, 0)
    with pytest.raises(ValueError):
        emap.mls_upsample(inp[:, :4].contiguous())
    with pytest.raises(ValueError):
        emap.mls_upsample(inp, {"upsampling": "voxel_grid_dilation"})


def test_seed_changes_samples_not_counts(emap):
    _, recs, o = mc.case_by_name("noisy_surface_order3")
    a, ia = emap.mls_upsample(dev(recs), dict(o, seed=1), info=True)
    b, ib = emap.mls_upsample(dev(recs), dict(o, seed=2), info=True)
    assert ia == ib and a.shape == b.shape and a.cpu().numpy().tobytes() != b.cpu().numpy().tobytes()


def test_cut_submap_dense():
    """cut_submap(dense=True) is [taken local map, its MLS points, grid cloud]; dense=False is unchanged.  Three maps are
    driven alike: one cut dense, one cut plain, one taken and exported step by step"""
    res, L = 0.1, 200
    scene = synth.make_scene()
    maps = [gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res) for _ in range(3)]
    pos = np.array((0.3, -0.2, 1.7), np.float32)
    for k in range(8):
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([0.5, 0.1, 0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        f = gem_b200.make_frame(T, gem_b200.LaserSensorProcessor())
        for g in maps:
            centre, _, shift = g.move(pos)
            if k > 0:
                g.harvest_to_local_map(centre, shift)
            g.add(fr["xyzi"], fr["rgba"], f)
            g.compute_features()
            g.snapshot_shown()
            g.raytracing()
    a, b, c = maps
    dense = a.cut_submap(dense=True, seed=11).cpu().numpy()
    plain = b.cut_submap().cpu().numpy()
    local = c.local_map_take().cpu().numpy()
    grid = c.export_grid_cloud("shown").cpu().numpy()
    assert local.shape[0] > 300
    extra, _ = mls_oracle.upsample(local, {"seed": 11})
    assert extra.shape[0] > local.shape[0]
    want = np.concatenate([local, extra, grid])
    assert dense.shape == want.shape and dense.tobytes() == want.tobytes()
    assert plain.tobytes() == np.concatenate([local, grid]).tobytes()
    assert a.local_map_size() == 0 and b.local_map_size() == 0


def test_facade_mls_program_runs():
    exe = native.facade_program("mls_smoke")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "mls ok" in r.stdout, r.stdout + r.stderr
