"""Local submaps, CPU side: the grid-cloud oracle (tests/orc_grid_cloud.c) against a numpy restatement of
gridMaptoPointCloud (ElevationMapping.cpp:1204-1223) on show()'s masked layers, the local-map order definition, and the
C++ facade's local-submap calls compiling and linking."""
import subprocess

import numpy as np
import pytest

import native
import submap_oracle
from oracle_lib import export_from_feature


def np_grid_cloud(f, L, centre, start, res):
    """:1204-1223 over visualMap_ = export_from_feature's masked layers, GridMapIterator order (ix fastest)"""
    v = export_from_feature(f, L)                          # (L, L), a[ix, iy], NaN where show() cleared the cell
    e, t = v["elevation"], v["traver"]
    take = (e != -10) & (t != -10) & ~np.isnan(t)
    i = np.flatnonzero(take.ravel(order="F"))
    ix, iy = i % L, i // L
    half = 0.5 * (L * res) - 0.5 * res
    out = np.empty((i.size, 8), np.float32)
    out[:, 0] = ((np.float64(centre[0]) + half) - res * ((ix + L - start[0]) % L)).astype(np.float32)
    out[:, 1] = ((np.float64(centre[1]) + half) - res * ((iy + L - start[1]) % L)).astype(np.float32)
    out[:, 2] = e[ix, iy]
    out[:, 3] = 1.0
    r, g, b = (v[c][ix, iy].astype(np.uint32) for c in ("color_r", "color_g", "color_b"))
    out[:, 4] = (b | (g << 8) | (r << 16) | np.uint32(0xff000000)).view(np.float32)
    out[:, 5] = v["variance"][ix, iy]
    out[:, 6] = v["intensity"][ix, iy]
    out[:, 7] = t[ix, iy]
    return out


def features(L, seed):
    rng = np.random.default_rng(seed)
    n = L * L
    tr = rng.choice(np.array([0.0, 0.37, 1.0, -0.25, -3.5, -9.999, -10.0, np.nan], np.float32), n)
    el = rng.uniform(-2, 2, n).astype(np.float32)
    el[rng.random(n) < 0.1] = -10.0
    return {"elevation": el, "variance": rng.uniform(0, 0.5, n).astype(np.float32), "traver": tr,
            "color_r": rng.integers(0, 256, n).astype(np.int32), "color_g": rng.integers(0, 256, n).astype(np.int32),
            "color_b": rng.integers(0, 256, n).astype(np.int32), "intensity": rng.uniform(0, 255, n).astype(np.float32),
            "rough": np.zeros(n, np.float32), "slope": np.zeros(n, np.float32)}


@pytest.mark.parametrize("L,res,seed", [(37, 0.1, 1), (64, 0.05, 2), (200, 0.1, 3)])
def test_grid_cloud_oracle_matches_numpy_restatement(L, res, seed):
    f = features(L, seed)
    rng = np.random.default_rng(seed + 10)
    centre = rng.uniform(-50, 50, 2).astype(np.float32)
    start = rng.integers(0, L, 2).astype(np.int32)
    got = submap_oracle.grid_cloud(f, L, centre, start, res)
    want = np_grid_cloud(f, L, centre, start, res)
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # :1208 is not the harvest's traver >= 0 (:725): negative traversabilities other than -10 are taken, -10 is not
    el, tr = f["elevation"], f["traver"]
    neg = (el != -10) & (tr > -10) & (tr < 0)
    assert neg.sum() > 100
    t = got[:, 7]
    assert np.count_nonzero((t > -10) & (t < 0)) == neg.sum()
    assert not np.any(t == -10) and not np.any(np.isnan(t)) and not np.any(got[:, 2] == -10)
    assert got.shape[0] == np.count_nonzero((el != -10) & (tr != -10) & ~np.isnan(tr))


def test_local_map_order_definition():
    """the dict of :740-747 iterates like "all harvests concatenated, last occurrence of each key kept", which is how
    gem_local_map_take orders its records"""
    rng = np.random.default_rng(4)
    d = submap_oracle.LocalMapDict()
    log = []
    for _ in range(6):
        rec = np.zeros((rng.integers(0, 300), 8), np.float32)
        rec[:, 0] = rng.integers(0, 40, rec.shape[0]) * np.float32(0.1)
        rec[:, 1] = rng.integers(0, 40, rec.shape[0]) * np.float32(0.1)
        rec[:, 2] = rng.uniform(0, 1, rec.shape[0])
        d.insert_all(rec)
        log.append(rec)
    log = np.concatenate(log)
    keys = log[:, :2].copy().view(np.uint64).ravel()
    last = {k: i for i, k in enumerate(keys.tolist())}
    keep = np.array(sorted(last.values()))
    assert np.array_equal(d.records().view(np.uint32), log[keep].view(np.uint32))
    assert len(d) < log.shape[0]


def test_local_submap_facade_compiles_and_links():
    exe = native.facade_program("local_submap_smoke")
    out = subprocess.run(["nm", "-C", "--undefined-only", exe], capture_output=True, text=True).stdout
    for sym in ("gem_export_grid_cloud", "gem_harvest_to_local_map", "gem_local_map_take", "gem_local_map_clear"):
        assert sym in out, sym
