"""The feature kernel and the ray clean-up against the oracle on the crafted map cases (tests/map_cases.py).

Every case goes through untiled handles: the nine Map_feature outputs, the traver layer (stale values in the empty
cells included), the grid_map write-back (export_layers, which reads traver_out), then the ray clean-up: elevation,
lowest (reset to 10) and the map state.  The start-0 cases also go through tile handles, world 2 and 4 on one GPU,
with tiles that are not multiples of the 16-cell feature tile.  Every comparison is bit for bit, NaN as a class."""
import numpy as np
import pytest

import gem_b200
import map_cases as mc
from gem_b200 import tiled
from oracle_lib import OracleMap

pytestmark = pytest.mark.gpu
f32 = np.float32
FEATURE_OUT = ["elevation", "variance", "color_r", "color_g", "color_b", "rough", "slope", "traver", "intensity"]


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype.kind != "f":
        return a == b
    a, b = a.astype(f32), b.astype(f32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _assert_same(g, o, what):
    ok = _same(g, o)
    if not ok.all():
        bad = np.argwhere(~ok.reshape(np.shape(g)))
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {bad.shape[0]} cells differ, first at {i}: gpu={np.asarray(g)[i]!r} "
                             f"oracle={np.asarray(o)[i]!r}")


def _pair(c):
    g = gem_b200.ElevationMap(c.L, c.res, obstacle_threshold=c.obstacle_threshold, compat_box_filter=False)
    o = OracleMap(c.L, c.res, obstacle_threshold=c.obstacle_threshold, compat_box_filter=False)
    for m in (g, o):
        c.apply(m)
    gs, os_ = g.state(), o.state()
    assert np.array_equal(gs[1], os_[1]) and tuple(gs[1]) == c.start, (gs, os_)
    assert np.array_equal(gs[0].view(np.uint32), os_[0].view(np.uint32)) and gs[2] == os_[2] == f32(c.sensor_z)
    return g, o


def _run_untiled(c):
    g, o = _pair(c)
    try:
        fg, fo = g.map_feature(), o.map_feature()
        for name in FEATURE_OUT:
            _assert_same(fg[name], fo[name], f"{c.name} map_feature {name}")
        _assert_same(g.get_layer("traver"), o.get_layer("traver"), f"{c.name} traver layer")
        eg, eo = g.export_layers(), o.export_layers()
        for name in eg:
            _assert_same(eg[name], eo[name], f"{c.name} export_layers {name}")
        for m in (g, o):
            c.apply_ray(m)
            m.raytracing()
        _assert_same(g.get_layer("elevation"), o.get_layer("elevation"), f"{c.name} raytracing elevation")
        _assert_same(g.get_layer("lowest"), o.get_layer("lowest"), f"{c.name} raytracing lowest")
        assert (g.get_layer("lowest") == 10).all()
        gs, os_ = g.state(), o.state()
        assert np.array_equal(gs[0].view(np.uint32), os_[0].view(np.uint32)) and np.array_equal(gs[1], os_[1])
        assert gs[2] == os_[2]
    finally:
        g.close()
        o.close()


CASES = mc.all_cases()


@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_case_untiled(c):
    _run_untiled(c)


def test_long_rays_L1024():
    _run_untiled(mc.long_ray_case())


# ---- tiled handles ---------------------------------------------------------------------------------------------------
TILED = [c for c in CASES if c.tileable and c.L in (200, 66, 34)]


def _tile_layer(t, name, rows, cols):
    import torch
    out = torch.empty((rows, cols), dtype=torch.int32 if name.startswith("color") else torch.float32, device="cuda:0")
    t.get_layer_device(name, out)
    t.sync()
    return out


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("c", TILED, ids=[c.name for c in TILED])
def test_case_tiled(c, world):
    import torch
    L = c.L
    boxes = [tiled.tile_of_rank(r, world, L) for r in range(world)]
    if min(min(b[1], b[3]) for b in boxes) < 2:
        pytest.skip("tiles narrower than 2 cells are outside what border_pack supports")
    o = OracleMap(L, c.res, obstacle_threshold=c.obstacle_threshold, compat_box_filter=False)
    c.apply(o)
    tiles = [gem_b200.ElevationMap(L, c.res, obstacle_threshold=c.obstacle_threshold, compat_box_filter=False, tile=b)
             for b in boxes]
    try:
        sl = lambda a, b: np.ascontiguousarray(a[b[0]:b[0] + b[1], b[2]:b[2] + b[3]])
        for t, b in zip(tiles, boxes):
            t.move(c.position())
            for name in ("elevation", "variance", "traver", "lowest"):
                t.set_layer(name, sl(getattr(c, name), b))
        # features: the 2-cell halo comes from the neighbouring tiles
        elev = [_tile_layer(t, "elevation", b[1], b[3]) for t, b in zip(tiles, boxes)]
        borders = torch.stack([tiled.border_pack(e) for e in elev])
        for r, t in enumerate(tiles):
            t.compute_features_tiled(tiled.padded_from_borders(elev[r], borders, r, world).contiguous())
            t.sync()
        fo = o.map_feature()
        want = {"rough": fo["rough"], "slope": fo["slope"], "traver_out": fo["traver"]}
        for name, full in list(want.items()) + [("traver", o.get_layer("traver"))]:
            full = full.reshape(L, L)
            for r, (t, b) in enumerate(zip(tiles, boxes)):
                _assert_same(_tile_layer(t, name, b[1], b[3]).cpu().numpy(), sl(full, b), f"{c.name} world {world} tile {r} {name}")
        # ray clean-up on the replicated, map-wide lowest layer
        for m in [o] + tiles:
            if c.ray_traver is not None:
                if m is o:
                    o.set_layer("traver", c.ray_traver)
                else:
                    m.set_layer("traver", sl(c.ray_traver, boxes[tiles.index(m)]))
        glob = tiled.global_from_tiles([_tile_layer(t, "lowest", b[1], b[3]) for t, b in zip(tiles, boxes)], world, L)
        assert np.array_equal(glob.cpu().numpy().view(np.uint32), c.lowest.view(np.uint32))
        for t in tiles:
            t.raytracing_tiled(glob)
            t.sync()
        o.raytracing()
        for name in ("elevation", "lowest"):
            full = o.get_layer(name)
            for r, (t, b) in enumerate(zip(tiles, boxes)):
                _assert_same(t.get_layer(name), sl(full, b), f"{c.name} world {world} tile {r} raytracing {name}")
    finally:
        for t in tiles:
            t.close()
        o.close()
