"""The navigation costmaps, CPU side: the oracle (tests/orc_costmap.c) against the independent numpy restatement of
tests/costmap_cases.py, bit for bit (grids, counts, exact double bounds), on every crafted case; the ctypes mirrors of
gem_costmap_window / gem_costmap_marks against the C compiler; the rolling-window helper's bounds and rect arithmetic; the
C++ facade program compiles."""

import numpy as np
import pytest

import costmap_cases as cc
import costmap_oracle
import native
from gem_b200 import costmap

POINTS = cc.point_cases()
MAPS = cc.map_cases()
ROLLS = cc.roll_cases()
COMBINES = cc.combine_cases()


def same_marks(a, b):
    for k in ("marked", "lethal"):
        assert a[k] == b[k], (k, a[k], b[k])
    for k in ("min_x", "min_y", "max_x", "max_y"):
        assert np.float64(a[k]).tobytes() == np.float64(b[k]).tobytes(), (k, a[k], b[k])


@pytest.mark.parametrize("name", [c[0] for c in POINTS])
def test_mark_points_oracle_matches_restatement(name):
    _, rec, w, th, g0 = next(c for c in POINTS if c[0] == name)
    got, gm = costmap_oracle.mark_points(rec, w, g0, th)
    want, wm = cc.np_mark_points(rec, w, g0, th)
    assert np.array_equal(got, want.reshape(got.shape)), name
    same_marks(gm, wm)
    if name == "empty":
        assert gm["marked"] == 0 and gm["min_x"] == np.inf and gm["max_y"] == -np.inf and np.array_equal(got, g0)
    if name == "nonfinite":
        assert gm["marked"] == 2
    if name.startswith("thresh_0.7"):   # 0.7f is below 0.7 and equal to float(0.7f): LETHAL either way; NaN is LETHAL
        assert gm["lethal"] >= 5


@pytest.mark.parametrize("name", [c[0] for c in MAPS])
def test_mark_map_oracle_matches_restatement(name):
    _, tr, L, gres, centre, start, w, th, mu, g0 = next(c for c in MAPS if c[0] == name)
    got, gm = costmap_oracle.mark_map(tr, L, gres, centre, start, w, g0, th, mu)
    want, wm = cc.np_mark_map(tr, L, gres, centre, start, w, g0, th, mu)
    assert np.array_equal(got, want.reshape(got.shape)), name
    same_marks(gm, wm)
    assert gm["marked"] > 0


@pytest.mark.parametrize("name", ["map_L64_w0_unknown_0.7", "map_L50_w0_known_0.7"])
def test_seam_cases_tell_iterator_from_geographic_order(name):
    """the crafted maps whose wrap seam crosses the window give other grids when the last cell in geographic order wins,
    so the iterator-order comparison above is not vacuous"""
    _, tr, L, gres, centre, start, w, th, mu, g0 = next(c for c in MAPS if c[0] == name)
    got, _ = costmap_oracle.mark_map(tr, L, gres, centre, start, w, g0, th, mu)
    geo, _ = cc.np_mark_map(tr, L, gres, centre, start, w, g0, th, mu, geographic=True)
    assert np.count_nonzero(got != geo) > 0


def test_mark_map_last_cell_in_iterator_order_wins():
    """four 0.05 m cells per 0.2 m costmap column: the one latest in GridMapIterator order decides the cell"""
    L, gres = 8, 0.05
    tr = np.full((L, L), 0.9, np.float32)
    tr[:, 3] = 0.1                          # iy = 3 comes after iy = 0..2 in iterator order
    w = (-0.2, -0.2, 0.2, 2, 2)
    g, m = costmap_oracle.mark_map(tr, L, gres, (0.0, 0.0), (0, 0), w, np.full((2, 2), 255, np.uint8), 0.5)
    want, _ = cc.np_mark_map(tr, L, gres, (0.0, 0.0), (0, 0), w, np.full((2, 2), 255, np.uint8), 0.5)
    assert np.array_equal(g, want) and m["marked"] == L * L


@pytest.mark.parametrize("name", [c[0] for c in ROLLS])
def test_update_origin_oracle_matches_restatement(name):
    _, w, seq, fill, g0 = next(c for c in ROLLS if c[0] == name)
    wo, go, wn, gn = w, g0, w, g0
    for nx, ny in seq:
        wo, go = costmap_oracle.update_origin(wo, nx, ny, fill, go)
        wn, gn = cc.np_update_origin(wn, nx, ny, fill, gn)
        assert np.float64(wo[:3]).tobytes() == np.float64(wn[:3]).tobytes(), (name, wo, wn)
        assert np.array_equal(go, gn), name
    if name == "fractional_half_cell":
        assert wo == w and np.array_equal(go, g0)
    if name == "200_rolls":   # the window follows the robot in whole cells
        assert wo[0] != w[0] and abs(wo[0] - (seq[-1][0])) < w[2]


def test_update_origin_defined_errors():
    w = (0.0, 0.0, 0.2, 4, 4)
    g = np.arange(16, dtype=np.uint8).reshape(4, 4)
    for nx, ny in [(np.nan, 0.0), (0.0, np.inf), (0.2 * 2.0 ** 31 + 1.0, 0.0)]:
        assert costmap_oracle.update_origin(w, nx, ny, 0, g) is None
        assert cc.np_update_origin(w, nx, ny, 0, g) is None


@pytest.mark.parametrize("name", [c[0] for c in COMBINES])
def test_combine_oracle_matches_restatement(name):
    _, mode, lay, mas, sx, sy, rect = next(c for c in COMBINES if c[0] == name)
    got = costmap_oracle.combine(mode, lay, mas, sx, sy, rect)
    want = cc.np_combine(mode, lay, mas, sx, sy, rect)
    assert np.array_equal(got, want), name
    if name.startswith("empty"):
        assert np.array_equal(got, mas)


def test_update_rect_arithmetic():
    w = (-7.5, 3.0, 0.2, 75, 75)
    inf = float("inf")
    # nothing marked: the bounds stay at +-1e30 and the reference returns before resetting anything
    assert costmap.update_rect(w, {"min_x": inf, "min_y": inf, "max_x": -inf, "max_y": -inf}) is None
    # below the origin -> 0; at origin + res * size -> size - 1, then + 1
    r = costmap.update_rect(w, {"min_x": -100.0, "min_y": 2.0, "max_x": -7.5 + 0.2 * 75, "max_y": 1e9})
    assert r == (0, 0, 75, 75)
    # inside: truncated quotients, the upper one + 1
    r = costmap.update_rect(w, {"min_x": -7.5 + 0.2 * 3.5, "min_y": 3.0 + 0.2 * 10.0, "max_x": -7.5 + 0.2 * 9.99,
                                "max_y": 3.0 + 0.2 * 10.0})
    assert r == (3, int((3.0 + 0.2 * 10.0 - 3.0) / 0.2), 10, int((3.0 + 0.2 * 10.0 - 3.0) / 0.2) + 1)
    # one point: a 1 x 1 rect
    x = -7.5 + 0.2 * 20.5
    assert costmap.update_rect(w, {"min_x": x, "min_y": 3.1, "max_x": x, "max_y": 3.1}) == (20, 0, 21, 1)
    assert costmap.world_to_map_enforce_bounds(w, float("-inf"), float("inf")) == (0, 74)


def test_size_in_meters_and_roll_target():
    """getSizeInMetersX = (size_x - 1 + 0.5) * resolution; the rolling origin is robot - that / 2"""
    cm = costmap.Costmap.__new__(costmap.Costmap)
    cm.window = (0.0, 0.0, 0.2, 75, 1000)
    assert cm.size_in_meters() == ((75 - 1 + 0.5) * 0.2, (1000 - 1 + 0.5) * 0.2)


def test_costmap_structs_match_the_header():
    import gem_b200._lib as L
    consts = {"GEM_COST_FREE": L.COST_FREE, "GEM_COST_LETHAL": L.COST_LETHAL, "GEM_COST_UNKNOWN": L.COST_UNKNOWN,
              "GEM_COSTMAP_MAX": L.COSTMAP_MODES["max"], "GEM_COSTMAP_OVERWRITE": L.COSTMAP_MODES["overwrite"]}
    native.assert_struct_layouts({"gem_costmap_window": L.GemCostmapWindow, "gem_costmap_marks": L.GemCostmapMarks}, consts)


def test_facade_program_with_costmaps_compiles():
    native.facade_compiles("costmap_smoke")
