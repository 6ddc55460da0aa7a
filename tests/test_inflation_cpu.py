"""InflationLayer (DESIGN.md f14) on the host: the oracle tests/orc_inflate.c bit for bit against the independent Python
restatement of tests/inflation_oracle.py on every crafted case, the witnesses shown to be witnesses, the footprint's
inscribed radius, the bounds sequence of InflationLayer.update_bounds, Costmap.update without inflation unchanged, and
the ctypes struct against the C compiler."""

import numpy as np
import pytest

import inflation_cases as ic
import inflation_oracle as O
import native
from gem_b200 import costmap

CASES = {c[0]: c for c in ic.all_cases()}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_restatement(name):
    _, g, res, p, rect = CASES[name]
    got = O.inflate(g, res, p, rect)
    assert np.array_equal(got, O.brushfire(g, res, p, rect)), name


def test_crafted_cases_reach_their_rule():
    changed = {n: int((O.inflate(g, res, p, rect) != g).sum()) for n, g, res, p, rect in ic.crafted()}
    for n in ("radius_zero", "rect_beyond", "single_cell", "all_lethal", "no_lethal"):
        assert changed[n] == 0, n
    for n in ("inscribed_exact", "weight_zero", "unknown_master", "widening_seeds", "clamped_corners",
              "propagation_leaves_rect", "row", "column", "unknown_master_weight_high"):
        assert changed[n] > 0, n
    _, g, res, p, rect = CASES["inscribed_exact"]
    out = O.inflate(g, res, p, rect)
    assert out[5, 7] == 253 and out[5, 3] == 253 and out[6, 7] < 253        # distance 2 at the edge; sqrt(5) beyond it
    _, g, res, p, rect = CASES["weight_zero"]
    out = O.inflate(g, res, p, rect)
    assert out[5, 7] == 252 and out[5, 6] == 253                            # 252 beyond the inscribed radius
    _, g, res, p, rect = CASES["truncation_half"]
    assert O.inflate(g, res, p, rect)[6, 9] in (125, 126)                   # 252 * exp(-ln 2) at the truncation
    a = O.inflate(*CASES["unknown_master"][1:])
    b = O.inflate(*CASES["unknown_master_inflated"][1:])
    assert not np.array_equal(a, b) and ((a == 255) & (b != 255)).any()
    _, g, res, p, rect = CASES["widening_seeds"]
    out = O.inflate(g, res, p, rect)
    assert out[3, 4] == 0 and out[3, 3] == 254 and out[10, 5] > 0 and out[10, 14] > 0   # (3, 3) is beyond the widening
    _, g, res, p, rect = CASES["propagation_leaves_rect"]
    assert (O.inflate(g, res, p, rect)[:, :12] > 0).any()


@pytest.mark.parametrize("seed", ic.ORDER_WITNESSES)
def test_order_witnesses(seed):
    _, g, res, p, rect = ic.witness(seed)
    assert not np.array_equal(O.inflate(g, res, p, rect), O.brushfire(g, res, p, rect, reverse=True))


@pytest.mark.parametrize("seed", ic.EDT_WITNESSES)
def test_edt_witnesses(seed):
    _, g, res, p, rect = ic.witness(seed)
    assert not np.array_equal(O.inflate(g, res, p, rect), O.nearest_obstacle(g, res, p, rect))


def test_random_grids_oracle_equals_restatement():
    for seed in range(40):
        rng = np.random.default_rng(seed)
        sy, sx = int(rng.integers(1, 24)), int(rng.integers(1, 24))
        g = ic.random_grid(seed, sy, sx, float(rng.choice([0.02, 0.1, 0.3, 0.5])), unknown=float(rng.choice([0.0, 0.2])))
        p = O.params(float(rng.uniform(0.0, 1.0)), float(rng.uniform(0.0, 15.0)), float(rng.uniform(0.0, 0.3)),
                     bool(rng.integers(0, 2)))
        rect = tuple(int(v) for v in (rng.integers(-3, sx), rng.integers(-3, sy), rng.integers(0, sx + 3), rng.integers(0, sy + 3)))
        assert np.array_equal(O.inflate(g, 0.1, p, rect), O.brushfire(g, 0.1, p, rect)), seed


def test_inscribed_radius_of_footprints():
    assert costmap.inscribed_radius(costmap.GEM_FOOTPRINT) == 0.4
    assert abs(costmap.inscribed_radius(costmap.GEM_FOOTPRINT, 0.01) - 0.41) < 1e-15
    assert abs(costmap.inscribed_radius(costmap.GEM_FOOTPRINT, 0.1) - 0.5) < 1e-15
    # an off-centre triangle: the nearest edge is the one the origin projects onto inside it
    tri = ((-0.2, -0.5), (0.9, -0.5), (-0.2, 0.6))
    assert abs(costmap.inscribed_radius(tri) - 0.2) < 1e-15
    # a segment whose projection parameter leaves [0, 1]: the vertex is nearer
    sq = ((0.3, 0.3), (1.0, 0.3), (1.0, 1.0), (0.3, 1.0))
    assert costmap.inscribed_radius(sq) == float(np.hypot(0.3, 0.3))
    assert costmap.inscribed_radius(((0.1, 0.1), (0.2, 0.2))) == 1.7976931348623157e308


def test_bounds_sequence():
    lay = costmap.InflationLayer(0.55, 10.0, 0.4)
    F = costmap.FLT_MAX
    assert lay.update_bounds((1.0, 2.0, 3.0, 4.0)) == (-F, -F, F, F)                  # first update: the whole grid
    assert lay.update_bounds((0.5, 2.5, 2.0, 5.0)) == (0.5 - 0.55, 2.0 - 0.55, 3.0 + 0.55, 5.0 + 0.55)
    assert lay.update_bounds((1e30, 1e30, -1e30, -1e30)) == (0.5 - 0.55, 2.5 - 0.55, 2.0 + 0.55, 5.0 + 0.55)
    assert lay.update_bounds((7.0, 7.0, 8.0, 8.0)) == (7.0 - 0.55, 7.0 - 0.55, 8.0 + 0.55, 8.0 + 0.55)
    lay.set_parameters(0.55, 10.0, 0.4)                                                # unchanged: no re-inflation
    assert lay.update_bounds((7.0, 7.0, 8.0, 8.0)) == (7.0 - 0.55, 7.0 - 0.55, 8.0 + 0.55, 8.0 + 0.55)
    lay.set_parameters(1.0, 10.0, 0.4)
    assert lay.update_bounds((3.0, 3.0, 4.0, 4.0)) == (-F, -F, F, F)
    assert lay.update_bounds((3.5, 2.0, 4.0, 4.5)) == (3.0 - 1.0, 2.0 - 1.0, 4.0 + 1.0, 4.5 + 1.0)
    w = (0.0, 0.0, 0.2, 100, 50)
    assert costmap.update_rect(w, dict(zip(("min_x", "min_y", "max_x", "max_y"), (-F, -F, F, F)))) == (0, 0, 100, 50)


class _FakeMap:
    """records the library calls Costmap.update makes (no device needed)"""

    def __init__(self):
        self.calls = []

    def costmap_update_origin(self, window, ox, oy, fill, grid):
        self.calls.append(("roll",))
        return window

    def costmap_combine(self, mode, layer, master, sx, sy, rect):
        self.calls.append(("combine", mode, rect))

    def costmap_inflate(self, window, params, master, rect):
        self.calls.append(("inflate", params["inflation_radius"], rect))

    def torch_stream(self):
        return None


def _costmaps(fake):
    import torch
    out = []
    for fill in (0, 255):
        c = costmap.Costmap.__new__(costmap.Costmap)
        c.emap, c.window, c.fill = fake, (0.0, 0.0, 0.2, 50, 40), fill
        c.grid = torch.zeros((40, 50), dtype=torch.uint8)
        out.append(c)
    return out


def test_update_without_inflation_and_radius_zero(monkeypatch):
    import torch
    monkeypatch.setattr(torch.cuda, "stream", lambda s: __import__("contextlib").nullcontext())
    marks = {"marked": 3, "lethal": 1, "min_x": 1.0, "min_y": 2.0, "max_x": 3.0, "max_y": 4.0}
    fake = _FakeMap()
    master, layer = _costmaps(fake)
    rect, m = master.update(layer, (5.0, 4.0), "overwrite", lambda l: marks)
    assert rect == costmap.update_rect(master.window, marks) == (5, 10, 16, 21) and m is marks
    assert fake.calls == [("roll",), ("roll",), ("combine", "overwrite", rect)]
    rect0, _ = master.update(layer, (5.0, 4.0), "overwrite", lambda l: marks, inflation=None)
    assert rect0 == rect
    # with the layer: its first update re-inflates the whole grid, later ones widen by the radius
    fake.calls.clear()
    lay = costmap.InflationLayer(0.0, 10.0, 0.4)
    rect1, _ = master.update(layer, (5.0, 4.0), "overwrite", lambda l: marks, inflation=lay)
    assert rect1 == (0, 0, 50, 40) and fake.calls[-1] == ("inflate", 0.0, rect1)
    rect2, _ = master.update(layer, (5.0, 4.0), "overwrite", lambda l: marks, inflation=lay)
    assert rect2 == rect and fake.calls[-1] == ("inflate", 0.0, rect)


def test_inflation_struct_matches_the_header():
    import gem_b200._lib as L
    native.assert_struct_layouts({"gem_costmap_inflation": L.GemCostmapInflation})


def test_facade_program_with_inflation_compiles():
    native.facade_compiles("inflation_smoke")
