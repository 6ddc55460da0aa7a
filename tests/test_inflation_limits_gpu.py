"""gem_costmap_inflate (DESIGN.md f14) at its limits, byte for byte against the oracle tests/orc_inflate.c: the radius
bound GEM_INFLATE_MAX_CELLS, and one handle whose cached tables and key buffer are replaced as the parameters and grid
sizes change."""
import numpy as np
import pytest
import torch

import inflation_cases as ic
import inflation_oracle as O
import gem_b200
from gem_b200 import _lib

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def run(emap, g, res, p, rect):
    grid = dev(g)
    emap.costmap_inflate((0.0, 0.0, float(res), int(g.shape[1]), int(g.shape[0])), p, grid, rect)
    emap.sync()
    return grid.cpu().numpy()


def test_radius_above_the_table_bound_is_refused():
    """r above GEM_INFLATE_MAX_CELLS (after the diagonal cap) is GEM_ERR_INVALID and writes nothing; the bound itself works"""
    g = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)
    n = 3000
    g0 = np.zeros((n, n), np.uint8)
    g0[1500, 1500] = 254
    grid = dev(g0)
    w = (0.0, 0.0, 0.01, n, n)
    with pytest.raises(gem_b200.GemError, match="GEM_INFLATE_MAX_CELLS"):
        g.costmap_inflate(w, O.params(0.01 * (_lib.INFLATE_MAX_CELLS + 1), 1.0, 0.0), grid, (0, 0, n, n))
    g.sync()
    assert torch.equal(grid, dev(g0))
    small = ic.random_grid(11, 40, 50, 0.05)
    p = O.params(0.01 * _lib.INFLATE_MAX_CELLS, 1.0, 0.0)   # capped at the small grid's diagonal
    assert np.array_equal(run(g, small, 0.01, p, (0, 0, 50, 40)), O.inflate(small, 0.01, p, (0, 0, 50, 40)))


def test_tables_follow_parameter_changes():
    """alternating radii and weights on one handle, with the tables and the key buffer regrown in between"""
    g = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)
    for k, (radius, weight, n) in enumerate(((0.3, 10.0, 50), (4.0, 2.0, 90), (0.3, 10.0, 400), (4.0, 2.0, 90),
                                             (4.0, 3.0, 90), (0.3, 10.0, 800), (0.3, 10.0, 60))):
        gr = ic.random_grid(900 + k, n, n + 7, 0.03, unknown=0.1)
        p = O.params(radius, weight, 0.15, bool(k & 1))
        assert np.array_equal(run(g, gr, 0.1, p, (2, 3, n, n - 5)), O.inflate(gr, 0.1, p, (2, 3, n, n - 5))), k
