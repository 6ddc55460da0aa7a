"""Crafted cases of gem_costmap_inflate (DESIGN.md f14): one small grid per rule, and the witness grids on which the
order inside a bin (ORDER_WITNESSES) or the brushfire's propagated sources (EDT_WITNESSES) decide bytes.

A case is (name, grid, resolution, params, rect)."""
from __future__ import annotations

import math

import numpy as np

from inflation_oracle import FREE, LETHAL, UNKNOWN, params


def _grid(sy, sx, fill=FREE, lethal=(), unknown=()):
    g = np.full((sy, sx), fill, np.uint8)
    for i, j in lethal:
        g[j, i] = LETHAL
    for i, j in unknown:
        g[j, i] = UNKNOWN
    return g


def random_grid(seed, sy, sx, density, unknown=0.0):
    rng = np.random.default_rng(seed)
    u = rng.random((sy, sx))
    g = rng.integers(0, 120, (sy, sx)).astype(np.uint8)      # some costs below the inflated ones
    g[u < unknown] = UNKNOWN
    g[u > 1.0 - density] = LETHAL
    return g


def crafted():
    cases = []
    full = lambda g: (0, 0, g.shape[1], g.shape[0])   # noqa: E731
    g = _grid(9, 9, lethal=[(4, 4)])
    cases.append(("radius_zero", g, 0.2, params(0.0), full(g)))
    cases.append(("radius_below_one_cell", g, 0.2, params(0.05), full(g)))
    # dist * res == inscribed exactly: at res 0.5 and inscribed 1.0 the cells at distance 2 are 253, sqrt(5) is not
    g = _grid(11, 11, lethal=[(5, 5)])
    cases.append(("inscribed_exact", g, 0.5, params(2.0, 3.0, 1.0), full(g)))
    cases.append(("weight_zero", g, 0.5, params(2.5, 0.0, 0.5), full(g)))
    # the factor lands on 0.5 at distance 3 (252 * 0.5 = 126), with the truncations around it
    g = _grid(13, 13, lethal=[(6, 6)])
    cases.append(("truncation_half", g, 0.1, params(0.6, math.log(2.0) / (0.3 - 0.1), 0.1), full(g)))
    cases.append(("truncation_steep", g, 0.05, params(0.3, 37.0, 0.0), full(g)))
    # NO_INFORMATION masters: inflated only at >= 253, or at > FREE with inflate_unknown
    g = _grid(12, 12, fill=UNKNOWN, lethal=[(3, 3), (8, 7)])
    g[0:4, 6:12] = FREE
    cases.append(("unknown_master", g, 0.1, params(0.5, 4.0, 0.15), full(g)))
    cases.append(("unknown_master_inflated", g, 0.1, params(0.5, 4.0, 0.15, unknown=True), full(g)))
    cases.append(("unknown_master_weight_high", g, 0.1, params(0.5, 20.0, 0.0, unknown=True), full(g)))
    # lethal cells just outside the rect but inside the widening (r = 3), and one beyond it
    g = _grid(20, 20, lethal=[(4, 10), (15, 10), (10, 3), (10, 16), (3, 3)])
    cases.append(("widening_seeds", g, 0.1, params(0.3, 5.0, 0.1), (7, 7, 13, 13)))
    # widening clamped at every edge, and rects partly or wholly outside the grid
    g = _grid(10, 14, lethal=[(0, 0), (13, 0), (0, 9), (13, 9), (6, 5)])
    cases.append(("clamped_corners", g, 0.1, params(0.4, 3.0, 0.1), (1, 1, 13, 9)))
    cases.append(("rect_outside", g, 0.1, params(0.4, 3.0, 0.1), (-50, -50, 100, 100)))
    cases.append(("rect_empty", g, 0.1, params(0.4, 3.0, 0.1), (5, 5, 5, 8)))
    cases.append(("rect_beyond", g, 0.1, params(0.4, 3.0, 0.1), (40, 40, 50, 50)))
    # propagation leaves the rect: a seed in a tiny rect writes the whole radius around it
    g = _grid(25, 25, lethal=[(12, 12)])
    cases.append(("propagation_leaves_rect", g, 0.1, params(0.9, 2.0, 0.2), (12, 12, 13, 13)))
    # 1 x N and N x 1
    g = _grid(1, 30, lethal=[(3, 0), (17, 0), (18, 0)])
    cases.append(("row", g, 0.1, params(0.7, 3.0, 0.2), full(g)))
    g = _grid(30, 1, lethal=[(0, 0), (0, 29), (0, 11)])
    cases.append(("column", g, 0.1, params(0.7, 3.0, 0.2), full(g)))
    g = _grid(1, 1, lethal=[(0, 0)])
    cases.append(("single_cell", g, 0.1, params(0.5), full(g)))
    g = np.full((7, 9), LETHAL, np.uint8)
    cases.append(("all_lethal", g, 0.1, params(0.3), full(g)))
    g = random_grid(3, 10, 12, 0.0)
    g[g == LETHAL] = 0
    cases.append(("no_lethal", g, 0.1, params(0.5), full(g)))
    # the radius beyond the grid's diagonal (capped) and a master with mixed costs
    g = random_grid(4, 6, 8, 0.1, unknown=0.2)
    cases.append(("radius_beyond_diagonal", g, 0.1, params(100.0, 1.0, 0.0), full(g)))
    cases.append(("mixed_master", random_grid(5, 16, 16, 0.08, unknown=0.1), 0.1, params(0.6, 2.0, 0.15), (2, 3, 11, 14)))
    return cases


# Random grids on which walking each bin backwards changes bytes (order witnesses) and on which the exact nearest-seed
# cost differs from the brushfire's (EDT witnesses).  Found once with the restatements of inflation_oracle.py; the CPU
# suite shows that each still is one.
def witness(seed):
    rng = np.random.default_rng(1000 + seed)
    sy, sx = int(rng.integers(6, 20)), int(rng.integers(6, 20))
    g = random_grid(seed, sy, sx, float(rng.choice([0.03, 0.08, 0.15])))
    r = int(rng.integers(2, 8))
    return (f"witness_{seed}", g, 0.1, params(0.1 * r - 0.01, 1.5, 0.05), (0, 0, sx, sy))


ORDER_WITNESSES = [20, 116, 129, 138, 160, 165]
EDT_WITNESSES = [15, 23, 31, 50, 92, 107]


def all_cases():
    return crafted() + [witness(s) for s in sorted(set(ORDER_WITNESSES + EDT_WITNESSES))]
