"""The table bound of gem_costmap_inflate (GEM_INFLATE_MAX_CELLS, DESIGN.md f14) in the ctypes module against the C
compiler's view of the header."""
import native


def test_table_bound_matches_the_header():
    import gem_b200._lib as L
    assert native.c_values(["GEM_INFLATE_MAX_CELLS"]) == {"GEM_INFLATE_MAX_CELLS": L.INFLATE_MAX_CELLS}
