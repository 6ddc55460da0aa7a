"""The costmap topics and the footprint clearing without a GPU (DESIGN.md f17): T against its formula, the struct encoder of
tests/costmap_pub_oracle.py against its decoder and the stated sizes, the library's host code (gem_rosfmt.h W9-W11 and
P1-P4, gem_footprint.h F1-F4, built with g++) against the encoder, the publisher restatement and the two footprint
oracles, and the gem_costmap_publisher layout against the C compiler."""
import ctypes as C
import math

import numpy as np
import pytest

import costmap_pub_oracle as cp
import native
import rosmsg_oracle as ro
from gem_b200 import _lib

SIZES = [(1, 1), (1, 37), (41, 1), (75, 75), (257, 33), (1000, 1000)]
FRAME_ID_LENGTHS = list(range(21)) + [300]


def frame_id(n):
    return ("odom/" * 80)[:n].encode()


def hdr(fl, seq=3):
    fid = frame_id(fl)
    return (seq, 1700000000 + fl, 1000 * fl, fid), ro.header(seq, 1700000000 + fl, 1000 * fl, fid)


def all_costs_grid(sx, sy, seed):
    """every cost value 0-255 where the grid has room, the rest random"""
    g = np.random.default_rng(seed).integers(0, 256, sx * sy, dtype=np.uint8)
    g[:min(256, g.size)] = np.arange(min(256, g.size), dtype=np.uint8)
    return g.reshape(sy, sx)


def test_translation_table():
    lib = cp.host()
    for c in range(256):
        want = 0 if c == 0 else 99 if c == 253 else 100 if c == 254 else -1 if c == 255 else 1 + (97 * (c - 1)) // 251
        assert cp.translate(c) == want == lib.cp_translate(c) == int(cp.TABLE[c]), c
    assert cp.TABLE[1] == 1 and cp.TABLE[252] == 98 and set(cp.TABLE[1:253]) == set(range(1, 99))


@pytest.mark.parametrize("size", SIZES)
def test_full_grid_encode_decode_and_host(size):
    sx, sy = size
    grid = all_costs_grid(sx, sy, sx * 7 + sy)
    window = (-12.3 + sx, 4.56 - sy, 0.05, sx, sy)
    for fl in FRAME_ID_LENGTHS if sx * sy < 10**5 else (0, 7, 20, 300):
        h, hb = hdr(fl)
        msg = cp.occupancy_grid(hb, window, grid)
        assert len(msg) == cp.size_grid(fl, sx, sy)
        assert msg[92 + fl:96 + fl] == np.uint32(sx * sy).tobytes()        # the int8[] field: its count, then the bytes
        assert msg[96 + fl:] == cp.TABLE[grid.reshape(-1)].tobytes()
        d = cp.decode_occupancy_grid(msg)
        assert d["header"] == {"seq": 3, "stamp": (h[1], h[2]), "frame_id": h[3]} and d["map_load_time"] == (0, 0)
        assert d["resolution"] == np.float32(0.05) and (d["width"], d["height"]) == (sx, sy)
        assert d["position"] == (window[0] + 0.5 * 0.05 - 0.05 / 2, window[1] + 0.5 * 0.05 - 0.05 / 2, 0.0)
        assert d["orientation"] == (0.0, 0.0, 0.0, 1.0) and d["data"].tobytes() == cp.TABLE[grid.reshape(-1)].tobytes()
        kind, rect, got = cp.HostPublisher().publish(h, window, grid)
        assert (kind, rect) == ("full", (0, 0, sx, sy)) and got == msg


@pytest.mark.parametrize("size", SIZES)
def test_updates_encode_decode_and_host(size):
    sx, sy = size
    grid = all_costs_grid(sx, sy, sx + 3 * sy)
    window = (1.0, 2.0, 0.2, sx, sy)
    rects = {(0, 0, sx, sy), (0, 0, 1, 1), (sx - 1, sy - 1, 1, 1), (0, sy // 2, sx, 1), (sx // 3, 0, sx - sx // 3, sy),
             (0, 0, sx, 0), (sx // 2, sy, sx - sx // 2, 0), (min(5, sx - 1), 0, min(17, sx - min(5, sx - 1)), min(3, sy))}
    for fl in (0, 1, 13, 20, 300):
        h, hb = hdr(fl)
        for x, y, w, hh in sorted(rects):
            if w == 0:
                continue
            msg = cp.grid_update(hb, x, y, w, hh, grid)
            assert len(msg) == cp.size_update(fl, w, hh)
            d = cp.decode_grid_update(msg)
            assert (d["x"], d["y"], d["width"], d["height"]) == (x, y, w, hh)
            assert np.array_equal(d["data"].reshape(hh, w), cp.TABLE[grid[y:y + hh, x:x + w]])
            pub = cp.HostPublisher()
            assert pub.publish(h, window, grid)[0] == "full"
            pub.bounds(x, x + w, y, y + hh)
            kind, rect, got = pub.publish(h, window, grid)
            assert (kind, rect) == ("update", (x, y, w, hh)) and got == msg


def test_full_origin_not_bit_equal_to_the_window_origin():
    """W9's origin is (origin + 0.5 res) - res / 2 in double: not always the origin's bits"""
    found = None
    for k in range(1, 2000):
        ox = 0.1 * k + 1e-3
        if (ox + 0.5 * 0.15) - 0.15 / 2 != ox:
            found = ox
            break
    assert found is not None
    window = (found, -found, 0.15, 75, 75)
    grid = all_costs_grid(75, 75, 1)
    h, hb = hdr(4)
    d = cp.decode_occupancy_grid(cp.HostPublisher().publish(h, window, grid)[2])
    assert d["position"][0] == (found + 0.5 * 0.15) - 0.15 / 2 != found
    assert d["position"][0] == cp.decode_occupancy_grid(cp.occupancy_grid(hb, window, grid))["position"][0]


@pytest.mark.parametrize("fl", [0, 5, 20, 300])
def test_footprint_message_encode_decode_and_host(fl):
    h, hb = hdr(fl, seq=0)
    for fp in (cp.GEM_FOOTPRINT, [], [(0.3, -0.2)], [(1e-3 * k, math.sin(k)) for k in range(40)]):
        for rx, ry, yaw in ((0.0, 0.0, 0.0), (12.345, -6.7, 1.2345), (-100.1, 55.5, -3.0)):
            verts = cp.transform(fp, rx, ry, yaw)
            msg = cp.polygon_stamped(hb, verts)
            assert len(msg) == cp.size_polygon(fl, len(fp))
            d = cp.decode_polygon_stamped(msg)
            assert d["points"] == [(float(np.float32(x)), float(np.float32(y)), 0.0) for x, y in verts]
            assert cp.host_footprint_msg(h, fp, rx, ry, yaw) == msg


# ---- the footprint ----------------------------------------------------------------------------------------------------
LOCAL = (-7.45, -7.45, 0.2, 75, 75)


def footprint_cases():
    out = []
    for k in range(24):                                   # GEM's rectangle at yaws over [0, 2 pi), positions +- half a cell
        for dx, dy in ((0.0, 0.0), (0.1, 0.0), (-0.1, 0.1), (0.1, -0.1)):
            out.append((f"gem_yaw{k}_{dx}_{dy}", LOCAL, cp.GEM_FOOTPRINT, 0.03 + dx, -0.02 + dy, 2 * math.pi * k / 24))
    out += [
        ("vertex_on_cell_edge", LOCAL, [(0.0, 0.0), (0.6, 0.0), (0.6, 0.4)], 0.05, 0.05, 0.0),
        ("vertex_on_window_edge", (0.0, 0.0, 0.25, 20, 20), [(0.0, 0.0), (1.0, 0.0), (1.0, 1.0)], 0.0, 0.0, 0.0),
        ("vertex_outside", LOCAL, cp.GEM_FOOTPRINT, 7.0, 0.0, 0.3),
        ("vertex_below_origin", LOCAL, cp.GEM_FOOTPRINT, -7.0, 0.0, 0.0),
        ("two_vertices", LOCAL, [(-0.5, 0.0), (0.5, 0.2)], 0.0, 0.0, 0.4),
        ("one_vertex", LOCAL, [(0.1, 0.1)], 0.0, 0.0, 0.0),
        ("no_vertex", LOCAL, [], 0.0, 0.0, 0.0),
        ("collinear", LOCAL, [(-1.0, -0.5), (0.0, 0.0), (1.0, 0.5)], 0.0, 0.0, 0.0),
        ("collinear_vertical", LOCAL, [(0.0, -1.0), (0.0, 0.0), (0.0, 1.3)], 0.01, 0.0, 0.0),
        ("degenerate_point", LOCAL, [(0.0, 0.0)] * 3, 0.01, 0.01, 0.0),
        ("thin_diagonal", LOCAL, [(-1.5, -1.0), (1.5, 1.1), (1.5, 1.25)], 0.0, 0.0, 0.0),
        ("thin_steep", LOCAL, [(-0.1, -2.0), (0.15, 2.0), (0.3, 2.0)], 0.0, 0.0, 0.0),
        ("skewed_quad", LOCAL, [(-2.0, -0.3), (-1.0, 0.1), (2.0, 0.9), (1.0, 0.2)], 0.0, 0.0, 0.2),
        ("triangle_single_columns", LOCAL, [(-1.0, 0.0), (1.0, 0.9), (1.05, -0.9)], 0.0, 0.0, 0.0),
        ("pentagon", LOCAL, [(1.0, 0.0), (0.3, 0.95), (-0.8, 0.6), (-0.8, -0.6), (0.3, -0.95)], 0.2, -0.3, 0.7),
        ("large", (0.0, 0.0, 0.2, 300, 300), [(-20, -10), (25, -12), (18, 22), (-15, 19)], 30.0, 30.0, 0.1),
    ]
    rng = np.random.default_rng(17)
    for k in range(60):                                    # random thin and skewed triangles and quads
        n = 3 + k % 2
        pts = [(float(x), float(y)) for x, y in rng.uniform(-2.5, 2.5, (n, 2)) * (1.0, rng.uniform(0.05, 1.0))]
        out.append((f"random{k}", LOCAL, pts, float(rng.uniform(-1, 1)), float(rng.uniform(-1, 1)), float(rng.uniform(0, 6.3))))
    return out


@pytest.mark.parametrize("case", footprint_cases(), ids=lambda c: c[0])
def test_footprint_cells_three_ways(case):
    name, window, fp, rx, ry, yaw = case
    pv, pc = cp.footprint_cells(window, fp, rx, ry, yaw)
    ov, oc = cp.orc_footprint_cells(window, fp, rx, ry, yaw)
    hv, hc = cp.host_footprint_cells(window, fp, rx, ry, yaw)
    assert np.array(pv, np.float64).tobytes() == np.array(ov, np.float64).tobytes() == np.array(hv, np.float64).tobytes()
    assert pc == oc == hc, name
    if name.startswith("vertex_outside") or name == "vertex_below_origin":
        assert pc is None
    if name in ("two_vertices", "one_vertex", "no_vertex"):
        assert pc == []
    if name.startswith("gem_yaw"):
        assert len(set(pc)) >= 20        # the 1.28 m x 0.80 m rectangle covers about 26 cells of 0.2 m


def test_footprint_fill_is_the_column_fill_of_the_outline():
    """through raytraceLine's closed outline every column holds two cells or more, so the walk's pairing stays inside a
    column and the literal fill is every cell between each column's lowest and highest outline cell"""
    for name, window, fp, rx, ry, yaw in footprint_cases():
        _, cells = cp.footprint_cells(window, fp, rx, ry, yaw)
        if cells:
            ol = cp.outline(window, fp, rx, ry, yaw)
            assert min(np.unique([c[0] for c in ol], return_counts=True)[1]) >= 2, name
            assert set(cells) == cp.true_fill(ol), name


def test_column_walk_quirk_on_crafted_lists():
    """F4 on lists with a column of one cell: the pairing runs across columns and pairs appended cells, so the literal
    result differs from the column fill; the C oracle, the library's header and the Python restatement agree"""
    cases = [[(0, 5), (1, 2), (1, 7), (2, 3), (2, 4)], [(3, 1), (4, 9), (4, 0), (5, 5), (6, 2), (6, 8), (7, 4)],
             [(0, 0), (2, 6), (2, 1)], [(5, 5)], [], [(1, 1), (1, 1)], [(2, 9), (0, 3), (1, 0), (0, 8)]]
    rng = np.random.default_rng(3)
    cases += [[(int(x), int(y)) for x, y in rng.integers(0, 12, (int(rng.integers(1, 30)), 2))] for _ in range(200)]
    differ = 0
    for cells in cases:
        o, h = cp.walk_both(cells)
        assert o == h == cp.column_walk(list(cells)), cells
        differ += bool(cells) and set(o) != cp.true_fill(cells)
    assert cp.column_walk([(0, 5), (1, 2), (1, 7), (2, 3), (2, 4)])[5:] == [(0, 2), (0, 3), (0, 4), (1, 3), (1, 4), (1, 5),
                                                                          (1, 6), (2, 2), (2, 3)]
    assert differ >= 100


def test_footprint_on_a_cell_edge_maps_up():
    """worldToMap truncates: a vertex exactly on the line between cells 3 and 4 falls in cell 4"""
    w = (0.0, 0.0, 0.25, 20, 20)
    assert cp.to_map(w, 1.0, 0.5) == (4, 2)
    _, cells = cp.host_footprint_cells(w, [(1.0, 0.5), (2.0, 0.5), (2.0, 1.5)], 0.0, 0.0, 0.0)
    assert min(c[0] for c in cells) == 4 and min(c[1] for c in cells) == 2


# ---- the publisher ----------------------------------------------------------------------------------------------------
def run_sequence(steps, always=False):
    """steps: ("bounds", x0, xn, y0, yn) | ("publish", window) | ("force", window) | ("query", window) | ("small", window);
    the library's host publisher and the restatement side by side; returns the kinds"""
    lib, py = cp.HostPublisher(always), cp.Publisher(always)
    kinds = []
    h = (0, 0, 0, b"map")
    for st in steps:
        if st[0] == "bounds":
            lib.bounds(*st[1:])
            py.bounds(*st[1:])
            continue
        window = st[1]
        grid = all_costs_grid(window[3], window[4], 5)
        before = lib.state()
        if st[0] in ("query", "small"):
            kind, rect, n = lib.publish(h, window, grid, query=st[0] == "query", capacity=None if st[0] == "query" else 10)
            assert lib.state() == before, st
            assert isinstance(n, int) and n >= 0
            kinds.append("kept")
            continue
        kind, rect, msg = lib.publish(h, window, grid, force_full=st[0] == "force")
        want = py.publish(window, force_full=st[0] == "force")
        assert (kind, rect) == want, (st, kind, rect, want)
        assert (lib.s.x0, lib.s.xn, lib.s.y0, lib.s.yn) == (py.x0, py.xn, py.y0, py.yn)
        if kind == "full":
            assert msg == cp.occupancy_grid(ro.header(0, 0, 0, b"map"), window, grid)
        elif kind == "update":
            assert msg == cp.grid_update(ro.header(0, 0, 0, b"map"), *rect, grid)
        else:
            assert msg == b""
        kinds.append(kind)
    return kinds


W = (-7.45, -7.45, 0.2, 75, 75)
ROLLED = (-7.25, -7.45, 0.2, 75, 75)


def test_publisher_first_full_then_update_then_roll():
    assert run_sequence([("bounds", 3, 9, 4, 8), ("publish", W), ("bounds", 3, 9, 4, 8), ("publish", W), ("bounds", 0, 75, 0, 75),
                         ("publish", ROLLED), ("publish", ROLLED)]) == ["full", "update", "full", "none"]


def test_publisher_empty_bounds_and_height_zero():
    assert run_sequence([("publish", W), ("publish", W), ("bounds", 5, 5, 0, 9), ("publish", W), ("bounds", 2, 7, 6, 6),
                         ("publish", W), ("bounds", 2, 7, 9, 3), ("bounds", 3, 4, 3, 3), ("publish", W)]) == ["full", "none", "none",
                                                                                                             "update", "update"]


def test_publisher_always_full_and_forced_full():
    assert run_sequence([("publish", W), ("bounds", 1, 2, 1, 2), ("publish", W)], always=True) == ["full", "full"]
    # onNewSubscription: a full message that leaves the accumulated bounds
    assert run_sequence([("publish", W), ("bounds", 1, 9, 2, 5), ("force", W), ("publish", W)]) == ["full", "full", "update"]
    # a forced full before anything else saves the window; the INT_MAX initial bounds stay empty
    assert run_sequence([("force", W), ("publish", W), ("bounds", 0, 4, 0, 4), ("publish", W)]) == ["full", "none", "update"]


def test_publisher_bounds_accumulate_over_skipped_publishes_and_stale_bounds():
    # no subscriber: publish is not called and the rects add up; getBounds after an early return repeats the last rect
    assert run_sequence([("publish", W), ("bounds", 10, 20, 10, 12), ("bounds", 30, 31, 5, 6), ("bounds", 30, 31, 5, 6),
                         ("publish", W), ("bounds", 30, 31, 5, 6), ("publish", W)]) == ["full", "update", "update"]


def test_publisher_query_and_small_capacity_keep_the_state():
    assert run_sequence([("query", W), ("small", W), ("publish", W), ("bounds", 1, 70, 2, 60), ("query", W), ("small", W),
                         ("publish", W), ("bounds", 1, 3, 1, 3), ("small", ROLLED), ("publish", ROLLED)]) == [
        "kept", "kept", "full", "kept", "kept", "update", "kept", "full"]


def test_publisher_window_changes():
    w_res = (-7.45, -7.45, 0.2 + 1e-12, 75, 75)        # the same float resolution: not a change
    w_last_bit = (np.nextafter(-7.45, 0.0), -7.45, 0.2, 75, 75)
    assert run_sequence([("publish", W), ("bounds", 0, 1, 0, 1), ("publish", w_res)]) == ["full", "update"]
    assert run_sequence([("publish", W), ("bounds", 0, 1, 0, 1), ("publish", w_last_bit)]) == ["full", "full"]
    assert run_sequence([("publish", W), ("publish", (-7.45, -7.45, 0.2, 75, 74))]) == ["full", "full"]


def test_publisher_refuses_bounds_outside_the_grid():
    pub = cp.HostPublisher()
    grid = all_costs_grid(75, 75, 2)
    h = (0, 0, 0, b"map")
    assert pub.publish(h, W, grid)[0] == "full"
    for b in ((-1, 3, 0, 3), (70, 76, 0, 3), (0, 3, 0, 76), (0, 3, 5, 2)):
        p = cp.HostPublisher()
        p.publish(h, W, grid)
        p.bounds(*b)
        before = p.state()
        assert p.publish(h, W, grid)[2] == -1 and p.state() == before


def test_publisher_struct_layout():
    native.assert_struct_layouts({"gem_costmap_publisher": _lib.GemCostmapPublisher})
    assert C.sizeof(_lib.GemCostmapPublisher) == C.sizeof(cp.PublisherState)
    assert _lib.GemCostmapPublisher._fields_ == cp.PublisherState._fields_
