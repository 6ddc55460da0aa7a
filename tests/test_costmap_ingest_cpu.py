"""The costmap plugins fed from their messages, CPU side (DESIGN.md f18): the C oracle (tests/orc_gridmsg.c) against the
independent Python restatement of tests/gridmsg_oracle.py, and the library's grid_map_msgs/GridMap reader
(gem_gridmsg.h, built with g++) against both, on messages from the general encoder and on every refusal, the message
truncated at every byte included; the oracle's whole-record PointCloud2 decode against the numpy restatement of f12;
the gem_grid_map_layer layout against the C compiler."""
import ctypes as C

import numpy as np
import pytest

import costmap_cases as cc
import gridmsg_oracle as gm
import pc2_cases as pc
import pc2_oracle
import rosmsg_oracle as ro
from gem_b200 import _lib

CASES = {c[0]: c for c in gm.cases()}
REFUSALS = {c[0]: c for c in gm.refusals()}


def bits(d):
    """a descriptor with its doubles as their bit patterns"""
    return None if d is None else {k: (np.float64(v).tobytes() if isinstance(v, float) else v) for k, v in d.items()}


@pytest.mark.parametrize("name", sorted(CASES))
def test_parse_three_ways(name):
    _, msg, layer = CASES[name]
    want = gm.parse(msg, layer)
    assert want is not None, name
    assert bits(gm.host_parse(msg, layer)) == bits(want)
    assert bits(gm.orc_parse(msg, layer)) == bits(want)
    assert want["offset"] % 1 == 0 and want["offset"] + 4 * want["floats"] <= len(msg) - 4


def test_what_the_cases_show():
    d = gm.parse(CASES["repeated_name_last_wins"][1])
    first = gm.parse(CASES["repeated_name_last_wins"][1].replace(b"traver", b"travex", 2).replace(b"travex", b"traver", 1))
    assert first is not None and d["offset"] > first["offset"]            # the later "traver" wins
    d = gm.parse(CASES["length_not_multiple"][1])
    assert (d["size_x"], d["size_y"]) == (30, 19) and d["length_x"] == 30 * 0.07 and d["length_y"] == 19 * 0.07
    d = gm.parse(CASES["length_half_up"][1])
    assert (d["size_x"], d["size_y"]) == (9, 11)                           # 8.5 and 10.5 round away from zero
    d = gm.parse(CASES["start_beyond_size"][1])
    assert (d["start_x"], d["start_y"]) == (65535, 1000)
    phases = {(gm.parse(CASES[f"frame_id_{fl}"][1])["offset"]) % 16 for fl in (0, 1, 2, 3, 5, 13, 16, 64, 255, 256, 300)}
    assert len(phases) >= 8


def test_the_library_message_layout():
    """the offsets W2 states for the messages gem_ros_grid_map writes: layer k's floats at 277 + |frame_id| + k (57 + 4 L^2)"""
    L = 8
    for fl in (0, 4, 19):
        fid = (b"odom/" * 10)[:fl]
        data = [gm.array(np.arange(L * L, dtype=np.float32) + k, L, L) for k in range(9)]
        names = [b"elevation", b"variance", b"rough", b"slope", b"traver", b"color_r", b"color_g", b"color_b", b"intensity"]
        msg = gm.encode(0.05, (L * 0.05, L * 0.05), (1.0, 2.0), names, data, start=(3, 5), frame_id=fid)
        assert len(msg) == 737 + fl + 36 * L * L
        for k, n in enumerate(names):
            d = gm.host_parse(msg, n)
            assert d["offset"] == 277 + fl + k * (57 + 4 * L * L)
            assert np.array_equal(gm.layer_floats(msg, d), data[k]["floats"])


@pytest.mark.parametrize("name", sorted(REFUSALS))
def test_refusals(name):
    _, msg, layer, nb = REFUSALS[name]
    assert gm.parse(msg, layer) is None
    assert gm.host_parse(msg, layer, nb) is None
    assert gm.orc_parse(msg, layer, nb) is None


@pytest.mark.parametrize("name", ["square_c1", "rect_tall", "frame_id_3", "extra_floats", "repeated_name_last_wins"])
def test_truncated_at_every_byte(name):
    _, msg, layer = CASES[name]
    n = len(msg)
    host, orc = gm.host(), gm.orc()
    buf = C.create_string_buffer(msg, n)
    for cut in range(n):
        for fn in (host.gm_parse, orc.orc_grid_map_parse):
            g = gm.Layer.from_buffer_copy(gm.SENTINEL)
            assert fn(buf, cut, layer, C.byref(g)) == 1, (name, cut)
            assert bytes(g) == bytes(gm.SENTINEL)
        if cut % 97 == 0 or cut > n - 8:
            assert gm.parse(msg[:cut], layer) is None
    assert gm.host_parse(msg + b"\x00" * 5, layer) == gm.host_parse(msg, layer)   # bytes after the message are ignored


def test_library_descriptor_check():
    d = gm.parse(CASES["rect_tall"][1])
    assert gm.host().gm_layer_ok(C.byref(gm.layer_struct(d))) == 1
    for k, v in (("resolution", 0.0), ("resolution", float("nan")), ("floats", d["floats"] + 1), ("column_major", 0),
                 ("size_x", -1), ("length_x", float("inf"))):
        e = dict(d, **{k: v})
        assert gm.host().gm_layer_ok(C.byref(gm.layer_struct(e))) == 0, k


def windows(d):
    """a few costmap windows over and around the layer"""
    lx, ly = d["length_x"], d["length_y"]
    cx, cy = d["position_x"], d["position_y"]
    return [(cx - 0.5 * lx - 0.3, cy - 0.5 * ly - 0.3, 0.2, int(lx / 0.2) + 4, int(ly / 0.2) + 4),
            (cx - 0.5 * lx, cy - 0.5 * ly, d["resolution"], d["size_x"], d["size_y"]),
            (cx - 0.01, cy + 0.02, 0.05, 13, 9),
            (cx - 0.5 * lx + 0.77 * d["resolution"], cy - 0.5 * ly + 0.31 * d["resolution"], 0.5 * d["resolution"],
             2 * d["size_x"] + 1, d["size_y"] + 3)]


@pytest.mark.parametrize("name", sorted(CASES))
def test_mark_oracle_equals_restatement(name):
    _, msg, layer = CASES[name]
    d = gm.parse(msg, layer)
    v = gm.layer_floats(msg, d)
    rng = np.random.default_rng(len(msg))
    for w in windows(d):
        g0 = cc.random_grid(rng, w)
        for th in (0.7, 0.5, float(np.float32(0.7)), 0.0):
            for mu in (True, False):
                g1, m1 = gm.orc_mark_grid(d, v, w, g0, th, mu)
                g2, m2 = gm.mark_grid(d, v, w, g0, th, mu)
                assert np.array_equal(g1.reshape(-1), g2.reshape(-1)), (name, w, th, mu)
                assert m1["marked"] == m2["marked"] and m1["lethal"] == m2["lethal"], (name, w, th, mu)
                for k in ("min_x", "min_y", "max_x", "max_y"):
                    assert np.float64(m1[k]).tobytes() == np.float64(m2[k]).tobytes(), (name, w, k)


def test_mark_positions_generalise_the_square_map():
    """on a square map G4's positions are GridMapFrame's: cx + half - res * ((i + L - s) % L)"""
    _, msg, _ = CASES["square_c1"]
    d = gm.parse(msg)
    px, py = gm.positions(d)
    L, res = d["size_x"], d["resolution"]
    half = 0.5 * (L * res) - 0.5 * res
    k = np.arange(L * L)
    assert np.array_equal(px, d["position_x"] + half - res * ((k % L + L - d["start_x"]) % L).astype(np.float64))
    assert np.array_equal(py, d["position_y"] + half - res * ((k // L + L - d["start_y"]) % L).astype(np.float64))


@pytest.mark.parametrize("name", pc.case_names())
def test_record_oracle_equals_numpy(name):
    case = pc.case_by_name(name)
    n = case["width"] * case["height"]
    want = pc.np_decode(case)
    c, keep = pc2_oracle._cloud(case)
    data = np.ascontiguousarray(case["data"], np.uint8)
    rec = np.zeros((max(n, 1), 32), np.uint8)
    rc = gm.orc().orc_pc2_records(C.addressof(c), data.ctypes.data, int(case.get("data_bytes", data.nbytes)), rec.ctypes.data)
    if want is None:
        assert rc == 1
        return
    assert rc == 0 and np.array_equal(rec[:n], want[0]), name


def test_layer_struct_layout():
    out = (C.c_longlong * 13)()
    gm.host().gm_layout(out)
    want = [C.sizeof(_lib.GemGridMapLayer)] + [getattr(_lib.GemGridMapLayer, k).offset for k in gm.FIELDS]
    assert list(out) == want
    assert [f[0] for f in _lib.GemGridMapLayer._fields_] == list(gm.FIELDS) and bytes(gm.Layer()) == bytes(_lib.GemGridMapLayer())


def test_encoder_writes_what_gem_ros_grid_map_writes():
    """tests/rosmsg_oracle.py's W2 encoder (the bytes gem_ros_grid_map writes) and the general encoder agree byte for byte"""
    L, res = 6, 0.05
    layers = {n: np.arange(L * L, dtype=np.float32).reshape(L, L) * (k + 1) for k, n in enumerate(ro.GRID_LAYERS)}
    a = ro.grid_map(ro.header(1, 1700000000, 5, b"odom"), L, res, 1.0, 2.0, (3, 4), layers)
    data = [gm.array(layers[n].reshape(-1, order="F"), L, L) for n in ro.GRID_LAYERS]
    b = gm.encode(res, (L * res, L * res), (1.0, 2.0), [n.encode() for n in ro.GRID_LAYERS], data, start=(3, 4))
    assert a == b
