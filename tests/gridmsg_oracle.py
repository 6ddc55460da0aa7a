"""The f18 ingest without a GPU (DESIGN.md f18).  TEST INFRASTRUCTURE ONLY.

- encode(): a general grid_map_msgs/GridMap encoder (ROS1 wire format, W1): any geometry, layer list, dims, data_offset,
  float counts, start indices and frame_id, so that messages the library never writes can be crafted.
- parse(): an independent Python restatement of G1-G3 (fromMessage of grid_map 1.6 for one layer): a dict of the
  descriptor's fields, or None where the library refuses.
- mark_grid(): ElevationMapLayer::updateBounds over a parsed layer (G4 order and positions, last writer wins) in numpy.
- orc(): tests/orc_gridmsg.c, the literal C oracle; host(): the library's reader (gem_gridmsg.h) through
  tests/gridmsg_host.cpp, built with g++.  Both compiled into a temporary directory (the checkout may be read-only).
- cases(): the crafted messages."""
from __future__ import annotations

import ctypes as C
import math
import os
import struct

import numpy as np

import costmap_oracle as co
import native

HERE = os.path.dirname(os.path.abspath(__file__))
FIELDS = ("resolution", "position_x", "position_y", "length_x", "length_y", "size_x", "size_y", "start_x", "start_y",
          "offset", "floats", "column_major")
INT_MAX = 2**31 - 1


class Layer(C.Structure):
    """gem_grid_map_layer / orc_grid_layer"""
    _fields_ = [("resolution", C.c_double), ("position_x", C.c_double), ("position_y", C.c_double), ("length_x", C.c_double),
                ("length_y", C.c_double), ("size_x", C.c_int), ("size_y", C.c_int), ("start_x", C.c_int), ("start_y", C.c_int),
                ("offset", C.c_ulonglong), ("floats", C.c_longlong), ("column_major", C.c_int)]


def as_dict(g) -> dict:
    return {k: getattr(g, k) for k in FIELDS}


# ---- the encoder ---------------------------------------------------------------------------------------------------------
def _str(b: bytes) -> bytes:
    return struct.pack("<I", len(b)) + b


def array(floats, rows: int | None = None, cols: int | None = None, labels=(b"column_index", b"row_index"), dims=None,
          data_offset: int = 0) -> dict:
    """a Float32MultiArray: the floats (any count) and its layout; dims overrides the two default dims"""
    f = np.ascontiguousarray(floats, np.float32).reshape(-1)
    if dims is None:
        dims = [(labels[0], cols, rows * cols), (labels[1], rows, rows)]
    return {"dims": dims, "data_offset": data_offset, "floats": f}


def encode(res, length, position, layers, data, basic=(b"elevation",), start=(0, 0), frame_id=b"odom", seq=1,
           stamp=(1700000000, 5), pose_z=0.0, orientation=(0.0, 0.0, 0.0, 1.0)) -> bytes:
    """the message's bytes.  layers: names (bytes); data: array() dicts, one per layer or any other number"""
    out = [struct.pack("<III", seq, *stamp), _str(frame_id),
           struct.pack("<3d", res, length[0], length[1]), struct.pack("<3d", position[0], position[1], pose_z),
           struct.pack("<4d", *orientation), struct.pack("<I", len(layers))]
    out += [_str(n) for n in layers]
    out.append(struct.pack("<I", len(basic)))
    out += [_str(n) for n in basic]
    out.append(struct.pack("<I", len(data)))
    for a in data:
        out.append(struct.pack("<I", len(a["dims"])))
        for label, size, stride in a["dims"]:
            out.append(_str(label) + struct.pack("<II", size, stride))
        out.append(struct.pack("<II", a["data_offset"], a["floats"].size))
        out.append(a["floats"].tobytes())
    out.append(struct.pack("<HH", *start))
    return b"".join(out)


# ---- G1-G3 restated --------------------------------------------------------------------------------------------------------
class _Truncated(Exception):
    pass


def _round(x: float) -> float:
    """std::round: halves away from zero (x >= 0 here)"""
    f = math.floor(x)
    return f + 1.0 if x - f >= 0.5 else f


def parse(msg: bytes, layer: bytes = b"traver"):
    """the descriptor as a dict, or None where fromMessage throws, asserts or reads out of bounds"""
    pos = 0

    def take(n):
        nonlocal pos
        if n > len(msg) - pos:
            raise _Truncated
        pos += n
        return msg[pos - n:pos]

    def u32():
        return struct.unpack("<I", take(4))[0]

    def string():
        return take(u32())

    try:
        take(12)
        string()
        res, lx, ly, px, py = struct.unpack("<5d", take(40))
        take(40)
        names = [string() for _ in range(u32())]
        [string() for _ in range(u32())]
        arrays = []
        for _ in range(u32()):
            dims = [(string(), u32(), u32()) for _ in range(u32())]
            u32()
            nf = u32()
            at = pos
            take(4 * nf)
            arrays.append((dims, nf, at))
        sx, sy = struct.unpack("<HH", take(4))
    except _Truncated:
        return None
    if len(names) != len(arrays):
        return None
    hits = [i for i, n in enumerate(names) if n == layer]
    if not hits:
        return None
    dims, nf, at = arrays[hits[-1]]
    if len(dims) < 2 or dims[0][0] != b"column_index":
        return None
    if not (math.isfinite(res) and res > 0):
        return None
    sizes = []
    for length in (lx, ly):
        if not (math.isfinite(length) and length > 0):
            return None
        q = _round(length / res)
        if not q <= INT_MAX:
            return None
        sizes.append(int(q))
    if sizes[0] * sizes[1] > INT_MAX:
        return None
    rows, cols = dims[1][1], dims[0][1]
    if (rows, cols) != tuple(sizes) or nf < rows * cols:
        return None
    return {"resolution": res, "position_x": px, "position_y": py, "length_x": sizes[0] * res, "length_y": sizes[1] * res,
            "size_x": sizes[0], "size_y": sizes[1], "start_x": sx, "start_y": sy, "offset": at, "floats": sizes[0] * sizes[1],
            "column_major": 1}


def layer_floats(msg: bytes, d: dict) -> np.ndarray:
    return np.frombuffer(msg, np.float32, d["floats"], d["offset"]) if d["floats"] else np.zeros(0, np.float32)


# ---- G4 and updateBounds restated --------------------------------------------------------------------------------------------
def positions(d: dict):
    """G4: every element's position, in element order"""
    k = np.arange(d["floats"], dtype=np.int64)
    sx, sy = d["size_x"], d["size_y"]
    ix, iy = k % sx, k // sx
    ux, uy = (ix - d["start_x"]) % sx, (iy - d["start_y"]) % sy
    res = d["resolution"]
    ox = d["position_x"] + (0.5 * d["length_x"] - 0.5 * res)
    oy = d["position_y"] + (0.5 * d["length_y"] - 0.5 * res)
    return ox + res * (-ux).astype(np.float64), oy + res * (-uy).astype(np.float64)


def mark_grid(d: dict, floats, window, grid, thresh: float, mark_unknown: bool):
    """(grid, marks) after ElevationMapLayer::updateBounds over the layer"""
    ox, oy, res, sx, sy = window
    v = np.asarray(floats, np.float32)
    px, py = positions(d)
    keep = np.ones(v.size, bool) if mark_unknown else ~np.isnan(v)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        qx, qy = (px - ox) / res, (py - oy) / res
        keep &= ~((px < ox) | (py < oy)) & np.isfinite(px) & np.isfinite(py) & (qx < 2.0**31) & (qy < 2.0**31)
        mx = np.where(keep, qx, 0).astype(np.int64)
        my = np.where(keep, qy, 0).astype(np.int64)
    keep &= (mx < sx) & (my < sy)
    lethal = v.astype(np.float64) < thresh
    g = np.array(grid, np.uint8).reshape(-1).copy()
    cells = (my * sx + mx)[keep]
    cost = np.where(lethal[keep], co_lethal(), 0).astype(np.uint8)
    if cells.size:
        _, first = np.unique(cells[::-1], return_index=True)            # the last writer of each cell
        last = cells.size - 1 - first
        g[cells[last]] = cost[last]
    n = int(keep.sum())
    marks = {"marked": n, "lethal": int((lethal & keep).sum()),
             "min_x": float(px[keep].min()) + 0.0 if n else math.inf, "min_y": float(py[keep].min()) + 0.0 if n else math.inf,
             "max_x": float(px[keep].max()) + 0.0 if n else -math.inf, "max_y": float(py[keep].max()) + 0.0 if n else -math.inf}
    return g.reshape(sy, sx), marks


def co_lethal():
    return 254


# ---- the C oracle and the library's host build ---------------------------------------------------------------------------------
_orc = _host = None


def orc():
    global _orc
    if _orc is None:
        lib = native.shared_library("orc_gridmsg", [os.path.join(HERE, "orc_gridmsg.c")], native.ORACLE_C + ["-I", HERE], ["-lm"])
        P = C.c_void_p
        lib.orc_grid_map_parse.argtypes = [C.c_char_p, C.c_ulonglong, C.c_char_p, C.POINTER(Layer)]
        lib.orc_grid_map_parse.restype = C.c_int
        lib.orc_mark_grid.argtypes = [C.POINTER(Layer), P, C.POINTER(co.Window), C.c_double, C.c_int, P, C.POINTER(co.Marks)]
        lib.orc_mark_grid.restype = None
        lib.orc_pc2_records.argtypes = [P, P, C.c_ulonglong, P]
        lib.orc_pc2_records.restype = C.c_int
        _orc = lib
    return _orc


def host():
    global _host
    if _host is None:
        lib = native.shared_library("gridmsg_host", [os.path.join(HERE, "gridmsg_host.cpp")], native.HOST_CXX)
        lib.gm_parse.argtypes = [C.c_char_p, C.c_ulonglong, C.c_char_p, C.POINTER(Layer)]
        lib.gm_parse.restype = C.c_int
        lib.gm_layer_ok.argtypes = [C.POINTER(Layer)]
        lib.gm_layer_ok.restype = C.c_int
        lib.gm_layout.argtypes = [C.POINTER(C.c_longlong)]
        lib.gm_layout.restype = None
        _host = lib
    return _host


SENTINEL = Layer(-1.0, -2.0, -3.0, -4.0, -5.0, -6, -7, -8, -9, 12345, -10, -11)


def _parse_with(fn, msg: bytes, layer: bytes, nbytes=None):
    g = Layer.from_buffer_copy(SENTINEL)
    rc = fn(msg, len(msg) if nbytes is None else nbytes, layer, C.byref(g))
    if rc:
        assert bytes(g) == bytes(SENTINEL), "a refused parse wrote its output"
        return None
    return as_dict(g)


def host_parse(msg: bytes, layer: bytes = b"traver", nbytes=None):
    return _parse_with(host().gm_parse, msg, layer, nbytes)


def orc_parse(msg: bytes, layer: bytes = b"traver", nbytes=None):
    return _parse_with(orc().orc_grid_map_parse, msg, layer, nbytes)


def layer_struct(d: dict) -> Layer:
    return Layer(*[d[k] for k in FIELDS])


def orc_mark_grid(d: dict, floats, window, grid, thresh: float, mark_unknown: bool):
    g = np.ascontiguousarray(grid, np.uint8).copy()
    v = np.ascontiguousarray(floats, np.float32)
    w = co.Window(*window)
    mk = co.Marks()
    orc().orc_mark_grid(C.byref(layer_struct(d)), C.c_void_p(v.ctypes.data), C.byref(w), float(thresh), 1 if mark_unknown else 0,
                        C.c_void_p(g.ctypes.data), C.byref(mk))
    return g, {k: getattr(mk, k) for k, _ in co.Marks._fields_}


# ---- crafted messages ---------------------------------------------------------------------------------------------------------
def traver_values(rng, n):
    """traversabilities around the thresholds, NaN (cleared cells), -0, +-inf"""
    v = rng.uniform(-0.2, 1.2, n).astype(np.float32)
    pick = rng.random(n)
    v[pick < 0.15] = np.nan
    v[(pick >= 0.15) & (pick < 0.2)] = np.float32(0.7)
    v[(pick >= 0.2) & (pick < 0.22)] = np.float32(0.5)
    v[(pick >= 0.22) & (pick < 0.23)] = -0.0
    if n > 2:
        v[0], v[1] = np.inf, -np.inf
    return v


def cases():
    """(name, msg bytes, layer name) of accepted messages"""
    rng = np.random.default_rng(18)
    out = []

    def add(name, res, sizes, position, start, names, pick, frame_id=b"odom", extra=0, lengths=None, dims_swap=False,
            basic=(b"elevation",)):
        sx, sy = sizes
        lengths = lengths or (sx * res, sy * res)
        data = []
        for n in names:
            f = traver_values(rng, sx * sy + extra)
            data.append(array(f, sx, sy))
        out.append((name, encode(res, lengths, position, list(names), data, basic=basic, start=start, frame_id=frame_id), pick))

    add("square_c1", 0.05, (64, 64), (1.25, -3.5), (0, 0), [b"elevation", b"traver"], b"traver")
    add("rect_tall", 0.1, (7, 33), (-12.0, 40.3), (3, 30), [b"traver"], b"traver")
    add("rect_wide", 0.2, (41, 5), (100.0, -0.05), (40, 4), [b"a", b"traver", b"b"], b"traver")
    add("start_beyond_size", 0.05, (16, 24), (0.3, 0.7), (65535, 1000), [b"traver"], b"traver")
    add("start_at_size", 0.05, (16, 24), (0.3, 0.7), (16, 24), [b"traver"], b"traver")
    add("length_not_multiple", 0.07, (30, 19), (2.0, -1.0), (5, 7), [b"traver"], b"traver", lengths=(30 * 0.07 + 0.02, 19 * 0.07 - 0.03))
    add("length_half_up", 0.25, (9, 11), (0.0, 0.0), (0, 1), [b"traver"], b"traver", lengths=(8.5 * 0.25, 10.5 * 0.25))
    add("repeated_name_last_wins", 0.1, (12, 12), (5.0, 5.0), (2, 9), [b"traver", b"x", b"traver"], b"traver")
    add("other_layer", 0.1, (12, 10), (5.0, 5.0), (2, 9), [b"traver", b"slope"], b"slope")
    add("extra_floats", 0.1, (10, 13), (-4.0, 2.0), (9, 12), [b"traver"], b"traver", extra=37)
    add("no_basic_layers", 0.1, (10, 13), (-4.0, 2.0), (1, 1), [b"traver"], b"traver", basic=())
    add("utm_position", 0.05, (32, 20), (453210.125, 5412345.875), (31, 0), [b"traver"], b"traver")
    add("one_cell", 0.2, (1, 1), (0.1, 0.1), (0, 0), [b"traver"], b"traver")
    add("one_row", 0.2, (1, 17), (0.1, 0.1), (0, 3), [b"traver"], b"traver")
    for fl in (0, 1, 2, 3, 5, 13, 16, 64, 255, 256, 300):
        add(f"frame_id_{fl}", 0.1, (9, 6), (0.5, -0.5), (4, 2), [b"elevation", b"traver"], b"traver", frame_id=(b"map/" * 80)[:fl])
    return out


def refusals():
    """(name, msg bytes, layer, nbytes) the parser refuses"""
    rng = np.random.default_rng(81)
    f = traver_values(rng, 6 * 4)
    ok = dict(res=0.1, length=(0.6, 0.4), position=(0.0, 0.0), layers=[b"traver"], data=[array(f, 6, 4)])

    def msg(**kw):
        a = dict(ok)
        a.update(kw)
        return encode(**a)

    out = [("layers_ne_data_more", msg(layers=[b"traver", b"x"]), b"traver"),
           ("layers_ne_data_fewer", msg(data=[array(f, 6, 4), array(f, 6, 4)]), b"traver"),
           ("layer_missing", msg(), b"elevation"),
           ("layer_prefix", msg(), b"trave"),
           ("no_dims", msg(data=[array(f, dims=[])]), b"traver"),
           ("one_dim", msg(data=[array(f, dims=[(b"column_index", 4, 24)])]), b"traver"),
           ("row_major", msg(data=[array(f, 6, 4, labels=(b"row_index", b"column_index"))]), b"traver"),
           ("bad_label", msg(data=[array(f, 6, 4, labels=(b"column_indeX", b"row_index"))]), b"traver"),
           ("rows_cols_swapped", msg(data=[array(f, 4, 6)]), b"traver"),
           ("too_few_floats", msg(data=[array(f[:23], 6, 4)]), b"traver"),
           ("zero_resolution", msg(res=0.0), b"traver"),
           ("negative_resolution", msg(res=-0.1), b"traver"),
           ("nan_resolution", msg(res=float("nan")), b"traver"),
           ("inf_resolution", msg(res=float("inf")), b"traver"),
           ("zero_length", msg(length=(0.0, 0.4)), b"traver"),
           ("negative_length", msg(length=(0.6, -0.4)), b"traver"),
           ("inf_length", msg(length=(float("inf"), 0.4)), b"traver"),
           ("nan_length", msg(length=(0.6, float("nan"))), b"traver"),
           ("size_overflows_int", msg(length=(0.1 * 2.0**31, 0.4)), b"traver"),
           ("product_overflows_int", msg(length=(0.1 * 65536, 0.1 * 65536), data=[array(f, dims=[(b"column_index", 65536, 0),
                                                                                               (b"row_index", 65536, 0)])]),
            b"traver"),
           ("the_repeat_is_bad", msg(layers=[b"traver", b"traver"], data=[array(f, 6, 4), array(f[:5], 6, 4)]), b"traver")]
    # a string or array count running past the end
    good = msg()
    fl = 4                                                              # "odom"
    out.append(("frame_id_count_past_end", good[:12] + struct.pack("<I", len(good)) + good[16:], b"traver"))
    at_layers = 12 + 4 + fl + 80
    out.append(("layers_count_huge", good[:at_layers] + struct.pack("<I", 0xFFFFFFFF) + good[at_layers + 4:], b"traver"))
    out.append(("layer_name_past_end", good[:at_layers + 4] + struct.pack("<I", 0x7FFFFFFF) + good[at_layers + 8:], b"traver"))
    at_floats = len(good) - 4 - 4 * f.size - 4
    out.append(("float_count_past_end", good[:at_floats] + struct.pack("<I", f.size + 1) + good[at_floats + 4:], b"traver"))
    return [(n, m, l, len(m)) for n, m, l in out]
