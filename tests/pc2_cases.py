"""Crafted sensor_msgs/PointCloud2 messages for the PointCloud2 ingest (DESIGN.md f12) and an independent numpy
restatement of PCL 1.8's createMapping<PointXYZRGBICT> + fromPCLPointCloud2 built on structured-dtype views.

A case is a dict {name, fields: [(name, offset, datatype, count)], width, height, point_step, row_step, is_bigendian,
data: uint8 array, data_bytes (optional, default len(data)), refused: bool}.  Every byte of a message that no field value
fills is random, so the bytes a merged span or the whole-point copy carries over are visible."""
from __future__ import annotations

import numpy as np

F32, F64, U8, U16, U32, I8 = 7, 8, 2, 4, 6, 1
NAMES = ["x", "y", "z", "rgb", "intensity", "covariance", "travers"]
STRUCT = {"x": 0, "y": 4, "z": 8, "rgb": 16, "intensity": 24, "covariance": 20, "travers": 28}
NP_TYPES = {1: "i1", 2: "u1", 3: "<i2", 4: "<u2", 5: "<i4", 6: "<u4", 7: "<f4", 8: "<f8"}

# the drivers' layouts: (fields, point_step)
LAYOUTS = {
    # KITTI velodyne bins as published by kitti2bag: x, y, z, intensity
    "kitti16": ([("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("intensity", 12, F32, 1)], 16),
    # velodyne_pointcloud PointXYZIR (PCL_ADD_POINT4D, float intensity, uint16 ring; 16-byte aligned)
    "xyzir32": ([("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("intensity", 16, F32, 1), ("ring", 20, U16, 1)], 32),
    # the packed variant: x, y, z, intensity, uint16 ring, float time -> floats at odd 2-byte offsets every other point
    "xyzir22": ([("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("intensity", 12, F32, 1), ("ring", 16, U16, 1),
                 ("time", 18, F32, 1)], 22),
    # Hesai PandarQT (simple_demo): x, y, z, intensity, float64 timestamp, uint16 ring
    "pandarqt": ([("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("intensity", 16, F32, 1), ("timestamp", 24, F64, 1),
                  ("ring", 32, U16, 1)], 48),
    # an Ouster-like layout whose intensity is a uint16: no FLOAT32 intensity, so intensity is 0
    "ouster": ([("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("t", 16, U32, 1), ("intensity", 20, U16, 1),
                ("reflectivity", 22, U16, 1), ("ring", 24, U8, 1), ("ambient", 26, U16, 1), ("range", 28, U32, 1)], 48),
    # a structured-light driver's organised cloud: x, y, z, packed rgb
    "d435": ([("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("rgb", 12, F32, 1)], 16),
    # GEM's own published PointXYZRGBICT (the whole-point copy)
    "xyzrgbict": ([("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("rgb", 16, F32, 1), ("intensity", 24, F32, 1),
                   ("covariance", 20, F32, 1), ("travers", 28, F32, 1)], 32),
}


def message(name, fields, point_step, width, height=1, row_step=None, values=None, seed=0, is_bigendian=0, data_bytes=None,
            refused=False, extra=0):
    """a message with random bytes everywhere, then values[k] (an (n,) array) written into every field named k"""
    rng = np.random.Generator(np.random.PCG64(seed))
    row_step = width * point_step if row_step is None else row_step
    size = max((height - 1) * row_step + width * point_step, 0) + extra
    data = rng.integers(0, 256, size, dtype=np.uint8)
    n = width * height
    for fname, off, dt, cnt in fields:
        if values is None or fname not in values or n == 0:
            continue
        v = np.asarray(values[fname]).astype(NP_TYPES[dt]).reshape(height, width)
        k = np.dtype(NP_TYPES[dt]).itemsize
        for r in range(height):
            base = r * row_step + off
            idx = base + np.arange(width)[:, None] * point_step + np.arange(k)[None, :]
            data[idx] = np.frombuffer(v[r].tobytes(), np.uint8).reshape(width, k)
    c = {"name": name, "fields": list(fields), "width": width, "height": height, "point_step": point_step,
         "row_step": row_step, "is_bigendian": is_bigendian, "data": data, "refused": refused}
    if data_bytes is not None:
        c["data_bytes"] = data_bytes
    return c


def from_xyzi(name, layout, xyzi, width=None, height=1, row_pad=0, seed=0, rgb=None):
    """a real layout filled from an (n, 4) float32 cloud (intensity cast to the field's type; rgb as packed bytes)"""
    fields, ps = LAYOUTS[layout]
    xyzi = np.asarray(xyzi, np.float32)
    width = xyzi.shape[0] if width is None else width
    vals = {"x": xyzi[:, 0], "y": xyzi[:, 1], "z": xyzi[:, 2], "intensity": xyzi[:, 3]}
    if rgb is not None:
        vals["rgb"] = np.ascontiguousarray(rgb, np.uint8).reshape(-1, 4).view(np.float32).reshape(-1)
    return message(name, fields, ps, width, height, width * ps + row_pad, vals, seed)


def _special_bits():
    bits = np.array([0x7FC00000, 0x7FC00001, 0xFFFFFFFF, 0x7F800001, 0xFF800000, 0x7F800000, 0x80000000, 0x00000000,
                     0x00000001, 0x807FFFFF, 0x3F800000, 0xBF800000], np.uint32)
    return bits.view(np.float32)


def cases():
    from gem_b200 import synth
    out = []
    hdl = synth.hdl64_frame(0)["xyzi"][:3000]
    for lay in ("kitti16", "xyzir32", "xyzir22", "pandarqt", "ouster", "xyzrgbict"):
        out.append(from_xyzi(lay, lay, hdl, seed=len(out) + 1))
    out.append(from_xyzi("xyzir22_odd_count", "xyzir22", hdl[:1001], seed=40))
    d435 = synth.d435_frame(0)
    out.append(from_xyzi("d435_organised_padded", "d435", d435["xyzi"], width=640, height=480, row_pad=64, seed=41,
                         rgb=d435["rgba"]))
    out.append(from_xyzi("d435_organised_odd_pad", "d435", d435["xyzi"][:640 * 7], width=640, height=7, row_pad=13, seed=42))
    n, rnd = 257, np.random.Generator(np.random.PCG64(5)).standard_normal((257, 4)).astype(np.float32)
    v = {"x": rnd[:, 0], "y": rnd[:, 1], "z": rnd[:, 2], "intensity": rnd[:, 3]}
    base = [("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("intensity", 12, F32, 1)]
    out += [
        message("reverse_order", list(reversed(LAYOUTS["xyzrgbict"][0])), 36, n, values=v, seed=10),
        message("duplicate_names", [("x", 12, F32, 1), ("x", 0, F32, 1), ("y", 4, F64, 1), ("y", 16, F32, 1), ("z", 8, F32, 1)],
                24, n, values=None, seed=11),
        message("count_0_and_2", [("x", 0, F32, 0), ("y", 4, F32, 2), ("z", 12, F32, 1), ("intensity", 16, F32, 1)], 20, n,
                values=v, seed=12),
        message("float64_x", [("x", 0, F64, 1), ("y", 8, F32, 1), ("z", 12, F32, 1), ("intensity", 16, F32, 1)], 20, n,
                values=v, seed=13),
        message("float64_y_filled_by_merge", [("x", 0, F32, 1), ("y", 4, F64, 1), ("z", 8, F32, 1), ("intensity", 12, F32, 1)],
                16, n, seed=14),
        message("merge_overwrites_intensity", [("intensity", 0, F32, 1), ("x", 4, F32, 1), ("travers", 32, F32, 1)], 36, n,
                values=v, seed=15),
        message("one_span_point_step_32", [("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("ring", 12, U16, 1)], 32, n,
                values=v, seed=16),
        message("special_bits", base, 16, 12 * 4, values={k: np.tile(_special_bits(), 4) for k in ("x", "y", "z", "intensity")},
                seed=17),
        message("is_bigendian", base, 16, n, values=v, seed=18, is_bigendian=1),
        message("empty_width", base, 16, 0, 5, seed=19),
        message("empty_height", base, 16, 7, 0, seed=20),
        message("no_fields", [], 12, 33, seed=21),
        message("unmatched_types", [("x", 0, I8, 1), ("y", 1, U32, 1), ("z", 5, F64, 1)], 13, 40, seed=22),
        message("huge_point_step", base, 40000, 3, seed=23),
        message("point_step_0", [("ring", 0, U8, 0)], 0, 9, seed=24),
        message("longer_data", base, 16, 100, seed=25, extra=37),
        message("padded_rows_wide", base, 16, 700, 3, 700 * 16 + 4, values=None, seed=26),
        message("width_1_tall", base, 16, 1, 300, 20, seed=27),
        # refusals
        message("short_data", base, 16, 20, 2, data_bytes=2 * 20 * 16 - 1, seed=30, refused=True),
        message("short_row_step", base, 16, 20, 2, 20 * 16 - 1, seed=31, refused=True),
        message("field_past_point_step", [("x", 0, F32, 1), ("intensity", 14, F32, 1)], 16, 10, seed=32, refused=True),
        message("overlapping_fields", [("x", 0, F32, 1), ("y", 2, F32, 1)], 16, 10, seed=33, refused=True),
        message("bad_datatype", [("x", 0, F32, 1), ("ring", 4, 9, 1)], 16, 10, seed=34, refused=True),
        message("bad_datatype_0", [("x", 0, F32, 1), ("ring", 4, 0, 1)], 16, 10, seed=35, refused=True),
    ]
    return out


def case_names():
    return [c["name"] for c in cases()]


_CACHE = {}


def case_by_name(name):
    if not _CACHE:
        _CACHE.update({c["name"]: c for c in cases()})
    return _CACHE[name]


# ---- the numpy restatement: structured dtypes over the message and the records ------------------------------------
def np_decode(case):
    """(records (n, 32) uint8, mapping dict) or None when the layout is refused"""
    fields, w, h = case["fields"], case["width"], case["height"]
    ps, rs = case["point_step"], case["row_step"]
    data = np.ascontiguousarray(case["data"], np.uint8)
    nbytes = case.get("data_bytes", data.nbytes)
    if any(not 1 <= dt <= 8 for _, _, dt, _ in fields) or w * h > 2 ** 31 - 1:
        return None
    matched = {}
    for k in NAMES:   # registration order; the first field with the name, FLOAT32 and count 0 or 1
        for fname, off, dt, cnt in fields:
            if fname == k and dt == F32 and cnt in (0, 1):
                matched[k] = off
                break
    n = w * h
    order = sorted(matched, key=lambda k: matched[k])
    need = 0
    if n:
        if any(matched[k] + 4 > ps for k in order):
            return None
        if any(matched[a] + 4 > matched[b] for a, b in zip(order, order[1:])):
            return None
        if rs < w * ps:
            return None
        need = (h - 1) * rs + w * ps
        if nbytes < need:
            return None
    # groups of fields the coalescing joins: same message-minus-struct shift as the group's first field, in offset order
    groups = []
    for k in order:
        if groups and matched[k] - matched[groups[-1][0]] == STRUCT[k] - STRUCT[groups[-1][0]]:
            groups[-1].append(k)
        else:
            groups.append([k])
    spans = [(matched[g[0]], STRUCT[g[0]], STRUCT[g[-1]] + 4 - STRUCT[g[0]]) for g in groups]
    fast = len(spans) == 1 and spans[0][:2] == (0, 0) and ps == 32
    mp = {"spans": spans, "fast_path": fast, "matched": [k for k in NAMES if k in matched], "points": n,
          "bytes": need}
    rec = np.zeros((h, w), np.dtype([("b", "V32")]))
    if n == 0:
        return rec.view(np.uint8).reshape(0, 32), mp
    copies = [(0, 0, 32)] if fast else spans
    for j, (ser, st, size) in enumerate(copies):
        src_t = np.dtype({"names": ["f"], "formats": [f"V{size}"], "offsets": [ser], "itemsize": max(ps, ser + size)})
        dst_t = np.dtype({"names": ["f"], "formats": [f"V{size}"], "offsets": [st], "itemsize": 32})
        src = np.ndarray((h, w), src_t, buffer=data, offset=0, strides=(rs, ps))
        rec.view(dst_t)["f"][...] = src["f"]
    return rec.view(np.uint8).reshape(n, 32), mp
