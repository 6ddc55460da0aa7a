"""Oracle of the gem_ros_* messages (DESIGN.md f15 W1-W8).  TEST INFRASTRUCTURE ONLY.

- The encoder builds each message with `struct` from the values it carries: oracle layers (oracle_lib's orc_show /
  export_layers), images, records and octree streams.
- The decoder is written independently of the encoder (a cursor over the bytes, field by field, as a ROS1 subscriber
  reads them) and returns the fields as a dict, so that every encoded message can be checked to decode to the values it
  was built from.
- fmt_host(): the library's host framing (gem_b200/csrc/gem_rosfmt.h through tests/rosmsg_fmt_host.cpp), compiled into
  a temporary directory, rendering a whole message from a payload.
"""
from __future__ import annotations

import ctypes as C
import os
import struct

import numpy as np

import native

HERE = os.path.dirname(os.path.abspath(__file__))

GRID_LAYERS = ["elevation", "variance", "rough", "slope", "traver", "color_r", "color_g", "color_b", "intensity"]
ICT_FIELDS = [("x", 0), ("y", 4), ("z", 8), ("rgb", 16), ("intensity", 24), ("covariance", 20), ("travers", 28)]
RGB_FIELDS = [("x", 0), ("y", 4), ("z", 8), ("rgb", 16)]


# ---- W1 ----------------------------------------------------------------------------------------------------------------
def _u32(v):
    return struct.pack("<I", v)


def _string(s: bytes):
    return _u32(len(s)) + s


def header(seq=0, sec=0, nsec=0, frame_id=b""):
    return struct.pack("<III", seq, sec, nsec) + _string(frame_id)


# ---- the encoder ------------------------------------------------------------------------------------------------------
def grid_map(hdr: bytes, L: int, res: float, cx: float, cy: float, start, layers: dict) -> bytes:
    """W2: `layers` maps each of the 9 names to an (L, L) float32 array in grid_map's column-major storage order"""
    out = [hdr, struct.pack("<3d", res, L * res, L * res), struct.pack("<7d", cx, cy, 0.0, 0.0, 0.0, 0.0, 1.0)]
    out.append(_u32(9) + b"".join(_string(n.encode()) for n in GRID_LAYERS))
    out.append(_u32(1) + _string(b"elevation"))
    out.append(_u32(9))
    for n in GRID_LAYERS:
        dims = _u32(2) + _string(b"column_index") + struct.pack("<II", L, L * L) + _string(b"row_index") + struct.pack("<II", L, L)
        data = np.asarray(layers[n], np.float32).reshape(-1, order="F").tobytes()
        out.append(dims + _u32(0) + _u32(L * L) + data)
    out.append(struct.pack("<HH", int(start[0]), int(start[1])))
    return b"".join(out)


def image(hdr: bytes, L: int, bgr: bytes) -> bytes:
    """W3"""
    assert len(bgr) == 3 * L * L
    return hdr + struct.pack("<II", L, L) + _string(b"bgr8") + b"\0" + _u32(3 * L) + _string(bgr)


def cloud(hdr: bytes, fields, records: bytes, is_dense: bool = True) -> bytes:
    """W4: n = len(records) / 32"""
    n = len(records) // 32
    assert len(records) == 32 * n and 32 * n < 1 << 32
    fl = _u32(len(fields)) + b"".join(_string(name.encode()) + struct.pack("<IBI", off, 7, 1) for name, off in fields)
    return hdr + struct.pack("<II", 1, n) + fl + b"\0" + struct.pack("<II", 32, 32 * n) + _string(records) + bytes([int(bool(is_dense))])


def ict_cloud(hdr: bytes, records, is_dense: bool = True) -> bytes:
    """W5 of (n, 8) 32-bit records"""
    return cloud(hdr, ICT_FIELDS, np.ascontiguousarray(records).tobytes(), is_dense)


def visual_records(xyz, rgb) -> np.ndarray:
    """W6's records: {x, y, z, 1.0f, b, g, r, 0xff, 12 zero bytes}"""
    n = xyz.shape[0]
    rec = np.zeros((n, 8), np.uint32)
    rec[:, :3] = np.asarray(xyz, np.float32).view(np.uint32)
    rec[:, 3] = np.float32(1.0).view(np.uint32)
    r, g, b = (np.asarray(rgb[:, k], np.uint32) for k in range(3))
    rec[:, 4] = b | (g << 8) | (r << 16) | np.uint32(0xFF000000)
    return rec


def visual_points(hdr: bytes, xyz, rgb) -> bytes:
    """W6"""
    return cloud(hdr, RGB_FIELDS, visual_records(xyz, rgb).tobytes(), True)


def octomap(hdr: bytes, res: float, stream: bytes) -> bytes:
    """W7"""
    return hdr + b"\0" + _string(b"ColorOcTree") + struct.pack("<d", res) + _string(stream)


def submap(cloud_msg: bytes, keyframe: bytes, image_msg: bytes, pose) -> bytes:
    """W8"""
    return cloud_msg + keyframe + image_msg + struct.pack("<7d", *pose)


# the sizes W2-W7 state
def size_grid_map(f, L):
    return 737 + f + 36 * L * L


def size_image(f, L):
    return 41 + f + 3 * L * L


def size_ict(f, n):
    return 165 + f + 32 * n


def size_visual(f, n):
    return 100 + f + 32 * n


def size_octomap(f, nbytes):
    return 44 + f + nbytes


def grid_layer_offset(f, L, k):
    return 277 + f + k * (57 + 4 * L * L)


# ---- the decoder ------------------------------------------------------------------------------------------------------
class Reader:
    def __init__(self, b: bytes, pos: int = 0):
        self.b, self.p = memoryview(b), pos

    def take(self, n):
        if self.p + n > len(self.b):
            raise ValueError("message too short")
        v = bytes(self.b[self.p:self.p + n])
        self.p += n
        return v

    def num(self, fmt):
        return struct.unpack("<" + fmt, self.take(struct.calcsize("<" + fmt)))[0]

    def string(self):
        return self.take(self.num("I"))

    def header(self):
        return {"seq": self.num("I"), "stamp": (self.num("I"), self.num("I")), "frame_id": self.string()}

    def end(self):
        if self.p != len(self.b):
            raise ValueError(f"{len(self.b) - self.p} bytes left over")


def decode_grid_map(b: bytes) -> dict:
    r = Reader(b)
    d = {"header": r.header(), "resolution": r.num("d"), "length": (r.num("d"), r.num("d")),
         "position": tuple(r.num("d") for _ in range(3)), "orientation": tuple(r.num("d") for _ in range(4))}
    d["layers"] = [r.string().decode() for _ in range(r.num("I"))]
    d["basic_layers"] = [r.string().decode() for _ in range(r.num("I"))]
    d["data"] = []
    for _ in range(r.num("I")):
        dims = [(r.string().decode(), r.num("I"), r.num("I")) for _ in range(r.num("I"))]
        off = r.num("I")
        n = r.num("I")
        d["data"].append({"dims": dims, "data_offset": off, "data": np.frombuffer(r.take(4 * n), "<f4")})
    d["start"] = (r.num("H"), r.num("H"))
    r.end()
    return d


def decode_image(b: bytes, pos: int = 0, whole: bool = True):
    r = Reader(b, pos)
    d = {"header": r.header(), "height": r.num("I"), "width": r.num("I"), "encoding": r.string().decode(),
         "is_bigendian": r.num("B"), "step": r.num("I")}
    d["data"] = r.string()
    if whole:
        r.end()
    return (d, r.p) if not whole else d


def decode_cloud(b: bytes, pos: int = 0, whole: bool = True):
    r = Reader(b, pos)
    d = {"header": r.header(), "height": r.num("I"), "width": r.num("I")}
    d["fields"] = [(r.string().decode(), r.num("I"), r.num("B"), r.num("I")) for _ in range(r.num("I"))]
    d.update(is_bigendian=r.num("B"), point_step=r.num("I"), row_step=r.num("I"))
    d["data"] = r.string()
    d["is_dense"] = r.num("B")
    if whole:
        r.end()
    return (d, r.p) if not whole else d


def decode_octomap(b: bytes) -> dict:
    r = Reader(b)
    d = {"header": r.header(), "binary": r.num("B"), "id": r.string().decode(), "resolution": r.num("d"), "data": r.string()}
    r.end()
    return d


def decode_submap(b: bytes, keyframe_len: int) -> dict:
    """W8 with a keyframe message of keyframe_len bytes (it is opaque here)"""
    sub, p = decode_cloud(b, 0, whole=False)
    kf = b[p:p + keyframe_len]
    img, p = decode_image(b, p + keyframe_len, whole=False)
    pose = struct.unpack("<7d", b[p:p + 56])
    if p + 56 != len(b):
        raise ValueError("bytes left over")
    return {"submap": sub, "keyframePC": kf, "orthoImage": img, "pose": pose}


# ---- the library's host framing (gem_rosfmt.h) ------------------------------------------------------------------------
_fmt = None


def fmt_host():
    """ctypes binding of tests/rosmsg_fmt_host.cpp (g++, into a temporary directory)"""
    global _fmt
    if _fmt is None:
        lib = native.shared_library("rosfmt_host", [os.path.join(HERE, "rosmsg_fmt_host.cpp")], native.FORMAT_CXX)
        ll, P = C.c_longlong, C.c_void_p
        hdr = [C.c_uint, C.c_uint, C.c_uint, C.c_char_p]
        lib.ros_fmt_grid_map.argtypes = hdr + [C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, C.c_int, P, P, ll]
        lib.ros_fmt_image.argtypes = hdr + [C.c_int, P, P, ll]
        lib.ros_fmt_cloud.argtypes = hdr + [C.c_int, ll, C.c_int, P, P, ll]
        lib.ros_fmt_octomap.argtypes = hdr + [C.c_double, ll, P, P, ll]
        for f in (lib.ros_fmt_grid_map, lib.ros_fmt_image, lib.ros_fmt_cloud, lib.ros_fmt_octomap):
            f.restype = ll
        _fmt = lib
    return _fmt


def host_render(kind: str, hdr: tuple, args: tuple, payload: bytes, capacity: int | None = None):
    """the message gem_rosfmt.h frames around `payload` (the payload runs back to back); returns bytes, or the call's
    negative status as an int when the framing refuses"""
    lib = fmt_host()
    seq, sec, nsec, fid = hdr
    pay = np.frombuffer(payload, np.uint8) if payload else np.zeros(1, np.uint8)
    cap = capacity if capacity is not None else 4096 + len(payload) + 2 * len(fid)
    out = np.full(max(cap, 1), 0xA5, np.uint8)
    fn = {"grid_map": lib.ros_fmt_grid_map, "image": lib.ros_fmt_image, "cloud": lib.ros_fmt_cloud,
          "octomap": lib.ros_fmt_octomap}[kind]
    n = fn(seq, sec, nsec, fid, *args, pay.ctypes.data, out.ctypes.data, cap)
    if n < 0:
        return n
    return out[:n].tobytes()
