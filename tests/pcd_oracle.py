"""Oracles of gem_pcd_header / gem_pcd_format (DESIGN.md f13).  TEST INFRASTRUCTURE ONLY.

- header() / data(): ctypes binding of tests/orc_pcd.c, the C restatement of PCL's generateHeader / writeASCII /
  writeBinary for PointXYZRGBICT (glibc's snprintf("%.8g") per value).
- py_header() / py_data(): an independent Python restatement ('%.8g' % v is CPython's own dtoa, not glibc's).
- the host build of the library's formatter (tests/pcd_fmt_host.cpp + gem_b200/csrc/gem_pcdfmt.h): fmt_one(),
  fmt_compare_range(), fmt_compare_list() (against snprintf) and fmt_ascii() (a whole data section).

Both libraries are compiled into a temporary directory (the checkout may be read-only).  Records are (n, 8) float32 or
uint32 arrays (32-byte PointXYZRGBICT records); flags are GEM_PCD_BINARY = 1 and GEM_PCD_RGB_UINT32 = 2."""
from __future__ import annotations

import ctypes as C
import math
import os
import struct

import numpy as np

import native

HERE = os.path.dirname(os.path.abspath(__file__))
BINARY, RGB_UINT32 = 1, 2
FIELDS = ["x", "y", "z", "rgb", "intensity", "covariance", "travers"]
WORDS = [0, 1, 2, 4, 6, 5, 7]     # each field's 32-bit word in the record, in registration order
_orc = None
_fmt = None


def load():
    global _orc
    if _orc is None:
        lib = native.shared_library("orc_pcd", [os.path.join(HERE, "orc_pcd.c")], native.FORMAT_C, ["-lm"])
        lib.orc_pcd_header.argtypes = [C.c_longlong, C.c_int, C.c_char_p, C.c_int]
        lib.orc_pcd_header.restype = C.c_int
        lib.orc_pcd_data.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p, C.c_longlong]
        lib.orc_pcd_data.restype = C.c_longlong
        _orc = lib
    return _orc


def load_fmt():
    global _fmt
    if _fmt is None:
        lib = native.shared_library("pcd_fmt_host", [os.path.join(HERE, "pcd_fmt_host.cpp")], native.FORMAT_CXX, ["-lm"])
        lib.pcd_fmt_one.argtypes = [C.c_uint32, C.c_int, C.c_char_p]
        lib.pcd_fmt_one.restype = C.c_int
        lib.pcd_fmt_compare_range.argtypes = [C.c_uint64, C.c_uint64, C.POINTER(C.c_uint32)]
        lib.pcd_fmt_compare_range.restype = C.c_longlong
        lib.pcd_fmt_compare_list.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.POINTER(C.c_uint32)]
        lib.pcd_fmt_compare_list.restype = C.c_longlong
        lib.pcd_fmt_ascii.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p]
        lib.pcd_fmt_ascii.restype = C.c_longlong
        _fmt = lib
    return _fmt


def _records(rec):
    return np.ascontiguousarray(np.asarray(rec).reshape(-1, 8)).view(np.uint32)


# ---- the C oracle ---------------------------------------------------------------------------------------------------
def header(n, flags=0):
    """the header bytes, or None where PCL throws"""
    buf = C.create_string_buffer(1024)
    k = load().orc_pcd_header(int(n), int(flags), buf, 1024)
    return None if k < 0 else buf.raw[:k]


def data(rec, flags=0):
    """the data section bytes, or None where PCL throws"""
    r = _records(rec)
    n = r.shape[0]
    k = load().orc_pcd_data(C.c_void_p(r.ctypes.data), n, int(flags), None, 0)
    if k < 0:
        return None
    out = np.empty(max(k, 1), np.uint8)
    load().orc_pcd_data(C.c_void_p(r.ctypes.data), n, int(flags), C.c_void_p(out.ctypes.data), k)
    return out[:k].tobytes()


def file_bytes(rec, flags=0):
    """what savePCDFile writes: header and data"""
    return header(_records(rec).shape[0], flags) + data(rec, flags)


# ---- the Python restatement -----------------------------------------------------------------------------------------
def py_header(n, flags=0):
    if n <= 0 or flags & ~3:
        return None
    return ("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\n"
            f"FIELDS {' '.join(FIELDS)}\nSIZE {' '.join(['4'] * 7)}\nTYPE {' '.join(['F'] * 7)}\n"
            f"COUNT {' '.join(['1'] * 7)}\nWIDTH {n}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\n"
            f"DATA {'binary' if flags & BINARY else 'ascii'}\n").encode()


def py_value(bits, as_uint=False):
    if as_uint:
        return str(int(bits))
    v = struct.unpack("<f", struct.pack("<I", int(bits)))[0]
    return "nan" if math.isnan(v) else "%.8g" % v


def py_data(rec, flags=0):
    r = _records(rec)
    if r.shape[0] == 0 or flags & ~3:
        return None
    if flags & BINARY:
        return np.ascontiguousarray(r[:, WORDS]).tobytes()
    uint_rgb = bool(flags & RGB_UINT32)
    lines = [" ".join(py_value(row[w], uint_rgb and f == 3) for f, w in enumerate(WORDS)) + "\n" for row in r.tolist()]
    return "".join(lines).encode()


# ---- the library's formatter, host build ----------------------------------------------------------------------------
def fmt_one(bits, as_uint=False):
    buf = C.create_string_buffer(32)
    k = load_fmt().pcd_fmt_one(int(bits) & 0xFFFFFFFF, 1 if as_uint else 0, buf)
    return buf.raw[:k].decode()


def fmt_compare_range(lo, hi):
    """(mismatches against snprintf over the bit patterns [lo, hi), the first one)"""
    first = C.c_uint32(0)
    bad = load_fmt().pcd_fmt_compare_range(int(lo), int(hi), C.byref(first))
    return bad, (first.value if bad else None)


def fmt_compare_list(bits, as_uint=False):
    """(mismatches against snprintf -- "%.8g", or "%u" with as_uint -- over the listed bit patterns, the first one)"""
    b = np.ascontiguousarray(bits, np.uint32)
    first = C.c_uint32(0)
    bad = load_fmt().pcd_fmt_compare_list(C.c_void_p(b.ctypes.data), b.size, 1 if as_uint else 0, C.byref(first))
    return bad, (first.value if bad else None)


def fmt_ascii(rec, rgb_uint32=False):
    """the ASCII data section the formatter's host build assembles"""
    r = _records(rec)
    out = np.empty(max(r.shape[0] * 105, 1), np.uint8)
    k = load_fmt().pcd_fmt_ascii(C.c_void_p(r.ctypes.data), r.shape[0], 1 if rgb_uint32 else 0, C.c_void_p(out.ctypes.data))
    return out[:k].tobytes()
