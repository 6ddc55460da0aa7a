"""The PCD writer's definitions without a GPU (DESIGN.md f13): the C oracle (tests/orc_pcd.c, glibc's snprintf) against
the independent Python restatement on crafted clouds; gem_pcd_header (host code) against both; the library's float
formatter (gem_b200/csrc/gem_pcdfmt.h, host build) against snprintf("%.8g") on every exponent's first and last mantissas,
every exact tie at the 9th digit, decade and style boundaries, the special values and 10^7 seeded random patterns; the
rgb field over every colour with a = 0xff and a = 0, as a float and as a uint32."""
import ctypes as C

import numpy as np
import pytest

import gem_b200
import pcd_cases as pc
import pcd_oracle as po
from gem_b200 import GemError, _lib

FLAGS = [0, po.BINARY, po.RGB_UINT32, po.BINARY | po.RGB_UINT32]


@pytest.mark.parametrize("name", pc.case_names())
@pytest.mark.parametrize("flags", FLAGS)
def test_oracle_matches_python_restatement(name, flags):
    rec = pc.cloud(name)
    got = po.data(rec, flags)
    assert got is not None and got == po.py_data(rec, flags)
    if flags & po.BINARY:
        assert len(got) == 28 * rec.shape[0]
    else:
        lines = got.split(b"\n")
        assert lines[-1] == b"" and len(lines) == rec.shape[0] + 1
        assert max(len(s) for s in lines) + 1 <= _lib.PCD_LINE_MAX
        assert all(len(s.split(b" ")) == 7 for s in lines[:-1])


def test_oracle_refuses_what_pcl_throws_on():
    assert po.data(np.zeros((0, 8), np.uint32)) is None and po.py_data(np.zeros((0, 8), np.uint32)) is None
    assert po.header(0) is None and po.py_header(0) is None
    assert po.data(pc.harvest_like(3), 4) is None


@pytest.mark.parametrize("n", [1, 2, 7, 255, 256, 1 << 20, (1 << 31) - 1, 1 << 31, 10 ** 18])
@pytest.mark.parametrize("flags", FLAGS)
def test_header_matches_oracles(n, flags):
    want = po.header(n, flags)
    assert want == po.py_header(n, flags)
    assert gem_b200.ElevationMap.pcd_header(n, bool(flags & po.BINARY), bool(flags & po.RGB_UINT32)) == want
    lib, k = _lib.load(), C.c_int(-1)
    assert lib.gem_pcd_header(n, flags, None, 0, C.byref(k)) == 0 and k.value == len(want)   # size query
    buf = C.create_string_buffer(b"S" * 600, 600)
    assert lib.gem_pcd_header(n, flags, buf, len(want), C.byref(k)) == 0 and k.value == len(want)   # no room for the NUL
    assert buf.raw == b"S" * 600
    assert lib.gem_pcd_header(n, flags, buf, len(want) + 1, C.byref(k)) == 0
    assert buf.raw[:len(want) + 1] == want + b"\0" and buf.raw[len(want) + 1:] == b"S" * (599 - len(want))
    assert len(want) < _lib.PCD_HEADER_MAX


@pytest.mark.parametrize("n,flags", [(0, 0), (0, 1), (-1, 0), (5, 4), (5, -1), (5, 8)])
def test_header_refusals_write_nothing(n, flags):
    lib, k = _lib.load(), C.c_int(-1)
    buf = C.create_string_buffer(b"S" * 600, 600)
    assert lib.gem_pcd_header(n, flags, buf, 600, C.byref(k)) == 1 and k.value == 0
    assert buf.raw == b"S" * 600
    if flags in (0, 1):
        with pytest.raises(GemError):
            gem_b200.ElevationMap.pcd_header(n, binary=bool(flags))


def _formatter_agrees(bits, as_uint=False):
    bad, first = po.fmt_compare_list(bits, as_uint)
    assert bad == 0, f"{bad} patterns differ from snprintf, first 0x{first:08x}: {po.fmt_one(first)!r}"


def test_formatter_examples():
    want = [(0.0, "0"), (-0.0, "-0"), (1.0, "1"), (2.0 ** -12, "0.00024414062"), (0.000732421875, "0.00073242188"),
            (2.0 ** -149, "1.4012985e-45"), (3.4028234663852886e38, "3.4028235e+38"), (float("inf"), "inf"),
            (float("-inf"), "-inf"), (12345678.0, "12345678"), (99999999.0, "1e+08"), (123456789.0, "1.2345679e+08"),
            (-1.2345678e-38, "-1.2345678e-38"), (-0.00012345678, "-0.00012345678"), (0.1, "0.1")]
    for v, s in want:
        assert po.fmt_one(int(pc.f2u(v))) == s, v
    assert po.fmt_one(0x7FC00000) == "nan" and po.fmt_one(0xFFC00001) == "nan"
    # %g's style follows the exponent after rounding: the floats on either side of 1e-4 and of 1e8
    b = int(pc.f2u(1e-4))
    assert (po.fmt_one(b), po.fmt_one(b + 1)) == ("9.9999997e-05", "0.0001")
    b = int(pc.f2u(1e8))
    assert (po.fmt_one(b - 1), po.fmt_one(b)) == ("99999992", "1e+08")
    assert po.fmt_one(0xFF000000, as_uint=True) == "4278190080"


def test_formatter_every_exponent_edge():
    _formatter_agrees(pc.exponent_edges(16))


def test_formatter_every_tie():
    t = pc.ties()
    assert t.size > 10 ** 7 and int(t[0]) == int(pc.f2u(2.0 ** -12))
    # every one is a tie: 9 significant digits ending in 5
    for b in t[:: t.size // 997]:
        s = "%.9e" % float(np.uint32(b).view(np.float32))
        assert s[9] == "5" and float(s) == float(np.uint32(b).view(np.float32))
    _formatter_agrees(t)
    _formatter_agrees(t[::7] | np.uint32(0x80000000))


def test_formatter_boundaries_and_specials():
    _formatter_agrees(pc.boundaries(8))
    _formatter_agrees(pc.specials())
    assert po.fmt_compare_range(0, 1 << 20) == (0, None)                       # every subnormal below 2^-129
    assert po.fmt_compare_range(0x7F800000, 0x7F800000 + (1 << 20)) == (0, None)   # inf and NaNs


def test_formatter_random_patterns():
    bits = np.random.default_rng(20261018).integers(0, 1 << 32, 10 ** 7 + 1, dtype=np.uint64).astype(np.uint32)
    _formatter_agrees(bits)


def test_rgb_every_colour_both_forms():
    c = np.arange(1 << 24, dtype=np.uint32)
    for a in (0xFF000000, 0):
        _formatter_agrees(c | np.uint32(a))
        _formatter_agrees(c | np.uint32(a), as_uint=True)
    # both forms inside whole lines (the other fields as the oracle prints them)
    rec = pc.harvest_like(4096, 9)
    for a in (0xFF000000, 0):
        rec[:, 4] = c[::4096] | np.uint32(a)
        for flags in (0, po.RGB_UINT32):
            assert po.fmt_ascii(rec, bool(flags)) == po.data(rec, flags) == po.py_data(rec, flags)
    # a = 0xff makes the float form lose the colour: nan, -inf or a huge negative number
    assert po.fmt_one(0xFF80FFFF) == "nan" and po.fmt_one(0xFF800000) == "-inf" and po.fmt_one(0xFF7F0000).startswith("-3.3")
