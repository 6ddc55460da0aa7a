"""The PointCloud2 ingest, CPU side (DESIGN.md f12): the oracle (tests/orc_pointcloud2.c) against the independent numpy
restatement of tests/pc2_cases.py, record bytes and mapping, on every crafted case; gem_pointcloud2_mapping (host code,
no GPU) against both; what the crafted cases are there to show; the ctypes mirrors of the new structs against the C
compiler's layout of include/gem_b200.h."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import native
import pc2_cases as pc
import pc2_oracle
from gem_b200 import ElevationMap, GemError, PointCloud2Layout, _lib


def layout(case):
    return PointCloud2Layout(case["fields"], case["width"], case["height"], case["point_step"], case["row_step"],
                             case["is_bigendian"])


def data_bytes(case):
    return case.get("data_bytes", case["data"].nbytes)


@pytest.mark.parametrize("name", pc.case_names())
def test_oracle_matches_restatement_and_library_mapping(name):
    case = pc.case_by_name(name)
    got, want = pc2_oracle.decode(case), pc.np_decode(case)
    if case["refused"]:
        assert got is None and want is None, name
        with pytest.raises(GemError):
            ElevationMap.pointcloud2_mapping(layout(case), data_bytes(case))
        return
    assert got is not None and want is not None, name
    (grec, gmap), (wrec, wmap) = got, want
    assert gmap == wmap, (name, gmap, wmap)
    assert grec.shape == wrec.shape and grec.tobytes() == wrec.tobytes(), name
    assert ElevationMap.pointcloud2_mapping(layout(case), data_bytes(case)) == gmap


def rec_f32(case, field):
    rec, _ = pc2_oracle.decode(case)
    return rec[:, pc.STRUCT[field]:pc.STRUCT[field] + 4].copy().view(np.uint32).reshape(-1)


def msg_u32(case, off):
    d, w, ps = case["data"], case["width"], case["point_step"]
    idx = np.arange(w)[:, None] * ps + off + np.arange(4)[None, :]
    return d[idx].copy().view(np.uint32).reshape(-1)


def test_what_the_cases_show():
    c = pc.case_by_name
    # fast path: whole points, unmapped bytes too
    m = pc2_oracle.decode(c("one_span_point_step_32"))[1]
    assert m["fast_path"] and m["spans"] == [(0, 0, 12)] and m["matched"] == ["x", "y", "z"]
    assert (rec_f32(c("one_span_point_step_32"), "intensity") == msg_u32(c("one_span_point_step_32"), 24)).all()
    assert pc2_oracle.decode(c("xyzrgbict"))[1]["fast_path"]
    assert not pc2_oracle.decode(c("xyzir32"))[1]["fast_path"]
    # a float64 y between matched x and z takes the 4 message bytes between them
    m = pc2_oracle.decode(c("float64_y_filled_by_merge"))[1]
    assert m["spans"] == [(0, 0, 12), (12, 24, 4)] and "y" not in m["matched"]
    assert (rec_f32(c("float64_y_filled_by_merge"), "y") == msg_u32(c("float64_y_filled_by_merge"), 4)).all()
    # the merged x..travers span is copied after intensity's own and overwrites it with message bytes 28..31
    m = pc2_oracle.decode(c("merge_overwrites_intensity"))[1]
    assert m["spans"] == [(0, 24, 4), (4, 0, 32)]
    assert (rec_f32(c("merge_overwrites_intensity"), "intensity") == msg_u32(c("merge_overwrites_intensity"), 28)).all()
    # first equal name wins, a FLOAT64 or count-2 field does not match
    assert pc2_oracle.decode(c("duplicate_names"))[1]["spans"] == [(8, 8, 4), (12, 0, 8)]
    assert pc2_oracle.decode(c("count_0_and_2"))[1]["matched"] == ["x", "z", "intensity"]
    assert pc2_oracle.decode(c("float64_x"))[1]["matched"] == ["y", "z", "intensity"]
    assert (rec_f32(c("float64_x"), "x") == 0).all()
    # uint16 intensity: DEFINED 0 (stale bytes in the reference)
    assert (rec_f32(c("ouster"), "intensity") == 0).all()
    # the field order of the message does not matter; is_bigendian is not read
    assert pc2_oracle.decode(c("reverse_order"))[1]["spans"] == [(0, 0, 32)]
    a, b = pc2_oracle.decode(c("is_bigendian"))[0], pc.np_decode(dict(c("is_bigendian"), is_bigendian=0))[0]
    assert a.tobytes() == b.tobytes()
    # bit patterns survive
    sb = pc2_oracle.xyzi(pc2_oracle.decode(c("special_bits"))[0]).view(np.uint32)
    assert (sb[:12, 0] == pc._special_bits().view(np.uint32)).all()
    assert pc2_oracle.decode(c("empty_width"))[0].shape == (0, 32)
    # the organised D435 cloud: padded rows, rgb matched, intensity 0
    rec, m = pc2_oracle.decode(c("d435_organised_padded"))
    assert rec.shape == (307200, 32) and m["matched"] == ["x", "y", "z", "rgb"] and len(m["spans"]) == 2
    assert (rec[:, 24:28] == 0).all()


def test_real_layouts_carry_the_cloud():
    from gem_b200 import synth
    hdl = synth.hdl64_frame(0)["xyzi"][:3000]
    for lay in ("kitti16", "xyzir32", "xyzir22", "pandarqt", "xyzrgbict"):
        got = pc2_oracle.xyzi(pc2_oracle.decode(pc.case_by_name(lay))[0])
        assert got.tobytes() == hdl.tobytes(), lay


def test_mapping_refusals_leave_the_output_alone():
    lib = _lib.load()
    case = pc.case_by_name("overlapping_fields")
    L = layout(case)
    mp = _lib.GemPc2Mapping()
    mp.nspans = 77
    assert lib.gem_pointcloud2_mapping(C.byref(L.c), 10 ** 6, C.byref(mp)) == 1 and mp.nspans == 77
    assert b"overlap" in lib.gem_last_error(None)
    assert lib.gem_pointcloud2_mapping(None, 0, C.byref(mp)) == 1
    assert lib.gem_pointcloud2_mapping(C.byref(L.c), 0, None) == 1


def test_numpy_dtype_layout():
    dt = np.dtype({"names": ["x", "y", "z", "intensity", "t", "ring"], "formats": ["<f4", "<f4", "<f4", "<f4", "<f8", "<u2"],
                   "offsets": [0, 4, 8, 16, 24, 32], "itemsize": 48})
    L = PointCloud2Layout(dt, 10)
    assert L.point_step == 48 and L.row_step == 480
    assert L.fields == [("x", 0, 7, 1), ("y", 4, 7, 1), ("z", 8, 7, 1), ("intensity", 16, 7, 1), ("t", 24, 8, 1), ("ring", 32, 4, 1)]
    assert ElevationMap.pointcloud2_mapping(L)["spans"] == [(0, 0, 12), (16, 24, 4)]
    L2 = PointCloud2Layout(np.dtype([("x", "<f4", (2,)), ("z", "<f4")]), 1)
    assert L2.fields == [("x", 0, 7, 2), ("z", 8, 7, 1)]


STRUCTS = {
    "gem_pointfield": (_lib.GemPointField, ["name", "offset", "datatype", "count"]),
    "gem_pointcloud2": (_lib.GemPointCloud2, ["width", "height", "point_step", "row_step", "is_bigendian", "nfields", "fields"]),
    "gem_pc2_span": (_lib.GemPc2Span, ["serialized_offset", "struct_offset", "size"]),
    "gem_pc2_mapping": (_lib.GemPc2Mapping, ["nspans", "spans", "fast_path", "matched", "points", "bytes"]),
    "gem_camera_image": (_lib.GemCameraImage, ["T_camera", "T_lidar", "encoding", "width", "height", "step", "data"]),
}


def test_struct_layouts_match_the_header():
    for s, (cls, fields) in STRUCTS.items():
        assert set(fields) <= {f for f, _ in cls._fields_}, s
    native.assert_struct_layouts({s: cls for s, (cls, _) in STRUCTS.items()}, std=None)
    # the oracle's mirrors too
    for cls, ref in ((pc2_oracle.Field, _lib.GemPointField), (pc2_oracle.Cloud, _lib.GemPointCloud2),
                     (pc2_oracle.Mapping, _lib.GemPc2Mapping)):
        assert C.sizeof(cls) == C.sizeof(ref)


FACADE = r"""
#include <cstdio>
#include "gem_b200/elevation_map.hpp"
int main()
{
    gem_b200::PointCloud2Layout lay(10, 1, 22, 220);   // velodyne XYZIRT, packed
    lay.addField("x", 0, GEM_PF_FLOAT32, 1); lay.addField("y", 4, GEM_PF_FLOAT32, 1); lay.addField("z", 8, GEM_PF_FLOAT32, 1);
    lay.addField("intensity", 12, GEM_PF_FLOAT32, 1); lay.addField("ring", 16, GEM_PF_UINT16, 1); lay.addField("time", 18, GEM_PF_FLOAT32, 1);
    const gem_pc2_mapping m = lay.mapping(220);
    std::printf("%d %u %u %u %u %u %u %d %u\n", m.nspans, m.spans[0].serialized_offset, m.spans[0].struct_offset, m.spans[0].size,
                m.spans[1].serialized_offset, m.spans[1].struct_offset, m.spans[1].size, m.fast_path, m.matched);
    try { lay.mapping(219); } catch (const std::runtime_error &) { std::printf("refused\n"); }
    return 0;
}
"""


def test_cxx_facade_layout_and_mapping(tmp_path):
    src = tmp_path / "f.cpp"
    src.write_text(FACADE)
    exe = native.facade_program("f", tmp_path, sources=[str(src)], flags=["-std=c++14", "-Wall", "-Wextra", "-Werror"])
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split("\n")
    assert out[0] == "2 0 0 12 12 24 4 0 23" and out[1] == "refused", out
