"""The ROS message definitions without a GPU (DESIGN.md f15): the struct encoder of tests/rosmsg_oracle.py decodes
back to the values it was built from, its messages have the sizes W2-W7 state, the library's host framing
(gem_b200/csrc/gem_rosfmt.h) renders the oracle's bytes for every map size, frame_id length and cloud, and refuses what
the framing decides (32 n >= 2^32, negative counts)."""
import struct

import numpy as np
import pytest

import rosmsg_cases as rc
import rosmsg_oracle as ro
from oracle_lib import OracleMap

f32 = np.float32


def _layers(L, seed):
    rng = np.random.default_rng(seed)
    out = {}
    for n in ro.GRID_LAYERS:
        a = rng.integers(0, 1 << 32, (L, L), dtype=np.uint64).astype(np.uint32).view(f32)
        out[n] = np.asfortranarray(a)
    return out


def _hdr(fid_len, seq=7):
    fid = rc.frame_id(fid_len).encode()
    return (seq, 1700000000 + fid_len, 123456 * fid_len, fid), ro.header(seq, 1700000000 + fid_len, 123456 * fid_len, fid)


def _payload_grid(layers):
    return b"".join(np.asarray(layers[n], f32).reshape(-1, order="F").tobytes() for n in ro.GRID_LAYERS)


@pytest.mark.parametrize("L", rc.MAP_SIZES)
def test_grid_map_encode_decode_size_and_host_framing(L):
    layers = _layers(L, L)
    for fl in rc.FRAME_ID_LENGTHS:
        h, hb = _hdr(fl)
        msg = ro.grid_map(hb, L, 0.1, 1.25, -3.5, (L // 3, L - 1), layers)
        assert len(msg) == ro.size_grid_map(fl, L)
        for k, n in enumerate(ro.GRID_LAYERS):
            o = ro.grid_layer_offset(fl, L, k)
            assert msg[o:o + 4 * L * L] == np.asarray(layers[n], f32).reshape(-1, order="F").tobytes()
        d = ro.decode_grid_map(msg)
        assert d["header"] == {"seq": 7, "stamp": (h[1], h[2]), "frame_id": h[3]}
        assert d["resolution"] == 0.1 and d["length"] == (L * 0.1, L * 0.1)
        assert d["position"] == (1.25, -3.5, 0.0) and d["orientation"] == (0.0, 0.0, 0.0, 1.0)
        assert d["layers"] == ro.GRID_LAYERS and d["basic_layers"] == ["elevation"] and d["start"] == (L // 3, L - 1)
        for k, n in enumerate(ro.GRID_LAYERS):
            e = d["data"][k]
            assert e["dims"] == [("column_index", L, L * L), ("row_index", L, L)] and e["data_offset"] == 0
            assert e["data"].tobytes() == np.asarray(layers[n], f32).reshape(-1, order="F").tobytes()
        assert ro.host_render("grid_map", h, (L, 0.1, 1.25, -3.5, L // 3, L - 1), _payload_grid(layers)) == msg
    # every layer meets all 16 byte phases over the frame_id lengths 0-15
    for k in range(9):
        assert {ro.grid_layer_offset(fl, L, k) % 16 for fl in range(16)} == set(range(16))


@pytest.mark.parametrize("L", rc.MAP_SIZES)
def test_image_encode_decode_size_and_host_framing(L):
    bgr = np.random.default_rng(L).integers(0, 256, 3 * L * L, dtype=np.uint8).tobytes()
    for fl in (0, 1, 5, 17, 300):
        h, hb = _hdr(fl, seq=0)
        msg = ro.image(hb, L, bgr)
        assert len(msg) == ro.size_image(fl, L)
        d = ro.decode_image(msg)
        assert (d["height"], d["width"], d["encoding"], d["is_bigendian"], d["step"], d["data"]) == (L, L, "bgr8", 0, 3 * L, bgr)
        assert ro.host_render("image", h, (L,), bgr) == msg


@pytest.mark.parametrize("name", sorted(rc.cloud_parts()))
def test_clouds_encode_decode_size_and_host_framing(name):
    parts = rc.cloud_parts()[name]
    rec = np.concatenate(parts) if parts else np.zeros((0, 8), np.uint32)
    n = rec.shape[0]
    for fl in (0, 3, 20, 300):
        h, hb = _hdr(fl)
        for dense in (True, False):
            msg = ro.ict_cloud(hb, rec, dense)
            assert len(msg) == ro.size_ict(fl, n)
            d = ro.decode_cloud(msg)
            assert (d["height"], d["width"], d["is_bigendian"], d["point_step"], d["row_step"], d["is_dense"]) == (1, n, 0, 32, 32 * n, int(dense))
            assert d["fields"] == [(f, o, 7, 1) for f, o in ro.ICT_FIELDS] and d["data"] == rec.tobytes()
            assert ro.host_render("cloud", h, (0, n, int(dense)), rec.tobytes()) == msg
        xyz = rec[:, :3].view(f32)
        rgb = (rec[:, 4:7] & 255).astype(np.uint8)
        msg = ro.visual_points(hb, xyz, rgb)
        assert len(msg) == ro.size_visual(fl, n)
        d = ro.decode_cloud(msg)
        assert d["fields"] == [(f, o, 7, 1) for f, o in ro.RGB_FIELDS] and d["is_dense"] == 1
        got = np.frombuffer(d["data"], np.uint32).reshape(-1, 8)
        assert got[:, :3].tobytes() == xyz.tobytes() and (got[:, 3] == 0x3F800000).all() and (got[:, 5:] == 0).all()
        assert (got[:, 4] == ((rgb[:, 2].astype(np.uint32)) | (rgb[:, 1].astype(np.uint32) << 8) |
                              (rgb[:, 0].astype(np.uint32) << 16) | 0xFF000000)).all()
        assert ro.host_render("cloud", h, (1, n, 1), ro.visual_records(xyz, rgb).tobytes()) == msg


@pytest.mark.parametrize("nbytes", [0, 8, 8 * 12345])
def test_octomap_encode_decode_size_and_host_framing(nbytes):
    stream = np.random.default_rng(nbytes).integers(0, 256, nbytes, dtype=np.uint8).tobytes()
    for fl in (0, 9, 300):
        h, hb = _hdr(fl, seq=0)
        msg = ro.octomap(hb, 0.2, stream)
        assert len(msg) == ro.size_octomap(fl, nbytes)
        d = ro.decode_octomap(msg)
        assert (d["binary"], d["id"], d["resolution"], d["data"]) == (0, "ColorOcTree", 0.2, stream)
        assert ro.host_render("octomap", h, (0.2, nbytes), stream) == msg


def test_submap_encode_decode():
    rec = rc.records(40, 9)
    _, hb = _hdr(3, seq=0)
    cloud = ro.ict_cloud(hb, rec)
    kf = b"\x01\x02keyframe bytes as received"
    img = ro.image(ro.header(), 2, bytes(range(12)))
    pose = (1.0, -2.0, 0.5, 0.0, 0.0, 0.38268343236508984, 0.9238795325112867)
    msg = ro.submap(cloud, kf, img, pose)
    assert len(msg) == len(cloud) + len(kf) + len(img) + 56
    d = ro.decode_submap(msg, len(kf))
    assert d["submap"]["data"] == rec.tobytes() and d["keyframePC"] == kf and d["orthoImage"]["data"] == bytes(range(12))
    assert d["pose"] == pose


def test_framing_refusals():
    h = (0, 0, 0, b"map")
    assert ro.host_render("cloud", h, (0, 1 << 27, 1), b"") == -1          # 32 n == 2^32
    assert ro.host_render("cloud", h, (0, -1, 1), b"") == -1
    assert ro.host_render("cloud", h, (1, (1 << 27) - 1, 1), b"", capacity=16) == -2   # framed, larger than the buffer
    assert ro.host_render("octomap", h, (0.1, -8), b"") == -1
    assert ro.host_render("octomap", h, (0.1, 1 << 32), b"") == -1
    assert ro.host_render("grid_map", h, (32768, 0.1, 0.0, 0.0, 0, 0), b"") == -1   # 4 L^2 == 2^32
    assert ro.host_render("grid_map", h, (0, 0.1, 0.0, 0.0, 0, 0), b"") == -1


@pytest.mark.parametrize("name", ["L5_scrolled", "L33_opt_move"])
def test_oracle_show_messages_decode(name):
    c = rc.case(name)
    o = OracleMap(c.L, c.res, compat_box_filter=False)
    c.apply(o)
    layers = o.export_layers()
    img, xyz, rgb = o.show()
    centre, start, _ = o.state()
    hb = ro.header(0, 0, 0, b"map")
    msg = ro.grid_map(hb, c.L, float(f32(c.res)), float(centre[0]), float(centre[1]), start, layers)
    d = ro.decode_grid_map(msg)
    assert d["start"] == tuple(int(s) for s in start) and d["position"][:2] == (float(centre[0]), float(centre[1]))
    for k, n in enumerate(ro.GRID_LAYERS):
        assert d["data"][k]["data"].tobytes() == layers[n].reshape(-1, order="F").tobytes()
    assert ro.decode_image(ro.image(ro.header(), c.L, img.tobytes()))["data"] == img.tobytes()
    v = ro.decode_cloud(ro.visual_points(hb, xyz, rgb))
    assert v["width"] == xyz.shape[0] and struct.unpack_from("<3f", v["data"], 0) == tuple(float(x) for x in xyz[0])
