"""PCD files on the device (DESIGN.md f13): gem_pcd_format's bytes equal the oracle's (tests/orc_pcd.c) in ASCII and
binary, with rgb as a float and as a uint32, on one record, the crafted clouds of tests/pcd_cases.py, the records the
library's producers make (harvests, the grid cloud, the local map, the dense keyframe cut, the MLS points) and a 2 M
record cloud; the device formatter equals its host build on 2^26 random bit patterns and snprintf on 2^24 of them;
save_pcd's files (host and device records, chunked and one-shot) equal the oracle's; refusals write nothing; the C++
facade's files equal Python's."""
import ctypes as C
import subprocess

import numpy as np
import pytest
import torch

import gem_b200
import native
import pcd_cases as pc
import pcd_oracle as po
from gem_b200 import GemError, _lib, synth

pytestmark = pytest.mark.gpu
FLAGS = [0, po.BINARY, po.RGB_UINT32, po.BINARY | po.RGB_UINT32]


@pytest.fixture(scope="module")
def emap():
    return gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)


def dev(rec):
    return torch.from_numpy(np.ascontiguousarray(rec).view(np.float32).reshape(-1, 8)).to("cuda:0")


def kw(flags):
    return {"binary": bool(flags & po.BINARY), "rgb_uint32": bool(flags & po.RGB_UINT32)}


def same_bytes(got, want, what):
    if got != want:
        k = next(i for i in range(min(len(got), len(want)) + 1) if i == min(len(got), len(want)) or got[i] != want[i])
        raise AssertionError((what, len(got), len(want), k, got[max(0, k - 60):k + 60], want[max(0, k - 60):k + 60]))


def check_device(emap, rec, what):
    d = dev(rec)
    for flags in FLAGS:
        got = emap.format_pcd(d, **kw(flags)).cpu().numpy().tobytes()
        same_bytes(got, po.data(rec, flags), (what, flags))


@pytest.mark.parametrize("name", pc.case_names())
def test_format_matches_oracle(emap, name):
    check_device(emap, pc.cloud(name), name)


def test_format_from_every_producer(emap):
    res, L = 0.1, 200
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    pos = np.array((0.3, -0.2, 1.7), np.float32)
    harvested = []
    for k in range(8):
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([0.5, 0.1, 0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        centre, _, shift = g.move(pos)
        if k > 0:
            rec, n = g.harvest_to_local_map(centre, shift, records=True)
            harvested.append(rec)
        g.add(fr["xyzi"], fr["rgba"], gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
        g.compute_features()
        g.snapshot_shown()
        g.raytracing()
    visual = np.concatenate(harvested)        # visualCloud_, as savingMap writes it
    assert visual.shape[0] > 300
    clouds = {"visual": visual, "grid": g.export_grid_cloud("shown").cpu().numpy()}
    local = g.local_map_take()
    clouds["local"] = local.cpu().numpy()
    clouds["mls"] = g.mls_upsample(local).cpu().numpy()
    g.harvest_to_local_map(*g.move(pos + np.array([2.0, 0.0, 0.0], np.float32))[0::2])
    clouds["dense_cut"] = g.cut_submap(dense=True, seed=3).cpu().numpy()
    for name, rec in clouds.items():
        assert rec.shape[0] > 0, name
        check_device(emap, rec.view(np.uint32), name)


def test_large_cloud(emap):
    rec = pc.harvest_like(2_100_000, 11)
    check_device(emap, rec, "2M")


def test_random_patterns_match_host_build_and_snprintf(emap):
    n = (1 << 26) // 7 + 1
    rec = np.random.default_rng(7).integers(0, 1 << 32, (n, 8), dtype=np.uint64).astype(np.uint32)
    got = emap.format_pcd(dev(rec)).cpu().numpy().tobytes()
    same_bytes(got, po.fmt_ascii(rec), "host build")
    k = (1 << 24) // 7 + 1
    cut = sum(len(s) + 1 for s in got[:200 * k].split(b"\n", k)[:k])
    same_bytes(got[:cut], po.data(rec[:k]), "snprintf")


@pytest.mark.parametrize("flags", FLAGS)
def test_save_pcd_files(emap, tmp_path, flags):
    rec = pc.harvest_like(5000, 4)
    rec[::97, :] = pc.records(pc.specials())[0]
    want = po.file_bytes(rec, flags)
    host = rec.view(np.float32)
    d = dev(rec)
    one = emap.pcd_header(rec.shape[0], **kw(flags)) + emap.format_pcd(d, **kw(flags)).cpu().numpy().tobytes()
    same_bytes(one, want, "one-shot")
    for src, chunk in ((host, None), (host, 7), (host, 1000), (d, None), (d, 999), (torch.from_numpy(host), 4096)):
        p = tmp_path / f"m_{chunk}.pcd"
        size = emap.save_pcd(str(p), src, chunk=chunk, **kw(flags))
        got = p.read_bytes()
        assert size == len(got)
        same_bytes(got, want, (flags, chunk, type(src)))


def test_refusals_write_nothing(emap, tmp_path):
    lib, h = _lib.load(), emap.handle
    rec = dev(pc.harvest_like(300, 5))
    need = C.c_longlong(-1)
    assert lib.gem_pcd_format(h, C.c_void_p(rec.data_ptr()), 300, 0, None, 0, C.byref(need)) == 0 and need.value > 0
    out = torch.full((need.value + 64,), 0xA5, dtype=torch.uint8, device="cuda:0")
    o = C.c_void_p(out.data_ptr() + 3)
    nb = C.c_longlong(-1)
    # one byte short: GEM_OK, the size, nothing written
    assert lib.gem_pcd_format(h, C.c_void_p(rec.data_ptr()), 300, 0, o, need.value - 1, C.byref(nb)) == 0
    assert nb.value == need.value and bool((out == 0xA5).all())
    nb.value = -1
    assert lib.gem_pcd_format(h, C.c_void_p(rec.data_ptr()), 300, po.BINARY, o, 28 * 300 - 1, C.byref(nb)) == 0
    assert nb.value == 28 * 300 and bool((out == 0xA5).all())
    # errors: *bytes_out is 0, nothing written
    for n, flags, ptr in ((0, 0, rec.data_ptr()), (-1, 0, rec.data_ptr()), (300, 4, rec.data_ptr()), (300, -1, rec.data_ptr()),
                          (299, 0, rec.data_ptr() + 4), (300, 0, 0)):
        nb.value = -1
        assert lib.gem_pcd_format(h, C.c_void_p(ptr) if ptr else None, n, flags, o, out.numel() - 3, C.byref(nb)) == 1, (n, flags)
        assert nb.value == 0 and bool((out == 0xA5).all()), (n, flags)
    # the output may not overlap the records
    assert lib.gem_pcd_format(h, C.c_void_p(rec.data_ptr()), 300, po.BINARY, C.c_void_p(rec.data_ptr()), 300 * 32, C.byref(nb)) == 1
    emap.sync()
    # an empty cloud: no file (PCL throws IOException before opening it)
    p = tmp_path / "empty.pcd"
    for empty in (np.zeros((0, 8), np.float32), rec[:0]):
        with pytest.raises(GemError):
            emap.save_pcd(str(p), empty)
        assert not p.exists()
    with pytest.raises(GemError):
        emap.format_pcd(rec[:0])
    # the records are unchanged by every call
    assert rec.cpu().numpy().tobytes() == pc.harvest_like(300, 5).tobytes()


def test_facade_pcd_program(emap, tmp_path):
    exe = native.facade_program("pcd_smoke", tmp_path)
    rec = pc.harvest_like(1000, 6)
    rec[::37, :] = pc.records(pc.specials())[1]
    (tmp_path / "rec.bin").write_bytes(rec.tobytes())
    r = subprocess.run([exe, str(tmp_path / "rec.bin"), str(tmp_path / "cxx")], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "pcd ok" in r.stdout, r.stdout + r.stderr
    for suffix, flags in (("ascii", 0), ("chunked", 0), ("binary", po.BINARY), ("rgbu", po.RGB_UINT32)):
        py = tmp_path / f"py.{suffix}.pcd"
        emap.save_pcd(str(py), rec.view(np.float32), **kw(flags))
        cx = (tmp_path / f"cxx.{suffix}.pcd").read_bytes()
        assert cx == py.read_bytes() == po.file_bytes(rec, flags), suffix
