"""The global map's submap stack on the device (gem_global_map_*, DESIGN.md f16) byte for byte against the oracle
(tests/orc_global_map.c) on every crafted call sequence of tests/global_map_cases.py in both precedence modes; against the
existing host loop submaps.update_global_map on poses whose relative transforms are exact in float; the packed run
through gem_ros_cloud and the submaps through save_submaps; growth past the reserve, the refusals, an update beside the
add path on the same handle, and the C++ façade."""
import ctypes as C
import os
import subprocess
import threading
import time

import numpy as np
import pytest
import torch

import gem_b200
import global_map_cases as gc
import global_map_oracle as go
import native
import pcd_oracle
import rosmsg_oracle as ro
from gem_b200 import submaps as sm
from gem_b200 import synth

pytestmark = pytest.mark.gpu
GEM_ERR_INVALID = 1


def dev(a):
    return torch.from_numpy(np.array(a, np.float32, copy=True).reshape(-1, 8)).to("cuda:0")


class DeviceStack:
    """the stack of a gem_b200.ElevationMap with the methods gc.run expects"""

    def __init__(self, emap):
        self.m = emap
        self.m.global_map_reset()

    def reset(self):
        self.m.global_map_reset()

    def push(self, records, pose):
        self.m.global_map_push(dev(records), pose)

    def update(self, opt_poses, resolution, radius=25.0, compat=True):
        return self.m.global_map_update(opt_poses, resolution, radius, compat)

    def state(self):
        subs = [s.cpu().numpy() for s in self.m.global_map_submaps()]
        poses, centres = self.m.global_map_poses()
        packed = self.m.global_map_records().cpu().numpy()
        assert packed.tobytes() == b"".join(s.tobytes() for s in subs), "the stack is not packed"
        return subs, poses, centres


@pytest.fixture(scope="module")
def emap():
    return gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)


@pytest.mark.parametrize("compat", [True, False], ids=["compat", "weighted"])
@pytest.mark.parametrize("name", list(gc.CASES))
def test_crafted(emap, name, compat):
    ops = gc.CASES[name]()
    fo, so = gc.run(go.OracleStack(), ops, compat)
    fd, sd = gc.run(DeviceStack(emap), ops, compat)
    assert fd == fo, (name, fd, fo)
    for step, (a, b) in enumerate(zip(sd, so)):
        assert go.stack_difference(a, b) is None, (name, step, go.stack_difference(a, b))


def exact_chain(K=6, res=0.125):
    """submaps under poses whose relative transforms are exact in float: 90-degree yaws, shifts by multiples of res"""
    q = [gc.pose(0.0, 0.0, 0.0)]
    for s in range(1, K + 1):
        P = np.eye(4, dtype=np.float32)
        P[:2, :2] = np.array([[0, -1], [1, 0]], np.float32) if s % 2 else np.eye(2, dtype=np.float32)
        P[:2, 3] = (2.0 * s, 1.0 * (s % 3))
        q.append(P)
    subs = [gc.submap(f"exact/{s}", *q[s][:2, 3], [900, 1200, 700, 1500, 1000, 800][s], res=res) for s in range(K)]
    opt = []
    for s, P in enumerate(q):
        O = P.copy()
        if s % 2:
            O[:2, :2] = -O[:2, :2]                      # a 180-degree turn on top
        O[:2, 3] += np.float32(res) * np.float32([(s % 3) - 1, 2 - (s % 4)])
        opt.append(O)
    return subs, q, np.array(opt, np.float32)


@pytest.mark.parametrize("compat", [True, False], ids=["compat", "weighted"])
def test_equals_host_loop_on_exact_poses(emap, compat):
    subs, kf, opt = exact_chain()
    K = len(subs)
    st = DeviceStack(emap)
    for s in range(K):
        st.push(subs[s], kf[s + 1])
    fused = st.update(opt, 0.125, 25.0, compat)
    old = [kf[s] for s in range(K)]
    centres = [(float(P[0, 3]), float(P[1, 3])) for P in old]
    for i in range(1, K):                       # the relative transforms really are exact
        assert (go.relative_pose(opt[i], old[i]) == (opt[i].astype(np.float64) @ np.linalg.inv(old[i].astype(np.float64)))).all()
    host, fh = sm.update_global_map(emap, [dev(s) for s in subs], old, opt[:K], centres, 0.125, 25.0, compat)
    assert fused == fh and fused > 100
    got = st.state()[0]
    for k, (a, b) in enumerate(zip(got, host)):
        assert go.stack_difference(([a], np.zeros(0), np.zeros(0)), ([b.cpu().numpy()], np.zeros(0), np.zeros(0))) is None, k


def test_ros_cloud_and_save_submaps(emap, tmp_path):
    ops = gc.CASES["sequence"]()[:6]
    fo, so = gc.run(go.OracleStack(), ops)
    gc.run(DeviceStack(emap), ops)
    subs = so[-1][0]
    h = gem_b200.RosHeader(seq=3, stamp_sec=7, frame_id="map")
    want = ro.ict_cloud(ro.header(3, 7, 0, b"map"), np.concatenate(subs))
    got = emap.ros_cloud(h, [emap.global_map_records()]).cpu().numpy().tobytes()
    dsubs = [s.cpu().numpy() for s in emap.global_map_submaps()]
    assert go.stack_difference((dsubs, np.zeros(0), np.zeros(0)), (subs, np.zeros(0), np.zeros(0))) is None
    assert got == ro.ict_cloud(ro.header(3, 7, 0, b"map"), np.concatenate(dsubs))
    assert len(got) == len(want)
    for binary in (False, True):
        d = tmp_path / ("bin" if binary else "ascii")
        d.mkdir()
        paths = emap.save_submaps(str(d), binary=binary)
        assert [os.path.basename(p) for p in paths] == [f"{i}.pcd" for i in range(len(dsubs)) if dsubs[i].shape[0]]
        for p in paths:
            i = int(os.path.basename(p)[:-4])
            assert open(p, "rb").read() == pcd_oracle.file_bytes(dsubs[i], gem_b200._lib.PCD_BINARY if binary else 0), p


def test_growth_past_reserve(emap):
    emap.global_map_reset()
    emap.global_map_reserve(1000, 2)
    ops = gc.chain("growth", gc._line(8), [1500, 3000, 2500, 4000, 100, 3500, 5000, 2000])
    ops.append(("update", gc.perturbed([gc.pose(0.0, *c) for c in gc._line(8)], 21), 0.1, 25.0))
    fo, so = gc.run(go.OracleStack(), ops)
    fd, sd = gc.run(DeviceStack(emap), ops)
    assert fd == fo and fo[0] > 0
    assert go.stack_difference(sd[-1], so[-1]) is None
    assert emap.global_map_info() == (8, 9, sum(s.shape[0] for s in so[-1][0]))


def test_refusals(emap):
    lib, h = emap._lib, emap._h
    st = DeviceStack(emap)
    for op in gc.chain("refusals", gc._line(3), [300, 400, 500]):
        st.push(op[1], op[2])
    before = st.state()
    eye = (C.c_float * 16)(*np.eye(4, dtype=np.float32).reshape(-1).tolist())
    opt = (C.c_float * 48)(*np.tile(np.eye(4, dtype=np.float32).reshape(-1), 3).tolist())
    fused = C.c_int(-7)
    nan, inf = float("nan"), float("inf")
    for k, p, res, rad in ((-1, opt, 0.1, 25.0), (2, None, 0.1, 25.0), (3, opt, 0.0, 25.0), (3, opt, -0.1, 25.0), (3, opt, nan, 25.0),
                           (3, opt, inf, 25.0), (3, opt, 0.1, -1.0), (3, opt, 0.1, nan)):
        assert lib.gem_global_map_update(h, p, k, res, rad, 1, C.byref(fused)) == GEM_ERR_INVALID, (k, res, rad)
    assert fused.value == -7
    buf = dev(np.zeros((4, 8), np.float32))
    host = np.zeros((4, 8), np.float32)
    pinned = torch.zeros((4, 8), dtype=torch.float32).pin_memory()
    for rec, n, pose in ((C.c_void_p(buf.data_ptr()), -1, eye), (None, 3, eye), (C.c_void_p(host.ctypes.data), 4, eye),
                         (C.c_void_p(pinned.data_ptr()), 4, eye), (C.c_void_p(buf.data_ptr()), 4, None)):
        assert lib.gem_global_map_push(h, rec, n, pose) == GEM_ERR_INVALID
    p, cnt, c = C.c_void_p(), C.c_int(), (C.c_float * 2)()
    for i in (-1, 3):
        assert lib.gem_global_map_submap(h, i, C.byref(p), C.byref(cnt)) == GEM_ERR_INVALID
    for i in (-1, 4):
        assert lib.gem_global_map_pose(h, i, eye, c) == GEM_ERR_INVALID
    assert lib.gem_global_map_reserve(h, -1, 0) == GEM_ERR_INVALID and lib.gem_global_map_reserve(h, 0, -1) == GEM_ERR_INVALID
    assert go.stack_difference(st.state(), before) is None
    assert lib.gem_global_map_push(h, None, 0, eye) == 0 and lib.gem_global_map_update(h, None, 0, 0.1, 25.0, 1, None) == 0
    assert emap.global_map_info() == (4, 5, sum(s.shape[0] for s in before[0]))


def _add_loop(g, frames, stamps=None, stop=None):
    out = []
    f = gem_b200.make_frame(frames[0]["T"], gem_b200.LaserSensorProcessor())
    for q, fr in enumerate(frames):
        f = gem_b200.make_frame(fr["T"], gem_b200.LaserSensorProcessor())
        g.move(fr["position"])
        g.add(fr["xyzi"], fr["rgba"], f)
        g.compute_features()
        out.append({k: v.copy() for k, v in g.export_layers().items()})
        if stamps is not None:
            stamps.append(time.perf_counter())
    return out


def _big_stack(g, K=12, n=250_000):
    g.global_map_reset()
    g.global_map_reserve(K * n, K)
    cen = gc._line(K, 1.0)
    for s in range(K):
        g.global_map_push(dev(gc.submap(f"big/{s}", *cen[s], n, spread=700)), gc.pose(0.0, *cen[s + 1]))
    return gc.perturbed([gc.pose(0.0, *c) for c in cen], 31)


def test_update_beside_the_add_path():
    """one thread updates the global map while another adds, computes features and exports on the same handle: both
    results equal the sequential run's, and the add thread finishes frames while the update runs"""
    frames = [synth.hdl64_frame(q) for q in range(12)]
    ref = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False)
    opt = _big_stack(ref)
    want_fused = ref.global_map_update(opt, 0.1)
    want_stack = ref.global_map_records().cpu().numpy()
    want_layers = _add_loop(ref, frames)

    g = gem_b200.ElevationMap(200, 0.1, compat_box_filter=False)
    _big_stack(g)
    stamps, span, res = [], [], {}

    def upd():
        t0 = time.perf_counter()
        res["fused"] = g.global_map_update(opt, 0.1)
        span.extend([t0, time.perf_counter()])

    th = threading.Thread(target=upd)
    loop = threading.Thread(target=lambda: res.setdefault("layers", _add_loop(g, frames * 4, stamps)))
    loop.start()
    while not stamps:
        time.sleep(0.001)
    th.start()
    th.join()
    loop.join()
    assert res["fused"] == want_fused and want_fused > 1000
    assert g.global_map_records().cpu().numpy().tobytes() == want_stack.tobytes()
    for a, b in zip(res["layers"][:len(frames)], want_layers):
        for k in b:
            assert a[k].tobytes() == b[k].tobytes(), k
    during = [t for t in stamps if span[0] < t < span[1]]
    print(f"update {1e3 * (span[1] - span[0]):.1f} ms, {len(during)} add frames finished during it")
    assert during, "no add frame finished while the update ran"


def test_facade_global_map_program(emap, tmp_path):
    exe = native.facade_program("global_map_smoke", tmp_path, ["-I", "/usr/local/cuda/include"],
                                ["-L", "/usr/local/cuda/lib64", "-lcudart"])
    subs, kf, opt = exact_chain()
    with open(tmp_path / "in.bin", "wb") as f:
        f.write(np.int32(len(subs)).tobytes())
        for s, rec in enumerate(subs):
            f.write(np.int32(rec.shape[0]).tobytes() + kf[s + 1].tobytes() + rec.tobytes())
        f.write(np.int32(opt.shape[0]).tobytes() + opt.tobytes() + np.float64(0.125).tobytes())
    out = str(tmp_path / "cxx") + "/"
    os.mkdir(out)
    r = subprocess.run([exe, str(tmp_path / "in.bin"), out], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "global_map ok" in r.stdout, r.stdout + r.stderr
    st = DeviceStack(emap)
    for s in range(len(subs)):
        st.push(subs[s], kf[s + 1])
    fused = st.update(opt, 0.125)
    assert f"fused={fused}" in r.stdout
    assert open(out + "packed.bin", "rb").read() == emap.global_map_records().cpu().numpy().tobytes()
    assert open(out + "poses.bin", "rb").read() == emap.global_map_poses()[0].tobytes()
    for i, s in enumerate(emap.global_map_submaps()):
        assert open(out + f"{i}.pcd", "rb").read() == pcd_oracle.file_bytes(s.cpu().numpy())
