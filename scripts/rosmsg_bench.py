"""Time of the map topics as ROS messages (DESIGN.md f15) on the c1 (200 x 200, 0.1 m), c2 (1024 x 1024, 0.05 m) and c3
(512 x 512, 0.02 m) map shapes, filled from synth frames, in one run:

- device time of gem_ros_grid_map into device memory and into pinned host memory, next to export_layers into pinned
  host arrays (k_export_colmajor into device scratch, then DMA copies) in the same run;
- gem_ros_visual_points and gem_ros_orthomosaic into device memory;
- gem_ros_cloud of 10 M records from one device part and from one pinned host part, into device memory;
- GB/s of each = the message's bytes over the time;
- a host stand-in: one CPU thread serialising the exported layers with the struct encoder of tests/rosmsg_oracle.py (a
  lower bound on grid_map's toMessage plus roscpp's serialiser, which copy more).

Every time is CUDA events on the library's stream around one call (the message calls are asynchronous, except
visual_points), median of CALLS after WARM.  Prints one JSON line with the GPU name, SM clock and power limit read by
nvidia-smi in the same run (also written to $GEM_BENCH_OUT/rosmsg_bench.json when that is set)."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import gem_b200  # noqa: E402
import rosmsg_oracle as ro  # noqa: E402
from gem_b200 import RosHeader, synth  # noqa: E402

WARM, CALLS = 3, 20
SHAPES = {"c1": (200, 0.1), "c2": (1024, 0.05), "c3": (512, 0.02)}


def gpu_info():
    q = "name,clocks.sm,clocks.max.sm,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:
        return {"error": str(e)}


def timed(g, fn):
    st = g.torch_stream()
    times = []
    for i in range(WARM + CALLS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        fn()
        e1.record(st)
        e1.synchronize()
        if i >= WARM:
            times.append(e0.elapsed_time(e1))
    return float(np.median(times))


def entry(ms, nbytes):
    return {"ms": round(ms, 4), "bytes": int(nbytes), "GBps": round(nbytes / (ms * 1e6), 2)}


def ros_call(g, fn, h, out):
    nb = C.c_longlong()
    rc = fn(g.handle, C.byref(h), C.c_void_p(out.data_ptr()), out.numel(), C.byref(nb))
    assert rc == 0 and nb.value <= out.numel()
    return nb.value


def fill(L, res):
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    scene = synth.make_scene()
    pos = np.array((0.3, -0.2, 1.7), np.float32)
    for k in range(4):
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([0.4, 0.1, 0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        g.move(pos)
        g.add(fr["xyzi"], fr["rgba"], gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
    g.compute_features()
    return g


def bench_shape(name, L, res):
    g = fill(L, res)
    lib = g._lib
    h = RosHeader(frame_id="map").c()
    size = ro.size_grid_map(3, L)
    dev = torch.empty(size + 16, dtype=torch.uint8, device="cuda:0")
    pin = torch.empty(size + 16, dtype=torch.uint8).pin_memory()
    out = {"L": L, "res": res}
    d1 = dev[1:]
    p1 = pin[1:]
    layers = {n: np.empty((L, L), np.float32, order="F") for n in ro.GRID_LAYERS}
    layers_pinned = {n: torch.empty(L * L, dtype=torch.float32).pin_memory() for n in ro.GRID_LAYERS}
    lp = {n: layers_pinned[n].numpy().reshape(L, L, order="F") for n in ro.GRID_LAYERS}
    out["export_layers_to_pinned"] = entry(timed(g, lambda: g.export_layers(lp)), 36 * L * L)
    out["grid_map_device"] = entry(timed(g, lambda: ros_call(g, lib.gem_ros_grid_map, h, d1)), size)
    out["grid_map_pinned"] = entry(timed(g, lambda: ros_call(g, lib.gem_ros_grid_map, h, p1)), size)
    g.sync()
    msg = d1[:size].cpu().numpy().tobytes()
    g.export_layers(layers)
    c, s, _ = g.state()
    want = ro.grid_map(ro.header(0, 0, 0, b"map"), L, res, float(c[0]), float(c[1]), s, layers)
    out["grid_map_equals_oracle"] = msg == want == p1[:size].numpy().tobytes()
    t0 = time.perf_counter()
    for _ in range(3):
        ro.grid_map(ro.header(0, 0, 0, b"map"), L, res, float(c[0]), float(c[1]), s, layers)
    out["host_encoder_grid_map"] = entry((time.perf_counter() - t0) / 3 * 1e3, size)
    n_vis = ros_call(g, lib.gem_ros_visual_points, h, d1)
    out["visual_points_device"] = entry(timed(g, lambda: ros_call(g, lib.gem_ros_visual_points, h, d1)), n_vis)
    n_img = ros_call(g, lib.gem_ros_orthomosaic, h, d1)
    out["orthomosaic_device"] = entry(timed(g, lambda: ros_call(g, lib.gem_ros_orthomosaic, h, d1)), n_img)
    return g, out


def bench_cloud(g):
    n = 10_000_000
    rec_d = torch.randint(0, 1 << 30, (n, 8), dtype=torch.int32, device="cuda:0").view(torch.float32)
    rec_p = rec_d.cpu().pin_memory()
    h = RosHeader(frame_id="map").c()
    size = ro.size_ict(3, n)
    out_d = torch.empty(size + 16, dtype=torch.uint8, device="cuda:0")[1:]
    res = {}
    for where, rec in (("device_part", rec_d), ("pinned_part", rec_p)):
        part = (gem_b200._lib.GemRosPart * 1)(gem_b200._lib.GemRosPart(rec.data_ptr(), n))

        def call():
            nb = C.c_longlong()
            assert g._lib.gem_ros_cloud(g.handle, C.byref(h), part, 1, 1, C.c_void_p(out_d.data_ptr()), out_d.numel(), C.byref(nb)) == 0
        res[where] = entry(timed(g, call), size)
    g.sync()
    res["equals_records"] = bool(torch.equal(out_d[164 + 3:164 + 3 + 32 * n], rec_d.view(torch.uint8).view(-1)))
    return res


def main():
    if not torch.cuda.is_available():
        raise SystemExit("rosmsg_bench: no GPU")
    result = {"gpu": gpu_info(), "shapes": {}}
    g = None
    for name, (L, res) in SHAPES.items():
        g, result["shapes"][name] = bench_shape(name, L, res)
    result["cloud_10M"] = bench_cloud(g)
    line = json.dumps(result)
    print(line)
    d = os.environ.get("GEM_BENCH_OUT")
    if d:
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "rosmsg_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
