"""Host wall time per call of the local-submap calls at the c2 geometry (1024^2 at 0.05 m, 1 m per frame along x: about
20 columns leave the window per frame), each next to the call it is compared with:
  gem_harvest_to_local_map (no host copy)        vs gem_harvest_scrolled_out (records to host memory)
  gem_export_grid_cloud (shown, device records)  vs gem_export_visual_points (xyz + rgb to host memory)
  gem_local_map_take after FRAMES frames (one cut per run).
Every call is host-synchronous; the wall time is perf_counter around the C-ABI call.  Prints one JSON line with the GPU
name, its SM clock and power limit as nvidia-smi reports them; writes nothing."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gem_b200  # noqa: E402
from gem_b200 import synth  # noqa: E402

L, RES, FRAMES, NF = 1024, 0.05, 50, 16


def gpu_info():
    q = "name,clocks.sm,clocks.max.sm,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except Exception:
        return {"name": torch.cuda.get_device_name(0)}


def stats(us):
    a = np.asarray(us)
    return {"median_us": round(float(np.median(a)), 1), "mean_us": round(float(a.mean()), 1), "min_us": round(float(a.min()), 1),
            "calls": int(a.size)}


def main():
    scene = synth.make_scene()
    frames = [synth.hdl64_frame(k, scene=scene) for k in range(NF)]
    xd = [torch.from_numpy(fr["xyzi"]).cuda() for fr in frames]
    rd = [torch.from_numpy(fr["rgba"]).cuda() for fr in frames]
    m = gem_b200.ElevationMap(L, RES, compat_box_filter=False, grid_resolution=RES)
    lib, h, nc = m._lib, m.handle, L * L
    host_rec = np.empty((nc, 8), np.float32)
    host_xyz, host_rgb = np.empty((nc, 3), np.float32), np.empty((nc, 3), np.uint8)
    dev_rec = torch.empty((nc, 8), dtype=torch.float32, device="cuda")
    cnt = C.c_int()
    t = {"harvest_scrolled_out": [], "harvest_to_local_map": [], "export_visual_points": [], "export_grid_cloud": []}
    counts = {"harvested": [], "grid": []}

    def timed(name, fn):
        t0 = time.perf_counter()
        rc = fn()
        t[name].append((time.perf_counter() - t0) * 1e6)
        assert rc == 0, (name, lib.gem_last_error(h))

    torch.cuda.synchronize()
    for k in range(FRAMES + 1):
        fr = frames[k % NF]
        pos = np.array([1.0 * k, 0.0, 1.7], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        f = gem_b200.make_frame(T, gem_b200.LaserSensorProcessor())
        cur, _, shift = m.move(pos)
        if k > 0:
            cp = (C.c_float * 2)(*cur.tolist())
            sp = (C.c_float * 2)(*shift.tolist())
            timed("harvest_scrolled_out", lambda: lib.gem_harvest_scrolled_out(h, cp, sp, C.c_void_p(host_rec.ctypes.data), nc, C.byref(cnt)))
            timed("harvest_to_local_map", lambda: lib.gem_harvest_to_local_map(h, cp, sp, None, 0, C.byref(cnt)))
            counts["harvested"].append(cnt.value)
        m.add(xd[k % NF], rd[k % NF], f)
        m.compute_features()
        timed("export_visual_points", lambda: lib.gem_export_visual_points(h, C.c_void_p(host_xyz.ctypes.data),
                                                                           C.c_void_p(host_rgb.ctypes.data), nc, C.byref(cnt)))
        timed("export_grid_cloud", lambda: lib.gem_export_grid_cloud(h, 0, C.c_void_p(dev_rec.data_ptr()), nc, C.byref(cnt)))
        counts["grid"].append(cnt.value)
        m.snapshot_shown()
        m.raytracing()
    m.sync()
    size = m.local_map_size()
    out = torch.empty((size, 8), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rc = lib.gem_local_map_take(h, C.c_void_p(out.data_ptr()), size, C.byref(cnt))
    take_us = (time.perf_counter() - t0) * 1e6
    assert rc == 0 and cnt.value == size
    # the first frames include one-time allocations (staging, the store's first growths): reported apart
    res = {"gpu": gpu_info(), "geometry": {"L": L, "res": RES, "metres_per_frame": 1.0, "frames": FRAMES},
           "records_per_harvest_median": int(np.median(counts["harvested"])), "grid_cloud_points_median": int(np.median(counts["grid"])),
           "local_map_records_after_frames": size,
           "per_call": {k: stats(v[5:]) for k, v in t.items()},
           "first_calls_us": {k: [round(x, 1) for x in v[:3]] for k, v in t.items()},
           "local_map_take_us": round(take_us, 1)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
