"""Host wall time of gem_grid_cloud_split (composingGlobalMap's statistical outlier removal + road / obstacle split) at the
c2 geometry (1024^2 at 0.05 m): FRAMES synthetic HDL-64 frames are fused along a 0.3 m-per-frame track, the features
computed and the shown map snapshotted (the node's prevMap_), then the call is timed CALLS times after WARM warm-up calls
(perf_counter around the host-synchronous C-ABI call, mean_k = 20, stddev_mul = 1, travers_threshold = 0, device
outputs).  One extra profiled call gives the per-kernel device time (CUDA events of gem_profile_*, all these kernels are
class "other"; torch.profiler names them).  For context, the same filter on the host's cores: the C oracle
(tests/orc_grid_split.c, one thread) and the scipy cKDTree restatement (tests/split_cases.py) -- CPU restatements, not PCL.
Both are also checked against the device result.  Prints one JSON line with the GPU name, SM clock and power limit as
nvidia-smi reports them in the same run; writes nothing."""
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
from gem_b200 import synth  # noqa: E402

L, RES, FRAMES, NF, WARM, CALLS = 1024, 0.05, 40, 16, 5, 60


def gpu_info():
    q = "name,clocks.sm,clocks.max.sm,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except Exception:
        return {"name": torch.cuda.get_device_name(0)}


def main():
    scene = synth.make_scene()
    m = gem_b200.ElevationMap(L, RES, compat_box_filter=False, grid_resolution=RES)
    lib, h, nc = m._lib, m.handle, L * L
    for k in range(FRAMES):
        fr = synth.hdl64_frame(k % NF, scene=scene)
        pos = np.array([0.3 * k, 0.1 * k, 1.7], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        m.move(pos)
        m.add(torch.from_numpy(fr["xyzi"]).cuda(), torch.from_numpy(fr["rgba"]).cuda(),
              gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
    m.compute_features()
    m.snapshot_shown()
    m.sync()
    road = torch.empty((nc, 8), dtype=torch.float32, device="cuda")
    obst = torch.empty((nc, 8), dtype=torch.float32, device="cuda")
    dist = torch.empty((nc,), dtype=torch.float32, device="cuda")
    st = gem_b200._lib.GemGridSplit()

    def call():
        return lib.gem_grid_cloud_split(h, 1, 20, 1.0, 0.0, C.c_void_p(road.data_ptr()), nc, C.c_void_p(obst.data_ptr()), nc,
                                        C.c_void_p(dist.data_ptr()), nc, C.byref(st))

    torch.cuda.synchronize()
    us = []
    for i in range(WARM + CALLS):
        t0 = time.perf_counter()
        rc = call()
        dt = (time.perf_counter() - t0) * 1e6
        assert rc == 0, lib.gem_last_error(h)
        if i >= WARM:
            us.append(dt)
    m.profile_enable(True)
    m.profile_read(reset=True)
    assert call() == 0
    prof = m.profile_read(reset=True)
    m.profile_enable(False)
    kernels = {}
    try:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as p:
            assert call() == 0
        for e in p.key_averages():
            if e.device_type.name == "CUDA" and ("split" in e.key or "compact" in e.key):
                kernels[e.key[:90]] = round(e.device_time_total, 1)
    except Exception as exc:   # per-kernel names are optional context
        kernels = {"unavailable": str(exc)[:200]}
    n = st.points
    res = {"gpu": gpu_info(), "geometry": {"L": L, "res": RES, "frames": FRAMES}, "points": n, "valid": st.valid,
           "road": st.road, "obstacle": st.obstacle, "mean": st.mean, "stddev": st.stddev, "threshold": st.threshold,
           "gem_grid_cloud_split_us": {"median": round(float(np.median(us)), 1), "min": round(float(np.min(us)), 1),
                                       "max": round(float(np.max(us)), 1), "calls": len(us)},
           "profile_ms": {"other": round(prof["ms"]["other"], 4), "launches": prof["count"]["other"]},
           "kernels_us": kernels}
    cloud = m.export_grid_cloud("snapshot").cpu().numpy()
    import split_cases
    import split_oracle
    cpu = {"note": "CPU restatements, not PCL", "cores": os.cpu_count()}
    t0 = time.perf_counter()
    o = split_oracle.grid_split(cloud, 20, 1.0, 0.0)
    cpu["c_oracle_ms_one_thread"] = round((time.perf_counter() - t0) * 1e3, 1)
    t0 = time.perf_counter()
    r = split_cases.np_grid_split(cloud, 20, 1.0, 0.0)
    cpu["scipy_ckdtree_restatement_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    d = dist[:n].cpu().numpy()
    res["device_equals_c_oracle"] = bool(np.array_equal(d.view(np.uint32), o["dist"].view(np.uint32)) and
                                         o["road"].shape[0] == st.road and o["threshold"] == st.threshold)
    res["scipy_equals_c_oracle"] = bool(np.array_equal(r["dist"].view(np.uint32), o["dist"].view(np.uint32)))
    res["cpu"] = cpu
    print(json.dumps(res))


if __name__ == "__main__":
    main()
