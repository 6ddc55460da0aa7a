"""Time of the costmap topics and the footprint clearing (DESIGN.md f17), in one run:

- gem_ros_costmap full (OccupancyGrid) of GEM's 1000 x 1000 global and 75 x 75 local costmaps, into device memory and
  into pinned host memory;
- an update (OccupancyGridUpdate) of a 75 x 75 rectangle of the global grid, into pinned memory;
- gem_costmap_footprint of GEM's footprint on the local layer grid;
- beside them, the host path a user has without the library: the 1000 x 1000 grid copied to pageable host memory, the
  numpy table lookup and the struct encoder of tests/costmap_pub_oracle.py.

Device calls are timed with CUDA events on the library's stream around one call, the host path with a wall clock around
work that ends in a device synchronise; each is the median of CALLS after WARM.  Prints one JSON line with the GPU name,
SM clock and power limit read by nvidia-smi in the same run (also written to $GEM_BENCH_OUT/costmap_publish_bench.json
when that is set)."""
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
import costmap_pub_oracle as cp  # noqa: E402
import rosmsg_oracle as ro  # noqa: E402
from gem_b200 import RosHeader, costmap  # noqa: E402

WARM, CALLS = 5, 50


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


def wall(fn):
    times = []
    for i in range(WARM + CALLS):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        if i >= WARM:
            times.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(times))


def main():
    if not torch.cuda.is_available():
        raise SystemExit("costmap_publish_bench needs a GPU")
    info = gpu_info()
    g = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)
    lib, h = g._lib, RosHeader(frame_id="odom")
    rng = np.random.default_rng(0)
    res = {"gpu": info, "unit": "ms", "warm": WARM, "calls": CALLS}
    windows = {"global": (-100.0, -100.0, 0.2, 1000, 1000), "local": (-7.45, -7.45, 0.2, 75, 75)}
    grids = {k: torch.from_numpy(rng.choice(np.array([0, 0, 0, 254, 255, 128], np.uint8), (w[4], w[3]))).to("cuda:0")
             for k, w in windows.items()}
    torch.cuda.synchronize()   # the grids are written on torch's stream, the library reads them on its own
    kind, nb = C.c_int(), C.c_longlong()

    def publish(name, out, force=1, pub=None):
        w = g._cost_window(windows[name])
        p = pub or costmap.CostmapPublisher()
        hc = h.c()
        grid = C.c_void_p(grids[name].data_ptr())
        return lambda: lib.gem_ros_costmap(g._h, C.byref(hc), C.byref(w), grid, C.byref(p.state), force, C.c_void_p(out.data_ptr()),
                                           out.numel(), C.byref(nb), C.byref(kind))

    for name in windows:
        sx, sy = windows[name][3:]
        dev = torch.empty(sx * sy + 256, dtype=torch.uint8, device="cuda:0")
        pin = torch.empty(sx * sy + 256, dtype=torch.uint8, pin_memory=True)
        res[f"full_{name}_device"] = timed(g, publish(name, dev))
        res[f"full_{name}_pinned"] = timed(g, publish(name, pin))
        res[f"full_{name}_bytes"] = nb.value
    # an update of a 75 x 75 rectangle of the global grid: the bounds fed before every call
    pub = costmap.CostmapPublisher()
    pin = torch.empty(1 << 21, dtype=torch.uint8, pin_memory=True)
    publish("global", pin, 0, pub)()
    upd = publish("global", pin, 0, pub)

    def update():
        pub.bounds(462, 537, 462, 537)
        upd()
    res["update_75x75_of_global_pinned"] = timed(g, update)
    assert kind.value == 2 and nb.value == 36 + 4 + 75 * 75
    layer = torch.zeros((75, 75), dtype=torch.uint8, device="cuda:0")
    res["footprint_clear_local"] = timed(g, lambda: g.costmap_footprint(windows["local"], costmap.GEM_FOOTPRINT, 0.03, -0.02, 0.7, layer))
    # the host path: D2H of the grid, the table lookup, the struct encoder
    hb = ro.header(0, 0, 0, b"odom")
    res["host_path_full_global"] = wall(lambda: cp.occupancy_grid(hb, windows["global"], grids["global"].cpu().numpy()))
    res["d2h_global_grid_pageable"] = wall(lambda: grids["global"].cpu())
    pin_grid = torch.empty((1000, 1000), dtype=torch.uint8, pin_memory=True)
    res["d2h_global_grid_pinned"] = wall(lambda: pin_grid.copy_(grids["global"], non_blocking=True))
    # the kernel alone, from a torch.profiler trace of device-memory full messages
    from torch.profiler import ProfilerActivity, profile
    dev = torch.empty(1000 * 1000 + 256, dtype=torch.uint8, device="cuda:0")
    call = publish("global", dev)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            call()
        g.sync()
    ks = [e for e in prof.events() if "k_ros_costmap" in e.name]
    res["k_ros_costmap_global_us"] = float(np.median([getattr(e, "device_time", None) or e.cuda_time for e in ks])) if ks else None
    line = json.dumps(res)
    print(line)
    out = os.environ.get("GEM_BENCH_OUT")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "costmap_publish_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
