"""Time of the costmap plugins fed from their messages (DESIGN.md f18), as move_base runs them, in one run:

- ElevationMapLayer: on_message + update_bounds of the c1 (200 x 200, 0.1 m), c2 (1024 x 1024, 0.05 m) and c3
  (512 x 512, 0.02 m) visual_map (gem_ros_grid_map's bytes), the message in pageable and in pinned host memory, into
  GEM's local costmap (75 x 75 at 0.2 m around the map centre);
- PointMapLayer: on_message + update_bounds of a 1 M and a 10 M record history_point, the PointCloud2 data in device
  memory and in pinned host memory, into GEM's global costmap (1000 x 1000 at 0.2 m);
- the same two paths as the C++ facade's ElevationMapLayer / PointMapLayer run them, with their buffers in pinned host
  memory the kernels read and write across PCIe (the floats memcpy'd into a pinned buffer, then the mark; the decode
  into pinned records, then the mark; the re-mark alone);
- beside each, the C oracle on one host thread (tests/orc_gridmsg.c: parse + mark; orc_pc2_decode + mark), a stand-in
  for move_base's fromMessage / fromPCLPointCloud2 and updateBounds on the CPU (which copy more).

Each time is a host clock around one on_message + update_bounds pair (update_bounds is host-synchronous, so the pair ends
with the work done), median of CALLS after WARM.  Prints one JSON line with the GPU name, SM clock and power limit read
by nvidia-smi in the same run (also written to $GEM_BENCH_OUT/costmap_ingest_bench.json when that is set)."""
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
import costmap_oracle  # noqa: E402
import gridmsg_oracle as gm  # noqa: E402
import pc2_oracle  # noqa: E402
from gem_b200 import PointCloud2Layout, RosHeader, _lib, costmap, synth  # noqa: E402

WARM, CALLS = 3, 15
SHAPES = {"c1": (200, 0.1), "c2": (1024, 0.05), "c3": (512, 0.02)}
ICT = [("x", 0, 7, 1), ("y", 4, 7, 1), ("z", 8, 7, 1), ("rgb", 16, 7, 1), ("intensity", 24, 7, 1), ("covariance", 20, 7, 1),
       ("travers", 28, 7, 1)]


def gpu_info():
    q = "name,clocks.sm,clocks.max.sm,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:
        return {"error": str(e)}


def clock(fn, warm=WARM, calls=CALLS):
    times = []
    for i in range(warm + calls):
        t0 = time.perf_counter()
        fn()
        t1 = time.perf_counter()
        if i >= warm:
            times.append((t1 - t0) * 1e3)
    return round(float(np.median(times)), 4)


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


def elevation_leg(nav, name, L, res):
    g = fill(L, res)
    msg = g.ros_grid_map(RosHeader(1, 2, 3, "odom")).cpu()
    del g
    pageable = msg.numpy().tobytes()
    pinned = msg.pin_memory()
    d = gm.parse(pageable)
    c = (d["position_x"], d["position_y"])
    layer = costmap.Costmap(nav, 75, 75, 0.2, c[0] - 7.45, c[1] - 7.45)
    el = costmap.ElevationMapLayer(nav, 0.7)

    def once(src):
        assert el.on_message(src)
        el.update_bounds(layer)

    r = {"message_bytes": len(pageable), "layer_bytes": 4 * d["floats"],
         "pageable_ms": clock(lambda: once(pageable)), "pinned_ms": clock(lambda: once(pinned))}
    # the C++ ElevationMapLayer: a host memcpy of the floats into its pinned buffer, the kernel reading them across PCIe
    lib = _lib.load()
    g = _lib.GemGridMapLayer()
    fl = torch.empty(4 * d["floats"], dtype=torch.uint8).pin_memory()
    src = np.frombuffer(pageable, np.uint8)
    w = _lib.GemCostmapWindow(*layer.window)
    mk = _lib.GemCostmapMarks()

    def cxx():
        assert lib.gem_grid_map_msg_parse(C.c_char_p(pageable), len(pageable), b"traver", C.byref(g)) == 0
        fl.numpy()[:] = src[g.offset:g.offset + 4 * g.floats]
        assert lib.gem_costmap_mark_grid(nav.handle, C.byref(g), C.c_void_p(fl.data_ptr()), C.byref(w), 0.7, 1,
                                         C.c_void_p(layer.grid.data_ptr()), C.byref(mk)) == 0
    r["cxx_pinned_buffer_ms"] = clock(cxx)
    floats = gm.layer_floats(pageable, d)
    grid = layer.grid.cpu().numpy()

    def oracle():
        gm.orc_parse(pageable)
        gm.orc_mark_grid(d, floats, layer.window, grid, 0.7, True)
    r["oracle_ms"] = clock(oracle, 1, 3)
    return r


def points_leg(nav, n):
    rng = np.random.default_rng(n)
    rec = np.zeros((n, 8), np.float32)
    rec[:, 0] = rng.uniform(-110.0, 110.0, n)
    rec[:, 1] = rng.uniform(-110.0, 110.0, n)
    rec[:, 2] = rng.uniform(-1.0, 2.0, n)
    rec[:, 3] = 1.0
    rec[:, 7] = rng.uniform(0.0, 1.0, n)
    raw = rec.view(np.uint8).reshape(-1)
    dev = torch.from_numpy(raw).cuda()
    pinned = torch.from_numpy(raw).pin_memory()
    lay = PointCloud2Layout(ICT, n, 1, 32)
    layer = costmap.Costmap(nav, 1000, 1000, 0.2, -100.0, -100.0, fill=costmap.COST_UNKNOWN)
    pl = costmap.PointMapLayer(nav, 0.7)

    def once(src):
        pl.on_message(lay, src)
        pl.update_bounds(layer)

    r = {"points": n, "data_bytes": 32 * n, "device_ms": clock(lambda: once(dev)), "pinned_ms": clock(lambda: once(pinned)),
         "update_bounds_only_ms": clock(lambda: pl.update_bounds(layer))}
    # the C++ PointMapLayer: the message bytes in pinned memory, decoded into pinned records, marked from them
    lib = _lib.load()
    recs = torch.empty(32 * n, dtype=torch.uint8).pin_memory()
    w = _lib.GemCostmapWindow(*layer.window)
    mk = _lib.GemCostmapMarks()

    def cxx_decode():
        assert lib.gem_decode_pointcloud2_records(nav.handle, C.byref(lay.c), C.c_void_p(pinned.data_ptr()), 32 * n,
                                                  C.c_void_p(recs.data_ptr())) == 0
        nav.sync()

    def cxx_mark():
        assert lib.gem_costmap_mark_points(nav.handle, C.c_void_p(recs.data_ptr()), n, C.byref(w), 0.7,
                                           C.c_void_p(layer.grid.data_ptr()), C.byref(mk)) == 0

    r["cxx_pinned_buffers_ms"] = clock(lambda: (cxx_decode(), cxx_mark()))
    r["cxx_update_bounds_only_ms"] = clock(cxx_mark)
    case = {"fields": ICT, "width": n, "height": 1, "point_step": 32, "row_step": 32 * n, "data": raw}
    grid = layer.grid.cpu().numpy()

    def oracle():
        recs, _ = pc2_oracle.decode(case)
        costmap_oracle.mark_points(recs.view(np.float32).reshape(-1, 8), layer.window, grid, 0.7)
    r["oracle_ms"] = clock(oracle, 0, 1 if n > 2_000_000 else 3)
    return r


def main():
    nav = gem_b200.ElevationMap(1, 0.1, compat_box_filter=False)          # move_base's handle: the smallest one
    out = {"gpu": gpu_info(), "elevation": {}, "points": {}}
    for name, (L, res) in SHAPES.items():
        out["elevation"][name] = elevation_leg(nav, name, L, res)
    for n in (1_000_000, 10_000_000):
        out["points"][f"{n // 1_000_000}M"] = points_leg(nav, n)
    line = json.dumps(out)
    print(line)
    if os.environ.get("GEM_BENCH_OUT"):
        os.makedirs(os.environ["GEM_BENCH_OUT"], exist_ok=True)
        with open(os.path.join(os.environ["GEM_BENCH_OUT"], "costmap_ingest_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
