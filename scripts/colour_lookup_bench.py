"""Time of the colour lookup in its two modes (DESIGN.md f19), in one run:

- gem_colourise_points per call, IMAGE and NODE, on the organised D435 frame (640 x 480 points into its 640 x 480 image)
  and on the 64-beam cloud at 0.08 degrees of azimuth into the KITTI camera's 1241 x 376 image;
- gem_add_pointcloud2_host_async of the same clouds (velodyne XYZIR 32-byte points, pageable) with a bgr8 image, IMAGE
  and NODE, into a fresh map per mode, each call ending in a synchronise;
- the literal loop of tests/orc_colour_lookup.c on one host thread, a stand-in for the node's own loop.

Device calls are timed with CUDA events on the library's stream around one call; the add calls and the oracle with a
wall clock around work that ends in a synchronise.  Each figure is the median of CALLS after WARM.  Outputs at the timed
sizes are checked equal to the oracle.  Prints one JSON line with the GPU name, SM clock and power limit read by
nvidia-smi in the same run (also written to $GEM_BENCH_OUT/colour_lookup_bench.json when that is set)."""
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
import colour_lookup_cases as cc  # noqa: E402
import colour_lookup_oracle as clo  # noqa: E402
import pc2_cases as pc  # noqa: E402
from gem_b200 import CameraImage, PointCloud2Layout, _lib, synth  # noqa: E402

WARM, CALLS = 5, 50


def gpu_info():
    q = "name,clocks.sm,clocks.max.sm,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:
        return {"error": str(e)}


def events(g, fn):
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


def wall(fn, warm=WARM, calls=CALLS):
    times = []
    for i in range(warm + calls):
        t0 = time.perf_counter()
        fn()
        if i >= warm:
            times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times))


def colourise_leg(g, c, mode):
    g.set_colour_lookup(mode)
    n = c["xyzi"].shape[0]
    src = torch.from_numpy(c["xyzi"]).cuda()
    x = src.clone()
    img = torch.from_numpy(c["img"]).cuda()
    out = torch.empty((n, 4), dtype=torch.uint8, device="cuda:0")
    tc = (C.c_double * 12)(*np.asarray(c["T_camera"], np.float64).reshape(-1))
    tl = (C.c_double * 16)(*np.asarray(c["T_lidar"], np.float64).reshape(-1))
    lib = _lib.load()
    torch.cuda.synchronize()

    def call():
        assert lib.gem_colourise_points(g.handle, C.c_void_p(x.data_ptr()), n, tc, tl, C.c_void_p(img.data_ptr()), c["width"],
                                        c["height"], c["row_stride"], C.c_void_p(out.data_ptr())) == 0

    ms = events(g, call)
    g.sync()
    return ms, x.cpu().numpy(), out.cpu().numpy()


def add_leg(c, mode, T, pos, depth):
    g = gem_b200.ElevationMap(120 if depth else 200, 0.05 if depth else 0.1, compat_box_filter=False)
    g.set_colour_lookup(mode)
    sp = gem_b200.StructuredLightSensorProcessor() if depth else gem_b200.LaserSensorProcessor()
    f = gem_b200.make_frame(T, sp)
    case = pc.from_xyzi("b", "xyzir32", c["xyzi"], width=640 if depth else None, height=480 if depth else 1, seed=9)
    lay = PointCloud2Layout(case["fields"], case["width"], case["height"], case["point_step"], case["row_step"],
                            case["is_bigendian"])
    W, H = c["width"], c["height"]
    cam = CameraImage(c["T_camera"], c["T_lidar"], "bgr8", np.ascontiguousarray(c["img"][:, :3 * W]), W, H, 3 * W)
    g.move(pos)

    def call():
        g.add_pointcloud2_host_async(lay, case["data"], f, cam)
        g.sync()

    return wall(call)


def main():
    res = {"gpu": gpu_info(), "warm": WARM, "calls": CALLS, "legs": {}}
    g = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)
    for name, c, (T, pos) in (("d435", cc.d435(), synth.d435_pose(0)), ("lidar_008", cc.lidar_008(), synth.hdl64_pose(0))):
        leg = {"points": int(c["xyzi"].shape[0]), "image": [c["width"], c["height"]]}
        t_o = time.perf_counter()
        want = clo.node(c["xyzi"], c["T_camera"], c["T_lidar"], c["img"], c["width"])
        leg["oracle_first_ms"] = (time.perf_counter() - t_o) * 1e3
        leg["oracle_loop_ms"] = wall(lambda: clo.node(c["xyzi"], c["T_camera"], c["T_lidar"], c["img"], c["width"]), 1, 5)
        leg["in_image"] = int((want[1][:, 3] == 255).sum())
        for mode in ("image", "node"):
            ms, x, rgba = colourise_leg(g, c, mode)
            leg[f"colourise_{mode}_ms"] = ms
            if mode == "node":
                leg["node_equals_oracle"] = bool(x.tobytes() == want[0].tobytes() and np.array_equal(rgba, want[1]))
            else:
                image_rgba = rgba
        leg["differs_from_image"] = int((image_rgba != want[1]).any(axis=1).sum())
        for mode in ("image", "node"):
            leg[f"add_pointcloud2_{mode}_ms"] = add_leg(c, mode, T, pos, name == "d435")
        res["legs"][name] = leg
    line = json.dumps(res)
    print(line)
    out = os.environ.get("GEM_BENCH_OUT")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "colour_lookup_bench.json"), "w") as fh:
            fh.write(line + "\n")
    if not all(leg["node_equals_oracle"] for leg in res["legs"].values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
