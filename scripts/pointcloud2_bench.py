"""The PointCloud2 ingest (DESIGN.md f12) timed on the frames of the add benchmarks, beside the C oracle on one host thread.

- decode kernel: gem_decode_pointcloud2 on the c2 frame (one synthetic HDL-64 frame, ~125 k points) in velodyne's XYZIR
  32-byte and packed 22-byte layouts, and on the organised 640 x 480 D435 frame (c3, 16-byte points, padded rows); CUDA
  events on the library's stream around DECODE_REPS back-to-back launches, per launch;
- frames: gem_add_pointcloud2_host_async on the message bytes against gem_add_points_host_async on the same frame
  pre-packed as xyzi (c2 into 200 x 200 @ 0.1 m, c3 into 512 x 512 @ 0.02 m), both from pinned host memory, no image,
  FRAMES calls each after WARM, the host clock around the
  calls plus the final gem_sync, in Gpoints/s;
- the oracle (tests/orc_pointcloud2.c) decoding the same messages on one host thread, a stand-in for the node's
  fromPCLPointCloud2 (median of ORACLE_RUNS).

Every decode output is checked equal to the oracle's, and the two maps of each frame comparison are checked equal cell
for cell.  Prints one JSON line with the GPU name and power limit read by nvidia-smi in the same run (also written to
$GEM_BENCH_OUT/pointcloud2_bench.json when that is set)."""
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
import pc2_cases as pc  # noqa: E402
import pc2_oracle  # noqa: E402

WARM, FRAMES, DECODE_REPS, ORACLE_RUNS = 10, 200, 200, 3
LAYERS = ("elevation", "variance", "intensity", "color_r", "color_g", "color_b", "lowest")


def gpu_info():
    q = "name,clocks.sm,clocks.max.sm,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:   # the numbers are then reported without the card's state
        return {"error": str(e)}


def layout(case):
    return gem_b200.PointCloud2Layout(case["fields"], case["width"], case["height"], case["point_step"], case["row_step"])


def messages():
    c2 = synth.hdl64_frame(0)
    d435 = synth.d435_frame(0)
    return {
        "c2_xyzir32": (pc.from_xyzi("c2_xyzir32", "xyzir32", c2["xyzi"], seed=1), c2, gem_b200.LaserSensorProcessor(), 200, 0.1),
        "c2_xyzir22": (pc.from_xyzi("c2_xyzir22", "xyzir22", c2["xyzi"], seed=2), c2, gem_b200.LaserSensorProcessor(), 200, 0.1),
        "c3_d435_organised": (pc.from_xyzi("c3", "d435", d435["xyzi"], width=640, height=480, row_pad=64, seed=3,
                                           rgb=d435["rgba"]), d435, gem_b200.StructuredLightSensorProcessor(), 512, 0.02),
    }


def decode_us(g, case):
    L = layout(case)
    data = torch.from_numpy(case["data"]).cuda()
    out = torch.empty((L.points, 4), dtype=torch.float32, device="cuda:0")
    g.decode_pointcloud2(L, data, out)
    g.sync()
    want = pc2_oracle.xyzi(pc2_oracle.decode(case)[0])
    assert out.cpu().numpy().tobytes() == want.tobytes(), case["name"]
    lib, h, pL = g._lib, g.handle, C.byref(L.c)
    dp, op, nb = C.c_void_p(data.data_ptr()), C.c_void_p(out.data_ptr()), case["data"].nbytes
    st = g.torch_stream()
    for _ in range(WARM):
        lib.gem_decode_pointcloud2(h, pL, dp, nb, op)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    for _ in range(DECODE_REPS):
        lib.gem_decode_pointcloud2(h, pL, dp, nb, op)
    b.record(st)
    b.synchronize()
    return a.elapsed_time(b) * 1000.0 / DECODE_REPS


def frames_gpts(case, fr, sp, length, resolution):
    """(Gpoints/s of the PointCloud2 call, of the pre-packed xyzi call); the two maps must agree"""
    L = layout(case)
    n = L.points
    f = gem_b200.make_frame(fr["T"], sp)
    raw = torch.from_numpy(case["data"]).pin_memory()
    xyzi = torch.from_numpy(pc2_oracle.xyzi(pc2_oracle.decode(case)[0])).pin_memory()
    res, maps = [], []
    for mode in ("pointcloud2", "xyzi"):
        g = gem_b200.ElevationMap(length, resolution, compat_box_filter=False)
        g.move(fr["position"])
        fref = C.byref(f)
        if mode == "pointcloud2":
            def call():
                g.add_pointcloud2_host_async(L, raw, f)
        else:
            xp = C.c_void_p(xyzi.data_ptr())

            def call():
                g.add_host_async_fast(xp, None, n, fref)
        for _ in range(WARM):
            call()
        g.sync()
        t0 = time.perf_counter()
        for _ in range(FRAMES):
            call()
        g.sync()
        dt = time.perf_counter() - t0
        res.append(n * FRAMES / dt / 1e9)
        maps.append({k: g.get_layer(k) for k in LAYERS})
        g.close()
    for k in LAYERS:
        a, b = maps[0][k], maps[1][k]
        assert a.tobytes() == b.tobytes(), ("maps differ", case["name"], k)
    return res


def oracle_ms(case):
    t = []
    for _ in range(ORACLE_RUNS):
        t0 = time.perf_counter()
        pc2_oracle.decode(case)
        t.append((time.perf_counter() - t0) * 1000.0)
    return float(np.median(t))


def main():
    if not torch.cuda.is_available():
        raise SystemExit("pointcloud2_bench: no CUDA device")
    info = gpu_info()
    g = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)
    out = {"gpu": info, "rows": []}
    for name, (case, fr, sp, length, res) in messages().items():
        row = {"frame": name, "map": f"{length}x{length}@{res}m", "points": case["width"] * case["height"], "point_step": case["point_step"],
               "message_bytes": int(case["data"].nbytes)}
        row["decode_us"] = round(decode_us(g, case), 2)
        row["decode_GBps_read"] = round(case["data"].nbytes / row["decode_us"] / 1e3, 1)
        p2, xy = frames_gpts(case, fr, sp, length, res)
        row["add_pointcloud2_host_async_Gpts"] = round(p2, 3)
        row["add_points_host_async_prepacked_Gpts"] = round(xy, 3)
        row["oracle_decode_ms_1thread"] = round(oracle_ms(case), 3)
        out["rows"].append(row)
    line = json.dumps(out)
    print(line)
    od = os.environ.get("GEM_BENCH_OUT")
    if od:
        os.makedirs(od, exist_ok=True)
        with open(os.path.join(od, "pointcloud2_bench.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
