"""Time per call of the navigation costmap calls (DESIGN.md f8) at GEM's sizes, beside the C oracle on one host thread.

- gem_costmap_mark_map from the shown c2 map (1024^2 at 0.05 m, 40 synthetic HDL-64 frames) into the local window
  (75 x 75 at 0.2 m) and the global one (1000 x 1000 at 0.2 m), mark_unknown = 1;
- gem_costmap_mark_points over 1 M and 4 M records (the c2 grid cloud, repeated and jittered) into 1000 x 1000;
- gem_costmap_update_origin of a 1000 x 1000 grid by (3, -2) cells;
- gem_costmap_combine over the whole 1000 x 1000 grid (max and overwrite);
- gem_costmap_inflate (DESIGN.md f14) of GEM's global costmap, 1000 x 1000 at 0.2 m whose master is PointMapLayer's
  overwrite of the c2 grid cloud, over the update rect at GEM's 0.0 m (a no-op), costmap_2d's default 0.55 m (r = 3) and
  2.0 m (r = 10), and over the whole grid at 0.55 m (the first update); and of a 4000 x 4000 grid at 0.05 m with the
  same cloud marked, r = 40, over the whole grid, to show the cost of its many distance bins.  Factor 10, GEM's
  footprint's inscribed radius 0.40 m.  Every call inflates the same master copy again, which is the same work.

Each time is CUDA events on the library's stream around one Python call, the median of CALLS calls after WARM.  The
interval therefore also holds the host's time between the launches (argument checks, waiting for the torch stream) and,
for the host-synchronous mark calls, the accumulator upload, the read-back of the marks and the stream synchronisation:
it is close to the wall time of a call, not the kernels' time alone.  The oracle (tests/orc_costmap.c, compiled and
given host copies before any clock starts) is timed for the same work on one host thread (median of ORACLE_RUNS), and
the grids and marks are checked equal to it.  Prints one JSON line with the GPU name, SM clock and power limit read by nvidia-smi in
the same run."""
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
import costmap_oracle  # noqa: E402
import inflation_oracle  # noqa: E402
from gem_b200 import costmap  # noqa: E402

WARM, CALLS, ORACLE_RUNS = 5, 50, 3


def gpu_info():
    q = "name,clocks.sm,clocks.max.sm,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:   # the numbers are then reported without the card's state
        return {"error": str(e)}


def device_ms(g, fn):
    st = g.torch_stream()
    for _ in range(WARM):
        fn()
    t = []
    for _ in range(CALLS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        fn()
        b.record(st)
        b.synchronize()
        t.append(a.elapsed_time(b))
    return float(np.median(t))


def host_ms(fn):
    t = []
    for _ in range(ORACLE_RUNS):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def inflation_rows(g, cloud, centre, out):
    ok = True
    ins = costmap.inscribed_radius(costmap.GEM_FOOTPRINT)
    cx, cy = float(centre[0]), float(centre[1])
    for size, res, runs in ((1000, 0.2, (("0.0", None), ("0.55", None), ("2.0", None), ("0.55", "whole"))),
                            (4000, 0.05, (("2.0", "whole"),))):
        w = (cx - size * res / 2, cy - size * res / 2, res, size, size)
        layer = torch.full((size, size), 255, dtype=torch.uint8, device="cuda:0")
        marks = g.costmap_mark_points(cloud, w, layer, 0.7)
        rect = costmap.update_rect(w, marks)
        master0 = costmap_oracle.combine(1, layer.cpu().numpy(), np.zeros((size, size), np.uint8), size, size, rect)
        out[f"inflate_{size}_lethal_cells"] = int((master0 == 254).sum())
        out[f"inflate_{size}_rect"] = list(rect)
        for radius, where in runs:
            p = inflation_oracle.params(float(radius), 10.0, ins)
            r = (0, 0, size, size) if where else rect
            key = f"inflate_{size}_{radius}m" + ("_whole" if where else "")
            grid = torch.from_numpy(master0).cuda()
            out[f"{key}_ms"] = device_ms(g, lambda: g.costmap_inflate(w, p, grid, r))
            out[f"{key}_oracle_ms"] = host_ms(lambda: inflation_oracle.inflate(master0, res, p, r))
            grid = torch.from_numpy(master0).cuda()
            g.costmap_inflate(w, p, grid, r)
            g.sync()
            want = inflation_oracle.inflate(master0, res, p, r)
            out[f"{key}_cells_changed"] = int((want != master0).sum())
            ok &= np.array_equal(grid.cpu().numpy(), want)
    return ok


def main():
    L, res = 1024, 0.05
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    for k in range(40):
        fr = synth.hdl64_frame(k % 16, scene=scene)
        pos = np.array([0.3 * k, 0.1 * k, 1.7], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        g.move(pos)
        g.add(torch.from_numpy(fr["xyzi"]).cuda(), torch.from_numpy(fr["rgba"]).cuda(),
              gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
    g.compute_features()
    centre, start, _ = g.state()
    tr = np.array(g.export_layers()["traver"])
    cx, cy = float(centre[0]), float(centre[1])
    windows = {"local_75": (cx - 7.45, cy - 7.45, 0.2, 75, 75), "global_1000": (cx - 100.0, cy - 100.0, 0.2, 1000, 1000)}
    costmap_oracle.load()
    out = {"gpu": gpu_info(), "map": f"c2 {L}^2 at {res} m", "warm": WARM, "calls": CALLS, "oracle_runs": ORACLE_RUNS}
    ok = True
    for name, w in windows.items():
        grid = torch.full((w[4], w[3]), 255, dtype=torch.uint8, device="cuda:0")
        out[f"mark_map_{name}_ms"] = device_ms(g, lambda: g.costmap_mark_map(w, grid, 0.7, "shown", True))
        g0 = np.full((w[4], w[3]), 255, np.uint8)
        want, wm = costmap_oracle.mark_map(tr, L, res, centre, start, w, g0, 0.7, True)
        out[f"mark_map_{name}_oracle_ms"] = host_ms(lambda: costmap_oracle.mark_map(tr, L, res, centre, start, w, g0, 0.7, True))
        grid.fill_(255)
        m = g.costmap_mark_map(w, grid, 0.7, "shown", True)
        ok &= np.array_equal(grid.cpu().numpy(), want) and m == wm
    cloud = g.export_grid_cloud("shown")
    rng = np.random.default_rng(1)
    w = windows["global_1000"]
    for n in (1 << 20, 1 << 22):
        base = cloud.cpu().numpy()
        rec = base[rng.integers(0, base.shape[0], n)].copy()
        rec[:, :2] += rng.uniform(-0.1, 0.1, (n, 2)).astype(np.float32)
        d = torch.from_numpy(rec).cuda()
        grid = torch.full((1000, 1000), 255, dtype=torch.uint8, device="cuda:0")
        out[f"mark_points_{n}_ms"] = device_ms(g, lambda: g.costmap_mark_points(d, w, grid, 0.7))
        g0 = np.full((1000, 1000), 255, np.uint8)
        want, wm = costmap_oracle.mark_points(rec, w, g0, 0.7)
        out[f"mark_points_{n}_oracle_ms"] = host_ms(lambda: costmap_oracle.mark_points(rec, w, g0, 0.7))
        m = g.costmap_mark_points(d, w, grid, 0.7)
        ok &= np.array_equal(grid.cpu().numpy(), want) and m == wm
    grid0 = np.random.default_rng(2).integers(0, 256, (1000, 1000)).astype(np.uint8)
    grid = torch.from_numpy(grid0).cuda()
    flip = [0]

    def roll():   # back and forth by (3, -2) cells, so every call moves the grid
        s = 1 if flip[0] == 0 else -1
        flip[0] ^= 1
        g.costmap_update_origin((0.0, 0.0, 0.2, 1000, 1000), s * 0.61, -s * 0.41, 0, grid)
    out["update_origin_ms"] = device_ms(g, roll)
    out["update_origin_oracle_ms"] = host_ms(lambda: costmap_oracle.update_origin((0.0, 0.0, 0.2, 1000, 1000), 0.61, -0.41, 0, grid0))
    grid = torch.from_numpy(grid0).cuda()
    nw, got = g.costmap_update_origin((0.0, 0.0, 0.2, 1000, 1000), 0.61, -0.41, 0, grid), None
    g.sync()
    ww, want = costmap_oracle.update_origin((0.0, 0.0, 0.2, 1000, 1000), 0.61, -0.41, 0, grid0)
    ok &= nw == ww and np.array_equal(grid.cpu().numpy(), want)
    lay0 = np.random.default_rng(3).integers(0, 256, (1000, 1000)).astype(np.uint8)
    lay = torch.from_numpy(lay0).cuda()
    for mode, mid in (("max", 0), ("overwrite", 1)):
        mas = torch.from_numpy(grid0).cuda()
        out[f"combine_{mode}_ms"] = device_ms(g, lambda: g.costmap_combine(mode, lay, mas, 1000, 1000, (0, 0, 1000, 1000)))
        out[f"combine_{mode}_oracle_ms"] = host_ms(lambda: costmap_oracle.combine(mid, lay0, grid0, 1000, 1000, (0, 0, 1000, 1000)))
        mas = torch.from_numpy(grid0).cuda()
        g.costmap_combine(mode, lay, mas, 1000, 1000, (0, 0, 1000, 1000))
        g.sync()
        ok &= np.array_equal(mas.cpu().numpy(), costmap_oracle.combine(mid, lay0, grid0, 1000, 1000, (0, 0, 1000, 1000)))
    ok &= inflation_rows(g, cloud, centre, out)
    out["outputs_equal_oracle"] = bool(ok)
    print(json.dumps(out))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
