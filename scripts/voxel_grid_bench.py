"""Time per call of gem_voxel_grid (DESIGN.md f9), the VoxelGrid nodelet of GEM's demo launches, beside the C oracle on
one host thread.

- a raw c2 frame (one synthetic HDL-64 frame, ~125 k points) under filter.launch (leaf 0.1 m, x in [-10, 10]);
- the same frame through filter_kitti.launch's chain of three calls (leaf 0.2 m; x, then z, then y), timed as a whole;
- random clouds of 1 M and 4 M points in a 100 m cube at leaf 0.1 m (almost every point in its own voxel);
- the worst case of the centroid pass: 1 M points in one voxel (one sequential chain of 1 M float additions).

Each time is CUDA events on the library's stream around the Python call(s), the median of CALLS after WARM.  The call is
host-synchronous, so the interval holds its two synchronisations, the read-backs and the host's work between launches:
close to the wall time of a call.  The oracle (tests/orc_voxel_grid.c, compiled and given host copies before any clock
starts) is timed for the same work on one host thread (median of ORACLE_RUNS), and every output and info field is
checked equal to it.  Prints one JSON line with the GPU name, SM clock and power limit read by nvidia-smi in the same
run."""
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
import voxel_oracle  # noqa: E402

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


def cloud(rng, n, lo, hi):
    p = np.empty((n, 4), np.float32)
    p[:, :3] = rng.uniform(lo, hi, (n, 3))
    p[:, 3] = rng.uniform(0.0, 255.0, n)
    return p


def main():
    if not torch.cuda.is_available():
        raise SystemExit("voxel_grid_bench: no CUDA device (timings are only taken on the GPU)")
    info = gpu_info()
    g = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)
    voxel_oracle.load()
    rng = np.random.default_rng(1)
    c2 = synth.hdl64_frame(0)["xyzi"]
    inputs = {"c2_filter_launch": (c2, voxel_oracle.FILTER_LAUNCH),
              "c2_kitti_chain": (c2, voxel_oracle.FILTER_KITTI_LAUNCH),
              "random_1m": (cloud(rng, 1 << 20, -50.0, 50.0), [(0.1, None, (-3.4e38, 3.4e38), False)]),
              "random_4m": (cloud(rng, 4 << 20, -50.0, 50.0), [(0.1, None, (-3.4e38, 3.4e38), False)]),
              "one_voxel_1m": (cloud(rng, 1 << 20, 0.01, 0.09), [(0.1, None, (-3.4e38, 3.4e38), False)])}
    res = {"gpu": info, "calls": CALLS, "warmup": WARM, "oracle_runs": ORACLE_RUNS, "cases": {}}
    all_equal = True
    for name, (pts, steps) in inputs.items():
        x = torch.from_numpy(pts).cuda()
        bufs = [torch.empty_like(x) for _ in range(2)]
        torch.cuda.synchronize()

        def run():
            cur, inf = x, []
            for k, (leaf, field, limits, neg) in enumerate(steps):
                cur, i = g.voxel_grid(cur, leaf, field, limits, neg, out=bufs[k % 2])
                inf.append(i)
            return cur, inf

        got, ginfo = run()
        want, winfo = voxel_oracle.chain(pts, steps)
        equal = ginfo == winfo and got.cpu().numpy().tobytes() == want.tobytes()
        all_equal &= equal
        res["cases"][name] = {"points": int(pts.shape[0]), "count": ginfo[-1]["count"], "used": ginfo[0]["used"],
                              "device_ms": round(device_ms(g, run), 4),
                              "oracle_ms": round(host_ms(lambda: voxel_oracle.chain(pts, steps)), 2),
                              "equal_to_oracle": bool(equal)}
    res["all_equal_to_oracle"] = bool(all_equal)
    out = os.environ.get("GEM_BENCH_OUT")
    line = json.dumps(res)
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "voxel_grid_bench.json"), "w") as f:
            f.write(line + "\n")
    print(line)
    return 0 if all_equal else 1


if __name__ == "__main__":
    sys.exit(main())
