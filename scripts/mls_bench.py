"""Time per call of gem_mls_upsample (DESIGN.md f10), the MLS densification of GEM's dense_mapping signal, beside the C
oracle on one host thread.

- the local map harvested from the synthetic c2 stream at 0.05 m (GEM's settings: r 0.5 m, order 5, density 1000: a few
  hundred neighbours, every point fitted);
- a KITTI-like 0.2 m map (about 20 neighbours: no fit, 25 samples per point);
- the worst case: a dense 3D blob with thousands of neighbours per point (every list sorted in global memory).

Each time is CUDA events on the library's stream around one C call with an output buffer that holds the result, the median
of CALLS after WARM.  The call is host-synchronous, so the interval holds its two synchronisations and the host's work
between launches.  The oracle (tests/orc_mls.c, brute-force neighbours) is timed once on one host thread, and every output
and info field is checked equal to it.  Prints one JSON line with the GPU name, SM clock and power limit read by
nvidia-smi in the same run (also written to $GEM_BENCH_OUT/mls_bench.json when that is set)."""
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
from gem_b200 import _lib, synth  # noqa: E402
import mls_cases  # noqa: E402
import mls_oracle  # noqa: E402

WARM, CALLS = 5, 50


def gpu_info():
    q = "name,clocks.sm,clocks.max.sm,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:   # the numbers are then reported without the card's state
        return {"error": str(e)}


def c2_local_map(res, L, frames):
    """the local map the node holds after `frames` frames of the synthetic c2 stream, moving 0.4 m per frame"""
    scene = synth.make_scene()
    g = gem_b200.ElevationMap(L, res, compat_box_filter=False, grid_resolution=res)
    pos = np.array((0.3, -0.2, 1.7), np.float32)
    for k in range(frames):
        fr = synth.hdl64_frame(k, scene=scene)
        pos = pos + np.array([0.4, 0.15, 0], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        centre, _, shift = g.move(pos)
        if k > 0:
            g.harvest_to_local_map(centre, shift)
        g.add(fr["xyzi"], fr["rgba"], gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
        g.compute_features()
        g.snapshot_shown()
        g.raytracing()
    rec = g.local_map_take().cpu().numpy()
    g.close()
    return rec


def main():
    if not torch.cuda.is_available():
        raise SystemExit("mls_bench: no CUDA device (timings are only taken on the GPU)")
    info = gpu_info()
    g = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False)
    mls_oracle.load()
    inputs = {"c2_local_map_005": (c2_local_map(0.05, 400, 10), {}),
              "kitti_like_02": (mls_cases.kitti_like(), {}),
              "dense_blob": (mls_cases.blob(4000, 0.12), {})}
    res = {"gpu": info, "calls": CALLS, "warmup": WARM, "oracle_runs": 1, "cases": {}}
    all_equal = True
    st = g.torch_stream()
    for name, (recs, o) in inputs.items():
        x = torch.from_numpy(recs).cuda()
        t0 = time.perf_counter()
        want, winfo = mls_oracle.upsample(recs, o)
        oracle_ms = (time.perf_counter() - t0) * 1e3
        out = torch.empty((max(winfo["count"], 1), 8), dtype=torch.float32, device="cuda")
        p = mls_oracle.params(o)
        pp = _lib.GemMlsParams(*[getattr(p, k) for k, _ in _lib.GemMlsParams._fields_])
        gi = _lib.GemMlsInfo()
        torch.cuda.synchronize()

        def run():
            rc = g._lib.gem_mls_upsample(g.handle, C.c_void_p(x.data_ptr()), x.shape[0], C.byref(pp), C.c_void_p(out.data_ptr()),
                                         out.shape[0], C.byref(gi))
            assert rc == 0

        run()
        got = out[:gi.count].cpu().numpy()
        ginfo = {k: getattr(gi, k) for k, _ in _lib.GemMlsInfo._fields_}
        equal = ginfo == winfo and got.tobytes() == want.tobytes()
        all_equal &= equal
        for _ in range(WARM):
            run()
        t = []
        for _ in range(CALLS):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st)
            run()
            b.record(st)
            b.synchronize()
            t.append(a.elapsed_time(b))
        res["cases"][name] = {"points": int(recs.shape[0]), **ginfo, "device_ms": round(float(np.median(t)), 4),
                              "device_ms_min": round(float(np.min(t)), 4), "device_ms_max": round(float(np.max(t)), 4),
                              "oracle_ms": round(oracle_ms, 1), "equal_to_oracle": bool(equal)}
    res["all_equal_to_oracle"] = bool(all_equal)
    line = json.dumps(res)
    outdir = os.environ.get("GEM_BENCH_OUT")
    if outdir:
        os.makedirs(outdir, exist_ok=True)
        with open(os.path.join(outdir, "mls_bench.json"), "w") as f:
            f.write(line + "\n")
    print(line)
    return 0 if all_equal else 1


if __name__ == "__main__":
    sys.exit(main())
