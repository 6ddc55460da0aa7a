"""Time per frame of gem_add_points_stream with each of the four sensor models (laser, structured light, stereo,
perfect) on the c3 shape: the raw organised 640x480 synthetic D435 frame (NaNs left in) into a 512^2 map at 0.02 m.

Laser and structured light run the headline instantiations of the bin kernel; stereo and perfect run the every-model
instantiation (one point per thread, transform_point<true>).  The models alternate round by round so that drift of the
shared host or card hits all four alike.  A round is FRAMES pipelined calls of one model between CUDA events on the
library's stream (the last fold issued by a flush inside the interval); the figure is the median over ROUNDS rounds, in
milliseconds per frame.  Prints one JSON line with the GPU name, SM clock and power limit read by nvidia-smi in the same
run.  The script needs a GPU; it has no CPU fallback."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import gem_b200  # noqa: E402
from gem_b200 import synth  # noqa: E402

ROUNDS, FRAMES, WARM = 15, 30, 2
ASLAM = dict(p_1=0.03287, p_2=-0.0001276, p_3=0.4850, p_4=399.1046, p_5=0.000006735, lateral_factor=0.001376915,
             depth_to_disparity_factor=47.3, cloud_width=640)
MODELS = {
    "laser": gem_b200.LaserSensorProcessor(ignore_points_above=float("inf"), ignore_points_below=float("-inf")),
    "structured_light": gem_b200.StructuredLightSensorProcessor(),
    "stereo": gem_b200.StereoSensorProcessor(**ASLAM),
    "perfect": gem_b200.PerfectSensorProcessor(),
}


def gpu_info():
    q = "name,clocks.sm,clocks.max.sm,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:   # the numbers are then reported without the card's state
        return {"error": str(e)}


def main():
    if not torch.cuda.is_available():
        raise SystemExit("sensor_model_bench: no CUDA device")
    fr = synth.d435_frame(0)
    n = fr["xyzi"].shape[0]
    x = torch.from_numpy(fr["xyzi"]).cuda()
    r = torch.from_numpy(fr["rgba"]).cuda()
    g = gem_b200.ElevationMap(512, 0.02, compat_box_filter=False)
    frames = {k: gem_b200.make_frame(fr["T"], s, base_z=float(fr["position"][2])) for k, s in MODELS.items()}
    refs = {k: C.byref(f) for k, f in frames.items()}
    xp, rp = C.c_void_p(x.data_ptr()), C.c_void_p(r.data_ptr())
    st = g.torch_stream()
    times = {k: [] for k in MODELS}
    for rnd in range(WARM + ROUNDS):
        for k in MODELS:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st)
            for _ in range(FRAMES):
                g.add_stream_fast(xp, rp, n, refs[k])
            g.flush()
            b.record(st)
            b.synchronize()
            if rnd >= WARM:
                times[k].append(a.elapsed_time(b) / FRAMES)
    out = {"bench": "sensor_model_stream_add", "shape": "640x480 D435 raw -> 512^2 @ 0.02 m", "points": n,
           "rounds": ROUNDS, "frames_per_round": FRAMES, "gpu": gpu_info(),
           "ms_per_frame": {k: round(float(np.median(v)), 4) for k, v in times.items()},
           "spread_ms": {k: [round(float(np.min(v)), 4), round(float(np.max(v)), 4)] for k, v in times.items()}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
