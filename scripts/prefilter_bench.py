"""Per-frame time of the demos' ingest with the VoxelGrid pre-filter (DESIGN.md f20): raw c2 frames (synthetic HDL-64,
~125 k points) as 32-byte XYZIR PointCloud2 messages in pinned memory, with a 640 x 480 bgr8 image in pinned memory,
under filter.launch and filter_kitti.launch, in both colour lookup modes.  Two arms, alternated in one run:

- (a) the synchronous chain: H2D copies of the message and the image (then a synchronise), gem_decode_pointcloud2,
  gem_voxel_grid per step (host-synchronous), gem_colourise_points, gem_add_points_stream;
- (b) gem_add_pointcloud2_filtered_host_async, one call per frame.

Each arm has its own map and gets the same frames and moves.  A window is a fixed number of frames (sized so that arm
(a)'s window lasts a second or more) and ends in gem_sync; the per-frame time is the host wall time of the window over
its frames, and raw Mpoints/s the raw points over it.  ROUNDS windows per arm, alternated, median reported.  At the end
both maps are read back and must be byte-equal on every layer.  With --profile, a separate run records a few frames of
each arm under torch.profiler (CUDA activities) and reports the device time of the filter's kernels per frame (k_vox_*
and the cub sort, run-length and scan kernels, which only the filter launches in the image lookup mode).  Prints one
JSON line with the GPU name and power limit read by nvidia-smi in the same run."""
import argparse
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
from gem_b200 import CameraImage, PointCloud2Layout, _lib, synth  # noqa: E402
import pc2_cases as pc  # noqa: E402
import voxel_oracle  # noqa: E402

NFRAMES, ROUNDS, WINDOW_S = 8, 3, 1.0
W, H = 640, 480
TC = np.array([[385.0, 0, 320.0, 0], [0, 385.0, 240.0, 0], [0, 0, 1, 0]], np.float64)
TL = np.array([[0, -1, 0, 0.0], [0, 0, -1, -0.08], [1, 0, 0, -0.27], [0, 0, 0, 1]], np.float64)
LAUNCHES = {"filter": voxel_oracle.FILTER_LAUNCH, "kitti": voxel_oracle.FILTER_KITTI_LAUNCH}
LAYERS = ("elevation", "variance", "intensity", "color_r", "color_g", "color_b", "traver", "lowest")


def gpu_info():
    q = "name,clocks.sm,clocks.max.sm,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:   # the numbers are then reported without the card's state
        return {"error": str(e)}


class Frames:
    def __init__(self):
        self.items = []
        for k in range(NFRAMES):
            fr = synth.hdl64_frame(k)
            case = pc.from_xyzi("f", "xyzir32", fr["xyzi"], seed=k)
            lay = PointCloud2Layout(case["fields"], case["width"], case["height"], case["point_step"], case["row_step"])
            data = torch.from_numpy(case["data"]).pin_memory()
            img = torch.from_numpy(np.random.default_rng(k).integers(0, 256, (H, 3 * W)).astype(np.uint8)).pin_memory()
            f = gem_b200.make_frame(fr["T"], gem_b200.LaserSensorProcessor())
            pos = (C.c_float * 3)(*[float(v) for v in fr["position"]])
            self.items.append((lay, data, img, f, pos, int(fr["xyzi"].shape[0])))
        self.nmax = max(it[5] for it in self.items)


class SyncChain:
    """arm (a): H2D, decode, gem_voxel_grid per step, gem_colourise_points, gem_add_points_stream"""

    def __init__(self, g, frames, steps):
        self.g, self.lib, self.h = g, g._lib, g.handle
        self.steps = [gem_b200.ElevationMap.prefilter([s]).step[0] for s in steps]
        n = frames.nmax
        self.msg = [torch.empty(max(it[1].numel() for it in frames.items), dtype=torch.uint8, device="cuda") for _ in range(3)]
        self.img = [torch.empty((H, 3 * W), dtype=torch.uint8, device="cuda") for _ in range(3)]
        self.dec = torch.empty((n, 4), dtype=torch.float32, device="cuda")
        self.buf = [[torch.empty((n, 4), dtype=torch.float32, device="cuda") for _ in range(2)] for _ in range(3)]
        self.rgba = [torch.empty((n, 4), dtype=torch.uint8, device="cuda") for _ in range(3)]
        self.tc = (C.c_double * 12)(*TC.reshape(-1))
        self.tl = (C.c_double * 16)(*TL.reshape(-1))
        self.info = _lib.GemVoxelGridInfo()
        self.i = 0

    def __call__(self, item):
        lay, data, img, f, pos, n = item
        b = self.i % 3
        self.i += 1
        lib, h = self.lib, self.h
        # the uploads on torch's stream, waited for as the voxel recipe before f20 did (the library's stream is the
        # handle's, and torch's pinned allocator must not record its events there)
        self.msg[b][:data.numel()].copy_(data, non_blocking=True)
        self.img[b].copy_(img, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        _lib.check(lib.gem_decode_pointcloud2(h, C.byref(lay.c), C.c_void_p(self.msg[b].data_ptr()), data.numel(),
                                              C.c_void_p(self.dec.data_ptr())), h, "decode")
        cur, count = self.dec, n
        for k, p in enumerate(self.steps):
            out = self.buf[b][k % 2]
            _lib.check(lib.gem_voxel_grid(h, C.c_void_p(cur.data_ptr()) if count else None, count, C.byref(p),
                                          C.c_void_p(out.data_ptr()), n, C.byref(self.info)), h, "voxel_grid")
            cur, count = out, self.info.count
        if count:
            _lib.check(lib.gem_colourise_points(h, C.c_void_p(cur.data_ptr()), count, self.tc, self.tl,
                                                C.c_void_p(self.img[b].data_ptr()), W, H, 3 * W,
                                                C.c_void_p(self.rgba[b].data_ptr())), h, "colourise")
        _lib.check(lib.gem_add_points_stream(h, C.c_void_p(cur.data_ptr()) if count else None,
                                             C.c_void_p(self.rgba[b].data_ptr()), count, C.byref(f)), h, "add")


class OneCall:
    """arm (b): gem_add_pointcloud2_filtered_host_async"""

    def __init__(self, g, frames, steps):
        self.lib, self.h = g._lib, g.handle
        self.pf = gem_b200.ElevationMap.prefilter(steps)
        self.cams = [CameraImage(TC, TL, "bgr8", it[2], W, H) for it in frames.items]

    def __call__(self, item, k):
        lay, data, img, f, pos, n = item
        _lib.check(self.lib.gem_add_pointcloud2_filtered_host_async(self.h, C.byref(lay.c), C.c_void_p(data.data_ptr()),
                                                                    data.numel(), C.byref(self.cams[k].c), C.byref(self.pf),
                                                                    C.byref(f)), self.h, "filtered")


def window(g, run, frames, nframes, start):
    t0 = time.perf_counter()
    for j in range(nframes):
        k = (start + j) % NFRAMES
        g.move_fast(frames.items[k][4])
        run(k)
    g.flush()
    g.sync()
    return time.perf_counter() - t0


def config(frames, launch, mode, profile):
    steps = LAUNCHES[launch]
    ga = gem_b200.ElevationMap(400, 0.1, compat_box_filter=False)
    gb = gem_b200.ElevationMap(400, 0.1, compat_box_filter=False)
    for g in (ga, gb):
        g.set_colour_lookup(mode)
    a, b = SyncChain(ga, frames, steps), OneCall(gb, frames, steps)
    ra = lambda k: a(frames.items[k])          # noqa: E731
    rb = lambda k: b(frames.items[k], k)       # noqa: E731
    raw = sum(it[5] for it in frames.items) / NFRAMES
    pos = 0
    # warm-up (every buffer and graph), then size the window from arm (a)
    for g, r in ((ga, ra), (gb, rb)):
        window(g, r, frames, 2 * NFRAMES, 0)
    pos = 2 * NFRAMES
    t = window(ga, ra, frames, 4 * NFRAMES, pos)
    window(gb, rb, frames, 4 * NFRAMES, pos)
    pos += 4 * NFRAMES
    nwin = max(NFRAMES, int(np.ceil(WINDOW_S / (t / (4 * NFRAMES)))))
    ta, tb = [], []
    for _ in range(ROUNDS):
        ta.append(window(ga, ra, frames, nwin, pos) / nwin)
        tb.append(window(gb, rb, frames, nwin, pos) / nwin)
        pos += nwin
    equal = all(ga.get_layer(n).tobytes() == gb.get_layer(n).tobytes() for n in LAYERS)
    res = {"frames_per_window": nwin, "raw_points_per_frame": raw,
           "sync_chain_ms": round(1e3 * float(np.median(ta)), 4), "one_call_ms": round(1e3 * float(np.median(tb)), 4),
           "sync_chain_ms_all": [round(1e3 * v, 4) for v in ta], "one_call_ms_all": [round(1e3 * v, 4) for v in tb],
           "sync_chain_raw_mpts_s": round(raw / float(np.median(ta)) / 1e6, 2),
           "one_call_raw_mpts_s": round(raw / float(np.median(tb)) / 1e6, 2),
           "maps_byte_equal": bool(equal)}
    if profile:
        from torch.profiler import ProfilerActivity, profile as prof
        for arm, g, r in (("sync_chain", ga, ra), ("one_call", gb, rb)):
            with prof(activities=[ProfilerActivity.CUDA]) as p:
                window(g, r, frames, NFRAMES, pos)
            filt = 0.0
            for e in p.key_averages():
                if "k_vox" in e.key or "cub" in e.key.lower():
                    filt += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            res[f"{arm}_filter_kernel_ms_per_frame"] = round(filt / 1e3 / NFRAMES, 4)
    ga.close()
    gb.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--profile", action="store_true", help="also record the filter's kernel time under torch.profiler")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prefilter_bench: no CUDA device (timings are only taken on the GPU)")
    res = {"gpu": gpu_info(), "rounds": ROUNDS, "window_s": WINDOW_S, "configs": {}}
    frames = Frames()
    ok = True
    for launch in LAUNCHES:
        for mode in ("image", "node"):
            if args.profile and mode == "node":
                continue      # the node lookup sorts too: the cub kernels would not be the filter's alone
            r = config(frames, launch, mode, args.profile)
            ok &= r["maps_byte_equal"]
            res["configs"][f"{launch}_{mode}"] = r
    res["maps_byte_equal"] = bool(ok)
    del frames                # the pinned buffers go while the CUDA context is still up
    torch.cuda.synchronize()
    line = json.dumps(res)
    out = os.environ.get("GEM_BENCH_OUT")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "prefilter_bench" + ("_profile" if args.profile else "") + ".json"), "w") as f:
            f.write(line + "\n")
    print(line)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
