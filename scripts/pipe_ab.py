"""A/B of the frame pipeline: gem_add_points_stream (one CUDA graph per call, `graph`) against the plain
gem_add_points call (`plain`).  Prints us/frame (device, CUDA events on the handle's stream) and the host enqueue time."""
import os, sys, time, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import gem_b200
from bench import gen_frames, pingpong, laser_frame

F, K = 32, 600
frames = gen_frames(F)
fobjs = [laser_frame(fr) for fr in frames]
dev = torch.device("cuda", 0)
xd = [torch.from_numpy(fr["xyzi"]).to(dev) for fr in frames]
rd = [torch.from_numpy(fr["rgba"]).to(dev) for fr in frames]
npts = [fr["xyzi"].shape[0] for fr in frames]
pos_c = [(C.c_float * 3)(*[float(v) for v in fr["position"]]) for fr in frames]
xp = [C.c_void_p(t.data_ptr()) for t in xd]; rp = [C.c_void_p(t.data_ptr()) for t in rd]
fref = [C.byref(f) for f in fobjs]
for mode in (sys.argv[1:] or ["graph", "plain"]):
    m = gem_b200.ElevationMap(1024, 0.05, compat_box_filter=False)
    st = m.torch_stream()
    def step(s):
        k = pingpong(s, F)
        m.move_fast(pos_c[k])
        (m.add_fast if mode == "plain" else m.add_stream_fast)(xp[k], rp[k], npts[k], fref[k])
        return npts[k]
    for s in range(40): step(s)
    m.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter(); e0.record(st); pts = 0
    for s in range(K): pts += step(40 + s)
    m.flush(); e1.record(st); host = (time.perf_counter() - t0) * 1e6 / K
    m.sync()
    ms = e0.elapsed_time(e1)
    print(f"{mode:7s} {ms*1e3/K:7.2f} us/frame device  {host:6.2f} us/frame host enqueue  {pts/ms/1e3:8.1f} Mpoints/s  stats {m.stats()}", flush=True)
    m.close()
