"""Plain c2 add loop for ncu: python scripts/add_loop.py [steps] [mode: plain|stream] ; prints per-kernel event timings
(serial schedule) when run without a profiler."""
import os, sys, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import gem_b200
from bench import gen_frames, pingpong, laser_frame

K = int(sys.argv[1]) if len(sys.argv) > 1 else 40
mode = sys.argv[2] if len(sys.argv) > 2 else "plain"
F = 16
frames = gen_frames(F)
fobjs = [laser_frame(fr) for fr in frames]
dev = torch.device("cuda", 0)
xd = [torch.from_numpy(fr["xyzi"]).to(dev) for fr in frames]
rd = [torch.from_numpy(fr["rgba"]).to(dev) for fr in frames]
npts = [fr["xyzi"].shape[0] for fr in frames]
m = gem_b200.ElevationMap(1024, 0.05, compat_box_filter=False)
def step(s):
    k = pingpong(s, F)
    m.move(frames[k]["position"])
    if mode == "plain":
        m.add(xd[k], rd[k], fobjs[k], n=npts[k])
    else:
        m.add_stream_fast(C.c_void_p(xd[k].data_ptr()), C.c_void_p(rd[k].data_ptr()), npts[k], C.byref(fobjs[k]))
for s in range(K): step(s)
m.sync()
if os.environ.get("ADD_LOOP_PROFILE", "1") == "1":
    m.profile_read(reset=True)
    m.profile_enable(True)
    for s in range(200): step(K + s)
    pr = m.profile_read(reset=True)
    print({k: (round(v / max(1, pr["count"][k]) * 1e3, 2), pr["count"][k]) for k, v in pr["ms"].items() if pr["count"][k]}, m.stats())
if os.environ.get("ADD_LOOP_STAMPS", "0") == "1":
    res = []
    for s in range(30):
        m.debug_stamps(True)
        step(K + 300 + s)
        st = m.debug_stamps(True)
        res.append([(st[i] - st[8]) / 1e3 if st[i] else np.nan for i in (9, 13, 10, 14, 12)] + [st[i] / 1e3 for i in (3, 4, 7, 5, 6)])
    res = np.nanmedian(np.array(res), axis=0)
    print("us since k_fold's first block started: k_fold (latest first warp of any block): marks queued %.2f, short lists done %.2f, end %.2f; k_fold_long: last list of 9..40 folded %.2f, last list of > 40 folded %.2f || slowest list of > 40 since its own start: k known %.2f, records arrived %.2f, positions counted %.2f, intensities in place %.2f, folded %.2f" % tuple(res))
