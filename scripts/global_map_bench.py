"""Loop-closure update of the global map (DESIGN.md f16): gem_global_map_update, one call, against the host loop
gem_b200.submaps.update_global_map over device tensors (one gem_transform_cloud per submap, one gem_refuse_submaps per
pair), on the same submaps and poses.  Two shapes:
  kitti: the kitti demo map, L = 75 at 0.2 m, K = 64 keyframes 20 m apart around a closed square loop;
  c2:    L = 1024 at 0.05 m, about 10^6 records per submap, K = 16 keyframes 20 m apart around a square loop.
Keyframe yaws are multiples of 90 degrees and the optimised poses shift them by multiples of the resolution, so every
relative transform is exact in float and the two outputs must be equal byte for byte (checked every round).  The two
are alternated, after one warm-up round each; host wall time around each call (both end in a synchronisation), median
of the rounds.  Prints one JSON line per shape with the pair count, the records, the GPU's name, SM clock and power
limit as nvidia-smi reports them in the same run; writes nothing."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gem_b200  # noqa: E402
from gem_b200 import submaps as sm  # noqa: E402

SHAPES = {"kitti": dict(L=75, res=0.2, K=64, rounds=7), "c2": dict(L=1024, res=0.05, K=16, rounds=5)}


def gpu_info():
    q = "name,clocks.sm,clocks.max.sm,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except Exception:
        return {"name": torch.cuda.get_device_name(0)}


def square_loop(K, step=20.0):
    """K keyframe poses (row-major 4 x 4) around a square of side K / 4 * step, yaw along the path"""
    side = K // 4
    poses = []
    for k in range(K):
        e, s = divmod(k, side)
        yaw = e * np.pi / 2
        c, d = np.float32(np.round(np.cos(yaw))), np.float32(np.round(np.sin(yaw)))
        start = [(0, 0), (side, 0), (side, side), (0, side)][e]
        x, y = (start[0] + c * s) * step, (start[1] + d * s) * step
        P = np.eye(4, dtype=np.float32)
        P[:2, :2] = [[c, -d], [d, c]]
        P[:2, 3] = (x, y)
        poses.append(P)
    return poses


def submap(rng, cx, cy, L, res):
    """the records of a keyframe cut: about half the window's cells, each cell at most twice (local map + grid cloud)"""
    n = L * L
    cells = rng.choice(L * L, n // 2, replace=False)
    cells = np.concatenate([cells, rng.choice(cells, n - n // 2)])
    ix, iy = cells // L - L // 2 + int(round(cx / res)), cells % L - L // 2 + int(round(cy / res))
    p = np.zeros((n, 8), np.float32)
    p[:, 0] = ((ix - 0.5 + 0.8 * (rng.random(n) - 0.5)) * res).astype(np.float32)
    p[:, 1] = ((iy - 0.5 + 0.8 * (rng.random(n) - 0.5)) * res).astype(np.float32)
    p[:, 2] = rng.uniform(-1, 1, n).astype(np.float32)
    p[:, 3] = 1
    p.view(np.uint32)[:, 4] = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    p[:, 5] = rng.choice(np.array([0.05, 0.2, 0.5, 1.0], np.float32), n)
    p[:, 6] = rng.integers(0, 256, n).astype(np.float32)
    p[:, 7] = rng.random(n).astype(np.float32)
    return p


def run(name, L, res, K, rounds):
    rng = np.random.default_rng(7)
    kf = [np.eye(4, dtype=np.float32)] + square_loop(K)
    subs = [torch.from_numpy(submap(rng, kf[s][0, 3], kf[s][1, 3], L, res)).cuda() for s in range(K)]
    opt = []
    for P in kf:
        O = P.copy()
        O[:2, 3] += np.float32(res) * rng.integers(-3, 4, 2).astype(np.float32)
        opt.append(O)
    opt = np.array(opt, np.float32)
    centres = [(float(P[0, 3]), float(P[1, 3])) for P in kf[:K]]
    pairs = sum(max(0, len(nb) - 1) - (i in nb[1:]) for i, nb in ((i, sm.neighbours(centres, i)) for i in range(K)) if len(nb) > 2)
    m = gem_b200.ElevationMap(64, res, compat_box_filter=False)
    total = sum(int(s.shape[0]) for s in subs)
    m.global_map_reserve(total, K)
    t_one, t_loop, equal = [], [], True
    for r in range(rounds + 1):
        m.global_map_reset()
        for s in range(K):
            m.global_map_push(subs[s], kf[s + 1])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fused = m.global_map_update(opt, res)
        t1 = time.perf_counter()
        work = [s.clone() for s in subs]
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        out, fh = sm.update_global_map(m, work, kf[:K], opt[:K], centres, res)
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        got = m.global_map_records()
        equal &= fused == fh and torch.equal(got.view(torch.int32), torch.cat(out).view(torch.int32))
        if r:
            t_one.append((t1 - t0) * 1e3)
            t_loop.append((t3 - t2) * 1e3)
    print(json.dumps({"shape": name, "L": L, "resolution": res, "submaps": K, "pairs": pairs, "records": total,
                      "records_after": int(m.global_map_info()[2]), "fused": fused, "equal": bool(equal),
                      "one_call_ms": round(float(np.median(t_one)), 3), "host_loop_ms": round(float(np.median(t_loop)), 3),
                      "rounds": rounds, "gpu": gpu_info()}), flush=True)


if __name__ == "__main__":
    for name in (sys.argv[1:] or list(SHAPES)):
        run(name, **SHAPES[name])
