"""Host wall time of composingGlobalMap's octrees on the device at the c2 geometry (1024^2 at 0.05 m): FRAMES synthetic
HDL-64 frames are fused along a 0.3 m-per-frame track, the features computed and the shown map snapshotted (the node's
prevMap_), as in grid_split_bench.py.  Timed, CALLS times each after WARM warm-up calls, perf_counter around
host-synchronous calls (the time ends with the call's last host synchronisation):
  * global_octrees: grid_cloud_split (one synchronisation) + the road tree at 0.2 m + the obstacle tree at 0.1 m (three
    each: gem_color_octree synchronises twice, for its sizes and its counts, and the stream read once), plus the
    Python wrapper's stream synchronisations and its size query of the grid cloud;
  * each build alone: gem_color_octree + gem_color_octree_read into a device buffer on the split's device outputs
    (road 0.2 m, obstacle 0.1 m): three host synchronisations per call.
For context, the same two trees built by the C oracle (tests/orc_color_octree.c, a literal pointer octree, one thread) on
the host's cores: a CPU restatement of octomap, not octomap.  The oracle is compiled and the clouds copied to the host
before its clock starts; each tree is timed ORACLE_RUNS times (build + stream write, median).  The device streams are
checked against it.
The worst case of the design: a cloud that fills an aligned cube of side^3 voxels (one maximal full subtree, simulated by
one thread; up to 32^3 in shared memory, 64^3 in global scratch) with PER_VOXEL points per voxel in random order, device
build (median of CUBE_CALLS) beside the C oracle.
Prints one JSON line with the GPU name, SM clock and power limit as nvidia-smi reports them in the same run; writes
nothing."""
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

L, RES, FRAMES, NF, WARM, CALLS = 1024, 0.05, 40, 16, 5, 60
ORACLE_RUNS, CUBE_SIDES, PER_VOXEL, CUBE_CALLS = 5, (8, 16, 32, 64), 8, 3


def gpu_info():
    q = "name,clocks.sm,clocks.max.sm,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except Exception:
        return {"name": torch.cuda.get_device_name(0)}


def timed(fn, warm=WARM, calls=CALLS):
    ms = []
    for i in range(warm + calls):
        t0 = time.perf_counter()
        fn()
        dt = (time.perf_counter() - t0) * 1e3
        if i >= warm:
            ms.append(dt)
    return {"median": round(float(np.median(ms)), 3), "min": round(float(np.min(ms)), 3), "max": round(float(np.max(ms)), 3),
            "calls": len(ms)}


def main():
    scene = synth.make_scene()
    m = gem_b200.ElevationMap(L, RES, compat_box_filter=False, grid_resolution=RES)
    lib, h = m._lib, m.handle
    for k in range(FRAMES):
        fr = synth.hdl64_frame(k % NF, scene=scene)
        pos = np.array([0.3 * k, 0.1 * k, 1.7], np.float32)
        T = fr["T"].copy()
        T[:3, 3] = pos
        m.move(pos)
        m.add(torch.from_numpy(fr["xyzi"]).cuda(), torch.from_numpy(fr["rgba"]).cuda(),
              gem_b200.make_frame(T, gem_b200.LaserSensorProcessor()))
    m.compute_features()
    m.snapshot_shown()
    m.sync()
    road, obst, st = m.grid_cloud_split("snapshot")
    torch.cuda.synchronize()
    out = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    info = gem_b200._lib.GemOctree()

    def build(cloud, res):
        def call():
            assert lib.gem_color_octree(h, C.c_void_p(cloud.data_ptr()), cloud.shape[0], res, C.byref(info)) == 0, lib.gem_last_error(h)
            assert lib.gem_color_octree_read(h, C.c_void_p(out.data_ptr()), out.numel()) == 0, lib.gem_last_error(h)
        return call

    res = {"gpu": gpu_info(), "geometry": {"L": L, "res": RES, "frames": FRAMES}, "grid_cloud_points": st["points"],
           "road_points": st["road"], "obstacle_points": st["obstacle"]}
    res["global_octrees_ms"] = timed(lambda: m.global_octrees())
    res["road_build_0.2m_ms"] = timed(build(road, 0.2))
    road_info = {k: getattr(info, k) for k, _ in gem_b200._lib.GemOctree._fields_}
    res["obstacle_build_0.1m_ms"] = timed(build(obst, 0.1))
    obst_info = {k: getattr(info, k) for k, _ in gem_b200._lib.GemOctree._fields_}
    res["road_tree"], res["obstacle_tree"] = road_info, obst_info
    rs, os_, _ = m.global_octrees()
    import octree_cases
    import octree_oracle
    octree_oracle.load()                                    # compiled before any clock starts
    road_h, obst_h = road.cpu().numpy(), obst.cpu().numpy()
    want = {}

    def oracle(key, cloud, r):
        def call():
            want[key] = octree_oracle.color_octree(cloud, r)[0]
        return call

    cpu = {"note": "C oracle: a CPU restatement of octomap 1.9, not octomap", "threads": 1,
           "road_0.2m_ms": timed(oracle("road", road_h, 0.2), 1, ORACLE_RUNS),
           "obstacle_0.1m_ms": timed(oracle("obstacle", obst_h, 0.1), 1, ORACLE_RUNS)}
    res["cpu_restatement"] = cpu
    res["device_equals_c_oracle"] = bool(np.array_equal(rs.cpu().numpy(), want["road"]) and
                                         np.array_equal(os_.cpu().numpy(), want["obstacle"]))
    rng = np.random.default_rng(1)
    cubes = {}
    for side in CUBE_SIDES:
        k = octree_cases.block_keys((0, 0, 0), side)
        k = np.repeat(k, PER_VOXEL, axis=0)[rng.permutation(k.shape[0] * PER_VOXEL)]
        rec = octree_cases.cloud(k, 0.1, rng.integers(0, 256, (k.shape[0], 3)))
        dev = torch.from_numpy(rec).cuda()
        torch.cuda.synchronize()
        c = {"points": int(rec.shape[0]), "device_ms": timed(build(dev, 0.1), 1, CUBE_CALLS)}
        c["tree"] = {f: getattr(info, f) for f, _ in gem_b200._lib.GemOctree._fields_}
        got = out[:info.bytes].cpu().numpy()
        c["c_oracle_ms"] = timed(oracle("cube", rec, 0.1), 1, 3)
        c["device_equals_c_oracle"] = bool(np.array_equal(got, want["cube"]))
        cubes[f"{side}^3"] = c
    res["full_cube_worst_case"] = {"per_voxel": PER_VOXEL, "resolution": 0.1, "order": "random", "cubes": cubes}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
