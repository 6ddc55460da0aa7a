"""The call scripts of tests/sequence_cases.py on the device map and the oracle side by side, under every schedule the
add path has: one CUDA graph per call (the default), profiling on (fully serial, with per-kernel event timing), the
padded shared-memory launch of GEM_B200_EXCLUSIVE and a small GEM_B200_FOLD_BLOCKS cap.  At every reader and at the end of a script everything observable is compared bit for bit:
all layers, the state after each move, map_feature, the exports, the orthomosaic, the visual cloud, harvested records,
process_points outputs and stats(); and at the later readers the grid clouds, the split and its stats, the octree
streams, the costmap grids, windows and marks, the ROS messages byte for byte, the device layers, the local map, the
cuts and the global-map stack.  A difference names the script, the step and the schedule."""
import ctypes as C

import numpy as np
import pytest

import gem_b200
import sequence_cases as sc

pytestmark = pytest.mark.gpu

SCHEDULES = {
    "graph": {},
    "profile": {},
    "exclusive": {"GEM_B200_EXCLUSIVE": "1"},
    "fold_blocks_8": {"GEM_B200_FOLD_BLOCKS": "8"},
}
ENV = ("GEM_B200_EXCLUSIVE", "GEM_B200_FOLD_BLOCKS", "GEM_B200_LONG_BLOCKS")
_ORACLE = {}


def _oracle_trace(name):
    """the oracle's outputs of a script (the same under every schedule)"""
    if name not in _ORACLE:
        _ORACLE[name] = sc.run_oracle(sc.script_by_name(name))
    return _ORACLE[name]


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return f"shape {a.shape} != {b.shape}"
    if a.dtype.kind == "f":
        a32, b32 = a.astype(np.float32), b.astype(np.float32)
        ok = (a32.view(np.uint32) == b32.view(np.uint32)) | (np.isnan(a32) & np.isnan(b32))
    else:
        ok = a == b
    if ok.all():
        return None
    bad = np.argwhere(~ok)
    i = tuple(bad[0])
    return f"{bad.shape[0]} values differ, first at {i}: device={a[i]!r} oracle={b[i]!r}"


class DeviceRun:
    def __init__(self, script, schedule):
        self.s = script
        self.schedule = schedule
        self.g = gem_b200.ElevationMap(script.L, script.res, compat_box_filter=False, max_points=sc.MAX_POINTS)
        if schedule == "profile":
            self.g.profile_enable()
        self.keep = []           # device and pinned inputs stay alive until the map is closed
        self.proc = None
        self.last_move = None
        self.cost = {}           # window size -> [window, layer grid]

    def check(self, where, what, got, want):
        d = _same(got, want)
        assert d is None, f"{self.s.name} step {where} [{self.schedule}]: {what}: {d}"

    def _device(self, a):
        import torch
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        torch.cuda.synchronize()                         # the library works on its own stream
        self.keep.append(t)
        return t

    def _pinned(self, a):
        import torch
        t = torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
        self.keep.append(t)
        return t

    def _add(self, variant, c, f):
        g = self.g
        n = c["xyzi"].shape[0]
        if variant == "host":
            g.add(c["xyzi"], c["rgba"], f)
        elif variant == "dev":
            g.add(self._device(c["xyzi"]), self._device(c["rgba"]), f)
        elif variant == "stream":
            x, r = self._device(c["xyzi"]), self._device(c["rgba"])
            g.add_stream_fast(C.c_void_p(x.data_ptr()), C.c_void_p(r.data_ptr()), n, C.byref(f))
        elif variant == "host_async":
            x, r = self._pinned(c["xyzi"]), self._pinned(c["rgba"])
            g.add_host_async_fast(C.c_void_p(x.data_ptr()), C.c_void_p(r.data_ptr()), n, C.byref(f))
        elif variant == "pcl":
            g.add_pcl(sc.pcl_records(c), f)
        else:
            raise ValueError(variant)

    def _empty(self, variant):
        g, f = self.g, sc.frame(np.eye(4))
        if variant == "host":
            g.add(np.zeros((0, 4), np.float32), None, f)
        elif variant == "dev":
            g.add_fast(None, None, 0, C.byref(f))
        elif variant == "stream":
            g.add_stream_fast(None, None, 0, C.byref(f))
        elif variant == "host_async":
            g.add_host_async_fast(None, None, 0, C.byref(f))
        elif variant == "pcl":
            g.add_pcl(np.zeros((0, 8), np.float32), f)
        else:
            x = self._device(np.zeros((1, 4), np.float32))
            g.add_multi(x, None, [0, 0], [f])

    def _stats(self, where, want):
        if want is not None:
            got = self.g.stats()
            assert got == want, f"{self.s.name} step {where} [{self.schedule}]: stats {got} != oracle {want}"

    def _layers(self, where, want):
        for name, b in want.items():
            self.check(where, f"layer {name}", self.g.get_layer(name), b)

    def _readouts(self, where, want):
        g = self.g
        f = g.map_feature()
        for k, b in want["feature"].items():
            self.check(where, f"map_feature {k}", f[k], b)
        e = g.export_layers()
        for k, b in want["export"].items():
            self.check(where, f"export {k}", e[k], b)
        self.check(where, "orthomosaic", g.export_orthomosaic(), want["ortho"])
        xyz, rgb, n = g.export_visual_points()
        self.check(where, "visual cloud xyz", xyz, want["vis_xyz"])
        self.check(where, "visual cloud rgb", rgb, want["vis_rgb"])

    def step(self, i, op, a, want):
        g = self.g
        where = f"{i} ({op})"
        if op == "move":
            got = g.move(a["pos"])
            for k, what in enumerate(("centre", "start", "shift")):
                self.check(where, f"move {what}", got[k], want["returned"][k])
            c, st, z = g.state()
            oc, ost, oz = want["state"]
            self.check(where, "state centre", c, oc)
            self.check(where, "state start", st, ost)
            assert z == oz, f"{self.s.name} step {where} [{self.schedule}]: sensor z {z} != {oz}"
            self.last_move = (got[0], got[2])
        elif op == "add":
            self._add(a["variant"], self.s.clouds[a["cloud"]], sc.frame(a["T"]))
            if a["variant"] not in sc.PIPELINED:
                self._stats(where, sc_stats(want, self.s, a))
        elif op == "multi":
            cl = [self.s.clouds[n] for n in a["clouds"]]
            x = self._device(np.concatenate([c["xyzi"] for c in cl]))
            r = self._device(np.concatenate([c["rgba"] for c in cl]))
            off = np.concatenate([[0], np.cumsum([c["xyzi"].shape[0] for c in cl])])
            g.add_multi(x, r, off, [sc.frame(T) for T in a["Ts"]])
        elif op == "empty":
            self._empty(a["variant"])
        elif op == "var_update":
            g.var_update(a["dv"])
        elif op == "set_variance":
            v = g.get_layer("variance")
            self.check(where, "variance before set_layer", v, want["variance_in"])
            g.set_layer("variance", sc.set_variance_values(v))
        elif op == "opt_move":
            self.check(where, "opt_move aligned", g.opt_move(a["p"], a["dh"]), want["aligned"])
        elif op == "closeloop":
            g.closeloop(a["p"], a["dh"])
        elif op == "process":
            c = self.s.clouds[a["cloud"]]
            x = c["xyzi"]
            got = g.process_points(x[:, 0], x[:, 1], x[:, 2], sc.frame(a["T"]))
            for k, what in enumerate(("key", "var", "x", "y", "z")):
                self.check(where, f"process_points {what}", got[k], want["process"][k])
            self.proc = (c, got)
        elif op == "fuse":
            c, (key, var, _, _, zt) = self.proc
            R, G, B = (c["rgba"][:, k].astype(np.int32) for k in range(3))
            g.fuse_points(key, R, G, B, c["xyzi"][:, 3], zt, var)
        elif op == "layers":
            self._layers(where, want["layers"])
        elif op == "observe":
            self._layers(where, want["layers"])
            self._readouts(where, want)
        elif op == "export_ray":
            f = g.map_feature()
            for k, b in want["feature"].items():
                self.check(where, f"map_feature {k}", f[k], b)
            L = self.s.L
            out = {k: self._pinned(np.zeros((L, L), np.float32)).numpy().T for k in want["export"]}   # Fortran order
            g.export_layers_begin(out)
            g.raytracing()                                # may run while the copies are in flight
            g.export_layers_end()
            for k, b in want["export"].items():
                self.check(where, f"export_layers_begin/_end {k}", out[k], b)
        elif op == "raytracing":
            g.raytracing()
        elif op == "snapshot":
            f = g.map_feature()
            for k, b in want["feature"].items():
                self.check(where, f"map_feature {k}", f[k], b)
            g.snapshot_shown()
        elif op == "harvest":
            centre, shift = self.last_move
            rec, n = g.harvest_scrolled_out(centre, shift)
            orec, on = want["harvest"]
            assert n == on, f"{self.s.name} step {where} [{self.schedule}]: harvested {n} != {on}"
            self.check(where, "harvested records", rec, orec)
        elif op == "sync":
            g.sync()
            self._stats(where, want["stats"])
        elif op in sc.READERS:
            self.reader(where, op, a, want)
        else:
            raise ValueError(op)

    # ---- the later readers ----------------------------------------------------------------------------------------------
    def _records(self, where, what, got, want):
        self.check(where, what, got.cpu().numpy() if hasattr(got, "cpu") else got, want)

    def _split_stats(self, where, st, want):
        for k in ("points", "valid", "road", "obstacle"):
            n = want[k].shape[0] if k in ("road", "obstacle") else want[k]
            assert st[k] == n, f"{self.s.name} step {where} [{self.schedule}]: split {k} {st[k]} != {n}"
        for k in ("mean", "stddev", "threshold"):
            self.check(where, f"split {k}", np.float64(st[k]).view(np.uint64), np.float64(want[k]).view(np.uint64))

    def _ros(self, where, name, call, want):
        """the message into guarded device and pinned buffers at an offset that is not 16-byte aligned"""
        import torch
        nb = C.c_longlong(-1)
        assert call(None, 0, C.byref(nb)) == 0 and nb.value == len(want), \
            f"{self.s.name} step {where} [{self.schedule}]: {name} size {nb.value} != {len(want)}"
        for kind, off in sc.ROS_OFFSETS.items():
            n = len(want) + off + 2 * sc.ROS_GUARD
            buf = torch.full((n,), 0xA5, dtype=torch.uint8, device="cuda") if kind == "cuda" else \
                torch.full((n,), 0xA5, dtype=torch.uint8).pin_memory()
            at = sc.ROS_GUARD + off
            assert call(C.c_void_p(buf.data_ptr() + at), len(want), C.byref(nb)) == 0 and nb.value == len(want)
            torch.cuda.synchronize()
            got = buf.cpu().numpy().tobytes()
            assert got[:at] == b"\xa5" * at and got[at + len(want):] == b"\xa5" * (n - at - len(want)), \
                f"{self.s.name} step {where} [{self.schedule}]: {name} wrote outside its bytes ({kind})"
            if got[at:at + len(want)] != want:
                k = next(i for i in range(len(want)) if got[at + i] != want[i])
                raise AssertionError(f"{self.s.name} step {where} [{self.schedule}]: {name} ({kind}) differs from byte {k} "
                                     f"of {len(want)}")

    def reader(self, where, op, a, want):
        import torch
        g, L = self.g, self.s.L
        if op == "grid_cloud":
            self._records(where, f"grid cloud {a['src']}", g.export_grid_cloud(a["src"]), want["cloud"])
        elif op == "split":
            road, obstacle, st = g.grid_cloud_split(a["src"])
            self._records(where, "split road", road, want["road"])
            self._records(where, "split obstacle", obstacle, want["obstacle"])
            self._split_stats(where, st, want)
        elif op == "octrees":
            rs, os_, st = g.global_octrees(a["src"])
            self._split_stats(where, st, want)
            self.check(where, "road octree", rs.cpu().numpy(), want["road_stream"])
            self.check(where, "obstacle octree", os_.cpu().numpy(), want["obstacle_stream"])
        elif op == "costmap":
            sx, sy = a["size"]
            if a["size"] not in self.cost:
                self.cost[a["size"]] = [sc.initial_window(sx, sy), torch.from_numpy(sc.initial_grid(sx, sy)).cuda()]
            w, grid = self.cost[a["size"]]
            nx, ny = sc.cost_origin(g.state()[0], sx, sy)
            w = g.costmap_update_origin(w, nx, ny, sc.COST_FILL, grid)
            self.cost[a["size"]][0] = w
            assert np.float64(w[:3]).tobytes() == np.float64(want["window"][:3]).tobytes(), \
                f"{self.s.name} step {where} [{self.schedule}]: costmap window {w} != {want['window']}"
            marks = g.costmap_mark_map(w, grid, sc.COST_THRESH, a["src"], True)
            self.check(where, f"costmap grid {a['size']}", grid.cpu().numpy(), want["grid"])
            for k, v in want["marks"].items():
                assert np.float64(marks[k]).tobytes() == np.float64(v).tobytes(), \
                    f"{self.s.name} step {where} [{self.schedule}]: costmap marks {k} {marks[k]} != {v}"
        elif op == "ros":
            hc = gem_b200.RosHeader(**sc.ROS_HEADER).c()
            lib, h = g._lib, g.handle
            for name in ("visual_points", "grid_map", "orthomosaic"):   # visual_points first: it reads the map first
                fn = getattr(lib, f"gem_ros_{name}")
                self._ros(where, name, lambda p, c, nb, fn=fn: fn(h, C.byref(hc), p, c, nb), want["ros"][name])
        elif op == "layer_device":
            for name, b in want["device_layers"].items():
                out = torch.full((L, L), -7, dtype=torch.int32 if name.startswith("color") else torch.float32, device="cuda")
                g.get_layer_device(name, out)
                torch.cuda.synchronize()
                self.check(where, f"device layer {name}", out.cpu().numpy(), b)
        elif op == "local":
            centre, shift = self.last_move
            rec, n = g.harvest_to_local_map(centre, shift, records=True)
            orec, on = want["local"]
            assert n == on, f"{self.s.name} step {where} [{self.schedule}]: harvested {n} != {on}"
            self.check(where, "harvested records", rec, orec)
            assert g.local_map_size() == want["local_size"], \
                f"{self.s.name} step {where} [{self.schedule}]: local map {g.local_map_size()} != {want['local_size']}"
        elif op == "cut":
            cut = g.cut_submap(dense=a["dense"], seed=sc.CUT_SEED)
            self._records(where, "dense cut" if a["dense"] else "cut", cut, want["cut"])
            assert g.local_map_size() == 0
            g.global_map_push(cut, a["pose"])
            submaps, _, records = g.global_map_info()
            assert (submaps, records) == (want["submaps"], want["global"].shape[0]), \
                f"{self.s.name} step {where} [{self.schedule}]: global map {submaps} submaps, {records} records"
            self._records(where, "global map", g.global_map_records(), want["global"])
        else:
            raise ValueError(op)


def sc_stats(want, s, a):
    """stats() of a serial add: the oracle's process_points keys of the call"""
    key = want["keys"]
    k = key[key >= 0]
    counts = np.bincount(k, minlength=s.L * s.L)
    return {"points_in": int(s.clouds[a["cloud"]]["xyzi"].shape[0]), "points_binned": int(k.size),
            "cells_touched": int((counts > 0).sum()), "max_points_per_cell": int(counts.max()) if k.size else 0}


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("name", sc.SCRIPT_NAMES)
def test_script_matches_oracle(name, schedule, monkeypatch):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in SCHEDULES[schedule].items():
        monkeypatch.setenv(k, v)                          # gem_create reads the schedule
    trace = _oracle_trace(name)
    s = sc.script_by_name(name)
    run = DeviceRun(s, schedule)
    try:
        for i, (op, a, want) in enumerate(trace):
            run.step(i, op, a, want)
        run.g.sync()
        if schedule == "profile":
            pr = run.g.profile_read()
            assert pr["count"]["bin"] > 0 and pr["count"]["fold"] > 0, f"{name} [{schedule}]: {pr}"
            assert pr["ms"]["bin"] > 0 and pr["ms"]["fold"] > 0, f"{name} [{schedule}]: {pr}"
    finally:
        run.g.close()
