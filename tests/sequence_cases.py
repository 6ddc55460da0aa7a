"""Call scripts for the add schedule of gem_api.cu: one map, a list of API calls, run against the oracle.

The library does not run the reference's arithmetic in the reference's order.  gem_move only queues its scroll clears
(RegionOps: row / column bands, two per axis when a band wraps the storage edge); the next fusing call executes them in
spare blocks of its bin kernel, a pipelined fold executes the NEXT call's clears itself (in_clear_region), readers flush
the clears early but keep their variance floor pending, more than MAX_REGION_OPS ops are launched on their own, and
gem_process_points parks the list.  The every-cell variance floor of each Fuse runs only where it can matter: cleared
bands, and every cell after the first fuse, after a negative gem_var_update and after gem_set_layer(variance).

Every hand-written script below targets one of those decisions and is named after it; tests/test_sequence_cases.py
checks on the oracle alone that each one reaches its hazard, tests/test_sequences_gpu.py runs every script on the
device under each schedule (the default graph, profiling, GEM_B200_EXCLUSIVE, GEM_B200_FOLD_BLOCKS) against the oracle.

A script is a list of steps (op, args).  Ops:
  move pos                       gem_move; the state and the returned centre / start / shift are compared
  add variant cloud T            variant: host (gem_add_points_host), dev (gem_add_points), stream, host_async, pcl
  multi clouds Ts                gem_add_points_multi, one segment per cloud, own frames
  empty variant                  an add call of n = 0 (every variant, and multi): a Fuse of no points
  var_update dv                  gem_var_update
  set_variance                   get_layer(variance), lower some of it below the floor, set_layer(variance)
  opt_move p dh / closeloop p dh
  process cloud T / fuse         gem_process_points (outputs compared), then gem_fuse of its outputs
  layers                         a reader: every layer compared
  observe                        layers, map_feature, export, orthomosaic, visual cloud
  export_ray                     map_feature, export_layers_begin, raytracing, export_layers_end
  raytracing
  snapshot / harvest             map_feature + snapshot_shown, then harvest_scrolled_out with the last move's centre
                                 and shift
  sync                           gem_sync, then stats() against the last add call

The later readers read the shown map as it stands: the live elevation, variance, intensity and colour, with the rough,
slope and traversability the last feature pass wrote (the oracle keeps that pass's outputs).  Their ops:
  grid_cloud src                 gem_export_grid_cloud of the shown map or the snapshot (src: shown / snapshot)
  split src                      gem_grid_cloud_split: road, obstacle and the filter's stats
  octrees src                    global_octrees: the split, then the 0.2 m road and 0.1 m obstacle ColorOcTree streams
  costmap src size               gem_costmap_update_origin of the layer grid of that window size to the map centre, then
                                 gem_costmap_mark_map into it: grid, window and marks (each size keeps its own grid, both
                                 calls share the handle's costmap scratch)
  ros                            gem_ros_visual_points, gem_ros_grid_map, gem_ros_orthomosaic into device and pinned
                                 memory at offsets that are not 16-byte aligned, guard bytes around them
  layer_device                   gem_get_layer_device of every layer, rough, slope and the feature traversability included
  local                          gem_harvest_to_local_map with the last move's centre and shift: records and store size
  cut dense pose                 cut_submap (dense: the MLS points of the taken local map between it and the grid cloud),
                                 then global_map_push of the cut: the whole global-map stack is compared

Hazards (kind, step) the CPU suite checks: long_clear, wrap, overflow, full_shift_pending, boundary, var_below_floor,
set_below_floor, pending_fold_and_clears, multi_frames and harvest (each at the step that raises it), and, in the scripts
named readers_after_*, at a later reader placed directly after
  reader_fold_in_flight          a pipelined add (stream, host_async) whose fold is still to be issued
  reader_queued_clears           a move whose bands are queued (wrapping the storage edge on both axes, or the whole map)
  reader_floor_pending           a negative var_update or a set_variance: the variance floor waits for the next Fuse
  reader_parked                  gem_process_points with its fuse still to come (the pending operations are parked)
"""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass, field

import numpy as np

import costmap_oracle
import mls_oracle
import np_reference
import octree_oracle
import oracle_lib
import rosmsg_oracle
import split_oracle
import submap_oracle
from oracle_lib import OracleMap

f32 = np.float32
MAX_REGION_OPS = 6                   # gem_kernels.cuh
MAX_POINTS = 1 << 16                 # per-launch capacity of the device maps the scripts run on
ADD_VARIANTS = ("host", "dev", "stream", "host_async", "pcl")
PIPELINED = ("stream", "host_async", "multi")
EMPTY_VARIANTS = ADD_VARIANTS + ("multi",)
READERS = ("grid_cloud", "split", "octrees", "costmap", "ros", "layer_device", "local", "cut")
READER_HAZARDS = ("reader_fold_in_flight", "reader_queued_clears", "reader_floor_pending", "reader_parked")
COST_RES, COST_THRESH, COST_FILL = 0.15, 0.7, 255      # costmap cells of 1.5 map cells: several map cells per costmap cell
COST_SIZES = ((23, 19), (41, 37))                       # inside the 64-cell window, and wider than it
ROS_HEADER = {"seq": 7, "stamp_sec": 1700000000, "stamp_nsec": 123456789, "frame_id": "map"}
ROS_OFFSETS = {"cuda": 7, "pinned": 13}                 # destination offsets that are not 16-byte aligned
ROS_GUARD = 64
CUT_SEED = 11                                           # the MLS seed of the dense cuts


def initial_window(sx, sy):
    return (-sx * COST_RES / 2, -sy * COST_RES / 2, COST_RES, sx, sy)


def initial_grid(sx, sy):
    """a costmap layer grid of free, lethal and unknown cells, so that a cell left unwritten shows"""
    return np.random.default_rng(1000 * sx + sy).choice(np.array([0, 254, 255], np.uint8), (sy, sx))


def cost_origin(centre, sx, sy):
    """the origin update_origin is asked for: the window centred on the map centre"""
    return float(centre[0]) - sx * COST_RES / 2, float(centre[1]) - sy * COST_RES / 2


# ---- gem_move's arithmetic, restated (gem_api.cu gem_move, oracle orc_move) ----------------------------------------------
def _d2i(d: float) -> int:
    if d != d:
        return 0
    if d >= 2147483648.0:
        return 2147483647
    if d <= -2147483649.0:
        return -2147483648
    return math.trunc(d)


def _index_to_range(index: int, L: int) -> int:
    if index < 0:
        index += ((-index // L) + 1) * L       # -index / L of non-negative ints
    return index % L


def _roundf(x: f32) -> float:
    """roundf: half away from zero (exact in double for a float argument)"""
    a = math.floor(abs(float(x)) + 0.5)
    return -a if x < 0 else a


def _position_to_range(p: f32, shift: f32, res: f32) -> f32:
    pi = _d2i(_roundf(f32(p / res)))
    si = _d2i(_roundf(f32(shift / res)))
    return f32(f32(pi + si) * res)


def index_shift(pos: float, centre: f32, res: f32) -> int:
    ps = f32(f32(pos) - centre)
    return _d2i(float(f32(ps / res)) + 0.5 * (1 if ps > 0 else -1))


def move_model(L: int, res: float, centre, start, pos):
    """gem_move on (centre, start): returns (centre, start, shift, ops); ops are the RegionOps it queues:
    ("rows" | "cols", first, n), or ("all",) for |shift| >= L"""
    res = f32(res)
    centre = [f32(c) for c in centre]
    start = [int(s) for s in start]
    shifts = [index_shift(pos[i], centre[i], res) for i in range(2)]
    aligned = [f32(f32(s) * res) for s in shifts]
    ops = []
    for i in range(2):
        s = shifts[i]
        kind = "rows" if i == 0 else "cols"
        if s != 0:
            if s >= L or s <= -L:
                ops.append(("all",))
            else:
                sign = 1 if s > 0 else -1
                first = start[i] - (1 if sign > 0 else 0)
                end = first + sign - s
                n = abs(s)
                index = _index_to_range(first if sign < 0 else end, L)
                if index + n <= L:
                    ops.append((kind, index, n))
                else:
                    ops.append((kind, index, L - index))
                    ops.append((kind, 0, n - (L - index)))
        start[i] = _index_to_range(start[i] - s, L)
        centre[i] = _position_to_range(centre[i], aligned[i], res)
    return centre, start, aligned, ops


def band_cells(L: int, ops) -> np.ndarray:
    """storage cells (row * L + col) the ops clear"""
    mask = np.zeros((L, L), bool)
    for op in ops:
        if op[0] == "all":
            mask[:] = True
        elif op[0] == "rows":
            mask[op[1]:op[1] + op[2], :] = True
        else:
            mask[:, op[1]:op[1] + op[2]] = True
    return np.flatnonzero(mask.reshape(-1))


# ---- clouds -------------------------------------------------------------------------------------------------------------
def sensor():
    import gem_b200
    return gem_b200.LaserSensorProcessor(ignore_points_above=100.0, ignore_points_below=-100.0)


def frame(T):
    import gem_b200
    return gem_b200.make_frame(np.asarray(T, np.float64), sensor())


def pose(x, y, z=0.0, yaw=0.0):
    c, s = math.cos(yaw), math.sin(yaw)
    T = np.eye(4)
    T[:2, :2] = [[c, -s], [s, c]]
    T[:3, 3] = (x, y, z)
    return T


def cloud(L, res, centre, seed, stripe=24, ks=(12, 20, 50, 90, 160), scale=1.0, sparse=1500, phase=0, T=None, relief=1.0):
    """dense patches on a diagonal stripe pattern of the window around `centre` (every row and every column of the
    storage holds cells with 9..40 and with more than 40 records, whatever the scroll), plus sparse points over and
    around the window, in random order.  World coordinates, expressed in the sensor frame of pose T (identity: None);
    relief scales the height differences (small: flat, traversable ground)."""
    rng = np.random.default_rng(seed)
    ix, iy = np.meshgrid(np.arange(L), np.arange(L), indexing="ij")
    cells = np.argwhere(((ix + iy + phase) % stripe) == 0)
    k = np.maximum(1, (np.asarray(ks)[(3 * cells[:, 0] + cells[:, 1] + phase) % len(ks)] * scale).astype(int))
    off = (L / 2 - 0.5) if L % 2 == 0 else L // 2
    cx = float(centre[0]) + (off - cells[:, 0]) * res
    cy = float(centre[1]) + (off - cells[:, 1]) * res
    base = 0.1 + relief * rng.uniform(-0.5, 0.5, cells.shape[0])
    rep = np.repeat(np.arange(cells.shape[0]), k)
    n = rep.shape[0]
    x = cx[rep] + rng.uniform(-0.3, 0.3, n) * res
    y = cy[rep] + rng.uniform(-0.3, 0.3, n) * res
    z = base[rep] + relief * rng.normal(0.0, 0.03, n)
    jump = rng.uniform(size=n) < 0.06                     # points the Mahalanobis gate has to decide
    z[jump] += relief * rng.uniform(0.2, 1.0, jump.sum())
    half = L * res / 2 * 1.15
    xs = float(centre[0]) + rng.uniform(-half, half, sparse)
    ys = float(centre[1]) + rng.uniform(-half, half, sparse)
    zs = 0.1 + relief * rng.uniform(-0.6, 0.9, sparse)
    xyz = np.concatenate([np.stack([x, y, z], 1), np.stack([xs, ys, zs], 1)])
    if T is not None:
        T = np.asarray(T, np.float64)
        xyz = (xyz - T[:3, 3]) @ T[:3, :3]                   # world -> sensor
    m = xyz.shape[0]
    inten = rng.integers(0, 256, m).astype(np.float32)
    inten[rng.uniform(size=m) < 0.05] = 0
    rgba = rng.integers(0, 256, (m, 4)).astype(np.uint8)
    rgba[rng.uniform(size=m) < 0.1, rng.integers(0, 3)] = 0
    perm = rng.permutation(m)
    xyzi = np.concatenate([xyz.astype(np.float32), inten[:, None]], 1)[perm]
    return {"xyzi": np.ascontiguousarray(xyzi, np.float32), "rgba": np.ascontiguousarray(rgba[perm])}


def pcl_records(c):
    """PointXYZRGBICT records of a cloud: x y z _ bgr(as float) _ intensity _"""
    n = c["xyzi"].shape[0]
    rec = np.zeros((n, 8), np.float32)
    rec[:, 0:3] = c["xyzi"][:, :3]
    bgr = (c["rgba"][:, 2].astype(np.uint32) | (c["rgba"][:, 1].astype(np.uint32) << 8) |
           (c["rgba"][:, 0].astype(np.uint32) << 16))
    rec[:, 4] = bgr.view(np.float32)
    rec[:, 6] = c["xyzi"][:, 3]
    return rec


# ---- scripts ------------------------------------------------------------------------------------------------------------
@dataclass
class Script:
    name: str
    L: int
    res: float
    steps: list = field(default_factory=list)
    clouds: dict = field(default_factory=dict)
    hazards: list = field(default_factory=list)   # (kind, step index) the CPU suite checks


class Builder:
    """writes a script while tracking the map's centre / start with move_model, so that clouds land in the window"""

    def __init__(self, name, L=64, res=0.1, seed=0):
        self.s = Script(name, L, res)
        self.centre = [f32(0), f32(0)]
        self.start = [0, 0]
        self.seed = seed * 1000 + 7
        self.last_move = None

    def _step(self, op, **args):
        self.s.steps.append((op, args))
        return len(self.s.steps) - 1

    def hazard(self, kind, idx):
        self.s.hazards.append((kind, idx))

    def new_cloud(self, T=None, **kw):
        self.seed += 1
        name = f"c{len(self.s.clouds)}"
        self.s.clouds[name] = cloud(self.s.L, self.s.res, self.centre, self.seed, T=T, phase=self.seed % 7, **kw)
        return name

    def move(self, x, y, z=0.0):
        pos = (float(f32(x)), float(f32(y)), float(f32(z)))
        self.centre, self.start, _, _ = move_model(self.s.L, self.s.res, self.centre, self.start, pos)
        self.last_move = pos
        return self._step("move", pos=pos)

    def move_cells(self, dx, dy, z=0.0):
        """a move of (dx, dy) cells (aligned positions, no rounding question)"""
        r = self.s.res
        return self.move(float(self.centre[0]) + dx * r, float(self.centre[1]) + dy * r, z)

    def move_to_start(self, sx, sy):
        """a move that leaves the storage start at (sx, sy), by a shift of less than L / 2 cells per axis"""
        L = self.s.L
        d = [(self.start[i] - t) % L for i, t in enumerate((sx, sy))]
        d = [v - L if v >= L // 2 else v for v in d]
        i = self.move_cells(d[0], d[1])
        assert self.start == [sx, sy], (self.start, sx, sy)
        return i

    def cut(self, dense):
        return self._step("cut", dense=dense, pose=pose(float(self.centre[0]), float(self.centre[1]), 0.5))

    def add(self, variant="stream", T=None, **kw):
        if variant == "multi":
            return self.multi(**kw)
        T = np.eye(4) if T is None else T
        return self._step("add", variant=variant, cloud=self.new_cloud(T=T, **kw), T=T)

    def multi(self, nseg=3, yaw0=0.0, scale=0.3):
        Ts = [pose(0.05 * k - 0.1, -0.03 * k, 0.02 * k, yaw0 + 0.3 * k) for k in range(nseg)]
        names = [self.new_cloud(T=T, scale=scale, sparse=300, stripe=32) for T in Ts]
        return self._step("multi", clouds=names, Ts=Ts)

    def empty(self, variant):
        return self._step("empty", variant=variant)

    def op(self, op, **args):
        return self._step(op, **args)

    def done(self):
        if not self.s.steps or self.s.steps[-1][0] != "observe":
            self._step("observe")
        return self.s


def boundary_position(res, centre, k, sign, before):
    """the float32 position nearest centre + sign * (k + 0.5) * res whose index shift is k (before=True) or k + 1, one ulp
    from the other: gem_move's d2i(ps / res + 0.5 sign) decides it"""
    res32 = f32(res)
    p = f32(float(centre) + sign * (k + 0.5) * res)
    away = f32(np.inf) * sign
    for _ in range(64):                                   # walk to the last position with shift k
        if abs(index_shift(float(p), f32(centre), res32)) > k:
            p = np.nextafter(p, -away)
        elif abs(index_shift(float(np.nextafter(p, away)), f32(centre), res32)) == k:
            p = np.nextafter(p, away)
        else:
            break
    assert abs(index_shift(float(p), f32(centre), res32)) == k
    return float(p) if before else float(np.nextafter(p, away))


def hand_written():
    out = []

    for axis in ("rows", "cols"):
        b = Builder(f"clear_rides_on_fold_{axis}", seed=1 if axis == "rows" else 2)
        b.add("stream")
        b.add("stream")
        i = b.move_cells(5, 0) if axis == "rows" else b.move_cells(0, -4)
        b.hazard("long_clear", i)
        b.add("stream")
        i = b.move_cells(3, 3)
        b.hazard("long_clear", i)
        b.add("stream")
        out.append(b.done())

    b = Builder("wrap_split_band", seed=3)
    b.add("stream")
    b.move_cells(3, 4)
    b.add("stream")
    i = b.move_cells(-6, -7)                              # from start (L-3, L-4): bands wrap on both axes
    b.hazard("wrap", i)
    b.hazard("long_clear", i)
    b.add("stream")
    b.op("layers")
    b.move_cells(2, -2)
    b.add("host")
    out.append(b.done())

    b = Builder("overflow_many_moves", seed=4)
    b.add("stream")
    for _ in range(4):                                    # 8 row / column bands, all distinct: the two oldest go alone
        i = b.move_cells(3, 3)
    b.hazard("overflow", i)
    b.add("stream")
    b.add("stream")
    for _ in range(3):
        b.move_cells(-2, 5)
    i = b.move_cells(-6, -6)
    b.hazard("overflow", i)
    b.add("host")
    out.append(b.done())

    b = Builder("full_shift_with_pending_fold", seed=5)
    L = b.s.L
    for dx, dy in ((L, 0), (-L - 3, 0), (0, L + 1), (0, -L)):
        b.add("stream")
        b.add("stream")
        i = b.move_cells(dx, dy)
        b.hazard("full_shift_pending", i)
        b.add("stream")
    b.add("stream")
    b.move_cells(L, 2)                                    # everything cleared, then a row band on top
    b.add("host")
    out.append(b.done())

    b = Builder("shift_boundary_ulp", seed=6)
    for k, sign, axis, before in ((2, 1, 0, True), (2, 1, 0, False), (3, -1, 1, True), (3, -1, 1, False),
                                  (0, 1, 1, True), (0, -1, 0, False)):
        b.add("stream")
        c = b.centre[axis]
        p = boundary_position(b.s.res, c, k, sign, before)
        pos = [float(b.centre[0]), float(b.centre[1])]
        pos[axis] = p
        i = b.move(pos[0], pos[1])
        b.hazard("boundary", i)
    b.add("stream")
    out.append(b.done())

    b = Builder("var_update_signs", seed=7)
    b.add("stream")
    b.add("stream")
    i = b.op("var_update", dv=-7.5e-5)                   # fused cells sit at the 1e-4 floor: they drop below it
    b.hazard("var_below_floor", i)
    b.add("stream", stripe=48)                           # touches few cells: the others need the all-cell floor
    b.op("layers")
    b.op("var_update", dv=2.5e-3)
    b.add("stream")
    b.op("var_update", dv=0.0)
    b.add("stream")
    i = b.op("var_update", dv=-9e-5)
    b.hazard("var_below_floor", i)
    b.move_cells(2, 0)
    b.add("dev", stripe=48)
    out.append(b.done())

    b = Builder("set_variance_between_pipelined", seed=8)
    b.add("stream")
    b.add("stream")
    i = b.op("set_variance")
    b.hazard("set_below_floor", i)
    b.add("stream", stripe=48)
    b.move_cells(1, 1)
    b.add("stream")
    out.append(b.done())

    b = Builder("opt_move_closeloop_pending", seed=9)
    b.add("stream")
    b.add("stream")
    b.move_cells(3, -2)
    i = b.op("opt_move", p=(0.37, -0.52), dh=0.125)       # a fold and two bands pending
    b.hazard("pending_fold_and_clears", i)
    b.centre = [f32(c) for c in _opt_move_centre(b.centre, (0.37, -0.52), b.s.res)]
    b.add("stream")
    b.move_cells(-2, 4)
    i = b.op("closeloop", p=(0.81, 0.33), dh=-0.25)
    b.hazard("pending_fold_and_clears", i)
    b.centre = [f32(c) for c in _closeloop_centre(b.centre, (0.81, 0.33), b.s.res)]
    b.add("stream")
    b.add("stream")
    out.append(b.done())

    b = Builder("parked_clears_process_points", seed=10)
    b.add("stream")
    b.add("stream")
    i = b.move_cells(4, -3)
    b.hazard("long_clear", i)
    b.op("process", cloud=b.new_cloud(), T=np.eye(4))
    b.op("layers")                                        # the clears parked across process_points are visible
    b.op("fuse")
    b.move_cells(2, 2)
    b.op("process", cloud=b.new_cloud(), T=np.eye(4))
    b.op("fuse")                                          # clears and floors parked, then taken by the fuse
    b.add("stream")
    out.append(b.done())

    b = Builder("empty_call_flushes", seed=11)
    for v in EMPTY_VARIANTS:
        b.add("stream")
        b.add("stream")
        i = b.move_cells(2, -1)
        b.hazard("long_clear", i)
        b.empty(v)
        b.op("layers")
    b.add("host")
    out.append(b.done())

    b = Builder("export_around_raytracing", seed=12)
    b.add("stream")
    b.move_cells(1, 2, z=1.5)
    b.add("stream")
    b.op("export_ray")
    b.add("stream")
    b.move_cells(-3, 1, z=2.0)
    b.add("stream")
    b.op("export_ray")
    b.add("host")
    out.append(b.done())

    b = Builder("snapshot_harvest_after_pipelined", seed=13)
    b.add("stream")
    b.add("stream", stripe=1, ks=(1, 2, 3), relief=0.01)              # every cell: the features give the whole window a traversability
    b.op("snapshot")
    b.move_cells(6, -5)
    b.hazard("harvest", b.op("harvest"))
    b.add("stream")
    b.add("stream", stripe=1, ks=(1, 2, 3), relief=0.01)
    b.op("snapshot")
    b.move_cells(-4, 7)
    b.hazard("harvest", b.op("harvest"))
    b.add("stream")
    out.append(b.done())

    b = Builder("multi_steady_state", seed=14)
    for k, nseg in enumerate((2, 5, 8, 3, 6, 4, 7)):
        i = b.multi(nseg=nseg, yaw0=0.4 * k)
        b.hazard("multi_frames", i)
        if k in (2, 4):
            b.move_cells(2, -1)
    b.op("sync")
    b.multi(nseg=2, yaw0=-0.7)
    b.multi(nseg=3, yaw0=1.1)
    out.append(b.done())

    b = Builder("host_async_alternating", seed=15)
    for v in ("stream", "host", "pcl", "dev", "stream"):
        b.add("host_async")
        b.add(v)
        b.move_cells(1, -1)
    b.add("host_async")
    b.add("host_async")
    b.op("sync")
    b.add("host_async")
    out.append(b.done())

    b = Builder("reader_between_pipelined", seed=16)
    b.add("stream")
    b.move_cells(2, 0)
    b.add("stream")
    b.op("layers")                                        # flushes the clears, keeps their floor pending
    b.move_cells(0, 3)
    b.op("layers")
    b.add("stream", stripe=48)
    b.op("raytracing")
    b.add("stream")
    b.op("sync")
    out.append(b.done())

    b = Builder("odd_length_scroll", L=65, seed=17)
    b.add("stream")
    i = b.move_cells(4, -6)
    b.hazard("long_clear", i)
    b.add("stream")
    b.move_cells(-9, 3)
    b.add("host")
    out.append(b.done())
    return out + readers_after_hazards() + [node_frame_loop()]


# ---- the later readers straight after each hazard ------------------------------------------------------------------------
def _reader_ops(k):
    """the readers of one readers_after_* script, in order: every op of READERS, the costmap at both sizes (its scratch
    alternates between the marks' ints and update_origin's bytes at both sizes), both sources, dense and plain cuts"""
    a, b = ("shown", "snapshot") if k % 2 == 0 else ("snapshot", "shown")
    return [("grid_cloud", {"src": "shown"}), ("split", {"src": a}), ("octrees", {"src": b}),
            ("costmap", {"src": "shown", "size": COST_SIZES[0]}), ("ros", {}), ("layer_device", {}), ("local", {}),
            ("cut", {"dense": True}), ("costmap", {"src": "shown", "size": COST_SIZES[1]}), ("grid_cloud", {"src": "snapshot"}),
            ("split", {"src": b}), ("octrees", {"src": a}), ("costmap", {"src": "snapshot", "size": COST_SIZES[0]}),
            ("cut", {"dense": False})]


def _fill(b):
    """an add that puts a few points into every cell of flat ground, then features + snapshot: the whole window is shown
    and traversable, so every reader has cells to read and the harvest has cells to take"""
    b.add("stream", stripe=1, ks=(1, 2, 3), relief=0.05)
    b.op("snapshot")


def _reader(b, op, args):
    return b.cut(args["dense"]) if op == "cut" else b.op(op, **args)


def readers_after_hazards():
    """one script per hazard: each round sets the map up, raises the hazard, and puts the next reader right after it"""
    out = []
    for k, (name, trigger) in enumerate((("readers_after_stream_fold", "stream"),
                                         ("readers_after_host_async_fold", "host_async"),
                                         ("readers_after_wrapping_clears", "wrap"), ("readers_after_full_shift", "full"),
                                         ("readers_after_negative_var_update", "var_update"),
                                         ("readers_after_set_variance", "set_variance"),
                                         ("readers_after_parked_process", "process"))):
        b = Builder(name, seed=20 + k)
        for op, args in _reader_ops(k):
            if trigger == "wrap":
                b.move_to_start(2, 3)
                _fill(b)
                h, kind = b.move_cells(5, 6), "reader_queued_clears"     # shifts above the start: both bands wrap
            elif trigger == "full":
                _fill(b)
                h, kind = b.move_cells(b.s.L + 1, -2), "reader_queued_clears"
            else:
                _fill(b)
                b.move_cells(3, -2)
                if trigger in ("stream", "host_async"):
                    h, kind = b.add(trigger, relief=0.3), "reader_fold_in_flight"
                elif trigger == "var_update":
                    b.add("stream", relief=0.3)
                    h, kind = b.op("var_update", dv=-7.5e-5), "reader_floor_pending"
                elif trigger == "set_variance":
                    b.add("stream", relief=0.3)
                    h, kind = b.op("set_variance"), "reader_floor_pending"
                else:
                    h, kind = b.op("process", cloud=b.new_cloud(relief=0.3), T=np.eye(4)), "reader_parked"
            i = _reader(b, op, args)
            assert i == h + 1
            b.hazard(kind, i)
            if trigger == "process":
                b.op("fuse")
        b.add("stream")                                   # a Fuse takes the last round's pending floor and clears
        out.append(b.done())
    return out


NODE_FRAMES = 14


def node_frame_loop():
    """the node's per-frame order on one handle: Move, harvest into the local map, add, features + snapshot, the grid
    cloud, the map topics, the local costmap; every third frame the global map's split and octrees and a keyframe cut
    (every other one dense); then the ray clean-up.  The first frames fill the window with small moves, the later ones
    scroll it away in long moves over sparse clouds, and the costmap window widens and narrows again: the grid cloud,
    the harvest and the costmap each grow and later shrink."""
    b = Builder("node_frame_loop", seed=31)
    sizes = [(9, 7), (15, 13), (23, 19), (31, 27), (41, 37), (49, 45), (49, 45), (41, 37), (31, 27), (23, 19), (15, 13),
             (9, 7), (9, 7), (15, 13)]
    variants = ("stream", "stream", "host_async", "host", "stream", "dev", "stream")
    for k in range(NODE_FRAMES):
        if k < 6:
            b.move_cells(1, (k % 2) - 1)
        else:
            b.move_cells(7, -6)
        if k > 0:
            b.op("local")
        if k < 6:
            b.add(variants[k % len(variants)], sparse=500, relief=0.25)
        else:
            b.add(variants[k % len(variants)], stripe=64, sparse=80, scale=0.5, relief=0.25)
        b.op("snapshot")
        b.op("grid_cloud", src="shown")
        b.op("ros")
        b.op("costmap", src="shown", size=sizes[k])
        if k % 3 == 2:
            b.op("split", src="snapshot")
            b.op("octrees", src="snapshot")
            b.cut(dense=k % 6 == 5)
        b.op("raytracing")
    return b.done()


def _opt_move_centre(centre, p, res):
    res = f32(res)
    out = []
    for i in range(2):
        ps = f32(f32(p[i]) - centre[i])
        s = _d2i(float(f32(ps / res)) + 0.5 * (1 if ps > 0 else -1))
        out.append(f32(centre[i] + f32(res * f32(s))))
    return out


def _closeloop_centre(centre, p, res):
    res = f32(res)
    out = []
    for i in range(2):
        ps = f32(f32(p[i]) - centre[i])
        s = _d2i(float(f32(ps / res)) + 0.5 * (1 if ps > 0 else -1))
        out.append(_position_to_range(centre[i], f32(f32(s) * res), res))
    return out


# ---- random scripts -----------------------------------------------------------------------------------------------------
SEEDS = (101, 102, 103, 104)


def random_script(seed, n_steps=28):
    rng = np.random.default_rng(seed)
    L = int(rng.choice([64, 80, 96]))
    b = Builder(f"random_{seed}", L=L, seed=seed)
    vocab = ["add", "add", "add", "add", "move", "move", "move", "layers", "var_update", "set_variance", "opt_move",
             "closeloop", "process", "empty", "export_ray", "snapshot", "sync", "multi", "raytracing"] + list(READERS)
    snap = False
    for _ in range(n_steps):
        op = vocab[int(rng.integers(len(vocab)))]
        if op in ("grid_cloud", "split", "octrees", "costmap"):
            args = {"src": "snapshot" if snap and rng.uniform() < 0.4 else "shown"}
            if op == "costmap":
                args["size"] = COST_SIZES[int(rng.integers(len(COST_SIZES)))]
            b.op(op, **args)
        elif op == "local":
            b.op("local" if snap and b.last_move is not None else "layer_device")
        elif op == "cut":
            b.cut(dense=False)
        elif op == "add":
            b.add(str(rng.choice(ADD_VARIANTS + ("stream", "stream"))), stripe=int(rng.choice([16, 24, 48])))
        elif op == "multi":
            b.multi(nseg=int(rng.integers(2, 9)), yaw0=float(rng.uniform(-3, 3)))
        elif op == "move":
            r = rng.uniform()
            if r < 0.1:
                dx, dy = int(rng.choice([-1, 1])) * (L + int(rng.integers(0, 3))), int(rng.integers(-3, 4))
            else:
                dx, dy = (int(v) for v in rng.integers(-7, 8, 2))
            b.move_cells(dx, dy, z=float(rng.uniform(0.5, 2.0)))
            if snap and rng.uniform() < 0.7:
                b.op("harvest")
        elif op == "var_update":
            b.op("var_update", dv=float(rng.choice([-8e-5, -2e-5, 0.0, 1e-3])))
        elif op in ("opt_move", "closeloop"):
            p = (float(b.centre[0] + rng.uniform(-0.3, 0.3)), float(b.centre[1] + rng.uniform(-0.3, 0.3)))
            dh = float(rng.uniform(-0.2, 0.2))
            b.op(op, p=p, dh=dh)
            fn = _opt_move_centre if op == "opt_move" else _closeloop_centre
            b.centre = [f32(c) for c in fn(b.centre, p, b.s.res)]
        elif op == "process":
            b.op("process", cloud=b.new_cloud(scale=0.5), T=np.eye(4))
            b.op("fuse")
        elif op == "empty":
            b.empty(str(rng.choice(EMPTY_VARIANTS)))
        elif op == "snapshot":
            b.op("snapshot")
            snap = True
        else:
            b.op(op)
    return b.done()


@functools.lru_cache(maxsize=1)
def all_scripts():
    return tuple(hand_written() + [random_script(s) for s in SEEDS])


SCRIPT_NAMES = [s.name for s in all_scripts()]


def script_by_name(name):
    for s in all_scripts():
        if s.name == name:
            return s
    raise KeyError(name)


# ---- the oracle's side of a script --------------------------------------------------------------------------------------
def segment_arrays(c):
    return c["xyzi"], c["rgba"]


class OracleRun:
    """executes a script's steps on an OracleMap; every step returns what the device map must reproduce, plus the facts
    the CPU suite checks hazards with (counts per storage cell of an add, the queued bands of a move, ...)"""

    def __init__(self, script: Script):
        self.s = script
        self.o = OracleMap(script.L, script.res, compat_box_filter=False)
        self.proc = None
        self.last_move = None
        self.stats = None
        n = script.L * script.L
        # the outputs of the last feature pass (the device map starts with rough = slope = 0, traversability -10)
        self.feat = {"rough": np.zeros(n, f32), "slope": np.zeros(n, f32), "traver": np.full(n, f32(-10))}
        self.local = submap_oracle.LocalMapDict()
        self.pushed = []                                 # the global map's submaps
        self.cost = {}                                   # window size -> (window, grid) of that costmap layer

    def close(self):
        self.o.close()

    def _process(self, xyzi, rgba, T):
        f = frame(T)
        xyzi, rgba = self.o.clean_point_cloud(xyzi, rgba, f)
        key, var, xt, yt, zt = self.o.process_points(xyzi[:, 0], xyzi[:, 1], xyzi[:, 2], f)
        return xyzi, rgba, key, var, xt, yt, zt

    def _fuse(self, xyzi, rgba, key, var, zt):
        R, G, B = (rgba[:, k].astype(np.int32) for k in range(3))
        self.o.fuse_points(key, R, G, B, xyzi[:, 3], zt, var)

    def _expect_stats(self, n_in, key):
        k = key[key >= 0]
        counts = np.bincount(k, minlength=self.s.L * self.s.L)
        return {"points_in": int(n_in), "points_binned": int(k.size), "cells_touched": int((counts > 0).sum()),
                "max_points_per_cell": int(counts.max()) if k.size else 0}

    def step(self, op, a):
        o, L = self.o, self.s.L
        out = {}
        if op == "move":
            before = o.state()
            ops = move_model(L, self.s.res, before[0], before[1], a["pos"])[3]
            out["band_filled"] = int((o.get_layer("elevation").reshape(-1)[band_cells(L, ops)] != f32(-10)).sum())
            out["returned"] = o.move(a["pos"])
            out["state"] = o.state()
            out["ops"] = ops
            self.last_move = (out["returned"][0], out["returned"][2])
        elif op == "add":
            c = self.s.clouds[a["cloud"]]
            xyzi, rgba, key, var, xt, yt, zt = self._process(c["xyzi"], c["rgba"], a["T"])
            self._fuse(xyzi, rgba, key, var, zt)
            out["keys"] = key
            self.stats = self._expect_stats(c["xyzi"].shape[0], key)
        elif op == "multi":
            low0 = o.get_layer("lowest")
            keys, geos, hs, hvs, n_in = [], [], [], [], 0
            for name, T in zip(a["clouds"], a["Ts"]):
                c = self.s.clouds[name]
                n_in += c["xyzi"].shape[0]
                xyzi, rgba, key, var, xt, yt, zt = self._process(c["xyzi"], c["rgba"], T)
                self._fuse(xyzi, rgba, key, var, zt)
                geo = np.array([o.points_to_index(px, py)[0] if k >= 0 else -1 for px, py, k in zip(xt, yt, key)],
                               np.int64)
                keys.append(key); geos.append(geo); hs.append(zt); hvs.append(var)
            # one call's lowest over all segments (the ORACLE DEFINITION of gpu.cu:432-438 on geographic indices)
            o.set_layer("lowest", np_reference.lowest_update(low0, np.concatenate(geos), np.concatenate(hs),
                                                             np.concatenate(hvs)))
            out["keys"] = np.concatenate(keys)
            out["frames"] = [np.asarray(T) for T in a["Ts"]]
            self.stats = self._expect_stats(n_in, out["keys"])
        elif op == "empty":
            # an add of no points is still a Fuse: the variance floor of gpu.cu:533-534 runs over every cell
            o.fuse_points(np.zeros(0, np.int32), None, None, None, None, np.zeros(0, f32), np.zeros(0, f32))
            self.stats = None
        elif op == "var_update":
            o.var_update(a["dv"])
            out["variance"] = o.get_layer("variance")
        elif op == "set_variance":
            v = o.get_layer("variance")
            out["variance_in"] = v
            nv = set_variance_values(v)
            o.set_layer("variance", nv)
            out["variance"] = nv
        elif op == "opt_move":
            out["aligned"] = o.opt_move(a["p"], a["dh"])
        elif op == "closeloop":
            o.closeloop(a["p"], a["dh"])
        elif op == "process":
            c = self.s.clouds[a["cloud"]]
            xyzi, rgba, key, var, xt, yt, zt = self._process(c["xyzi"], c["rgba"], a["T"])
            self.proc = (xyzi, rgba, key, var, zt)
            out["process"] = (key, var, xt, yt, zt)
            self.stats = None
        elif op == "fuse":
            xyzi, rgba, key, var, zt = self.proc
            self._fuse(xyzi, rgba, key, var, zt)
            self.stats = None
        elif op == "layers":
            out["layers"] = self.layers()
        elif op == "observe":
            out["layers"] = self.layers()
            out.update(self.readouts())
        elif op == "export_ray":
            out["feature"] = self._features()
            out["export"] = o.export_layers()            # what the node reads: taken before the ray clean-up
            o.raytracing()
        elif op == "raytracing":
            o.raytracing()
        elif op == "snapshot":
            out["feature"] = self._features()            # the node snapshots what show() just drew
            o.snapshot_shown()
        elif op == "harvest":
            centre, shift = self.last_move
            out["harvest"] = o.harvest_scrolled_out(centre, shift)
        elif op == "sync":
            out["stats"] = self.stats
        elif op in READERS:
            out["shown"] = self.shown_mask()
            out.update(self.reader(op, a))
        else:
            raise ValueError(op)
        return out

    def layers(self):
        return {n: self.o.get_layer(n) for n in LAYERS}

    # ---- the later readers ----------------------------------------------------------------------------------------------
    def _features(self):
        f = self.o.map_feature()
        self.feat = {k: f[k].copy() for k in ("rough", "slope", "traver")}
        return f

    def shown(self):
        """the shown map as the readers take it: live cells, the last feature pass's rough / slope / traversability"""
        f = {n: self.o.get_layer(n).reshape(-1) for n in ("elevation", "variance", "intensity", "color_r", "color_g", "color_b")}
        f.update(self.feat)
        return f

    def shown_mask(self):
        f = self.shown()
        return (f["elevation"] != f32(-10)) & (f["traver"] != f32(-10)) & ~np.isnan(f["traver"])

    def grid_res(self):
        return float(f32(self.s.res))

    def grid_cloud(self, src):
        if src == "shown":
            centre, start, _ = self.o.state()
            return submap_oracle.grid_cloud(self.shown(), self.s.L, centre, start, self.grid_res())
        f, centre, start = self.o._prev
        return submap_oracle.grid_cloud(f, self.s.L, centre, start, self.grid_res())

    def show(self):
        """orc_show of the shown map: orthomosaic, visual cloud xyz and rgb"""
        f, L = self.shown(), self.s.L
        img = np.empty((L, L, 3), np.uint8)
        xyz = np.empty((L * L, 3), f32)
        rgb = np.empty((L * L, 3), np.uint8)
        cnt = oracle_lib.C.c_int()
        p = oracle_lib._p
        self.o.lib.orc_show(self.o.m, 0.0, p(f["elevation"]), p(f["traver"]), p(f["color_r"]), p(f["color_g"]), p(f["color_b"]),
                            p(img), p(xyz), p(rgb), oracle_lib.C.byref(cnt))
        return img, xyz[:cnt.value].copy(), rgb[:cnt.value].copy()

    def cost_traver(self, src):
        """show()'s traversability [ix, iy], NaN where the cell is not shown, and that grid's centre and start"""
        L = self.s.L
        if src == "shown":
            f = self.shown()
            centre, start, _ = self.o.state()
            t = np.where(self.shown_mask(), f["traver"], f32(np.nan))
        else:
            f, centre, start = self.o._prev
            t = oracle_lib.export_from_feature(f, L)["traver"]
        return np.asarray(t, f32).reshape(L, L), centre, start

    def reader(self, op, a):
        o, L = self.o, self.s.L
        if op == "grid_cloud":
            return {"cloud": self.grid_cloud(a["src"])}
        if op in ("split", "octrees"):
            cloud = self.grid_cloud(a["src"])
            sp = split_oracle.grid_split(cloud)
            out = {"road": sp["road"], "obstacle": sp["obstacle"], "points": int(cloud.shape[0])}
            out.update({k: sp[k] for k in ("valid", "mean", "stddev", "threshold")})
            if op == "octrees":
                out["road_stream"] = octree_oracle.color_octree(sp["road"], 0.2)[0]
                out["obstacle_stream"] = octree_oracle.color_octree(sp["obstacle"], 0.1)[0]
            return out
        if op == "costmap":
            sx, sy = a["size"]
            if a["size"] not in self.cost:
                self.cost[a["size"]] = (initial_window(sx, sy), initial_grid(sx, sy))
            w, grid = self.cost[a["size"]]
            nx, ny = cost_origin(o.state()[0], sx, sy)
            w, grid = costmap_oracle.update_origin(w, nx, ny, COST_FILL, grid)
            t, centre, start = self.cost_traver(a["src"])
            grid, marks = costmap_oracle.mark_map(t, L, self.grid_res(), centre, start, w, grid, COST_THRESH, True)
            self.cost[a["size"]] = (w, grid)
            return {"window": w, "grid": grid, "marks": marks}
        if op == "ros":
            ro = rosmsg_oracle
            h = ro.header(ROS_HEADER["seq"], ROS_HEADER["stamp_sec"], ROS_HEADER["stamp_nsec"], ROS_HEADER["frame_id"].encode())
            img, xyz, rgb = self.show()
            centre, start, _ = o.state()
            layers = oracle_lib.export_from_feature(self.shown(), L)
            return {"ros": {"visual_points": ro.visual_points(h, xyz, rgb),
                            "grid_map": ro.grid_map(h, L, self.grid_res(), float(centre[0]), float(centre[1]), start, layers),
                            "orthomosaic": ro.image(h, L, img.tobytes())}}
        if op == "layer_device":
            out = {n: o.get_layer(n) for n in LAYERS}
            out.update({n: self.feat[k].reshape(L, L) for n, k in (("rough", "rough"), ("slope", "slope"),
                                                                   ("traver_out", "traver"))})
            return {"device_layers": out}
        if op == "local":
            centre, shift = self.last_move
            rec, n = o.harvest_scrolled_out(centre, shift)
            self.local.insert_all(rec)
            return {"local": (rec, n), "local_size": len(self.local)}
        if op == "cut":
            local = self.local.records()
            parts = [local]
            if a["dense"] and local.shape[0]:
                parts.append(mls_oracle.upsample(local, {"seed": CUT_SEED})[0])
            parts.append(self.grid_cloud("shown"))
            cut = np.concatenate(parts)
            self.local.clear()
            self.pushed.append(cut)
            return {"cut": cut, "local_taken": int(local.shape[0]), "global": np.concatenate(self.pushed),
                    "submaps": len(self.pushed)}
        raise ValueError(op)

    def readouts(self):
        o = self.o
        out = {"feature": self._features(), "export": o.export_layers()}
        out["ortho"], out["vis_xyz"], out["vis_rgb"] = o.show()
        return out


LAYERS = ["elevation", "variance", "intensity", "color_r", "color_g", "color_b", "lowest", "traver"]


def set_variance_values(v):
    """the variance layer a set_variance step writes: halved where set, and some set cells pushed below the floor"""
    v = np.asarray(v, np.float32)
    out = np.where(v == f32(-10), v, f32(0.5) * v).astype(np.float32)
    low = (np.arange(v.size).reshape(v.shape) % 7 == 0) & (v != f32(-10))
    out[low] = f32(2e-5)
    return out


def run_oracle(script: Script):
    """all steps on the oracle alone: [(op, args, out)]"""
    r = OracleRun(script)
    try:
        return [(op, a, r.step(op, a)) for op, a in script.steps]
    finally:
        r.close()
