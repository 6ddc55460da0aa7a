"""A costmap_2d grid on the device and LayeredCostmap::updateMap around one layer (DESIGN.md f8).

GEM's navigation stack runs two single-layer costmaps: the local one (ElevationMapLayer, 15 m x 15 m at 0.2 m, combined
into the master with updateWithMax) and the global one (PointMapLayer, 200 m x 200 m at 0.2 m, which overwrites the
master).  Both roll with the robot.  `Costmap` owns one window and its grid; `update` does, on the host, what
LayeredCostmap::updateMap does around the layer, so that a caller does not have to reproduce the grid-aligned origin
drift of the rolling window or the bounds-to-rect arithmetic.  The cell work is the library's
(gem_costmap_* of include/gem_b200.h).

GEM's global costmap also lists costmap_2d's InflationLayer after the point layer; `InflationLayer` holds its parameters
and bounds state, and `Costmap.update(..., inflation=layer)` runs it as LayeredCostmap::updateMap does with the two
plugins (DESIGN.md f14).

What Costmap2DROS publishes, and ObstacleLayer's footprint clearing (DESIGN.md f17): `CostmapPublisher` is
Costmap2DPublisher's decision between a full grid, an update and nothing, with the bytes written on the device;
`Costmap.update(..., robot_yaw=, footprint=)` clears the footprint in the layer grid; `Costmap` keeps LayeredCostmap's
getBounds rect and its initialized flag for the publisher.

The two plugins as move_base runs them, fed from their subscribed messages (DESIGN.md f18): `ElevationMapLayer` takes
the serialised grid_map_msgs/GridMap bytes of visual_map, `PointMapLayer` the PointCloud2 of history_point; either is
passed to `Costmap.update` as its `mark`."""
from __future__ import annotations

import math

import ctypes as C

import numpy as np

from . import _lib
from ._lib import COST_FREE, COST_LETHAL, COST_UNKNOWN  # noqa: F401

FLT_MAX = 3.4028234663852886e38   # std::numeric_limits<float>::max(), as a double

# GEM's robot footprint (move_base's costmap_common_params); its inscribed radius is 0.40 m
GEM_FOOTPRINT = ((-0.64, -0.40), (-0.64, 0.40), (0.64, 0.40), (0.64, -0.40))


def _distance_to_line(px, py, x0, y0, x1, y1):
    """costmap_math's distanceToLine: the distance to the segment, its projection parameter clamped to [0, 1]"""
    a, b, c, d = px - x0, py - y0, x1 - x0, y1 - y0
    dot = a * c + b * d
    len_sq = c * c + d * d
    param = dot / len_sq if len_sq != 0 else math.copysign(math.inf, dot) if dot != 0 else math.nan
    if param < 0:
        xx, yy = x0, y0
    elif param > 1:
        xx, yy = x1, y1
    else:
        xx, yy = x0 + param * c, y0 + param * d
    return math.hypot(px - xx, py - yy)


def inscribed_radius(footprint, padding: float = 0.0) -> float:
    """calculateMinAndMaxDistances' minimum (footprint.cpp) over the footprint padded as padFootprint does (each
    coordinate moved away from 0 by `padding`): the least distance from the origin to a vertex or an edge.  A footprint
    of two points or fewer gives DBL_MAX, as the reference's initial value."""
    sign0 = lambda v: -1.0 if v < 0 else (1.0 if v > 0 else 0.0)   # noqa: E731
    pts = [(float(x) + sign0(float(x)) * padding, float(y) + sign0(float(y)) * padding) for x, y in footprint]
    best = 1.7976931348623157e308
    if len(pts) <= 2:
        return best
    for k in range(len(pts)):
        (x0, y0), (x1, y1) = pts[k], pts[(k + 1) % len(pts)]
        best = min(best, min(math.hypot(x0, y0), _distance_to_line(0.0, 0.0, x0, y0, x1, y1)))
    return best


def transform_footprint(footprint, robot_x: float, robot_y: float, robot_yaw: float):
    """footprint.cpp's transformFootprint: each vertex (fx, fy) at the pose as (x + (fx cos t - fy sin t), y + (fx sin t +
    fy cos t)) in double, cos and sin from the host's libm.  The published footprint (W11) is these as float32."""
    c, s = math.cos(float(robot_yaw)), math.sin(float(robot_yaw))
    return [(float(robot_x) + (float(fx) * c - float(fy) * s), float(robot_y) + (float(fx) * s + float(fy) * c))
            for fx, fy in footprint]


def world_to_map_enforce_bounds(window, wx: float, wy: float):
    """Costmap2D::worldToMapEnforceBounds: below the origin -> 0, at or beyond origin + resolution * size -> size - 1,
    else the truncated quotient"""
    ox, oy, res, sx, sy = window

    def one(w, o, n):
        if w < o:
            return 0
        if w >= res * n + o:
            return n - 1
        return int((w - o) / res)
    return one(wx, ox, sx), one(wy, oy, sy)


def update_rect(window, marks):
    """the rect LayeredCostmap::updateMap resets and hands to updateCosts, from the layer's touch bounds (the bounds start
    at +-1e30): (x0, y0, xn, yn), or None when the reference returns early (xn < x0 or yn < y0)"""
    _, _, _, sx, sy = window
    min_x, min_y = min(1e30, marks["min_x"]), min(1e30, marks["min_y"])
    max_x, max_y = max(-1e30, marks["max_x"]), max(-1e30, marks["max_y"])
    x0, y0 = world_to_map_enforce_bounds(window, min_x, min_y)
    xn, yn = world_to_map_enforce_bounds(window, max_x, max_y)
    x0, y0 = max(0, x0), max(0, y0)
    xn, yn = min(sx, xn + 1), min(sy, yn + 1)
    if xn < x0 or yn < y0:
        return None
    return x0, y0, xn, yn


class Costmap:
    """One costmap_2d grid: a window (origin_x, origin_y, resolution, size_x, size_y), a uint8 CUDA tensor of
    (size_y, size_x) cells filled with `fill` (the grid's default_value_) and the ElevationMap whose stream works on it.
    A master grid of GEM's configs has fill FREE (track_unknown_space false); the elevation layer FREE; the point layer
    NO_INFORMATION."""

    def __init__(self, emap, size_x: int, size_y: int, resolution: float, origin_x: float = 0.0, origin_y: float = 0.0,
                 fill: int = COST_FREE):
        import torch
        self.emap = emap
        self.window = (float(origin_x), float(origin_y), float(resolution), int(size_x), int(size_y))
        self.fill = int(fill)
        dev = torch.device("cuda", emap._device_index())
        self.grid = torch.full((int(size_y), int(size_x)), self.fill, dtype=torch.uint8, device=dev)
        # LayeredCostmap's getBounds rect (bx0, bxn, by0, byn) and initialized_: set by an update that reaches updateCosts;
        # one that returns early leaves them, and a node feeds those stale bounds to the publisher again
        self.bx0 = self.bxn = self.by0 = self.byn = 0
        self.initialized = False

    def size_in_meters(self):
        """Costmap2D::getSizeInMetersX / Y: (size - 1 + 0.5) * resolution"""
        _, _, res, sx, sy = self.window
        return (sx - 1 + 0.5) * res, (sy - 1 + 0.5) * res

    def roll(self, robot_xy):
        """the rolling window: updateOrigin(robot - getSizeInMeters() / 2); the origin moves in whole cells"""
        mx, my = self.size_in_meters()
        self.window = self.emap.costmap_update_origin(self.window, float(robot_xy[0]) - mx / 2, float(robot_xy[1]) - my / 2,
                                                      self.fill, self.grid)

    def mark_map(self, travers_thresh: float = 0.7, source: str = "shown", mark_unknown: bool = True) -> dict:
        """ElevationMapLayer::updateBounds into this grid"""
        return self.emap.costmap_mark_map(self.window, self.grid, travers_thresh, source, mark_unknown)

    def mark_points(self, points, travers_thresh: float = 0.7) -> dict:
        """PointMapLayer::updateBounds into this grid"""
        return self.emap.costmap_mark_points(points, self.window, self.grid, travers_thresh)

    def update(self, layer: "Costmap", robot_xy, mode: str, mark, inflation: "InflationLayer | None" = None,
               robot_yaw: float | None = None, footprint=None):
        """LayeredCostmap::updateMap of this master grid with one layer: roll the master and the layer, let the layer
        mark (`mark(layer)` returns its marks, e.g. lambda l: l.mark_map(0.7)), turn the touch bounds into the rect,
        reset the rect to the master's fill and combine the layer into it ("max" for ElevationMapLayer, "overwrite" for
        PointMapLayer).  With `inflation`, that InflationLayer is the second plugin: its update_bounds follows the
        layer's, and its update_costs follows the combine.  With `footprint` (the padded footprint's vertices) and
        `robot_yaw`, the "max" layer clears it as ObstacleLayer does (DESIGN.md f17): the vertices widen the bounds and
        the footprint's cells become FREE in the layer grid; PointMapLayer ("overwrite") has no footprint clearing, so a
        footprint with it is refused.  Returns (rect or None, marks), the marks with the footprint's bounds merged in."""
        import torch
        if footprint is not None and (mode != "max" or robot_yaw is None):
            raise ValueError("update: footprint clearing needs mode \"max\" (ElevationMapLayer) and robot_yaw")
        self.roll(robot_xy)
        layer.roll(robot_xy)
        marks = mark(layer)
        if footprint is not None:
            fm = self.emap.costmap_footprint(layer.window, footprint, robot_xy[0], robot_xy[1], robot_yaw, layer.grid)
            marks = dict(marks, min_x=min(marks["min_x"], fm["min_x"]), min_y=min(marks["min_y"], fm["min_y"]),
                         max_x=max(marks["max_x"], fm["max_x"]), max_y=max(marks["max_y"], fm["max_y"]))
        if inflation is None:
            rect = update_rect(self.window, marks)
        else:
            b = inflation.update_bounds((min(1e30, marks["min_x"]), min(1e30, marks["min_y"]),
                                         max(-1e30, marks["max_x"]), max(-1e30, marks["max_y"])))
            rect = update_rect(self.window, dict(zip(("min_x", "min_y", "max_x", "max_y"), b)))
        if rect is None:
            return None, marks
        x0, y0, xn, yn = rect
        with torch.cuda.stream(self.emap.torch_stream()):   # resetMap, ordered with the library's calls
            self.grid[y0:yn, x0:xn].fill_(self.fill)
        _, _, _, sx, sy = self.window
        self.emap.costmap_combine(mode, layer.grid, self.grid, sx, sy, rect)
        if inflation is not None:
            inflation.update_costs(self, rect)
        self.bx0, self.bxn, self.by0, self.byn = x0, xn, y0, yn
        self.initialized = True
        return rect, marks


def _host_u8(a):
    """host bytes (bytes, bytearray, memoryview, numpy or a CPU tensor) as a flat uint8 CPU tensor sharing their memory"""
    import torch
    import warnings
    if isinstance(a, torch.Tensor):
        return a.reshape(-1).view(torch.uint8)
    with warnings.catch_warnings():      # read-only bytes: the tensor is only ever read
        warnings.simplefilter("ignore", UserWarning)
        return torch.from_numpy(np.frombuffer(memoryview(a).cast("B"), np.uint8))


NO_MARKS = {"marked": 0, "lethal": 0, "min_x": math.inf, "min_y": math.inf, "max_x": -math.inf, "max_y": -math.inf}


class ElevationMapLayer:
    """ElevationMapLayer (layers/src/elevationMap_layer.cpp) fed from visual_map messages.  `on_message` is
    elevationMapCB with its elevation_map_available_ gate: a message is kept only when none is pending; keeping it is
    gem_grid_map_msg_parse of the bytes and one H2D copy of the `layer` floats alone into a device buffer this object
    owns (on torch's current stream, which the mark waits for).  `update_bounds` (or calling the object, as Costmap.update's `mark`) marks the layer grid
    from the pending message and consumes it; with none pending it marks nothing.  DEFINED: a message the parser refuses
    raises GemError and leaves the layer as it was (the reference sets elevation_map_available_ after a failed
    fromMessage and marks whatever that left, or throws in operator[] when no message ever had the layer).
    travers_thresh defaults to the plugin's 0.5; GEM's yaml sets 0.7."""

    def __init__(self, emap, travers_thresh: float = 0.5, mark_unknown: bool = True, layer: str = "traver"):
        self.emap = emap
        self.travers_thresh = float(travers_thresh)
        self.mark_unknown = bool(mark_unknown)
        self.layer = str(layer)
        self.desc = None           # the pending message's gem_grid_map_layer, None when none is pending
        self._buf = None           # the pending layer's floats (uint8 CUDA tensor, grown on demand)

    @property
    def available(self) -> bool:
        """elevation_map_available_"""
        return self.desc is not None

    def on_message(self, msg) -> bool:
        """elevationMapCB on the serialised message (bytes, numpy or a CPU tensor, pinned or pageable); returns whether
        it was kept"""
        import torch
        from .elevation_map import ElevationMap
        if self.desc is not None:
            return False
        g = ElevationMap.grid_map_msg_parse(msg, self.layer)
        src = _host_u8(msg)
        nb = 4 * int(g.floats)
        dev = torch.device("cuda", self.emap._device_index())
        if self._buf is None or self._buf.numel() < nb:
            self.emap.sync()       # the previous buffer may still be read on the map's stream
            self._buf = torch.empty(max(nb, 4), dtype=torch.uint8, device=dev)
        # the copy runs on torch's current stream, which costmap_mark_grid synchronises before it marks.  Not on the
        # map's stream: torch ties a pinned source block to the stream of its copy and records an event there when the
        # block is freed, which must not outlive the stream (the map's is destroyed with the map)
        self._buf[:nb].copy_(src[g.offset:g.offset + nb], non_blocking=src.is_pinned())
        self.desc = g
        return True

    def update_bounds(self, layer_costmap: "Costmap") -> dict:
        """updateBounds into the layer grid: the marks (NO_MARKS when no message is pending)"""
        if self.desc is None:
            return dict(NO_MARKS)
        g, self.desc = self.desc, None
        if layer_costmap.emap is not self.emap:
            self.emap.sync()       # the copy ran on this layer's handle, the mark runs on the costmap's
        return layer_costmap.emap.costmap_mark_grid(g, self._buf, layer_costmap.window, layer_costmap.grid,
                                                    self.travers_thresh, self.mark_unknown)

    __call__ = update_bounds


class PointMapLayer:
    """PointMapLayer (layers/src/pointMap_layer.cpp) fed from history_point messages.  `on_message(layout, data)` is
    pointMapCB: the cloud replaces the stored one (ob_pointCloud = *pointCloud), decoded on the device into whole
    PointXYZRGBICT records in a buffer this object owns and grows.  `update_bounds` (or calling the object) re-marks the
    stored cloud every time, as the reference does; before any message it marks nothing.  DEFINED: the reference races
    the callback against updateBounds; here calls take effect in call order.  travers_thresh defaults to the plugin's
    0.5; GEM's yaml sets 0.7."""

    def __init__(self, emap, travers_thresh: float = 0.5):
        self.emap = emap
        self.travers_thresh = float(travers_thresh)
        self.n = None              # points of the stored cloud, None before any message
        self._buf = None           # (capacity, 8) float32 CUDA tensor

    @property
    def points(self):
        """the stored cloud's records, an (n, 8) float32 CUDA tensor view (None before any message)"""
        return None if self.n is None else self._buf[:self.n]

    def on_message(self, layout, data, data_bytes: int | None = None):
        """pointMapCB on a PointCloud2 of `layout` (an elevation_map.PointCloud2Layout) whose bytes are `data`: a CUDA
        tensor, or host memory (bytes, numpy or a CPU tensor) that is copied to the device first.  A layout the library
        refuses raises GemError before anything changes: the stored cloud stays as it was (DEFINED, as for
        ElevationMapLayer)."""
        import torch
        from .elevation_map import ElevationMap
        dev = torch.device("cuda", self.emap._device_index())
        if isinstance(data, torch.Tensor) and data.is_cuda:
            nb = int(data.numel() * data.element_size()) if data_bytes is None else int(data_bytes)
            ElevationMap.pointcloud2_mapping(layout, nb)           # validates the layout first (raises GemError)
        else:
            host = _host_u8(data)
            nb = host.numel() if data_bytes is None else int(data_bytes)
            ElevationMap.pointcloud2_mapping(layout, nb)
            data = host.to(dev)
            # the decode reads this staging copy on the map's stream after on_message returns: the caching allocator
            # must not hand its memory out before that work is done
            data.record_stream(self.emap.torch_stream())
        n = layout.points
        if self._buf is None or self._buf.shape[0] < n:
            self.emap.sync()       # the previous buffer may still be read on the map's stream
            self._buf = torch.empty((max(n + n // 4, 1024), 8), dtype=torch.float32, device=dev)
        self.emap.decode_pointcloud2_records(layout, data, out=self._buf, data_bytes=nb)
        self.n = n

    def update_bounds(self, layer_costmap: "Costmap") -> dict:
        """updateBounds into the layer grid: the marks (NO_MARKS before any message)"""
        if self.n is None:
            return dict(NO_MARKS)
        if layer_costmap.emap is not self.emap:
            self.emap.sync()       # the decode ran on this layer's handle, the mark runs on the costmap's
        return layer_costmap.mark_points(self._buf[:self.n], self.travers_thresh)

    __call__ = update_bounds


class CostmapPublisher:
    """Costmap2DPublisher (navigation 1.14; DESIGN.md f17 P1-P4) of one costmap: the saved window and the accumulated
    bounds in a gem_costmap_publisher, the decision and the message bytes in the library.  The subscriber gate and the
    publish timer stay with the caller: skipping `publish` is what the reference does without subscribers."""

    def __init__(self, always_send_full: bool = False):
        self.state = _lib.GemCostmapPublisher()
        _lib.load().gem_costmap_publisher_init(C.byref(self.state), 1 if always_send_full else 0)

    def bounds(self, x0: int, xn: int, y0: int, yn: int):
        """Costmap2DPublisher::updateBounds: the rect merged into the accumulated bounds with min / max"""
        _lib.load().gem_costmap_publisher_bounds(C.byref(self.state), int(x0), int(xn), int(y0), int(yn))

    def update_bounds(self, costmap: Costmap):
        """what Costmap2DROS::mapUpdateLoop feeds after every update: getBounds, once the costmap is initialised"""
        if costmap.initialized:
            self.bounds(costmap.bx0, costmap.bxn, costmap.by0, costmap.byn)

    def publish(self, master: Costmap, header, out=None, force_full: bool = False):
        """publishCostmap of the master grid (force_full: onNewSubscription's full grid, which leaves the bounds):
        (kind, message) with kind "full", "update" or "none"; see ElevationMap.ros_costmap"""
        return master.emap.ros_costmap(header, master.window, master.grid, self.state, force_full, out)


class InflationLayer:
    """costmap_2d's InflationLayer (navigation 1.14): its parameters, need_reinflation and the last bounds.  Defaults are
    costmap_2d's (0.55 m, factor 10); inscribed_radius is inscribed_radius(footprint) of the robot's footprint."""

    def __init__(self, inflation_radius: float = 0.55, cost_scaling_factor: float = 10.0, inscribed_radius: float = 0.0,
                 inflate_unknown: bool = False):
        self.params = {}
        self.need_reinflation = True
        self.last = None
        self.set_parameters(inflation_radius, cost_scaling_factor, inscribed_radius, inflate_unknown)

    def set_parameters(self, inflation_radius: float, cost_scaling_factor: float, inscribed_radius: float,
                       inflate_unknown: bool = False):
        """a changed value makes the next update re-inflate the whole grid"""
        p = {"inflation_radius": float(inflation_radius), "cost_scaling_factor": float(cost_scaling_factor),
             "inscribed_radius": float(inscribed_radius), "inflate_unknown": bool(inflate_unknown)}
        if p != self.params:
            self.need_reinflation = True
        self.params = p

    def update_bounds(self, bounds):
        """InflationLayer::updateBounds on (min_x, min_y, max_x, max_y): after a (re)configuration the bounds become the
        float range, the whole grid; otherwise they are widened by the radius over the union with the last ones"""
        last, self.last = self.last, tuple(float(v) for v in bounds)
        if self.need_reinflation:
            self.need_reinflation = False
            return (-FLT_MAX, -FLT_MAX, FLT_MAX, FLT_MAX)
        r = self.params["inflation_radius"]
        return (min(last[0], bounds[0]) - r, min(last[1], bounds[1]) - r, max(last[2], bounds[2]) + r,
                max(last[3], bounds[3]) + r)

    def update_costs(self, master: Costmap, rect):
        """InflationLayer::updateCosts of the master grid over rect = (min_i, min_j, max_i, max_j), on the device"""
        master.emap.costmap_inflate(master.window, self.params, master.grid, rect)
