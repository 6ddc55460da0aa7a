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
getBounds rect and its initialized flag for the publisher."""
from __future__ import annotations

import math

import ctypes as C

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
