"""A costmap_2d grid on the device and LayeredCostmap::updateMap around one layer (DESIGN.md f8).

GEM's navigation stack runs two single-layer costmaps: the local one (ElevationMapLayer, 15 m x 15 m at 0.2 m, combined
into the master with updateWithMax) and the global one (PointMapLayer, 200 m x 200 m at 0.2 m, which overwrites the
master).  Both roll with the robot.  `Costmap` owns one window and its grid; `update` does, on the host, what
LayeredCostmap::updateMap does around the layer, so that a caller does not have to reproduce the grid-aligned origin
drift of the rolling window or the bounds-to-rect arithmetic.  The cell work is the library's
(gem_costmap_* of include/gem_b200.h)."""
from __future__ import annotations

from ._lib import COST_FREE, COST_LETHAL, COST_UNKNOWN  # noqa: F401


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

    def update(self, layer: "Costmap", robot_xy, mode: str, mark):
        """LayeredCostmap::updateMap of this master grid with one layer: roll the master and the layer, let the layer
        mark (`mark(layer)` returns its marks, e.g. lambda l: l.mark_map(0.7)), turn the touch bounds into the rect,
        reset the rect to the master's fill and combine the layer into it ("max" for ElevationMapLayer, "overwrite" for
        PointMapLayer).  Returns (rect or None, marks)."""
        import torch
        self.roll(robot_xy)
        layer.roll(robot_xy)
        marks = mark(layer)
        rect = update_rect(self.window, marks)
        if rect is None:
            return None, marks
        x0, y0, xn, yn = rect
        with torch.cuda.stream(self.emap.torch_stream()):   # resetMap, ordered with the library's calls
            self.grid[y0:yn, x0:xn].fill_(self.fill)
        _, _, _, sx, sy = self.window
        self.emap.costmap_combine(mode, layer.grid, self.grid, sx, sy, rect)
        return rect, marks
