// gem_footprint.h -- ObstacleLayer's footprint clearing (DESIGN.md f17 F1-F4) and Costmap2DROS's published footprint
// (W11's points): the robot's footprint at its pose, worldToMap, and costmap_2d's setConvexPolygonCost cell list
// (polygonOutlineCells, raytraceLine / bresenham2D, convexFillCells), restated literally from navigation 1.14 (unpinned),
// quirks included.  Host code (tens to hundreds of cells); the library and tests/costmap_pub_host.cpp (built by the CPU
// suite with g++) compile the same definitions.  worldToMap is also the device's (gem_costmap.cuh).
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include <vector>

#ifdef __CUDACC__
#define GEM_FP __host__ __device__ __forceinline__
#else
#define GEM_FP inline
#endif

namespace gem_fp {

// f8 item 4, Costmap2D::worldToMap in double: false if wx < origin_x || wy < origin_y; otherwise mx = (int)((wx -
// origin_x) / res) (same for my), accepted iff mx < size_x && my < size_y.  DEFINED: a non-finite coordinate is
// rejected, and so is a quotient >= 2^31, where the reference's cast is undefined.  (NaN fails `>=`; -inf is below the
// origin; +inf gives an infinite quotient.)
GEM_FP bool world_to_map(double ox, double oy, double res, int sx, int sy, double wx, double wy, int &mx, int &my)
{
    if (!(wx >= ox) || !(wy >= oy)) return false;
    const double qx = (wx - ox) / res, qy = (wy - oy) / res;
    if (!(qx < 2147483648.0) || !(qy < 2147483648.0)) return false;
    mx = (int)qx;
    my = (int)qy;
    return mx < sx && my < sy;
}

struct Point {
    double x, y;
};
struct Cell { // costmap_2d's MapLocation
    unsigned x, y;
};

// footprint.cpp's transformFootprint: x + (fx cos t - fy sin t), y + (fx sin t + fy cos t) in double, cos and sin from
// the host's libm (DEFINED).  W11 stores each as float; ObstacleLayer keeps the doubles.
inline void transform(const double *spec_xy, int n, double rx, double ry, double yaw, std::vector<Point> &out)
{
    out.clear();
    const double c = cos(yaw), s = sin(yaw);
    for (int i = 0; i < n; i++) {
        const double fx = spec_xy[2 * i], fy = spec_xy[2 * i + 1];
        out.push_back(Point{rx + (fx * c - fy * s), ry + (fx * s + fy * c)});
    }
}

// costmap_2d's sign(): -1 for 0 (never applied to a zero step: bresenham2D's error term never reaches abs_da then)
inline int sign(int x) { return x > 0 ? 1 : -1; }

// F3 Costmap2D::raytraceLine with max_length UINT_MAX (scale 1) into PolygonOutlineCells: bresenham2D visits
// abs_da cells and then the end cell, each offset turned back into (mx, my) by indexToCells
inline void raytrace(unsigned sx, unsigned x0, unsigned y0, unsigned x1, unsigned y1, std::vector<Cell> &cells)
{
    const int dx = (int)(x1 - x0), dy = (int)(y1 - y0);
    const unsigned abs_dx = (unsigned)abs(dx), abs_dy = (unsigned)abs(dy);
    const int offset_dx = sign(dx), offset_dy = sign(dy) * (int)sx;
    unsigned offset = y0 * sx + x0;
    unsigned abs_da, abs_db;
    int error_b, offset_a, offset_b;
    if (abs_dx >= abs_dy) {
        abs_da = abs_dx; abs_db = abs_dy; error_b = (int)(abs_dx / 2); offset_a = offset_dx; offset_b = offset_dy;
    } else {
        abs_da = abs_dy; abs_db = abs_dx; error_b = (int)(abs_dy / 2); offset_a = offset_dy; offset_b = offset_dx;
    }
    auto at = [&](unsigned off) { cells.push_back(Cell{off - (off / sx) * sx, off / sx}); };
    for (unsigned i = 0; i < abs_da; ++i) {
        at(offset);
        offset += (unsigned)offset_a;
        error_b += (int)abs_db;
        if ((unsigned)error_b >= abs_da) {
            offset += (unsigned)offset_b;
            error_b -= (int)abs_da;
        }
    }
    at(offset);
}

// F4 convexFillCells after the outline, literally: the adjacent-swap sort by x, then the column walk that pairs cells
// i, i + 1 and appends each column's inner cells to the list it walks.  A column of one cell would pair it with the next
// column's first; through F3's outline that cannot happen (the closed outline crosses every column between its ends twice,
// so each holds two cells or more), but the walk is kept as the reference's for any list.
inline void column_walk(std::vector<Cell> &cells)
{
    if (cells.empty()) return;
    size_t i = 0;
    while (i < cells.size() - 1) {
        if (cells[i].x > cells[i + 1].x) {
            const Cell t = cells[i];
            cells[i] = cells[i + 1];
            cells[i + 1] = t;
            if (i > 0) --i;
        } else {
            ++i;
        }
    }
    i = 0;
    Cell min_pt{0, 0}, max_pt{0, 0};
    const unsigned min_x = cells[0].x, max_x = cells[cells.size() - 1].x;
    for (unsigned x = min_x; x <= max_x; ++x) {
        if (i >= cells.size() - 1) break;
        if (cells[i].y < cells[i + 1].y) {
            min_pt = cells[i];
            max_pt = cells[i + 1];
        } else {
            min_pt = cells[i + 1];
            max_pt = cells[i];
        }
        i += 2;
        while (i < cells.size() && cells[i].x == x) {
            if (cells[i].y < min_pt.y) min_pt = cells[i];
            else if (cells[i].y > max_pt.y) max_pt = cells[i];
            ++i;
        }
        for (unsigned y = min_pt.y; y < max_pt.y; ++y) cells.push_back(Cell{x, y});
    }
}

// F2-F4 Costmap2D::convexFillCells: nothing below 3 vertices, else polygonOutlineCells and the column walk
inline void convex_fill(unsigned sx, const std::vector<Cell> &polygon, std::vector<Cell> &cells)
{
    if (polygon.size() < 3) return;
    for (size_t i = 0; i + 1 < polygon.size(); ++i) raytrace(sx, polygon[i].x, polygon[i].y, polygon[i + 1].x, polygon[i + 1].y, cells);
    raytrace(sx, polygon.back().x, polygon.back().y, polygon[0].x, polygon[0].y, cells);
    column_walk(cells);
}

// F1 Costmap2D::setConvexPolygonCost's cells: every vertex through worldToMap, one outside fills nothing (false)
inline bool polygon_cells(double ox, double oy, double res, int sx, int sy, const std::vector<Point> &poly, std::vector<Cell> &cells)
{
    cells.clear();
    std::vector<Cell> map_polygon;
    for (const Point &p : poly) {
        int mx, my;
        if (!world_to_map(ox, oy, res, sx, sy, p.x, p.y, mx, my)) return false;
        map_polygon.push_back(Cell{(unsigned)mx, (unsigned)my});
    }
    convex_fill((unsigned)sx, map_polygon, cells);
    return true;
}

} // namespace gem_fp
