// gem_globalmap.h -- the host half of updateGlobalMap (ElevationMapping.cpp:773-905; DESIGN.md f16): the pose arithmetic
// of :800 and the pair schedule of :812-891.  Host code only, compiled by nvcc's host compiler into the library and by
// g++ into the CPU tests, both without FMA contraction (-ffp-contract=off), so the two builds agree bit for bit.
#pragma once
#include <algorithm>
#include <utility>
#include <vector>

namespace gem_gmap {

// a 3-term dot product, left to right in float: (a0 b0 + a1 b1) + a2 b2
inline float dot3(float a0, float a1, float a2, float b0, float b1, float b2) { return (a0 * b0 + a1 * b1) + a2 * b2; }

// T = P_new * P_old^-1 (:800, optGlobalMapLoc_[i] * trajectory_[i].inverse()) the way Eigen's Isometry3f evaluates it
// (DEFINED, unpinned: Eigen is not available): inverse = (R^T, -(R^T t)), product = (R_n R_o^T, R_n t_inv + t_n).  Poses are
// row-major 4 x 4 floats whose row 3 is ignored; T's row 3 is written as 0 0 0 1.
inline void relative_pose(const float *pn, const float *po, float *T)
{
    float ri[3][3], ti[3];
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) ri[r][c] = po[4 * c + r];
    for (int r = 0; r < 3; r++) ti[r] = -dot3(ri[r][0], ri[r][1], ri[r][2], po[3], po[7], po[11]);
    for (int r = 0; r < 3; r++) {
        const float *n = pn + 4 * r;
        for (int c = 0; c < 3; c++) T[4 * r + c] = dot3(n[0], n[1], n[2], ri[0][c], ri[1][c], ri[2][c]);
        T[4 * r + 3] = dot3(n[0], n[1], n[2], ti[0], ti[1], ti[2]) + n[3];
    }
    T[12] = T[13] = T[14] = 0.0f;
    T[15] = 1.0f;
}

// KdTreeFLANN::radiusSearch over the first K centres (x, y pairs) around centre i (:816-838): the indices whose squared
// float distance (dx dx + dy dy) is <= (float)radius * (float)radius, nearest first, ties by index (DEFINED: FLANN's tie
// order is unspecified).  A NaN centre is within no distance of anything, itself included, so it has no neighbours (the
// reference reads pointIdx[0] out of bounds there).
inline void neighbours(const float *centres, int K, int i, double radius, std::vector<int> &out)
{
    const float rr = (float)radius * (float)radius;
    std::vector<std::pair<float, int>> d;
    for (int j = 0; j < K; j++) {
        const float dx = centres[2 * j] - centres[2 * i], dy = centres[2 * j + 1] - centres[2 * i + 1];
        const float d2 = dx * dx + dy * dy;
        if (d2 <= rr) d.push_back(std::make_pair(d2, j));
    }
    std::sort(d.begin(), d.end());
    out.clear();
    for (const auto &e : d) out.push_back(e.second);
}

// the re-fusion pairs (new = neighbour j, old = submap i) in the order :812-891 runs them: for every i < K with more than
// two results, every result after the first, i itself skipped (DEFINED: a tie can put i after the first result)
inline void pair_schedule(const float *centres, int K, double radius, std::vector<std::pair<int, int>> &pairs)
{
    pairs.clear();
    std::vector<int> nb;
    for (int i = 0; i < K; i++) {
        neighbours(centres, K, i, radius, nb);
        if (nb.size() <= 2) continue;
        for (size_t q = 1; q < nb.size(); q++)
            if (nb[q] != i) pairs.push_back(std::make_pair(nb[q], i));
    }
}

} // namespace gem_gmap
