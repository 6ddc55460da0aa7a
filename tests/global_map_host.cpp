// The host half of gem_global_map_update (gem_globalmap.h) as a C ABI for the CPU tests.  TEST INFRASTRUCTURE ONLY.
#include "gem_globalmap.h"

extern "C" {
void gm_relative_pose(const float *pn, const float *po, float *T) { gem_gmap::relative_pose(pn, po, T); }
// the pair schedule of K centres as (j, i) int pairs; returns the number of pairs (written up to cap)
int gm_pair_schedule(const float *centres, int K, double radius, int *out, int cap)
{
    std::vector<std::pair<int, int>> pairs;
    gem_gmap::pair_schedule(centres, K, radius, pairs);
    for (int q = 0; q < (int)pairs.size() && q < cap; q++) { out[2 * q] = pairs[q].first; out[2 * q + 1] = pairs[q].second; }
    return (int)pairs.size();
}
}
