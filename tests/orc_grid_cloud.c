/* orc_grid_cloud.c -- CPU oracle of gem_export_grid_cloud: ElevationMapping::gridMaptoPointCloud
 * (ElevationMapping.cpp:1198-1226).  TEST INFRASTRUCTURE ONLY: compiled by tests/submap_oracle.py next to the pinned
 * oracle library (oracle/gem_oracle.c), which it leaves untouched.  Same conventions as orc_harvest there
 * (-ffp-contract=off, GridMapIterator order, grid_map positions).
 *
 * PARITY UNPINNED (grid_map): the input grid is a visualMap_, i.e. Map_feature's outputs as show() writes them
 * (ElevationMap.cpp:101-111: the cell's values where show() takes it, NaN everywhere else) with the centre / start index
 * of that frame.  Cell-centre positions restate grid_map's getPositionFromIndex as orc_show does (ORACLE DEFINITION).
 * w = 1 and a = 255 are defined here; the reference leaves them uninitialised (`Anypoint point;` at :1200). */
#include <math.h>
#include <string.h>

void orc_grid_cloud(int L, double grid_res, const float centre[2], const int start[2], const float *elevation,
                    const float *variance, const float *traver, const int *R, const int *G, const int *B,
                    const float *intensity, float *out, int *count)
{
    const double res = grid_res, half = 0.5 * ((double)L * res) - 0.5 * res;
    const float nan = (float)NAN;
    int n = 0, i;
    for (i = 0; i < L * L; i++) {
        const int ix = i % L, iy = i / L, index = ix * L + iy;
        /* visualMap_ after show(): ElevationMap.cpp:101 decides, cleared cells are NaN in every layer */
        const int shown = elevation[index] != -10 && traver[index] != -10 && !isnan(traver[index]);
        const float e = shown ? elevation[index] : nan, t = shown ? traver[index] : nan;
        /* :1208.  Not the harvest's traver >= 0 (:725): negative traversabilities other than -10 are taken. */
        if (e != -10 && t != -10 && !isnan(t)) {
            if (out) {
                float *o = out + 8 * (size_t)n;
                const unsigned r = (unsigned char)(float)R[index], g = (unsigned char)(float)G[index],
                               b = (unsigned char)(float)B[index];
                const unsigned bgra = b | (g << 8) | (r << 16) | 0xff000000u;
                o[0] = (float)((double)centre[0] + half - res * (double)((ix + L - start[0]) % L));
                o[1] = (float)((double)centre[1] + half - res * (double)((iy + L - start[1]) % L));
                o[2] = e; o[3] = 1.0f;
                memcpy(&o[4], &bgra, 4);
                o[5] = variance[index]; o[6] = intensity[index]; o[7] = t;
            }
            n++;
        }
    }
    if (count) *count = n;
}
