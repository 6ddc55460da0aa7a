// gridmsg_host.cpp -- the host build of the library's grid_map_msgs/GridMap reader (gem_b200/csrc/gem_gridmsg.h, G1-G3)
// for tests/test_costmap_ingest_cpu.py.
// TEST INFRASTRUCTURE ONLY: compiled by tests/gridmsg_oracle.py into a temporary directory.
#include <stddef.h>

#include "gem_gridmsg.h"

extern "C" {

// 0 and *out filled, or 1 (refused) with *out untouched
int gm_parse(const void *msg, unsigned long long bytes, const char *layer, gem_grid_map_layer *out)
{
    return gem_gridmsg::parse(msg, bytes, layer, out) ? 1 : 0;
}

int gm_layer_ok(const gem_grid_map_layer *g) { return gem_gridmsg::layer_ok(*g) ? 1 : 0; }

// sizeof(gem_grid_map_layer), then the offset of each field in declaration order
void gm_layout(long long *out)
{
    const long long v[] = {(long long)sizeof(gem_grid_map_layer), (long long)offsetof(gem_grid_map_layer, resolution),
                           (long long)offsetof(gem_grid_map_layer, position_x), (long long)offsetof(gem_grid_map_layer, position_y),
                           (long long)offsetof(gem_grid_map_layer, length_x), (long long)offsetof(gem_grid_map_layer, length_y),
                           (long long)offsetof(gem_grid_map_layer, size_x), (long long)offsetof(gem_grid_map_layer, size_y),
                           (long long)offsetof(gem_grid_map_layer, start_x), (long long)offsetof(gem_grid_map_layer, start_y),
                           (long long)offsetof(gem_grid_map_layer, offset), (long long)offsetof(gem_grid_map_layer, floats),
                           (long long)offsetof(gem_grid_map_layer, column_major)};
    for (size_t k = 0; k < sizeof v / sizeof v[0]; k++) out[k] = v[k];
}

} // extern "C"
