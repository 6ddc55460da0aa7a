// The device-side decision of a VoxelGrid step (gem_voxgrid.h, the arithmetic k_vox_decide runs) built by the host
// compiler, for tests/test_prefilter_cpu.py.
#include "gem_voxgrid.h"

extern "C" int voxgrid_layout(const float *mn, const float *mx, const float *inv, double *minb, unsigned long long *radix)
{
    return gem_vox_layout(mn, mx, inv, minb, &radix[0], &radix[1], &radix[2]);
}
