// pcd_fmt_host.cpp -- the host build of the library's float formatter (gem_b200/csrc/gem_pcdfmt.h) and its comparison
// with glibc's snprintf("%.8g"), for tests/test_pcd_cpu.py, tests/test_pcd_gpu.py and scripts/pcd_float_exhaustive.py.
// TEST INFRASTRUCTURE ONLY: compiled by tests/pcd_oracle.py into a temporary directory.
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "gem_pcdfmt.h"

extern "C" {

// one value as the formatter prints it: float (uint32 = 0) or unsigned decimal (uint32 = 1); returns the length
int pcd_fmt_one(uint32_t bits, int uint32, char *out)
{
    return gem_pcd_put(uint32 ? gem_pcd_uint(bits) : gem_pcd_float(bits), out);
}

// what PCL's writer prints for one float: "nan" for any NaN, else %.8g of the value as a double
static int ref_one(uint32_t bits, char *out)
{
    float f;
    memcpy(&f, &bits, 4);
    if (isnan(f)) return snprintf(out, 32, "nan");
    return snprintf(out, 32, "%.8g", (double)f);
}

static int differs(uint32_t bits, int uint32)
{
    char a[32], b[32];
    const int na = pcd_fmt_one(bits, uint32, a), nb = uint32 ? snprintf(b, sizeof b, "%u", bits) : ref_one(bits, b);
    if (na > GEM_PCD_VALUE_MAX || na != nb) return 1;
    if (na != gem_pcd_len(uint32 ? gem_pcd_uint(bits) : gem_pcd_float(bits))) return 1;
    return memcmp(a, b, (size_t)na) != 0;
}

// the bit patterns in [lo, hi) whose formatting differs from snprintf: returns their number, the first in *first_bad
long long pcd_fmt_compare_range(uint64_t lo, uint64_t hi, uint32_t *first_bad)
{
    long long bad = 0;
    for (uint64_t b = lo; b < hi; b++)
        if (differs((uint32_t)b, 0)) {
            if (!bad) *first_bad = (uint32_t)b;
            bad++;
        }
    return bad;
}

// the same over a list of patterns, printed as floats (uint32 = 0) or as unsigned decimals against "%u" (uint32 = 1)
long long pcd_fmt_compare_list(const uint32_t *bits, long long n, int uint32, uint32_t *first_bad)
{
    long long bad = 0;
    for (long long i = 0; i < n; i++)
        if (differs(bits[i], uint32)) {
            if (!bad) *first_bad = bits[i];
            bad++;
        }
    return bad;
}

// the ASCII data section of n PointXYZRGBICT records built from the formatter, line by line as gem_pcd_format defines
// it (fields x y z rgb intensity covariance travers, one space between, '\n' after); returns the bytes written
long long pcd_fmt_ascii(const uint32_t *rec, long long n, int rgb_uint32, char *out)
{
    static const int word[7] = {0, 1, 2, 4, 6, 5, 7};
    long long o = 0;
    for (long long i = 0; i < n; i++) {
        for (int f = 0; f < 7; f++) {
            const uint32_t b = rec[8 * i + word[f]];
            o += gem_pcd_put(f == 3 && rgb_uint32 ? gem_pcd_uint(b) : gem_pcd_float(b), out + o);
            out[o++] = f == 6 ? '\n' : ' ';
        }
    }
    return o;
}

} // extern "C"
