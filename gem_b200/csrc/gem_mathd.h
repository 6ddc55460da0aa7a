/* gem_mathd.h -- exp, atan2 and sincos in double, built only from + - * / floor and exact power-of-two scaling, in a
 * form that both nvcc (device and host) and a C compiler accept.  The MLS kernels (gem_mls.cuh) and their C oracle
 * (tests/orc_mls.c) include this one source, so that both evaluate these functions bit for bit alike.  Both sides are
 * compiled without FMA contraction (-fmad=false, -ffp-contract=off).
 *
 * gem_atan2_d and gem_sincos_d are the definitions of gem_math.cuh's detail::atan2_d / sincos_d, term for term; those
 * stay where they are so that the code of the existing kernels does not move.  gem_exp_d is new: k = floor(x log2(e) +
 * 1/2), r = (x - k ln2_hi) - k ln2_lo (|r| <= 0.35, ln2_hi has 11 trailing zero bits so k ln2_hi is exact), the Taylor
 * series of e^r through r^13 in Horner form, then the exact scaling by 2^k (in two steps near the ends of the range, so
 * that a subnormal result is rounded once).  Over [-745, 709] it lies within 2 ulp of glibc's exp (tests/test_mls_cpu.py
 * measures it); NaN gives NaN, x > 709.79 gives +inf, x < -745.2 gives +0. */
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define GEM_MD static __host__ __device__ __forceinline__
#else
#define GEM_MD static inline
#endif

GEM_MD double gem_sin_k(double r)
{
    const double r2 = r * r;
    double p = -2.81145725434552076320e-15;
    p = p * r2 + 7.64716373181981647590e-13;
    p = p * r2 + -1.60590438368216145994e-10;
    p = p * r2 + 2.50521083854417187751e-08;
    p = p * r2 + -2.75573192239858906526e-06;
    p = p * r2 + 1.98412698412698412698e-04;
    p = p * r2 + -8.33333333333333333333e-03;
    p = p * r2 + 1.66666666666666666667e-01;
    return r - (r * r2) * p;
}
GEM_MD double gem_cos_k(double r)
{
    const double r2 = r * r;
    double p = -1.56192069685862264622e-16;
    p = p * r2 + 4.77947733238738529744e-14;
    p = p * r2 + -1.14707455977297247139e-11;
    p = p * r2 + 2.08767569878680989792e-09;
    p = p * r2 + -2.75573192239858906526e-07;
    p = p * r2 + 2.48015873015873015873e-05;
    p = p * r2 + -1.38888888888888888889e-03;
    p = p * r2 + 4.16666666666666666667e-02;
    p = p * r2 + -0.5;
    return 1.0 + r2 * p;
}
GEM_MD void gem_sincos_d(double x, double *s, double *c)
{
    if (!(x == x) || x - x != 0.0) {
        *s = x - x;
        *c = x - x;
        return;
    }
    const double kd = floor(x * 0.63661977236758134308 + 0.5);
    const double r = (x - kd * 1.57079632673412561417e+00) - kd * 6.07710050650619224932e-11;
    const long long k = (long long)kd;
    const double sr = gem_sin_k(r), cr = gem_cos_k(r);
    switch (k & 3) {
    case 0: *s = sr; *c = cr; break;
    case 1: *s = cr; *c = -sr; break;
    case 2: *s = -sr; *c = -cr; break;
    default: *s = -cr; *c = sr; break;
    }
}
GEM_MD double gem_atan_poly(double t)
{
    /* odd Maclaurin series through t^43, Horner in t^2; the coefficients 1/n are correctly rounded quotients */
    const double t2 = t * t;
    double p = 0.0;
    for (int n = 43; n >= 3; n -= 2) {
        double coef = 1.0 / (double)n;
        if (((n - 1) / 2) & 1) coef = -coef;
        p = (p + coef) * t2;
    }
    return t + t * p;
}
GEM_MD double gem_atan_core(double z)
{
    if (z > 0.41421356237309503) {
        const double t = (z - 1.0) / (z + 1.0);
        return 0.78539816339744830962 + gem_atan_poly(t);
    }
    return gem_atan_poly(z);
}
GEM_MD double gem_atan2_d(double y, double x)
{
    if (y != y || x != x) return y + x;
    const double ax = fabs(x), ay = fabs(y);
    double a;
    if (ax == 0.0 && ay == 0.0)
        a = 0.0;
    else if (ay <= ax)
        a = gem_atan_core(ay / ax);
    else
        a = 1.57079632679489661923 - gem_atan_core(ax / ay);
    if (x < 0.0) a = 3.14159265358979323846 - a;
    if (y < 0.0) a = -a;
    return a;
}

/* 2^k for -1022 <= k <= 1023, exactly */
GEM_MD double gem_pow2_d(int k)
{
    const uint64_t b = (uint64_t)(k + 1023) << 52;
    double d;
    memcpy(&d, &b, sizeof d);
    return d;
}
GEM_MD double gem_exp_d(double x)
{
    if (x != x) return x + x;
    if (x > 709.79) return 1.0 / 0.0;
    if (x < -745.2) return 0.0;
    const double kd = floor(x * 1.44269504088896338700e+00 + 0.5);
    const double r = (x - kd * 6.93147180369123816490e-01) - kd * 1.90821492927058770002e-10;
    double p = 1.0 / 6227020800.0; /* 1/13! */
    p = p * r + 1.0 / 479001600.0;
    p = p * r + 1.0 / 39916800.0;
    p = p * r + 1.0 / 3628800.0;
    p = p * r + 1.0 / 362880.0;
    p = p * r + 1.0 / 40320.0;
    p = p * r + 1.0 / 5040.0;
    p = p * r + 1.0 / 720.0;
    p = p * r + 1.0 / 120.0;
    p = p * r + 1.0 / 24.0;
    p = p * r + 1.0 / 6.0;
    p = p * r + 0.5;
    p = p * r + 1.0;
    p = p * r + 1.0;
    const int k = (int)kd;
    if (k < -1000) return (p * gem_pow2_d(k + 54)) * gem_pow2_d(-54);
    if (k > 1000) return (p * gem_pow2_d(k - 2)) * 4.0;
    return p * gem_pow2_d(k);
}
