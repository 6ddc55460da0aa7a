/* gem_pcdfmt.h -- one float as glibc's printf("%.8g") prints it, exactly, in a form that both nvcc (device and host) and
 * a C++ compiler accept.  The PCD kernels (gem_pcd.cuh) and the host build the tests and scripts/pcd_float_exhaustive.py
 * check against snprintf (tests/pcd_fmt_host.cpp) include this one source.  PCL's ASCII writer prints a float field
 * with `ostream << value` at precision 8 in the classic locale, which libstdc++ hands to vsnprintf("%.*g").
 *
 * Method: a finite non-zero float is m 2^e with an integer m < 2^24.  With E = floor(log2 |v|) and
 * kest = floor(E log10 2) = (E * 78913) >> 18, the decimal exponent k = floor(log10 |v|) is kest or kest + 1, so
 * T = floor(|v| / 10^(kest - 8)) has 9 or 10 digits.  T is computed exactly with 32-bit limbs: for kest >= 8 as
 * (m << e) divided by 10^(kest - 8) (at most 128 bits), otherwise as m 10^(8 - kest) (at most 201 bits) shifted right by
 * -e, with a sticky bit for every discarded non-zero remainder.  A 10-digit T drops one more digit into the sticky bit
 * (k = kest + 1).  The 9th digit and the sticky bit then round the 8 digits to nearest, ties to even (glibc rounds the
 * exact binary value in the current rounding mode); a carry to 10^8 moves k up by one.  %g's style comes from k after
 * rounding: exponent style when k < -4 or k >= 8, fixed otherwise; trailing zeros and a trailing '.' are dropped and the
 * exponent has two digits (|k| <= 45).  NaN of any sign or payload is "nan" (PCL tests isnan before printing); -0, inf
 * and -inf print as "-0", "inf" and "-inf".  The longest result is 14 characters ("-1.2345678e-38",
 * "-0.00012345678"). */
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define GEM_PF static __host__ __device__ __forceinline__
#else
#define GEM_PF static inline
#endif

#define GEM_PCD_VALUE_MAX 14

enum { GEM_PCD_FINITE = 0, GEM_PCD_ZERO = 1, GEM_PCD_INF = 2, GEM_PCD_NAN = 3, GEM_PCD_UINT = 4 };

/* one value ready to print: kind, sign, the 8 rounded digits (or the unsigned value) and the decimal exponent */
typedef struct gem_pcd_val {
    uint32_t d;   /* GEM_PCD_FINITE: 10^7 <= d < 10^8; GEM_PCD_UINT: the value */
    int k;        /* GEM_PCD_FINITE: the decimal exponent after rounding */
    int kind;
    int neg;
    int nd;       /* digits printed: GEM_PCD_FINITE: of d without trailing zeros; GEM_PCD_UINT: of d */
} gem_pcd_val;

GEM_PF int gem_pcd_clz32(uint32_t x)
{
#ifdef __CUDA_ARCH__
    return __clz((int)x);
#else
    return __builtin_clz(x);
#endif
}

/* 10^p for 0 <= p <= 9 */
GEM_PF uint32_t gem_pcd_pow10(int p)
{
    uint32_t r = 1u;
    for (int i = 0; i < p; i++) r *= 10u;
    return r;
}

/* floor(x / d) in place over limbs [0, nl) (little-endian); returns the remainder */
GEM_PF uint32_t gem_pcd_divmod(uint32_t *x, int nl, uint32_t d)
{
    uint64_t r = 0;
    for (int i = nl - 1; i >= 0; i--) {
        const uint64_t cur = (r << 32) | x[i];
        x[i] = (uint32_t)(cur / d);
        r = cur % d;
    }
    return (uint32_t)r;
}

/* x *= f in place; *nl grows by the carry limb */
GEM_PF void gem_pcd_mul(uint32_t *x, int *nl, uint32_t f)
{
    uint64_t c = 0;
    for (int i = 0; i < *nl; i++) {
        const uint64_t p = (uint64_t)x[i] * f + c;
        x[i] = (uint32_t)p;
        c = p >> 32;
    }
    if (c) x[(*nl)++] = (uint32_t)c;
}

/* the 8 digits and decimal exponent of a finite non-zero float (sign ignored) */
GEM_PF void gem_pcd_digits(uint32_t bits, uint32_t *d_out, int *k_out)
{
    const uint32_t ex = (bits >> 23) & 0xffu, man = bits & 0x7fffffu;
    const uint32_t m = ex ? (man | 0x800000u) : man;
    const int e = ex ? (int)ex - 150 : -149;
    const int E = e + 31 - gem_pcd_clz32(m);
    const int kest = (E * 78913) >> 18; /* arithmetic shift: floor for negative E as well */
    uint32_t x[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
    uint64_t T;
    int sticky = 0;
    if (kest >= 8) { /* v >= 10^8 > 2^24: e > 0, m << e < 2^128 */
        const int w = e >> 5, b = e & 31;
        const uint64_t s = (uint64_t)m << b;
        x[w] = (uint32_t)s;
        x[w + 1] = (uint32_t)(s >> 32);
        int nl = w + 2, p = kest - 8;
        for (; p >= 9; p -= 9) sticky |= gem_pcd_divmod(x, nl, 1000000000u) != 0;
        if (p > 0) sticky |= gem_pcd_divmod(x, nl, gem_pcd_pow10(p)) != 0;
        T = ((uint64_t)x[1] << 32) | x[0];
    } else {
        int nl = 1, q = 8 - kest;
        x[0] = m;
        for (; q >= 9; q -= 9) gem_pcd_mul(x, &nl, 1000000000u);
        if (q > 0) gem_pcd_mul(x, &nl, gem_pcd_pow10(q));
        if (e >= 0) { /* v < 10^8 and e >= 0: e <= 3, x < 2^61 */
            T = (((uint64_t)x[1] << 32) | x[0]) << e;
        } else {
            const int s = -e, w = s >> 5, b = s & 31;
            for (int i = 0; i < w; i++) sticky |= x[i] != 0;
            if (b) sticky |= (x[w] & ((1u << b) - 1u)) != 0;
            const uint64_t lo = ((uint64_t)x[w + 1] << 32) | x[w];
            T = b ? (lo >> b) | ((uint64_t)x[w + 2] << (64 - b)) : lo;
        }
    }
    int k = kest;
    if (T >= 1000000000ull) {
        sticky |= (T % 10u) != 0;
        T /= 10u;
        k++;
    }
    const uint32_t t = (uint32_t)T;
    uint32_t d = t / 10u;
    const uint32_t r = t % 10u;
    if (r > 5u || (r == 5u && (sticky || (d & 1u)))) d++;
    if (d == 100000000u) {
        d = 10000000u;
        k++;
    }
    *d_out = d;
    *k_out = k;
}

/* the value of a float field */
GEM_PF gem_pcd_val gem_pcd_float(uint32_t bits)
{
    gem_pcd_val v;
    v.d = 0u;
    v.k = 0;
    v.neg = (int)(bits >> 31);
    v.nd = 1;
    const uint32_t ex = (bits >> 23) & 0xffu, man = bits & 0x7fffffu;
    if (ex == 0xffu) {
        v.kind = man ? GEM_PCD_NAN : GEM_PCD_INF;
        if (man) v.neg = 0;
        return v;
    }
    if ((bits & 0x7fffffffu) == 0u) {
        v.kind = GEM_PCD_ZERO;
        return v;
    }
    v.kind = GEM_PCD_FINITE;
    gem_pcd_digits(bits, &v.d, &v.k);
    uint32_t d = v.d;
    int nd = 8;
    while (d % 10u == 0u) { /* d >= 10^7 has a non-zero leading digit */
        d /= 10u;
        nd--;
    }
    v.nd = nd;
    return v;
}

/* the value of a field printed as an unsigned 32-bit integer (newer PCL's rgb) */
GEM_PF gem_pcd_val gem_pcd_uint(uint32_t bits)
{
    gem_pcd_val v;
    v.d = bits;
    v.k = 0;
    v.kind = GEM_PCD_UINT;
    v.neg = 0;
    int nd = 1;
    for (uint32_t t = bits; t >= 10u; t /= 10u) nd++;
    v.nd = nd;
    return v;
}

/* characters gem_pcd_put writes for v */
GEM_PF int gem_pcd_len(gem_pcd_val v)
{
    int n = v.neg;
    switch (v.kind) {
    case GEM_PCD_NAN: return 3;
    case GEM_PCD_INF: return n + 3;
    case GEM_PCD_ZERO: return n + 1;
    case GEM_PCD_UINT: return v.nd;
    default: break;
    }
    if (v.k < -4 || v.k >= 8) return n + v.nd + (v.nd > 1) + 4;  /* d[.ddd]e+XX */
    if (v.k >= 0) return n + v.k + 1 + (v.nd > v.k + 1 ? v.nd - v.k : 0);
    return n + 1 - v.k + v.nd;                                     /* 0.000ddd */
}

/* writes v's characters to out (no terminator); returns their number */
GEM_PF int gem_pcd_put(gem_pcd_val v, char *out)
{
    int n = 0;
    if (v.kind == GEM_PCD_NAN) {
        out[0] = 'n'; out[1] = 'a'; out[2] = 'n';
        return 3;
    }
    if (v.neg) out[n++] = '-';
    if (v.kind == GEM_PCD_INF) {
        out[n] = 'i'; out[n + 1] = 'n'; out[n + 2] = 'f';
        return n + 3;
    }
    if (v.kind == GEM_PCD_ZERO) {
        out[n] = '0';
        return n + 1;
    }
    char dig[10];
    const int nd = v.kind == GEM_PCD_UINT ? v.nd : 8;
    uint32_t d = v.d;
    for (int i = nd - 1; i >= 0; i--) {
        dig[i] = (char)('0' + d % 10u);
        d /= 10u;
    }
    if (v.kind == GEM_PCD_UINT) {
        for (int i = 0; i < nd; i++) out[n++] = dig[i];
        return n;
    }
    const int k = v.k;
    if (k < -4 || k >= 8) {
        out[n++] = dig[0];
        if (v.nd > 1) {
            out[n++] = '.';
            for (int i = 1; i < v.nd; i++) out[n++] = dig[i];
        }
        const int a = k < 0 ? -k : k;
        out[n++] = 'e';
        out[n++] = k < 0 ? '-' : '+';
        out[n++] = (char)('0' + a / 10);
        out[n++] = (char)('0' + a % 10);
    } else if (k >= 0) {
        for (int i = 0; i <= k; i++) out[n++] = dig[i];
        if (v.nd > k + 1) {
            out[n++] = '.';
            for (int i = k + 1; i < v.nd; i++) out[n++] = dig[i];
        }
    } else {
        out[n++] = '0';
        out[n++] = '.';
        for (int i = 0; i < -k - 1; i++) out[n++] = '0';
        for (int i = 0; i < v.nd; i++) out[n++] = dig[i];
    }
    return n;
}
