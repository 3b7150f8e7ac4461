/* gm_math.h -- the occupancy grid's double log and exp, shared by the kernel (gm_grid.cu) and its C oracle (oracle/gm_oracle.c).
 *
 * libm's and CUDA's log / exp are different functions, so neither can stand in for the other bit for bit.  These two are
 * evaluated in double-double arithmetic out of plain IEEE operations and explicit fma only, with no table, so a host build
 * without FP contraction (-ffp-contract=off, SSE2) and a device build with -fmad=false compute the same bits.  The result is the
 * double-double value (relative error below about 2^-96) rounded once to double, so it is the correctly rounded value except when
 * the exact result lies within that error of a rounding boundary.  0, +-inf, NaN, subnormal arguments, overflow and gradual
 * underflow behave as in libm.  DESIGN.md "Occupancy grid" has the measured agreement with glibc.
 *
 * log: x = 2^e m, m in [sqrt(1/2), sqrt(2)); log m = 2 atanh f, f = (m - 1) / (m + 1), |f| < 0.1716, by its odd series to f^41.
 * exp: x = k log 2 + r, |r| <= log(2) / 2; exp(r / 256) - 1 by its Taylor series, squared eight times as e <- 2 e + e^2. */
#ifndef GM_MATH_H
#define GM_MATH_H

#include <math.h>
#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define GM_FN static __host__ __device__ __forceinline__
#else
#define GM_FN static inline
#endif

typedef struct { double hi, lo; } gm_dd;

GM_FN gm_dd gm_two_sum(double a, double b)
{
    gm_dd r;
    const double s = a + b, bb = s - a;
    r.hi = s;
    r.lo = (a - (s - bb)) + (b - bb);
    return r;
}
GM_FN gm_dd gm_fast_two_sum(double a, double b)      /* |a| >= |b| or a == 0 */
{
    gm_dd r;
    const double s = a + b;
    r.hi = s;
    r.lo = b - (s - a);
    return r;
}
GM_FN gm_dd gm_dd_add(gm_dd x, gm_dd y)
{
    gm_dd s = gm_two_sum(x.hi, y.hi);
    const gm_dd t = gm_two_sum(x.lo, y.lo);
    s = gm_fast_two_sum(s.hi, s.lo + t.hi);
    return gm_fast_two_sum(s.hi, s.lo + t.lo);
}
GM_FN gm_dd gm_dd_mul(gm_dd x, gm_dd y)
{
    const double p = x.hi * y.hi;
    double e = fma(x.hi, y.hi, -p);
    e = e + (x.hi * y.lo + x.lo * y.hi);
    return gm_fast_two_sum(p, e);
}
GM_FN gm_dd gm_dd_make(double hi, double lo)
{
    gm_dd r;
    r.hi = hi;
    r.lo = lo;
    return r;
}
GM_FN double gm_pow2(int k)                           /* 2^k, -1022 <= k <= 1023 */
{
    const uint64_t b = (uint64_t)(k + 1023) << 52;
    double r;
    memcpy(&r, &b, 8);
    return r;
}

#define GM_LN2_HI 0x1.62e42fefa39efp-1
#define GM_LN2_LO 0x1.abc9e3b39803fp-56

GM_FN double gm_log(double x)
{
    if (x != x) return x + x;
    if (x < 0.0) return NAN;
    if (x == 0.0) return -INFINITY;
    if (x == INFINITY) return x;
    int e = 0;
    if (x < 0x1p-1022) { x = x * 0x1p54; e = -54; }
    uint64_t b;
    memcpy(&b, &x, 8);
    e += (int)(b >> 52) - 1023;
    b = (b & 0x000fffffffffffffull) | 0x3ff0000000000000ull;
    double m;
    memcpy(&m, &b, 8);
    if (m > 0x1.6a09e667f3bcdp+0) { m = m * 0.5; e += 1; }
    /* f = (m - 1) / (m + 1): m - 1 is exact, m + 1 a two-sum, the quotient refined by its exact fma residual */
    const double num = m - 1.0;
    const gm_dd den = gm_two_sum(m, 1.0);
    const double q1 = num / den.hi;
    double rr = fma(-q1, den.hi, num);
    rr = rr - q1 * den.lo;
    const gm_dd f = gm_fast_two_sum(q1, rr / den.hi);
    const gm_dd f2 = gm_dd_mul(f, f);
    /* 1 + f^2 / 3 + f^4 / 5 + ...: the terms from f^22 on (below 2^-56 relative) in double, the rest in double-double */
    const double z = f2.hi;
    double t = 0x1.8f9c18f9c18fap-6;                                        /* 1/41 */
    t = t * z + 0x1.a41a41a41a41ap-6; t = t * z + 0x1.bacf914c1bad0p-6;     /* 1/39, 1/37 */
    t = t * z + 0x1.d41d41d41d41dp-6; t = t * z + 0x1.f07c1f07c1f08p-6;     /* 1/35, 1/33 */
    t = t * z + 0x1.0842108421084p-5; t = t * z + 0x1.1a7b9611a7b96p-5;     /* 1/31, 1/29 */
    t = t * z + 0x1.2f684bda12f68p-5; t = t * z + 0x1.47ae147ae147bp-5;     /* 1/27, 1/25 */
    t = t * z + 0x1.642c8590b2164p-5;                                       /* 1/23 */
    gm_dd p = gm_dd_make(t, 0.0);
#define GM_STEP(h, l) p = gm_dd_add(gm_dd_mul(p, f2), gm_dd_make(h, l))
    GM_STEP(0x1.8618618618618p-5, 0x1.8618618618618p-59);                   /* 1/21 */
    GM_STEP(0x1.af286bca1af28p-5, 0x1.af286bca1af28p-59);                   /* 1/19 */
    GM_STEP(0x1.e1e1e1e1e1e1ep-5, 0x1.e1e1e1e1e1e1ep-61);                   /* 1/17 */
    GM_STEP(0x1.1111111111111p-4, 0x1.1111111111111p-60);                   /* 1/15 */
    GM_STEP(0x1.3b13b13b13b14p-4, -0x1.3b13b13b13b14p-58);                  /* 1/13 */
    GM_STEP(0x1.745d1745d1746p-4, -0x1.745d1745d1746p-59);                  /* 1/11 */
    GM_STEP(0x1.c71c71c71c71cp-4, 0x1.c71c71c71c71cp-58);                   /* 1/9 */
    GM_STEP(0x1.2492492492492p-3, 0x1.2492492492492p-57);                   /* 1/7 */
    GM_STEP(0x1.999999999999ap-3, -0x1.999999999999ap-57);                  /* 1/5 */
    GM_STEP(0x1.5555555555555p-2, 0x1.5555555555555p-56);                   /* 1/3 */
    GM_STEP(1.0, 0.0);
#undef GM_STEP
    gm_dd l = gm_dd_mul(f, p);
    l.hi = 2.0 * l.hi;
    l.lo = 2.0 * l.lo;
    const double de = (double)e;
    const double eh = de * GM_LN2_HI;
    const gm_dd el = gm_fast_two_sum(eh, fma(de, GM_LN2_HI, -eh) + de * GM_LN2_LO);
    return gm_dd_add(el, l).hi;
}

GM_FN double gm_exp(double x)
{
    if (x != x) return x + x;
    if (x > 710.0) return INFINITY;
    if (x < -746.0) return 0.0;
    /* k = round(x / log 2) by the 1.5 * 2^52 shift; r = x - k log 2 in double-double */
    double kd = x * 0x1.71547652b82fep+0 + 0x1.8p52;
    kd = kd - 0x1.8p52;
    const int k = (int)kd;
    const double ph = kd * GM_LN2_HI;
    const gm_dd pk = gm_fast_two_sum(ph, fma(kd, GM_LN2_HI, -ph) + kd * GM_LN2_LO);
    gm_dd r = gm_dd_add(gm_dd_make(x, 0.0), gm_dd_make(-pk.hi, -pk.lo));
    r.hi = r.hi * 0x1p-8;
    r.lo = r.lo * 0x1p-8;
    /* e = exp(s) - 1 = s (1 + s / 2 + s^2 / 6 + ...), |s| < 2^-9.5: the terms from s^6 / 7! on in double */
    double t = 0x1.27e4fb7789f5cp-22;                                       /* 1/10! */
    t = t * r.hi + 0x1.71de3a556c734p-19;                                   /* 1/9! */
    t = t * r.hi + 0x1.a01a01a01a01ap-16;                                   /* 1/8! */
    t = t * r.hi + 0x1.a01a01a01a01ap-13;                                   /* 1/7! */
    gm_dd p = gm_dd_make(t, 0.0);
#define GM_STEP(h, l) p = gm_dd_add(gm_dd_mul(p, r), gm_dd_make(h, l))
    GM_STEP(0x1.6c16c16c16c17p-10, -0x1.f49f49f49f49fp-65);                 /* 1/6! */
    GM_STEP(0x1.1111111111111p-7, 0x1.1111111111111p-63);                   /* 1/5! */
    GM_STEP(0x1.5555555555555p-5, 0x1.5555555555555p-59);                   /* 1/4! */
    GM_STEP(0x1.5555555555555p-3, 0x1.5555555555555p-57);                   /* 1/3! */
    GM_STEP(0.5, 0.0);
    GM_STEP(1.0, 0.0);
#undef GM_STEP
    gm_dd e = gm_dd_mul(p, r);
    for (int i = 0; i < 8; i++) e = gm_dd_add(gm_dd_make(2.0 * e.hi, 2.0 * e.lo), gm_dd_mul(e, e));
    const gm_dd y = gm_dd_add(gm_dd_make(1.0, 0.0), e);
    if (k >= -1021 || (k == -1022 && y.hi >= 1.0)) {              /* a normal result */
        if (k > 1023) return (y.hi * gm_pow2(k - 1)) * 2.0;   /* overflows to inf iff the rounded value exceeds DBL_MAX */
        return y.hi * gm_pow2(k);
    }
    /* subnormal result: round y 2^(k + 1074) to an integer n once (ties to even), then n 2^-1074 is exact */
    const double sc = gm_pow2(k + 1074);
    const double H = y.hi * sc, L = y.lo * sc;
    double n = (H + 0x1p52) - 0x1p52;
    const double d = H - n;
    if (d == 0.5 && L > 0.0) n = n + 1.0;
    else if (d == -0.5 && L < 0.0) n = n - 1.0;
    return n * 0x1p-1074;
}

#endif /* GM_MATH_H */
