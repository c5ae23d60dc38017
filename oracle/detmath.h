/*
 * oracle/detmath.h -- TEST INFRASTRUCTURE (CPU oracle). Not part of the product.
 *
 * "DETMATH": a fixed, written-down evaluation of the transcendental functions
 * the reference's GLSL leaves to the Vulkan driver (sin, cos, exp, log, pow,
 * tanh, atan(y,x), inversesqrt).  Every function is a finite sequence of
 * IEEE-754 binary64 add/mul/div/fma operations (round-to-nearest-even) whose
 * result is then rounded ONCE to binary32.  Because only correctly-rounded
 * basic operations are used, the same sequence executed by gcc on x86-64
 * (-ffp-contract=off, explicit fma()) and by nvcc on sm_90a (-fmad=false,
 * explicit fma()) yields bit-identical results.  The binary64 results are
 * accurate to ~1e-14 relative, so the binary32 result equals the correctly
 * rounded value of the true function except with probability ~1e-6 per call
 * (checked against glibc libm in tests/test_oracle_detmath.py).
 *
 * The CUDA product carries its own, independently written copy of this spec
 * (godotoceanwaves_b200/csrc/detmath.cuh); the spec itself (constants and
 * operation order) is stated in DESIGN.md section "DETMATH".
 *
 * Reference call sites that need these functions:
 *   assets/shaders/compute/spectrum_compute.glsl:46-48 (log, cos, sin)
 *   assets/shaders/compute/spectrum_compute.glsl:60,84 (tanh)
 *   assets/shaders/compute/spectrum_compute.glsl:72,77,83,94,95,113 (inversesqrt, pow, cos, exp)
 *   assets/shaders/compute/spectrum_compute.glsl:107 (atan(y,x))
 *   assets/shaders/compute/spectrum_modulate.glsl:33,49 (cos, sin, tanh)
 *   assets/shaders/compute/fft_butterfly.glsl:15 (cos, sin)
 *   assets/shaders/compute/fft_unpack.glsl:62 (exp)
 */
#ifndef ORACLE_DETMATH_H
#define ORACLE_DETMATH_H
#include <math.h>
#include <stdint.h>
#include <string.h>

static inline double dm_from_bits(uint64_t b) { double d; memcpy(&d, &b, 8); return d; }
static inline uint64_t dm_to_bits(double d) { uint64_t b; memcpy(&b, &d, 8); return b; }

/* ---- sin / cos ----------------------------------------------------------
 * n = rint(x*2/pi); r = x - n*pi/2 by two-term Cody-Waite (PIO2_1 has 33
 * significant bits so n*PIO2_1 is exact for |n| < 2^20); Taylor polynomials
 * on |r| <= pi/4: sin through r^13, cos through r^14.                        */
#define DM_TWO_OVER_PI 0x1.45f306dc9c883p-1
#define DM_PIO2_1 0x1.921fb54400000p+0
#define DM_PIO2_2 0x1.0b4611a626331p-34
static inline void dm_sincos(double x, double *s, double *c) {
    double fn = rint(x * DM_TWO_OVER_PI);
    double r = fma(-fn, DM_PIO2_1, x);
    r = fma(-fn, DM_PIO2_2, r);
    int q = (int)(((int64_t)fn) & 3);
    double z = r * r;
    double ps = 0x1.6124613a86d09p-33;
    ps = fma(ps, z, -0x1.ae64567f544e4p-26);
    ps = fma(ps, z, 0x1.71de3a556c734p-19);
    ps = fma(ps, z, -0x1.a01a01a01a01ap-13);
    ps = fma(ps, z, 0x1.1111111111111p-7);
    ps = fma(ps, z, -0x1.5555555555555p-3);
    double sr = fma(r * z, ps, r);
    double pc = -0x1.93974a8c07c9dp-37;
    pc = fma(pc, z, 0x1.1eed8eff8d898p-29);
    pc = fma(pc, z, -0x1.27e4fb7789f5cp-22);
    pc = fma(pc, z, 0x1.a01a01a01a01ap-16);
    pc = fma(pc, z, -0x1.6c16c16c16c17p-10);
    pc = fma(pc, z, 0x1.5555555555555p-5);
    pc = fma(pc, z, -0x1.0000000000000p-1);
    double cr = fma(z, pc, 1.0);
    switch (q) {
        case 0: *s = sr;  *c = cr;  break;
        case 1: *s = cr;  *c = -sr; break;
        case 2: *s = -sr; *c = -cr; break;
        default: *s = -cr; *c = sr; break;
    }
}

/* ---- exp ---------------------------------------------------------------
 * argument clamped to [-110, 90] (binary32 results under/overflow outside);
 * n = rint(x*log2e); r = x - n*ln2 (two-term); Taylor through r^13; * 2^n.   */
#define DM_LOG2E 0x1.71547652b82fep+0
#define DM_LN2_HI 0x1.62e42ff000000p-1
#define DM_LN2_LO -0x1.718432a1b0e26p-35
static inline double dm_exp(double x) {
    if (x != x) return x;
    if (x < -110.0) x = -110.0;
    if (x > 90.0) x = 90.0;
    double fn = rint(x * DM_LOG2E);
    double r = fma(-fn, DM_LN2_HI, x);
    r = fma(-fn, DM_LN2_LO, r);
    double p = 0x1.6124613a86d09p-33;            /* 1/13! */
    p = fma(p, r, 0x1.1eed8eff8d898p-29);         /* 1/12! */
    p = fma(p, r, 0x1.ae64567f544e4p-26);         /* 1/11! */
    p = fma(p, r, 0x1.27e4fb7789f5cp-22);         /* 1/10! */
    p = fma(p, r, 0x1.71de3a556c734p-19);         /* 1/9!  */
    p = fma(p, r, 0x1.a01a01a01a01ap-16);         /* 1/8!  */
    p = fma(p, r, 0x1.a01a01a01a01ap-13);         /* 1/7!  */
    p = fma(p, r, 0x1.6c16c16c16c17p-10);         /* 1/6!  */
    p = fma(p, r, 0x1.1111111111111p-7);          /* 1/5!  */
    p = fma(p, r, 0x1.5555555555555p-5);          /* 1/4!  */
    p = fma(p, r, 0x1.5555555555555p-3);          /* 1/3!  */
    p = fma(p, r, 0x1.0000000000000p-1);          /* 1/2!  */
    double e = fma(r * r, p, r) + 1.0;
    uint64_t sb = (uint64_t)((int64_t)fn + 1023) << 52;
    return e * dm_from_bits(sb);
}

/* ---- log (x a non-negative binary32 value widened to binary64) ---------- */
#define DM_SQRT2 0x1.6a09e667f3bcdp+0
static inline double dm_log(double x) {
    if (x != x) return x;
    if (x < 0.0) return NAN;
    if (x == 0.0) return -INFINITY;
    if (x == INFINITY) return x;
    uint64_t b = dm_to_bits(x);
    int64_t e = (int64_t)(b >> 52) - 1023;
    double m = dm_from_bits((b & 0x000fffffffffffffULL) | 0x3ff0000000000000ULL);
    if (m > DM_SQRT2) { m = m * 0.5; e += 1; }
    double f = m - 1.0;
    double s = f / (2.0 + f);
    double z = s * s;
    double p = 0x1.8618618618618p-5;              /* 1/21 */
    p = fma(p, z, 0x1.af286bca1af28p-5);          /* 1/19 */
    p = fma(p, z, 0x1.e1e1e1e1e1e1ep-5);          /* 1/17 */
    p = fma(p, z, 0x1.1111111111111p-4);          /* 1/15 */
    p = fma(p, z, 0x1.3b13b13b13b14p-4);          /* 1/13 */
    p = fma(p, z, 0x1.745d1745d1746p-4);          /* 1/11 */
    p = fma(p, z, 0x1.c71c71c71c71cp-4);          /* 1/9  */
    p = fma(p, z, 0x1.2492492492492p-3);          /* 1/7  */
    p = fma(p, z, 0x1.999999999999ap-3);          /* 1/5  */
    p = fma(p, z, 0x1.5555555555555p-2);          /* 1/3  */
    double lm = 2.0 * fma(s * z, p, s);
    double de = (double)e;
    return fma(de, DM_LN2_HI, fma(de, DM_LN2_LO, lm));
}

/* ---- pow for x >= 0 ------------------------------------------------------ */
static inline double dm_pow(double x, double y) {
    if (y == 0.0) return 1.0;
    if (x == 0.0) return (y > 0.0) ? 0.0 : INFINITY;
    return dm_exp(y * dm_log(x));
}

/* ---- tanh ---------------------------------------------------------------- */
static inline double dm_tanh(double a) {
    if (a != a) return a;
    double aa = fabs(a), r;
    if (aa < 0x1.0624dd2f1a9fcp-10) {             /* 1e-3: odd Taylor series */
        double z = aa * aa;
        double p = fma(z, 0x1.1111111111111p-3, -0x1.5555555555555p-2); /* 2/15, -1/3 */
        r = fma(aa * z, p, aa);
    } else {
        double t = dm_exp(-2.0 * aa);
        r = (1.0 - t) / (1.0 + t);
    }
    return (a < 0.0) ? -r : r;
}

/* ---- atan2(y, x); atan2(0,0) := 0 ---------------------------------------- */
#define DM_PI 0x1.921fb54442d18p+1
#define DM_PIO2 0x1.921fb54442d18p+0
static const double DM_ATAN_TAB[9] = {
    0x0.0p+0, 0x1.fd5ba9aac2f6ep-4, 0x1.f5b75f92c80ddp-3, 0x1.6f61941e4def1p-2,
    0x1.dac670561bb4fp-2, 0x1.1e00babdefeb4p-1, 0x1.4978fa3269ee1p-1,
    0x1.700a7c5784634p-1, 0x1.921fb54442d18p-1 };
static inline double dm_atan2(double y, double x) {
    double ax = fabs(x), ay = fabs(y);
    if (ax == 0.0 && ay == 0.0) return 0.0;
    int swap = ay > ax;
    double t = swap ? ax / ay : ay / ax;
    double fi = rint(t * 8.0);
    double c = fi * 0.125;
    double u = (t - c) / fma(t, c, 1.0);
    double z = u * u;
    double p = -0x1.1111111111111p-4;             /* -1/15 */
    p = fma(p, z, 0x1.3b13b13b13b14p-4);          /*  1/13 */
    p = fma(p, z, -0x1.745d1745d1746p-4);         /* -1/11 */
    p = fma(p, z, 0x1.c71c71c71c71cp-4);          /*  1/9  */
    p = fma(p, z, -0x1.2492492492492p-3);         /* -1/7  */
    p = fma(p, z, 0x1.999999999999ap-3);          /*  1/5  */
    p = fma(p, z, -0x1.5555555555555p-2);         /* -1/3  */
    double r = fma(u * z, p, u) + DM_ATAN_TAB[(int)fi];
    if (swap) r = DM_PIO2 - r;
    if (x < 0.0) r = DM_PI - r;
    return (y < 0.0) ? -r : r;
}
#endif
