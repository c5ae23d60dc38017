// detmath.cuh -- device-side DETMATH (spec: DESIGN.md "DETMATH").
//
// The reference's GLSL leaves sin/cos/exp/log/pow/tanh/atan precision to the Vulkan
// driver (assets/shaders/compute/*.glsl).  This product fixes them as explicit sequences
// of IEEE-754 binary64 add/mul/div/fma operations whose result is rounded once to
// binary32, so results are reproducible bit for bit on any IEEE machine.  Compile with
// -fmad=false: every fused operation below is an explicit fma().
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace detmath {

// ---- sin/cos: two-term Cody-Waite by pi/2 (33-bit head, one fma per term), Taylor kernels on r ----
// The constants live in constant memory: a binary64 immediate costs two UMOVs per use, a constant-bank
// operand costs one uniform load that the compiler can hoist out of loops.
__constant__ double c_sincos[16] = {
    0x1.45f306dc9c883p-1,    // [0]  2/pi
    0x1.921fb54400000p+0,    // [1]  pi/2 head (33 bits)
    0x1.0b4611a626331p-34,   // [2]  pi/2 tail
    0x1.6124613a86d09p-33,   // [3]  sin:  1/13!
    -0x1.ae64567f544e4p-26,  // [4]       -1/11!
    0x1.71de3a556c734p-19,   // [5]        1/9!
    -0x1.a01a01a01a01ap-13,  // [6]       -1/7!
    0x1.1111111111111p-7,    // [7]        1/5!
    -0x1.5555555555555p-3,   // [8]       -1/3!
    -0x1.93974a8c07c9dp-37,  // [9]  cos: -1/14!
    0x1.1eed8eff8d898p-29,   // [10]       1/12!
    -0x1.27e4fb7789f5cp-22,  // [11]      -1/10!
    0x1.a01a01a01a01ap-16,   // [12]       1/8!
    -0x1.6c16c16c16c17p-10,  // [13]      -1/6!
    0x1.5555555555555p-5,    // [14]       1/4!
    -0x1.0000000000000p-1 }; // [15]      -1/2!

// Quadrant of n: the low two bits of n converted to int64 with saturation, NaN giving 0 (|n| >= 2^63, i.e. |x| >= 1.45e19,
// gives INT64_MAX / INT64_MIN).  __double2ll_rz is the PTX instruction cvt.rzi.s64.f64, whose out-of-range results the PTX ISA
// defines that way (clamped to the destination range, NaN -> 0); a C++ cast would be undefined behaviour there.  The CUDA
// headers do not promise the out-of-range result of the intrinsic, so tests/test_gpu_device_math.py pins it against the C
// copy (oracle/detmath.h spells the rule out) at every exponent beyond 2^63.  (An explicit clamp costs the bench kernel 20
// bytes of spill.)  The result for such x is meaningless but the same on both sides.
__device__ __forceinline__ int quadrant(double fn) {
    return (int)(__double2ll_rz(fn) & 3);
}

__device__ __forceinline__ void sincos64(double x, double& s, double& c) {
    const double fn = rint(x * c_sincos[0]);
    double r = fma(-fn, c_sincos[1], x);
    r = fma(-fn, c_sincos[2], r);
    const int q = quadrant(fn);
    const double z = r * r;
    double ps = c_sincos[3];
    ps = fma(ps, z, c_sincos[4]);
    ps = fma(ps, z, c_sincos[5]);
    ps = fma(ps, z, c_sincos[6]);
    ps = fma(ps, z, c_sincos[7]);
    ps = fma(ps, z, c_sincos[8]);
    const double sr = fma(r * z, ps, r);
    double pc = c_sincos[9];
    pc = fma(pc, z, c_sincos[10]);
    pc = fma(pc, z, c_sincos[11]);
    pc = fma(pc, z, c_sincos[12]);
    pc = fma(pc, z, c_sincos[13]);
    pc = fma(pc, z, c_sincos[14]);
    pc = fma(pc, z, c_sincos[15]);
    const double cr = fma(z, pc, 1.0);
    const double s0 = (q & 1) ? cr : sr;
    const double c0 = (q & 1) ? sr : cr;
    s = (q & 2) ? -s0 : s0;
    c = ((q + 1) & 2) ? -c0 : c0;
}

// ---- exp: clamp to [-110, 90]; n = rint(x*log2e); two-term ln2 reduction; Taylor to r^13 ----
// (exp64 / log64 are real functions, not inlined: the spectrum kernel calls them a dozen times per texel quad and was an
//  instruction-cache-bound 61 KB of straight-line code with every call expanded)
static __device__ __noinline__ double exp64(double x) {   // static: the header is compiled into more than one object
    if (x != x) return x;
    if (x < -110.0) x = -110.0;
    if (x > 90.0) x = 90.0;
    const double fn = rint(x * 0x1.71547652b82fep+0);
    double r = fma(-fn, 0x1.62e42ff000000p-1, x);
    r = fma(-fn, -0x1.718432a1b0e26p-35, r);
    double p = 0x1.6124613a86d09p-33;
    p = fma(p, r, 0x1.1eed8eff8d898p-29);
    p = fma(p, r, 0x1.ae64567f544e4p-26);
    p = fma(p, r, 0x1.27e4fb7789f5cp-22);
    p = fma(p, r, 0x1.71de3a556c734p-19);
    p = fma(p, r, 0x1.a01a01a01a01ap-16);
    p = fma(p, r, 0x1.a01a01a01a01ap-13);
    p = fma(p, r, 0x1.6c16c16c16c17p-10);
    p = fma(p, r, 0x1.1111111111111p-7);
    p = fma(p, r, 0x1.5555555555555p-5);
    p = fma(p, r, 0x1.5555555555555p-3);
    p = fma(p, r, 0x1.0000000000000p-1);
    const double e = fma(r * r, p, r) + 1.0;
    const long long sb = ((long long)fn + 1023LL) << 52;
    return e * __longlong_as_double(sb);
}

// ---- log of a non-negative binary32 value widened to binary64 ----
static __device__ __noinline__ double log64(double x) {
    if (x != x) return x;
    if (x < 0.0) return __longlong_as_double(0x7ff8000000000000LL);
    if (x == 0.0) return __longlong_as_double(0xfff0000000000000LL);
    if (x == __longlong_as_double(0x7ff0000000000000LL)) return x;
    const long long b = __double_as_longlong(x);
    long long e = (b >> 52) - 1023;
    double m = __longlong_as_double((b & 0x000fffffffffffffLL) | 0x3ff0000000000000LL);
    if (m > 0x1.6a09e667f3bcdp+0) { m = m * 0.5; e += 1; }
    const double f = m - 1.0;
    const double s = f / (2.0 + f);
    const double z = s * s;
    double p = 0x1.8618618618618p-5;
    p = fma(p, z, 0x1.af286bca1af28p-5);
    p = fma(p, z, 0x1.e1e1e1e1e1e1ep-5);
    p = fma(p, z, 0x1.1111111111111p-4);
    p = fma(p, z, 0x1.3b13b13b13b14p-4);
    p = fma(p, z, 0x1.745d1745d1746p-4);
    p = fma(p, z, 0x1.c71c71c71c71cp-4);
    p = fma(p, z, 0x1.2492492492492p-3);
    p = fma(p, z, 0x1.999999999999ap-3);
    p = fma(p, z, 0x1.5555555555555p-2);
    const double lm = 2.0 * fma(s * z, p, s);
    const double de = (double)e;
    return fma(de, 0x1.62e42ff000000p-1, fma(de, -0x1.718432a1b0e26p-35, lm));
}

__device__ __forceinline__ double pow64(double x, double y) {   // x >= 0
    if (y == 0.0) return 1.0;
    if (x == 0.0) return (y > 0.0) ? 0.0 : __longlong_as_double(0x7ff0000000000000LL);
    return exp64(y * log64(x));
}

__device__ __forceinline__ double tanh64(double a) {
    if (a != a) return a;
    const double aa = fabs(a);
    double r;
    if (aa < 0x1.0624dd2f1a9fcp-10) {
        const double z = aa * aa;
        const double p = fma(z, 0x1.1111111111111p-3, -0x1.5555555555555p-2);
        r = fma(aa * z, p, aa);
    } else {
        const double t = exp64(-2.0 * aa);
        r = (1.0 - t) / (1.0 + t);
    }
    return (a < 0.0) ? -r : r;
}

// atan(i/8), i = 0..8 (constant memory: a local array would live on the thread's stack)
__constant__ double c_atan_tab[9] = {
    0x0.0p+0, 0x1.fd5ba9aac2f6ep-4, 0x1.f5b75f92c80ddp-3, 0x1.6f61941e4def1p-2,
    0x1.dac670561bb4fp-2, 0x1.1e00babdefeb4p-1, 0x1.4978fa3269ee1p-1,
    0x1.700a7c5784634p-1, 0x1.921fb54442d18p-1 };
__device__ __forceinline__ double atan2_64(double y, double x) {   // atan2(0,0) := 0
    const double ax = fabs(x), ay = fabs(y);
    if (ax == 0.0 && ay == 0.0) return 0.0;
    const bool swap = ay > ax;
    const double t = swap ? ax / ay : ay / ax;
    if (t != t) return t;                 // an argument NaN, or both infinite: NaN, before t indexes the table
    const double fi = rint(t * 8.0);
    const double c = fi * 0.125;
    const double u = (t - c) / fma(t, c, 1.0);
    const double z = u * u;
    double p = -0x1.1111111111111p-4;
    p = fma(p, z, 0x1.3b13b13b13b14p-4);
    p = fma(p, z, -0x1.745d1745d1746p-4);
    p = fma(p, z, 0x1.c71c71c71c71cp-4);
    p = fma(p, z, -0x1.2492492492492p-3);
    p = fma(p, z, 0x1.999999999999ap-3);
    p = fma(p, z, -0x1.5555555555555p-2);
    double r = fma(u * z, p, u) + c_atan_tab[(int)fi];
    if (swap) r = 0x1.921fb54442d18p+0 - r;
    if (x < 0.0) r = 0x1.921fb54442d18p+1 - r;
    return (y < 0.0) ? -r : r;
}

// ---- binary32 front-ends (one rounding) ----
// binary32 sin/cos of a binary32 argument.  Same value as rounding sincos64's outputs: the quadrant swap and
// negation commute with the (sign-symmetric) rounding, so they are applied to the two rounded kernel values.
__device__ __forceinline__ void sincosf_det(float x, float& s, float& c) {
    const double xd = (double)x;
    const double fn = rint(xd * c_sincos[0]);
    double r = fma(-fn, c_sincos[1], xd);
    r = fma(-fn, c_sincos[2], r);
    const int q = quadrant(fn);
    const double z = r * r;
    double ps = c_sincos[3];
    ps = fma(ps, z, c_sincos[4]);
    ps = fma(ps, z, c_sincos[5]);
    ps = fma(ps, z, c_sincos[6]);
    ps = fma(ps, z, c_sincos[7]);
    ps = fma(ps, z, c_sincos[8]);
    const float sr = (float)fma(r * z, ps, r);
    double pc = c_sincos[9];
    pc = fma(pc, z, c_sincos[10]);
    pc = fma(pc, z, c_sincos[11]);
    pc = fma(pc, z, c_sincos[12]);
    pc = fma(pc, z, c_sincos[13]);
    pc = fma(pc, z, c_sincos[14]);
    pc = fma(pc, z, c_sincos[15]);
    const float cr = (float)fma(z, pc, 1.0);
    const float s0 = (q & 1) ? cr : sr;
    const float c0 = (q & 1) ? sr : cr;
    s = (q & 2) ? -s0 : s0;
    c = ((q + 1) & 2) ? -c0 : c0;
}
// K independent arguments at once: every table constant is fetched once and the K chains advance in lockstep, so the
// binary64 dependency chains overlap.  Values identical to sincosf_det.
template <int K>
__device__ __forceinline__ void sincosf_det_n(const float (&x)[K], float (&s)[K], float (&c)[K]) {
    double fn[K], r[K], z[K], ps[K], pc[K];
#pragma unroll
    for (int e = 0; e < K; ++e) {
        const double xd = (double)x[e];
        fn[e] = rint(xd * c_sincos[0]);
        r[e] = fma(-fn[e], c_sincos[1], xd);
        r[e] = fma(-fn[e], c_sincos[2], r[e]);
        z[e] = r[e] * r[e];
        ps[e] = c_sincos[3];
        pc[e] = c_sincos[9];
    }
#pragma unroll
    for (int j = 0; j < 5; ++j) {
#pragma unroll
        for (int e = 0; e < K; ++e) {
            ps[e] = fma(ps[e], z[e], c_sincos[4 + j]);
            pc[e] = fma(pc[e], z[e], c_sincos[10 + j]);
        }
    }
#pragma unroll
    for (int e = 0; e < K; ++e) {
        pc[e] = fma(pc[e], z[e], c_sincos[15]);
        const float sr = (float)fma(r[e] * z[e], ps[e], r[e]);
        const float cr = (float)fma(z[e], pc[e], 1.0);
        const int q = quadrant(fn[e]);
        const float s0 = (q & 1) ? cr : sr;
        const float c0 = (q & 1) ? sr : cr;
        s[e] = (q & 2) ? -s0 : s0;
        c[e] = ((q + 1) & 2) ? -c0 : c0;
    }
}
__device__ __forceinline__ float cosf_det(float x) { double s, c; sincos64((double)x, s, c); return (float)c; }
__device__ __forceinline__ float expf_det(float x) { return (float)exp64((double)x); }
__device__ __forceinline__ float logf_det(float x) { return (float)log64((double)x); }
__device__ __forceinline__ float powf_det(float x, float y) { return (float)pow64((double)x, (double)y); }
__device__ __forceinline__ float tanhf_det(float x) { return (float)tanh64((double)x); }
__device__ __forceinline__ float atan2f_det(float y, float x) { return (float)atan2_64((double)y, (double)x); }
__device__ __forceinline__ float inversesqrtf_det(float x) { return (float)(1.0 / sqrt((double)x)); }

}  // namespace detmath
