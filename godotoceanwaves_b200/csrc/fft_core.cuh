// fft_core.cuh -- register-resident radix-2 Stockham passes on lane pairs of fp32 (sm_90a).
//
// The reference's inverse FFT (assets/shaders/compute/fft_butterfly.glsl:24-34 + fft_compute.glsl:47-58)
// is a radix-2 decimation-in-time Stockham network: stage s (stride = 2^s, mid = N >> (s+1))
//     out[stride*(2i+b) + j] = in[stride*i + j] +/- tw(s, j) * in[stride*(i+mid) + j],   j < stride, i < mid
// with tw(s, j) = (cos, sin)(fp32(PI) / 2^s * j).  To stay bit-identical with it the butterflies below
// perform exactly that arithmetic (FMA contraction mode of the oracle), but log2(R) consecutive stages
// are composed on R values held in registers, so data crosses threads (through shared memory) only
// between radix-R passes.  Index algebra (DESIGN.md "FFT plan"): at the start of a pass whose first
// stage is LS0 the natural index is idx = 2^LS0 * i + j; group g = (i', j) owns the R elements
// a*(N/R) + g, and output b of that group lands on 2^LS0*R*i' + 2^LS0*b + j.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace ocean {

constexpr int kMaxMapSizeFft = 1024;
constexpr int kTwiddleTableSize = kMaxMapSizeFft;   // entries (1<<s)-1+j, j < 2^s, s < 10  (+1 pad)

// Universal twiddle table; warp-uniform lookups (first pass) read it from the constant bank.
__constant__ float2 c_twiddles[kTwiddleTableSize];

typedef unsigned long long u64;

__device__ __forceinline__ u64 pk(float lo, float hi) {
    u64 r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ void upk(u64 v, float& lo, float& hi) {
    asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
// Lane-wise operations on a pair.  sm_90 has no packed fp32 instruction: each lane is one scalar FFMA / FMUL / FADD
// with an explicit .rn rounding, which ptxas never contracts, so every lane rounds exactly once as the GLSL text does.
__device__ __forceinline__ u64 fma2(u64 a, u64 b, u64 c) {
    float a0, a1, b0, b1, c0, c1;
    upk(a, a0, a1); upk(b, b0, b1); upk(c, c0, c1);
    return pk(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ u64 mul2(u64 a, u64 b) {
    float a0, a1, b0, b1;
    upk(a, a0, a1); upk(b, b0, b1);
    return pk(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ u64 add2(u64 a, u64 b) {
    float a0, a1, b0, b1;
    upk(a, a0, a1); upk(b, b0, b1);
    return pk(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ u64 sub2(u64 a, u64 b) {
    float a0, a1, b0, b1;
    upk(a, a0, a1); upk(b, b0, b1);
    return pk(__fsub_rn(a0, b0), __fsub_rn(a1, b1));
}

// Two complex numbers (spectrum layers a and b of one layer pair) in SoA form.
struct C2 {
    u64 re;  // (re_a, re_b)
    u64 im;  // (im_a, im_b)
};
__device__ __forceinline__ C2 c2_from(float4 v) { return C2{pk(v.x, v.y), pk(v.z, v.w)}; }
__device__ __forceinline__ float4 c2_to(const C2& c) {
    float4 v;
    upk(c.re, v.x, v.y);
    upk(c.im, v.z, v.w);
    return v;
}

// One radix-2 butterfly of fft_compute.glsl:55-57 for both layers of the pair:
//   p = mul_complex(l, tw) = (fma(l.re, tx, -(l.im*ty)), fma(l.re, ty, l.im*tx));  o0 = u + p
//   o1 = u + mul_complex(l, -tw) = u - p      (negation commutes with round-to-nearest, except for the sign of an exact
//   zero: -(a + b) is -0 and (-a) + (-b) is +0 when a + b is a zero sum of opposite zeros)
__device__ __forceinline__ void butterfly(const C2& u, const C2& l, float2 tw, C2& o0, C2& o1) {
    const u64 txx = pk(tw.x, tw.x), tyy = pk(tw.y, tw.y), nty = pk(-tw.y, -tw.y);
    const u64 pre = fma2(l.re, txx, mul2(l.im, nty));
    const u64 pim = fma2(l.re, tyy, mul2(l.im, txx));
    o0.re = add2(u.re, pre);
    o0.im = add2(u.im, pim);
    o1.re = sub2(u.re, pre);
    o1.im = sub2(u.im, pim);
}
// tw == (1, 0) exactly (j == 0 of every stage): l*tw == l for finite l up to the sign of an exact zero
// (fma(x, 1, -(y*0)) == x and fma(x, 0, y*1) == y for every finite x, y != 0), so the product is skipped.  For infinite
// lanes the reference's product is NaN (inf*0) where the skip passes inf or a finite value through: once a binary32
// intermediate overflows, the two sides no longer agree NaN for NaN.  Computing the product instead cost 3.5 % of the bench
// step (H100, 400 W power limit; the measurement is recorded in DESIGN.md section 2).
__device__ __forceinline__ void butterfly_unit(const C2& u, const C2& l, C2& o0, C2& o1) {
    o0.re = add2(u.re, l.re);
    o0.im = add2(u.im, l.im);
    o1.re = sub2(u.re, l.re);
    o1.im = sub2(u.im, l.im);
}

// Stage LS0+T of a radix-R pass on registers.  j (< 2^LS0) = already produced low output index.
template <int R, int T, int LS0>
__device__ __forceinline__ void stockham_stage(const C2 (&in)[R], C2 (&out)[R], int j, const float2* __restrict__ tw_g) {
    constexpr int SL = 1 << T;          // local stride
    constexpr int ML = R >> (T + 1);    // local "mid"
    constexpr int BASE = (1 << (LS0 + T)) - 1;
#pragma unroll
    for (int jl = 0; jl < SL; ++jl) {
        if (LS0 == 0 && jl == 0) {                                     // twiddle (1,0), known at compile time
#pragma unroll
            for (int il = 0; il < ML; ++il)
                butterfly_unit(in[SL * il + jl], in[SL * (il + ML) + jl], out[SL * 2 * il + jl], out[SL * (2 * il + 1) + jl]);
        } else {
            float2 tw;
            if (LS0 == 0) tw = c_twiddles[BASE + jl];                  // warp-uniform: constant bank
            else tw = tw_g[BASE + j + (jl << LS0)];                    // table copy in shared memory
#pragma unroll
            for (int il = 0; il < ML; ++il)
                butterfly(in[SL * il + jl], in[SL * (il + ML) + jl], tw, out[SL * 2 * il + jl], out[SL * (2 * il + 1) + jl]);
        }
    }
}

template <int R, int LS0>
__device__ __forceinline__ void radix_pass(C2 (&v)[R], int j, const float2* __restrict__ tw_g) {
    static_assert(R == 2 || R == 4 || R == 8 || R == 16, "radix");
    C2 w[R];
    stockham_stage<R, 0, LS0>(v, w, j, tw_g);
    if (R == 2) {
#pragma unroll
        for (int i = 0; i < R; ++i) v[i] = w[i];
        return;
    }
    if (R >= 4) stockham_stage<R, (R >= 4 ? 1 : 0), LS0>(w, v, j, tw_g);
    if (R == 4) return;
    if (R >= 8) stockham_stage<R, (R >= 8 ? 2 : 0), LS0>(v, w, j, tw_g);
    if (R == 8) {
#pragma unroll
        for (int i = 0; i < R; ++i) v[i] = w[i];
        return;
    }
    if (R >= 16) stockham_stage<R, (R >= 16 ? 3 : 0), LS0>(w, v, j, tw_g);
}

// FFT plans: radices of the register passes (product = N, each <= 16).
template <int N> struct Plan;
template <> struct Plan<128>  { static constexpr int NP = 2; static constexpr int R0 = 16, R1 = 8,  R2 = 1; };
template <> struct Plan<256>  { static constexpr int NP = 2; static constexpr int R0 = 16, R1 = 16, R2 = 1; };
template <> struct Plan<512>  { static constexpr int NP = 3; static constexpr int R0 = 16, R1 = 16, R2 = 2; };
template <> struct Plan<1024> { static constexpr int NP = 3; static constexpr int R0 = 16, R1 = 16, R2 = 4; };

constexpr int kE = 16;                                    // elements per thread per layer pair
__host__ __device__ constexpr int ilog2(int v) { return v <= 1 ? 0 : 1 + ilog2(v >> 1); }
__device__ __forceinline__ int pad16(int idx) { return idx + (idx >> 4); }

// pad16(x + c) == pad16(x) + pad16(c) whenever x or c is a multiple of 16.  The passes below split a padded index into the
// thread's part, computed once, and a compile-time part, so that every element is an immediate offset from one address.
// Loads the kE elements a thread owns in a pass of radix R from a (padded) shared buffer:
// group g = t + TT*u, element a of the group sits at natural index a*(N/R) + g.
template <int N, int R>
__device__ __forceinline__ void pass_load(C2 (&v)[kE], const float4* __restrict__ buf, int t) {
    constexpr int TT = N / kE;
    constexpr bool SPLIT = (N / R) % 16 == 0 && TT % 16 == 0;     // a*(N/R) + TT*u is a multiple of 16
    const float4* base = SPLIT ? buf + pad16(t) : buf;
#pragma unroll
    for (int u = 0; u < kE / R; ++u)
#pragma unroll
        for (int a = 0; a < R; ++a)
            v[u * R + a] = c2_from(SPLIT ? base[pad16(a * (N / R) + TT * u)] : buf[pad16(a * (N / R) + t + TT * u)]);
}
// Natural index of output b of group g after a pass of radix R that started at stride 2^LS0.
template <int R, int LS0>
__device__ __forceinline__ int out_index(int g, int b) {
    return ((g >> LS0) << (LS0 + ilog2(R))) + (b << LS0) + (g & ((1 << LS0) - 1));
}
template <int N, int R, int LS0>
__device__ __forceinline__ void pass_compute(C2 (&v)[kE], int t, const float2* __restrict__ tw_g) {
    constexpr int TT = N / kE;
#pragma unroll
    for (int u = 0; u < kE / R; ++u) {
        const int g = t + TT * u;
        radix_pass<R, LS0>(reinterpret_cast<C2(&)[R]>(v[u * R]), g & ((1 << LS0) - 1), tw_g);
    }
}
template <int N, int R, int LS0>
__device__ __forceinline__ void pass_store(const C2 (&v)[kE], float4* __restrict__ buf, int t) {
    constexpr int TT = N / kE;
    // with TT a multiple of 2^LS0, out_index(t + TT*u, b) = out_index(t, 0) + TT*u*R + (b << LS0); the thread's part is a multiple
    // of 16 when LS0 == 0 and R == 16, the element part when LS0 >= 4
    constexpr bool SPLIT = TT % (1 << LS0) == 0 && ((LS0 == 0 && R % 16 == 0) || (LS0 >= 4 && (TT * R) % 16 == 0));
    float4* base = SPLIT ? buf + pad16(out_index<R, LS0>(t, 0)) : buf;
#pragma unroll
    for (int u = 0; u < kE / R; ++u)
#pragma unroll
        for (int b = 0; b < R; ++b) {
            if (SPLIT) base[pad16(TT * u * R + (b << LS0))] = c2_to(v[u * R + b]);
            else buf[pad16(out_index<R, LS0>(t + TT * u, b))] = c2_to(v[u * R + b]);
        }
}
// Natural output index of register slot i (= u*RL + b) after the last pass, for 0 <= t < TT.  The group g = t + TT*u is below
// TT * kE/RL = 2^LSL, so out_index<RL, LSL>(g, b) = g + (b << LSL): the thread's t plus a compile-time offset.
template <int N>
__device__ __forceinline__ int final_index(int t, int i) {
    using P = Plan<N>;
    constexpr int TT = N / kE;
    constexpr int RL = P::NP == 3 ? P::R2 : P::R1;
    constexpr int LSL = ilog2(N) - ilog2(RL);
    static_assert(TT * (kE / RL) == (1 << LSL), "groups of the last pass");
    return out_index<RL, LSL>(t + TT * (i / RL), i % RL);
}

// For 0 <= t < TT the group g = t + TT*u of the last pass is below TT * kE/RL = 2^LSL, so final_index(t, i) = t + final_offset(i):
// stores of the final outputs are compile-time offsets from the thread's first output.
template <int N>
__device__ __forceinline__ constexpr int final_offset(int i) {
    using P = Plan<N>;
    constexpr int TT = N / kE;
    constexpr int RL = P::NP == 3 ? P::R2 : P::R1;
    constexpr int LSL = ilog2(N) - ilog2(RL);
    static_assert(TT * (kE / RL) == (1 << LSL), "groups of the last pass");
    return TT * (i / RL) + ((i % RL) << LSL);
}

// Barrier among the N/16 threads that share one FFT's exchange buffer: they sit in one warp when
// N <= 512 (consecutive lanes), otherwise the whole CTA synchronises.
template <int N>
__device__ __forceinline__ void fft_group_sync() {
    if (N / kE <= 32) __syncwarp();
    else __syncthreads();
}

// Passes 1.. of an FFT whose pass 0 has been computed in registers (outputs in v), exchanging
// through `buf`, which only the N/16 threads of this FFT touch.  On return v holds the final outputs
// (slot i -> natural index final_index<N>(t, i)).
template <int N>
__device__ __forceinline__ void remaining_passes(C2 (&v)[kE], float4* __restrict__ buf, int t, const float2* __restrict__ tw_g) {
    using P = Plan<N>;
    constexpr int LS1 = ilog2(P::R0);
    pass_store<N, P::R0, 0>(v, buf, t);
    fft_group_sync<N>();
    pass_load<N, P::R1>(v, buf, t);
    pass_compute<N, P::R1, LS1>(v, t, tw_g);
    if (P::NP == 3) {
        constexpr int LS2 = LS1 + ilog2(P::R1);
        constexpr int R2 = P::R2 > 1 ? P::R2 : 2;
        fft_group_sync<N>();
        pass_store<N, P::R1, LS1>(v, buf, t);
        fft_group_sync<N>();
        pass_load<N, R2>(v, buf, t);
        pass_compute<N, R2, LS2>(v, t, tw_g);
    }
}

}  // namespace ocean
