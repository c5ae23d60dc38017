// wake_sample.cuh -- the wake layer's bilinear sample (oracle/wake.py sample(), ocean_sample_wake), shared by the wake kernels
// (ocean_wake.cu) and the ops that read the layer: the ray cast (ocean_sample.cu) and spray (ocean_spray.cu).
// Numeric policy: binary32 in the specification's order with explicit _rn operations, no contraction.
#pragma once
#include <cuda_runtime.h>

namespace ocean {

// h at window cell (i, j) of the field f ([n][n]), 0 outside
__device__ __forceinline__ float cell(const float* __restrict__ f, int n, int i, int j) {
    return (unsigned)i < (unsigned)n && (unsigned)j < (unsigned)n ? f[(size_t)j * n + i] : 0.0f;
}

__device__ __forceinline__ float grad_x(const float* __restrict__ h, int n, int i, int j, float two_dx) {
    return __fdiv_rn(__fsub_rn(cell(h, n, i + 1, j), cell(h, n, i - 1, j)), two_dx);
}
__device__ __forceinline__ float grad_z(const float* __restrict__ h, int n, int i, int j, float two_dx) {
    return __fdiv_rn(__fsub_rn(cell(h, n, i, j + 1), cell(h, n, i, j - 1)), two_dx);
}

__device__ __forceinline__ float bilerp(float f00, float f10, float f01, float f11, float fu, float fv) {
    const float top = __fadd_rn(f00, __fmul_rn(fu, __fsub_rn(f10, f00)));
    const float bot = __fadd_rn(f01, __fmul_rn(fu, __fsub_rn(f11, f01)));
    return __fadd_rn(top, __fmul_rn(fv, __fsub_rn(bot, top)));
}

// oracle/wake.py sample() of the field h at world point p: r[0] = bilinear h and, with kGradients, r[1], r[2] = bilinear
// central differences; r is left as it is (the caller's zeros) outside the window
template <bool kGradients>
__device__ __forceinline__ void sample_field(const float* __restrict__ h, int n, float dx, float x0, float z0, float2 p, float* r) {
    const float ext = __fmul_rn((float)n, dx);
    if (p.x >= x0 && p.x < __fadd_rn(x0, ext) && p.y >= z0 && p.y < __fadd_rn(z0, ext)) {
        const float u = __fsub_rn(__fdiv_rn(__fsub_rn(p.x, x0), dx), 0.5f);
        const float v = __fsub_rn(__fdiv_rn(__fsub_rn(p.y, z0), dx), 0.5f);
        const float fi = floorf(u), fj = floorf(v);
        const float fu = __fsub_rn(u, fi), fv = __fsub_rn(v, fj);
        const int i = (int)fi, j = (int)fj;
        const float two_dx = __fmul_rn(2.0f, dx);
        r[0] = bilerp(cell(h, n, i, j), cell(h, n, i + 1, j), cell(h, n, i, j + 1), cell(h, n, i + 1, j + 1), fu, fv);
        if constexpr (kGradients) {
            // central differences of cells outside the window are 0, like their heights
            auto gx = [&](int ii, int jj) { return (unsigned)ii < (unsigned)n && (unsigned)jj < (unsigned)n ? grad_x(h, n, ii, jj, two_dx) : 0.0f; };
            auto gz = [&](int ii, int jj) { return (unsigned)ii < (unsigned)n && (unsigned)jj < (unsigned)n ? grad_z(h, n, ii, jj, two_dx) : 0.0f; };
            r[1] = bilerp(gx(i, j), gx(i + 1, j), gx(i, j + 1), gx(i + 1, j + 1), fu, fv);
            r[2] = bilerp(gz(i, j), gz(i + 1, j), gz(i, j + 1), gz(i + 1, j + 1), fu, fv);
        }
    }
}

}  // namespace ocean
