// ocean_texture.cuh -- texture() of the reference's spatial shaders on the generator's RGBA16F maps: exact-weight bilinear
// filter with REPEAT addressing, binary32, round to nearest, no contraction (oracle/sampling.py is the specification).
// Shared by the map-query, surface-query and velocity-query ops (ocean_sample.cu), the spray-candidate op (ocean_spray.cu),
// the drag reduction of the body-forces op (ocean_buoyancy.cu) and the drifters (ocean_drift.cu); sample_point is the
// water shader's whole sampling contract at one point (water.gdshader:27-39,42-84).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace ocean {
namespace {

__device__ __forceinline__ float4 texel(const uint2* __restrict__ layer, int N, int x, int y) {
    const uint2 t = __ldg(&layer[(size_t)y * N + x]);
    const __half2 lo = *reinterpret_cast<const __half2*>(&t.x), hi = *reinterpret_cast<const __half2*>(&t.y);
    const float2 a = __half22float2(lo), b = __half22float2(hi);
    return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float mixf(float a, float b, float t) { return a * (1.0f - t) + b * t; }   // GLSL mix
__device__ __forceinline__ float4 mix4(const float4 a, const float4 b, float t) {
    return make_float4(mixf(a.x, b.x, t), mixf(a.y, b.y, t), mixf(a.z, b.z, t), mixf(a.w, b.w, t));
}

// REPEAT texel index of floor(x): x0 mod N.  N is a power of two (128..1024), so the wrap is a mask.  The conversion to
// int64 saturates beyond +-2^63, so x0 is clamped to [-2^62, 2^62] first; that is exact, because every binary32 of
// magnitude >= 2^62 is a multiple of 2^39, hence of N, and so is 2^62.  fmaxf sends NaN to -2^62, i.e. to texel 0.
__device__ __forceinline__ int wrap_texel(float x0, int N) {
    return (int)(long long)fminf(fmaxf(x0, -0x1p62f), 0x1p62f) & (N - 1);
}

// texture(): bilinear, REPEAT.
__device__ __forceinline__ float4 texture_bilinear(const uint2* __restrict__ layer, int N, float u, float v) {
    const float n = (float)N;
    const float x = u * n - 0.5f, y = v * n - 0.5f;
    const float x0 = floorf(x), y0 = floorf(y);
    const float fx = x - x0, fy = y - y0;
    const int ix0 = wrap_texel(x0, N), iy0 = wrap_texel(y0, N);
    const int ix1 = (ix0 + 1) & (N - 1), iy1 = (iy0 + 1) & (N - 1);
    const float4 t00 = texel(layer, N, ix0, iy0), t10 = texel(layer, N, ix1, iy0);
    const float4 t01 = texel(layer, N, ix0, iy1), t11 = texel(layer, N, ix1, iy1);
    return mix4(mix4(t00, t10, fx), mix4(t01, t11, fx), fy);
}

// texture() plus the exact derivatives of the bilinear interpolant with respect to u and v, from the same four texels
// (oracle/surface.py, bilinear_slopes): d/du = mix(t10 - t00, t11 - t01, fy) * N, d/dv = mix(t01 - t00, t11 - t10, fx) * N.
// The value is computed operation for operation as texture_bilinear computes it.
__device__ __forceinline__ float4 texture_bilinear_slopes(const uint2* __restrict__ layer, int N, float u, float v, float4& du, float4& dv) {
    const float n = (float)N;
    const float x = u * n - 0.5f, y = v * n - 0.5f;
    const float x0 = floorf(x), y0 = floorf(y);
    const float fx = x - x0, fy = y - y0;
    const int ix0 = wrap_texel(x0, N), iy0 = wrap_texel(y0, N);
    const int ix1 = (ix0 + 1) & (N - 1), iy1 = (iy0 + 1) & (N - 1);
    const float4 t00 = texel(layer, N, ix0, iy0), t10 = texel(layer, N, ix1, iy0);
    const float4 t01 = texel(layer, N, ix0, iy1), t11 = texel(layer, N, ix1, iy1);
    const float4 a = make_float4(t10.x - t00.x, t10.y - t00.y, t10.z - t00.z, t10.w - t00.w);
    const float4 b = make_float4(t11.x - t01.x, t11.y - t01.y, t11.z - t01.z, t11.w - t01.w);
    const float4 c = make_float4(t01.x - t00.x, t01.y - t00.y, t01.z - t00.z, t01.w - t00.w);
    const float4 d = make_float4(t11.x - t10.x, t11.y - t10.y, t11.z - t10.z, t11.w - t10.w);
    const float4 su = mix4(a, b, fy), sv = mix4(c, d, fx);
    du = make_float4(su.x * n, su.y * n, su.z * n, su.w * n);
    dv = make_float4(sv.x * n, sv.y * n, sv.z * n, sv.w * n);
    return mix4(mix4(t00, t10, fx), mix4(t01, t11, fx), fy);
}

// Cascade c's term of the displacement sum of the water shader's vertex() (water.gdshader:34-35), added to (dx, dy, dz).
// On the velocity maps (v = dD/dt, so the displacement scale applies) it is the cascade's term of the water velocity.
__device__ __forceinline__ void add_displacement(const uint2* __restrict__ layer, int N, float u, float v, float scale, float& dx, float& dy,
                                                 float& dz) {
    const float4 d = texture_bilinear(layer, N, u, v);
    dx = dx + d.x * scale;
    dy = dy + d.y * scale;
    dz = dz + d.z * scale;
}

// water.gdshader:42-51
__device__ __forceinline__ void cubic_weights(float a, float (&w)[4]) {
    const float a2 = a * a, a3 = a2 * a;
    w[0] = (-a3 + a2 * 3.0f - a * 3.0f + 1.0f) / 6.0f;
    w[1] = (a3 * 3.0f - a2 * 6.0f + 4.0f) / 6.0f;
    w[2] = (-a3 * 3.0f + a2 * 3.0f + a * 3.0f + 1.0f) / 6.0f;
    w[3] = a3 / 6.0f;
}

// water.gdshader:55-70
__device__ __forceinline__ float4 texture_bicubic(const uint2* __restrict__ layer, int N, float u, float v) {
    const float dims = (float)N, dims_inv = 1.0f / dims;
    const float ux = u * dims + 0.5f, vy = v * dims + 0.5f;
    const float flx = floorf(ux), fly = floorf(vy);
    float wx[4], wy[4];
    cubic_weights(ux - flx, wx);
    cubic_weights(vy - fly, wy);
    const float gx = wx[0] + wx[1], gy = wx[2] + wx[3], gz = wy[0] + wy[1], gw = wy[2] + wy[3];
    const float hx = (wx[1] / gx + -1.5f + flx) * dims_inv;
    const float hy = (wx[3] / gy + 0.5f + flx) * dims_inv;
    const float hz = (wy[1] / gz + -1.5f + fly) * dims_inv;
    const float hw = (wy[3] / gw + 0.5f + fly) * dims_inv;
    const float wxx = gx / (gx + gy), wyy = gz / (gz + gw);
    return mix4(mix4(texture_bilinear(layer, N, hy, hw), texture_bilinear(layer, N, hx, hw), wxx),
                mix4(texture_bilinear(layer, N, hy, hz), texture_bilinear(layer, N, hx, hz), wxx), wyy);
}

// The sampling contract at one point p: displacement (vertex(), :27-39) and gradient/foam (fragment(), :72-84).
__device__ __forceinline__ void sample_point(const uint2* __restrict__ displacement, const uint2* __restrict__ normal, int N, int C, float2 p,
                                             const float4* __restrict__ scales, float3& disp, float3& grad) {
    float dx = 0.0f, dy = 0.0f, dz = 0.0f, gx = 0.0f, gy = 0.0f, gf = 0.0f;
    for (int c = 0; c < C; ++c) {
        const float4 s = __ldg(&scales[c]);
        const float u = p.x * s.x, v = p.y * s.y;
        const size_t layer = (size_t)c * N * N;
        add_displacement(displacement + layer, N, u, v, s.z, dx, dy, dz);                           // :34-35
        const float ppm = (float)N * fminf(s.x, s.y);                                             // :80
        const float t = fminf(1.0f, ppm * 0.1f);
        const float4 m = mix4(texture_bicubic(normal + layer, N, u, v), texture_bilinear(normal + layer, N, u, v), t);   // :83
        gx = gx + m.x * s.w;
        gy = gy + m.y * s.w;
        gf = gf + m.w * 1.0f;
    }
    disp = make_float3(dx, dy, dz);
    grad = make_float3(gx, gy, gf);
}

}  // namespace
}  // namespace ocean
