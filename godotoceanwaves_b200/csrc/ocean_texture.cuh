// ocean_texture.cuh -- texture() of the reference's spatial shaders on the generator's RGBA16F maps: exact-weight bilinear
// filter with REPEAT addressing, binary32, round to nearest, no contraction (oracle/sampling.py is the specification).
// Shared by the map-query, surface-query and velocity-query ops (ocean_sample.cu), the spray-candidate op (ocean_spray.cu)
// and the drag reduction of the body-forces op (ocean_buoyancy.cu).
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

}  // namespace
}  // namespace ocean
