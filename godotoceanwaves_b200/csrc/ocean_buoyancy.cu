// ocean_buoyancy.cu -- per-body hydrostatic force and torque from hull sample points on the displaced surface
// (ocean_buoyancy; oracle/buoyancy.py is the specification).
//
// A call runs three steps on the generator's stream:
//   k_buoyancy_transform  one thread per world point (body-major; the host's exclusive prefix of num_points gives each body
//                         its start, a binary search over it gives a thread its body): r = R p, w = r + t, Q = (w.x, w.z)
//   launch_query_surface  the surface query (ocean_sample.cu), unchanged, on those Q
//   k_buoyancy_reduce     one warp per body, lane l takes j = l, l + 32, ...: recomputes r from the body and the hull point
//                         (the same operations, so the same bits), reads the height and the residual from the record and
//                         sums v, v r.x, v r.y, v r.z in the specification's order -- each lane from +0 in increasing j, then
//                         __shfl_down_sync with offsets 16, 8, 4, 2, 1 -- and lane 0 writes the body's record.
// No shared memory and no atomics: a body of any size is a longer lane loop, and the result does not depend on the schedule.
//
// The body-forces op (ocean_body_forces; oracle/drag.py is the specification) runs the same three steps and then
//   k_drag_reduce         one warp per body in the same lane order: recomputes r and f as k_buoyancy_reduce does; for a
//                         submerged point (f > 0) gathers the velocity maps at the record's source point (4 texels per
//                         cascade), and sums the quadratic drag force, its torque about the body origin and f * C_d A.
//   k_drag_reduce_wake    the same with the wake layer's vertical velocity per world point added to the water velocity
//                         (ocean_wake_set_coupling); both kernels are one inlined template, k_drag_reduce its uncoupled form.
// Numeric policy: binary32, the specification's operation order, no contraction (-fmad=false).
#include "../../include/ocean.h"
#include "ocean_kernels.cuh"
#include "ocean_texture.cuh"

namespace ocean {

namespace {

// r = R p of the specification: ((R[k][0] p.x + R[k][1] p.y) + R[k][2] p.z), row k of the 3 x 4 row-major transform
__device__ __forceinline__ float3 rotate(const float* __restrict__ T, const float* __restrict__ p) {
    float3 r;
    r.x = (T[0] * p[0] + T[1] * p[1]) + T[2] * p[2];
    r.y = (T[4] * p[0] + T[5] * p[1]) + T[6] * p[2];
    r.z = (T[8] * p[0] + T[9] * p[1]) + T[10] * p[2];
    return r;
}

// f of the specification: the submerged fraction of a column of half height h centred at height wy, under water height eta
__device__ __forceinline__ float submerged_fraction(float eta, float wy, float h) {
    return h > 0.0f ? fminf(fmaxf(__fdiv_rn(eta - (wy - h), h + h), 0.0f), 1.0f) : (wy <= eta ? 1.0f : 0.0f);
}

__global__ void __launch_bounds__(256) k_buoyancy_transform(const ocean_buoyancy_body* __restrict__ bodies, const int* __restrict__ offsets,
                                                            int num_bodies, const ocean_buoyancy_point* __restrict__ points, int n,
                                                            float2* __restrict__ q) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int lo = 0, hi = num_bodies - 1;              // the last body whose start is <= i (it has points: the next start is > i)
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(&offsets[mid]) <= i) lo = mid; else hi = mid - 1;
    }
    const ocean_buoyancy_body& b = bodies[lo];
    const ocean_buoyancy_point& p = points[b.first_point + (i - __ldg(&offsets[lo]))];
    const float3 r = rotate(b.transform, p.position);
    q[i] = make_float2(r.x + b.transform[3], r.z + b.transform[11]);
}

__global__ void __launch_bounds__(256) k_buoyancy_reduce(const ocean_buoyancy_body* __restrict__ bodies, const int* __restrict__ offsets,
                                                         int num_bodies, const ocean_buoyancy_point* __restrict__ points,
                                                         const ocean_surface_sample* __restrict__ samples, float rho_g, float tol,
                                                         ocean_buoyancy_result* __restrict__ out) {
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (warp >= (size_t)num_bodies) return;        // whole warps: the shuffles below see all 32 lanes
    const int body = (int)warp;
    const int lane = threadIdx.x & 31;
    const ocean_buoyancy_body& b = bodies[body];
    const int count = b.num_points;
    if (count == 0) {
        if (lane == 0) out[body] = ocean_buoyancy_result{};
        return;
    }
    const ocean_buoyancy_point* hull = points + b.first_point;
    const ocean_surface_sample* rec = samples + offsets[body];
    const float ty = b.transform[7];
    float s0 = 0.0f, sx = 0.0f, sy = 0.0f, sz = 0.0f, max_res = __int_as_float(0x7fffffff);
    unsigned missed = 0;
    for (int j = lane; j < count; j += 32) {
        const float3 r = rotate(b.transform, hull[j].position);
        const float wy = r.y + ty;
        const float h = hull[j].half_height;
        const float eta = rec[j].displacement[1];
        const float res = rec[j].residual;
        const float f = submerged_fraction(eta, wy, h);
        const float v = f * hull[j].volume;
        s0 = s0 + v;
        sx = sx + v * r.x;
        sy = sy + v * r.y;
        sz = sz + v * r.z;
        max_res = fmaxf(max_res, res);
        missed += !(res <= tol);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {              // p[l] = p[l] + p[l + o]: the specification's tree
        s0 = s0 + __shfl_down_sync(0xffffffffu, s0, o);
        sx = sx + __shfl_down_sync(0xffffffffu, sx, o);
        sy = sy + __shfl_down_sync(0xffffffffu, sy, o);
        sz = sz + __shfl_down_sync(0xffffffffu, sz, o);
        max_res = fmaxf(max_res, __shfl_down_sync(0xffffffffu, max_res, o));
        missed += __shfl_down_sync(0xffffffffu, missed, o);
    }
    if (lane != 0) return;
    ocean_buoyancy_result o;
    o.force[0] = 0.0f;
    o.force[1] = rho_g * s0;
    o.force[2] = 0.0f;
    o.torque[0] = -(rho_g * sz);
    o.torque[1] = 0.0f;
    o.torque[2] = rho_g * sx;
    o.submerged_volume = s0;
    const bool pos = s0 > 0.0f;
    o.center_offset[0] = pos ? __fdiv_rn(sx, s0) : 0.0f;
    o.center_offset[1] = pos ? __fdiv_rn(sy, s0) : 0.0f;
    o.center_offset[2] = pos ? __fdiv_rn(sz, s0) : 0.0f;
    o.max_residual = max_res;
    o.unconverged = missed;
    out[body] = o;
}

// d = u - (v + w x r) per submerged point, F = ((f * cda) * |d|) d, T = r x F; per body half_rho * sum F, half_rho * sum T,
// sum f * cda and the NaN-dropping max of |d| (from 0), each summed in k_buoyancy_reduce's order.  With kWake, u.y also gets
// the wake layer's vertical velocity wv of the world point.
template <bool kWake>
__device__ __forceinline__ void drag_reduce(const ocean_buoyancy_body* __restrict__ bodies, const ocean_body_velocity* __restrict__ velocities,
                                            const int* __restrict__ offsets, int num_bodies, const ocean_buoyancy_point* __restrict__ points,
                                            const float* __restrict__ drag_areas, const ocean_surface_sample* __restrict__ samples,
                                            const uint2* __restrict__ velocity, int N, int C, const float4* __restrict__ scales,
                                            float half_rho, ocean_drag_result* __restrict__ out, const float* __restrict__ wv) {
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (warp >= (size_t)num_bodies) return;        // whole warps: the shuffles below see all 32 lanes
    const int body = (int)warp;
    const int lane = threadIdx.x & 31;
    const ocean_buoyancy_body& b = bodies[body];
    const int count = b.num_points;
    if (count == 0) {
        if (lane == 0) out[body] = ocean_drag_result{};
        return;
    }
    const ocean_buoyancy_point* hull = points + b.first_point;
    const float* cda = drag_areas + b.first_point;
    const ocean_surface_sample* rec = samples + offsets[body];
    const float* wake = kWake ? wv + offsets[body] : nullptr;
    const ocean_body_velocity bv = velocities[body];
    const float ty = b.transform[7];
    float sfx = 0.0f, sfy = 0.0f, sfz = 0.0f, stx = 0.0f, sty = 0.0f, stz = 0.0f, sa = 0.0f, max_s = 0.0f;
    for (int j = lane; j < count; j += 32) {
        const float3 r = rotate(b.transform, hull[j].position);
        const float f = submerged_fraction(rec[j].displacement[1], r.y + ty, hull[j].half_height);
        if (!(f > 0.0f)) continue;                  // a dry point gathers nothing and adds nothing
        const float px = rec[j].source_x, pz = rec[j].source_z;
        float ux = 0.0f, uy = 0.0f, uz = 0.0f;
        for (int c = 0; c < C; ++c) {
            const float4 s = __ldg(&scales[c]);
            add_displacement(velocity + (size_t)c * N * N, N, px * s.x, pz * s.y, s.z, ux, uy, uz);
        }
        if constexpr (kWake) uy = uy + __ldg(&wake[j]);
        const float dx = ux - (bv.linear[0] + (bv.angular[1] * r.z - bv.angular[2] * r.y));
        const float dy = uy - (bv.linear[1] + (bv.angular[2] * r.x - bv.angular[0] * r.z));
        const float dz = uz - (bv.linear[2] + (bv.angular[0] * r.y - bv.angular[1] * r.x));
        const float speed = __fsqrt_rn((dx * dx + dy * dy) + dz * dz);
        const float a = f * __ldg(&cda[j]);
        const float k = a * speed;
        const float Fx = k * dx, Fy = k * dy, Fz = k * dz;
        sfx = sfx + Fx;
        sfy = sfy + Fy;
        sfz = sfz + Fz;
        stx = stx + (r.y * Fz - r.z * Fy);
        sty = sty + (r.z * Fx - r.x * Fz);
        stz = stz + (r.x * Fy - r.y * Fx);
        sa = sa + a;
        max_s = fmaxf(max_s, speed);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {              // p[l] = p[l] + p[l + o]: the specification's tree
        sfx = sfx + __shfl_down_sync(0xffffffffu, sfx, o);
        sfy = sfy + __shfl_down_sync(0xffffffffu, sfy, o);
        sfz = sfz + __shfl_down_sync(0xffffffffu, sfz, o);
        stx = stx + __shfl_down_sync(0xffffffffu, stx, o);
        sty = sty + __shfl_down_sync(0xffffffffu, sty, o);
        stz = stz + __shfl_down_sync(0xffffffffu, stz, o);
        sa = sa + __shfl_down_sync(0xffffffffu, sa, o);
        max_s = fmaxf(max_s, __shfl_down_sync(0xffffffffu, max_s, o));
    }
    if (lane != 0) return;
    ocean_drag_result o;
    o.force[0] = half_rho * sfx;
    o.force[1] = half_rho * sfy;
    o.force[2] = half_rho * sfz;
    o.torque[0] = half_rho * stx;
    o.torque[1] = half_rho * sty;
    o.torque[2] = half_rho * stz;
    o.wetted_drag_area = sa;
    o.max_relative_speed = max_s;
    out[body] = o;
}


__global__ void __launch_bounds__(256) k_drag_reduce(const ocean_buoyancy_body* __restrict__ bodies, const ocean_body_velocity* __restrict__ velocities,
                                                     const int* __restrict__ offsets, int num_bodies, const ocean_buoyancy_point* __restrict__ points,
                                                     const float* __restrict__ drag_areas, const ocean_surface_sample* __restrict__ samples,
                                                     const uint2* __restrict__ velocity, int N, int C, const float4* __restrict__ scales,
                                                     float half_rho, ocean_drag_result* __restrict__ out) {
    drag_reduce<false>(bodies, velocities, offsets, num_bodies, points, drag_areas, samples, velocity, N, C, scales, half_rho, out, nullptr);
}

// k_drag_reduce with the wake layer's vertical velocity per world point (ocean_wake_set_coupling)
__global__ void __launch_bounds__(256) k_drag_reduce_wake(const ocean_buoyancy_body* __restrict__ bodies,
                                                          const ocean_body_velocity* __restrict__ velocities, const int* __restrict__ offsets,
                                                          int num_bodies, const ocean_buoyancy_point* __restrict__ points,
                                                          const float* __restrict__ drag_areas, const ocean_surface_sample* __restrict__ samples,
                                                          const uint2* __restrict__ velocity, int N, int C, const float4* __restrict__ scales,
                                                          float half_rho, ocean_drag_result* __restrict__ out, const float* __restrict__ wv) {
    drag_reduce<true>(bodies, velocities, offsets, num_bodies, points, drag_areas, samples, velocity, N, C, scales, half_rho, out, wv);
}

}  // namespace

cudaError_t launch_buoyancy_transform(const ocean_buoyancy_body* bodies_dev, const int* offsets_dev, int num_bodies,
                                      const ocean_buoyancy_point* points_dev, int n, float2* q_dev, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    k_buoyancy_transform<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(bodies_dev, offsets_dev, num_bodies, points_dev, n, q_dev);
    return cudaGetLastError();
}

cudaError_t launch_buoyancy_reduce(const ocean_buoyancy_body* bodies_dev, const int* offsets_dev, int num_bodies,
                                   const ocean_buoyancy_point* points_dev, const ocean_surface_sample* samples_dev, float rho_g,
                                   float tolerance, ocean_buoyancy_result* results_dev, cudaStream_t stream) {
    if (num_bodies <= 0) return cudaSuccess;
    const unsigned blocks = (unsigned)(((size_t)num_bodies * 32 + 255) / 256);      // 8 bodies per block
    k_buoyancy_reduce<<<blocks, 256, 0, stream>>>(bodies_dev, offsets_dev, num_bodies, points_dev, samples_dev, rho_g, tolerance, results_dev);
    return cudaGetLastError();
}

cudaError_t launch_drag_reduce(const ocean_buoyancy_body* bodies_dev, const ocean_body_velocity* velocities_dev, const int* offsets_dev,
                               int num_bodies, const ocean_buoyancy_point* points_dev, const float* drag_areas_dev,
                               const ocean_surface_sample* samples_dev, const uint2* velocity_dev, int map_size, int num_cascades,
                               const float4* scales_dev, float half_rho, ocean_drag_result* results_dev, const float* wake_wv_dev,
                               cudaStream_t stream) {
    if (num_bodies <= 0) return cudaSuccess;
    const unsigned blocks = (unsigned)(((size_t)num_bodies * 32 + 255) / 256);      // 8 bodies per block
    if (wake_wv_dev)
        k_drag_reduce_wake<<<blocks, 256, 0, stream>>>(bodies_dev, velocities_dev, offsets_dev, num_bodies, points_dev, drag_areas_dev,
                                                       samples_dev, velocity_dev, map_size, num_cascades, scales_dev, half_rho, results_dev,
                                                       wake_wv_dev);
    else
        k_drag_reduce<<<blocks, 256, 0, stream>>>(bodies_dev, velocities_dev, offsets_dev, num_bodies, points_dev, drag_areas_dev, samples_dev,
                                                  velocity_dev, map_size, num_cascades, scales_dev, half_rho, results_dev);
    return cudaGetLastError();
}

}  // namespace ocean
