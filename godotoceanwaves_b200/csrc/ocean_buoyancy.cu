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
// Numeric policy: binary32, the specification's operation order, no contraction (-fmad=false).
#include "../../include/ocean.h"
#include "ocean_kernels.cuh"

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
        const float f = h > 0.0f ? fminf(fmaxf(__fdiv_rn(eta - (wy - h), h + h), 0.0f), 1.0f) : (wy <= eta ? 1.0f : 0.0f);
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

}  // namespace

cudaError_t launch_buoyancy_transform(const void* bodies_dev, const int* offsets_dev, int num_bodies, const void* points_dev, int n,
                                      float2* q_dev, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    k_buoyancy_transform<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(static_cast<const ocean_buoyancy_body*>(bodies_dev), offsets_dev,
                                                                         num_bodies, static_cast<const ocean_buoyancy_point*>(points_dev), n, q_dev);
    return cudaGetLastError();
}

cudaError_t launch_buoyancy_reduce(const void* bodies_dev, const int* offsets_dev, int num_bodies, const void* points_dev,
                                   const void* samples_dev, float rho_g, float tolerance, void* results_dev, cudaStream_t stream) {
    if (num_bodies <= 0) return cudaSuccess;
    const unsigned blocks = (unsigned)(((size_t)num_bodies * 32 + 255) / 256);      // 8 bodies per block
    k_buoyancy_reduce<<<blocks, 256, 0, stream>>>(static_cast<const ocean_buoyancy_body*>(bodies_dev), offsets_dev, num_bodies,
                                                  static_cast<const ocean_buoyancy_point*>(points_dev),
                                                  static_cast<const ocean_surface_sample*>(samples_dev), rho_g, tolerance,
                                                  static_cast<ocean_buoyancy_result*>(results_dev));
    return cudaGetLastError();
}

}  // namespace ocean
