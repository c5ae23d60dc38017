// ocean_bodies.cu -- the floating-body integrator (ocean_simulate_bodies; oracle/bodies.py is the specification): the body
// state stays on the device, and every sub-step runs the body-forces sequence of ocean_buoyancy.cu unchanged on pose and
// velocity tables these kernels write.
//
// A call runs, on the generator's stream:
//   k_bodies_prepare     one warp per body: r2 = the NaN-dropping max of |p|^2 over the body's hull points (lanes, then the
//                        shuffle tree; max is exact, so the order does not matter), and the first sub-step's pose table
//                        (ocean_buoyancy_body: [R(q) | position], the range) and velocity table (ocean_body_velocity)
//   then per sub-step    k_buoyancy_transform, the surface query, k_buoyancy_reduce, k_drag_reduce (unchanged), and
//   k_bodies_integrate   one thread per body: the semi-implicit step of the specification from the state, the pose the
//                        sub-step started from and its two records; writes the new state, the next sub-step's pose and
//                        velocity rows, and on the last sub-step the 3 x 4 transform of the final state when asked to.
// ocean_simulate_hull_bodies (ocean_hull.cu) runs k_hull_prepare, the same prepare over a hull mesh's vertices, in place of
// k_bodies_prepare, and k_bodies_integrate on pose rows of ocean_hull_body (ocean_buoyancy_body's layout).
// ocean_simulate_driven_bodies runs k_bodies_integrate_driven instead, the same step on the forces and denominators of
// ocean_drive.cu's reduce (both are forms of one inlined template).
// Nothing crosses PCIe between sub-steps.  Numeric policy: binary32, the specification's operation order, no contraction
// (-fmad=false), IEEE division and square root.
#include "../../include/ocean.h"
#include "ocean_kernels.cuh"

namespace ocean {

namespace {

constexpr float kG = 9.81f;      // wave_generator.gd:5, as the buoyancy op's rho_g

// [R(q) | t] of the specification: the standard unit-quaternion rotation, q = (x, y, z, w), 3 x 4 row-major
__device__ __forceinline__ void pose_transform(const float* __restrict__ q, const float* __restrict__ t, float* __restrict__ T) {
    const float x = q[0], y = q[1], z = q[2], w = q[3];
    const float xx = x * x, yy = y * y, zz = z * z;
    const float xy = x * y, xz = x * z, yz = y * z;
    const float wx = w * x, wy = w * y, wz = w * z;
    T[0] = 1.0f - 2.0f * (yy + zz);
    T[1] = 2.0f * (xy - wz);
    T[2] = 2.0f * (xz + wy);
    T[3] = t[0];
    T[4] = 2.0f * (xy + wz);
    T[5] = 1.0f - 2.0f * (xx + zz);
    T[6] = 2.0f * (yz - wx);
    T[7] = t[1];
    T[8] = 2.0f * (xz - wy);
    T[9] = 2.0f * (yz + wx);
    T[10] = 1.0f - 2.0f * (xx + yy);
    T[11] = t[2];
}

__global__ void __launch_bounds__(256) k_bodies_prepare(const ocean_floating_body* __restrict__ bodies, const ocean_body_state* __restrict__ states,
                                                        int num_bodies, const ocean_buoyancy_point* __restrict__ points, float* __restrict__ r2,
                                                        ocean_buoyancy_body* __restrict__ pose, ocean_body_velocity* __restrict__ vel) {
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (warp >= (size_t)num_bodies) return;        // whole warps: the shuffles below see all 32 lanes
    const int body = (int)warp;
    const int lane = threadIdx.x & 31;
    const ocean_floating_body b = bodies[body];
    const ocean_buoyancy_point* hull = points + b.first_point;
    float m = 0.0f;
    for (int j = lane; j < b.num_points; j += 32) {
        const float* p = hull[j].position;
        m = fmaxf(m, (p[0] * p[0] + p[1] * p[1]) + p[2] * p[2]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_down_sync(0xffffffffu, m, o));
    if (lane != 0) return;
    r2[body] = m;
    const ocean_body_state& s = states[body];
    ocean_buoyancy_body pb;
    pose_transform(s.orientation, s.position, pb.transform);
    pb.first_point = b.first_point;
    pb.num_points = b.num_points;
    pose[body] = pb;
    ocean_body_velocity v;
    for (int k = 0; k < 3; ++k) {
        v.linear[k] = s.linear_velocity[k];
        v.angular[k] = s.angular_velocity[k];
    }
    vel[body] = v;
}

// One sub-step of the specification's step per body.  The plain form (k_bodies_integrate) forms F, tau and the denominators
// m + h c_v, I + h c_w from the two records; the driven form (k_bodies_integrate_driven, ocean_drive.cu's reduce) reads them
// from the body's DriveSum, where the drive contributions are already added.
template <bool kDriven>
__device__ __forceinline__ void bodies_integrate(const ocean_floating_body* __restrict__ bodies, const float* __restrict__ r2, int num_bodies,
                                                 const ocean_buoyancy_result* __restrict__ hyd, const ocean_drag_result* __restrict__ drg,
                                                 float density, float h, ocean_body_state* __restrict__ states, ocean_buoyancy_body* __restrict__ pose,
                                                 ocean_body_velocity* __restrict__ vel, float* __restrict__ transforms,
                                                 const DriveSum* __restrict__ sums) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= num_bodies) return;
    const ocean_floating_body b = bodies[i];
    ocean_body_state s = states[i];
    float R[12];                                    // the pose this sub-step started from: [R(q) | position]
    for (int k = 0; k < 12; ++k) R[k] = pose[i].transform[k];
    ocean_buoyancy_result fh{};
    ocean_drag_result fd{};
    DriveSum ds{};
    if constexpr (kDriven) ds = sums[i]; else { fh = hyd[i]; fd = drg[i]; }
    const float cv = (density * fd.wetted_drag_area) * fd.max_relative_speed;
    const float cw = kDriven ? 0.0f : cv * __ldg(&r2[i]);
    // linear: v' = v + (h / (m + h c_v)) F
    float F[3];
    for (int k = 0; k < 3; ++k) F[k] = kDriven ? ds.force[k] : fh.force[k] + fd.force[k];
    F[1] = F[1] - b.mass * kG;
    const float kv = __fdiv_rn(h, kDriven ? ds.den_v : b.mass + h * cv);
    for (int k = 0; k < 3; ++k) s.linear_velocity[k] = s.linear_velocity[k] + kv * F[k];
    // angular, in body axes: w_b' = w_b + h tau_b / (I + h c_w), then w' = R w_b'
    float tau[3], tb[3], wb[3];
    for (int k = 0; k < 3; ++k) tau[k] = kDriven ? ds.torque[k] : fh.torque[k] + fd.torque[k];
    for (int k = 0; k < 3; ++k) {
        tb[k] = (R[k] * tau[0] + R[4 + k] * tau[1]) + R[8 + k] * tau[2];
        wb[k] = (R[k] * s.angular_velocity[0] + R[4 + k] * s.angular_velocity[1]) + R[8 + k] * s.angular_velocity[2];
    }
    for (int k = 0; k < 3; ++k) wb[k] = wb[k] + __fdiv_rn(h * tb[k], kDriven ? ds.den_w[k] : b.inertia[k] + h * cw);
    for (int k = 0; k < 3; ++k) s.angular_velocity[k] = (R[4 * k] * wb[0] + R[4 * k + 1] * wb[1]) + R[4 * k + 2] * wb[2];
    // position and orientation: p' = p + h v',  q' = normalize(q + (h/2) (w' (x) q))
    for (int k = 0; k < 3; ++k) s.position[k] = s.position[k] + h * s.linear_velocity[k];
    const float* w = s.angular_velocity;
    float* q = s.orientation;
    const float dq[4] = {(w[0] * q[3] + w[1] * q[2]) - w[2] * q[1],
                         (w[1] * q[3] + w[2] * q[0]) - w[0] * q[2],
                         (w[2] * q[3] + w[0] * q[1]) - w[1] * q[0],
                         -((w[0] * q[0] + w[1] * q[1]) + w[2] * q[2])};
    const float hh = 0.5f * h;
    for (int k = 0; k < 4; ++k) q[k] = q[k] + hh * dq[k];
    const float n = __fsqrt_rn(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]);
    for (int k = 0; k < 4; ++k) q[k] = __fdiv_rn(q[k], n);
    states[i] = s;
    // the next sub-step's tables (the range in the pose row stays as k_bodies_prepare wrote it)
    pose_transform(s.orientation, s.position, R);
    for (int k = 0; k < 12; ++k) pose[i].transform[k] = R[k];
    ocean_body_velocity v;
    for (int k = 0; k < 3; ++k) {
        v.linear[k] = s.linear_velocity[k];
        v.angular[k] = s.angular_velocity[k];
    }
    vel[i] = v;
    if (transforms)
        for (int k = 0; k < 12; ++k) transforms[(size_t)i * 12 + k] = R[k];
}

__global__ void __launch_bounds__(256) k_bodies_integrate(const ocean_floating_body* __restrict__ bodies, const float* __restrict__ r2,
                                                          int num_bodies, const ocean_buoyancy_result* __restrict__ hyd,
                                                          const ocean_drag_result* __restrict__ drg, float density, float h,
                                                          ocean_body_state* __restrict__ states, ocean_buoyancy_body* __restrict__ pose,
                                                          ocean_body_velocity* __restrict__ vel, float* __restrict__ transforms) {
    bodies_integrate<false>(bodies, r2, num_bodies, hyd, drg, density, h, states, pose, vel, transforms, nullptr);
}

__global__ void __launch_bounds__(256) k_bodies_integrate_driven(const ocean_floating_body* __restrict__ bodies, int num_bodies,
                                                                 const DriveSum* __restrict__ sums, float h, ocean_body_state* __restrict__ states,
                                                                 ocean_buoyancy_body* __restrict__ pose, ocean_body_velocity* __restrict__ vel,
                                                                 float* __restrict__ transforms) {
    bodies_integrate<true>(bodies, nullptr, num_bodies, nullptr, nullptr, 0.0f, h, states, pose, vel, transforms, sums);
}

// r2 = the NaN-dropping max of |p|^2 over the mesh's vertices, the first sub-step's pose row ([R(q) | position], the mesh) and
// velocity row: k_bodies_prepare on a hull mesh; and the body's ocean_floating_body row (its mass and inertia, the mesh's
// vertex range), the table k_bodies_integrate reads.
__global__ void __launch_bounds__(256) k_hull_prepare(const ocean_floating_hull* __restrict__ bodies, const ocean_body_state* __restrict__ states,
                                                      int num_bodies, const ocean_hull_mesh* __restrict__ meshes,
                                                      const float* __restrict__ vertices, float* __restrict__ r2, ocean_hull_body* __restrict__ pose,
                                                      ocean_body_velocity* __restrict__ vel, ocean_floating_body* __restrict__ rows) {
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (warp >= (size_t)num_bodies) return;        // whole warps: the shuffles below see all 32 lanes
    const int body = (int)warp;
    const int lane = threadIdx.x & 31;
    const ocean_floating_hull b = bodies[body];
    const ocean_hull_mesh mesh = meshes[b.mesh];
    const float* p0 = vertices + 3 * (size_t)mesh.first_vertex;
    float m = 0.0f;
    for (int j = lane; j < mesh.num_vertices; j += 32) {
        const float* p = p0 + 3 * (size_t)j;
        m = fmaxf(m, (p[0] * p[0] + p[1] * p[1]) + p[2] * p[2]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_down_sync(0xffffffffu, m, o));
    if (lane != 0) return;
    r2[body] = m;
    rows[body] = ocean_floating_body{b.mass, {b.inertia[0], b.inertia[1], b.inertia[2]}, mesh.first_vertex, mesh.num_vertices};
    const ocean_body_state& s = states[body];
    ocean_hull_body pb;
    pose_transform(s.orientation, s.position, pb.transform);
    pb.mesh = b.mesh;
    pb.reserved = 0;
    pose[body] = pb;
    ocean_body_velocity v;
    for (int k = 0; k < 3; ++k) {
        v.linear[k] = s.linear_velocity[k];
        v.angular[k] = s.angular_velocity[k];
    }
    vel[body] = v;
}

}  // namespace

cudaError_t launch_bodies_prepare(const ocean_floating_body* bodies_dev, const ocean_body_state* states_dev, int num_bodies,
                                  const ocean_buoyancy_point* points_dev, float* r2_dev, ocean_buoyancy_body* pose_dev,
                                  ocean_body_velocity* velocities_dev, cudaStream_t stream) {
    if (num_bodies <= 0) return cudaSuccess;
    const unsigned blocks = (unsigned)(((size_t)num_bodies * 32 + 255) / 256);      // 8 bodies per block
    k_bodies_prepare<<<blocks, 256, 0, stream>>>(bodies_dev, states_dev, num_bodies, points_dev, r2_dev, pose_dev, velocities_dev);
    return cudaGetLastError();
}

cudaError_t launch_bodies_integrate(const ocean_floating_body* bodies_dev, const float* r2_dev, int num_bodies,
                                    const ocean_buoyancy_result* hydrostatic_dev, const ocean_drag_result* drag_dev, float density, float h,
                                    ocean_body_state* states_dev, ocean_buoyancy_body* pose_dev, ocean_body_velocity* velocities_dev,
                                    float* transforms_dev, cudaStream_t stream) {
    if (num_bodies <= 0) return cudaSuccess;
    k_bodies_integrate<<<(unsigned)((num_bodies + 255) / 256), 256, 0, stream>>>(bodies_dev, r2_dev, num_bodies, hydrostatic_dev, drag_dev,
                                                                                 density, h, states_dev, pose_dev, velocities_dev,
                                                                                 transforms_dev);
    return cudaGetLastError();
}

cudaError_t launch_bodies_integrate_driven(const ocean_floating_body* bodies_dev, int num_bodies, const DriveSum* sums_dev, float h,
                                           ocean_body_state* states_dev, ocean_buoyancy_body* pose_dev, ocean_body_velocity* velocities_dev,
                                           float* transforms_dev, cudaStream_t stream) {
    if (num_bodies <= 0) return cudaSuccess;
    k_bodies_integrate_driven<<<(unsigned)((num_bodies + 255) / 256), 256, 0, stream>>>(bodies_dev, num_bodies, sums_dev, h, states_dev, pose_dev,
                                                                                        velocities_dev, transforms_dev);
    return cudaGetLastError();
}

cudaError_t launch_hull_prepare(const ocean_floating_hull* bodies_dev, const ocean_body_state* states_dev, int num_bodies,
                                const ocean_hull_mesh* meshes_dev, const float* vertices_dev, float* r2_dev, ocean_hull_body* pose_dev,
                                ocean_body_velocity* velocities_dev, ocean_floating_body* rows_dev, cudaStream_t stream) {
    if (num_bodies <= 0) return cudaSuccess;
    const unsigned blocks = (unsigned)(((size_t)num_bodies * 32 + 255) / 256);      // 8 bodies per block
    k_hull_prepare<<<blocks, 256, 0, stream>>>(bodies_dev, states_dev, num_bodies, meshes_dev, vertices_dev, r2_dev, pose_dev, velocities_dev,
                                               rows_dev);
    return cudaGetLastError();
}

}  // namespace ocean
