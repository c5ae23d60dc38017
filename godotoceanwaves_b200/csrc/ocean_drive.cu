// ocean_drive.cu -- thrusters, hull foils, applied loads and tethers of the driven floating-body integrator
// (ocean_simulate_driven_bodies; oracle/drive.py is the specification).
//
// Per sub-step, around ocean_simulate_bodies' sequence on the same pose and velocity tables:
//   k_actuator_transform  one thread per actuator (the thrusters, then the foils): r = R p, w = r + t, and Q = (w.x, w.z) at
//                         world point world + k, after the hull's, so one surface query serves both
//   k_tethers             one thread per tether: the tension from the end points' poses and velocities the sub-step starts
//                         from, its force and the torques on both bodies, and the tension output
//   k_drive_reduce        one warp per body over the body's incidence list (its thrusters, foils and tether ends in array
//                         order, built on the host): the lanes evaluate 32 entries at a time, then every lane adds them onto
//                         F = hyd + drg and tau in list order, so the sums do not depend on the schedule; then the load, and
//                         the step's denominators; lane 0 writes the DriveSum k_bodies_integrate_driven reads and the drive
//                         record.
// A term that does not act (a dry actuator, a slack tether) is skipped, not added as zero, so a body with nothing acting
// keeps the plain step's bits, signed zeros included.  No atomics.  Numeric policy: binary32, the specification's operation
// order, no contraction (-fmad=false), IEEE division and square root.
#include "../../include/ocean.h"
#include "ocean_kernels.cuh"
#include "ocean_texture.cuh"

namespace ocean {

namespace {

// r = R p: ((R[k][0] p.x + R[k][1] p.y) + R[k][2] p.z), row k of the 3 x 4 row-major transform (ocean_buoyancy.cu's)
__device__ __forceinline__ float3 rotate(const float* __restrict__ T, const float* __restrict__ p) {
    float3 r;
    r.x = (T[0] * p[0] + T[1] * p[1]) + T[2] * p[2];
    r.y = (T[4] * p[0] + T[5] * p[1]) + T[6] * p[2];
    r.z = (T[8] * p[0] + T[9] * p[1]) + T[10] * p[2];
    return r;
}

__device__ __forceinline__ float3 cross(float3 a, float3 b) {
    return make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

// the velocity of the body point at lever r: v + w x r, each bracket rounded as drag.py's
__device__ __forceinline__ float3 point_velocity(const ocean_body_velocity& v, float3 r) {
    return make_float3(v.linear[0] + (v.angular[1] * r.z - v.angular[2] * r.y), v.linear[1] + (v.angular[2] * r.x - v.angular[0] * r.z),
                       v.linear[2] + (v.angular[0] * r.y - v.angular[1] * r.x));
}

__device__ __forceinline__ float submerged_fraction(float eta, float wy, float h) {
    return h > 0.0f ? fminf(fmaxf(__fdiv_rn(eta - (wy - h), h + h), 0.0f), 1.0f) : (wy <= eta ? 1.0f : 0.0f);
}

__device__ __forceinline__ float norm2(const float* p) { return (p[0] * p[0] + p[1] * p[1]) + p[2] * p[2]; }

// ocean_thruster and ocean_foil share one layout: body, position, a direction, a magnitude, half_height
static_assert(sizeof(ocean_thruster) == sizeof(ocean_foil), "actuator layouts");

__global__ void __launch_bounds__(256) k_actuator_transform(const ocean_thruster* __restrict__ thrusters, int num_thrusters,
                                                            const ocean_foil* __restrict__ foils, int n, const ocean_buoyancy_body* __restrict__ pose,
                                                            float2* __restrict__ q) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int body;
    const float* p;
    if (i < num_thrusters) {
        body = thrusters[i].body;
        p = thrusters[i].position;
    } else {
        body = foils[i - num_thrusters].body;
        p = foils[i - num_thrusters].position;
    }
    const float* T = pose[body].transform;
    const float3 r = rotate(T, p);
    q[i] = make_float2(r.x + T[3], r.z + T[11]);
}

__global__ void __launch_bounds__(256) k_tethers(const ocean_tether* __restrict__ tethers, int n, const ocean_buoyancy_body* __restrict__ pose,
                                                 const ocean_body_velocity* __restrict__ vel, TetherForce* __restrict__ out,
                                                 float* __restrict__ tensions) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const ocean_tether t = tethers[i];
    const float* Ta = pose[t.body_a].transform;
    const float3 ra = rotate(Ta, t.point_a);
    const float3 va = point_velocity(vel[t.body_a], ra);
    float3 rb = make_float3(0.0f, 0.0f, 0.0f), xb = make_float3(t.point_b[0], t.point_b[1], t.point_b[2]), vb = rb;
    if (t.body_b >= 0) {
        const float* Tb = pose[t.body_b].transform;
        rb = rotate(Tb, t.point_b);
        xb = make_float3(rb.x + Tb[3], rb.y + Tb[7], rb.z + Tb[11]);
        vb = point_velocity(vel[t.body_b], rb);
    }
    const float dx = xb.x - (ra.x + Ta[3]), dy = xb.y - (ra.y + Ta[7]), dz = xb.z - (ra.z + Ta[11]);
    const float L = __fsqrt_rn((dx * dx + dy * dy) + dz * dz);
    const float3 u = make_float3(__fdiv_rn(dx, L), __fdiv_rn(dy, L), __fdiv_rn(dz, L));
    const float ex = vb.x - va.x, ey = vb.y - va.y, ez = vb.z - va.z;
    const float s = t.stiffness * (L - t.rest_length) + t.damping * ((ex * u.x + ey * u.y) + ez * u.z);
    TetherForce f{};
    if (L > 0.0f && s > 0.0f) {
        const float3 fa = make_float3(s * u.x, s * u.y, s * u.z);
        const float3 fb = make_float3(-fa.x, -fa.y, -fa.z);
        const float3 ta = cross(ra, fa), tb = cross(rb, fb);
        f = TetherForce{{fa.x, fa.y, fa.z}, {ta.x, ta.y, ta.z}, {tb.x, tb.y, tb.z}, s};
    }
    out[i] = f;
    if (tensions) tensions[i] = f.tension;
}

// One evaluated incidence entry: its force and torque, whether it acts, and what it adds to the bounds.
struct Term {
    float F[3], T[3];
    float a, dn;                    // foil: f * area, |dn|
    float v, w;                     // taut tether end: h c + h^2 k, (h c) |p|^2 + (h^2 k) |p|^2
    float p2;                       // foil: |p|^2
    int kind;                       // 0 none / dry, 1 thruster, 2 foil (wet), 3 dry foil, 4 taut tether end
};

__global__ void __launch_bounds__(256) k_drive_reduce(DriveArgs d, int num_bodies, const ocean_floating_body* __restrict__ bodies,
                                                      const float* __restrict__ r2, const ocean_buoyancy_body* __restrict__ pose,
                                                      const ocean_body_velocity* __restrict__ vel, const ocean_buoyancy_result* __restrict__ hyd,
                                                      const ocean_drag_result* __restrict__ drg, const ocean_surface_sample* __restrict__ samples,
                                                      const float* __restrict__ wv, const TetherForce* __restrict__ tforces,
                                                      const uint2* __restrict__ velocity, int N, int C, const float4* __restrict__ scales,
                                                      float density, float h, DriveSum* __restrict__ sums, ocean_drive_result* __restrict__ drive) {
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (warp >= (size_t)num_bodies) return;        // whole warps: the shuffles below see all 32 lanes
    const int body = (int)warp;
    const int lane = threadIdx.x & 31;
    const float* T = pose[body].transform;
    const ocean_body_velocity bv = vel[body];
    const float half_rho = 0.5f * density;
    const float hh = h * h;
    const ocean_buoyancy_result fh = hyd[body];
    const ocean_drag_result fd = drg[body];
    float F[3], tau[3], D[3] = {0.0f, 0.0f, 0.0f}, DT[3] = {0.0f, 0.0f, 0.0f};
    for (int k = 0; k < 3; ++k) F[k] = fh.force[k] + fd.force[k];
    for (int k = 0; k < 3; ++k) tau[k] = fh.torque[k] + fd.torque[k];
    float sa = 0.0f, max_dn = 0.0f, rf2 = 0.0f, tv = 0.0f, tw = 0.0f;
    bool foiled = false, taut = false;
    const int first = d.incidence_offsets[body], last = d.incidence_offsets[body + 1];
    const int nt = d.num_thrusters, nf = d.num_foils;
    for (int base = first; base < last; base += 32) {
        Term e{};
        const int j = base + lane;
        if (j < last) {
            const int id = d.incidence[j];
            if (id < nt + nf) {                     // an actuator: world point id after the hull's
                const bool thruster = id < nt;
                const ocean_thruster& a = thruster ? d.thrusters[id] : reinterpret_cast<const ocean_thruster*>(d.foils)[id - nt];
                const float3 r = rotate(T, a.position);
                const float f = submerged_fraction(samples[id].displacement[1], r.y + T[7], a.half_height);
                const float3 n = rotate(T, a.direction);
                if (!thruster) e.p2 = norm2(a.position);
                e.kind = thruster ? 0 : 3;
                if (f > 0.0f) {
                    float3 Fo;
                    if (thruster) {
                        const float g = f * a.thrust;
                        Fo = make_float3(g * n.x, g * n.y, g * n.z);
                        e.kind = 1;
                    } else {
                        const float px = samples[id].source_x, pz = samples[id].source_z;
                        float ux = 0.0f, uy = 0.0f, uz = 0.0f;
                        for (int c = 0; c < C; ++c) {
                            const float4 s = __ldg(&scales[c]);
                            add_displacement(velocity + (size_t)c * N * N, N, px * s.x, pz * s.y, s.z, ux, uy, uz);
                        }
                        if (wv) uy = uy + __ldg(&wv[id]);
                        const float3 vp = point_velocity(bv, r);
                        const float dx = ux - vp.x, dy = uy - vp.y, dz = uz - vp.z;
                        const float dn = (dx * n.x + dy * n.y) + dz * n.z;
                        const float adn = fabsf(dn);
                        e.a = f * a.thrust;         // the foil's area
                        const float g = ((half_rho * e.a) * dn) * adn;
                        Fo = make_float3(g * n.x, g * n.y, g * n.z);
                        e.dn = adn;
                        e.kind = 2;
                    }
                    const float3 To = cross(r, Fo);
                    e.F[0] = Fo.x; e.F[1] = Fo.y; e.F[2] = Fo.z;
                    e.T[0] = To.x; e.T[1] = To.y; e.T[2] = To.z;
                }
            } else {                                // a tether end
                const int k = (id - nt - nf) >> 1, end = (id - nt - nf) & 1;
                const TetherForce tf = tforces[k];
                if (tf.tension > 0.0f) {
                    const ocean_tether& t = d.tethers[k];
                    for (int c = 0; c < 3; ++c) {
                        e.F[c] = end ? -tf.force[c] : tf.force[c];
                        e.T[c] = end ? tf.torque_b[c] : tf.torque_a[c];
                    }
                    const float p2 = norm2(end ? t.point_b : t.point_a);
                    const float hc = h * t.damping, hk = hh * t.stiffness;
                    e.v = hc + hk;
                    e.w = hc * p2 + hk * p2;
                    e.kind = 4;
                }
            }
        }
        const int count = min(32, last - base);
        for (int l = 0; l < count; ++l) {           // in list order: every lane adds entry base + l
            const int kind = __shfl_sync(0xffffffffu, e.kind, l);
            float Fl[3], Tl[3];
            for (int c = 0; c < 3; ++c) {
                Fl[c] = __shfl_sync(0xffffffffu, e.F[c], l);
                Tl[c] = __shfl_sync(0xffffffffu, e.T[c], l);
            }
            const float al = __shfl_sync(0xffffffffu, e.a, l), dnl = __shfl_sync(0xffffffffu, e.dn, l);
            const float vl = __shfl_sync(0xffffffffu, e.v, l), wl = __shfl_sync(0xffffffffu, e.w, l);
            const float p2l = __shfl_sync(0xffffffffu, e.p2, l);
            if (kind == 2 || kind == 3) {
                foiled = true;
                rf2 = fmaxf(rf2, p2l);
            }
            if (kind == 1 || kind == 2 || kind == 4) {
                for (int c = 0; c < 3; ++c) {
                    F[c] = F[c] + Fl[c];
                    tau[c] = tau[c] + Tl[c];
                    D[c] = D[c] + Fl[c];
                    DT[c] = DT[c] + Tl[c];
                }
            }
            if (kind == 2) {
                sa = sa + al;
                max_dn = fmaxf(max_dn, dnl);
            }
            if (kind == 4) {
                taut = true;
                tv = tv + vl;
                tw = tw + wl;
            }
        }
    }
    if (lane != 0) return;
    if (d.loads) {
        const ocean_body_load ld = d.loads[body];
        for (int c = 0; c < 3; ++c) {
            F[c] = F[c] + ld.force[c];
            tau[c] = tau[c] + ld.torque[c];
            D[c] = D[c] + ld.force[c];
            DT[c] = DT[c] + ld.torque[c];
        }
    }
    const ocean_floating_body b = bodies[body];
    float cv = (density * fd.wetted_drag_area) * fd.max_relative_speed;
    float cw = cv * __ldg(&r2[body]);
    if (foiled) {
        const float cf = (density * sa) * max_dn;
        cv = cv + cf;
        cw = cw + cf * rf2;
    }
    DriveSum out;
    for (int c = 0; c < 3; ++c) {
        out.force[c] = F[c];
        out.torque[c] = tau[c];
    }
    out.den_v = b.mass + h * cv;
    for (int c = 0; c < 3; ++c) out.den_w[c] = b.inertia[c] + h * cw;
    if (taut) {
        out.den_v = out.den_v + tv;
        for (int c = 0; c < 3; ++c) out.den_w[c] = out.den_w[c] + tw;
    }
    sums[body] = out;
    ocean_drive_result r;
    for (int c = 0; c < 3; ++c) {
        r.force[c] = D[c];
        r.torque[c] = DT[c];
    }
    r.wetted_foil_area = sa;
    r.max_normal_speed = max_dn;
    drive[body] = r;
}

}  // namespace

cudaError_t launch_actuator_transform(const DriveArgs& d, const ocean_buoyancy_body* pose_dev, float2* q_dev, cudaStream_t stream) {
    const int n = d.num_thrusters + d.num_foils;
    if (n <= 0) return cudaSuccess;
    k_actuator_transform<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(d.thrusters, d.num_thrusters, d.foils, n, pose_dev, q_dev);
    return cudaGetLastError();
}

cudaError_t launch_tethers(const DriveArgs& d, const ocean_buoyancy_body* pose_dev, const ocean_body_velocity* velocities_dev,
                           TetherForce* forces_dev, float* tensions_dev, cudaStream_t stream) {
    if (d.num_tethers <= 0) return cudaSuccess;
    k_tethers<<<(unsigned)((d.num_tethers + 255) / 256), 256, 0, stream>>>(d.tethers, d.num_tethers, pose_dev, velocities_dev, forces_dev,
                                                                           tensions_dev);
    return cudaGetLastError();
}

cudaError_t launch_drive_reduce(const DriveArgs& d, int num_bodies, const ocean_floating_body* bodies_dev, const float* r2_dev,
                                const ocean_buoyancy_body* pose_dev, const ocean_body_velocity* velocities_dev,
                                const ocean_buoyancy_result* hydrostatic_dev, const ocean_drag_result* drag_dev,
                                const ocean_surface_sample* actuator_samples_dev, const float* actuator_wv_dev, const TetherForce* tether_forces_dev,
                                const uint2* velocity_dev, int map_size, int num_cascades, const float4* scales_dev, float density, float h,
                                DriveSum* sums_dev, ocean_drive_result* drive_dev, cudaStream_t stream) {
    if (num_bodies <= 0) return cudaSuccess;
    const unsigned blocks = (unsigned)(((size_t)num_bodies * 32 + 255) / 256);      // 8 bodies per block
    k_drive_reduce<<<blocks, 256, 0, stream>>>(d, num_bodies, bodies_dev, r2_dev, pose_dev, velocities_dev, hydrostatic_dev, drag_dev,
                                               actuator_samples_dev, actuator_wv_dev, tether_forces_dev, velocity_dev, map_size, num_cascades,
                                               scales_dev, density, h, sums_dev, drive_dev);
    return cudaGetLastError();
}

}  // namespace ocean
