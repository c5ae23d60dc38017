// ocean_hull.cu -- floating bodies on triangle-mesh hulls: hydrostatic pressure and drag integrated over the wetted triangles
// (ocean_hull_forces, ocean_simulate_hull_bodies; oracle/hull.py is the specification).
//
// A forces call runs, on the generator's stream:
//   k_hull_transform      one thread per world vertex (body-major; the host's exclusive prefix of the meshes' num_vertices gives
//                         each body its start, a binary search over it gives a thread its body): r = R p, writes (r, r.y + t.y)
//                         and the query point (w.x, w.z)
//   launch_query_surface  the surface query (ocean_sample.cu), unchanged, on those points
//   k_hull_vertex         one thread per world vertex: the depth d = eta - w.y and the water velocity u at the record's source
//                         point (plus the wake's vertical velocity while the coupling is live), each vertex gathered once
//   k_hull_reduce         one warp per body, lane l takes triangles j = l, l + 32, ...: clips each at d = 0, integrates pressure
//                         and drag over its wet pieces (their sum first), and sums in the specification's order -- each lane from
//                         +0 in increasing j, then __shfl_down_sync with offsets 16, 8, 4, 2, 1; lane 0 writes both records.
// The integrator (ocean_simulate_hull_bodies) adds k_hull_prepare, ocean_bodies.cu's k_bodies_prepare for hull meshes, and runs
// ocean_bodies.cu's k_bodies_integrate unchanged on the pose rows, which have ocean_buoyancy_body's layout.
// No shared memory and no atomics.  Numeric policy: binary32, the specification's operation order, no contraction
// (-fmad=false), IEEE division and square root.
#include "../../include/ocean.h"
#include "ocean_kernels.cuh"
#include "ocean_texture.cuh"

namespace ocean {

namespace {

// r = R p of the specification (ocean_buoyancy.cu's rotate)
__device__ __forceinline__ float3 rotate(const float* __restrict__ T, const float* __restrict__ p) {
    float3 r;
    r.x = (T[0] * p[0] + T[1] * p[1]) + T[2] * p[2];
    r.y = (T[4] * p[0] + T[5] * p[1]) + T[6] * p[2];
    r.z = (T[8] * p[0] + T[9] * p[1]) + T[10] * p[2];
    return r;
}

__device__ __forceinline__ float3 sub(float3 a, float3 b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float3 add(float3 a, float3 b) { return make_float3(a.x + b.x, a.y + b.y, a.z + b.z); }
// a x b, each component (a.y b.z - a.z b.y, ...) rounded as written
__device__ __forceinline__ float3 cross(float3 a, float3 b) {
    return make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

// A corner of a wet piece: its position r (rotated, not translated), depth d and water velocity u.
struct Corner {
    float3 r;
    float d;
    float3 u;
};

// X_ab of the specification: the crossing of edge a -> b from the wet corner a, t = d_a / (d_a - d_b), with d = 0.
__device__ __forceinline__ Corner clip(const Corner& a, const Corner& b) {
    const float t = __fdiv_rn(a.d, a.d - b.d);
    Corner x;
    x.r = make_float3(a.r.x + t * (b.r.x - a.r.x), a.r.y + t * (b.r.y - a.r.y), a.r.z + t * (b.r.z - a.r.z));
    x.d = 0.0f;
    x.u = make_float3(a.u.x + t * (b.u.x - a.u.x), a.u.y + t * (b.u.y - a.u.y), a.u.z + t * (b.u.z - a.u.z));
    return x;
}

// The sums of one triangle (or of its pieces): pressure (f = sum a sd, tq = sum m x a, q = sum a.y m), drag (g = sum F,
// gt = sum r_c x F, area = sum (C_n + C_t) A) and the max of |d_c|.
struct Sums {
    float3 f, tq, q, g, gt;
    float area, speed;
};

// One wet piece (c0, c1, c2) of the specification onto s.
__device__ __forceinline__ void piece(const Corner& c0, const Corner& c1, const Corner& c2, const ocean_body_velocity& bv, float cn, float ct,
                                      float cnt, Sums& s) {
    const float3 e = cross(sub(c2.r, c0.r), sub(c1.r, c0.r));
    const float3 a = make_float3(0.5f * e.x, 0.5f * e.y, 0.5f * e.z);
    const float sd = (c0.d + c1.d) + c2.d;
    const float sdd = (c0.d * c0.d + c1.d * c1.d) + c2.d * c2.d;
    float3 m;                                       // sum d_i r_i + sum d sum r (y: + (sum d^2 + (sum d)^2) / 2)
    m.x = ((c0.d * c0.r.x + c1.d * c1.r.x) + c2.d * c2.r.x) + sd * ((c0.r.x + c1.r.x) + c2.r.x);
    m.y = ((c0.d * c0.r.y + c1.d * c1.r.y) + c2.d * c2.r.y) + sd * ((c0.r.y + c1.r.y) + c2.r.y);
    m.z = ((c0.d * c0.r.z + c1.d * c1.r.z) + c2.d * c2.r.z) + sd * ((c0.r.z + c1.r.z) + c2.r.z);
    const float my = m.y + 0.5f * (sdd + sd * sd);
    s.f = add(s.f, make_float3(a.x * sd, a.y * sd, a.z * sd));
    s.tq = add(s.tq, cross(m, a));
    s.q = add(s.q, make_float3(a.y * m.x, a.y * my, a.y * m.z));
    const float A = __fsqrt_rn((a.x * a.x + a.y * a.y) + a.z * a.z);
    if (!(A > 0.0f)) return;                        // a zero-area piece adds no drag
    // relative velocities u - (v + w x r) at the corners, and their mean
    auto rel = [&](const Corner& c) {
        return make_float3(c.u.x - (bv.linear[0] + (bv.angular[1] * c.r.z - bv.angular[2] * c.r.y)),
                           c.u.y - (bv.linear[1] + (bv.angular[2] * c.r.x - bv.angular[0] * c.r.z)),
                           c.u.z - (bv.linear[2] + (bv.angular[0] * c.r.y - bv.angular[1] * c.r.x)));
    };
    const float3 d0 = rel(c0), d1 = rel(c1), d2 = rel(c2);
    const float3 dc = make_float3(__fdiv_rn((d0.x + d1.x) + d2.x, 3.0f), __fdiv_rn((d0.y + d1.y) + d2.y, 3.0f),
                                  __fdiv_rn((d0.z + d1.z) + d2.z, 3.0f));
    const float3 n = make_float3(__fdiv_rn(a.x, A), __fdiv_rn(a.y, A), __fdiv_rn(a.z, A));
    const float dn = (dc.x * n.x + dc.y * n.y) + dc.z * n.z;
    const float3 dt = make_float3(dc.x - dn * n.x, dc.y - dn * n.y, dc.z - dn * n.z);
    const float st = __fsqrt_rn((dt.x * dt.x + dt.y * dt.y) + dt.z * dt.z);
    const float kt = (ct * A) * st;
    const float kn = dn < 0.0f ? (cn * A) * (dn * dn) : 0.0f;
    const float3 F = make_float3(kt * dt.x - kn * n.x, kt * dt.y - kn * n.y, kt * dt.z - kn * n.z);
    const float3 rc = make_float3(__fdiv_rn((c0.r.x + c1.r.x) + c2.r.x, 3.0f), __fdiv_rn((c0.r.y + c1.r.y) + c2.r.y, 3.0f),
                                  __fdiv_rn((c0.r.z + c1.r.z) + c2.r.z, 3.0f));
    s.g = add(s.g, F);
    s.gt = add(s.gt, cross(rc, F));
    s.area = s.area + cnt * A;
    s.speed = fmaxf(s.speed, __fsqrt_rn((dc.x * dc.x + dc.y * dc.y) + dc.z * dc.z));
}

__device__ __forceinline__ int body_of(const int* __restrict__ offsets, int num_bodies, int i) {
    int lo = 0, hi = num_bodies - 1;                // the last body whose start is <= i (it has vertices: the next start is > i)
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(&offsets[mid]) <= i) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(256) k_hull_transform(const ocean_hull_body* __restrict__ bodies, const int* __restrict__ offsets,
                                                        int num_bodies, const ocean_hull_mesh* __restrict__ meshes,
                                                        const float* __restrict__ vertices, int n, float2* __restrict__ q,
                                                        float4* __restrict__ corner_r) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int body = body_of(offsets, num_bodies, i);
    const ocean_hull_body& b = bodies[body];
    const int v = meshes[b.mesh].first_vertex + (i - __ldg(&offsets[body]));
    const float p[3] = {__ldg(&vertices[3 * (size_t)v]), __ldg(&vertices[3 * (size_t)v + 1]), __ldg(&vertices[3 * (size_t)v + 2])};
    const float3 r = rotate(b.transform, p);
    q[i] = make_float2(r.x + b.transform[3], r.z + b.transform[11]);
    corner_r[i] = make_float4(r.x, r.y, r.z, r.y + b.transform[7]);
}

// d = eta - w.y into corner_r[i].w, u into corner_u[i]
__global__ void __launch_bounds__(256) k_hull_vertex(const ocean_surface_sample* __restrict__ samples, int n, const uint2* __restrict__ velocity,
                                                     int N, int C, const float4* __restrict__ scales, const float* __restrict__ wv,
                                                     float4* __restrict__ corner_r, float4* __restrict__ corner_u) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const ocean_surface_sample& rec = samples[i];
    const float px = rec.source_x, pz = rec.source_z;
    float ux = 0.0f, uy = 0.0f, uz = 0.0f;
    for (int c = 0; c < C; ++c) {
        const float4 s = __ldg(&scales[c]);
        add_displacement(velocity + (size_t)c * N * N, N, px * s.x, pz * s.y, s.z, ux, uy, uz);
    }
    if (wv) uy = uy + __ldg(&wv[i]);
    corner_r[i].w = rec.displacement[1] - corner_r[i].w;
    corner_u[i] = make_float4(ux, uy, uz, 0.0f);
}

__device__ __forceinline__ Corner load_corner(const float4* __restrict__ corner_r, const float4* __restrict__ corner_u, int k) {
    const float4 r = __ldg(&corner_r[k]), u = __ldg(&corner_u[k]);
    return Corner{make_float3(r.x, r.y, r.z), r.w, make_float3(u.x, u.y, u.z)};
}

__global__ void __launch_bounds__(256) k_hull_reduce(const ocean_hull_body* __restrict__ bodies, const ocean_body_velocity* __restrict__ velocities,
                                                     const int* __restrict__ offsets, int num_bodies, const ocean_hull_mesh* __restrict__ meshes,
                                                     const int* __restrict__ triangles, const float4* __restrict__ corner_r,
                                                     const float4* __restrict__ corner_u, const ocean_surface_sample* __restrict__ samples,
                                                     float rho_g, float half_rho, float tol, ocean_buoyancy_result* __restrict__ hyd,
                                                     ocean_drag_result* __restrict__ drg) {
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (warp >= (size_t)num_bodies) return;        // whole warps: the shuffles below see all 32 lanes
    const int body = (int)warp;
    const int lane = threadIdx.x & 31;
    const ocean_hull_mesh mesh = meshes[bodies[body].mesh];
    if (mesh.num_vertices == 0) {
        if (lane == 0) {
            hyd[body] = ocean_buoyancy_result{};
            drg[body] = ocean_drag_result{};
        }
        return;
    }
    const int base = offsets[body];
    const ocean_body_velocity bv = velocities[body];
    const float cn = mesh.normal_drag, ct = mesh.tangential_drag, cnt = cn + ct;
    const int* tri = triangles + 3 * (size_t)mesh.first_triangle;
    const float3 zero = make_float3(0.0f, 0.0f, 0.0f);
    Sums s{zero, zero, zero, zero, zero, 0.0f, 0.0f};
    for (int j = lane; j < mesh.num_triangles; j += 32) {
        Corner c0 = load_corner(corner_r, corner_u, base + __ldg(&tri[3 * j]));
        Corner c1 = load_corner(corner_r, corner_u, base + __ldg(&tri[3 * j + 1]));
        Corner c2 = load_corner(corner_r, corner_u, base + __ldg(&tri[3 * j + 2]));
        if (isnan(c0.d) || isnan(c1.d) || isnan(c2.d)) continue;     // a NaN depth drops the triangle
        const bool w0 = c0.d > 0.0f, w1 = c1.d > 0.0f, w2 = c2.d > 0.0f;
        const int wet = (int)w0 + (int)w1 + (int)w2;
        if (wet == 0) continue;
        // rotate the corners in winding order: the one wet corner, or the corner after the one dry corner, first
        if ((wet == 1 && w1) || (wet == 2 && !w0)) {
            const Corner t = c0; c0 = c1; c1 = c2; c2 = t;
        } else if ((wet == 1 && w2) || (wet == 2 && !w1)) {
            const Corner t = c2; c2 = c1; c1 = c0; c0 = t;
        }
        Sums t{zero, zero, zero, zero, zero, 0.0f, s.speed};
        if (wet == 3) {
            piece(c0, c1, c2, bv, cn, ct, cnt, t);
        } else if (wet == 1) {
            piece(c0, clip(c0, c1), clip(c0, c2), bv, cn, ct, cnt, t);
        } else {
            const Corner x12 = clip(c1, c2), x20 = clip(c0, c2);
            piece(c0, c1, x12, bv, cn, ct, cnt, t);
            piece(c0, x12, x20, bv, cn, ct, cnt, t);
        }
        s.f = add(s.f, t.f);
        s.tq = add(s.tq, t.tq);
        s.q = add(s.q, t.q);
        s.g = add(s.g, t.g);
        s.gt = add(s.gt, t.gt);
        s.area = s.area + t.area;
        s.speed = t.speed;
    }
    float max_res = __int_as_float(0x7fffffff);
    unsigned missed = 0;
    for (int j = lane; j < mesh.num_vertices; j += 32) {
        const float res = samples[base + j].residual;
        max_res = fmaxf(max_res, res);
        missed += !(res <= tol);
    }
    float v[17] = {s.f.x, s.f.y, s.f.z, s.tq.x, s.tq.y, s.tq.z, s.q.x, s.q.y, s.q.z, s.g.x, s.g.y, s.g.z, s.gt.x, s.gt.y, s.gt.z, s.area, s.speed};
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {              // p[l] = p[l] + p[l + o]: the specification's tree
#pragma unroll
        for (int k = 0; k < 16; ++k) v[k] = v[k] + __shfl_down_sync(0xffffffffu, v[k], o);
        v[16] = fmaxf(v[16], __shfl_down_sync(0xffffffffu, v[16], o));
        max_res = fmaxf(max_res, __shfl_down_sync(0xffffffffu, max_res, o));
        missed += __shfl_down_sync(0xffffffffu, missed, o);
    }
    if (lane != 0) return;
    ocean_buoyancy_result h;
    const float fy = __fdiv_rn(v[1], 3.0f);
    h.force[0] = -(rho_g * __fdiv_rn(v[0], 3.0f));
    h.force[1] = -(rho_g * fy);
    h.force[2] = -(rho_g * __fdiv_rn(v[2], 3.0f));
    for (int k = 0; k < 3; ++k) h.torque[k] = -(rho_g * __fdiv_rn(v[3 + k], 12.0f));
    const float V = -fy;
    h.submerged_volume = V;
    const bool pos = V > 0.0f;
    for (int k = 0; k < 3; ++k) h.center_offset[k] = pos ? __fdiv_rn(-__fdiv_rn(v[6 + k], 12.0f), V) : 0.0f;
    h.max_residual = max_res;
    h.unconverged = missed;
    hyd[body] = h;
    ocean_drag_result d;
    for (int k = 0; k < 3; ++k) {
        d.force[k] = half_rho * v[9 + k];
        d.torque[k] = half_rho * v[12 + k];
    }
    d.wetted_drag_area = v[15];
    d.max_relative_speed = v[16];
    drg[body] = d;
}

}  // namespace

cudaError_t launch_hull_transform(const ocean_hull_body* bodies_dev, const int* offsets_dev, int num_bodies, const ocean_hull_mesh* meshes_dev,
                                  const float* vertices_dev, int n, float2* q_dev, float4* corner_r_dev, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    k_hull_transform<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(bodies_dev, offsets_dev, num_bodies, meshes_dev, vertices_dev, n, q_dev,
                                                                      corner_r_dev);
    return cudaGetLastError();
}

cudaError_t launch_hull_vertex(const ocean_surface_sample* samples_dev, int n, const uint2* velocity_dev, int map_size, int num_cascades,
                               const float4* scales_dev, const float* wake_wv_dev, float4* corner_r_dev, float4* corner_u_dev,
                               cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    k_hull_vertex<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(samples_dev, n, velocity_dev, map_size, num_cascades, scales_dev, wake_wv_dev,
                                                                   corner_r_dev, corner_u_dev);
    return cudaGetLastError();
}

cudaError_t launch_hull_reduce(const ocean_hull_body* bodies_dev, const ocean_body_velocity* velocities_dev, const int* offsets_dev,
                               int num_bodies, const ocean_hull_mesh* meshes_dev, const int* triangles_dev, const float4* corner_r_dev,
                               const float4* corner_u_dev, const ocean_surface_sample* samples_dev, float rho_g, float half_rho,
                               float tolerance, ocean_buoyancy_result* hydrostatic_dev, ocean_drag_result* drag_dev, cudaStream_t stream) {
    if (num_bodies <= 0) return cudaSuccess;
    const unsigned blocks = (unsigned)(((size_t)num_bodies * 32 + 255) / 256);      // 8 bodies per block
    k_hull_reduce<<<blocks, 256, 0, stream>>>(bodies_dev, velocities_dev, offsets_dev, num_bodies, meshes_dev, triangles_dev, corner_r_dev,
                                              corner_u_dev, samples_dev, rho_g, half_rho, tolerance, hydrostatic_dev, drag_dev);
    return cudaGetLastError();
}

}  // namespace ocean
