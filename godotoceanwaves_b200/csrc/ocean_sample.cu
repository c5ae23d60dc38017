// ocean_sample.cu -- batched map queries: the sampling contract of the reference's water shader as a CUDA op
// (SURVEY 8f row f2; what buoyancy / gameplay code and the spray emitter need from the generator's outputs).
//
// Reference: assets/shaders/spatial/water.gdshader
//   vertex()   :27-39   displacement(UV) = sum_i texture(displacements, vec3(UV*scales_i.xy, i)).xyz * scales_i.z
//   cubic_weights / texture_bicubic :42-70
//   fragment() :72-84   gradient/foam(UV) = sum_i mix(texture_bicubic(normals, c_i), texture(normals, c_i),
//                                                       min(1, ppm_i*0.1)).xyw * vec3(scales_i.ww, 1)
// with map_scales[i] = (1/tile_length.x, 1/tile_length.y, displacement_scale, normal_scale), water.gd:102-110.
//
// Numeric policy (oracle/sampling.py is the specification): binary32, round to nearest, the shader's operation order,
// no contraction (-fmad=false); texture() = exact-weight bilinear filter with REPEAT addressing on the RGBA16F texels.
// One thread per query point; the texel gathers are 8 B reads served by L2 (the maps of a frame are L2-resident for
// N <= 1024 x 8 cascades = 128 MiB only partly -- the op is sector-bound, see DESIGN.md).
//
// The surface query (ocean_query_surface; oracle/surface.py is the specification) inverts the horizontal displacement
// first: for a world position Q it solves P + D_xz(P) = Q by damped Newton steps (four displacement texels per cascade and
// trial give D and its exact bilinear Jacobian), then samples the maps at P with the same per-point body as k_sample_maps.
// The ray cast (ocean_raycast; oracle/raycast.py is the specification) marches each ray through the height slab of the maps
// with the same inversion, warm-started from sample to sample, and refines the first crossing.  Its wake form
// (ocean_wake_set_readers; oracle/wake_readers.py) adds the wake free surface e to the height of every evaluation, widens
// the slab by e's bounds (k_raycast_wake_bound) and adds e's sample and slopes to the record.
#include "../../include/ocean.h"
#include "ocean_kernels.cuh"
#include "ocean_texture.cuh"
#include "wake_sample.cuh"

namespace ocean {

namespace {

__global__ void __launch_bounds__(256) k_sample_maps(const uint2* __restrict__ displacement, const uint2* __restrict__ normal, int N, int C,
                                                     const float2* __restrict__ points, int n, const float4* __restrict__ scales,
                                                     float* __restrict__ disp_out, float* __restrict__ grad_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float3 d, g;
    sample_point(displacement, normal, N, C, points[i], scales, d, g);
    disp_out[3 * (size_t)i + 0] = d.x;
    disp_out[3 * (size_t)i + 1] = d.y;
    disp_out[3 * (size_t)i + 2] = d.z;
    grad_out[3 * (size_t)i + 0] = g.x;
    grad_out[3 * (size_t)i + 1] = g.y;
    grad_out[3 * (size_t)i + 2] = g.z;
}

// The water velocity at undisplaced points: the displacement half of k_sample_maps on the velocity maps (v = dD/dt, so the
// displacement scale applies).
__global__ void __launch_bounds__(256) k_sample_velocity(const uint2* __restrict__ velocity, int N, int C, const float2* __restrict__ points, int n,
                                                         const float4* __restrict__ scales, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float2 p = points[i];
    float vx = 0.0f, vy = 0.0f, vz = 0.0f;
    for (int c = 0; c < C; ++c) {
        const float4 s = __ldg(&scales[c]);
        add_displacement(velocity + (size_t)c * N * N, N, p.x * s.x, p.y * s.y, s.z, vx, vy, vz);
    }
    out[3 * (size_t)i + 0] = vx;
    out[3 * (size_t)i + 1] = vy;
    out[3 * (size_t)i + 2] = vz;
}

// ---- surface query: the surface at a world position (oracle/surface.py is the specification) ----
// The shader reads the maps at the undisplaced point P and moves the vertex to P + D_xz(P) (:28,37), so the query solves
// P + D_xz(P) = Q by damped Newton steps on the displacement layers, then samples the maps at P.

struct SurfaceEval {         // D_xz(P) and J = dD_xz/dP
    float dx, dz, jxx, jxz, jzx, jzz;
};

__device__ __forceinline__ SurfaceEval surface_eval(const uint2* __restrict__ displacement, int N, int C, const float4* __restrict__ scales,
                                                    float px, float pz) {
    SurfaceEval e = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    for (int c = 0; c < C; ++c) {
        const float4 s = __ldg(&scales[c]);
        float4 du, dv;
        const float4 d = texture_bilinear_slopes(displacement + (size_t)c * N * N, N, px * s.x, pz * s.y, du, dv);
        e.dx = e.dx + d.x * s.z;
        e.dz = e.dz + d.z * s.z;
        e.jxx = e.jxx + (du.x * s.x) * s.z;
        e.jxz = e.jxz + (dv.x * s.y) * s.z;
        e.jzx = e.jzx + (du.z * s.x) * s.z;
        e.jzz = e.jzz + (dv.z * s.y) * s.z;
    }
    return e;
}

__device__ __forceinline__ float surface_residual(float px, float pz, const SurfaceEval& e, float2 q, float& ex, float& ez) {
    ex = (px + e.dx) - q.x;
    ez = (pz + e.dz) - q.y;
    return fmaxf(fabsf(ex), fabsf(ez));
}

// One start from (px, pz): damped Newton steps until r <= tol, max_iterations steps, or a step finds no trial that does
// not raise the residual.  Leaves the end point in (px, pz), returns its residual; `steps` receives the steps taken.
__device__ float surface_solve(const uint2* __restrict__ displacement, int N, int C, const float4* __restrict__ scales, float2 q,
                               float& px, float& pz, float tol, int max_iterations, int& steps) {
    SurfaceEval e = surface_eval(displacement, N, C, scales, px, pz);
    float ex, ez;
    float r = surface_residual(px, pz, e, q, ex, ez);
    steps = 0;
    while (steps < max_iterations && r > tol) {
        const float a = 1.0f + e.jxx, b = e.jxz, c = e.jzx, d = 1.0f + e.jzz;
        const float det = a * d - b * c;
        float sx = __fdiv_rn(d * ex - b * ez, det), sz = __fdiv_rn(a * ez - c * ex, det);
        if (!(det > 1e-3f) || !isfinite(sx) || !isfinite(sz)) { sx = ex; sz = ez; }    // fixed-point step
        bool taken = false;
        float lam = 1.0f;
        for (int k = 0; k < 5 && !taken; ++k, lam *= 0.5f) {
            const float tx = px - lam * sx, tz = pz - lam * sz;
            const SurfaceEval et = surface_eval(displacement, N, C, scales, tx, tz);
            float etx, etz;
            const float rt = surface_residual(tx, tz, et, q, etx, etz);
            if (rt <= r) {
                px = tx; pz = tz; e = et; ex = etx; ez = etz; r = rt;
                taken = true;
            }
        }
        ++steps;
        if (!taken) break;
    }
    return r;
}

__device__ __forceinline__ void surface_write(const uint2* __restrict__ displacement, const uint2* __restrict__ normal, int N, int C,
                                              const float4* __restrict__ scales, float px, float pz, float r, uint32_t iterations,
                                              ocean_surface_sample* __restrict__ out) {
    float3 d, g;
    sample_point(displacement, normal, N, C, make_float2(px, pz), scales, d, g);
    ocean_surface_sample s;
    s.source_x = px;
    s.source_z = pz;
    s.displacement[0] = d.x; s.displacement[1] = d.y; s.displacement[2] = d.z;
    s.gradient_foam[0] = g.x; s.gradient_foam[1] = g.y; s.gradient_foam[2] = g.z;
    s.residual = r;
    s.iterations = iterations;
    *out = s;
}

// First start, P0 = Q, for every query.  A converged query (or max_iterations == 0) writes its record; any other writes
// its end point, residual and steps into its own record and appends its index to `pending` for k_surface_restart.
__global__ void __launch_bounds__(256) k_surface_first(const uint2* __restrict__ displacement, const uint2* __restrict__ normal, int N, int C,
                                                       const float2* __restrict__ points, int n, const float4* __restrict__ scales, float tol,
                                                       int max_iterations, ocean_surface_sample* __restrict__ out, int* __restrict__ pending_count,
                                                       int* __restrict__ pending) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float2 q = points[i];
    float px = q.x, pz = q.y;
    int steps;
    const float r = surface_solve(displacement, N, C, scales, q, px, pz, tol, max_iterations, steps);
    if (r <= tol || max_iterations == 0) {
        surface_write(displacement, normal, N, C, scales, px, pz, r, (uint32_t)steps, &out[i]);
        return;
    }
    out[i].source_x = px;
    out[i].source_z = pz;
    out[i].residual = r;
    out[i].iterations = (uint32_t)steps;
    pending[atomicAdd(pending_count, 1)] = i;
}

// Per layer, max over the texels of max(|x|, |z|) (non-negative floats order as their bit patterns: atomicMax on the bits).
__global__ void __launch_bounds__(256) k_surface_bound(const uint2* __restrict__ displacement, int N, unsigned* __restrict__ layer_max) {
    const size_t texels = (size_t)N * N;
    const uint2* layer = displacement + blockIdx.y * texels;
    float m = 0.0f;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < texels; t += (size_t)gridDim.x * blockDim.x) {
        const float4 v = texel(layer, N, (int)t, 0);        // texel t of the row-major layer
        m = fmaxf(m, fmaxf(fabsf(v.x), fabsf(v.z)));
    }
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(&layer_max[blockIdx.y], __float_as_uint(m));
}

// The restarts of the queries the first start left unconverged: seeds Q - D_xz(Q), then Q +- rho along x and z, each until
// one converges; the end point with the smallest residual (the earlier start on ties) is sampled and written.
// Small blocks spread the few pending queries over the SMs; (64, 8) lets ptxas keep the solve in registers (no spill).
constexpr int kRestartBlock = 64;
__global__ void __launch_bounds__(kRestartBlock, 8) k_surface_restart(const uint2* __restrict__ displacement, const uint2* __restrict__ normal, int N, int C,
                                                         const float2* __restrict__ points, const float4* __restrict__ scales, float tol,
                                                         int max_iterations, ocean_surface_sample* __restrict__ out, const int* __restrict__ pending_count,
                                                         const int* __restrict__ pending, const unsigned* __restrict__ layer_max) {
    const int count = *pending_count;
    float rho = 0.0f;
    for (int c = 0; c < C; ++c) rho = rho + fabsf(__ldg(&scales[c]).z) * __uint_as_float(layer_max[c]);
    rho = rho * 0.5f;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < count; j += gridDim.x * blockDim.x) {
        const int i = pending[j];
        const float2 q = points[i];
        float bx = out[i].source_x, bz = out[i].source_z, br = out[i].residual;
        int total = (int)out[i].iterations;
        const SurfaceEval eq = surface_eval(displacement, N, C, scales, q.x, q.y);
        for (int s = 0; s < 5; ++s) {
            float px = q.x, pz = q.y;
            switch (s) {
                case 0: px = q.x - eq.dx; pz = q.y - eq.dz; break;
                case 1: px = q.x + rho; break;
                case 2: pz = q.y + rho; break;
                case 3: px = q.x - rho; break;
                default: pz = q.y - rho; break;
            }
            int steps;
            const float r = surface_solve(displacement, N, C, scales, q, px, pz, tol, max_iterations, steps);
            total += steps;
            if (r < br) { bx = px; bz = pz; br = r; }
            if (r <= tol) break;
        }
        surface_write(displacement, normal, N, C, scales, bx, bz, br, (uint32_t)total, &out[i]);
    }
}

// ---- ray cast: the first crossing of each ray with the displaced surface (oracle/raycast.py is the specification) ----

constexpr int kRayRefineSteps = 32;

// Signed floats as unsigned keys in the same order (atomicMax over signed values).
__device__ __forceinline__ unsigned order_key(float f) {
    const unsigned b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float order_value(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// Per layer, three maxima over the texels (NaN-dropping): [0] y, [1] -y (as order_key), [2] max(|x|, |z|) from 0 (bits, as
// k_surface_bound).  bounds must be zero on entry.
__global__ void __launch_bounds__(256) k_raycast_bound(const uint2* __restrict__ displacement, int N, unsigned* __restrict__ bounds) {
    const size_t texels = (size_t)N * N;
    const uint2* layer = displacement + blockIdx.y * texels;
    float hi = -INFINITY, nlo = -INFINITY, m = 0.0f;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < texels; t += (size_t)gridDim.x * blockDim.x) {
        const float4 v = texel(layer, N, (int)t, 0);
        hi = fmaxf(hi, v.y);
        nlo = fmaxf(nlo, -v.y);
        m = fmaxf(m, fmaxf(fabsf(v.x), fabsf(v.z)));
    }
    for (int o = 16; o > 0; o >>= 1) {
        hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        nlo = fmaxf(nlo, __shfl_xor_sync(0xffffffffu, nlo, o));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMax(&bounds[3 * blockIdx.y + 0], order_key(hi));
        atomicMax(&bounds[3 * blockIdx.y + 1], order_key(nlo));
        atomicMax(&bounds[3 * blockIdx.y + 2], __float_as_uint(m));
    }
}

// The NaN-dropping extrema of the wake free surface e ([n][n]) as k_raycast_bound's: bounds[0] = max e, bounds[1] = max -e
// (as order_key).  bounds must be zero on entry.
__global__ void __launch_bounds__(256) k_raycast_wake_bound(const float* __restrict__ e, int n, unsigned* __restrict__ bounds) {
    const size_t cells = (size_t)n * n;
    float hi = -INFINITY, nlo = -INFINITY;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < cells; t += (size_t)gridDim.x * blockDim.x) {
        const float v = e[t];
        hi = fmaxf(hi, v);
        nlo = fmaxf(nlo, -v);
    }
    for (int o = 16; o > 0; o >>= 1) {
        hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        nlo = fmaxf(nlo, __shfl_xor_sync(0xffffffffu, nlo, o));
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMax(&bounds[0], order_key(hi));
        atomicMax(&bounds[1], order_key(nlo));
    }
}

// An evaluated point of a ray: parameter, position, source point P, inversion residual, gap.
struct RayPoint {
    float t, x, y, z, px, pz, r, g;
};

// One gap evaluation at parameter t, started at Q or (warm) from the evaluated point `base` shifted by the ray's horizontal
// advance since it, with the surface query's restarts when that start does not converge.  With Wake the gap is taken to
// eta + we, we = the sample of the wake free surface w.field at (x, z).
template <bool Wake>
__device__ __forceinline__ RayPoint ray_gap(const uint2* __restrict__ displacement, int N, int C, const float4* __restrict__ scales,
                                            const ocean_ray& ray, float t, bool warm, float base_x, float base_z, float base_px, float base_pz,
                                            float tol, int max_iterations, float rho, uint32_t& iterations, uint32_t& unconverged,
                                            const WakeRead& w) {
    RayPoint e;
    e.t = t;
    e.x = ray.origin[0] + t * ray.direction[0];
    e.y = ray.origin[1] + t * ray.direction[1];
    e.z = ray.origin[2] + t * ray.direction[2];
    const float2 q = make_float2(e.x, e.z);
    float px = q.x, pz = q.y;
    if (warm && max_iterations > 0) {
        px = base_px + (e.x - base_x);
        pz = base_pz + (e.z - base_z);
    }
    // start -1 is the first (from Q or warm); starts 0..4 are k_surface_restart's seeds, in its order.  One solve site keeps
    // the solve inlined.
    float r = 0.0f;
    int total = 0;
    SurfaceEval eq;
    for (int s = -1; s < 5; ++s) {
        float sx = px, sz = pz;
        if (s >= 0) {
            if (s == 0) eq = surface_eval(displacement, N, C, scales, q.x, q.y);
            sx = q.x; sz = q.y;
            switch (s) {
                case 0: sx = q.x - eq.dx; sz = q.y - eq.dz; break;
                case 1: sx = q.x + rho; break;
                case 2: sz = q.y + rho; break;
                case 3: sx = q.x - rho; break;
                default: sz = q.y - rho; break;
            }
        }
        int steps;
        const float rs = surface_solve(displacement, N, C, scales, q, sx, sz, tol, max_iterations, steps);
        total += steps;
        if (s < 0) {
            r = rs;
            px = sx; pz = sz;
            if (r <= tol || max_iterations == 0) break;
        } else {
            if (rs < r) { px = sx; pz = sz; r = rs; }
            if (rs <= tol) break;
        }
    }
    float hx = 0.0f, eta = 0.0f, hz = 0.0f;
    for (int c = 0; c < C; ++c) {
        const float4 s = __ldg(&scales[c]);
        add_displacement(displacement + (size_t)c * N * N, N, px * s.x, pz * s.y, s.z, hx, eta, hz);
    }
    e.px = px;
    e.pz = pz;
    e.r = r;
    if constexpr (Wake) {
        float we = 0.0f;
        sample_field<false>(w.field, w.n, w.cell, w.x0, w.z0, q, &we);
        e.g = e.y - (eta + we);
    } else {
        e.g = e.y - eta;
    }
    iterations += (uint32_t)total;
    unconverged += (r <= tol) ? 0u : 1u;
    return e;
}

// One thread per ray: slab clip, march, Illinois refinement, and the map sample at the reported point.  bounds = the
// per-layer maxima of k_raycast_bound.  (128, 4) lets ptxas keep the ray's state in registers (no spill).  With Wake (the
// coupled surface) bounds[3C], bounds[3C + 1] are k_raycast_wake_bound's extrema of w.field = e, and the reported point's
// record carries e's sample and slopes as ocean_query_surface's coupled record.
template <bool Wake>
__global__ void __launch_bounds__(128, 4) k_raycast(const uint2* __restrict__ displacement, const uint2* __restrict__ normal, int N, int C,
                                                 const ocean_ray* __restrict__ rays, int n, const float4* __restrict__ scales, float step,
                                                 int max_samples, float tol, int max_iterations, const unsigned* __restrict__ bounds,
                                                 ocean_ray_hit* __restrict__ out, const WakeRead w) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const ocean_ray ray = rays[i];
    ocean_ray_hit hit = {};
    const bool finite = isfinite(ray.origin[0]) && isfinite(ray.origin[1]) && isfinite(ray.origin[2]) && isfinite(ray.direction[0]) &&
                        isfinite(ray.direction[1]) && isfinite(ray.direction[2]);
    if (!finite || (ray.direction[0] == 0.0f && ray.direction[1] == 0.0f && ray.direction[2] == 0.0f) || !(ray.t_max >= 0.0f)) {
        hit.status = OCEAN_RAY_INVALID;
        out[i] = hit;
        return;
    }
    // height slab and rho
    float y_lo = 0.0f, y_hi = 0.0f, acc = 0.0f, rho = 0.0f;
    for (int c = 0; c < C; ++c) {
        const float s = __ldg(&scales[c]).z;
        const float ymax = order_value(bounds[3 * c + 0]), ymin = -order_value(bounds[3 * c + 1]);
        const float a = s * ymin, b = s * ymax;
        y_lo = y_lo + fminf(a, b);
        y_hi = y_hi + fmaxf(a, b);
        acc = acc + fabsf(s) * fmaxf(fabsf(ymin), fabsf(ymax));
        rho = rho + fabsf(s) * __uint_as_float(bounds[3 * c + 2]);
    }
    if constexpr (Wake) {
        // the sample of e is 0 outside its window, and its bilinear interpolant lies between its extrema
        const float emax = order_value(bounds[3 * C + 0]), emin = -order_value(bounds[3 * C + 1]);
        y_lo = y_lo + fminf(emin, 0.0f);
        y_hi = y_hi + fmaxf(emax, 0.0f);
        acc = acc + fmaxf(fabsf(emin), fabsf(emax));
    }
    rho = rho * 0.5f;
    const float pad = tol + acc * 0x1p-13f;
    const float lo = y_lo - pad, hi = y_hi + pad;
    float t_in, t_out;
    bool enters;
    if (ray.direction[1] == 0.0f) {
        t_in = 0.0f;
        t_out = ray.t_max;
        enters = lo <= ray.origin[1] && ray.origin[1] <= hi;
    } else {
        const float ta = __fdiv_rn(lo - ray.origin[1], ray.direction[1]), tb = __fdiv_rn(hi - ray.origin[1], ray.direction[1]);
        const float tn = ta < tb ? ta : tb, tf = ta < tb ? tb : ta;
        t_in = tn > 0.0f ? tn : 0.0f;
        t_out = tf < ray.t_max ? tf : ray.t_max;
        enters = t_in <= t_out && isfinite(t_in);
    }
    if (!enters) {
        hit.status = OCEAN_RAY_MISS;
        hit.position[0] = ray.origin[0]; hit.position[1] = ray.origin[1]; hit.position[2] = ray.origin[2];
        out[i] = hit;
        return;
    }
    const float h = __fdiv_rn(step, __fsqrt_rn(ray.direction[0] * ray.direction[0] + ray.direction[2] * ray.direction[2]));
    uint32_t evaluations = 0, iterations = 0, unconverged = 0, status = OCEAN_RAY_MISS;
    // One evaluation per trip, so that ray_gap is inlined once.  March: a = the previous sample.  Refinement: [a, b] is the
    // bracket, wa / wb its Illinois weights, last = 1 (2) when the previous step replaced a (b).
    RayPoint a = {}, b = {}, rep = {};
    bool above = false, refining = false;
    float t = t_in, base_x = 0.0f, base_z = 0.0f, base_px = 0.0f, base_pz = 0.0f, wa = 0.0f, wb = 0.0f;
    int k = 0, steps = 0, last = 0;
    for (;;) {
        const RayPoint e = ray_gap<Wake>(displacement, N, C, scales, ray, t, evaluations > 0, base_x, base_z, base_px, base_pz, tol,
                                         max_iterations, rho, iterations, unconverged, w);
        ++evaluations;
        if (isnan(e.g)) { status = OCEAN_RAY_INVALID; rep = e; break; }
        if (!refining) {
            const bool side = e.g > 0.0f;
            if (k == 0) above = side;
            if (k == 0 || side == above) {
                rep = e;
                if (t == t_out) break;                                      // MISS
                if (evaluations == (uint32_t)max_samples) { status = OCEAN_RAY_TRUNCATED; break; }
                ++k;
                float tn = t_in + (float)k * h;
                if (!(tn < t_out)) tn = t_out;
                if (!isfinite(tn)) break;                                   // MISS
                a = e;
                t = tn;
                base_x = e.x; base_z = e.z; base_px = e.px; base_pz = e.pz;
                continue;
            }
            refining = true;
            b = e;
            wa = a.g;
            wb = b.g;
            status = above ? OCEAN_RAY_HIT_FROM_ABOVE : OCEAN_RAY_HIT_FROM_BELOW;
        } else {
            ++steps;
            if ((e.g > 0.0f) == above) {
                if (last == 1) wb = wb * 0.5f;
                a = e; wa = e.g; last = 1;
            } else {
                if (last == 2) wa = wa * 0.5f;
                b = e; wb = e.g; last = 2;
            }
        }
        rep = fabsf(a.g) <= fabsf(b.g) ? a : b;
        if (steps == kRayRefineSteps || fabsf(a.g) <= tol || fabsf(b.g) <= tol) break;
        const float w = __fdiv_rn(wa, wa - wb);
        const float tn = a.t + w * (b.t - a.t);
        if (!(tn > a.t && tn < b.t)) break;
        const bool near_a = (tn - a.t) <= (b.t - tn);
        base_x = near_a ? a.x : b.x; base_z = near_a ? a.z : b.z; base_px = near_a ? a.px : b.px; base_pz = near_a ? a.pz : b.pz;
        t = tn;
    }
    float3 d, g;
    sample_point(displacement, normal, N, C, make_float2(rep.px, rep.pz), scales, d, g);
    if constexpr (Wake) {
        float r[3] = {0.0f, 0.0f, 0.0f};
        sample_field<true>(w.field, w.n, w.cell, w.x0, w.z0, make_float2(rep.x, rep.z), r);
        d.y = __fadd_rn(d.y, r[0]);
        g.x = __fadd_rn(g.x, r[1]);
        g.y = __fadd_rn(g.y, r[2]);
    }
    hit.t = rep.t;
    hit.position[0] = rep.x; hit.position[1] = rep.y; hit.position[2] = rep.z;
    hit.source_x = rep.px;
    hit.source_z = rep.pz;
    hit.displacement[0] = d.x; hit.displacement[1] = d.y; hit.displacement[2] = d.z;
    hit.gradient_foam[0] = g.x; hit.gradient_foam[1] = g.y; hit.gradient_foam[2] = g.z;
    hit.gap = rep.g;
    hit.residual = rep.r;
    hit.status = status;
    hit.evaluations = evaluations;
    hit.iterations = iterations;
    hit.unconverged = unconverged;
    out[i] = hit;
}

}  // namespace

cudaError_t launch_sample_maps(const DeviceBuffers& b, int num_cascades, const float2* points_dev, int n, const float4* scales_dev,
                               float* disp_out_dev, float* grad_out_dev, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    k_sample_maps<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(b.displacement, b.normal, b.map_size, num_cascades, points_dev, n, scales_dev,
                                                                  disp_out_dev, grad_out_dev);
    return cudaGetLastError();
}

cudaError_t launch_sample_velocity(const uint2* velocity_dev, int map_size, int num_cascades, const float2* points_dev, int n,
                                   const float4* scales_dev, float* out_dev, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    k_sample_velocity<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(velocity_dev, map_size, num_cascades, points_dev, n, scales_dev, out_dev);
    return cudaGetLastError();
}

size_t surface_scratch_ints(int num_cascades, int n) { return 1 + (size_t)num_cascades + (size_t)n; }

// scratch_dev: [surface_scratch_ints(num_cascades, n)] ints = pending count, per-layer displacement maxima, pending list.
// Kernels: k_surface_first over all queries; with max_iterations > 0 also k_surface_bound (rho) and k_surface_restart over
// the pending list, whose length only the device knows: a grid-stride loop on a grid sized for up to one query per thread.
cudaError_t launch_query_surface(const DeviceBuffers& b, int num_cascades, const float2* points_dev, int n, const float4* scales_dev,
                                 float tolerance, int max_iterations, ocean_surface_sample* out_dev, int* scratch_dev, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    const int N = b.map_size;
    int* count = scratch_dev;
    unsigned* layer_max = reinterpret_cast<unsigned*>(scratch_dev + 1);
    int* pending = scratch_dev + 1 + num_cascades;
    cudaError_t e = cudaMemsetAsync(scratch_dev, 0, sizeof(int) * (size_t)(1 + num_cascades), stream);
    if (e != cudaSuccess) return e;
    k_surface_first<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(b.displacement, b.normal, N, num_cascades, points_dev, n, scales_dev,
                                                                    tolerance, max_iterations, out_dev, count, pending);
    if ((e = cudaGetLastError()) != cudaSuccess || max_iterations == 0) return e;
    const unsigned bound_blocks = (unsigned)(((size_t)N * N + 4095) / 4096);     // 16 texels per thread
    k_surface_bound<<<dim3(bound_blocks, (unsigned)num_cascades), 256, 0, stream>>>(b.displacement, N, layer_max);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    const int restart_blocks = (n + kRestartBlock - 1) / kRestartBlock < 2048 ? (n + kRestartBlock - 1) / kRestartBlock : 2048;
    k_surface_restart<<<restart_blocks, kRestartBlock, 0, stream>>>(b.displacement, b.normal, N, num_cascades, points_dev, scales_dev, tolerance,
                                                                   max_iterations, out_dev, count, pending, layer_max);
    return cudaGetLastError();
}

// bounds_dev: [3 * num_cascades] unsigned (+ 2 with a wake), cleared here, then filled by k_raycast_bound (and
// k_raycast_wake_bound, e is taken per call: it changes with every step call); k_raycast reads them.
cudaError_t launch_raycast(const DeviceBuffers& b, int num_cascades, const ocean_ray* rays_dev, int n, const float4* scales_dev, float step,
                           int max_samples, float tolerance, int max_iterations, unsigned* bounds_dev, ocean_ray_hit* out_dev,
                           const WakeRead* wake, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    const int N = b.map_size;
    cudaError_t e = cudaMemsetAsync(bounds_dev, 0, sizeof(unsigned) * (3 * (size_t)num_cascades + (wake ? 2 : 0)), stream);
    if (e != cudaSuccess) return e;
    const unsigned bound_blocks = (unsigned)(((size_t)N * N + 4095) / 4096);     // 16 texels per thread
    k_raycast_bound<<<dim3(bound_blocks, (unsigned)num_cascades), 256, 0, stream>>>(b.displacement, N, bounds_dev);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    const unsigned ray_blocks = (unsigned)((n + 127) / 128);
    if (!wake) {
        k_raycast<false><<<ray_blocks, 128, 0, stream>>>(b.displacement, b.normal, N, num_cascades, rays_dev, n, scales_dev, step, max_samples,
                                                         tolerance, max_iterations, bounds_dev, out_dev, WakeRead{});
        return cudaGetLastError();
    }
    const unsigned wake_blocks = (unsigned)(((size_t)wake->n * wake->n + 4095) / 4096);    // 16 cells per thread
    k_raycast_wake_bound<<<wake_blocks, 256, 0, stream>>>(wake->field, wake->n, bounds_dev + 3 * num_cascades);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    k_raycast<true><<<ray_blocks, 128, 0, stream>>>(b.displacement, b.normal, N, num_cascades, rays_dev, n, scales_dev, step, max_samples,
                                                    tolerance, max_iterations, bounds_dev, out_dev, *wake);
    return cudaGetLastError();
}

}  // namespace ocean
