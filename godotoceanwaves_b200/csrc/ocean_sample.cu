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
#include "ocean_kernels.cuh"
#include "ocean_texture.cuh"

namespace ocean {

namespace {

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
        const float4 d = texture_bilinear(displacement + layer, N, u, v);                         // :34-35
        dx = dx + d.x * s.z;
        dy = dy + d.y * s.z;
        dz = dz + d.z * s.z;
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

// ---- surface query: the surface at a world position (oracle/surface.py is the specification) ----
// The shader reads the maps at the undisplaced point P and moves the vertex to P + D_xz(P) (:28,37), so the query solves
// P + D_xz(P) = Q by damped Newton steps on the displacement layers, then samples the maps at P.

struct SurfaceSample {       // == ocean_surface_sample (include/ocean.h), 40 bytes
    float source_x, source_z;
    float displacement[3];
    float gradient_foam[3];
    float residual;
    uint32_t iterations;
};

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
                                              SurfaceSample* __restrict__ out) {
    float3 d, g;
    sample_point(displacement, normal, N, C, make_float2(px, pz), scales, d, g);
    SurfaceSample s;
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
                                                       int max_iterations, SurfaceSample* __restrict__ out, int* __restrict__ pending_count,
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
                                                         int max_iterations, SurfaceSample* __restrict__ out, const int* __restrict__ pending_count,
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

}  // namespace

cudaError_t launch_sample_maps(const DeviceBuffers& b, int num_cascades, const float2* points_dev, int n, const float4* scales_dev,
                               float* disp_out_dev, float* grad_out_dev, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    k_sample_maps<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(b.displacement, b.normal, b.map_size, num_cascades, points_dev, n, scales_dev,
                                                                  disp_out_dev, grad_out_dev);
    return cudaGetLastError();
}

size_t surface_scratch_ints(int num_cascades, int n) { return 1 + (size_t)num_cascades + (size_t)n; }

// scratch_dev: [surface_scratch_ints(num_cascades, n)] ints = pending count, per-layer displacement maxima, pending list.
// Kernels: k_surface_first over all queries; with max_iterations > 0 also k_surface_bound (rho) and k_surface_restart over
// the pending list, whose length only the device knows: a grid-stride loop on a grid sized for up to one query per thread.
cudaError_t launch_query_surface(const DeviceBuffers& b, int num_cascades, const float2* points_dev, int n, const float4* scales_dev,
                                 float tolerance, int max_iterations, void* out_dev, int* scratch_dev, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    const int N = b.map_size;
    SurfaceSample* out = static_cast<SurfaceSample*>(out_dev);
    int* count = scratch_dev;
    unsigned* layer_max = reinterpret_cast<unsigned*>(scratch_dev + 1);
    int* pending = scratch_dev + 1 + num_cascades;
    cudaError_t e = cudaMemsetAsync(scratch_dev, 0, sizeof(int) * (size_t)(1 + num_cascades), stream);
    if (e != cudaSuccess) return e;
    k_surface_first<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(b.displacement, b.normal, N, num_cascades, points_dev, n, scales_dev,
                                                                    tolerance, max_iterations, out, count, pending);
    if ((e = cudaGetLastError()) != cudaSuccess || max_iterations == 0) return e;
    const unsigned bound_blocks = (unsigned)(((size_t)N * N + 4095) / 4096);     // 16 texels per thread
    k_surface_bound<<<dim3(bound_blocks, (unsigned)num_cascades), 256, 0, stream>>>(b.displacement, N, layer_max);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    const int restart_blocks = (n + kRestartBlock - 1) / kRestartBlock < 2048 ? (n + kRestartBlock - 1) / kRestartBlock : 2048;
    k_surface_restart<<<restart_blocks, kRestartBlock, 0, stream>>>(b.displacement, b.normal, N, num_cascades, points_dev, scales_dev, tolerance,
                                                                   max_iterations, out, count, pending, layer_max);
    return cudaGetLastError();
}

}  // namespace ocean
