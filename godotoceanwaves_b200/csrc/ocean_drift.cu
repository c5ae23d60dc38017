// ocean_drift.cu -- the sea state (spectral moments of each cascade's spectrum texture) and the drifters (Lagrangian labels
// that drift with the spectrum's Stokes drift, a current and windage, rendered on the displaced surface).  include/ocean.h,
// ocean_get_sea_state and ocean_drift; oracle/sea_state.py and oracle/drifters.py are the specifications, bit for bit.
//
// Sea state: two kernels per launch of up to kMaxSeaStateLaunch cascades.
//   k_sea_state_partial   per cascade sea_state_blocks(N) blocks of 256 threads; thread t of the cascade sums the terms of
//                         texels t, t + T, t + 2T, ... (T = 256 * blocks = N^2 / 16) in binary64 from +0, then a warp shuffle
//                         tree (lane l += lane l + 16, + 8, + 4, + 2, + 1) and the 8 warp sums in warp order from +0
//   k_sea_state_finish    the block sums of a cascade in block order from +0, into the cascade's cached moments
// No floating-point atomics: the result is a function of the spectrum and the table alone.
//
// Drifters: one thread per drifter, k_drift.  Binary64 where the label moves, binary32 (explicit _rn operations, no
// contraction) where it samples and renders, as ocean_sample.cu.
#include "ocean_kernels.cuh"
#include "ocean_texture.cuh"
#include "wake_sample.cuh"
#include "detmath.cuh"

namespace ocean {

namespace {

constexpr int kSeaStateThreads = 256;
constexpr float kDepthF = 20.0f;      // wave_generator.gd:6, the depth of every dispersion table

struct SeaStateTable {                // jobs of one launch, by value (constant bank)
    SeaStateJob d[kMaxSeaStateLaunch];
};

// The kSeaStateMoments terms of texel i = y N + x (oracle/sea_state.py, texel_terms); false for an excluded texel.
__device__ __forceinline__ bool sea_state_terms(const float4* __restrict__ spec, const float4* __restrict__ tab, const float* __restrict__ kvyt,
                                                int N, int i, double (&t)[kSeaStateMoments]) {
    const int y = i / N, x = i & (N - 1);
    float omega, kvx, kvy, kux, kuy;
    if (y <= N / 2) {
        const float4 e = __ldg(&tab[(size_t)y * N + x]);
        omega = e.x; kvx = e.y; kuy = e.z; kux = e.w;
        kvy = __ldg(&kvyt[y]);
    } else {
        // the mirror row: same omega, k_vec and k_unit negated -- except in column 0, which is its own mirror along x
        const int ym = N - y, xm = (N - x) & (N - 1);
        const float4 e = __ldg(&tab[(size_t)ym * N + xm]);
        omega = e.x;
        kvx = (x == 0) ? e.y : -e.y;
        kux = (x == 0) ? e.w : -e.w;
        kuy = -e.z;
        kvy = -__ldg(&kvyt[ym]);
    }
    const float k = __fadd_rn(__fsqrt_rn(__fadd_rn(__fmul_rn(kvx, kvx), __fmul_rn(kvy, kvy))), 1e-6f);   // spectrum_modulate.glsl:60
    const float4 a = __ldg(&spec[i]);
    const double ax = (double)a.x, ay = (double)a.y;
    const double E = __dmul_rn(2.0, __dadd_rn(__dmul_rn(ax, ax), __dmul_rn(ay, ay)));
    const double q = (double)detmath::expf_det(-__fmul_rn(__fmul_rn(2.0f, k), kDepthF));
    const double omq = __dsub_rn(1.0, q);
    if ((x == N / 2 && y == N / 2) || E == 0.0 || omq == 0.0) return false;
    const double w = (double)omega, kd = (double)k;
    const double dx = -(double)kuy, dz = -(double)kux;          // direction of travel, world (x, z)
    const double kx = (double)kvy, kz = (double)kvx;            // world wave vector (the maps are the transpose)
    t[0] = __ddiv_rn(E, w);
    t[1] = E;
    t[2] = __dmul_rn(w, E);
    t[3] = __dmul_rn(__dmul_rn(w, w), E);
    t[4] = __dmul_rn(E, dx);
    t[5] = __dmul_rn(E, dz);
    t[6] = __dmul_rn(E, __dmul_rn(kx, kx));
    t[7] = __dmul_rn(E, __dmul_rn(kz, kz));
    const double F = __ddiv_rn(__dadd_rn(1.0, __dmul_rn(q, q)), __dmul_rn(omq, omq));
    const double c = __dmul_rn(__dmul_rn(__dmul_rn(__dmul_rn(2.0, w), kd), E), F);
    t[8] = __dmul_rn(c, dx);
    t[9] = __dmul_rn(c, dz);
    return true;
}

__global__ void __launch_bounds__(kSeaStateThreads) k_sea_state_partial(const float4* __restrict__ spectrum, const float4* __restrict__ table,
                                                                        const float* __restrict__ kvy, int N, double* __restrict__ partial,
                                                                        const __grid_constant__ SeaStateTable jobs) {
    const SeaStateJob j = jobs.d[blockIdx.y];
    const float4* spec = spectrum + (size_t)j.cascade * N * N;
    const float4* tab = table + (size_t)j.table_slot * (N / 2 + 1) * N;
    const float* kvyt = kvy + (size_t)j.table_slot * N;
    const int T = gridDim.x * kSeaStateThreads;
    double acc[kSeaStateMoments];
#pragma unroll
    for (int m = 0; m < kSeaStateMoments; ++m) acc[m] = 0.0;
    for (int i = blockIdx.x * kSeaStateThreads + threadIdx.x; i < N * N; i += T) {
        double t[kSeaStateMoments];
        if (!sea_state_terms(spec, tab, kvyt, N, i, t)) continue;
#pragma unroll
        for (int m = 0; m < kSeaStateMoments; ++m) acc[m] = __dadd_rn(acc[m], t[m]);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1)
#pragma unroll
        for (int m = 0; m < kSeaStateMoments; ++m) acc[m] = __dadd_rn(acc[m], __shfl_down_sync(0xffffffffu, acc[m], off));
    __shared__ double warp_sum[kSeaStateThreads / 32][kSeaStateMoments];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0)
#pragma unroll
        for (int m = 0; m < kSeaStateMoments; ++m) warp_sum[warp][m] = acc[m];
    __syncthreads();
    if (threadIdx.x < kSeaStateMoments) {
        double s = 0.0;
        for (int w = 0; w < kSeaStateThreads / 32; ++w) s = __dadd_rn(s, warp_sum[w][threadIdx.x]);
        partial[((size_t)blockIdx.y * gridDim.x + blockIdx.x) * kSeaStateMoments + threadIdx.x] = s;
    }
}

__global__ void __launch_bounds__(32) k_sea_state_finish(const double* __restrict__ partial, int blocks, double* __restrict__ moments,
                                                         const __grid_constant__ SeaStateTable jobs) {
    if (threadIdx.x >= kSeaStateMoments) return;
    const double* p = partial + (size_t)blockIdx.x * blocks * kSeaStateMoments + threadIdx.x;
    double s = 0.0;
    for (int b = 0; b < blocks; ++b) s = __dadd_rn(s, p[(size_t)b * kSeaStateMoments]);
    moments[(size_t)jobs.d[blockIdx.x].cascade * kSeaStateMoments + threadIdx.x] = s;
}

// normalize(v) = v / sqrt((v.x v.x + v.y v.y) + v.z v.z)
__device__ __forceinline__ float3 normalize3(float3 v) {
    const float l = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)), __fmul_rn(v.z, v.z)));
    return make_float3(__fdiv_rn(v.x, l), __fdiv_rn(v.y, l), __fdiv_rn(v.z, l));
}

// One drifter (oracle/drifters.py, drift): advance (dt > 0), wrap, and with kRender the MultiMesh instance.
template <bool kRender, bool kWake>
__global__ void __launch_bounds__(256) k_drift(const uint2* __restrict__ displacement, const uint2* __restrict__ normal, int N, int C,
                                               const float4* __restrict__ scales, const double* __restrict__ moments,
                                               const ocean_drift_params p, double dt, ocean_drifter* __restrict__ drifters, int n,
                                               float* __restrict__ instances, const WakeRead wake) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ocean_drifter d = drifters[i];
    if (dt > 0.0) {
        // the total Stokes drift of the surface as rendered: sum_c s_c^2 u_s,c in cascade order
        double usx = 0.0, usz = 0.0;
        for (int c = 0; c < C; ++c) {
            const double s = (double)__ldg(&scales[c]).z, s2 = __dmul_rn(s, s);
            usx = __dadd_rn(usx, __dmul_rn(s2, moments[(size_t)c * kSeaStateMoments + 8]));
            usz = __dadd_rn(usz, __dmul_rn(s2, moments[(size_t)c * kSeaStateMoments + 9]));
        }
        const double ss = (double)p.stokes_scale, wg = (double)d.windage;
        const double ux = __dadd_rn(__dadd_rn(__dmul_rn(ss, usx), (double)p.current[0]), __dmul_rn(wg, (double)p.wind[0]));
        const double uz = __dadd_rn(__dadd_rn(__dmul_rn(ss, usz), (double)p.current[1]), __dmul_rn(wg, (double)p.wind[1]));
        d.x = __dadd_rn(d.x, __dmul_rn(dt, ux));
        d.z = __dadd_rn(d.z, __dmul_rn(dt, uz));
        d.yaw = (float)__dadd_rn((double)d.yaw, __dmul_rn(dt, (double)d.yaw_rate));
        if (p.flags & OCEAN_DRIFT_WRAP) {
            const double rx = __dsub_rn(d.x, p.box[0]), rz = __dsub_rn(d.z, p.box[1]);
            d.x = __dadd_rn(p.box[0], __dsub_rn(rx, __dmul_rn(p.box[2], floor(__ddiv_rn(rx, p.box[2])))));
            d.z = __dadd_rn(p.box[1], __dsub_rn(rz, __dmul_rn(p.box[3], floor(__ddiv_rn(rz, p.box[3])))));
        }
        drifters[i] = d;
    }
    if constexpr (kRender) {
        float3 D, g;
        sample_point(displacement, normal, N, C, make_float2((float)d.x, (float)d.z), scales, D, g);
        const float X = (float)__dadd_rn(d.x, (double)D.x), Z = (float)__dadd_rn(d.z, (double)D.z);
        double y = (double)D.y;
        if constexpr (kWake) {
            float r[3] = {0.0f, 0.0f, 0.0f};
            sample_field<true>(wake.field, wake.n, wake.cell, wake.x0, wake.z0, make_float2(X, Z), r);
            y = __dadd_rn(y, (double)r[0]);
            g.x = __fadd_rn(g.x, r[1]);
            g.y = __fadd_rn(g.y, r[2]);
        }
        const float Y = (float)__dadd_rn(y, (double)d.offset);
        const float3 nrm = normalize3(make_float3(-g.x, 1.0f, -g.y));                        // water.gdshader:90
        const float3 ny = normalize3(make_float3(__fadd_rn(0.0f, __fmul_rn(d.tilt, __fsub_rn(nrm.x, 0.0f))),
                                                 __fadd_rn(1.0f, __fmul_rn(d.tilt, __fsub_rn(nrm.y, 1.0f))),
                                                 __fadd_rn(0.0f, __fmul_rn(d.tilt, __fsub_rn(nrm.z, 0.0f)))));
        float sn, cs;
        detmath::sincosf_det(d.yaw, sn, cs);
        // the yaw direction (the z column of Basis(UP, yaw)) projected onto the plane normal to ny
        const float f_n = __fadd_rn(__fadd_rn(__fmul_rn(sn, ny.x), __fmul_rn(0.0f, ny.y)), __fmul_rn(cs, ny.z));
        const float3 nz = normalize3(make_float3(__fsub_rn(sn, __fmul_rn(f_n, ny.x)), __fsub_rn(0.0f, __fmul_rn(f_n, ny.y)),
                                                 __fsub_rn(cs, __fmul_rn(f_n, ny.z))));
        const float3 nx = make_float3(__fsub_rn(__fmul_rn(ny.y, nz.z), __fmul_rn(ny.z, nz.y)),
                                      __fsub_rn(__fmul_rn(ny.z, nz.x), __fmul_rn(ny.x, nz.z)),
                                      __fsub_rn(__fmul_rn(ny.x, nz.y), __fmul_rn(ny.y, nz.x)));
        const float s = d.scale;
        float* o = instances + (size_t)i * 12;
        o[0] = __fmul_rn(nx.x, s); o[1] = __fmul_rn(ny.x, s); o[2] = __fmul_rn(nz.x, s); o[3] = X;
        o[4] = __fmul_rn(nx.y, s); o[5] = __fmul_rn(ny.y, s); o[6] = __fmul_rn(nz.y, s); o[7] = Y;
        o[8] = __fmul_rn(nx.z, s); o[9] = __fmul_rn(ny.z, s); o[10] = __fmul_rn(nz.z, s); o[11] = Z;
    }
}

}  // namespace

int sea_state_blocks(int map_size) { return map_size * map_size / (16 * kSeaStateThreads); }

cudaError_t launch_sea_state(const DeviceBuffers& b, const SeaStateJob* jobs_host, int count, double* partial_dev, double* moments_dev,
                             cudaStream_t stream, int* launched) {
    if (launched) *launched = 0;
    const int blocks = sea_state_blocks(b.map_size);
    for (int first = 0; first < count; first += kMaxSeaStateLaunch) {
        const int n = (count - first < kMaxSeaStateLaunch) ? count - first : kMaxSeaStateLaunch;
        SeaStateTable jobs;
        for (int i = 0; i < n; ++i) jobs.d[i] = jobs_host[first + i];
        k_sea_state_partial<<<dim3(blocks, n), kSeaStateThreads, 0, stream>>>(b.spectrum, b.disp_table, b.disp_kvy, b.map_size, partial_dev, jobs);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        k_sea_state_finish<<<n, 32, 0, stream>>>(partial_dev, blocks, moments_dev, jobs);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        if (launched) *launched += 2;
    }
    return cudaSuccess;
}

cudaError_t launch_drift(const DeviceBuffers& b, int num_cascades, const float4* scales_dev, const double* moments_dev,
                         const ocean_drift_params& params, double dt, ocean_drifter* drifters_dev, int n, float* instances_dev,
                         const WakeRead* wake, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    const dim3 grid((n + 255) / 256);
    const WakeRead w = wake ? *wake : WakeRead{};
    if (!instances_dev)
        k_drift<false, false><<<grid, 256, 0, stream>>>(b.displacement, b.normal, b.map_size, num_cascades, scales_dev, moments_dev, params, dt,
                                                        drifters_dev, n, nullptr, w);
    else if (wake)
        k_drift<true, true><<<grid, 256, 0, stream>>>(b.displacement, b.normal, b.map_size, num_cascades, scales_dev, moments_dev, params, dt,
                                                      drifters_dev, n, instances_dev, w);
    else
        k_drift<true, false><<<grid, 256, 0, stream>>>(b.displacement, b.normal, b.map_size, num_cascades, scales_dev, moments_dev, params, dt,
                                                       drifters_dev, n, instances_dev, w);
    return cudaGetLastError();
}

}  // namespace ocean
