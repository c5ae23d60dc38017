// ocean_spray.cu -- foam-driven spray candidates as a stream-compaction op (SURVEY 8f row f3).
//
// Reference: assets/shaders/spatial/sea_spray_particle.gdshader
//   process() :80-94   gradient = sum_i texture(normals, vec3(START_POS.xz * map_scales[i].xy, i)).xyw
//                      normal = normalize(vec3(-gradient.x, 1, -gradient.y)), foam = gradient.z
//                      normal_factor / foam_factor = mix(0.25, 1, min((v - lo) / (hi - lo), 1)),  ACTIVE = factors in range && foam > 0.9
//                      SCALE_FACTOR, PARTICLE_SCALE
// The reference runs this for every particle of the emitter and culls the inactive ones (README.md:29: "most particles are
// culled"); here the candidates are evaluated once and only the active ones are written out, in candidate order:
//   pass 1  one thread per candidate: evaluate, count the active ones per block of 256
//   scan    exclusive prefix sum of the block counts (one block)
//   pass 2  evaluate again (four texel gathers per cascade, L2-resident) and write the record at its final position
//           (block offset + rank inside the block from warp ballots) -- a STABLE compaction, deterministic output.
// Numeric policy: oracle/spray.py is the specification (binary32, shader operation order, no contraction, -fmad=false).
//
// The particle op (ocean_spray_particles, oracle/spray_particles.py) runs the same shader's start() and process() on an
// emitter's particle states, kept in device memory, and writes the live particles as MultiMesh instances:
//   update  one thread per particle: the restart schedule (binary64), start(), process() and the state write; the live
//           particles are counted per block of 256
//   scan    k_spray_scan on the block counts
//   write   the instances of the live particles at block offset + rank (warp ballots): a stable compaction in INDEX order
//
// The wake forms of k_spray_count, k_spray_write and k_spray_particles_update (ocean_wake_set_readers; oracle/wake_readers.py)
// add the wake layer's slopes and foam F at START_POS.xz to the spawn test's gradient and foam, and its height h to the
// particle's height: spray from the white water the render map shows on the wake.  Same launches.
#include "../../include/ocean.h"
#include "ocean_kernels.cuh"
#include "ocean_texture.cuh"
#include "detmath.cuh"
#include "wake_sample.cuh"

namespace ocean {

namespace {

struct SprayEval {
    bool active;
    float scale_factor, psx, psy, psz, foam;
};

struct SprayFactors {
    float normal_factor, foam_factor, foam;
};

// :80-87: the gradient and foam at START_POS.xz, and the two factors; with Wake plus the wake's (dh/dx, dh/dz) and F there
template <bool Wake>
__device__ __forceinline__ SprayFactors spray_factors(const uint2* __restrict__ normal, int N, int C, float2 p,
                                                      const float4* __restrict__ scales, const WakeRead& w) {
    float gx = 0.0f, gy = 0.0f, gf = 0.0f;
    for (int c = 0; c < C; ++c) {
        const float4 s = __ldg(&scales[c]);
        const float4 t = texture_bilinear(normal + (size_t)c * N * N, N, p.x * s.x, p.y * s.y);     // :83
        gx = gx + t.x;
        gy = gy + t.y;
        gf = gf + t.w;
    }
    if constexpr (Wake) {
        float r[3] = {0.0f, 0.0f, 0.0f}, fw = 0.0f;
        sample_field<true>(w.field, w.n, w.cell, w.x0, w.z0, p, r);
        if (w.foam) sample_field<false>(w.foam, w.n, w.cell, w.x0, w.z0, p, &fw);
        gx = gx + r[1];
        gy = gy + r[2];
        gf = gf + fw;
    }
    const float nx = -gx, nz = -gy;
    const float ny = __fdiv_rn(1.0f, __fsqrt_rn((nx * nx + 1.0f * 1.0f) + nz * nz));               // normalize(...).y  :84
    SprayFactors f;
    f.normal_factor = mixf(0.25f, 1.0f, fminf(__fdiv_rn(ny - 0.92f, 0.99f - 0.92f), 1.0f));        // :86
    f.foam_factor = mixf(0.25f, 1.0f, fminf(__fdiv_rn(gf - 0.9f, 1.0f - 0.9f), 1.0f));             // :87
    f.foam = gf;
    return f;
}

template <bool Wake>
__device__ __forceinline__ SprayEval spray_eval(const uint2* __restrict__ normal, int N, int C, float2 p, const float4* __restrict__ scales,
                                                float3 particle_scale, const WakeRead& w) {
    const SprayFactors f = spray_factors<Wake>(normal, N, C, p, scales, w);
    const float nf = f.normal_factor, ff = f.foam_factor, gf = f.foam;
    SprayEval e;
    e.active = nf >= 0.0f && nf <= 1.0f && gf > 0.9f;                                               // :89
    e.scale_factor = nf * ff;                                                                       // :90
    const float s0 = ff * (1.0f + 1e-3f);                                                           // :92
    e.psx = (s0 * 1.0f) * particle_scale.x;                                                         // :93-94
    e.psy = (s0 * nf) * particle_scale.y;
    e.psz = (s0 * 1.0f) * particle_scale.z;
    e.foam = gf;
    return e;
}

constexpr int kSprayBlock = 256;

template <bool Wake>
__global__ void __launch_bounds__(kSprayBlock) k_spray_count(const uint2* __restrict__ normal, int N, int C, const float2* __restrict__ points, int n,
                                                             const float4* __restrict__ scales, float3 particle_scale, int* __restrict__ block_counts,
                                                             const WakeRead w) {
    const int i = blockIdx.x * kSprayBlock + threadIdx.x;
    bool active = false;
    if (i < n) active = spray_eval<Wake>(normal, N, C, points[i], scales, particle_scale, w).active;
    const int total = __syncthreads_count(active);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = total;
}

// exclusive scan of `blocks` counts in place; counts[blocks] receives the total
__global__ void __launch_bounds__(1024) k_spray_scan(int* __restrict__ counts, int blocks) {
    __shared__ int s_warp[32];
    __shared__ int s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < blocks; base += 1024) {
        const int i = base + threadIdx.x;
        const int v = (i < blocks) ? counts[i] : 0;
        int incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, d);
            if ((threadIdx.x & 31) >= d) incl += t;
        }
        if ((threadIdx.x & 31) == 31) s_warp[threadIdx.x >> 5] = incl;
        __syncthreads();
        if (threadIdx.x < 32) {
            int w = s_warp[threadIdx.x];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, w, d);
                if (threadIdx.x >= d) w += t;
            }
            s_warp[threadIdx.x] = w;
        }
        __syncthreads();
        const int warp_off = (threadIdx.x >> 5) ? s_warp[(threadIdx.x >> 5) - 1] : 0;
        const int carry = s_carry;
        if (i < blocks) counts[i] = carry + warp_off + incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = carry + warp_off + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) counts[blocks] = s_carry;
}

template <bool Wake>
__global__ void __launch_bounds__(kSprayBlock) k_spray_write(const uint2* __restrict__ normal, int N, int C, const float2* __restrict__ points, int n,
                                                             const float4* __restrict__ scales, float3 particle_scale,
                                                             const int* __restrict__ block_offsets, ocean_spray_record* __restrict__ out,
                                                             int max_records, const WakeRead w) {
    __shared__ int s_warp[kSprayBlock / 32];
    const int i = blockIdx.x * kSprayBlock + threadIdx.x;
    SprayEval e;
    e.active = false;
    float2 p = make_float2(0.f, 0.f);
    if (i < n) {
        p = points[i];
        e = spray_eval<Wake>(normal, N, C, p, scales, particle_scale, w);
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, e.active);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    int off = block_offsets[blockIdx.x];
    for (int w = 0; w < warp; ++w) off += s_warp[w];
    off += __popc(ballot & ((1u << lane) - 1u));
    if (e.active && off < max_records) {
        ocean_spray_record r;
        r.index = (uint32_t)i;
        r.start_x = p.x;
        r.start_z = p.y;
        r.scale_factor = e.scale_factor;
        r.particle_scale[0] = e.psx;
        r.particle_scale[1] = e.psy;
        r.particle_scale[2] = e.psz;
        r.foam = e.foam;
        out[off] = r;
    }
}

// ---- the particle op ----

// :32-38
__device__ __forceinline__ float3 spray_hash32(uint32_t px, uint32_t py) {
    const uint32_t M = 1103515245u;
    const uint32_t x = M * ((px >> 1) ^ py), y = M * ((py >> 1) ^ px);
    const uint32_t h = M * (x ^ (y >> 3));
    const uint32_t n = h ^ (h >> 16);
    const float d = 2147483648.0f;                       // float(0x7FFFFFFF)
    return make_float3(__fdiv_rn(__uint2float_rn(n >> 1), d), __fdiv_rn(__uint2float_rn((n * 16807u) >> 1), d),
                       __fdiv_rn(__uint2float_rn((n * 48271u) >> 1), d));
}

// :39-43: basis column c = normalize(column c) * s_c
__device__ __forceinline__ void spray_set_scale(float* T, float sx, float sy, float sz) {
    const float s[3] = {sx, sy, sz};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float x = T[c], y = T[4 + c], z = T[8 + c];
        const float n = __fsqrt_rn((x * x + y * y) + z * z);
        T[c] = __fdiv_rn(x, n) * s[c];
        T[4 + c] = __fdiv_rn(y, n) * s[c];
        T[8 + c] = __fdiv_rn(z, n) * s[c];
    }
}

// :69-72
__device__ __forceinline__ float exp_impulse(float x, float k) {
    const float h = k * x;
    return h * detmath::expf_det(1.0f - h);
}

// r_k = L * ((double)k + (double)i / (double)amount)
__device__ __forceinline__ double restart_time(double L, long long k, double f) { return __dmul_rn(L, __dadd_rn((double)k, f)); }

// The cycle k of particle i's restart in [t0, t1), -1 for none: the largest k >= 0 with t0 <= r_k < t1.  r_k does not
// decrease with k, so the largest k with r_k < t1 is reached from an estimate by unit steps (t1 / L < 2^32 is validated).
__device__ __forceinline__ long long restart_cycle(double L, double f, double t0, double t1) {
    long long k = (long long)fmax(floor(__dadd_rn(__ddiv_rn(t1, L), -f)), -1.0);
    while (restart_time(L, k + 1, f) < t1) ++k;
    while (k >= 0 && restart_time(L, k, f) >= t1) --k;
    return (k >= 0 && restart_time(L, k, f) >= t0) ? k : -1;
}

// start() :45-66, after the restart's reset of TRANSFORM and CUSTOM
__device__ __forceinline__ void spray_start(ocean_spray_particle& p, const ocean_spray_emitter& e, uint32_t index, float time) {
    const uint32_t u = __float2uint_rz(time);
    const float3 rand = spray_hash32(p.number + u + e.random_seed, 1u + u + e.random_seed);
    const uint32_t t = __float2uint_rz(__fsqrt_rn(__uint2float_rn((uint32_t)e.num_particles)));
    const float tm1 = __uint2float_rn(t) - 1.0f;
    const float cx = (__fdiv_rn(__uint2float_rn(index / t), tm1) - 0.5f) * 10.0f;
    const float cz = (__fdiv_rn(__uint2float_rn(index % t), tm1) - 0.5f) * 10.0f;
    // TRANSFORM = EMISSION_TRANSFORM * TRANSFORM, the identity basis with origin (cx, 0, cz), as sums in index order
    const float* E = e.emission_transform;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const float e0 = E[4 * r], e1 = E[4 * r + 1], e2 = E[4 * r + 2], e3 = E[4 * r + 3];
        p.transform[4 * r + 0] = ((e0 * 1.0f + e1 * 0.0f) + e2 * 0.0f) + e3 * 0.0f;
        p.transform[4 * r + 1] = ((e0 * 0.0f + e1 * 1.0f) + e2 * 0.0f) + e3 * 0.0f;
        p.transform[4 * r + 2] = ((e0 * 0.0f + e1 * 0.0f) + e2 * 1.0f) + e3 * 0.0f;
        p.transform[4 * r + 3] = ((e0 * cx + e1 * 0.0f) + e2 * cz) + e3 * 1.0f;
    }
    p.custom[2] = rand.x;
    const float pl = e.lifetime - (e.lifetime * e.lifetime_randomness) * rand.y;
    p.userdata2[3] = pl;
    p.userdata1[0] = p.transform[3];
    p.userdata1[1] = p.transform[7];
    p.userdata1[2] = p.transform[11];
    p.userdata1[3] = time + rand.z * ((float)e.emitter_lifetime - pl);
    p.userdata3[3] = 0.0f;
    p.transform[3] = 0.0f;
    p.transform[7] = -1e10f;
    p.transform[11] = 0.0f;
    spray_set_scale(p.transform, 1e-3f, 1e-3f, 1e-3f);
}

// process() :74-126 of an ACTIVE particle; with Wake the spawn test reads the wake and the height adds its h at START_POS.xz
template <bool Wake>
__device__ __forceinline__ void spray_process(ocean_spray_particle& p, const ocean_spray_emitter& e, float time,
                                              const uint2* __restrict__ disp, const uint2* __restrict__ normal, int N, int C,
                                              const float4* __restrict__ scales, const WakeRead& w) {
    const float st = p.userdata1[3], pl = p.userdata2[3];
    if (time > st + pl) {
        p.flags &= ~OCEAN_SPRAY_ACTIVE;
        return;
    }
    if (!(time >= st)) return;
    const float2 sp = make_float2(p.userdata1[0], p.userdata1[2]);
    if (p.userdata3[3] == 0.0f) {                                                                  // :78-96
        const SprayFactors f = spray_factors<Wake>(normal, N, C, sp, scales, w);
        const float nf = f.normal_factor, ff = f.foam_factor;
        const bool active = nf >= 0.0f && nf <= 1.0f && f.foam > 0.9f;
        p.flags = active ? (p.flags | OCEAN_SPRAY_ACTIVE) : (p.flags & ~OCEAN_SPRAY_ACTIVE);
        p.userdata3[2] = nf * ff;
        const float s0 = ff * ((active ? 1.0f : 0.0f) + 1e-3f);
        p.userdata2[0] = (s0 * 1.0f) * e.particle_scale[0];
        p.userdata2[1] = (s0 * nf) * e.particle_scale[1];
        p.userdata2[2] = (s0 * 1.0f) * e.particle_scale[2];
        p.userdata3[3] = 1.0f;
    }
    if (!(p.flags & OCEAN_SPRAY_ACTIVE)) return;
    const float t = __fdiv_rn(time - st, pl);                                                      // :99
    p.custom[3] = exp_impulse(t, 10.0f);
    float dx = 0.0f, dy = 0.0f, dz = 0.0f;
    for (int c = 0; c < C; ++c) {                                                                  // :105-108
        const float4 s = __ldg(&scales[c]);
        add_displacement(disp + (size_t)c * N * N, N, sp.x * s.x, sp.y * s.y, s.z, dx, dy, dz);
    }
    if constexpr (Wake) {
        float hw = 0.0f;
        sample_field<false>(w.field, w.n, w.cell, w.x0, w.z0, sp, &hw);
        dy = dy + hw;
    }
    dx = dx * 0.75f;                                                                               // :111
    dy = dy * 1.0f;
    dz = dz * 0.75f;
    const float a = 2.5f * t - 0.45f;                                                              // :114, pow(a, 2) = a * a
    dx = dx + 0.0f;
    dy = dy + ((-5.0f * (a * a)) * p.userdata3[2] + 0.5f);
    dz = dz + 0.0f;
    p.transform[3] = sp.x + dx;                                                                    // :115
    p.transform[7] = p.userdata1[1] + dy;
    p.transform[11] = sp.y + dz;
    const float size = __fdiv_rn(pl, e.lifetime);                                                  // :118-123
    const float m = size * size;
    const float my = m * exp_impulse(t, 3.0f);
    const float lg = detmath::logf_det(1.0f + t);
    const float mx = m * lg, mz = m * lg;
    spray_set_scale(p.transform, p.userdata2[0] * mx, p.userdata2[1] * my, p.userdata2[2] * mz);
}

__device__ __forceinline__ bool spray_live(const ocean_spray_particle& p) {
    return (p.flags & OCEAN_SPRAY_ACTIVE) && p.userdata3[3] != 0.0f;
}

template <bool Wake>
__global__ void __launch_bounds__(kSprayBlock) k_spray_particles_update(const ocean_spray_emitter e, double t0, double t1, float time,
                                                                        const uint2* __restrict__ disp, const uint2* __restrict__ normal,
                                                                        int N, int C, const float4* __restrict__ scales,
                                                                        ocean_spray_particle* __restrict__ states,
                                                                        int* __restrict__ block_counts, const WakeRead w) {
    const int i = blockIdx.x * kSprayBlock + threadIdx.x;
    bool live = false;
    if (i < e.amount) {
        ocean_spray_particle p = states[i];
        const double f = __ddiv_rn((double)i, (double)e.amount);
        const long long k = restart_cycle(e.emitter_lifetime, f, t0, t1);
        if (k >= 0) {
            p.number = (uint32_t)k * (uint32_t)e.amount + (uint32_t)i;
#pragma unroll
            for (int j = 0; j < 12; ++j) p.transform[j] = (j % 5 == 0) ? 1.0f : 0.0f;
#pragma unroll
            for (int j = 0; j < 4; ++j) p.custom[j] = 0.0f;
            p.flags |= OCEAN_SPRAY_ACTIVE | OCEAN_SPRAY_EMITTED;
            spray_start(p, e, (uint32_t)i, time);
        }
        if (p.flags & OCEAN_SPRAY_ACTIVE) spray_process<Wake>(p, e, time, disp, normal, N, C, scales, w);
        states[i] = p;
        live = spray_live(p);
    }
    const int total = __syncthreads_count(live);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kSprayBlock) k_spray_particles_write(const ocean_spray_particle* __restrict__ states, int n,
                                                                       const int* __restrict__ block_offsets, float* __restrict__ instances,
                                                                       int max_instances) {
    __shared__ int s_warp[kSprayBlock / 32];
    const int i = blockIdx.x * kSprayBlock + threadIdx.x;
    const bool live = i < n && spray_live(states[i]);
    const unsigned ballot = __ballot_sync(0xffffffffu, live);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    int off = block_offsets[blockIdx.x];
    for (int w = 0; w < warp; ++w) off += s_warp[w];
    off += __popc(ballot & ((1u << lane) - 1u));
    if (live && off < max_instances) {
        const ocean_spray_particle& p = states[i];
        float* o = instances + (size_t)off * 16;
#pragma unroll
        for (int j = 0; j < 12; ++j) o[j] = p.transform[j];
#pragma unroll
        for (int j = 0; j < 4; ++j) o[12 + j] = p.custom[j];
    }
}

}  // namespace

int spray_blocks(int n) { return (n + kSprayBlock - 1) / kSprayBlock; }

// counts_dev: [spray_blocks(n) + 1] ints of scratch; on completion counts_dev[spray_blocks(n)] = number of active
// candidates (which may exceed max_records: the records beyond it are dropped, the count is not clamped).
cudaError_t launch_extract_spray(const DeviceBuffers& b, int num_cascades, const float2* points_dev, int n, const float4* scales_dev,
                                 float3 particle_scale, int* counts_dev, ocean_spray_record* records_dev, int max_records,
                                 const WakeRead* wake, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    const int blocks = spray_blocks(n);
    const WakeRead w = wake ? *wake : WakeRead{};
    if (wake)
        k_spray_count<true><<<blocks, kSprayBlock, 0, stream>>>(b.normal, b.map_size, num_cascades, points_dev, n, scales_dev, particle_scale,
                                                                counts_dev, w);
    else
        k_spray_count<false><<<blocks, kSprayBlock, 0, stream>>>(b.normal, b.map_size, num_cascades, points_dev, n, scales_dev, particle_scale,
                                                                 counts_dev, w);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    k_spray_scan<<<1, 1024, 0, stream>>>(counts_dev, blocks);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    if (wake)
        k_spray_write<true><<<blocks, kSprayBlock, 0, stream>>>(b.normal, b.map_size, num_cascades, points_dev, n, scales_dev, particle_scale,
                                                                counts_dev, records_dev, max_records, w);
    else
        k_spray_write<false><<<blocks, kSprayBlock, 0, stream>>>(b.normal, b.map_size, num_cascades, points_dev, n, scales_dev, particle_scale,
                                                                 counts_dev, records_dev, max_records, w);
    return cudaGetLastError();
}

// counts_dev: [spray_blocks(amount) + 1] ints of scratch; on completion counts_dev[spray_blocks(amount)] = number of live
// particles (which may exceed max_instances: the instances beyond it are dropped, the count is not clamped).
cudaError_t launch_spray_particles(const DeviceBuffers& b, int num_cascades, const float4* scales_dev, const ocean_spray_emitter& emitter,
                                   double t0, double t1, ocean_spray_particle* states_dev, int* counts_dev, float* instances_dev,
                                   int max_instances, const WakeRead* wake, cudaStream_t stream) {
    if (emitter.amount <= 0) return cudaSuccess;
    const int blocks = spray_blocks(emitter.amount);
    const WakeRead w = wake ? *wake : WakeRead{};
    if (wake)
        k_spray_particles_update<true><<<blocks, kSprayBlock, 0, stream>>>(emitter, t0, t1, (float)t1, b.displacement, b.normal, b.map_size,
                                                                           num_cascades, scales_dev, states_dev, counts_dev, w);
    else
        k_spray_particles_update<false><<<blocks, kSprayBlock, 0, stream>>>(emitter, t0, t1, (float)t1, b.displacement, b.normal, b.map_size,
                                                                            num_cascades, scales_dev, states_dev, counts_dev, w);
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) return err;
    k_spray_scan<<<1, 1024, 0, stream>>>(counts_dev, blocks);
    err = cudaGetLastError();
    if (err != cudaSuccess) return err;
    k_spray_particles_write<<<blocks, kSprayBlock, 0, stream>>>(states_dev, emitter.amount, counts_dev, instances_dev, max_instances);
    return cudaGetLastError();
}

}  // namespace ocean
