// ocean_velocity.cu -- velocity maps: the time derivative of the displacement map, computed on the device
// (include/ocean.h, ocean_update_velocity; oracle_velocity_update in oracle/velocity_oracle.c is the specification).
//
// h(t) = h0a e^{i w t} + h0b e^{-i w t}, so dh/dt = i w (h0a e^{i w t} - h0b e^{-i w t}): another inverse FFT of the same
// spectrum.  The three real fields (vx, vy, vz) pack as ONE layer pair -- layer 0 = vx + i vy, layer 1 = vz -- which is the
// C2 lane-pair form fft_core.cuh transforms, so a velocity layer costs half the FFT work of an update and has no foam
// read-modify-write.  Two kernels per launch of up to kMaxVelocityLaunch cascades:
//   k_velocity_rowfft   spectrum -> layer pair -> row IFFT -> scratch [C][N][N] float4 (re_0, re_1, im_0, im_1)
//   k_velocity_colfft   column IFFT -> sign_shift -> velocity map [C][N][N] 4 x half (+ binary32 tap)
// The map has the displacement map's orientation and layout, so ocean_texture.cuh samples it unchanged.
//
// Per texel, binary32, FMA only where the oracle's FMA mode has it (mul_complex), every other operation rounded on its own
// (-fmad=false):
//   w = dispersion table omega (bit-identical to sqrtf(G*k*tanh(k*depth)), spectrum_modulate.glsl:49)
//   m = sincos(w * time), pa = h0a * m, pb = h0b * conj(m), d = pa - pb
//   ht = (-(w*d.y), w*d.x),  hti = (-ht.y, ht.x),  vx = hti * k_unit.y,  vz = hti * k_unit.x
//   layer 0 = (vx.x - ht.y, vx.y + ht.x),  layer 1 = (vz.x, vz.y)
// The update's row pass derives a texel's mirror from the texel's own products (h(-k) == conj h(k)); for d = pa - pb that
// identity holds only up to the sign of exact zeros, so here every texel is evaluated from its own spectrum texel and its
// own k_unit.  Only the phase is shared: a texel and its mirror have the same omega bit for bit (k depends on k_vec^2),
// hence the same sincos.
#include "ocean_kernels.cuh"
#include "detmath.cuh"
#include "fft_core.cuh"

#include <cuda_fp16.h>

namespace ocean {

namespace {

// A team of THREADS threads transforms ROWS rows (row pass) or ROWS columns (column pass), T = N/16 threads per FFT.
template <int N>
struct VelTile {
    static constexpr int T = N / kE;
    static constexpr int ROWS = (128 / T) < 2 ? 2 : 128 / T;
    static constexpr int THREADS = ROWS * T;
    static constexpr int RB = N + N / 16;               // padded row buffer (float4 units), pad16 layout of fft_core.cuh
    static constexpr int CS = RB + 1;                   // column buffers: odd offset between the W columns of a row
    static constexpr size_t ROW_SMEM = sizeof(float4) * ROWS * RB + sizeof(float2) * N;
    static constexpr size_t COL_SMEM = sizeof(float4) * ROWS * CS + sizeof(float2) * N;
};

struct VelocityTable {      // dispatch records of one launch, by value (constant bank)
    VelocityDispatch d[kMaxVelocityLaunch];
};

__device__ __forceinline__ float2 mul_complex(float2 a, float2 b) {   // spectrum_modulate.glsl:37-39, FMA contraction mode
    return make_float2(__fmaf_rn(a.x, b.x, -(a.y * b.y)), __fmaf_rn(a.x, b.y, a.y * b.x));
}

// Layers 0 and 1 of one texel as the lanes of a C2 pair: (re_0, re_1, im_0, im_1).
__device__ __forceinline__ float4 velocity_texel(const float4 h0, float cs, float sn, float w, float kux, float kuy) {
    const float2 m = make_float2(cs, sn), mc = make_float2(cs, sn * -1.0f);
    const float2 pa = mul_complex(make_float2(h0.x, h0.y), m), pb = mul_complex(make_float2(h0.z, h0.w), mc);
    const float2 d = make_float2(pa.x - pb.x, pa.y - pb.y);
    const float2 ht = make_float2(-(w * d.y), w * d.x);
    const float2 hti = make_float2(-ht.y, ht.x);
    const float2 vx = make_float2(hti.x * kuy, hti.y * kuy);
    const float2 vz = make_float2(hti.x * kux, hti.y * kux);
    return make_float4(vx.x - ht.y, vz.x, vx.y + ht.x, vz.y);
}

template <int N>
__device__ __forceinline__ const float2* stage_twiddles(float2* tw_s, const float2* __restrict__ tw_g) {
    for (int i = threadIdx.x; i < N - 1; i += VelTile<N>::THREADS) tw_s[i] = __ldg(&tw_g[i]);
    return tw_s;
}

// Row pass.  A team holds RP = ROWS/2 mirror pairs of rows: pair q = (row q, row N-q) for q >= 1, pair 0 = rows 0 and N/2.
// Phase 1: the 2T threads of a pair evaluate texel (x, q) and its mirror ((N-x) mod N, N-q) with one sincos; rows 0 and
// N/2 mirror within themselves and are evaluated texel by texel.  Phase 2: one row IFFT per T consecutive threads.
template <int N>
__global__ void __launch_bounds__(VelTile<N>::THREADS) k_velocity_rowfft(const float4* __restrict__ spectrum, const float4* __restrict__ table,
                                                                      float4* __restrict__ scratch, const float2* __restrict__ tw_g,
                                                                      const __grid_constant__ VelocityTable jobs) {
    using VT = VelTile<N>;
    constexpr int T = VT::T, RB = VT::RB, RP = VT::ROWS / 2, SUB = 2 * T, ITER = N / SUB, TROWS = N / 2 + 1;
    static_assert(ITER % 4 == 0, "texels per thread");
    extern __shared__ float4 smem[];
    const float2* tw_s = stage_twiddles<N>(reinterpret_cast<float2*>(smem + VT::ROWS * RB), tw_g);
    const VelocityDispatch d = jobs.d[blockIdx.y];
    const int tid = threadIdx.x;
    const int ql = tid / SUB, xs = tid % SUB;
    const int q0 = blockIdx.x * RP, q = q0 + ql;
    float4* row_a = smem + (size_t)(2 * ql) * RB;        // row q (or row 0)
    float4* row_b = row_a + RB;                          // row N-q (or row N/2)
    const float4* spec = spectrum + (size_t)d.cascade * N * N;
    const float4* tab = table + (size_t)d.table_slot * TROWS * N;     // (omega, k_vec.x, k_unit.y, k_unit.x) of rows <= N/2
#pragma unroll
    for (int e0 = 0; e0 < ITER; e0 += 4) {
        float4 tb[4];
        float ph[4], sn[4], cs[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            tb[j] = __ldg(&tab[(size_t)q * N + xs + SUB * (e0 + j)]);
            ph[j] = tb[j].x * d.time;                                    // spectrum_modulate.glsl:65
        }
        detmath::sincosf_det_n<4>(ph, sn, cs);                          // :66
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int x = xs + SUB * (e0 + j);
            row_a[pad16(x)] = velocity_texel(__ldg(&spec[(size_t)q * N + x]), cs[j], sn[j], tb[j].x, tb[j].w, tb[j].z);
            if (q != 0) {
                // the mirror texel: same omega, k_unit negated -- except k_unit.x in column 0, whose k_vec.x is its own mirror
                const int xm = (N - x) & (N - 1);
                const float kux = (x == 0) ? tb[j].w : -tb[j].w;
                row_b[pad16(xm)] = velocity_texel(__ldg(&spec[(size_t)(N - q) * N + xm]), cs[j], sn[j], tb[j].x, kux, -tb[j].z);
            }
        }
    }
    if (q == 0) {                                        // row N/2: table row N/2 holds its own entries
#pragma unroll 1
        for (int e = 0; e < ITER; ++e) {
            const int x = xs + SUB * e;
            const float4 tb = __ldg(&tab[(size_t)(N / 2) * N + x]);
            float sn, cs;
            detmath::sincosf_det(tb.x * d.time, sn, cs);
            row_b[pad16(x)] = velocity_texel(__ldg(&spec[(size_t)(N / 2) * N + x]), cs, sn, tb.x, tb.w, tb.z);
        }
    }
    __syncthreads();

    const int fid = tid / T, t = tid % T;                // local row fid = 2 * pair + side
    float4* buf = smem + (size_t)fid * RB;
    C2 v[kE];
    pass_load<N, Plan<N>::R0>(v, buf, t);
    fft_group_sync<N>();
    pass_compute<N, Plan<N>::R0, 0>(v, t, tw_s);
    remaining_passes<N>(v, buf, t, tw_s);
    const int pq = q0 + (fid >> 1);
    const int row = (pq == 0) ? ((fid & 1) ? N / 2 : 0) : ((fid & 1) ? N - pq : pq);
    float4* out = scratch + ((size_t)d.cascade * N + row) * N;
#pragma unroll
    for (int i = 0; i < kE; ++i) out[final_index<N>(t, i)] = c2_to(v[i]);
}

__device__ __forceinline__ uint2 pack_half4(float a, float b, float c, float d) {
    const __half2 lo = __floats2half2_rn(a, b), hi = __floats2half2_rn(c, d);
    uint2 r;
    r.x = *reinterpret_cast<const uint32_t*>(&lo);
    r.y = *reinterpret_cast<const uint32_t*>(&hi);
    return r;
}

// Column pass: W = ROWS columns per team.  The W columns are read row by row (W float4 contiguous per row) into padded
// column buffers, transformed by T threads each, and written as rows of the map: map row = scratch column, map column =
// transform index (the reference never transposes back, wave_generator.gd:77-78).  Texel (x, y) =
// (l0.re, l0.im, l1.re, 0) * sign_shift (fft_unpack.glsl:38,50), half RTNE.
template <int N, bool TAPS>
__global__ void __launch_bounds__(VelTile<N>::THREADS) k_velocity_colfft(const float4* __restrict__ scratch, uint2* __restrict__ velocity,
                                                                      float4* __restrict__ velocity_f32, const float2* __restrict__ tw_g,
                                                                      const __grid_constant__ VelocityTable jobs) {
    using VT = VelTile<N>;
    constexpr int T = VT::T, W = VT::ROWS, CS = VT::CS;
    extern __shared__ float4 smem[];
    const float2* tw_s = stage_twiddles<N>(reinterpret_cast<float2*>(smem + W * CS), tw_g);
    const VelocityDispatch d = jobs.d[blockIdx.y];
    const int tid = threadIdx.x;
    const int c0 = blockIdx.x * W;
    const float4* src = scratch + (size_t)d.cascade * N * N + c0;
    for (int i = tid; i < N * W; i += VT::THREADS) {
        const int y = i / W, c = i % W;
        smem[c * CS + pad16(y)] = __ldcs(&src[(size_t)y * N + c]);     // read once
    }
    __syncthreads();

    const int c = tid / T, t = tid % T;
    float4* buf = smem + (size_t)c * CS;
    C2 v[kE];
    pass_load<N, Plan<N>::R0>(v, buf, t);
    fft_group_sync<N>();
    pass_compute<N, Plan<N>::R0, 0>(v, t, tw_s);
    remaining_passes<N>(v, buf, t, tw_s);
    const int yout = c0 + c;
    const size_t row_base = ((size_t)d.cascade * N + yout) * N;
#pragma unroll
    for (int i = 0; i < kE; ++i) {
        const int xo = final_index<N>(t, i);
        const float s = ((xo ^ yout) & 1) ? -1.0f : 1.0f;
        const float4 f = c2_to(v[i]);                    // (l0.re, l1.re, l0.im, l1.im)
        const float vx = f.x * s, vy = f.z * s, vz = f.y * s, vw = 0.0f * s;
        __stcs(&velocity[row_base + xo], pack_half4(vx, vy, vz, vw));
        if (TAPS) velocity_f32[row_base + xo] = make_float4(vx, vy, vz, vw);
    }
}

template <int N>
cudaError_t launch_velocity_n(const DeviceBuffers& b, const VelocityDispatch* jobs_host, int count, float4* scratch, uint2* velocity,
                              float4* velocity_f32, cudaStream_t stream, int* launched) {
    using VT = VelTile<N>;
    for (int first = 0; first < count; first += kMaxVelocityLaunch) {
        const int n = (count - first < kMaxVelocityLaunch) ? count - first : kMaxVelocityLaunch;
        VelocityTable jobs;
        for (int i = 0; i < n; ++i) jobs.d[i] = jobs_host[first + i];
        k_velocity_rowfft<N><<<dim3((N / 2) / (VT::ROWS / 2), n), VT::THREADS, VT::ROW_SMEM, stream>>>(b.spectrum, b.disp_table, scratch,
                                                                                                     b.twiddles, jobs);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        if (velocity_f32)
            k_velocity_colfft<N, true><<<dim3(N / VT::ROWS, n), VT::THREADS, VT::COL_SMEM, stream>>>(scratch, velocity, velocity_f32, b.twiddles, jobs);
        else
            k_velocity_colfft<N, false><<<dim3(N / VT::ROWS, n), VT::THREADS, VT::COL_SMEM, stream>>>(scratch, velocity, nullptr, b.twiddles, jobs);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        if (launched) *launched += 2;
    }
    return cudaSuccess;
}

}  // namespace

cudaError_t init_velocity_twiddles(const float2* twiddles_dev, cudaStream_t stream) {
    // this module's copy of the constant-bank twiddle table (the first radix pass reads it, fft_core.cuh)
    return cudaMemcpyToSymbolAsync(c_twiddles, twiddles_dev, sizeof(float2) * kTwiddleCount, 0, cudaMemcpyDeviceToDevice, stream);
}

cudaError_t launch_velocity(const DeviceBuffers& b, const VelocityDispatch* jobs_host, int count, float4* scratch, uint2* velocity,
                            float4* velocity_f32, cudaStream_t stream, int* launched) {
    if (launched) *launched = 0;
    if (count <= 0) return cudaSuccess;
    switch (b.map_size) {
        case 128: return launch_velocity_n<128>(b, jobs_host, count, scratch, velocity, velocity_f32, stream, launched);
        case 256: return launch_velocity_n<256>(b, jobs_host, count, scratch, velocity, velocity_f32, stream, launched);
        case 512: return launch_velocity_n<512>(b, jobs_host, count, scratch, velocity, velocity_f32, stream, launched);
        case 1024: return launch_velocity_n<1024>(b, jobs_host, count, scratch, velocity, velocity_f32, stream, launched);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace ocean
