// ocean_wake.cu -- the wake layer (include/ocean.h, "Wake layer"; oracle/wake.py is the specification, bit for bit): a
// local N x N height field advanced by sub-steps of the iWave scheme with a radius-6 stencil for sqrt(-laplacian), forced
// by the pressure head of moving sources.
//
//   k_wake_step     one sub-step; one CTA per 32 x 32 output tile (256 threads, 4 cells each).  The CTA culls the sources
//                   against its tile plus the 6-cell halo, 256 at a time, with a warp ballot and a prefix over the warps
//                   (index order is kept), and accumulates phi over its 44 x 44 halo cells in registers; then it stores
//                   s = h + phi (0 outside the window) in shared memory and each thread takes the 28-class symmetric
//                   convolution of its four cells from there.  The scroll is folded into the reads: h and h_prev are read at
//                   (i + di, j + dj), 0 outside, and on a scrolled sub-step the scrolled h is written as the new h_prev.
//   k_wake_step_foam  k_wake_step (one inlined template) that also advances the foam field F (ocean_wake_set_foam;
//                   oracle/wake_foam.py) in the same pass: the cull carries each kept source's |v|^2, the halo pass adds
//                   w^2 |v|^2 next to phi (kept per halo cell in shared memory), and each output cell
//                   updates F from its convolution c and that sum.  F is read at (i + di, j + dj) and written to a second
//                   field, as h is.
//   k_wake_step_obstacles, k_wake_step_foam_obstacles  the two sub-steps (the same template) while an obstacle mask is set
//                   (ocean_wake_set_obstacles; oracle/wake_obstacles.py): the halo pass reads the mask byte of each halo
//                   cell once, stores s = 0 on blocked cells and marks the blocked output cells in shared memory; those
//                   are written h = 0 (and F = 0).  h_prev is written unmasked.
//   k_wake_map      one thread per cell: (h, dh/dx, dh/dz, 0) as half, central differences; k_wake_map_foam writes F as
//                   the fourth channel.
//   k_wake_sample   one thread per point: bilinear h and central differences.
// The coupling of the layer to the surface query (ocean_wake_set_coupling; oracle/wake_coupling.py):
//   k_wake_free_surface  after a coupled step call: e = h + phi of the sources at the end of the call, one CTA per 32 x 32
//                        tile; the source cull and the rasterisation are k_wake_step's (one __device__ template, over the
//                        tile instead of the halo), without the convolution.  k_wake_free_surface_obstacles also writes
//                        e = 0 on blocked cells.
//   k_wake_couple        one thread per query point: k_wake_sample's bilinear sample of e added to the surface record, and
//                        on request the wake's vertical velocity (e - e_old) / T at the point for the drag pass.
// No atomics.  Numeric policy: binary32 in the specification's order with explicit _rn operations, no contraction
// (-fmad=false), IEEE division.
#include "../../include/ocean.h"
#include "ocean_kernels.cuh"
#include "wake_sample.cuh"

#include <cuda_fp16.h>

namespace ocean {

namespace {

constexpr int kR = 6;
constexpr int kTile = 32;
constexpr int kHalo = kTile + 2 * kR;           // 44
constexpr int kHaloCells = kHalo * kHalo;       // 1936
constexpr int kThreads = 256;
constexpr int kCellsPerThread = (kHaloCells + kThreads - 1) / kThreads;    // 8

// the 28 taps G[a][b], 0 <= b <= a <= 6, in the specification's order (tools/fit_wake_kernel.py)
__host__ __device__ constexpr float wake_tap(int t) {
    constexpr float k[28] = {
        0x1.cb69a8p+0f,   // G[0][0]
        -0x1.1ee9ap-4f,   // G[1][0]
        -0x1.0ffeap-3f,   // G[1][1]
        -0x1.43e97p-2f,   // G[2][0]
        -0x1.6504p-6f,    // G[2][1]
        0x1.7312ep-4f,    // G[2][2]
        0x1.1a2cp-2f,     // G[3][0]
        0x1.ad1f8p-6f,    // G[3][1]
        -0x1.142dp-4f,    // G[3][2]
        0x1.1c418p-6f,    // G[3][3]
        -0x1.b34d6p-3f,   // G[4][0]
        -0x1.97ccp-6f,    // G[4][1]
        0x1.228p-8f,      // G[4][2]
        -0x1.3e51p-7f,    // G[4][3]
        0x1.277dcp-5f,    // G[4][4]
        0x1.a86fp-4f,     // G[5][0]
        0x1.1e5p-6f,      // G[5][1]
        0x1.de36p-7f,     // G[5][2]
        0x1.323ap-7f,     // G[5][3]
        -0x1.c8dbp-6f,    // G[5][4]
        0x1.3535p-7f,     // G[5][5]
        -0x1.dfdbp-6f,    // G[6][0]
        -0x1.979cp-7f,    // G[6][1]
        -0x1.787bp-7f,    // G[6][2]
        -0x1.fc14p-8f,    // G[6][3]
        0x1.ae5p-9f,      // G[6][4]
        -0x1.28bp-9f,     // G[6][5]
        0x1.9ep-12f,      // G[6][6]
    };
    return k[t];
}
__host__ __device__ constexpr int tap_a(int t) { int a = 0; while ((a + 1) * (a + 2) / 2 <= t) ++a; return a; }
__host__ __device__ constexpr int tap_b(int t) { return t - tap_a(t) * (tap_a(t) + 1) / 2; }

// the sum of the values at the mirrored offsets (di, dj) of class (A, B), in the specification's order; s points at the
// centre of a row-major array of row stride kHalo
template <int A, int B>
__device__ __forceinline__ float orbit(const float* s) {
    constexpr int W = kHalo;
    if constexpr (A == 0) {
        return s[0];
    } else if constexpr (B == 0) {
        return __fadd_rn(__fadd_rn(__fadd_rn(s[A], s[-A]), s[A * W]), s[-A * W]);
    } else if constexpr (A == B) {
        return __fadd_rn(__fadd_rn(__fadd_rn(s[A + A * W], s[A - A * W]), s[-A + A * W]), s[-A - A * W]);
    } else {
        float v = __fadd_rn(s[A + B * W], s[A - B * W]);
        v = __fadd_rn(v, s[-A + B * W]);
        v = __fadd_rn(v, s[-A - B * W]);
        v = __fadd_rn(v, s[B + A * W]);
        v = __fadd_rn(v, s[B - A * W]);
        v = __fadd_rn(v, s[-B + A * W]);
        return __fadd_rn(v, s[-B - A * W]);
    }
}

template <int T>
__device__ __forceinline__ float convolve_from(const float* s, float c) {
    if constexpr (T == 28) {
        return c;
    } else {
        return convolve_from<T + 1>(s, __fadd_rn(c, __fmul_rn(wake_tap(T), orbit<tap_a(T), tap_b(T)>(s))));
    }
}

__device__ __forceinline__ float convolve(const float* s) { return convolve_from<1>(s, __fmul_rn(wake_tap(0), s[0])); }

// phi at the cells of the kSpan x kSpan square whose first cell is window cell (ti0, tj0): thread t holds square cells
// c = t + m * kThreads (row-major) in phi[m], and adds, in source index order, the sources of `a` at a.tau.  The CTA culls
// the sources against the square, 256 at a time, with a warp ballot and a prefix over the warps (index order is kept);
// list and warp_count are its shared scratch.  Cells outside the window are left as they are.  Args is WakeStepArgs or
// WakeFreeSurfaceArgs: the source, window and time fields of both have the same names.  With kStir the same pass adds
// (w w) |v|^2 of each source to the shared sigma[c] of the square's cell c (v its centre velocity, |v|^2 = vx vx + vz vz),
// the cull keeping |v|^2 of the kept sources in the shared speed2; the caller zeroes sigma, and each cell is only touched by
// the thread that holds it, so it needs no barrier.
template <int kSpan, bool kStir = false, typename Args>
__device__ __forceinline__ void rasterise(const Args& a, int ti0, int tj0, float4* list, int* warp_count,
                                          float (&phi)[(kSpan * kSpan + kThreads - 1) / kThreads], float* speed2 = nullptr,
                                          float* sigma = nullptr) {
    constexpr int kCells = kSpan * kSpan;
    constexpr int kPer = (kCells + kThreads - 1) / kThreads;
    const int t = threadIdx.x;
    const int n = a.n;
    const float dx = a.cell;
    if (a.num_sources > 0) {
        // the square's cell centres span [lo, hi] per axis; one cell of margin keeps the cull conservative under rounding
        const float xlo = __fadd_rn(a.x0, __fmul_rn(__fadd_rn((float)(ti0 - 1), 0.5f), dx));
        const float xhi = __fadd_rn(a.x0, __fmul_rn(__fadd_rn((float)(ti0 + kSpan), 0.5f), dx));
        const float zlo = __fadd_rn(a.z0, __fmul_rn(__fadd_rn((float)(tj0 - 1), 0.5f), dx));
        const float zhi = __fadd_rn(a.z0, __fmul_rn(__fadd_rn((float)(tj0 + kSpan), 0.5f), dx));
        for (int base = 0; base < a.num_sources; base += kThreads) {
            const int k = base + t;
            bool keep = false;
            float4 e = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
            float v2 = 0.0f;
            if (k < a.num_sources) {
                const ocean_wake_source src = a.sources[k];
                float cx = __fadd_rn(src.x, __fmul_rn(src.vx, a.tau));
                float cz = __fadd_rn(src.z, __fmul_rn(src.vz, a.tau));
                float vx = src.vx, vz = src.vz;
                bool ok = src.body < a.num_states;
                if (ok && src.body >= 0) {
                    const ocean_body_state& b = a.states[src.body];
                    cx = __fadd_rn(cx, __fadd_rn(b.position[0], __fmul_rn(b.linear_velocity[0], a.tau)));
                    cz = __fadd_rn(cz, __fadd_rn(b.position[2], __fmul_rn(b.linear_velocity[2], a.tau)));
                    if constexpr (kStir) {
                        vx = __fadd_rn(vx, b.linear_velocity[0]);
                        vz = __fadd_rn(vz, b.linear_velocity[2]);
                    }
                }
                if constexpr (kStir) v2 = __fadd_rn(__fmul_rn(vx, vx), __fmul_rn(vz, vz));
                const float r = src.radius;
                const float r2 = __fmul_rn(r, r);
                ok = ok && isfinite(cx) && isfinite(cz) && isfinite(src.head) && isfinite(r) && r > 0.0f && isfinite(r2);
                keep = ok && __fadd_rn(cx, r) >= xlo && __fsub_rn(cx, r) <= xhi && __fadd_rn(cz, r) >= zlo && __fsub_rn(cz, r) <= zhi;
                e = make_float4(cx, cz, r2, src.head);
            }
            const unsigned ballot = __ballot_sync(0xffffffffu, keep);
            const int lane = t & 31, warp = t >> 5;
            if (lane == 0) warp_count[warp] = __popc(ballot);
            __syncthreads();
            int offset = 0, total = 0;
#pragma unroll
            for (int w = 0; w < kThreads / 32; ++w) {
                offset += w < warp ? warp_count[w] : 0;
                total += warp_count[w];
            }
            if (keep) {
                const int slot = offset + __popc(ballot & ((1u << lane) - 1u));
                list[slot] = e;
                if constexpr (kStir) speed2[slot] = v2;
            }
            __syncthreads();
#pragma unroll
            for (int m = 0; m < kPer; ++m) {
                const int c = t + m * kThreads;
                const int i = ti0 + c % kSpan, j = tj0 + c / kSpan;
                if (c < kCells && (unsigned)i < (unsigned)n && (unsigned)j < (unsigned)n) {
                    const float px = __fadd_rn(a.x0, __fmul_rn(__fadd_rn((float)i, 0.5f), dx));
                    const float pz = __fadd_rn(a.z0, __fmul_rn(__fadd_rn((float)j, 0.5f), dx));
                    float p = phi[m];
                    float sg = 0.0f;
                    if constexpr (kStir) sg = sigma[c];
                    for (int q = 0; q < total; ++q) {
                        const float4 e2 = list[q];
                        const float ex = __fsub_rn(px, e2.x), ez = __fsub_rn(pz, e2.y);
                        const float d2 = __fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ez, ez));
                        if (d2 < e2.z) {
                            const float w = __fsub_rn(1.0f, __fdiv_rn(d2, e2.z));
                            const float ww = __fmul_rn(w, w);
                            p = __fadd_rn(p, __fmul_rn(e2.w, ww));
                            if constexpr (kStir) sg = __fadd_rn(sg, __fmul_rn(ww, speed2[q]));
                        }
                    }
                    phi[m] = p;
                    if constexpr (kStir) sigma[c] = sg;
                }
            }
            __syncthreads();                        // the list and the counts are rewritten by the next chunk
        }
    }
}

// whether window cell (i, j) of the call's window is blocked by the obstacle mask
__device__ __forceinline__ bool blocked(const WakeObstacles& o, int i, int j) {
    const int q = o.qx + i, r = o.qz + j;
    return (unsigned)q < (unsigned)o.width && (unsigned)r < (unsigned)o.depth && o.mask[(size_t)r * o.width + q] != 0;
}

// One sub-step over one 32 x 32 output tile: k_wake_step, and with kFoam k_wake_step_foam (f is its foam arguments, the
// foam-only shared arrays speed2 [kThreads] and sig [kHaloCells] are not null).  sigma lives in shared memory rather than
// in registers next to phi: eight more live registers per thread made the foam form spill.  With kObstacles (ob and the
// shared [kTile * kTile] out_blocked are not null) the halo pass reads the mask once per halo cell, stores s = 0 on blocked
// cells and marks the blocked output cells, which are then written 0 (h and F; h_prev is the scrolled h, unmasked).
template <bool kFoam, bool kObstacles = false>
__device__ __forceinline__ void wake_step(const WakeStepArgs& a, const WakeFoamStepArgs* f, float* s, float4* list, int* warp_count,
                                          float* speed2, float* sig, const WakeObstacles* ob = nullptr,
                                          unsigned char* out_blocked = nullptr) {
    const int t = threadIdx.x;
    const int n = a.n;
    const int ti0 = blockIdx.x * kTile - kR, tj0 = blockIdx.y * kTile - kR;   // window cell of halo cell (0, 0)

    float phi[kCellsPerThread];
#pragma unroll
    for (int m = 0; m < kCellsPerThread; ++m) phi[m] = 0.0f;
    if constexpr (kFoam) {
#pragma unroll
        for (int m = 0; m < kCellsPerThread; ++m)
            if (t + m * kThreads < kHaloCells) sig[t + m * kThreads] = 0.0f;
        rasterise<kHalo, true>(a, ti0, tj0, list, warp_count, phi, speed2, sig);
    } else {
        rasterise<kHalo>(a, ti0, tj0, list, warp_count, phi);
    }

    // s = h + phi over the halo, 0 outside the window
#pragma unroll
    for (int m = 0; m < kCellsPerThread; ++m) {
        const int c = t + m * kThreads;
        if (c < kHaloCells) {
            const int i = ti0 + c % kHalo, j = tj0 + c / kHalo;
            float v = 0.0f;
            if constexpr (kObstacles) {
                const bool b = (unsigned)i < (unsigned)n && (unsigned)j < (unsigned)n && blocked(*ob, i, j);
                if (!b && (unsigned)i < (unsigned)n && (unsigned)j < (unsigned)n) v = __fadd_rn(cell(a.h, n, i + a.di, j + a.dj), phi[m]);
                const int oi = c % kHalo - kR, oj = c / kHalo - kR;
                if ((unsigned)oi < (unsigned)kTile && (unsigned)oj < (unsigned)kTile) out_blocked[oj * kTile + oi] = b;
            } else {
                if ((unsigned)i < (unsigned)n && (unsigned)j < (unsigned)n) v = __fadd_rn(cell(a.h, n, i + a.di, j + a.dj), phi[m]);
            }
            s[c] = v;
        }
    }
    __syncthreads();

    const int li = t & 31;
#pragma unroll
    for (int r = 0; r < kTile / 8; ++r) {
        const int lj = (t >> 5) + 8 * r;
        const int i = blockIdx.x * kTile + li, j = blockIdx.y * kTile + lj;
        const float c = convolve(&s[(lj + kR) * kHalo + li + kR]);
        const float h = cell(a.h, n, i + a.di, j + a.dj);
        const float hp = cell(a.h_prev, n, i + a.di, j + a.dj);
        const int edge = min(min(i, j), min(n - 1 - i, n - 1 - j));
        const int ring = min(edge, a.sponge_cells);
        float hn = __fsub_rn(__fsub_rn(__fmul_rn(a.a1[ring], h), __fmul_rn(a.a2[ring], hp)), __fmul_rn(a.a3[ring], c));
        bool shut = false;
        if constexpr (kObstacles) {
            shut = out_blocked[lj * kTile + li] != 0;
            if (shut) hn = 0.0f;
        }
        const size_t o = (size_t)j * n + i;
        a.out_h[o] = hn;
        if (a.out_h_prev) a.out_h_prev[o] = h;
        if constexpr (kFoam) {
            // F' = clamp(F d + (gh max(c / dx - whitecap, 0) + sh sigma), 0, 1); "x > 0 ? x : 0" is fmaxf(x, 0) (NaN -> 0)
            // with -0 -> +0, so the result has one encoding
            const float beta = __fdiv_rn(c, a.cell);
            float b = __fsub_rn(beta, f->whitecap);
            b = b > 0.0f ? b : 0.0f;
            const float grow = __fadd_rn(__fmul_rn(f->grow, b), __fmul_rn(f->stir, sig[(lj + kR) * kHalo + li + kR]));
            const float v = __fadd_rn(__fmul_rn(cell(f->foam, n, i + a.di, j + a.dj), f->decay), grow);
            f->out_foam[o] = v > 0.0f && !shut ? fminf(v, 1.0f) : 0.0f;
        }
    }
}

__global__ void __launch_bounds__(kThreads) k_wake_step(const WakeStepArgs a) {
    __shared__ float s[kHaloCells];
    __shared__ float4 list[kThreads];               // culled sources: cx, cz, r2, head
    __shared__ int warp_count[kThreads / 32];
    wake_step<false>(a, nullptr, s, list, warp_count, nullptr, nullptr);
}

__global__ void __launch_bounds__(kThreads) k_wake_step_foam(const WakeFoamStepArgs f) {
    __shared__ float s[kHaloCells];
    __shared__ float4 list[kThreads];               // culled sources: cx, cz, r2, head
    __shared__ int warp_count[kThreads / 32];
    __shared__ float speed2[kThreads];              // |v|^2 of the culled sources
    __shared__ float sig[kHaloCells];               // sigma of the halo cells
    wake_step<true>(f.step, &f, s, list, warp_count, speed2, sig);
}

__global__ void __launch_bounds__(kThreads) k_wake_step_obstacles(const WakeStepArgs a, const WakeObstacles ob) {
    __shared__ float s[kHaloCells];
    __shared__ float4 list[kThreads];               // culled sources: cx, cz, r2, head
    __shared__ int warp_count[kThreads / 32];
    __shared__ unsigned char out_blocked[kTile * kTile];
    wake_step<false, true>(a, nullptr, s, list, warp_count, nullptr, nullptr, &ob, out_blocked);
}

__global__ void __launch_bounds__(kThreads) k_wake_step_foam_obstacles(const WakeFoamStepArgs f, const WakeObstacles ob) {
    __shared__ float s[kHaloCells];
    __shared__ float4 list[kThreads];               // culled sources: cx, cz, r2, head
    __shared__ int warp_count[kThreads / 32];
    __shared__ float speed2[kThreads];              // |v|^2 of the culled sources
    __shared__ float sig[kHaloCells];               // sigma of the halo cells
    __shared__ unsigned char out_blocked[kTile * kTile];
    wake_step<true, true>(f.step, &f, s, list, warp_count, speed2, sig, &ob, out_blocked);
}

// e = h + phi of the sources at a.tau over one 32 x 32 tile (256 threads, 4 cells each), into a.e, and into a.e_old when it
// is not null (the priming call writes both snapshots); with kObstacles e = 0 on blocked cells
template <bool kObstacles>
__device__ __forceinline__ void free_surface(const WakeFreeSurfaceArgs& a, const WakeObstacles* ob) {
    __shared__ float4 list[kThreads];
    __shared__ int warp_count[kThreads / 32];
    constexpr int kPer = kTile * kTile / kThreads;
    const int t = threadIdx.x;
    const int n = a.n;
    const int ti0 = blockIdx.x * kTile, tj0 = blockIdx.y * kTile;
    float phi[kPer];
#pragma unroll
    for (int m = 0; m < kPer; ++m) phi[m] = 0.0f;
    rasterise<kTile>(a, ti0, tj0, list, warp_count, phi);
#pragma unroll
    for (int m = 0; m < kPer; ++m) {
        const int c = t + m * kThreads;
        const size_t o = (size_t)(tj0 + c / kTile) * n + (ti0 + c % kTile);
        float e = __fadd_rn(a.h[o], phi[m]);
        if constexpr (kObstacles) {
            if (blocked(*ob, ti0 + c % kTile, tj0 + c / kTile)) e = 0.0f;
        }
        a.e[o] = e;
        if (a.e_old) a.e_old[o] = e;
    }
}

__global__ void __launch_bounds__(kThreads) k_wake_free_surface(const WakeFreeSurfaceArgs a) { free_surface<false>(a, nullptr); }

__global__ void __launch_bounds__(kThreads) k_wake_free_surface_obstacles(const WakeFreeSurfaceArgs a, const WakeObstacles ob) {
    free_surface<true>(a, &ob);
}

// (h, dh/dx, dh/dz, F) of one cell as half; F is 0 without kFoam
template <bool kFoam>
__device__ __forceinline__ void wake_map(const float* __restrict__ h, const float* __restrict__ foam, int n, float two_dx,
                                         __half2* __restrict__ out) {
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= n * n) return;
    const int i = o % n, j = o / n;
    out[2 * (size_t)o] = __halves2half2(__float2half_rn(h[o]), __float2half_rn(grad_x(h, n, i, j, two_dx)));
    out[2 * (size_t)o + 1] = __halves2half2(__float2half_rn(grad_z(h, n, i, j, two_dx)), __float2half_rn(kFoam ? foam[o] : 0.0f));
}

__global__ void __launch_bounds__(256) k_wake_map(const float* __restrict__ h, int n, float two_dx, __half2* __restrict__ out) {
    wake_map<false>(h, nullptr, n, two_dx, out);
}

__global__ void __launch_bounds__(256) k_wake_map_foam(const float* __restrict__ h, const float* __restrict__ foam, int n, float two_dx,
                                                       __half2* __restrict__ out) {
    wake_map<true>(h, foam, n, two_dx, out);
}

__global__ void __launch_bounds__(256) k_wake_sample(const float* __restrict__ h, int n, float dx, float x0, float z0,
                                                     const float2* __restrict__ xz, int count, float* __restrict__ out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    float r[3] = {0.0f, 0.0f, 0.0f};
    sample_field<true>(h, n, dx, x0, z0, xz[k], r);
    for (int m = 0; m < 3; ++m) out[3 * (size_t)k + m] = r[m];
}

// The coupling of the surface records to the wake free surface e: one thread per query point Q, (we, gx, gz) = sample(e, Q)
// added to (displacement[1], gradient_foam[0], gradient_foam[1]); with wv not null also wv = (we - sample(e_old, Q)[0]) / T.
__global__ void __launch_bounds__(256) k_wake_couple(const WakeCoupleArgs a, const float2* __restrict__ q, int count,
                                                     ocean_surface_sample* __restrict__ rec, float* __restrict__ wv) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    const float2 p = q[k];
    float r[3] = {0.0f, 0.0f, 0.0f};
    sample_field<true>(a.e, a.n, a.cell, a.x0, a.z0, p, r);
    ocean_surface_sample& s = rec[k];
    s.displacement[1] = __fadd_rn(s.displacement[1], r[0]);
    s.gradient_foam[0] = __fadd_rn(s.gradient_foam[0], r[1]);
    s.gradient_foam[1] = __fadd_rn(s.gradient_foam[1], r[2]);
    if (wv) {
        float o = 0.0f;
        sample_field<false>(a.e_old, a.n, a.cell, a.x0_old, a.z0_old, p, &o);
        wv[k] = __fdiv_rn(__fsub_rn(r[0], o), a.interval);
    }
}

}  // namespace

void wake_kernel_taps(float* out) {
    for (int t = 0; t < 28; ++t) out[t] = wake_tap(t);
}

cudaError_t launch_wake_step(const WakeStepArgs& args, const WakeFoamStepArgs* foam, const WakeObstacles* obstacles, cudaStream_t stream) {
    const dim3 grid((unsigned)(args.n / kTile), (unsigned)(args.n / kTile));
    if (foam) {
        WakeFoamStepArgs f = *foam;
        f.step = args;
        if (obstacles)
            k_wake_step_foam_obstacles<<<grid, kThreads, 0, stream>>>(f, *obstacles);
        else
            k_wake_step_foam<<<grid, kThreads, 0, stream>>>(f);
    } else if (obstacles) {
        k_wake_step_obstacles<<<grid, kThreads, 0, stream>>>(args, *obstacles);
    } else {
        k_wake_step<<<grid, kThreads, 0, stream>>>(args);
    }
    return cudaGetLastError();
}

cudaError_t launch_wake_free_surface(const WakeFreeSurfaceArgs& args, const WakeObstacles* obstacles, cudaStream_t stream) {
    const dim3 grid((unsigned)(args.n / kTile), (unsigned)(args.n / kTile));
    if (obstacles)
        k_wake_free_surface_obstacles<<<grid, kThreads, 0, stream>>>(args, *obstacles);
    else
        k_wake_free_surface<<<grid, kThreads, 0, stream>>>(args);
    return cudaGetLastError();
}

cudaError_t launch_wake_map(const WakeRead& wake, void* map_dev, cudaStream_t stream) {
    const int n = wake.n;
    const unsigned blocks = (unsigned)(((size_t)n * n + 255) / 256);
    if (wake.foam)
        k_wake_map_foam<<<blocks, 256, 0, stream>>>(wake.field, wake.foam, n, 2.0f * wake.cell, static_cast<__half2*>(map_dev));
    else
        k_wake_map<<<blocks, 256, 0, stream>>>(wake.field, n, 2.0f * wake.cell, static_cast<__half2*>(map_dev));    // exact
    return cudaGetLastError();
}

cudaError_t launch_wake_sample(const WakeRead& wake, const float2* xz_dev, int count, float* out_dev, cudaStream_t stream) {
    if (count <= 0) return cudaSuccess;
    k_wake_sample<<<(unsigned)((count + 255) / 256), 256, 0, stream>>>(wake.field, wake.n, wake.cell, wake.x0, wake.z0, xz_dev, count,
                                                                         out_dev);
    return cudaGetLastError();
}

cudaError_t launch_wake_couple(const WakeCoupleArgs& args, const float2* q_dev, int count, ocean_surface_sample* records_dev, float* wv_dev,
                               cudaStream_t stream) {
    if (count <= 0) return cudaSuccess;
    k_wake_couple<<<(unsigned)((count + 255) / 256), 256, 0, stream>>>(args, q_dev, count, records_dev, wv_dev);
    return cudaGetLastError();
}

}  // namespace ocean
