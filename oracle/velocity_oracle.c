/*
 * oracle/velocity_oracle.c -- TEST INFRASTRUCTURE.  The specification of the velocity maps (include/ocean.h,
 * ocean_update_velocity): the time derivative of the displacement map, bit for bit, in the numeric policy of
 * oracle/ocean_oracle.c.  Built by oracle/velocity.py into libocean_velocity_oracle.so, linked against
 * libocean_oracle.so: the transcendentals (oracle_cosf / oracle_sinf / oracle_tanhf), the row IFFT (oracle_fft_compute),
 * the transpose (oracle_transpose), the half conversion (oracle_float_to_half) and the numeric modes
 * (oracle_get_contract_mode) are that library's, so the two share one state and one FFT.
 *
 * Not part of the reference.  h(t) = h0a e^{i w t} + h0b e^{-i w t}, so dh/dt = i w (h0a e^{i w t} - h0b e^{-i w t}); the
 * displacement fields hx, hy, hz are linear in h (spectrum_modulate.glsl:69-74), so their derivatives pack like :86 with dh/dt
 * for h.  Per texel, binary32, every name as in oracle_spectrum_modulate:
 *   w   = sqrtf(G*k*tanh(k*depth))        (the factor of spectrum_modulate.glsl:49 that the phase multiplies by time, :65)
 *   m   = (cos(w*time), sin(w*time)),  pa = mul_complex(h0a, m),  pb = mul_complex(h0b, conj m)
 *   d   = (pa.x - pb.x, pa.y - pb.y)
 *   ht  = (-(w*d.y), w*d.x)              (i w d)
 *   hti = (-ht.y, ht.x)                  (i ht, like :69)
 *   vx  = hti*k_unit.y,  vy = ht,  vz = hti*k_unit.x                      (each product rounded on its own)
 *   layer 0 = (vx.x - vy.y, vx.y + vy.x),  layer 1 = (vz.x, vz.y)          (no "+ 0": that would turn -0 into +0)
 * then the reference's row IFFT, transpose and row IFFT, and the texel (l0.re*s, l0.im*s, l1.re*s, 0*s), s = sign_shift, as
 * fft_unpack.glsl:38,50 forms the displacement; half RTNE.  mul_complex follows the contraction mode of ocean_oracle.c
 * (policy item 4): FMA (fma(ax,bx,-(ay*by)), fma(ax,by,ay*bx)) or STRICT (four products, then the sums).
 *
 * Build flags as oracle/Makefile's: gcc -O2 -std=c11 -fPIC -shared -ffp-contract=off -fno-fast-math -fopenmp -mfma.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

#define PI_F 3.141592653589793f   /* GLSL "#define PI" as binary32 */
#define G_F 9.81f
#define NUM_SPECTRA 4

/* libocean_oracle.so */
float oracle_cosf(float x);
float oracle_sinf(float x);
float oracle_tanhf(float x);
int oracle_get_contract_mode(void);
uint16_t oracle_float_to_half(float f);
void oracle_fft_compute(const float *butterfly, float *fft_buffer, int map_size);
void oracle_transpose(float *fft_buffer, int map_size);

typedef struct {            /* == pc_spectrum_modulate of ocean_oracle.c (spectrum_modulate.glsl:24-29) */
    float tile_length[2];
    float depth, time;
    uint32_t cascade_index;
} pc_velocity;

typedef struct { float x, y; } vec2;

static inline vec2 mul_complex(vec2 a, vec2 b, int fma_mode) {
    vec2 r;
    if (fma_mode) {
        r.x = fmaf(a.x, b.x, -(a.y * b.y));
        r.y = fmaf(a.x, b.y, a.y * b.x);
    } else {
        float p0 = a.x * b.x, p1 = a.y * b.y, p2 = a.x * b.y, p3 = a.y * b.x;
        r.x = p0 - p1;
        r.y = p2 + p3;
    }
    return r;
}

/* fft_buffer: 2 halves x 4 layers x N*N vec2, as oracle_spectrum_modulate writes it.  Layers 0 and 1 receive the velocity
 * layer pair; layers 2 and 3 are written as +0 so that oracle_fft_compute transforms defined data (the unpack ignores them). */
void oracle_velocity_modulate(const float *spectrum, float *fft_buffer, int map_size, const pc_velocity *pc) {
    const int N = map_size;
    const size_t NN = (size_t)N * N;
    const int fma_mode = oracle_get_contract_mode();
#pragma omp parallel for schedule(static)
    for (int y = 0; y < N; ++y)
        for (int x = 0; x < N; ++x) {
            float half = (float)N * 0.5f;
            float kvx = ((float)x - half) * 2.0f * PI_F / pc->tile_length[0];
            float kvy = ((float)y - half) * 2.0f * PI_F / pc->tile_length[1];
            float k = sqrtf(kvx * kvx + kvy * kvy) + 1e-6f;
            float kux = kvx / k, kuy = kvy / k;
            const float *h0 = spectrum + ((size_t)y * N + x) * 4;
            float w = sqrtf(G_F * k * oracle_tanhf(k * pc->depth));
            float phase = w * pc->time;
            vec2 m = { oracle_cosf(phase), oracle_sinf(phase) };
            vec2 mc = { m.x, m.y * -1.0f };
            vec2 h0a = { h0[0], h0[1] }, h0b = { h0[2], h0[3] };
            vec2 pa = mul_complex(h0a, m, fma_mode), pb = mul_complex(h0b, mc, fma_mode);
            vec2 d = { pa.x - pb.x, pa.y - pb.y };
            vec2 ht = { -(w * d.y), w * d.x };
            vec2 hti = { -ht.y, ht.x };
            vec2 vx = { hti.x * kuy, hti.y * kuy };
            vec2 vy = ht;
            vec2 vz = { hti.x * kux, hti.y * kux };
            size_t o = (size_t)y * N + x;
            float *b = fft_buffer;
            b[(0 * NN + o) * 2 + 0] = vx.x - vy.y; b[(0 * NN + o) * 2 + 1] = vx.y + vy.x;
            b[(1 * NN + o) * 2 + 0] = vz.x;        b[(1 * NN + o) * 2 + 1] = vz.y;
            b[(2 * NN + o) * 2 + 0] = 0.0f;        b[(2 * NN + o) * 2 + 1] = 0.0f;
            b[(3 * NN + o) * 2 + 0] = 0.0f;        b[(3 * NN + o) * 2 + 1] = 0.0f;
        }
}

/* After oracle_fft_compute, oracle_transpose, oracle_fft_compute: velocity = N*N*4 halves, velocity_f32 (optional, may be
 * NULL) the binary32 values before the half conversion. */
void oracle_velocity_unpack(const float *fft_buffer, uint16_t *velocity, float *velocity_f32, int map_size) {
    const int N = map_size;
    const size_t NN = (size_t)N * N;
    const float *half1 = fft_buffer + NUM_SPECTRA * NN * 2;
#pragma omp parallel for schedule(static)
    for (int y = 0; y < N; ++y)
        for (int x = 0; x < N; ++x) {
            size_t o = (size_t)y * N + x;
            float sign_shift = (float)(-2 * ((x & 1) ^ (y & 1)) + 1);
            const float *l0 = half1 + (0 * NN + o) * 2, *l1 = half1 + (1 * NN + o) * 2;
            float v[4] = { l0[0] * sign_shift, l0[1] * sign_shift, l1[0] * sign_shift, 0.0f * sign_shift };
            for (int c = 0; c < 4; ++c) velocity[o * 4 + c] = oracle_float_to_half(v[c]);
            if (velocity_f32) memcpy(velocity_f32 + o * 4, v, sizeof v);
        }
}

/* One cascade's velocity map from its spectrum texture and the push constants of the update that built its maps. */
void oracle_velocity_update(const float *spectrum, float *fft_buffer, const float *butterfly, uint16_t *velocity,
                            float *velocity_f32, int map_size, const pc_velocity *pc) {
    oracle_velocity_modulate(spectrum, fft_buffer, map_size, pc);
    oracle_fft_compute(butterfly, fft_buffer, map_size);
    oracle_transpose(fft_buffer, map_size);
    oracle_fft_compute(butterfly, fft_buffer, map_size);
    oracle_velocity_unpack(fft_buffer, velocity, velocity_f32, map_size);
}
