"""CPU specification of the sea state (ocean_get_sea_state): the spectral moments of each cascade's spectrum texture, summed
in the library's fixed order, and the fields derived from them.

TEST INFRASTRUCTURE ONLY -- the product path (godotoceanwaves_b200/csrc) never imports or calls this module.

TABLE   the dispersion table of a (tile_length, depth) pair as k_dispersion_table builds it (spectrum_modulate.glsl:59-61,49),
        binary32 in the shader's order: kvx = ((x - N/2) * 2 * PI) / tile.x, kvy likewise with y, k = sqrt(kvx kvx + kvy kvy)
        + 1e-6, k_unit = k_vec / k, omega = sqrt((G k) tanh(k depth)) with DETMATH's tanh; rows y <= N/2 only.  Row y > N/2
        is the mirror of row N - y at column (N - x) mod N: omega the same, k_vec and k_unit negated, except k_vec.x and
        k_unit.x in column 0 (its own mirror along x).
TERMS   per texel (binary64 from the binary32 values, every operation rounded once, in the order written):
          E = 2 (A.x A.x + A.y A.y),  A = the texel's .xy
          q = DETMATH exp(-((2 k) 20)) (binary32),  F = (1 + q q) / ((1 - q)(1 - q))
          d = (-k_unit.y, -k_unit.x),  kw = (k_vec.y, k_vec.x)
          E / w,  E,  w E,  (w w) E,  E d.x,  E d.z,  E (kw.x kw.x),  E (kw.z kw.z),  c d.x,  c d.z  with c = (((2 w) k) E) F
        The DC texel (N/2, N/2) and texels with E == 0 or 1 - q == 0 contribute +0.
ORDER   T = N^2 / 16 threads; thread t sums texels t + j T, j = 0..15, from +0; lanes of a warp fold as lane l += lane l + off,
        off = 16, 8, 4, 2, 1; the 8 warp sums of each 256-thread block and then the N^2 / 4096 block sums are added in index
        order from +0.
"""
from __future__ import annotations

import math

import numpy as np

from . import pyoracle as po

F = np.float32
MOMENTS = 10
THREADS = 256
DEPTH = 20.0
PI32 = F(3.141592653589793)
G32 = F(9.81)

SEA_STATE = np.dtype([("m_minus1", np.float64), ("m0", np.float64), ("m1", np.float64), ("m2", np.float64),
                      ("direction", np.float64, 2), ("slope", np.float64, 2), ("stokes", np.float64, 2),
                      ("significant_wave_height", np.float64), ("mean_period", np.float64), ("zero_crossing_period", np.float64),
                      ("energy_period", np.float64), ("mean_direction", np.float64), ("directional_spread", np.float64),
                      ("mean_square_slope", np.float64), ("stokes_speed", np.float64)])          # struct ocean_sea_state


def dispersion_table(N: int, tile_length):
    """(omega, kvx, kuy, kux) [N/2 + 1][N] and kvy [N/2 + 1], binary32, as k_dispersion_table stores them."""
    half = F(N) * F(0.5)
    x = np.arange(N, dtype=np.float32)
    y = np.arange(N // 2 + 1, dtype=np.float32)
    kvx = ((x - half) * F(2.0) * PI32) / F(tile_length[0])
    kvy = ((y - half) * F(2.0) * PI32) / F(tile_length[1])
    KX = np.broadcast_to(kvx[None, :], (N // 2 + 1, N))
    KY = np.broadcast_to(kvy[:, None], (N // 2 + 1, N))
    k = np.sqrt(KX * KX + KY * KY) + F(1e-6)
    th = po.math_batch(po.MATH_TANH, k * F(DEPTH))[:, 0].reshape(k.shape)
    omega = np.sqrt(G32 * k * th)
    return omega, np.array(KX), KY / k, KX / k, kvy


def texel_terms(spectrum: np.ndarray, tile_length) -> np.ndarray:
    """[N * N][MOMENTS] binary64 terms of the spectrum texture [N][N][4] float32 (texel i = y N + x)."""
    N = spectrum.shape[0]
    omega_t, kvx_t, kuy_t, kux_t, kvy_t = dispersion_table(N, tile_length)
    ys, xs = np.meshgrid(np.arange(N), np.arange(N), indexing="ij")
    lower = ys <= N // 2
    ym = np.where(lower, ys, N - ys)
    xm = np.where(lower, xs, (N - xs) & (N - 1))
    own_x = lower | (xs == 0)
    omega = omega_t[ym, xm]
    kvx = np.where(own_x, kvx_t[ym, xm], -kvx_t[ym, xm])
    kux = np.where(own_x, kux_t[ym, xm], -kux_t[ym, xm])
    kuy = np.where(lower, kuy_t[ym, xm], -kuy_t[ym, xm])
    kvy = np.where(lower, kvy_t[ym], -kvy_t[ym])
    k = np.sqrt(kvx * kvx + kvy * kvy) + F(1e-6)
    ax = spectrum[..., 0].astype(np.float64)
    ay = spectrum[..., 1].astype(np.float64)
    E = 2.0 * (ax * ax + ay * ay)
    q = po.math_batch(po.MATH_EXP, -((F(2.0) * k) * F(DEPTH)))[:, 0].reshape(N, N).astype(np.float64)
    omq = 1.0 - q
    w = omega.astype(np.float64)
    kd = k.astype(np.float64)
    dx, dz = -kuy.astype(np.float64), -kux.astype(np.float64)
    kx, kz = kvy.astype(np.float64), kvx.astype(np.float64)
    with np.errstate(all="ignore"):
        Fq = (1.0 + q * q) / (omq * omq)
        c = (((2.0 * w) * kd) * E) * Fq
        t = np.stack([E / w, E, w * E, (w * w) * E, E * dx, E * dz, E * (kx * kx), E * (kz * kz), c * dx, c * dz], axis=-1)
    excluded = (E == 0.0) | (omq == 0.0)
    excluded[N // 2, N // 2] = True
    t[excluded] = 0.0
    return t.reshape(N * N, MOMENTS)


def fixed_sum(terms: np.ndarray) -> np.ndarray:
    """The library's fixed summation order (ORDER above) of [N * N][MOMENTS] terms."""
    n = terms.shape[0]
    T = n // 16
    B = T // THREADS
    per = terms.reshape(16, T, MOMENTS)
    acc = np.zeros((T, MOMENTS))
    for j in range(16):
        acc = acc + per[j]
    w = acc.reshape(T // 32, 32, MOMENTS)
    off = 16
    while off:
        w = w[:, :off] + w[:, off:2 * off]
        off //= 2
    warps = w[:, 0].reshape(B, THREADS // 32, MOMENTS)
    blocks = np.zeros((B, MOMENTS))
    for k in range(THREADS // 32):
        blocks = blocks + warps[:, k]
    total = np.zeros(MOMENTS)
    for b in range(B):
        total = total + blocks[b]
    return total


def cascade_moments(spectrum: np.ndarray, tile_length) -> np.ndarray:
    """The MOMENTS binary64 moments of one cascade (m-1, m0, m1, m2, E d.x, E d.z, E kx^2, E kz^2, u_s.x, u_s.z)."""
    return fixed_sum(texel_terms(spectrum, tile_length))


def total_moments(moments, map_scales) -> np.ndarray:
    """sum over the cascades in order of (s s) moments_i, s = (double)map_scales[i][2], from +0."""
    sc = np.asarray(map_scales, np.float32).reshape(-1, 4)
    total = np.zeros(MOMENTS)
    for m, s in zip(moments, sc[:, 2].astype(np.float64)):
        total = total + (s * s) * np.asarray(m, np.float64)
    return total


def record(m) -> np.ndarray:
    """A 0-d SEA_STATE of the moments m with the derived fields of include/ocean.h (binary64, 0 when m0 == 0)."""
    m = [float(v) for v in m]
    r = np.zeros((), SEA_STATE)
    r["m_minus1"], r["m0"], r["m1"], r["m2"] = m[0], m[1], m[2], m[3]
    r["direction"] = m[4:6]
    r["slope"] = m[6:8]
    r["stokes"] = m[8:10]
    m0 = m[1]
    if m0 == 0.0:
        return r
    two_pi = 2.0 * math.pi
    r["significant_wave_height"] = 4.0 * math.sqrt(m0)
    r["mean_period"] = two_pi * m0 / m[2]
    r["zero_crossing_period"] = two_pi * math.sqrt(m0 / m[3])
    r["energy_period"] = two_pi * m[0] / m0
    r["mean_direction"] = math.atan2(-m[5], -m[4]) * (180.0 / math.pi)
    R = math.hypot(m[4], m[5]) / m0
    r["directional_spread"] = math.sqrt(2.0 * max(0.0, 1.0 - R))
    r["mean_square_slope"] = m[6] + m[7]
    r["stokes_speed"] = math.hypot(m[8], m[9])
    return r
