"""Fits the wake layer's vertical-derivative stencil (include/ocean.h, "Wake layer"): the 28 taps G[a][b], 0 <= b <= a <= 6,
of a radius-6 radial 13 x 13 stencil whose symbol approximates |k| dx, the operator sqrt(-laplacian) of deep-water waves.

A minimax linear program (scipy linprog, HiGHS) over the taps and the error bound t:
    minimise t  subject to  |Ghat(k) / |k| - 1| <= t  for |k| in [K_LO, K_HI] (units of 1/dx), every direction;
                            sum G = 0                  (the k = 0 mode is neutral);
                            MU (2 - cos kx - cos kz) <= Ghat(k) <= CAP - MARGIN   on a dense grid of the Brillouin zone
                                                       (no mode grows, with room left for the grid and the rounding; CAP
                                                       sets the largest stable sub-step, h^2 <= 4 dx / (g CAP)).
The taps are then rounded to multiples of 2^-23 and the centre tap set to minus the sum of the others, which makes the sum
of the 169 binary32 taps exactly zero.
Ghat(k) = sum_ab G[a][b] S_ab(k), S_ab the sum of cos(k . o) over the up-to-8 mirrored offsets o of (a, b).

Prints the taps as C hex-float literals (0x1.cb69a8p+0f) that paste into csrc/ocean_wake.cu's wake_tap table, with their sum, the least and largest Ghat on a denser grid (the
library's stability check takes CAP as the bound) and the band error reached.  Run: python tools/fit_wake_kernel.py
"""
from __future__ import annotations

import numpy as np
from scipy.optimize import linprog

R = 6
K_LO, K_HI = 0.4, 2.0
CAP = 4.0
MU = 0.02
MARGIN = 0.01
OFFSETS = [(a, b) for a in range(R + 1) for b in range(a + 1)]   # the specification's tap order


def orbit(a: int, b: int):
    """The mirrored offsets (dx, dz) of class (a, b), in the order the step sums them."""
    if a == 0:
        return [(0, 0)]
    if b == 0:
        return [(a, 0), (-a, 0), (0, a), (0, -a)]
    if a == b:
        return [(a, a), (a, -a), (-a, a), (-a, -a)]
    return [(a, b), (a, -b), (-a, b), (-a, -b), (b, a), (b, -a), (-b, a), (-b, -a)]


def basis(kx: np.ndarray, kz: np.ndarray) -> np.ndarray:
    """[len(k)][28] symbols S_ab(k) of the 28 tap classes (binary64)."""
    cols = [sum(np.cos(kx * dx + kz * dz) for dx, dz in orbit(a, b)) for a, b in OFFSETS]
    return np.stack([np.broadcast_to(c, kx.shape) for c in cols], axis=1)


def zone(n: int):
    """The fundamental triangle 0 <= kz <= kx <= pi of the Brillouin zone on an n-point axis (the symbol is even in each
    component and symmetric under their exchange)."""
    ax = np.linspace(0.0, np.pi, n)
    kx, kz = np.meshgrid(ax, ax, indexing="ij")
    m = kz <= kx
    return kx[m], kz[m]


def band(nk: int = 64, nth: int = 24):
    k = np.linspace(K_LO, K_HI, nk)
    th = np.linspace(0.0, np.pi / 4, nth)
    kk, tt = np.meshgrid(k, th, indexing="ij")
    return (kk * np.cos(tt)).ravel(), (kk * np.sin(tt)).ravel()


def fit():
    bx, bz = band()
    kn = np.hypot(bx, bz)
    A = basis(bx, bz) / kn[:, None]                     # Ghat / |k|
    zx, zz = zone(161)
    Z = basis(zx, zz)
    floor = MU * (2.0 - np.cos(zx) - np.cos(zz))
    n = len(OFFSETS)
    ones = np.ones((len(kn), 1))
    A_ub = np.vstack([np.hstack([A, -ones]), np.hstack([-A, -ones]),                 # |A g - 1| <= t
                      np.hstack([-Z, np.zeros((len(Z), 1))]),                         # Ghat >= MU (2 - cos kx - cos kz)
                      np.hstack([Z, np.zeros((len(Z), 1))])])                         # Ghat <= CAP - MARGIN
    b_ub = np.concatenate([np.ones(len(kn)), -np.ones(len(kn)), -floor, np.full(len(Z), CAP - MARGIN)])
    counts = np.array([len(orbit(a, b)) for a, b in OFFSETS], float)
    A_eq = np.concatenate([counts, [0.0]])[None, :]                                   # sum over all 169 taps = 0
    c = np.zeros(n + 1)
    c[-1] = 1.0
    res = linprog(c, A_ub=A_ub, b_ub=b_ub, A_eq=A_eq, b_eq=[0.0], bounds=[(None, None)] * n + [(0, None)], method="highs")
    assert res.status == 0, res.message
    g = np.round(res.x[:n] * 2.0**23) / 2.0**23
    g[0] = -(counts[1:] @ g[1:])                    # a multiple of 2^-23 below 2 in magnitude: exact in binary32
    return g.astype(np.float32), res.x[-1]


def report(taps: np.ndarray) -> dict:
    """Sum, min / max of Ghat on a dense grid and the band error of binary32 taps (binary64 evaluation)."""
    g = taps.astype(np.float64)
    counts = np.array([len(orbit(a, b)) for a, b in OFFSETS], float)
    zx, zz = zone(801)
    gz = basis(zx, zz) @ g
    bx, bz = band(256, 64)
    rel = basis(bx, bz) @ g / np.hypot(bx, bz) - 1.0
    return dict(sum=float(counts @ g), min=float(gz.min()), max=float(gz.max()), band_error=float(np.abs(rel).max()))


def hex_literal(v) -> str:
    """A binary32 value as the C hex-float literal of ocean_wake.cu (exact: binary32 fits in the 13 hex digits)."""
    m, e = float(v).hex().split("p")
    if "." in m:
        m = m.rstrip("0").rstrip(".")
    return f"{m}p{e}f"


if __name__ == "__main__":
    taps, t = fit()
    r = report(taps)
    print(f"band [{K_LO}, {K_HI}] / dx, cap {CAP}: LP error {t:.5f}; binary32 taps: {r}")
    for (a, b), v in zip(OFFSETS, taps):
        print(f"        {hex_literal(v) + ',':<18}// G[{a}][{b}]")
