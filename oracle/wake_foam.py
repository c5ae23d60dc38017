"""Specification of the wake layer's foam (include/ocean.h, "Wake layer", ocean_wake_set_foam; csrc/ocean_wake.cu's
k_wake_step_foam and k_wake_map_foam match it bit for bit): a field F ([N][N] float32 in window order, values in [0, 1]) of
white water where the wake breaks and where sources stir it, advanced by every sub-step of the layer.

It composes oracle/wake.py and changes none of it: h and h_prev advance exactly as wake.Layer advances them, and F reads
them without feeding anything back.  Per call, in binary32:  d = ocean_detmath_expf(-(decay_rate * h)),
gh = grow_rate * h,  sh = stir_rate * h.  Per sub-step at tau_k, per cell, with c the sub-step's convolution of h + phi:
    beta  = c / dx                                   (wake.convolve's c; the cell's downward acceleration in units of g)
    sigma = sum over the sources that add to phi at the cell, in source index order, of (w w) * |v|^2
            (w = 1 - d2 / r2 of wake.rasterise; v = (vx, vz) + linear_velocity.xz of the body state when body >= 0,
            |v|^2 = vx vx + vz vz)
    b = beta - whitecap, 0 unless b > 0;   x = F d + (gh b + sh sigma);   F' = min(x, 1) if x > 0 else 0
F scrolls with the window as h does (wake.scroll).  "x > 0 ? x : 0" is fmaxf(x, 0) (NaN gives 0) that also maps -0 to +0.
"""
from __future__ import annotations

import numpy as np

from oracle import wake

f32 = np.float32
FOAM_PARAMS = np.dtype([("whitecap", np.float32), ("grow_rate", np.float32), ("stir_rate", np.float32),
                        ("decay_rate", np.float32)])                                         # struct ocean_wake_foam_params


def foam_params(whitecap=0.0, grow_rate=0.0, stir_rate=0.0, decay_rate=0.0) -> np.ndarray:
    p = np.zeros((), FOAM_PARAMS)
    p["whitecap"], p["grow_rate"], p["stir_rate"], p["decay_rate"] = whitecap, grow_rate, stir_rate, decay_rate
    return p


def detmath_exp(x) -> np.float32:
    """The cascades' host DETMATH exp of a binary32 argument (ocean_detmath_expf; no device needed)."""
    from godotoceanwaves_b200.native import load_library
    return f32(load_library().ocean_detmath_expf(float(f32(x))))


def constants(params, h):
    """(d, gh, sh) of a call with sub-step h: exp(-(decay_rate h)), grow_rate h, stir_rate h, each binary32."""
    p = np.asarray(params, FOAM_PARAMS).reshape(())
    h = f32(h)
    return detmath_exp(-(p["decay_rate"] * h)), f32(p["grow_rate"] * h), f32(p["stir_rate"] * h)


def speed2(sources, states) -> np.ndarray:
    """|v|^2 per source: v = (vx, vz), plus linear_velocity.xz of its body state when 0 <= body < len(states)."""
    s = np.asarray(sources, wake.SOURCE).reshape(-1)
    st = np.asarray(states, wake.STATE).reshape(-1) if states is not None else np.zeros(0, wake.STATE)
    vx, vz = s["vx"].copy(), s["vz"].copy()
    att = (s["body"] >= 0) & (s["body"] < len(st))
    with np.errstate(all="ignore"):
        if np.any(att):
            lv = st[s["body"][att]]["linear_velocity"]
            vx[att] = vx[att] + lv[:, 0]
            vz[att] = vz[att] + lv[:, 2]
        return vx * vx + vz * vz


def stir(n, cell_size, origin, sources, states, tau) -> np.ndarray:
    """sigma [N][N]: wake.rasterise's cells, sources, test and weight w, summing (w w) |v|^2 instead of head (w w)."""
    dx = f32(cell_size)
    x0, z0 = wake.world_origin(origin, dx)
    c = (np.arange(n, dtype=np.float32) + f32(0.5)) * dx
    px, pz = (x0 + c)[None, :], (z0 + c)[:, None]
    sigma = np.zeros((n, n), np.float32)
    cx, cz, r2, _, valid = wake.centres(sources, states, tau)
    v2 = speed2(sources, states)
    with np.errstate(all="ignore"):
        for k in np.flatnonzero(valid):
            ex, ez = px - cx[k], pz - cz[k]
            d2 = ex * ex + ez * ez
            inside = d2 < r2[k]
            w = f32(1.0) - d2 / r2[k]
            sigma = np.where(inside, sigma + (w * w) * v2[k], sigma)
    return sigma


def update(foam, c, sigma, cell_size, whitecap, d, gh, sh) -> np.ndarray:
    """F' of one sub-step from F, the convolution c and sigma."""
    with np.errstate(all="ignore"):
        b = c / f32(cell_size) - f32(whitecap)
        b = np.where(b > 0, b, f32(0.0)).astype(np.float32)
        x = foam * f32(d) + (f32(gh) * b + f32(sh) * sigma)
        return np.where(x > 0, np.minimum(x, f32(1.0)), f32(0.0)).astype(np.float32)


class Layer(wake.Layer):
    """wake.Layer with foam: its h, h_prev and origin, plus F and the foam parameters."""

    def __init__(self, params, foam=None):
        super().__init__(params)
        self.foam_params = np.asarray(foam if foam is not None else foam_params(), FOAM_PARAMS).reshape(()).copy()
        self.foam = np.zeros_like(self.h)
        self.betas = []                 # with record_beta, c / dx of every sub-step (for tests)
        self.record_beta = False

    def step(self, dt, substeps, origin, sources=None, states=None):
        """wake.Layer.step's scroll and sub-steps, with F advanced after each sub-step from its c and sigma."""
        h = wake.substep(dt, substeps)
        assert wake.stable(self.cell_size, h)
        di, dj = int(origin[0]) - self.origin[0], int(origin[1]) - self.origin[1]
        self.h, self.h_prev = wake.scroll(self.h, di, dj), wake.scroll(self.h_prev, di, dj)
        self.foam = wake.scroll(self.foam, di, dj)
        self.origin = (int(origin[0]), int(origin[1]))
        a1, a2, a3 = wake.coefficients(self.params, h)
        rg = wake.ring(self.n, int(self.params["sponge_cells"]))
        a1, a2, a3 = a1[rg], a2[rg], a3[rg]
        g = wake.taps()
        d, gh, sh = constants(self.foam_params, h)
        src = np.zeros(0, wake.SOURCE) if sources is None else np.asarray(sources, wake.SOURCE).reshape(-1)
        for k in range(int(substeps)):
            tau = f32(k) * h
            if len(src):
                phi = wake.rasterise(self.n, self.cell_size, self.origin, src, states, tau)
                sigma = stir(self.n, self.cell_size, self.origin, src, states, tau)
            else:
                phi = sigma = np.zeros_like(self.h)
            c = wake.convolve(self.h + phi, g)
            with np.errstate(all="ignore"):
                new = (a1 * self.h - a2 * self.h_prev) - a3 * c
            self.foam = update(self.foam, c, sigma, self.cell_size, self.foam_params["whitecap"], d, gh, sh)
            if self.record_beta:
                with np.errstate(all="ignore"):
                    self.betas.append(c / self.cell_size)
            self.h_prev, self.h = self.h, new
        return self

    def render_map(self) -> np.ndarray:
        return render_map(self.h, self.foam, self.cell_size)


def render_map(h: np.ndarray, foam: np.ndarray, cell_size) -> np.ndarray:
    """[N][N][4] float16 (h, dh/dx, dh/dz, F) in window order, each rounded to nearest even from binary32."""
    gx, gz = wake.gradients(h, cell_size)
    return np.stack([h, gx, gz, foam], axis=-1).astype(np.float16)
