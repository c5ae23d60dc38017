"""A binary64 model of the wake layer, written from include/ocean.h's "Wake layer" block and independent of the binary32
specification (oracle/wake.py, wake_foam.py, wake_coupling.py, wake_obstacles.py).  It shares only the 28 binary32 taps
(oracle.wake.taps, which reads them from the library) and the cascades' binary32 foam decay exp, which the header defines
the foam constant d by.

Everything else is binary64 and written the way the header words it, not the way the specification orders its sums:
  * the 13 x 13 stencil is assembled from the taps by orbit class -- offset (di, dj) carries G[max(|di|, |dj|)][min(..)] --
    and applied as a zero-padded correlation (scipy.ndimage.correlate, mode "constant");
  * the coefficients a1, a2, a3 are exact per ring, the ring of a cell being min(distance to the nearest edge, sponge_cells);
  * phi and sigma are evaluated at the exact cell centres ((ox + i + 1/2) dx, (oz + j + 1/2) dx);
  * the values the header defines as binary32 stay binary32: the sub-step h = (float)(dt / S), tau = (float)k * h, the
    source fields and the foam constants d, gh, sh.
Use: Model(params) holds h, h_prev, F (binary64 [N][N]) and the origin; Model.step(...) is one step call; bound_step in
tests/test_oracle_wake_model64.py propagates the binary32 error bound alongside.
"""
from __future__ import annotations

import numpy as np
from scipy import ndimage

from oracle.wake import taps as _taps       # the library's 28 binary32 taps, nothing else of the specification

G = 9.81
R = 6
f32 = np.float32


def kernel(taps=None) -> np.ndarray:
    """[13][13] binary64: entry [dj + 6][di + 6] is G[a][b] with a = max(|di|, |dj|), b = min(|di|, |dj|); the taps come in
    the order (0,0), (1,0), (1,1), (2,0), ... (6,6), class (a, b) at a (a + 1) / 2 + b."""
    g = (_taps() if taps is None else np.asarray(taps, np.float32)).astype(np.float64)
    k = np.zeros((2 * R + 1, 2 * R + 1))
    for dj in range(-R, R + 1):
        for di in range(-R, R + 1):
            a, b = max(abs(di), abs(dj)), min(abs(di), abs(dj))
            k[dj + R, di + R] = g[a * (a + 1) // 2 + b]
    return k


def convolve(s: np.ndarray, k: np.ndarray) -> np.ndarray:
    """c[j][i] = sum over (di, dj) of K[dj][di] s[j + dj][i + di], cells outside the window reading 0."""
    return ndimage.correlate(np.asarray(s, np.float64), k, mode="constant", cval=0.0)


def substep(dt, substeps) -> float:
    return float(f32(float(dt) / int(substeps)))


def coefficients(n, sponge_cells, cell_size, damping, sponge_damping, h):
    """(a1, a2, a3) [N][N] binary64, exact (not rounded to binary32): alpha = damping in the interior and
    damping + (sponge_damping - damping) t^2, t = (sponge_cells - r) / sponge_cells, on ring r < sponge_cells."""
    i = np.arange(n)
    e = np.minimum(i, n - 1 - i)
    r = np.minimum(np.minimum(e[None, :], e[:, None]), sponge_cells).astype(np.float64)
    d, ds = float(f32(damping)), float(f32(sponge_damping))
    if sponge_cells > 0:
        t = (sponge_cells - r) / sponge_cells
        alpha = np.where(r < sponge_cells, d + (ds - d) * t * t, d)
    else:
        alpha = np.full((n, n), d)
    ah = alpha * h
    dx = float(f32(cell_size))
    return (2.0 - ah) / (1.0 + ah), 1.0 / (1.0 + ah), G * h * h / (dx * (1.0 + ah))


def corner(origin, cell_size):
    """The header's binary32 world corner x0 = (float)((double)ox * dx), as a binary64 value (+-inf when it overflows)."""
    dx = float(f32(cell_size))
    with np.errstate(over="ignore"):
        return float(f32(float(int(origin[0])) * dx)), float(f32(float(int(origin[1])) * dx))


def cell_centres(n, cell_size, origin):
    """The exact cell centres (x[i], z[j]) in binary64: (ox + i + 1/2) dx, computed from the integer ox + i (exact to
    binary64 for |ox| < 2^52; beyond, rounded once)."""
    dx = float(f32(cell_size))
    i = np.arange(n)
    x = np.array([float(int(origin[0]) + int(k)) for k in i]) + 0.5
    z = np.array([float(int(origin[1]) + int(k)) for k in i]) + 0.5
    return x * dx, z * dx


def source_terms(sources, states, tau):
    """Per source: centre (cx, cz), radius r, head, |v|^2 in binary64 and whether it contributes (the header's rule)."""
    s = np.asarray(sources).reshape(-1)
    st = np.asarray(states).reshape(-1) if states is not None else None
    ns = 0 if st is None else len(st)
    tau = float(tau)
    cx = s["x"].astype(np.float64) + s["vx"].astype(np.float64) * tau
    cz = s["z"].astype(np.float64) + s["vz"].astype(np.float64) * tau
    vx, vz = s["vx"].astype(np.float64), s["vz"].astype(np.float64)
    body = s["body"].astype(np.int64)
    ok = body < ns
    for k in np.flatnonzero((body >= 0) & ok):
        b = st[body[k]]
        cx[k] += float(b["position"][0]) + float(b["linear_velocity"][0]) * tau
        cz[k] += float(b["position"][2]) + float(b["linear_velocity"][2]) * tau
        vx[k] += float(b["linear_velocity"][0])
        vz[k] += float(b["linear_velocity"][2])
    r = s["radius"].astype(np.float64)
    head = s["head"].astype(np.float64)
    with np.errstate(all="ignore"):
        r2_32 = s["radius"] * s["radius"]
        valid = ok & np.isfinite(cx) & np.isfinite(cz) & np.isfinite(head) & np.isfinite(r) & (r > 0) & np.isfinite(r2_32)
    return cx, cz, r, head, vx * vx + vz * vz, valid


def footprint(n, cell_size, origin, sources, states, tau):
    """phi and sigma [N][N] binary64 at the exact cell centres: per contributing source with q2 = |p - c|^2 / r^2 < 1,
    w = 1 - q2, phi += head w^2 and sigma += w^2 |v|^2."""
    px, pz = cell_centres(n, cell_size, origin)
    phi, sigma = np.zeros((n, n)), np.zeros((n, n))
    cx, cz, r, head, v2, valid = source_terms(sources, states, tau)
    for k in np.flatnonzero(valid):
        q2 = ((px[None, :] - cx[k]) ** 2 + (pz[:, None] - cz[k]) ** 2) / (r[k] * r[k])
        ww = np.where(q2 < 1.0, (1.0 - q2) ** 2, 0.0)
        phi += head[k] * ww
        sigma += v2[k] * ww
    return phi, sigma


def scroll(f: np.ndarray, di: int, dj: int) -> np.ndarray:
    """out[j][i] = f[j + dj][i + di], 0 outside (a move of N cells or more clears the field)."""
    n = f.shape[0]
    out = np.zeros_like(f)
    for j in range(n):
        if 0 <= j + dj < n:
            lo, hi = max(0, -di), min(n, n - di)
            if lo < hi:
                out[j, lo:hi] = f[j + dj, lo + di:hi + di]
    return out


def blocked(mask, mask_origin, origin, n) -> np.ndarray:
    """B[j][i]: world cell (ox + i, oz + j) lies in the mask rectangle and its byte is nonzero."""
    out = np.zeros((n, n), bool)
    if mask is None:
        return out
    m = np.asarray(mask) != 0
    depth, width = m.shape
    # mask column of window column i is (ox - mx) + i; an offset clamped to just outside [-n, width] selects the same cells
    qx = max(-n - 1, min(width + 1, int(origin[0]) - int(mask_origin[0]))) + np.arange(n)
    qz = max(-n - 1, min(depth + 1, int(origin[1]) - int(mask_origin[1]))) + np.arange(n)
    inx, inz = (qx >= 0) & (qx < width), (qz >= 0) & (qz < depth)
    out[np.ix_(inz, inx)] = m[np.ix_(qz[inz], qx[inx])]
    return out


def detmath_exp(x) -> float:
    from godotoceanwaves_b200.native import load_library
    return float(f32(load_library().ocean_detmath_expf(float(f32(x)))))


class Model:
    """The layer in binary64: h, h_prev, F and the origin; foam (whitecap, grow_rate, stir_rate, decay_rate) or None; a mask."""

    def __init__(self, params, foam=None, mask=None, mask_origin=(0, 0)):
        p = np.asarray(params).reshape(())
        self.n, self.sponge_cells = int(p["size"]), int(p["sponge_cells"])
        self.cell_size, self.damping, self.sponge_damping = float(p["cell_size"]), float(p["damping"]), float(p["sponge_damping"])
        self.h = np.zeros((self.n, self.n))
        self.h_prev = np.zeros((self.n, self.n))
        self.F = np.zeros((self.n, self.n))
        self.origin = (0, 0)
        self.foam = None if foam is None else tuple(float(f32(v)) for v in foam)
        self.mask, self.mask_origin = mask, mask_origin
        self.k = kernel()

    def step(self, dt, substeps, origin, sources=None, states=None, trace=None):
        """One call.  With `trace` (a list), each sub-step appends a dict of what a binary32 error bound needs."""
        h = substep(dt, substeps)
        di, dj = int(origin[0]) - self.origin[0], int(origin[1]) - self.origin[1]
        di, dj = max(-self.n, min(self.n, di)), max(-self.n, min(self.n, dj))
        self.h, self.h_prev, self.F = scroll(self.h, di, dj), scroll(self.h_prev, di, dj), scroll(self.F, di, dj)
        self.origin = (int(origin[0]), int(origin[1]))
        a1, a2, a3 = coefficients(self.n, self.sponge_cells, self.cell_size, self.damping, self.sponge_damping, h)
        B = blocked(self.mask, self.mask_origin, self.origin, self.n)
        dx = float(f32(self.cell_size))
        if self.foam is not None:
            wc, gr, sr, dr = self.foam
            d = detmath_exp(-(f32(dr) * f32(h)))
            gh, sh = float(f32(gr) * f32(h)), float(f32(sr) * f32(h))
        src = np.zeros(0, [("x", "f4")]) if sources is None else sources
        for k in range(int(substeps)):
            tau = float(f32(k) * f32(h))
            if len(src):
                phi, sigma = footprint(self.n, self.cell_size, self.origin, src, states, tau)
            else:
                phi = sigma = np.zeros((self.n, self.n))
            s = np.where(B, 0.0, self.h + phi)
            c = convolve(s, self.k)
            new = np.where(B, 0.0, (a1 * self.h - a2 * self.h_prev) - a3 * c)
            if trace is not None:
                trace.append(dict(h=self.h, h_prev=self.h_prev, phi=phi, sigma=sigma, s=s, c=c, a=(a1, a2, a3), B=B, tau=tau,
                                  F=self.F))
            if self.foam is not None:
                b = np.maximum(c / dx - wc, 0.0)
                x = self.F * d + (gh * b + sh * sigma)
                self.F = np.where(B, 0.0, np.where(x > 0, np.minimum(x, 1.0), 0.0))
                if trace is not None:
                    trace[-1].update(b=c / dx - wc, x=x, d=d, gh=gh, sh=sh)
            self.h_prev, self.h = self.h, new
        return self

    def free_surface(self, dt, substeps, sources=None, states=None) -> np.ndarray:
        """e = h + phi_end at tau_end = (float)S * h, +0 on blocked cells."""
        h = substep(dt, substeps)
        tau = float(f32(int(substeps)) * f32(h))
        phi = footprint(self.n, self.cell_size, self.origin, sources, states, tau)[0] if sources is not None and len(sources) \
            else np.zeros((self.n, self.n))
        return np.where(blocked(self.mask, self.mask_origin, self.origin, self.n), 0.0, self.h + phi)


def gradients(h: np.ndarray, cell_size):
    """Central differences (h[i + 1] - h[i - 1]) / (2 dx) and likewise along z, cells outside reading 0."""
    p = np.pad(np.asarray(h, np.float64), 1)
    two_dx = 2.0 * float(f32(cell_size))
    return (p[1:-1, 2:] - p[1:-1, :-2]) / two_dx, (p[2:, 1:-1] - p[:-2, 1:-1]) / two_dx


def render_map(h, cell_size, foam=None) -> np.ndarray:
    """[N][N][4] binary64 (h, dh/dx, dh/dz, F or 0), before any rounding to half."""
    gx, gz = gradients(h, cell_size)
    f = np.zeros_like(gx) if foam is None else np.asarray(foam, np.float64)
    return np.stack([np.asarray(h, np.float64), gx, gz, f], -1)


def sample(h, cell_size, origin, xz) -> np.ndarray:
    """[n][3] binary64 bilinear (h, dh/dx, dh/dz) at world points, on the lattice of the exact cell centres; 0 outside the
    window [ox dx, (ox + N) dx) x [oz dx, (oz + N) dx).  u = x / dx - ox - 1/2, i = floor(u)."""
    n = h.shape[0]
    dx = float(f32(cell_size))
    fields = [np.pad(np.asarray(f, np.float64), 1) for f in (h, *gradients(h, cell_size))]
    pts = np.asarray(xz, np.float64).reshape(-1, 2)
    out = np.zeros((len(pts), 3))
    for k, (x, z) in enumerate(pts):
        u, v = x / dx - int(origin[0]) - 0.5, z / dx - int(origin[1]) - 0.5
        if not (-0.5 <= u < n - 0.5 and -0.5 <= v < n - 0.5):
            continue
        i, j = int(np.floor(u)), int(np.floor(v))
        fu, fv = u - i, v - j
        for m, f in enumerate(fields):
            q = f[j + 1:j + 3, i + 1:i + 3]
            out[k, m] = (1 - fv) * ((1 - fu) * q[0, 0] + fu * q[0, 1]) + fv * ((1 - fu) * q[1, 0] + fu * q[1, 1])
    return out
