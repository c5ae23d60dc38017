"""Specification of the wake layer (include/ocean.h, "Wake layer"; csrc/ocean_wake.cu matches it bit for bit): a local
N x N height field of cell size dx at an integer cell origin, advanced by explicit sub-steps of the iWave scheme (Tessendorf,
"Interactive Water Surfaces", 2004) with a radius-6 stencil for sqrt(-laplacian), forced by the pressure head of sources.

Every operation is binary32 in the order written here unless it says binary64; numpy's float32 elementwise add, subtract,
multiply and divide are IEEE round-to-nearest, as the device's _rn operations.  Fields are [N][N] float32 in window order:
row j along z, column i along x; cell (i, j) covers world x in [(origin_x + i) dx, (origin_x + i + 1) dx).
"""
from __future__ import annotations

import ctypes

import numpy as np

G = 9.81                      # wave_generator.gd:5, as the cascades' dispersion
CAP = 4.0                     # the largest Ghat(k) of the stencil (tools/fit_wake_kernel.py): the stability bound's constant
RADIUS = 6
OFFSETS = [(a, b) for a in range(RADIUS + 1) for b in range(a + 1)]     # the 28 tap classes, in summation order

SOURCE = np.dtype([("x", np.float32), ("z", np.float32), ("vx", np.float32), ("vz", np.float32), ("radius", np.float32),
                   ("head", np.float32), ("body", np.int32)])                                 # struct ocean_wake_source
PARAMS = np.dtype([("size", np.int32), ("sponge_cells", np.int32), ("cell_size", np.float32), ("damping", np.float32),
                   ("sponge_damping", np.float32)])                                           # struct ocean_wake_params
STATE = np.dtype([("position", np.float32, 3), ("orientation", np.float32, 4), ("linear_velocity", np.float32, 3),
                  ("angular_velocity", np.float32, 3)])                                       # struct ocean_body_state
f32 = np.float32


def orbit(a: int, b: int):
    """The mirrored offsets (di, dj) of tap class (a, b) in the order their values are summed."""
    if a == 0:
        return [(0, 0)]
    if b == 0:
        return [(a, 0), (-a, 0), (0, a), (0, -a)]
    if a == b:
        return [(a, a), (a, -a), (-a, a), (-a, -a)]
    return [(a, b), (a, -b), (-a, b), (-a, -b), (b, a), (b, -a), (-b, a), (-b, -a)]


def taps() -> np.ndarray:
    """The 28 binary32 taps G[a][b] in OFFSETS order, from the library's host-only entry point (no device needed)."""
    from godotoceanwaves_b200.native import check, load_library
    out = np.zeros(28, np.float32)
    check(load_library().ocean_wake_kernel_taps(out.ctypes.data_as(ctypes.c_void_p)))
    return out


def symbol(g: np.ndarray, kx, kz):
    """Ghat(k) = sum_ab G[a][b] sum_orbit cos(k . o), binary64, k in units of 1/dx."""
    kx, kz = np.asarray(kx, np.float64), np.asarray(kz, np.float64)
    return sum(float(t) * sum(np.cos(kx * di + kz * dj) for di, dj in orbit(a, b)) for t, (a, b) in zip(g, OFFSETS))


def substep(dt: float, substeps: int) -> np.float32:
    """h = dt / S in binary64, rounded once."""
    return f32(float(dt) / int(substeps))


def stable(cell_size, h) -> bool:
    """The call's stability rule: a3 at zero damping, G h^2 / dx in binary64, times CAP must not exceed 4."""
    h = float(h)
    return G * h * h / float(f32(cell_size)) * CAP <= 4.0


def coefficients(params, h):
    """(a1, a2, a3) float32 [sponge_cells + 1]: ring r < sponge_cells (r cells from the window edge) has damping
    alpha = damping + (sponge_damping - damping) t^2, t = (sponge_cells - r) / sponge_cells; the last entry is the interior's
    (alpha = damping).  Binary64 from the binary32 parameters, each coefficient rounded to binary32 once."""
    p = np.asarray(params, PARAMS).reshape(())
    sc, dx = int(p["sponge_cells"]), float(p["cell_size"])
    d, ds, h = float(p["damping"]), float(p["sponge_damping"]), float(h)
    out = np.zeros((3, sc + 1), np.float32)
    for r in range(sc + 1):
        if r < sc:
            t = (sc - r) / sc
            alpha = d + (ds - d) * (t * t)
        else:
            alpha = d
        ah = alpha * h
        out[0, r] = (2.0 - ah) / (1.0 + ah)
        out[1, r] = 1.0 / (1.0 + ah)
        out[2, r] = G * h * h / (dx * (1.0 + ah))
    return out


def ring(n: int, sponge_cells: int) -> np.ndarray:
    """[N][N] index into the coefficient table: min(distance to the nearest window edge in cells, sponge_cells)."""
    i = np.arange(n)
    e = np.minimum(i, n - 1 - i)
    return np.minimum(np.minimum(e[:, None], e[None, :]), sponge_cells)


def scroll(f: np.ndarray, di: int, dj: int) -> np.ndarray:
    """The field of a window moved by (di, dj) cells: out[j][i] = f[j + dj][i + di], 0 where that lies outside."""
    n = f.shape[0]
    out = np.zeros_like(f)
    if abs(di) >= n or abs(dj) >= n:
        return out
    src = f[max(dj, 0):n + min(dj, 0), max(di, 0):n + min(di, 0)]
    out[max(-dj, 0):max(-dj, 0) + src.shape[0], max(-di, 0):max(-di, 0) + src.shape[1]] = src
    return out


def world_origin(origin, cell_size):
    """The window's world corner (x0, z0): (double)origin * (double)dx, rounded to binary32."""
    return f32(float(origin[0]) * float(f32(cell_size))), f32(float(origin[1]) * float(f32(cell_size)))


def centres(sources, states, tau):
    """Per source at sub-step time tau (binary32): centre c = (x + vx tau, z + vz tau), plus position.xz + linear_velocity.xz
    tau of its body when body >= 0, and whether it contributes: a body index inside the states, c, head and radius finite,
    radius > 0 and radius^2 finite.  Returns cx, cz, r2, head, valid."""
    s = np.asarray(sources, SOURCE).reshape(-1)
    st = np.asarray(states, STATE).reshape(-1) if states is not None else np.zeros(0, STATE)
    tau = f32(tau)
    with np.errstate(all="ignore"):
        cx = s["x"] + s["vx"] * tau
        cz = s["z"] + s["vz"] * tau
        b = s["body"]
        ok = b < len(st)
        att = (b >= 0) & ok
        if np.any(att):
            bs = st[b[att]]
            cx[att] = cx[att] + (bs["position"][:, 0] + bs["linear_velocity"][:, 0] * tau)
            cz[att] = cz[att] + (bs["position"][:, 2] + bs["linear_velocity"][:, 2] * tau)
        r2 = s["radius"] * s["radius"]
        valid = ok & np.isfinite(cx) & np.isfinite(cz) & np.isfinite(s["head"]) & np.isfinite(s["radius"]) & (s["radius"] > 0) \
            & np.isfinite(r2)
    return cx, cz, r2, s["head"].copy(), valid


def footprint_box(p: np.ndarray, c, r, margin: int = 2):
    """[lo, hi) of the cells along one axis that a source of centre c and radius r can reach, for non-decreasing binary32
    centres p (x0 + (i + 0.5) dx is monotone in i).  A cell with p > fl(c + r) has c + r < p exactly (rounding is monotone
    and p is a binary32), so fl(p - c) >= r, fl(ex ex) >= fl(r r) = r2 and d2 >= r2: it is outside; likewise below
    fl(c - r).  `margin` more cells on each side are visited as well."""
    lo = int(np.searchsorted(p, f32(c) - f32(r), "left"))
    hi = int(np.searchsorted(p, f32(c) + f32(r), "right"))
    return max(lo - margin, 0), min(hi + margin, len(p))


def rasterise(n, cell_size, origin, sources, states, tau, box=True) -> np.ndarray:
    """phi [N][N]: at each cell centre p = (x0 + (i + 0.5) dx, z0 + (j + 0.5) dz), in source index order, for each
    contributing source with d2 = (px - cx)^2 + (pz - cz)^2 < r2:  q2 = d2 / r2,  w = 1 - q2,  phi += head (w w).
    box=True visits only the cells of footprint_box (cells outside it cannot satisfy d2 < r2); box=False every cell.
    Both give the same bytes."""
    dx = f32(cell_size)
    x0, z0 = world_origin(origin, dx)
    c = (np.arange(n, dtype=np.float32) + f32(0.5)) * dx
    with np.errstate(all="ignore"):
        px, pz = x0 + c, z0 + c
    phi = np.zeros((n, n), np.float32)
    cx, cz, r2, head, valid = centres(sources, states, tau)
    radius = np.asarray(sources, SOURCE).reshape(-1)["radius"]
    with np.errstate(all="ignore"):
        for k in np.flatnonzero(valid):
            i0, i1 = footprint_box(px, cx[k], radius[k]) if box else (0, n)
            j0, j1 = footprint_box(pz, cz[k], radius[k]) if box else (0, n)
            if i0 >= i1 or j0 >= j1:
                continue
            ex, ez = px[None, i0:i1] - cx[k], pz[j0:j1, None] - cz[k]
            d2 = ex * ex + ez * ez
            inside = d2 < r2[k]
            w = f32(1.0) - d2 / r2[k]
            sub = phi[j0:j1, i0:i1]
            phi[j0:j1, i0:i1] = np.where(inside, sub + head[k] * (w * w), sub)
    return phi


def convolve(s: np.ndarray, g: np.ndarray) -> np.ndarray:
    """c = G[0][0] s + sum over the other 27 classes in OFFSETS order of G[a][b] (the orbit's values summed left to right);
    cells outside the window read 0."""
    n = s.shape[0]
    R = RADIUS
    p = np.zeros((n + 2 * R, n + 2 * R), np.float32)
    p[R:R + n, R:R + n] = s

    def at(di, dj):
        return p[R + dj:R + dj + n, R + di:R + di + n]

    c = None
    for t, (a, b) in zip(g, OFFSETS):
        o = orbit(a, b)
        acc = at(*o[0])
        for di, dj in o[1:]:
            acc = acc + at(di, dj)
        c = t * acc if c is None else c + t * acc
    return c


class Layer:
    """The wake layer's state: parameters, h, h_prev (float32 [N][N]) and the origin in cells (int x, z)."""

    def __init__(self, params):
        self.params = np.asarray(params, PARAMS).reshape(()).copy()
        n = int(self.params["size"])
        self.h = np.zeros((n, n), np.float32)
        self.h_prev = np.zeros((n, n), np.float32)
        self.origin = (0, 0)

    @property
    def n(self):
        return self.h.shape[0]

    @property
    def cell_size(self):
        return f32(self.params["cell_size"])

    def step(self, dt, substeps, origin, sources=None, states=None):
        """One call: the scroll to `origin`, then `substeps` sub-steps of h = dt / substeps with the sources at
        tau_k = (float)k * h."""
        h = substep(dt, substeps)
        assert stable(self.cell_size, h)
        di, dj = int(origin[0]) - self.origin[0], int(origin[1]) - self.origin[1]
        self.h, self.h_prev = scroll(self.h, di, dj), scroll(self.h_prev, di, dj)
        self.origin = (int(origin[0]), int(origin[1]))
        a1, a2, a3 = coefficients(self.params, h)
        rg = ring(self.n, int(self.params["sponge_cells"]))
        a1, a2, a3 = a1[rg], a2[rg], a3[rg]
        g = taps()
        src = np.zeros(0, SOURCE) if sources is None else np.asarray(sources, SOURCE).reshape(-1)
        for k in range(int(substeps)):
            phi = rasterise(self.n, self.cell_size, self.origin, src, states, f32(k) * h) if len(src) else np.zeros_like(self.h)
            c = convolve(self.h + phi, g)
            with np.errstate(all="ignore"):
                new = (a1 * self.h - a2 * self.h_prev) - a3 * c
            self.h_prev, self.h = self.h, new
        return self

    def render_map(self) -> np.ndarray:
        return render_map(self.h, self.cell_size)

    def sample(self, xz) -> np.ndarray:
        return sample(self.h, self.cell_size, self.origin, xz)


def gradients(h: np.ndarray, cell_size):
    """Central differences (h[i + 1] - h[i - 1]) / (2 dx) along x and z, cells outside the window reading 0."""
    n = h.shape[0]
    p = np.zeros((n + 2, n + 2), np.float32)
    p[1:-1, 1:-1] = h
    two_dx = f32(2.0) * f32(cell_size)
    with np.errstate(all="ignore"):
        gx = (p[1:-1, 2:] - p[1:-1, :-2]) / two_dx
        gz = (p[2:, 1:-1] - p[:-2, 1:-1]) / two_dx
    return gx, gz


def render_map(h: np.ndarray, cell_size) -> np.ndarray:
    """[N][N][4] float16 (h, dh/dx, dh/dz, 0) in window order, each rounded to nearest even from binary32."""
    gx, gz = gradients(h, cell_size)
    return np.stack([h, gx, gz, np.zeros_like(h)], axis=-1).astype(np.float16)


def sample(h: np.ndarray, cell_size, origin, xz) -> np.ndarray:
    """[n][3] float32 (h, dh/dx, dh/dz) at world points (x, z): 0 unless x0 <= x < x0 + N dx and likewise z (x0 + N dx in
    binary32 as (x0 + (float)N * dx)); else u = (x - x0) / dx - 0.5, i = floor(u), f = u - i (likewise v, j, g) and, per
    field (h and render_map's central differences, cells outside the window reading 0),
    top = f00 + f (f10 - f00),  bottom = f01 + f (f11 - f01),  value = top + g (bottom - top)."""
    n = h.shape[0]
    dx = f32(cell_size)
    x0, z0 = world_origin(origin, dx)
    pts = np.asarray(xz, np.float32).reshape(-1, 2)
    x, z = pts[:, 0], pts[:, 1]
    ext = f32(n) * dx
    out = np.zeros((len(pts), 3), np.float32)
    with np.errstate(all="ignore"):
        inside = (x >= x0) & (x < x0 + ext) & (z >= z0) & (z < z0 + ext)
        u = (x - x0) / dx - f32(0.5)
        v = (z - z0) / dx - f32(0.5)
        fi, fj = np.floor(u), np.floor(v)
        fu, fv = u - fi, v - fj
    gx, gz = gradients(h, dx)
    for k in np.flatnonzero(inside):
        i, j = int(fi[k]), int(fj[k])
        for m, f in enumerate((h, gx, gz)):
            def at(ii, jj):
                return f[jj, ii] if 0 <= ii < n and 0 <= jj < n else f32(0.0)
            with np.errstate(all="ignore"):
                top = at(i, j) + fu[k] * (at(i + 1, j) - at(i, j))
                bot = at(i, j + 1) + fu[k] * (at(i + 1, j + 1) - at(i, j + 1))
                out[k, m] = top + fv[k] * (bot - top)
    return out
