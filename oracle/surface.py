"""CPU specification of the surface query: water height, normal and foam at a WORLD position (ocean_query_surface).

TEST INFRASTRUCTURE ONLY -- the product path (godotoceanwaves_b200/csrc) never imports or calls this module.

The water shader reads its maps at the undisplaced grid point, UV = VERTEX.xz, and only then moves the vertex,
VERTEX += displacement (assets/shaders/spatial/water.gdshader:28,37).  The surface point that starts at P therefore sits
at P + D_xz(P).  For a world position Q the query solves P + D_xz(P) = Q for P and reads the maps there:

  evaluation at P   D(P) = sum_i bilinear(disp_i, P * s_i.xy).xyz * s_i.z, accumulated as sampling.sample_maps does;
                    J = dD_xz/dP, the exact derivative of the bilinear interpolant from the same four texels:
                      d/du = mix(t10 - t00, t11 - t01, fy) * N,  d/dv = mix(t01 - t00, t11 - t10, fx) * N,
                      J += (d/du * s_i.x) * s_i.z  (column x),  J += (d/dv * s_i.y) * s_i.z  (column z).
                    Only the displacement layers are read inside the solve.
  residual          E = (P + D_xz(P)) - Q,  r = max(|E.x|, |E.z|)
  step              (I + J) step = E by Cramer's rule; where det(I + J) <= 1e-3 (or is NaN) or the step is not finite,
                    step = E (a fixed-point step)
  damping           trials P - lam * step, lam = 1, 1/2, 1/4, 1/8, 1/16: the first trial whose residual does not exceed r
                    is taken.  If none qualifies, the start stays at P and ends there (every further step would repeat
                    the same trials); the step still counts.
  stopping          a start ends when r <= tolerance, after max_iterations steps, or when it stalls as above
  restarts          if the start from P0 = Q ends with r > tolerance (and max_iterations > 0), the same solve runs from
                    Q - D_xz(Q), then Q + (rho, 0), (0, rho), (-rho, 0), (0, -rho), in this order, until one converges;
                    rho = 0.5 * sum_i |s_i.z| * max over the texels of layer i of max(|x|, |z|), summed in cascade order
                    (half the horizontal displacement bound of the maps; it depends on the maps only)
  result            the end point with the smallest r over the starts (the earlier start on ties), P:
                    source_xz = P, (displacement, gradient_foam) = sampling.sample_maps at P, residual = r at P,
                    iterations = the steps taken over all starts.
  max_iterations = 0 returns sampling.sample_maps(Q) unchanged, source_xz = Q, iterations = 0.

Numeric policy (as oracle/sampling.py): every operation binary32, rounded once, in the order written here, no contraction;
divisions IEEE; max(a, b) of non-NaN values.  The CUDA kernels (ocean_sample.cu, -fmad=false) reproduce this bit for bit.
"""
from __future__ import annotations

import numpy as np

from .sampling import F, _mix, sample_maps, texture_bilinear, wrap_texel

RECORD = np.dtype([("source_x", np.float32), ("source_z", np.float32), ("displacement", np.float32, 3),
                   ("gradient_foam", np.float32, 3), ("residual", np.float32), ("iterations", np.uint32)])   # 40 B
DET_MIN = F(1e-3)
LAMBDAS = tuple(F(1.0) / F(1 << j) for j in range(5))


def bilinear_slopes(tex: np.ndarray, u: np.ndarray, v: np.ndarray):
    """d/du and d/dv of sampling.texture_bilinear (float32 [n][4] each), from the four texels the value reads."""
    N = tex.shape[0]
    n = F(N)
    x = u * n - F(0.5)
    y = v * n - F(0.5)
    x0 = np.floor(x)
    y0 = np.floor(y)
    fx = (x - x0)[:, None]
    fy = (y - y0)[:, None]
    ix0 = wrap_texel(x0, N)
    iy0 = wrap_texel(y0, N)
    ix1 = np.mod(ix0 + 1, N)
    iy1 = np.mod(iy0 + 1, N)
    t = tex.astype(np.float32)
    t00, t10 = t[iy0, ix0], t[iy0, ix1]
    t01, t11 = t[iy1, ix0], t[iy1, ix1]
    return _mix(t10 - t00, t11 - t01, fy) * n, _mix(t01 - t00, t11 - t10, fx) * n


def _evaluate(displacement, sc, px, pz):
    """D_xz(P) and J = dD_xz/dP: (dx, dz, jxx, jxz, jzx, jzz), float32 [n] each."""
    z = np.zeros(px.shape, np.float32)
    dx, dz, jxx, jxz, jzx, jzz = z, z, z, z, z, z
    for i in range(displacement.shape[0]):
        u = px * sc[i, 0]
        v = pz * sc[i, 1]
        d = texture_bilinear(displacement[i], u, v)
        du, dv = bilinear_slopes(displacement[i], u, v)
        dx = dx + d[:, 0] * sc[i, 2]
        dz = dz + d[:, 2] * sc[i, 2]
        jxx = jxx + (du[:, 0] * sc[i, 0]) * sc[i, 2]
        jxz = jxz + (dv[:, 0] * sc[i, 1]) * sc[i, 2]
        jzx = jzx + (du[:, 2] * sc[i, 0]) * sc[i, 2]
        jzz = jzz + (dv[:, 2] * sc[i, 1]) * sc[i, 2]
    return dx, dz, jxx, jxz, jzx, jzz


def _residual(px, pz, dx, dz, qx, qz):
    ex = (px + dx) - qx
    ez = (pz + dz) - qz
    return ex, ez, np.fmax(np.abs(ex), np.abs(ez))


def _solve(displacement, sc, qx, qz, px, pz, tolerance, max_iterations):
    """One start from (px, pz) for every query.  Returns the end point, its residual and the steps taken."""
    px, pz = px.copy(), pz.copy()
    ev = _evaluate(displacement, sc, px, pz)
    ex, ez, r = _residual(px, pz, ev[0], ev[1], qx, qz)
    steps = np.zeros(px.shape, np.uint32)
    live = r > tolerance
    for _ in range(max_iterations):
        k = np.nonzero(live)[0]
        if k.size == 0:
            break
        jxx, jxz, jzx, jzz = ev[2][k], ev[3][k], ev[4][k], ev[5][k]
        a, b, c, d = F(1.0) + jxx, jxz, jzx, F(1.0) + jzz
        det = a * d - b * c
        with np.errstate(all="ignore"):
            sx = (d * ex[k] - b * ez[k]) / det
            sz = (a * ez[k] - c * ex[k]) / det
        fixed = ~(det > DET_MIN) | ~np.isfinite(sx) | ~np.isfinite(sz)
        sx = np.where(fixed, ex[k], sx)
        sz = np.where(fixed, ez[k], sz)
        taken = np.zeros(k.size, bool)
        for lam in LAMBDAS:
            t = np.nonzero(~taken)[0]
            if t.size == 0:
                break
            kt = k[t]
            tx = px[kt] - lam * sx[t]
            tz = pz[kt] - lam * sz[t]
            evt = _evaluate(displacement, sc, tx, tz)
            etx, etz, rt = _residual(tx, tz, evt[0], evt[1], qx[kt], qz[kt])
            ok = rt <= r[kt]
            t, kt = t[ok], kt[ok]
            taken[t] = True
            px[kt], pz[kt], ex[kt], ez[kt], r[kt] = tx[ok], tz[ok], etx[ok], etz[ok], rt[ok]
            for a_, b_ in zip(ev, evt):
                a_[kt] = b_[ok]
        steps[k] += 1
        live[k] = taken & (r[k] > tolerance)
    return px, pz, r, steps


def displacement_bound(displacement: np.ndarray, map_scales: np.ndarray) -> np.float32:
    """rho = 0.5 * sum_i |s_i.z| * max over layer i of max(|x|, |z|): half the horizontal displacement bound of the maps."""
    sc = np.asarray(map_scales, np.float32)
    acc = F(0.0)
    for i in range(displacement.shape[0]):
        t = displacement[i].astype(np.float32)
        m = np.fmax(np.abs(t[..., 0]), np.abs(t[..., 2])).max()
        acc = acc + np.abs(sc[i, 2]) * m
    return acc * F(0.5)


def query_surface(displacement: np.ndarray, normal: np.ndarray, points_xz: np.ndarray, map_scales: np.ndarray,
                  tolerance: float = 1e-3, max_iterations: int = 8) -> np.ndarray:
    """displacement, normal: [C][N][N][4] float16; points_xz: [n][2] world x, z; map_scales: [C][4] float32.
    Returns RECORD [n]."""
    pts = np.ascontiguousarray(points_xz, np.float32).reshape(-1, 2)
    sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
    tol = F(tolerance)
    qx, qz = pts[:, 0].copy(), pts[:, 1].copy()
    px, pz, r, steps = _solve(displacement, sc, qx, qz, qx, qz, tol, max_iterations)
    pending = np.nonzero(r > tol)[0] if max_iterations > 0 else np.zeros(0, np.int64)
    if pending.size:
        rho = displacement_bound(displacement, sc)
        k = pending
        ev = _evaluate(displacement, sc, qx[k], qz[k])
        seeds = [(qx[k] - ev[0], qz[k] - ev[1]), (qx[k] + rho, qz[k]), (qx[k], qz[k] + rho), (qx[k] - rho, qz[k]),
                 (qx[k], qz[k] - rho)]
        live = np.ones(k.size, bool)
        for sx, sz in seeds:
            j = np.nonzero(live)[0]
            if j.size == 0:
                break
            kj = k[j]
            ex_, ez_, er, es = _solve(displacement, sc, qx[kj], qz[kj], sx[j], sz[j], tol, max_iterations)
            steps[kj] += es
            better = er < r[kj]
            px[kj[better]], pz[kj[better]], r[kj[better]] = ex_[better], ez_[better], er[better]
            live[j[er <= tol]] = False
    src = np.stack([px, pz], 1)
    d, g = sample_maps(displacement, normal, src, sc)
    out = np.zeros(pts.shape[0], RECORD)
    out["source_x"], out["source_z"] = px, pz
    out["displacement"], out["gradient_foam"] = d, g
    out["residual"] = r
    out["iterations"] = steps
    return out
