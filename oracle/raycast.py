"""CPU specification of the ray cast against the displaced water surface (ocean_raycast): the first crossing of each ray.

TEST INFRASTRUCTURE ONLY -- the product path (godotoceanwaves_b200/csrc) never imports or calls this module.

The surface is the one oracle/surface.py describes: the point that starts at the undisplaced P is rendered at
S(P) = (P.x + D.x(P), D.y(P), P.z + D.z(P)).  Along a ray r(t) = o + t d the gap is g(t) = r_y(t) - eta(r_xz(t)), eta the
water height over r_xz(t) from the surface inversion; a point is above the water iff g > 0.

  ray check    a ray is INVALID (every other field 0) unless o and d are finite, d != 0 and t_max >= 0 (+inf allowed)
  layer bounds per layer i, over its texels (NaN-dropping, as the device's fmaxf): ymax_i = max y, ymin_i = min y,
               m_i = max(max(|x|, |z|)) from 0
  slab         from 0, in cascade order:  a = s_i.z * ymin_i,  b = s_i.z * ymax_i,
                 Y_lo = Y_lo + fmin(a, b),  Y_hi = Y_hi + fmax(a, b),  acc = acc + |s_i.z| * fmax(|ymin_i|, |ymax_i|),
                 rho = rho + |s_i.z| * m_i;
               rho = rho * 0.5 (surface.displacement_bound, the restarts' rho),  pad = tolerance + acc * 2^-13,
               lo = Y_lo - pad,  hi = Y_hi + pad.  The heights of the maps lie in [Y_lo, Y_hi] up to rounding of their sums;
               pad covers that rounding for hundreds of cascades, and the tolerance.
  clip         d.y == 0:  t_in = 0, t_out = t_max, the ray enters iff lo <= o.y <= hi;
               otherwise  ta = (lo - o.y) / d.y,  tb = (hi - o.y) / d.y,  tn = ta < tb ? ta : tb,  tf = ta < tb ? tb : ta,
                          t_in = tn > 0 ? tn : 0,  t_out = tf < t_max ? tf : t_max,
                          the ray enters iff t_in <= t_out and t_in is finite.
               A ray that does not enter is a MISS with 0 evaluations, t = 0, position = o, every other field 0.
  march        hs = sqrt(d.x * d.x + d.z * d.z) (correctly rounded),  h = step / hs  (+inf for a vertical ray).
               Sample 0 is at t_in.  After sample k - 1 the next parameter is t = t_in + float(k) * h; where not t < t_out it
               is t_out, and where that is not finite the segment has ended (MISS, the record of sample k - 1).
               After each sample, in this order: a gap that is NaN stops the ray (INVALID, this sample's record); a side
               other than sample 0's brackets a crossing between the previous sample and this one (refinement); t == t_out
               ends the segment (MISS, this sample's record); max_samples samples taken ends the march (TRUNCATED, this
               sample's record).
  evaluation   at parameter t:  x = o.x + t * d.x,  y = o.y + t * d.y,  z = o.z + t * d.z,  Q = (x, z).  The start is Q for
               sample 0 and whenever max_iterations = 0; otherwise it is the warm start from an evaluated point e,
               (e.source_x + (x - e.x), e.source_z + (z - e.z)), e = the previous sample in the march and the nearer
               bracket end in the refinement.  surface._solve runs from the start; if its residual is not <= tolerance
               and max_iterations > 0, surface.query_surface's restarts follow (Q - D_xz(Q), then Q + (rho, 0), (0, rho),
               (-rho, 0), (0, -rho), each until one converges; the smallest residual wins, the earlier start on ties; the
               warm start counts as the first).  Sample 0 is thus ocean_query_surface(Q)'s solve, and max_iterations = 0
               gives eta = the map height at Q (a height-field march).  With P the end point:
                 eta = sum_i bilinear(disp_i, P * s_i.xy).y * s_i.z  (from 0, in cascade order: sampling.sample_maps' y),
                 g = y - eta.
               The evaluation's Newton steps add to `iterations`; it adds 1 to `unconverged` unless its residual is
               <= tolerance.
  refinement   on the bracket a = the earlier sample, b = the later one (g_a and g_b of opposite sides), with interpolation
               weights wa = g_a, wb = g_b, Illinois regula falsi.  While fewer than 32 steps have run and neither
               |g_a| <= tolerance nor |g_b| <= tolerance:
                 w = wa / (wa - wb),  t = t_a + w * (t_b - t_a); stop unless t_a < t < t_b;
                 evaluate at t, warm-started from a if (t - t_a) <= (t_b - t), else from b; a NaN gap stops the ray
                 (INVALID, this evaluation's record);
                 on a's side (g > 0 equals sample 0's side): if the previous step also replaced a, wb = wb * 0.5; a = the
                 new point, wa = g;  otherwise: if the previous step also replaced b, wa = wa * 0.5; b = the new point, wb = g.
               The reported point is a if |g_a| <= |g_b|, else b.  Status HIT_FROM_ABOVE when sample 0 was above, else
               HIT_FROM_BELOW.
  record       t, position = (x, y, z), source = P, (displacement, gradient_foam) = sampling.sample_maps at P, gap = g,
               residual = the inversion residual at P, status, evaluations (march samples + refinement evaluations),
               iterations, unconverged.

Numeric policy (as oracle/surface.py): every operation binary32, rounded once, in the order written here, no contraction;
divisions IEEE; fmin / fmax drop NaN.  The CUDA kernels (ocean_sample.cu, -fmad=false, __fdiv_rn / __fsqrt_rn) reproduce
this bit for bit.  Rays are independent: this module runs them in lock step, one sample or refinement step at a time.
"""
from __future__ import annotations

import numpy as np

from .sampling import F, sample_maps, texture_bilinear
from .surface import _evaluate, _solve

RAY = np.dtype([("origin", np.float32, 3), ("direction", np.float32, 3), ("t_max", np.float32)])          # 28 B
HIT = np.dtype([("t", np.float32), ("position", np.float32, 3), ("source_x", np.float32), ("source_z", np.float32),
                ("displacement", np.float32, 3), ("gradient_foam", np.float32, 3), ("gap", np.float32),
                ("residual", np.float32), ("status", np.uint32), ("evaluations", np.uint32), ("iterations", np.uint32),
                ("unconverged", np.uint32)])                                                                  # 72 B
MISS, HIT_FROM_ABOVE, HIT_FROM_BELOW, TRUNCATED, INVALID = range(5)
MAX_REFINE = 32
PAD_SCALE = F(2.0 ** -13)
# one row per gap evaluation (raycast(..., trace=True)); kind 0 = march sample, 1 = refinement
TRACE = np.dtype([("ray", np.int64), ("kind", np.uint8), ("t", np.float32), ("position", np.float32, 3),
                  ("source_x", np.float32), ("source_z", np.float32), ("residual", np.float32), ("iterations", np.uint32),
                  ("gap", np.float32)])


class _Widened(np.ndarray):
    """Displacement layers already widened to binary32, whose astype(float32) is the array itself: the shared sampling helpers
    widen their texture on every read, and widening half to binary32 is exact, so doing it once per call changes no bit."""

    def astype(self, dtype, *args, **kwargs):
        if np.dtype(dtype) == np.float32:
            return self
        return np.asarray(self).astype(dtype, *args, **kwargs)


def layer_bounds(displacement: np.ndarray):
    """(ymin, ymax, m) float32 [C] each: the y range of each layer and max(|x|, |z|) over it, NaN-dropping."""
    C = displacement.shape[0]
    ymin, ymax, m = (np.zeros(C, np.float32) for _ in range(3))
    ninf = F(-np.inf)
    with np.errstate(invalid="ignore"):
        for i in range(C):
            t = displacement[i].astype(np.float32).reshape(-1, 4)
            ymax[i] = np.fmax.reduce(t[:, 1], initial=ninf)
            ymin[i] = -np.fmax.reduce(-t[:, 1], initial=ninf)
            m[i] = np.fmax.reduce(np.fmax(np.abs(t[:, 0]), np.abs(t[:, 2])), initial=F(0.0))
    return ymin, ymax, m


def slab(displacement: np.ndarray, map_scales: np.ndarray, tolerance: float):
    """(lo, hi, y_lo, y_hi, rho) float32: the padded and unpadded height slab of the maps, and the restarts' rho."""
    sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
    ymin, ymax, m = layer_bounds(displacement)
    y_lo = y_hi = acc = rho = F(0.0)
    with np.errstate(all="ignore"):
        for i in range(displacement.shape[0]):
            s = sc[i, 2]
            a, b = s * ymin[i], s * ymax[i]
            y_lo = y_lo + np.fmin(a, b)
            y_hi = y_hi + np.fmax(a, b)
            acc = acc + np.abs(s) * np.fmax(np.abs(ymin[i]), np.abs(ymax[i]))
            rho = rho + np.abs(s) * m[i]
        rho = rho * F(0.5)
        pad = F(tolerance) + acc * PAD_SCALE
        return F(y_lo - pad), F(y_hi + pad), F(y_lo), F(y_hi), F(rho)


def _height(displacement, sc, px, pz):
    """sum_i bilinear(disp_i, P * s_i.xy).y * s_i.z: the y component of sampling.sample_maps' displacement."""
    eta = np.zeros(px.shape, np.float32)
    for i in range(displacement.shape[0]):
        eta = eta + texture_bilinear(displacement[i], px * sc[i, 0], pz * sc[i, 1])[:, 1] * sc[i, 2]
    return eta


def _gap(displacement, sc, tol, max_iterations, rho, x, y, z, sx, sz):
    """One gap evaluation per row: the inversion at Q = (x, z) from the start (sx, sz), with the surface query's restarts.
    Returns (source_x, source_z, residual, steps, gap)."""
    px, pz, r, steps = _solve(displacement, sc, x, z, sx, sz, tol, max_iterations)
    if max_iterations > 0:
        k = np.nonzero(~(r <= tol))[0]
        if k.size:
            ev = _evaluate(displacement, sc, x[k], z[k])
            seeds = [(x[k] - ev[0], z[k] - ev[1]), (x[k] + rho, z[k]), (x[k], z[k] + rho), (x[k] - rho, z[k]), (x[k], z[k] - rho)]
            live = np.ones(k.size, bool)
            for s_x, s_z in seeds:
                j = np.nonzero(live)[0]
                if j.size == 0:
                    break
                kj = k[j]
                ex_, ez_, er, es = _solve(displacement, sc, x[kj], z[kj], s_x[j], s_z[j], tol, max_iterations)
                steps[kj] += es
                better = er < r[kj]
                px[kj[better]], pz[kj[better]], r[kj[better]] = ex_[better], ez_[better], er[better]
                live[j[er <= tol]] = False
    return np.asarray(px), np.asarray(pz), np.asarray(r), np.asarray(steps), np.asarray(y - _height(displacement, sc, px, pz))


class _Points:
    """Evaluated points of a set of rays: t, position, source, residual, gap (float32 [n] each)."""
    FIELDS = ("t", "x", "y", "z", "px", "pz", "r", "g")

    def __init__(self, n):
        for f in self.FIELDS:
            setattr(self, f, np.zeros(n, np.float32))

    def put(self, idx, vals):
        for f, v in zip(self.FIELDS, vals):
            getattr(self, f)[idx] = v

    def take(self, idx):
        return tuple(getattr(self, f)[idx] for f in self.FIELDS)


def raycast(displacement: np.ndarray, normal: np.ndarray, rays: np.ndarray, map_scales: np.ndarray, step: float = 0.5,
            max_samples: int = 1024, tolerance: float = 1e-3, max_iterations: int = 8, trace: bool = False):
    """displacement, normal: [C][N][N][4] float16; rays: RAY [n]; map_scales: [C][4] float32.
    Returns HIT [n], and with trace=True also the TRACE rows of every gap evaluation, ray by ray in evaluation order."""
    rays = np.ascontiguousarray(rays, RAY).reshape(-1)
    sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
    tol, stp = F(tolerance), F(step)
    n = len(rays)
    o, d, t_max = rays["origin"], rays["direction"], rays["t_max"]
    ox, oy, oz = (o[:, c].copy() for c in range(3))
    dx, dy, dz = (d[:, c].copy() for c in range(3))
    out = np.zeros(n, HIT)
    rows = []

    with np.errstate(all="ignore"):
        valid = np.isfinite(o).all(1) & np.isfinite(d).all(1) & (d != 0).any(1) & (t_max >= 0)
        lo, hi, _, _, rho = slab(displacement, sc, tol)
        layers = displacement.astype(np.float32).view(_Widened)
        flat = dy == 0
        ta = (lo - oy) / dy
        tb = (hi - oy) / dy
        tn = np.where(ta < tb, ta, tb)
        tf = np.where(ta < tb, tb, ta)
        t_in = np.where(flat, F(0.0), np.where(tn > 0, tn, F(0.0))).astype(np.float32)
        t_out = np.where(flat, t_max, np.where(tf < t_max, tf, t_max)).astype(np.float32)
        enters = np.where(flat, (lo <= oy) & (oy <= hi), (t_in <= t_out) & np.isfinite(t_in)) & valid
        h = stp / np.sqrt(dx * dx + dz * dz)

        status = np.where(valid, MISS, INVALID).astype(np.uint32)
        evals, iters, unconv = (np.zeros(n, np.uint32) for _ in range(3))
        rep = _Points(n)                       # the reported point
        prev = _Points(n)                      # the previous march sample
        side0 = np.zeros(n, bool)
        k = np.zeros(n, np.int64)
        cur = t_in.copy()

        def evaluate(i, t, base, kind):
            """Gap evaluations of rays i at t; base = None (start at Q) or the warm start's (x, z, source_x, source_z)."""
            x, y, z = ox[i] + t * dx[i], oy[i] + t * dy[i], oz[i] + t * dz[i]
            if base is None or max_iterations == 0:
                sx, sz = x, z
            else:
                sx, sz = base[2] + (x - base[0]), base[3] + (z - base[1])
            px, pz, r, s, g = _gap(layers, sc, tol, max_iterations, rho, x, y, z, sx, sz)
            evals[i] += 1
            iters[i] += s
            unconv[i] += ~(r <= tol)
            if trace:
                tr = np.zeros(i.size, TRACE)
                tr["ray"], tr["kind"], tr["t"] = i, kind, t
                tr["position"] = np.stack([x, y, z], 1)
                tr["source_x"], tr["source_z"], tr["residual"], tr["iterations"], tr["gap"] = px, pz, r, s, g
                rows.append(tr)
            return (t, x, y, z, px, pz, r, g)

        # march
        live = enters.copy()
        while True:
            i = np.nonzero(live)[0]
            if i.size == 0:
                break
            first = k[i] == 0
            t = cur[i]
            warm = np.nonzero(~first)[0]
            e = [np.zeros(i.size, np.float32) for _ in range(8)]
            for sel, base in ((np.nonzero(first)[0], None), (warm, True)):
                if sel.size == 0:
                    continue
                b = None if base is None else (prev.x[i[sel]], prev.z[i[sel]], prev.px[i[sel]], prev.pz[i[sel]])
                for a_, v_ in zip(e, evaluate(i[sel], t[sel], b, 0)):
                    a_[sel] = v_
            g = e[7]
            side = g > 0
            side0[i[first]] = side[first]
            nan = np.isnan(g)
            crossed = ~first & (side != side0[i]) & ~nan
            rest = ~crossed & ~nan
            end = rest & (t == t_out[i])
            trunc = rest & ~end & (evals[i] == max_samples)
            cont = rest & ~end & ~trunc
            kn = k[i] + 1
            tn = t_in[i] + kn.astype(np.float32) * h[i]
            tn = np.where(tn < t_out[i], tn, t_out[i])
            gone = cont & ~np.isfinite(tn)
            cont &= ~gone
            # brackets keep the previous sample as end a; everything else reports this sample
            rep.put(i[~crossed], [v[~crossed] for v in e])
            status[i[nan]] = INVALID
            status[i[trunc]] = TRUNCATED
            live[i[~cont]] = False
            ic = i[crossed]
            if ic.size:
                _refine(ic, prev.take(ic), tuple(v[crossed] for v in e), side0[ic], evaluate, tol, status, rep)
            prev.put(i, e)
            k[i[cont]] = kn[cont]
            cur[i[cont]] = tn[cont]

        # the records
        out["status"] = status
        out["evaluations"], out["iterations"], out["unconverged"] = evals, iters, unconv
        miss0 = valid & ~enters
        out["position"][miss0] = o[miss0]
        ev = np.nonzero(enters)[0]
        if ev.size:
            out["t"][ev] = rep.t[ev]
            out["position"][ev] = np.stack([rep.x[ev], rep.y[ev], rep.z[ev]], 1)
            out["source_x"][ev], out["source_z"][ev] = rep.px[ev], rep.pz[ev]
            out["gap"][ev], out["residual"][ev] = rep.g[ev], rep.r[ev]
            dd, gg = sample_maps(displacement, normal, np.stack([rep.px[ev], rep.pz[ev]], 1), sc)
            out["displacement"][ev], out["gradient_foam"][ev] = dd, gg
    if not trace:
        return out
    tr = np.concatenate(rows) if rows else np.zeros(0, TRACE)
    return out, tr[np.argsort(tr["ray"], kind="stable")]


def _refine(i, a, b, above, evaluate, tol, status, rep):
    """Illinois regula falsi on the brackets [a, b] of rays i (tuples of _Points.FIELDS arrays); writes status and rep."""
    a = [v.copy() for v in a]
    b = [v.copy() for v in b]
    wa, wb = a[7].copy(), b[7].copy()
    last = np.zeros(i.size, np.int8)            # 1: the previous step replaced a, 2: it replaced b
    active = np.ones(i.size, bool)
    done_invalid = np.zeros(i.size, bool)
    for _ in range(MAX_REFINE):
        active &= ~((np.abs(a[7]) <= tol) | (np.abs(b[7]) <= tol))
        j = np.nonzero(active)[0]
        if j.size == 0:
            break
        w = wa[j] / (wa[j] - wb[j])
        t = a[0][j] + w * (b[0][j] - a[0][j])
        inside = (t > a[0][j]) & (t < b[0][j])
        active[j[~inside]] = False
        j, t = j[inside], t[inside]
        if j.size == 0:
            break
        near_a = (t - a[0][j]) <= (b[0][j] - t)
        base = tuple(np.where(near_a, a[f][j], b[f][j]) for f in (1, 3, 4, 5))     # x, z, source_x, source_z
        e = evaluate(i[j], t, base, 1)
        g = e[7]
        nan = np.isnan(g)
        done_invalid[j[nan]] = True
        active[j[nan]] = False
        repl_a = ~nan & ((g > 0) == above[j])
        repl_b = ~nan & ~repl_a
        ja, jb = j[repl_a], j[repl_b]
        wb[ja[last[ja] == 1]] *= F(0.5)
        wa[jb[last[jb] == 2]] *= F(0.5)
        for f in range(8):
            a[f][ja] = e[f][repl_a]
            b[f][jb] = e[f][repl_b]
        wa[ja] = g[repl_a]
        wb[jb] = g[repl_b]
        last[ja] = 1
        last[jb] = 2
        if nan.any():
            rep.put(i[j[nan]], [v[nan] for v in e])
    ok = ~done_invalid
    take_a = np.abs(a[7]) <= np.abs(b[7])
    best = [np.where(take_a, a[f], b[f]) for f in range(8)]
    rep.put(i[ok], [v[ok] for v in best])
    status[i[ok]] = np.where(above[ok], HIT_FROM_ABOVE, HIT_FROM_BELOW)
    status[i[done_invalid]] = INVALID
