"""Specification of the wake readers (include/ocean.h, "Wake layer", Readers; ocean_wake_set_readers): the ray cast and spray
reading the wake layer of oracle/wake.py.  csrc/ocean_sample.cu (k_raycast<true>, k_raycast_wake_bound) and
csrc/ocean_spray.cu (the <true> forms of k_spray_count, k_spray_write and k_spray_particles_update) match it bit for bit.

TEST INFRASTRUCTURE ONLY -- the product path (godotoceanwaves_b200/csrc) never imports or calls this module.

It composes oracle/raycast.py, oracle/spray.py and oracle/spray_particles.py and changes none of them: the march, the spawn
test and the particle process are restated here with the wake's additions, on those modules' helpers (the inversion, the
refinement, the restarts, start()), and with no wake they give those modules' bytes (tests/test_oracle_wake_readers.py).

  raycast   OCEAN_WAKE_READ_RAYCAST, while the coupling is live (oracle/wake_coupling.py live(): on and primed); otherwise
            raycast.raycast as it is.  The surface is the coupled one of wake_coupling.query_surface, the free surface e in
            its own window (origin_e):
              bounds   e_min = -fmax over the cells of -e, e_max = fmax over the cells of e (NaN-dropping, from -inf)
              slab     after the cascades:  y_lo = y_lo + fmin(e_min, 0),  y_hi = y_hi + fmax(e_max, 0),
                       acc = acc + fmax(|e_min|, |e_max|)   (the sample is 0 outside the window, and the bilinear sample
                       of e lies in [min(e_min, 0), max(e_max, 0)] up to the rounding acc * 2^-13 covers)
              gap      at each evaluation of raycast.py, after its eta:  we = wake.sample(e, cell, origin_e, Q)[0] at
                       Q = (x, z) of the evaluated point;  g = y - (eta + we)  (one binary32 add, then the subtraction).
                       The wake has no horizontal displacement: the inversion, warm starts, restarts, march and
                       refinement are unchanged; the trace rows carry this g.
              record   at the reported point, wake_coupling.couple's additions at Q = (position.x, position.z):
                       displacement[1] += we, gradient_foam[0] += gx, gradient_foam[1] += gz; gap == position.y -
                       displacement[1] as without the wake.
  spray     OCEAN_WAKE_READ_SPRAY, whenever a layer exists (no coupling needed).  With S = START_POS.xz,
            (hw, hgx, hgz) = wake.sample(h, cell, origin, S) of the layer's current h and window, and Fw = its sample of
            F (+0 while foam is off):
              spawn    spray.spray_candidates and spray_particles' spawn test, right after the cascade sum and before the
                       normalize:  gx = gx + hgx,  gy = gy + hgz,  gf = gf + Fw;  everything after is unchanged, and the
                       record's foam is the sum.
              height   spray_particles' process, right after the cascade displacement sum:  dy = dy + hw  (every frame).

Numeric policy as oracle/wake.py: binary32 in the order written, no contraction, IEEE division.
"""
from __future__ import annotations

import numpy as np

from . import raycast as rc
from . import spray as sp
from . import spray_particles as spp
from . import wake as wk
from . import wake_coupling as wc
from .sampling import F, _mix, sample_maps, texture_bilinear

f32 = np.float32


def sample(f: np.ndarray, cell_size, origin, x, z, gradients: bool = True) -> np.ndarray:
    """wake.sample(f, cell_size, origin, (x, z)) vectorised: [n][3] float32 (value, d/dx, d/dz), byte-identical (the same
    binary32 operations per point, cells outside the window reading 0 through one ring of zero padding)."""
    n = f.shape[0]
    dx = f32(cell_size)
    x0, z0 = wk.world_origin(origin, dx)
    x = np.asarray(x, np.float32).reshape(-1)
    z = np.asarray(z, np.float32).reshape(-1)
    out = np.zeros((len(x), 3), np.float32)
    with np.errstate(all="ignore"):
        inside = (x >= x0) & (x < x0 + f32(n) * dx) & (z >= z0) & (z < z0 + f32(n) * dx)
        k = np.flatnonzero(inside)
        if k.size == 0:
            return out
        u = (x[k] - x0) / dx - f32(0.5)
        v = (z[k] - z0) / dx - f32(0.5)
        fi, fj = np.floor(u), np.floor(v)
        fu, fv = u - fi, v - fj
        i, j = fi.astype(np.int64) + 1, fj.astype(np.int64) + 1          # indices into the padded fields
        fields = (f,) + (wk.gradients(f, dx) if gradients else ())
        for m, g in enumerate(fields):
            p = np.zeros((n + 2, n + 2), np.float32)
            p[1:-1, 1:-1] = g
            f00, f10, f01, f11 = p[j, i], p[j, i + 1], p[j + 1, i], p[j + 1, i + 1]
            top = f00 + fu * (f10 - f00)
            bot = f01 + fu * (f11 - f01)
            out[k, m] = top + fv * (bot - top)
    return out


def bounds(e: np.ndarray):
    """(e_min, e_max) float32: NaN-dropping extrema of e, as the device's fmaxf reductions from -inf."""
    t = np.asarray(e, np.float32).reshape(-1)
    ninf = f32(-np.inf)
    with np.errstate(invalid="ignore"):
        return f32(-np.fmax.reduce(-t, initial=ninf)), f32(np.fmax.reduce(t, initial=ninf))


class RaySurface:
    """The wake surface the ray cast reads: the coupling's e in its window."""

    def __init__(self, coupling: wc.Coupling):
        self.e = coupling.e
        self.origin = coupling.origin_e
        self.cell = coupling.cell_size
        self.bounds = bounds(self.e)

    def height(self, x, z) -> np.ndarray:
        return sample(self.e, self.cell, self.origin, x, z, gradients=False)[:, 0]

    def sample(self, x, z) -> np.ndarray:
        return sample(self.e, self.cell, self.origin, x, z)


class SprayLayer:
    """The wake layer spray reads: h and F (None while foam is off) in the current window."""

    def __init__(self, layer: wk.Layer, foam_on: bool = False):
        self.h = layer.h
        self.foam = layer.foam if foam_on else None
        self.origin = layer.origin
        self.cell = layer.cell_size

    def spray(self, x, z):
        """(hw, hgx, hgz, Fw) float32 [n] each at the points (x, z)."""
        s = sample(self.h, self.cell, self.origin, x, z)
        fw = np.zeros(len(s), np.float32) if self.foam is None else sample(self.foam, self.cell, self.origin, x, z, False)[:, 0]
        return s[:, 0], s[:, 1], s[:, 2], fw


# ---- the ray cast ----

def slab(displacement, map_scales, tolerance, wake_bounds=None):
    """raycast.slab, widened after the cascades by wake_bounds = (e_min, e_max) when given:
    y_lo += fmin(e_min, 0), y_hi += fmax(e_max, 0), acc += fmax(|e_min|, |e_max|).  Returns (lo, hi, rho)."""
    sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
    ymin, ymax, m = rc.layer_bounds(displacement)
    y_lo = y_hi = acc = rho = F(0.0)
    with np.errstate(all="ignore"):
        for i in range(displacement.shape[0]):
            s = sc[i, 2]
            a, b = s * ymin[i], s * ymax[i]
            y_lo = y_lo + np.fmin(a, b)
            y_hi = y_hi + np.fmax(a, b)
            acc = acc + np.abs(s) * np.fmax(np.abs(ymin[i]), np.abs(ymax[i]))
            rho = rho + np.abs(s) * m[i]
        if wake_bounds is not None:
            e_min, e_max = F(wake_bounds[0]), F(wake_bounds[1])
            y_lo = y_lo + np.fmin(e_min, F(0.0))
            y_hi = y_hi + np.fmax(e_max, F(0.0))
            acc = acc + np.fmax(np.abs(e_min), np.abs(e_max))
        rho = rho * F(0.5)
        pad = F(tolerance) + acc * rc.PAD_SCALE
        return F(y_lo - pad), F(y_hi + pad), F(rho)


def _gap(layers, sc, tol, max_iterations, rho, x, y, z, sx, sz, wake):
    """raycast._gap's inversion and restarts, the gap taken to eta + we (we = wake.height(x, z)); no wake: raycast._gap."""
    px, pz, r, steps, g = rc._gap(layers, sc, tol, max_iterations, rho, x, y, z, sx, sz)
    if wake is None:
        return px, pz, r, steps, g
    with np.errstate(all="ignore"):
        eta = rc._height(layers, sc, px, pz) + wake.height(x, z)
        return px, pz, r, steps, np.asarray(y - eta)


def _raycast(displacement, normal, rays, map_scales, step, max_samples, tolerance, max_iterations, trace, wake):
    """raycast.raycast's clip, march and records, with the wake surface `wake` (RaySurface or None) in the slab, every gap
    and the record.  The march is raycast.raycast's, line for line; the refinement is raycast._refine itself."""
    rays = np.ascontiguousarray(rays, rc.RAY).reshape(-1)
    sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
    tol, stp = F(tolerance), F(step)
    n = len(rays)
    o, d, t_max = rays["origin"], rays["direction"], rays["t_max"]
    ox, oy, oz = (o[:, c].copy() for c in range(3))
    dx, dy, dz = (d[:, c].copy() for c in range(3))
    out = np.zeros(n, rc.HIT)
    rows = []

    with np.errstate(all="ignore"):
        valid = np.isfinite(o).all(1) & np.isfinite(d).all(1) & (d != 0).any(1) & (t_max >= 0)
        lo, hi, rho = slab(displacement, sc, tol, None if wake is None else wake.bounds)
        layers = displacement.astype(np.float32).view(rc._Widened)
        flat = dy == 0
        ta = (lo - oy) / dy
        tb = (hi - oy) / dy
        tn = np.where(ta < tb, ta, tb)
        tf = np.where(ta < tb, tb, ta)
        t_in = np.where(flat, F(0.0), np.where(tn > 0, tn, F(0.0))).astype(np.float32)
        t_out = np.where(flat, t_max, np.where(tf < t_max, tf, t_max)).astype(np.float32)
        enters = np.where(flat, (lo <= oy) & (oy <= hi), (t_in <= t_out) & np.isfinite(t_in)) & valid
        h = stp / np.sqrt(dx * dx + dz * dz)

        status = np.where(valid, rc.MISS, rc.INVALID).astype(np.uint32)
        evals, iters, unconv = (np.zeros(n, np.uint32) for _ in range(3))
        rep = rc._Points(n)
        prev = rc._Points(n)
        side0 = np.zeros(n, bool)
        k = np.zeros(n, np.int64)
        cur = t_in.copy()

        def evaluate(i, t, base, kind):
            x, y, z = ox[i] + t * dx[i], oy[i] + t * dy[i], oz[i] + t * dz[i]
            if base is None or max_iterations == 0:
                sx, sz = x, z
            else:
                sx, sz = base[2] + (x - base[0]), base[3] + (z - base[1])
            px, pz, r, s, g = _gap(layers, sc, tol, max_iterations, rho, x, y, z, sx, sz, wake)
            evals[i] += 1
            iters[i] += s
            unconv[i] += ~(r <= tol)
            if trace:
                tr = np.zeros(i.size, rc.TRACE)
                tr["ray"], tr["kind"], tr["t"] = i, kind, t
                tr["position"] = np.stack([x, y, z], 1)
                tr["source_x"], tr["source_z"], tr["residual"], tr["iterations"], tr["gap"] = px, pz, r, s, g
                rows.append(tr)
            return (t, x, y, z, px, pz, r, g)

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
            rep.put(i[~crossed], [v[~crossed] for v in e])
            status[i[nan]] = rc.INVALID
            status[i[trunc]] = rc.TRUNCATED
            live[i[~cont]] = False
            ic = i[crossed]
            if ic.size:
                rc._refine(ic, prev.take(ic), tuple(v[crossed] for v in e), side0[ic], evaluate, tol, status, rep)
            prev.put(i, e)
            k[i[cont]] = kn[cont]
            cur[i[cont]] = tn[cont]

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
            if wake is not None:
                w = wake.sample(rep.x[ev], rep.z[ev])
                dd[:, 1] = dd[:, 1] + w[:, 0]
                gg[:, 0] = gg[:, 0] + w[:, 1]
                gg[:, 1] = gg[:, 1] + w[:, 2]
            out["displacement"][ev], out["gradient_foam"][ev] = dd, gg
    if not trace:
        return out
    tr = np.concatenate(rows) if rows else np.zeros(0, rc.TRACE)
    return out, tr[np.argsort(tr["ray"], kind="stable")]


def raycast(displacement, normal, rays, map_scales, step=0.5, max_samples=1024, tolerance=1e-3, max_iterations=8, trace=False,
            coupling: wc.Coupling | None = None, read: bool = True):
    """The ray cast with OCEAN_WAKE_READ_RAYCAST `read`: on the coupled surface while the coupling is live, otherwise
    raycast.raycast itself.  With trace=True also the TRACE rows, whose gap is the coupled one."""
    if not (read and wc.live(coupling)):
        return rc.raycast(displacement, normal, rays, map_scales, step, max_samples, tolerance, max_iterations, trace)
    return _raycast(displacement, normal, rays, map_scales, step, max_samples, tolerance, max_iterations, trace, RaySurface(coupling))


# ---- spray ----

def _spawn_gradient(normal, sx, sz, scales, wake):
    """The spawn test's gradient [n][3] (x, y, foam): the cascade sum of spray.py, then + (hgx, hgz, Fw) of `wake`."""
    grad = np.zeros((len(sx), 3), np.float32)
    for i in range(len(scales)):
        t = texture_bilinear(normal[i], sx * scales[i, 0], sz * scales[i, 1])             # :83
        grad = grad + t[:, [0, 1, 3]]
    if wake is not None:
        _, hgx, hgz, fw = wake.spray(sx, sz)
        with np.errstate(all="ignore"):
            grad = grad + np.stack([hgx, hgz, fw], axis=1)
    return grad


def _factors(grad):
    """(normal_factor, foam_factor, foam, active) of spray.py from the gradient; min is fmin (minNum), as the device's fminf
    and spray_particles.py (spray.py's np.minimum differs only for a NaN gradient, which finite maps do not give)."""
    gx, gy, foam = -grad[:, 0], -grad[:, 1], grad[:, 2]
    with np.errstate(invalid="ignore", over="ignore"):
        ny = F(1.0) / np.sqrt((gx * gx + F(1.0) * F(1.0)) + gy * gy)                            # :84
        nf = _mix(F(0.25), F(1.0), np.fmin((ny - F(0.92)) / (F(0.99) - F(0.92)), F(1.0)))       # :86
        ff = _mix(F(0.25), F(1.0), np.fmin((foam - F(0.9)) / (F(1.0) - F(0.9)), F(1.0)))        # :87
        active = (nf >= F(0.0)) & (nf <= F(1.0)) & (foam > F(0.9))                              # :89
    return nf, ff, foam, active


def _spray_candidates(normal, points_xz, map_scales, particle_scale, wake):
    """spray.spray_candidates with the wake (SprayLayer or None) in the spawn test."""
    pts = np.ascontiguousarray(points_xz, np.float32)
    sc = np.ascontiguousarray(map_scales, np.float32)
    ps = np.asarray(particle_scale, np.float32)
    nf, ff, foam, active = _factors(_spawn_gradient(normal, pts[:, 0], pts[:, 1], sc, wake))
    s = ff * (F(1.0) + F(1e-3))                                                                  # :92 (ACTIVE == true)
    out = np.zeros(int(active.sum()), sp.RECORD)
    k = np.nonzero(active)[0]
    out["index"] = k.astype(np.uint32)
    out["start_x"], out["start_z"] = pts[k, 0], pts[k, 1]
    out["scale_factor"] = (nf * ff)[k]                                                           # :90
    out["particle_scale"][:, 0] = ((s * F(1.0)) * ps[0])[k]                                      # :93-94
    out["particle_scale"][:, 1] = ((s * nf) * ps[1])[k]
    out["particle_scale"][:, 2] = ((s * F(1.0)) * ps[2])[k]
    out["foam"] = foam[k]
    return out


def spray_candidates(normal, points_xz, map_scales, particle_scale, layer: wk.Layer | None = None, foam_on: bool = False):
    """ocean_extract_spray with OCEAN_WAKE_READ_SPRAY: reading `layer` (None: no layer or the bit clear, spray.py itself)."""
    if layer is None:
        return sp.spray_candidates(normal, points_xz, map_scales, particle_scale)
    return _spray_candidates(normal, points_xz, map_scales, particle_scale, SprayLayer(layer, foam_on))


def _process(p, idx, e, TIME, displacement, normal, scales, wake):
    """spray_particles._process for the ACTIVE particles idx, with the wake (None: none) in the spawn test and hw added
    to d.y."""
    T32 = F(TIME)
    st, pl = p["userdata1"][idx, 3], p["userdata2"][idx, 3]
    over = T32 > st + pl
    p["flags"][idx[over]] &= ~spp.U32(spp.ACTIVE)
    now = idx[~over & (T32 >= st)]
    first = now[p["userdata3"][now, 3] == F(0.0)]
    if len(first):
        nf, ff, _, active = _factors(_spawn_gradient(normal, p["userdata1"][first, 0], p["userdata1"][first, 2], scales, wake))
        s = ff * (active.astype(np.float32) + F(1e-3))
        ps = np.asarray(e["particle_scale"], np.float32)
        p["flags"][first] = np.where(active, p["flags"][first] | spp.U32(spp.ACTIVE), p["flags"][first] & ~spp.U32(spp.ACTIVE))
        p["userdata3"][first, 2] = nf * ff
        p["userdata2"][first, :3] = np.stack([(s * F(1.0)) * ps[0], (s * nf) * ps[1], (s * F(1.0)) * ps[2]], axis=1)
        p["userdata3"][first, 3] = F(1.0)
    on = now[(p["flags"][now] & spp.U32(spp.ACTIVE)) != 0]
    if not len(on):
        return
    st, pl = p["userdata1"][on, 3], p["userdata2"][on, 3]
    t = (T32 - st) / pl
    p["custom"][on, 3] = spp._exp_impulse(t, 10.0)
    sx, sz = p["userdata1"][on, 0], p["userdata1"][on, 2]
    d = np.zeros((len(on), 3), np.float32)
    for i in range(len(scales)):
        tex = texture_bilinear(displacement[i], sx * scales[i, 0], sz * scales[i, 1])
        d = d + tex[:, :3] * scales[i, 2]
    if wake is not None:
        d[:, 1] = d[:, 1] + wake.spray(sx, sz)[0]
    d = d * np.array([0.75, 1.0, 0.75], np.float32)
    a = F(2.5) * t - F(0.45)
    d[:, 0] = d[:, 0] + F(0.0)
    d[:, 1] = d[:, 1] + ((F(-5.0) * (a * a)) * p["userdata3"][on, 2] + F(0.5))
    d[:, 2] = d[:, 2] + F(0.0)
    T = p["transform"][on]
    T[:, 3], T[:, 7], T[:, 11] = sx + d[:, 0], p["userdata1"][on, 1] + d[:, 1], sz + d[:, 2]
    size = pl / F(e["lifetime"])
    m = np.repeat((size * size)[:, None], 3, axis=1)
    m[:, 1] = m[:, 1] * spp._exp_impulse(t, 3.0)
    lg = spp._log(F(1.0) + t)
    m[:, 0] = m[:, 0] * lg
    m[:, 2] = m[:, 2] * lg
    spp._set_scale(T, p["userdata2"][on, :3] * m)
    p["transform"][on] = T


def _frame(states, emitter, t0, t1, displacement, normal, map_scales, max_instances, wake):
    """spray_particles.frame with _process above (the restart and start() are spray_particles' own)."""
    e = np.asarray(emitter, spp.EMITTER).reshape(())
    amount = int(e["amount"])
    p = np.array(states, spp.PARTICLE, copy=True).reshape(-1)
    assert len(p) == amount
    scales = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
    TIME = np.float32(t1)
    with np.errstate(all="ignore"):
        k = spp.restart_cycles(amount, float(e["emitter_lifetime"]), t0, t1)
        idx = np.nonzero(k >= 0)[0]
        if len(idx):
            number = ((k[idx].astype(np.uint64) * np.uint64(amount) + idx.astype(np.uint64)) & np.uint64(0xFFFFFFFF)).astype(spp.U32)
            p["transform"][idx] = np.eye(3, 4, dtype=np.float32).reshape(12)
            p["custom"][idx] = 0.0
            p["number"][idx] = number
            p["flags"][idx] |= spp.U32(spp.ACTIVE | spp.EMITTED)
            spp._start(p, idx, number, e, TIME)
        act = np.nonzero((p["flags"] & spp.U32(spp.ACTIVE)) != 0)[0]
        if len(act):
            _process(p, act, e, TIME, displacement, normal, scales, wake)
    live = ((p["flags"] & spp.U32(spp.ACTIVE)) != 0) & (p["userdata3"][:, 3] != F(0.0))
    count = int(live.sum())
    inst = np.concatenate([p["transform"][live], p["custom"][live]], axis=1).astype(np.float32)
    if max_instances is not None:
        inst = inst[:max_instances]
    return p, np.ascontiguousarray(inst), count


def frame(states, emitter, t0, t1, displacement, normal, map_scales, max_instances=None, layer: wk.Layer | None = None,
          foam_on: bool = False, wake=None):
    """ocean_spray_particles with OCEAN_WAKE_READ_SPRAY: reading `layer` (None: no layer or the bit clear,
    spray_particles.frame itself).  `wake` may replace SprayLayer(layer, foam_on) by any object with its spray(x, z)."""
    if wake is None and layer is not None:
        wake = SprayLayer(layer, foam_on)
    if wake is None:
        return spp.frame(states, emitter, t0, t1, displacement, normal, map_scales, max_instances)
    return _frame(states, emitter, t0, t1, displacement, normal, map_scales, max_instances, wake)
