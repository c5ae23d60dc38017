"""Specification of the wake coupling (include/ocean.h, "Wake layer", ocean_wake_set_coupling): the surface query, buoyancy,
body forces and the floating-body integrator reading the wake layer of oracle/wake.py on top of the FFT maps.
csrc/ocean_wake.cu (k_wake_free_surface, k_wake_couple) and csrc/ocean_buoyancy.cu (k_drag_reduce_wake) match it bit for bit.

TEST INFRASTRUCTURE ONLY -- the product path (godotoceanwaves_b200/csrc) never imports or calls this module.

What the physics reads is the wake FREE SURFACE e = h + phi_end, not h: the iWave stencil acts on s = h + phi, which is
exactly 0 at rest under a stationary source (h = -phi there), so a body that carries a source does not feel the depression
its own pressure head presses into the layer (that depression is the hull), while waves from other sources and the body's
own radiated waves pass through e unchanged.

  free surface  after a step call of S sub-steps of h_sub = dt / S:  e = h + rasterise(sources at tau_end), tau_end = (float)S
                * h_sub (the sub-step time one past the last sub-step; body-attached sources at position.xz +
                linear_velocity.xz * tau_end of the states the call was given)
  Coupling      (e, origin_e, e_old, origin_old, T, primed): the snapshot of the last coupled call, the one before it, each in
                the window of its own call, and T = tau_end of the last call.  A priming call (the first after the coupling
                is enabled or the layer's state is set) writes e into both snapshots, so that wv = 0.  Before it both are 0,
                the origins (0, 0) and T = 0, and the ops read nothing of the wake.
  couple        per query point Q, after the inversion: (we, gx, gz) = wake.sample(e, cell, origin_e, Q);
                displacement[1] += we, gradient_foam[0] += gx, gradient_foam[1] += gz.  The wake has no horizontal
                displacement, so the inversion and every other field are unchanged.
  buoyancy, body forces, simulate   the same on the world hull points Q = (w.x, w.z); the submerged fractions read the coupled
                height.  Drag adds the wake's vertical water velocity to u.y before d = u - vb:
                  wv = (sample(e, origin_e, Q)[0] - sample(e_old, origin_old, Q)[0]) / T
                each snapshot sampled in its own window (0 outside).  Every sub-step of a simulate call reads the same e and
                e_old, as it reads the same maps.

Numeric policy as oracle/wake.py and oracle/drag.py: binary32 in the order written, no contraction, IEEE division.
"""
from __future__ import annotations

import numpy as np

from . import bodies as bo
from . import buoyancy as bu
from . import drag as dr
from . import surface as su
from . import wake as wk
from .sampling import F

f32 = np.float32


class Coupling:
    """The coupling state of one layer: the snapshots e, e_old ([N][N] float32) with their origins (cells), T and primed."""

    def __init__(self, n: int, cell_size):
        self.cell_size = f32(cell_size)
        self.n = int(n)
        self.reset()

    def reset(self):
        """Unprimed: both snapshots 0 at origin (0, 0) and T = 0 (ocean_wake_set_coupling, ocean_wake_set_state)."""
        self.e = np.zeros((self.n, self.n), np.float32)
        self.e_old = np.zeros((self.n, self.n), np.float32)
        self.origin_e = (0, 0)
        self.origin_old = (0, 0)
        self.T = f32(0.0)
        self.primed = False
        return self


def free_surface(layer: wk.Layer, sources, states, dt, substeps) -> np.ndarray:
    """e = h + phi of the sources at tau_end = (float)S * h_sub, in the layer's current window, after a step call."""
    h = wk.substep(dt, substeps)
    tau = f32(int(substeps)) * h
    src = np.zeros(0, wk.SOURCE) if sources is None else np.asarray(sources, wk.SOURCE).reshape(-1)
    phi = wk.rasterise(layer.n, layer.cell_size, layer.origin, src, states, tau) if len(src) else np.zeros_like(layer.h)
    with np.errstate(all="ignore"):
        return layer.h + phi


def step(layer: wk.Layer, coupling: Coupling | None, dt, substeps, origin, sources=None, states=None) -> wk.Layer:
    """One step call of a layer whose coupling is `coupling` (None: off): Layer.step, then the free surface into the snapshots."""
    layer.step(dt, substeps, origin, sources, states)
    if coupling is None:
        return layer
    e = free_surface(layer, sources, states, dt, substeps)
    if coupling.primed:
        coupling.e_old, coupling.origin_old = coupling.e, coupling.origin_e
    else:
        coupling.e_old, coupling.origin_old = e.copy(), layer.origin
    coupling.e, coupling.origin_e = e, layer.origin
    coupling.T = f32(int(substeps)) * wk.substep(dt, substeps)
    coupling.primed = True
    return layer


def live(coupling: Coupling | None) -> bool:
    return coupling is not None and coupling.primed


def couple(records: np.ndarray, Q, coupling: Coupling, cell) -> np.ndarray:
    """Surface records (surface.RECORD [n]) with the wake free surface e at the query points Q [n][2] added."""
    out = np.array(records, su.RECORD, copy=True).reshape(-1)
    s = wk.sample(coupling.e, cell, coupling.origin_e, Q)
    with np.errstate(all="ignore"):
        out["displacement"][:, 1] = out["displacement"][:, 1] + s[:, 0]
        out["gradient_foam"][:, 0] = out["gradient_foam"][:, 0] + s[:, 1]
        out["gradient_foam"][:, 1] = out["gradient_foam"][:, 1] + s[:, 2]
    return out


def vertical_velocity(Q, coupling: Coupling, cell) -> np.ndarray:
    """wv [n] float32: (sample(e, origin_e, Q)[0] - sample(e_old, origin_old, Q)[0]) / T."""
    a = wk.sample(coupling.e, cell, coupling.origin_e, Q)[:, 0]
    b = wk.sample(coupling.e_old, cell, coupling.origin_old, Q)[:, 0]
    with np.errstate(all="ignore"):
        return (a - b) / f32(coupling.T)


def query_surface(displacement, normal, points_xz, map_scales, tolerance=1e-3, max_iterations=8, wake: Coupling | None = None):
    """surface.query_surface, coupled to the wake while `wake` is primed."""
    rec = su.query_surface(displacement, normal, points_xz, map_scales, tolerance, max_iterations)
    if not live(wake):
        return rec
    return couple(rec, np.asarray(points_xz, np.float32).reshape(-1, 2), wake, wake.cell_size)


def buoyancy(displacement, normal, bodies, points, map_scales, density=1025.0, tolerance=1e-3, max_iterations=8, return_samples=False,
             wake: Coupling | None = None):
    """buoyancy.buoyancy, its surface records coupled to the wake while `wake` is primed."""
    if not live(wake):
        return bu.buoyancy(displacement, normal, bodies, points, map_scales, density, tolerance, max_iterations, return_samples)
    bodies = np.ascontiguousarray(bodies, bu.BODY)
    points = np.ascontiguousarray(points, bu.POINT)
    B = len(bodies)
    body, j, r, w = bu.world_points(bodies, points)
    Q = np.stack([w[:, 0], w[:, 2]], 1)
    samples = query_surface(displacement, normal, Q, map_scales, tolerance, max_iterations, wake) if len(body) \
        else np.zeros(0, su.RECORD)
    # from here on buoyancy.buoyancy's lines, on the coupled records
    p = points[bodies["first_point"].astype(np.int64)[body] + j]
    f = bu.submerged_fraction(samples["displacement"][:, 1], w[:, 1], p["half_height"].astype(np.float32))
    with np.errstate(all="ignore"):
        v = f * p["volume"].astype(np.float32)
        terms = np.stack([v, v * r[:, 0], v * r[:, 1], v * r[:, 2]], 1)
    S = bu.lane_tree_sum(terms, body, j, B)
    S0, S1 = S[:, 0], S[:, 1:]
    rho_g = F(density) * bu.G
    out = np.zeros(B, bu.RESULT)
    with np.errstate(all="ignore"):
        out["submerged_volume"] = S0
        out["force"][:, 1] = rho_g * S0
        out["torque"][:, 0] = -(rho_g * S1[:, 2])
        out["torque"][:, 2] = rho_g * S1[:, 0]
        pos = S0 > F(0.0)
        out["center_offset"][pos] = S1[pos] / S0[pos, None]
    max_res = np.full(B, np.nan, np.float32)
    np.fmax.at(max_res, body, samples["residual"])
    out["max_residual"] = max_res
    missed = (~(samples["residual"] <= F(tolerance))).astype(np.float64)
    out["unconverged"] = np.bincount(body, weights=missed, minlength=B).astype(np.uint32)
    out[bodies["num_points"] == 0] = np.zeros(1, bu.RESULT)
    return (out, samples) if return_samples else out


def body_forces(displacement, normal, velocity, bodies, velocities, points, drag_areas, map_scales, density=1025.0, tolerance=1e-3,
                max_iterations=8, return_samples=False, wake: Coupling | None = None):
    """drag.body_forces, coupled to the wake while `wake` is primed: the coupled buoyancy records, and u.y + wv in the drag."""
    if not live(wake):
        return dr.body_forces(displacement, normal, velocity, bodies, velocities, points, drag_areas, map_scales, density, tolerance,
                              max_iterations, return_samples)
    bodies = np.ascontiguousarray(bodies, bu.BODY)
    points = np.ascontiguousarray(points, bu.POINT)
    velocities = np.ascontiguousarray(velocities, dr.VELOCITY)
    drag_areas = np.ascontiguousarray(drag_areas, np.float32)
    B = len(bodies)
    hydro, samples = buoyancy(displacement, normal, bodies, points, map_scales, density, tolerance, max_iterations, True, wake)
    body, j, r, w = bu.world_points(bodies, points)
    wv = vertical_velocity(np.stack([w[:, 0], w[:, 2]], 1), wake, wake.cell_size)
    # from here on drag.body_forces' lines, with wv added to u.y
    k_point = bodies["first_point"].astype(np.int64)[body] + j
    f = bu.submerged_fraction(samples["displacement"][:, 1], w[:, 1], points["half_height"][k_point].astype(np.float32))
    wet = f > F(0.0)
    body, j, r, f, k_point, wv = body[wet], j[wet], r[wet], f[wet], k_point[wet], wv[wet]
    src = np.stack([samples["source_x"][wet], samples["source_z"][wet]], 1)
    u = dr.water_velocity(velocity, src, map_scales)
    vel = velocities[body]
    with np.errstate(all="ignore"):
        u[:, 1] = u[:, 1] + wv
        vb = vel["linear"] + dr.cross(vel["angular"], r)
        d = u - vb
        s = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        a = f * drag_areas[k_point]
        k = a * s
        Fp = k[:, None] * d
        Tp = dr.cross(r, Fp)
    S = bu.lane_tree_sum(np.concatenate([Fp, Tp, a[:, None]], 1), body, j, B) if len(body) else np.zeros((B, 7), np.float32)
    half_rho = F(0.5) * F(density)
    out = np.zeros(B, dr.RESULT)
    with np.errstate(all="ignore"):
        out["force"] = half_rho * S[:, 0:3]
        out["torque"] = half_rho * S[:, 3:6]
    out["wetted_drag_area"] = S[:, 6]
    max_s = np.zeros(B, np.float32)
    np.fmax.at(max_s, body, s)
    out["max_relative_speed"] = max_s
    out[bodies["num_points"] == 0] = np.zeros(1, dr.RESULT)
    return (hydro, out, samples) if return_samples else (hydro, out)


def simulate(displacement, normal, velocity, bodies, states, points, drag_areas, map_scales, density=1025.0, dt=1.0 / 60.0, substeps=1,
             tolerance=1e-3, max_iterations=8, wake: Coupling | None = None):
    """bodies.simulate, every sub-step's forces those of body_forces coupled to the same wake snapshots."""
    if not live(wake):
        return bo.simulate(displacement, normal, velocity, bodies, states, points, drag_areas, map_scales, density, dt, substeps, tolerance,
                           max_iterations)
    bodies = np.ascontiguousarray(bodies, bo.BODY)
    s = np.array(states, bo.STATE, copy=True)
    h = F(dt) / F(substeps)
    r2 = bo.radius2(bodies, points)
    hyd, drg = np.zeros(len(bodies), bu.RESULT), np.zeros(len(bodies), dr.RESULT)
    world = int(bodies["num_points"].astype(np.int64).sum())
    for _ in range(substeps):
        table, vel = bo.pose(bodies, s)
        if world:
            with np.errstate(all="ignore"):
                hyd, drg = body_forces(displacement, normal, velocity, table, vel, points, drag_areas, map_scales, density, tolerance,
                                       max_iterations, wake=wake)
        s = bo.step(bodies, s, r2, hyd, drg, density, h)
    return s, hyd, drg, bo.transforms(s)
