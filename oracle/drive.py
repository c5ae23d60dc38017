"""CPU specification of the driven floating-body integrator (ocean_simulate_driven_bodies): oracle/bodies.py's sub-steps with
thrusters, hull foils, applied loads and tethers.  It composes bodies.py, buoyancy.py, drag.py (and wake_coupling.py while the
wake coupling is live) and changes none of them.

TEST INFRASTRUCTURE ONLY -- the product path (godotoceanwaves_b200/csrc) never imports or calls this module.

Inputs: those of bodies.simulate, plus THRUSTER [T], FOIL [F], LOAD [B] or None and TETHER [K] rows (include/ocean.h).  Per
sub-step, with R, t the pose ([R | t], bodies.pose) and v, w the velocity (linear, angular) the sub-step starts from, r = R p
for a hull-local point p (buoyancy.world_points' rotation), cross() and the point velocity vb = v + w x r as in drag.py:

  actuators  the thrusters, then the foils, are world points world + k of the sub-step's surface query (after the hull's; each
             query point's record depends only on its own position, so they are queried here on their own), with
             rec their records and f = buoyancy.submerged_fraction(rec.displacement.y, r.y + t.y, half_height).  An actuator
             with !(f > 0) is dry: it adds nothing.
  thruster   n = R direction;  g = f * thrust;  F = g * n;  T = r x F
  foil       n = R normal;  u = drag.water_velocity at (rec.source_x, rec.source_z) (u.y + wv while the coupling is live);
             d = u - vb;  dn = (d.x*n.x + d.y*n.y) + d.z*n.z;  a = f * area;  g = ((half_rho * a) * dn) * |dn|;  F = g * n;
             T = r x F
  tether     x_a = r_a + t_a, v_a = vb_a(r_a); x_b = r_b + t_b, v_b = vb_b(r_b), or x_b = point_b, r_b = v_b = 0 at an anchor
             (body_b = -1);  e = x_b - x_a;  L = sqrt((e.x*e.x + e.y*e.y) + e.z*e.z);  u = e / L;  dv = v_b - v_a;
             s = stiffness * (L - rest_length) + damping * ((dv.x*u.x + dv.y*u.y) + dv.z*u.z);
             tension = s if L > 0 and s > 0 else 0 (a slack tether adds nothing);  F_a = tension * u, T_a = r_a x F_a,
             F_b = -F_a, T_b = r_b x F_b
  sums       per body, from F = hyd.force + drg.force, tau = hyd.torque + drg.torque and D = DT = 0: its incidence list --
             its thrusters, then its foils, then its tether ends, each in array order -- adds each acting term in turn
             (F = F + F_e, tau = tau + T_e, D = D + F_e, DT = DT + T_e), then the load row (when loads are given) the same way.
             Over its foils: sa = sum a (wet ones, in order, from 0), max_dn = max(0, |dn| of the wet ones) (np.fmax),
             rf2 = max(0, |p|^2 of all of them), |p|^2 = (p.x*p.x + p.y*p.y) + p.z*p.z.  Over its taut tether ends, with p
             that end's hull-local point, hc = h * damping and hk = (h*h) * stiffness: tv = sum (hc + hk), tw = sum
             (hc*|p|^2 + hk*|p|^2), in order from 0.
  step       c_v = (density * drg.wetted_drag_area) * drg.max_relative_speed; c_w = c_v * r2 (bodies.py);
             with foils:  c_f = (density * sa) * max_dn;  c_v = c_v + c_f;  c_w = c_w + c_f * rf2
             den_v = mass + h*c_v;  den_w.k = inertia.k + h*c_w;  with a taut tether end: den_v = den_v + tv, den_w.k = den_w.k + tw
             then bodies.step's lines from F.y = F.y - mass * G on, with h / den_v and (h*tau_b.k) / den_w.k as the factors.

The drive record (RESULT) of a body is (D, DT, sa, max_dn) of the last sub-step; the tensions those of the last sub-step.  A
body with nothing attached and no load row gets bodies.step's bits (nothing is added, not even +0: signed zeros stay), and a
call with no thrusters, foils or tethers and loads None is bodies.simulate.

Why this step.  A foil's force is -1/2 rho f A |dn| dn n along n, whose Jacobian with respect to the body velocity is
-rho f A |dn| n n^T: its norm is at most rho f A |dn| <= c_f, and with |R p| = |p| the torque's is at most c_f rf2, so the
foils widen the drag's bounds c_v, c_w exactly as drag.py's points do, and the drag argument of bodies.py carries over.  A
tether is a spring-damper: with the end's lever p its force's Jacobian is -(k + c d/dt) along u, so it adds c to the
velocity Jacobian and k to the position one.  Take one body of mass m on an anchor, along the line, with k only: x' = x + h v',
v' = v + h (-k x) / (m + h^2 k).  The step is linear with matrix [[1 - a, h], [-a / h, 1]] in (x, v), a = h^2 k / (m + h^2 k):
determinant (1 - a) + a = 1 and trace 2 - a in (1, 2] for any h > 0 and k >= 0, so both eigenvalues lie on the unit circle
and the oscillation neither grows nor decays (explicit symplectic Euler, denominator m, is unstable once h^2 k / m > 4).  Two
bodies on one line: the extension x = x_b - x_a follows the same matrix with a = h^2 k (1 / (m_a + h^2 k) + 1 / (m_b + h^2 k))
in (0, 2), trace 2 - a in (0, 2).  A chain: with D = diag(m_i + h^2 k deg_i) and K the chain's stiffness Laplacian, K <= 2
diag(k deg_i), so every mode of h^2 D^-1 K has a in [0, 2): each mode's step has determinant 1 and trace in (0, 2].  Damping c
multiplies the determinant by 1 - h c / (m + h c + h^2 k) in (0, 1]: it only damps.  The same holds per body axis for the
angular step, with the end's lever p: c |p|^2 and k |p|^2 bound the torque's Jacobians.  As h -> 0 the added terms vanish next
to m and I, and the step becomes explicit Euler on the true forces.

Limits of the model: those of bodies.py; a thruster's push and a foil's force act at the point regardless of how deep it is
under the surface (f only scales them); no propeller wash, stall or lift (the plate has normal drag only); the tether is
massless and straight, with no sag and no breaking (a host reads the tensions and drops it); no contacts.

Numeric policy (as oracle/bodies.py): every operation binary32, rounded once, in the order written here, no contraction;
divisions and sqrt IEEE.  The CUDA kernels (ocean_drive.cu and k_bodies_integrate_driven in ocean_bodies.cu, -fmad=false)
reproduce this bit for bit.
"""
from __future__ import annotations

import numpy as np

from . import bodies as bo
from . import buoyancy as bu
from . import drag as dr
from . import wake_coupling as wc
from .sampling import F

THRUSTER = np.dtype([("body", np.int32), ("position", np.float32, 3), ("direction", np.float32, 3), ("thrust", np.float32),
                     ("half_height", np.float32)])                                                                  # 36 B
FOIL = np.dtype([("body", np.int32), ("position", np.float32, 3), ("normal", np.float32, 3), ("area", np.float32),
                 ("half_height", np.float32)])                                                                      # 36 B
LOAD = np.dtype([("force", np.float32, 3), ("torque", np.float32, 3)])                                              # 24 B
TETHER = np.dtype([("body_a", np.int32), ("body_b", np.int32), ("point_a", np.float32, 3), ("point_b", np.float32, 3),
                   ("rest_length", np.float32), ("stiffness", np.float32), ("damping", np.float32)])               # 44 B
RESULT = np.dtype([("force", np.float32, 3), ("torque", np.float32, 3), ("wetted_foil_area", np.float32),
                   ("max_normal_speed", np.float32)])                                                               # 32 B


def rotate(T: np.ndarray, p: np.ndarray) -> np.ndarray:
    """r = R p per row for transforms T [n][12] and points p [n][3]: float32 [n][3] (buoyancy.world_points' order)."""
    T = np.asarray(T, np.float32).reshape(-1, 3, 4)
    p = np.asarray(p, np.float32).reshape(-1, 3)
    with np.errstate(all="ignore"):
        return np.stack([(T[:, k, 0] * p[:, 0] + T[:, k, 1] * p[:, 1]) + T[:, k, 2] * p[:, 2] for k in range(3)], 1)


def point_velocity(vel: np.ndarray, r: np.ndarray) -> np.ndarray:
    """vb = v + w x r per row (drag.py's brackets)."""
    with np.errstate(all="ignore"):
        return vel["linear"] + dr.cross(vel["angular"], r)


def norm2(p: np.ndarray) -> np.ndarray:
    p = np.asarray(p, np.float32).reshape(-1, 3)
    with np.errstate(all="ignore"):
        return (p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2]


def tethers_pass(table: np.ndarray, vel: np.ndarray, tethers: np.ndarray):
    """The tether lines of the module docstring: (tension [K], F_a [K][3], T_a [K][3], T_b [K][3]) float32."""
    t = np.ascontiguousarray(tethers, TETHER)
    K = len(t)
    T = table["transform"].astype(np.float32)
    a = t["body_a"].astype(np.int64)
    b = t["body_b"].astype(np.int64)
    anchored = b < 0
    bb = np.where(anchored, 0, b)
    with np.errstate(all="ignore"):
        ra = rotate(T[a], t["point_a"])
        xa = ra + T[a][:, [3, 7, 11]]
        va = point_velocity(vel[a], ra)
        rb = rotate(T[bb], t["point_b"])
        xb = rb + T[bb][:, [3, 7, 11]]
        vb = point_velocity(vel[bb], rb)
        rb[anchored] = 0.0
        vb[anchored] = 0.0
        xb[anchored] = t["point_b"][anchored]
        e = xb - xa
        L = np.sqrt((e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2])
        u = e / L[:, None]
        dv = vb - va
        s = t["stiffness"] * (L - t["rest_length"]) + t["damping"] * ((dv[:, 0] * u[:, 0] + dv[:, 1] * u[:, 1]) + dv[:, 2] * u[:, 2])
    taut = (L > F(0.0)) & (s > F(0.0))
    tension = np.where(taut, s, F(0.0)).astype(np.float32)
    Fa = np.zeros((K, 3), np.float32)
    Ta = np.zeros((K, 3), np.float32)
    Tb = np.zeros((K, 3), np.float32)
    with np.errstate(all="ignore"):
        Fa[taut] = tension[taut, None] * u[taut]
        Ta[taut] = dr.cross(ra[taut], Fa[taut])
        Tb[taut] = dr.cross(rb[taut], -Fa[taut])
    return tension, Fa, Ta, Tb


def _query(displacement, normal, points_xz, map_scales, tolerance, max_iterations, wake):
    """The surface records of extra query points (the actuators), and wv there while the coupling is live (else None)."""
    with np.errstate(all="ignore"):
        rec = wc.query_surface(displacement, normal, points_xz, map_scales, tolerance, max_iterations, wake)
        wv = wc.vertical_velocity(points_xz, wake, wake.cell_size) if wc.live(wake) else None
    return rec, wv


def drive_terms(displacement, normal, velocity, table, vel, map_scales, density, tolerance, max_iterations, thrusters, foils, tethers, h,
                wake=None):
    """Every incidence entry's term for one sub-step: a dict of per-entry arrays in the order thrusters, foils, tether ends
    (end a of tether k before end b), with keys body, F, T (float32 [n][3]), acts, kind (0 thruster, 1 foil, 2 tether end),
    a, dn, p2 (foils), v, w (tether ends); and the tensions."""
    th = np.ascontiguousarray(thrusters, THRUSTER)
    fo = np.ascontiguousarray(foils, FOIL)
    te = np.ascontiguousarray(tethers, TETHER)
    T = table["transform"].astype(np.float32)
    act_body = np.concatenate([th["body"], fo["body"]]).astype(np.int64)
    act_pos = np.concatenate([th["position"], fo["position"]]).astype(np.float32).reshape(-1, 3)
    act_dir = np.concatenate([th["direction"], fo["normal"]]).astype(np.float32).reshape(-1, 3)
    act_val = np.concatenate([th["thrust"], fo["area"]]).astype(np.float32)
    act_hh = np.concatenate([th["half_height"], fo["half_height"]]).astype(np.float32)
    nT, A = len(th), len(act_body)
    half_rho = F(0.5) * F(density)
    Fe = np.zeros((A, 3), np.float32)
    Te = np.zeros((A, 3), np.float32)
    a = np.zeros(A, np.float32)
    dn_abs = np.zeros(A, np.float32)
    acts = np.zeros(A, bool)
    if A:
        with np.errstate(all="ignore"):
            r = rotate(T[act_body], act_pos)
            w = r + T[act_body][:, [3, 7, 11]]
            rec, wv = _query(displacement, normal, np.stack([w[:, 0], w[:, 2]], 1), map_scales, tolerance, max_iterations, wake)
            f = bu.submerged_fraction(rec["displacement"][:, 1], w[:, 1], act_hh)
            n = rotate(T[act_body], act_dir)
            acts = f > F(0.0)
            is_t = np.arange(A) < nT
            # thrusters
            g = f * act_val
            Ft = g[:, None] * n
            # foils
            u = dr.water_velocity(velocity, np.stack([rec["source_x"], rec["source_z"]], 1), map_scales)
            if wv is not None:
                u[:, 1] = u[:, 1] + wv
            d = u - point_velocity(vel[act_body], r)
            dn = (d[:, 0] * n[:, 0] + d[:, 1] * n[:, 1]) + d[:, 2] * n[:, 2]
            af = f * act_val
            gf = ((half_rho * af) * dn) * np.abs(dn)
            Ff = gf[:, None] * n
            Fo = np.where(is_t[:, None], Ft, Ff).astype(np.float32)
            Fe[acts] = Fo[acts]
            Te[acts] = dr.cross(r[acts], Fo[acts])
            foil_wet = acts & ~is_t
            a[foil_wet] = af[foil_wet]
            dn_abs[foil_wet] = np.abs(dn[foil_wet])
    p2 = norm2(act_pos)
    tension, Fa, Ta, Tb = tethers_pass(table, vel, te) if len(te) else (np.zeros(0, np.float32),) + (np.zeros((0, 3), np.float32),) * 3
    K = len(te)
    taut = tension > F(0.0)
    # tether ends: a then b per tether; anchored ends b are dropped below
    end_body = np.stack([te["body_a"], te["body_b"]], 1).reshape(-1).astype(np.int64)
    with np.errstate(all="ignore"):
        end_F = np.stack([Fa, -Fa], 1).reshape(-1, 3)
    end_T = np.stack([Ta, Tb], 1).reshape(-1, 3)
    end_p2 = np.stack([norm2(te["point_a"]), norm2(te["point_b"])], 1).reshape(-1)
    end_c = np.repeat(te["damping"].astype(np.float32), 2)
    end_k = np.repeat(te["stiffness"].astype(np.float32), 2)
    end_acts = np.repeat(taut, 2)
    keep = end_body >= 0
    with np.errstate(all="ignore"):
        hc = F(h) * end_c
        hk = (F(h) * F(h)) * end_k
        end_v = hc + hk
        end_w = hc * end_p2 + hk * end_p2
    z = np.zeros(A, np.float32)
    terms = dict(
        body=np.concatenate([act_body, end_body[keep]]),
        F=np.concatenate([Fe, end_F[keep]]).astype(np.float32).reshape(-1, 3),
        T=np.concatenate([Te, end_T[keep]]).astype(np.float32).reshape(-1, 3),
        acts=np.concatenate([acts, end_acts[keep]]),
        kind=np.concatenate([np.where(np.arange(A) < nT, 0, 1), np.full(int(keep.sum()), 2)]),
        a=np.concatenate([a, np.zeros(int(keep.sum()), np.float32)]),
        dn=np.concatenate([dn_abs, np.zeros(int(keep.sum()), np.float32)]),
        p2=np.concatenate([p2, np.zeros(int(keep.sum()), np.float32)]),
        v=np.concatenate([z, end_v[keep]]).astype(np.float32),
        w=np.concatenate([z, end_w[keep]]).astype(np.float32),
    )
    assert K == len(tension)
    return terms, tension


def incidence_order(body: np.ndarray) -> np.ndarray:
    """The entries' positions within their body's incidence list (stable: the list order is the entries' order)."""
    body = np.asarray(body, np.int64)
    order = np.argsort(body, kind="stable")
    rank = np.empty(len(body), np.int64)
    counts = np.bincount(body, minlength=1) if len(body) else np.zeros(1, np.int64)
    starts = np.cumsum(counts) - counts
    rank[order] = np.arange(len(body)) - starts[body[order]]
    return rank


def drive_step(bodies, states, r2, hyd, drg, terms, loads, density, h):
    """The sums and step lines of the module docstring: (states after one sub-step, RESULT [B])."""
    bodies = np.ascontiguousarray(bodies, bo.BODY)
    s = np.array(states, bo.STATE, copy=True)
    B = len(bodies)
    h = F(h)
    with np.errstate(all="ignore"):
        Fo = hyd["force"] + drg["force"]
        tau = hyd["torque"] + drg["torque"]
    D = np.zeros((B, 3), np.float32)
    DT = np.zeros((B, 3), np.float32)
    sa = np.zeros(B, np.float32)
    max_dn = np.zeros(B, np.float32)
    rf2 = np.zeros(B, np.float32)
    tv = np.zeros(B, np.float32)
    tw = np.zeros(B, np.float32)
    foiled = np.zeros(B, bool)
    taut = np.zeros(B, bool)
    body = terms["body"]
    rank = incidence_order(body)
    with np.errstate(all="ignore"):
        for q in range(int(rank.max()) + 1 if len(rank) else 0):     # one entry per body per rank: a plain vectorised add
            k = np.nonzero(rank == q)[0]
            bk = body[k]
            foil = terms["kind"][k] == 1
            foiled[bk[foil]] = True
            rf2[bk[foil]] = np.fmax(rf2[bk[foil]], terms["p2"][k[foil]])
            act = terms["acts"][k]
            ka, ba = k[act], bk[act]
            Fo[ba] = Fo[ba] + terms["F"][ka]
            tau[ba] = tau[ba] + terms["T"][ka]
            D[ba] = D[ba] + terms["F"][ka]
            DT[ba] = DT[ba] + terms["T"][ka]
            wf = act & foil
            sa[bk[wf]] = sa[bk[wf]] + terms["a"][k[wf]]
            max_dn[bk[wf]] = np.fmax(max_dn[bk[wf]], terms["dn"][k[wf]])
            te = act & (terms["kind"][k] == 2)
            taut[bk[te]] = True
            tv[bk[te]] = tv[bk[te]] + terms["v"][k[te]]
            tw[bk[te]] = tw[bk[te]] + terms["w"][k[te]]
        if loads is not None:
            ld = np.ascontiguousarray(loads, LOAD)
            Fo = Fo + ld["force"]
            tau = tau + ld["torque"]
            D = D + ld["force"]
            DT = DT + ld["torque"]
        m = bodies["mass"].astype(np.float32)
        inertia = bodies["inertia"].astype(np.float32)
        cv = (F(density) * drg["wetted_drag_area"]) * drg["max_relative_speed"]
        cw = cv * r2
        cf = (F(density) * sa) * max_dn
        cv = np.where(foiled, cv + cf, cv)
        cw = np.where(foiled, cw + cf * rf2, cw)
        den_v = m + h * cv
        den_w = inertia + (h * cw)[:, None]
        den_v = np.where(taut, den_v + tv, den_v)
        den_w = np.where(taut[:, None], den_w + tw[:, None], den_w)
        # bodies.step from the gravity line on
        R = bo.rotation(s["orientation"])
        Fo[:, 1] = Fo[:, 1] - m * bo.G
        v = s["linear_velocity"] + (h / den_v)[:, None] * Fo
        w = s["angular_velocity"]
        tb = np.stack([(R[:, 0, k] * tau[:, 0] + R[:, 1, k] * tau[:, 1]) + R[:, 2, k] * tau[:, 2] for k in range(3)], 1)
        wb = np.stack([(R[:, 0, k] * w[:, 0] + R[:, 1, k] * w[:, 1]) + R[:, 2, k] * w[:, 2] for k in range(3)], 1)
        wb = wb + (h * tb) / den_w
        w = np.stack([(R[:, k, 0] * wb[:, 0] + R[:, k, 1] * wb[:, 1]) + R[:, k, 2] * wb[:, 2] for k in range(3)], 1)
        pos = s["position"] + h * v
        q = s["orientation"]
        dq = np.stack([(w[:, 0] * q[:, 3] + w[:, 1] * q[:, 2]) - w[:, 2] * q[:, 1],
                       (w[:, 1] * q[:, 3] + w[:, 2] * q[:, 0]) - w[:, 0] * q[:, 2],
                       (w[:, 2] * q[:, 3] + w[:, 0] * q[:, 1]) - w[:, 1] * q[:, 0],
                       -((w[:, 0] * q[:, 0] + w[:, 1] * q[:, 1]) + w[:, 2] * q[:, 2])], 1)
        q = q + (F(0.5) * h) * dq
        n = np.sqrt(((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]) + q[:, 3] * q[:, 3])
        q = q / n[:, None]
    s["linear_velocity"] = v
    s["angular_velocity"] = w
    s["position"] = pos
    s["orientation"] = q
    out = np.zeros(B, RESULT)
    out["force"] = D
    out["torque"] = DT
    out["wetted_foil_area"] = sa
    out["max_normal_speed"] = max_dn
    return s, out


def simulate(displacement, normal, velocity, bodies, states, points, drag_areas, map_scales, density=1025.0, dt=1.0 / 60.0, substeps=1,
             tolerance=1e-3, max_iterations=8, thrusters=None, foils=None, loads=None, tethers=None, wake=None):
    """bodies.simulate's arguments (and wake_coupling.simulate's wake) plus THRUSTER, FOIL, LOAD [B] (or None) and TETHER rows.
    Returns (STATE [B], buoyancy.RESULT [B], drag.RESULT [B], RESULT [B], tensions float32 [K], float32 [B][12])."""
    th = np.zeros(0, THRUSTER) if thrusters is None else np.ascontiguousarray(thrusters, THRUSTER).reshape(-1)
    fo = np.zeros(0, FOIL) if foils is None else np.ascontiguousarray(foils, FOIL).reshape(-1)
    te = np.zeros(0, TETHER) if tethers is None else np.ascontiguousarray(tethers, TETHER).reshape(-1)
    bodies = np.ascontiguousarray(bodies, bo.BODY)
    B = len(bodies)
    if not len(th) and not len(fo) and not len(te) and loads is None:
        s, hyd, drg, T = wc.simulate(displacement, normal, velocity, bodies, states, points, drag_areas, map_scales, density, dt, substeps,
                                     tolerance, max_iterations, wake)
        return s, hyd, drg, np.zeros(B, RESULT), np.zeros(0, np.float32), T
    s = np.array(states, bo.STATE, copy=True)
    h = F(dt) / F(substeps)
    r2 = bo.radius2(bodies, points)
    hyd, drg = np.zeros(B, bu.RESULT), np.zeros(B, dr.RESULT)
    world = int(bodies["num_points"].astype(np.int64).sum())
    drive, tension = np.zeros(B, RESULT), np.zeros(len(te), np.float32)
    for _ in range(substeps):
        table, vel = bo.pose(bodies, s)
        if world:
            with np.errstate(all="ignore"):
                hyd, drg = wc.body_forces(displacement, normal, velocity, table, vel, points, drag_areas, map_scales, density, tolerance,
                                          max_iterations, wake=wake)
        terms, tension = drive_terms(displacement, normal, velocity, table, vel, map_scales, density, tolerance, max_iterations, th, fo, te,
                                     h, wake)
        s, drive = drive_step(bodies, s, r2, hyd, drg, terms, loads, density, h)
    return s, hyd, drg, drive, tension, bo.transforms(s)
