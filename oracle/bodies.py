"""CPU specification of the floating-body integrator (ocean_simulate_bodies): rigid bodies advanced by sub-steps of
buoyancy, quadratic drag and gravity, the forces those of oracle/drag.py.

TEST INFRASTRUCTURE ONLY -- the product path (godotoceanwaves_b200/csrc) never imports or calls this module.

Inputs: BODY (mass in kg, principal moments of inertia about the centre of mass in kg m^2 along the hull axes, and a range
[first_point, first_point + num_points) into the hull points and drag areas, as buoyancy.BODY's), STATE (the world position
of the body origin, which is its centre of mass; a unit quaternion q = (x, y, z, w) from body to world; the world-frame
linear velocity of the centre of mass and angular velocity), the hull points, drag areas, maps and scales of
drag.body_forces, density, dt and the number of sub-steps S.  h = dt / S (binary32).  Once per call, per body:

  r2    = max((p.x*p.x + p.y*p.y) + p.z*p.z over the body's hull points), NaN dropped (np.fmax), from 0

One sub-step, per body:

  pose    xx = x*x, yy = y*y, zz = z*z, xy = x*y, xz = x*z, yz = y*z, wx = w*x, wy = w*y, wz = w*z
          R = [[1 - 2*(yy + zz),  2*(xy - wz),      2*(xz + wy)    ],
               [2*(xy + wz),      1 - 2*(xx + zz),  2*(yz - wx)    ],
               [2*(xz - wy),      2*(yz + wx),      1 - 2*(xx + yy)]]
          transform = [R | position] (buoyancy.BODY, with the body's range); velocity = (linear_velocity, angular_velocity)
          (drag.VELOCITY: the origin is the centre of mass)
  forces  hyd, drg = drag.body_forces(...) for that transform and velocity
  step    c_v   = (density * drg.wetted_drag_area) * drg.max_relative_speed
          c_w   = c_v * r2
          F     = hyd.force + drg.force;  F.y = F.y - mass * G                     G = 9.81 (binary32)
          v'    = v + (h / (mass + h*c_v)) * F
          tau   = hyd.torque + drg.torque
          tau_b.k = (R[0][k]*tau.x + R[1][k]*tau.y) + R[2][k]*tau.z                 R^T tau
          w_b.k   = (R[0][k]*w.x + R[1][k]*w.y) + R[2][k]*w.z                       R^T w
          w_b'.k  = w_b.k + (h*tau_b.k) / (inertia.k + h*c_w)
          w'.k    = (R[k][0]*w_b'.x + R[k][1]*w_b'.y) + R[k][2]*w_b'.z               R w_b'
          position' = position + h*v'
          dq    = w' (x) q = ((w.x*q.w + w.y*q.z) - w.z*q.y,  (w.y*q.w + w.z*q.x) - w.x*q.z,
                              (w.z*q.w + w.x*q.y) - w.y*q.x,  -((w.x*q.x + w.y*q.y) + w.z*q.z))      (w = w')
          q~    = q + (0.5*h) * dq;  n = sqrt(((q~.x*q~.x + q~.y*q~.y) + q~.z*q~.z) + q~.w*q~.w);  q' = q~ / n

The call returns the states after S sub-steps, the records of the last sub-step (the forces at the pose that sub-step started
from) and transforms = [R(q') | position'] of the final states, 3 x 4 row-major ([B][12]).  A body with num_points = 0 is
ballistic: its records are all zero.  A NaN or infinite state affects only its own body.

Why this step.  The drag of a submerged point is 1/2 rho f C_dA |d| d with d = u - v_point; its Jacobian with respect to the
body velocity is -1/2 rho f C_dA (s I + d d^T / s), s = |d|, whose norm is at most rho f C_dA s.  Summed over the points,
|dF_drag/dv| <= rho * sum(f C_dA) * max s = c_v, and since |R p| = |p|, |dT_drag/dw| <= c_v * r2 = c_w.  For the drag
linearised about the current velocity, F = F0 - J (v - v0) with 0 <= J <= c_v along each eigendirection, and the step
v' = v + h F / (m + h c_v) moves the relative velocity by the factor 1 - h J / (m + h c_v), which lies in (0, 1]: the step
never overshoots the water velocity and is stable for any h, where explicit Euler (factor 1 - h J / m) overshoots once
h J > m and diverges once h J > 2 m.  As h -> 0 the bound's term h c_v vanishes next to m and the step becomes explicit Euler on
the true forces; at large h the bound only slows the approach to the water velocity.  The same holds per body axis for the
angular step, whose denominator inertia + h c_w bounds the drag torque's Jacobian; dividing per body axis is
w + h (I_w + h c_w 1)^-1 tau with I_w = R diag(inertia) R^T, without a 3 x 3 solve.

Limits of the model:
  * No added mass: the heave period is shorter than a real body's.
  * No gyroscopic term (w x I w): a body spinning off a principal axis does not precess.
  * No contacts between bodies.
  * The SURFACE water velocity at every depth (drag.py's limit).
  * Every sub-step of a call sees the same maps.
  * The hydrostatic spring is explicit in position: it needs h < T_heave / pi, T_heave = 2 pi sqrt(m / (rho G A_waterplane)).
  * The body origin is the centre of mass and the hull axes are the principal axes.  A Godot RigidBody3D with a custom
    center_of_mass c shifts its hull points by -c once (p - c), passes position = global_position + basis * c and writes
    back global_position = position - basis * c.

Numeric policy (as oracle/drag.py): every operation binary32, rounded once, in the order written here, no contraction;
divisions and sqrt IEEE.  The CUDA kernels (ocean_bodies.cu, -fmad=false) reproduce this bit for bit.
"""
from __future__ import annotations

import numpy as np

from . import buoyancy as bu
from . import drag as dr
from .sampling import F

BODY = np.dtype([("mass", np.float32), ("inertia", np.float32, 3), ("first_point", np.int32), ("num_points", np.int32)])     # 24 B
STATE = np.dtype([("position", np.float32, 3), ("orientation", np.float32, 4), ("linear_velocity", np.float32, 3),
                  ("angular_velocity", np.float32, 3)])                                                                     # 52 B
G = bu.G


def rotation(q: np.ndarray) -> np.ndarray:
    """R(q) of the module docstring for quaternions [n][4] (x, y, z, w): float32 [n][3][3]."""
    q = np.asarray(q, np.float32).reshape(-1, 4)
    x, y, z, w = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    one, two = F(1.0), F(2.0)
    with np.errstate(all="ignore"):
        xx, yy, zz = x * x, y * y, z * z
        xy, xz, yz = x * y, x * z, y * z
        wx, wy, wz = w * x, w * y, w * z
        R = np.stack([one - two * (yy + zz), two * (xy - wz), two * (xz + wy),
                      two * (xy + wz), one - two * (xx + zz), two * (yz - wx),
                      two * (xz - wy), two * (yz + wx), one - two * (xx + yy)], 1)
    return R.astype(np.float32).reshape(-1, 3, 3)


def transforms(states: np.ndarray) -> np.ndarray:
    """[R(q) | position] of each state, 3 x 4 row-major: float32 [n][12]."""
    states = np.ascontiguousarray(states, STATE)
    T = np.concatenate([rotation(states["orientation"]), states["position"].astype(np.float32)[:, :, None]], 2)
    return T.reshape(-1, 12)


def pose(bodies: np.ndarray, states: np.ndarray):
    """The body-forces inputs of one sub-step: (buoyancy.BODY [B], drag.VELOCITY [B])."""
    bodies = np.ascontiguousarray(bodies, BODY)
    states = np.ascontiguousarray(states, STATE)
    table = np.zeros(len(bodies), bu.BODY)
    table["transform"] = transforms(states)
    table["first_point"] = bodies["first_point"]
    table["num_points"] = bodies["num_points"]
    vel = np.zeros(len(bodies), dr.VELOCITY)
    vel["linear"] = states["linear_velocity"]
    vel["angular"] = states["angular_velocity"]
    return table, vel


def radius2(bodies: np.ndarray, points: np.ndarray) -> np.ndarray:
    """r2 of the module docstring: float32 [B]."""
    bodies = np.ascontiguousarray(bodies, BODY)
    points = np.ascontiguousarray(points, bu.POINT)
    counts = bodies["num_points"].astype(np.int64)
    body = np.repeat(np.arange(len(bodies)), counts)
    j = np.arange(int(counts.sum()), dtype=np.int64) - np.repeat(np.cumsum(counts) - counts, counts)
    p = points["position"][bodies["first_point"].astype(np.int64)[body] + j].astype(np.float32)
    with np.errstate(all="ignore"):
        d2 = (p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2]
    out = np.zeros(len(bodies), np.float32)
    np.fmax.at(out, body, d2)
    return out


def step(bodies: np.ndarray, states: np.ndarray, r2: np.ndarray, hyd: np.ndarray, drg: np.ndarray, density: float, h) -> np.ndarray:
    """The `step` lines of the module docstring: the states after one sub-step of h from their records (hyd, drg)."""
    bodies = np.ascontiguousarray(bodies, BODY)
    s = np.array(states, STATE, copy=True)
    h = F(h)
    R = rotation(s["orientation"])
    m = bodies["mass"].astype(np.float32)
    inertia = bodies["inertia"].astype(np.float32)
    with np.errstate(all="ignore"):
        cv = (F(density) * drg["wetted_drag_area"]) * drg["max_relative_speed"]
        cw = cv * r2
        Fo = hyd["force"] + drg["force"]
        Fo[:, 1] = Fo[:, 1] - m * G
        v = s["linear_velocity"] + (h / (m + h * cv))[:, None] * Fo
        tau = hyd["torque"] + drg["torque"]
        w = s["angular_velocity"]
        tb = np.stack([(R[:, 0, k] * tau[:, 0] + R[:, 1, k] * tau[:, 1]) + R[:, 2, k] * tau[:, 2] for k in range(3)], 1)
        wb = np.stack([(R[:, 0, k] * w[:, 0] + R[:, 1, k] * w[:, 1]) + R[:, 2, k] * w[:, 2] for k in range(3)], 1)
        wb = wb + (h * tb) / (inertia + (h * cw)[:, None])
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
    return s


def simulate(displacement: np.ndarray, normal: np.ndarray, velocity: np.ndarray, bodies: np.ndarray, states: np.ndarray,
             points: np.ndarray, drag_areas: np.ndarray, map_scales: np.ndarray, density: float = 1025.0, dt: float = 1.0 / 60.0,
             substeps: int = 1, tolerance: float = 1e-3, max_iterations: int = 8):
    """displacement, normal, velocity: [C][N][N][4] float16 (drag.body_forces'); bodies: BODY [B]; states: STATE [B];
    points: buoyancy.POINT [P]; drag_areas: [P] float32; map_scales: [C][4] float32.
    Returns (STATE [B], buoyancy.RESULT [B], drag.RESULT [B], float32 [B][12]): the states after `substeps` sub-steps of
    dt / substeps, the last sub-step's records and the final transforms."""
    bodies = np.ascontiguousarray(bodies, BODY)
    s = np.array(states, STATE, copy=True)
    h = F(dt) / F(substeps)
    r2 = radius2(bodies, points)
    hyd, drg = np.zeros(len(bodies), bu.RESULT), np.zeros(len(bodies), dr.RESULT)     # every body ballistic: all-zero records
    world = int(bodies["num_points"].astype(np.int64).sum())
    for _ in range(substeps):
        table, vel = pose(bodies, s)
        if world:
            with np.errstate(all="ignore"):
                hyd, drg = dr.body_forces(displacement, normal, velocity, table, vel, points, drag_areas, map_scales, density,
                                          tolerance, max_iterations)
        s = step(bodies, s, r2, hyd, drg, density, h)
    return s, hyd, drg, transforms(s)
