"""CPU specification of the body-forces op (ocean_body_forces): per body, the buoyancy record of oracle/buoyancy.py and a
quadratic drag record against the water velocity, both from one surface query.

TEST INFRASTRUCTURE ONLY -- the product path (godotoceanwaves_b200/csrc) never imports or calls this module.

Inputs: those of buoyancy.buoyancy, plus the velocity maps ([C][N][N][4] float16, ocean_copy_velocity_to_host), one
VELOCITY per body (world frame: `linear` is the velocity of the body ORIGIN t in m/s, `angular` the angular velocity in
rad/s) and drag_areas[P], C_d A in m^2 per hull point (parallel to the hull points, so shared hulls share their areas).
For world point j of body b, with r, w, the surface record `rec` and f exactly as in buoyancy.py, and a point with f > 0:

  u   = sum_i texture_bilinear(velocity_i, (rec.source_x, rec.source_z) * s_i.xy).xyz * s_i.z
        (the displacement half of sampling.sample_maps on the velocity maps, at the record's source point: the water
        velocity at w)
  vb  = v + (a.y*r.z - a.z*r.y,  a.z*r.x - a.x*r.z,  a.x*r.y - a.y*r.x)        v = linear, a = angular; each bracket
                                                                                rounded as written
  d   = u - vb
  s   = sqrt((d.x*d.x + d.y*d.y) + d.z*d.z)
  k   = (f * cda) * s
  F   = k * d
  T   = (r.y*F.z - r.z*F.y,  r.z*F.x - r.x*F.z,  r.x*F.y - r.y*F.x)             r x F, component order as vb's

A point with f = 0 (dry) gathers nothing and adds nothing: it is skipped, not added as zero.  Per body the sums of F, T and
f * cda use buoyancy.lane_tree_sum's order (lane j mod 32, increasing j within a lane, then the shuffle tree).  With
half_rho = 0.5 * density (binary32):

  force               half_rho * sum F
  torque              half_rho * sum T                 about the body origin t, like the buoyancy torque
  wetted_drag_area    sum f * cda
  max_relative_speed  max(0, s over the wet points), NaN dropped (np.fmax): 0 when there are none

A body with num_points = 0 gets an all-zero record.  The hydrostatic record is buoyancy.buoyancy(...) unchanged.

Limits of the model:
  * The water velocity is the SURFACE velocity at every submerged point.  The orbital velocity of a wave decays with depth
    z below the surface as e^(-k z); at 1 m of draft this overstates the longest wave of a 16 m tile about 1.5 times, and
    shorter waves by more.
  * No added mass, radiation or wave-making damping, skin friction, or separate normal and tangential coefficients.
  * Nothing is written back into the maps: no wake and no foam injection.
  * Quadratic drag is stiff for light bodies under explicit integration.  The op does not integrate;
    max_relative_speed is there so that a host can choose sub-steps.

Numeric policy (as oracle/buoyancy.py): every operation binary32, rounded once, in the order written here, no contraction;
sqrt IEEE.  The CUDA kernel (k_drag_reduce in ocean_buoyancy.cu, -fmad=false) reproduces this bit for bit.
"""
from __future__ import annotations

import numpy as np

from . import buoyancy as bu
from .sampling import F, texture_bilinear

VELOCITY = np.dtype([("linear", np.float32, 3), ("angular", np.float32, 3)])                                   # 24 B
RESULT = np.dtype([("force", np.float32, 3), ("torque", np.float32, 3), ("wetted_drag_area", np.float32),
                   ("max_relative_speed", np.float32)])                                                        # 32 B


def water_velocity(velocity: np.ndarray, points_xz: np.ndarray, map_scales: np.ndarray) -> np.ndarray:
    """u of the module docstring at UNDISPLACED points [n][2]: float32 [n][3] (ocean_sample_velocity)."""
    pts = np.ascontiguousarray(points_xz, np.float32).reshape(-1, 2)
    sc = np.ascontiguousarray(map_scales, np.float32)
    u = np.zeros((len(pts), 3), np.float32)
    with np.errstate(all="ignore"):
        for i in range(sc.shape[0]):
            u = u + texture_bilinear(velocity[i], pts[:, 0] * sc[i, 0], pts[:, 1] * sc[i, 1])[:, :3] * sc[i, 2]
    return u


def cross(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """a x b per row, [n][3] float32, each component (a.y*b.z - a.z*b.y, ...) rounded as written."""
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1],
                     a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def body_forces(displacement: np.ndarray, normal: np.ndarray, velocity: np.ndarray, bodies: np.ndarray, velocities: np.ndarray,
                points: np.ndarray, drag_areas: np.ndarray, map_scales: np.ndarray, density: float = 1025.0, tolerance: float = 1e-3,
                max_iterations: int = 8, return_samples: bool = False):
    """displacement, normal, velocity: [C][N][N][4] float16; bodies: buoyancy.BODY [B]; velocities: VELOCITY [B];
    points: buoyancy.POINT [P]; drag_areas: [P] float32; map_scales: [C][4] float32.
    Returns (buoyancy.RESULT [B], RESULT [B]), and with return_samples also the surface records in world-point order."""
    bodies = np.ascontiguousarray(bodies, bu.BODY)
    points = np.ascontiguousarray(points, bu.POINT)
    velocities = np.ascontiguousarray(velocities, VELOCITY)
    drag_areas = np.ascontiguousarray(drag_areas, np.float32)
    B = len(bodies)
    hydro, samples = bu.buoyancy(displacement, normal, bodies, points, map_scales, density, tolerance, max_iterations, return_samples=True)
    body, j, r, w = bu.world_points(bodies, points)
    k_point = bodies["first_point"].astype(np.int64)[body] + j
    f = bu.submerged_fraction(samples["displacement"][:, 1], w[:, 1], points["half_height"][k_point].astype(np.float32))
    wet = f > F(0.0)
    body, j, r, f, k_point = body[wet], j[wet], r[wet], f[wet], k_point[wet]
    src = np.stack([samples["source_x"][wet], samples["source_z"][wet]], 1)
    u = water_velocity(velocity, src, map_scales)
    vel = velocities[body]
    with np.errstate(all="ignore"):
        vb = vel["linear"] + cross(vel["angular"], r)
        d = u - vb
        s = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        a = f * drag_areas[k_point]
        k = a * s
        Fp = k[:, None] * d
        Tp = cross(r, Fp)
    S = bu.lane_tree_sum(np.concatenate([Fp, Tp, a[:, None]], 1), body, j, B) if len(body) else np.zeros((B, 7), np.float32)
    half_rho = F(0.5) * F(density)
    out = np.zeros(B, RESULT)
    with np.errstate(all="ignore"):
        out["force"] = half_rho * S[:, 0:3]
        out["torque"] = half_rho * S[:, 3:6]
    out["wetted_drag_area"] = S[:, 6]
    max_s = np.zeros(B, np.float32)
    np.fmax.at(max_s, body, s)
    out["max_relative_speed"] = max_s
    out[bodies["num_points"] == 0] = np.zeros(1, RESULT)
    return (hydro, out, samples) if return_samples else (hydro, out)
