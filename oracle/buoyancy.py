"""CPU specification of the buoyancy op (ocean_buoyancy): per-body hydrostatic force and torque from hull sample points on
the displaced water surface.

TEST INFRASTRUCTURE ONLY -- the product path (godotoceanwaves_b200/csrc) never imports or calls this module.

Inputs: hull points (POINT, body-local position, volume in m^3, half_height in m: a vertical column element of that volume,
centred on the point, reaching half_height above and below it) and bodies (BODY: a 3 x 4 row-major body-to-world matrix
[R | t], the layout of ocean_spray_grid's emission_transform, and a range [first_point, first_point + num_points) into the
hull points; ranges may overlap, so identical bodies share one hull).  World point j of body b (hull point
p = points[first_point + j]):

  r.k   = ((R[k][0]*p.x + R[k][1]*p.y) + R[k][2]*p.z)          k = x, y, z   (rotated, not translated)
  w.k   = r.k + t.k
  rec   = surface.query_surface at Q = (w.x, w.z)                             (the same tolerance and step budget)
  eta   = rec.displacement[1]                                                 water height over Q
  f     = h > 0 ? min(max((eta - (w.y - h)) / (h + h), 0), 1) : (w.y <= eta ? 1 : 0)      h = half_height
  v     = f * volume

min and max drop NaN (np.fmin / np.fmax), so a NaN height gives f = 0.  Per body S0 = sum v and S1.k = sum v * r.k, summed
in a FIXED order: point j goes to lane j mod 32, each lane starts from +0.0 and adds its points in increasing j, and the 32
partials are combined by the tree `for o in 16, 8, 4, 2, 1: p[l] = p[l] + p[l + o] for l < o` (one warp's
__shfl_down_sync reduction).  With rho_g = density * G (binary32):

  submerged_volume = S0
  force            = (0, rho_g * S0, 0)
  torque           = (-(rho_g * S1.z), 0, rho_g * S1.x)       about the body origin t: sum of r x F over the points
  center_offset    = S1 / S0 if S0 > 0 else (0, 0, 0)          centre of buoyancy = t + center_offset
  max_residual     = NaN-dropping max of the points' query residuals
  unconverged      = number of points with !(residual <= tolerance)

A body with num_points = 0 gets an all-zero record.

Numeric policy (as oracle/sampling.py): every operation binary32, rounded once, in the order written here, no contraction;
divisions IEEE.  The CUDA kernels (ocean_buoyancy.cu, -fmad=false) reproduce this bit for bit.
"""
from __future__ import annotations

import numpy as np

from .sampling import F
from .surface import RECORD as SURFACE_RECORD
from .surface import query_surface

POINT = np.dtype([("position", np.float32, 3), ("volume", np.float32), ("half_height", np.float32)])           # 20 B
BODY = np.dtype([("transform", np.float32, 12), ("first_point", np.int32), ("num_points", np.int32)])          # 56 B
RESULT = np.dtype([("force", np.float32, 3), ("torque", np.float32, 3), ("submerged_volume", np.float32),
                   ("center_offset", np.float32, 3), ("max_residual", np.float32), ("unconverged", np.uint32)])  # 48 B
G = F(9.81)        # wave_generator.gd:5
LANES = 32


def world_points(bodies: np.ndarray, points: np.ndarray):
    """The world points in body-major order: (body index [n], j [n], r [n][3], w [n][3]), r and w float32."""
    counts = bodies["num_points"].astype(np.int64)
    body = np.repeat(np.arange(len(bodies)), counts)
    start = np.repeat(np.cumsum(counts) - counts, counts)
    j = np.arange(int(counts.sum()), dtype=np.int64) - start
    p = points[bodies["first_point"].astype(np.int64)[body] + j]
    T = bodies["transform"].astype(np.float32)[body].reshape(-1, 3, 4)
    pos = p["position"].astype(np.float32)
    r = np.empty((len(body), 3), np.float32)
    for k in range(3):
        r[:, k] = (T[:, k, 0] * pos[:, 0] + T[:, k, 1] * pos[:, 1]) + T[:, k, 2] * pos[:, 2]
    w = r + T[:, :, 3]
    return body, j, r, w


def submerged_fraction(eta: np.ndarray, wy: np.ndarray, h: np.ndarray) -> np.ndarray:
    """f of the module docstring, float32 [n]."""
    with np.errstate(all="ignore"):
        column = np.fmin(np.fmax((eta - (wy - h)) / (h + h), F(0.0)), F(1.0))
    step = np.where(wy <= eta, F(1.0), F(0.0))
    return np.where(h > F(0.0), column, step).astype(np.float32)


def lane_tree_sum(values: np.ndarray, body: np.ndarray, j: np.ndarray, num_bodies: int) -> np.ndarray:
    """Per-body sums of values [n][k] in the fixed order: lane j mod 32, increasing j within a lane, then the shuffle tree.
    Returns float32 [num_bodies][k]."""
    vals = np.asarray(values, np.float32).reshape(len(body), -1)
    lanes = np.zeros((num_bodies, LANES, vals.shape[1]), np.float32)
    lane = j % LANES
    row = j // LANES
    order = np.argsort(row, kind="stable")
    bounds = np.searchsorted(row[order], np.arange(int(row.max()) + 2 if len(row) else 1))
    with np.errstate(all="ignore"):
        for q in range(len(bounds) - 1):       # one point per (body, lane) in each row: a plain vectorised add
            k = order[bounds[q]:bounds[q + 1]]
            lanes[body[k], lane[k]] = lanes[body[k], lane[k]] + vals[k]
        o = LANES // 2
        while o >= 1:
            lanes[:, :o] = lanes[:, :o] + lanes[:, o:2 * o]
            o //= 2
    return lanes[:, 0]


def buoyancy(displacement: np.ndarray, normal: np.ndarray, bodies: np.ndarray, points: np.ndarray, map_scales: np.ndarray,
             density: float = 1025.0, tolerance: float = 1e-3, max_iterations: int = 8, return_samples: bool = False):
    """displacement, normal: [C][N][N][4] float16; bodies: BODY [B]; points: POINT [P]; map_scales: [C][4] float32.
    Returns RESULT [B], and with return_samples also the surface records [sum of num_points] in world-point order."""
    bodies = np.ascontiguousarray(bodies, BODY)
    points = np.ascontiguousarray(points, POINT)
    B = len(bodies)
    body, j, r, w = world_points(bodies, points)
    samples = query_surface(displacement, normal, np.stack([w[:, 0], w[:, 2]], 1), map_scales, tolerance, max_iterations) \
        if len(body) else np.zeros(0, SURFACE_RECORD)
    p = points[bodies["first_point"].astype(np.int64)[body] + j]
    f = submerged_fraction(samples["displacement"][:, 1], w[:, 1], p["half_height"].astype(np.float32))
    with np.errstate(all="ignore"):
        v = f * p["volume"].astype(np.float32)
        terms = np.stack([v, v * r[:, 0], v * r[:, 1], v * r[:, 2]], 1)
    S = lane_tree_sum(terms, body, j, B)
    S0, S1 = S[:, 0], S[:, 1:]
    rho_g = F(density) * G
    out = np.zeros(B, RESULT)
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
    out[bodies["num_points"] == 0] = np.zeros(1, RESULT)
    return (out, samples) if return_samples else out
