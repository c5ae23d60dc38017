"""CPU specification of the hull-mesh ops (ocean_hull_forces, ocean_simulate_hull_bodies): floating bodies whose hull is a
closed triangle mesh, with hydrostatic pressure and drag integrated over the wetted triangles.

TEST INFRASTRUCTURE ONLY -- the product path (godotoceanwaves_b200/csrc) never imports or calls this module.

Inputs: MESH rows (a range of the vertices [V][3] float32, hull-local, and of the triangles [T][3] int32, indices local to the
mesh's vertex range, with the normal and tangential drag coefficients C_n, C_t), BODY rows (a 3 x 4 row-major transform
[R | t] and a mesh index, the layout of buoyancy.BODY) and one drag.VELOCITY per body.  Winding is Godot's: front faces are
clockwise seen from outside, so the outward area vector of triangle (P0, P1, P2) is a = 0.5 (P2 - P0) x (P1 - P0).

World vertex j of a body (p = its mesh's vertex j), in body-major order:

  r.k  = ((R[k][0]*p.x + R[k][1]*p.y) + R[k][2]*p.z)          (buoyancy.world_points' operations)
  rec  = surface.query_surface at Q = (r.x + t.x, r.z + t.z)   (wake_coupling.query_surface while a coupling is live)
  d    = rec.displacement[1] - (r.y + t.y)                     depth below the water surface
  u    = drag.water_velocity at (rec.source_x, rec.source_z), u.y + wake_coupling.vertical_velocity(Q) while coupled

Per triangle j of the body's mesh, with corners c = (r, d, u) in winding order.  It is dropped when a corner's d is NaN.
Corners with d > 0 are wet:
  0 wet   nothing
  3 wet   the piece (c0, c1, c2)
  1 wet   rotated (cyclically, which keeps the winding) so that c0 is wet: the piece (c0, X01, X02)
  2 wet   rotated so that c2 is dry: the pieces (c0, c1, X12) and (c0, X12, X20)
  X_ab    the crossing of edge a -> b from its wet corner a: t = d_a / (d_a - d_b), r = r_a + t*(r_b - r_a) per component,
          u = u_a + t*(u_b - u_a), d = 0
A corner at exactly d = 0 is dry.  The triangle's sums are its pieces' sums added to +0 in that order.

One piece (c0, c1, c2), every operation binary32 in the order written:

  a    = 0.5 * ((r2 - r0) x (r1 - r0))                        x: (a.y*b.z - a.z*b.y, a.z*b.x - a.x*b.z, a.x*b.y - a.y*b.x)
  sd   = (d0 + d1) + d2,   sdd = (d0*d0 + d1*d1) + d2*d2
  m.k  = ((d0*r0.k + d1*r1.k) + d2*r2.k) + sd*((r0.k + r1.k) + r2.k)
  my   = m.y + 0.5*(sdd + sd*sd)
  pressure sums   f += a*sd,   tq += m x a,   q += (a.y*m.x, a.y*my, a.y*m.z)
  A    = sqrt((a.x*a.x + a.y*a.y) + a.z*a.z); only when A > 0 (a zero-area or NaN piece adds no drag):
  e_i  = u_i - (v + w x r_i)                                  relative velocity of the water at corner i (v, w: the body's)
  dc   = ((e0 + e1) + e2) / 3,   n = a / A,   dn = (dc.x*n.x + dc.y*n.y) + dc.z*n.z
  dt   = dc - dn*n,   kt = (C_t*A) * |dt|,   kn = dn < 0 ? (C_n*A)*(dn*dn) : 0
  G    = kt*dt - kn*n,   rc = ((r0 + r1) + r2) / 3
  drag sums       g += G,   gt += rc x G,   area += (C_n + C_t)*A,   speed = max(speed, |dc|)

Per body the triangles' sums use buoyancy.lane_tree_sum's order (triangle j in lane j mod 32, increasing j, then the shuffle
tree); speed is the NaN-dropping max from 0.  With rho_g = density * G and half_rho = 0.5 * density (binary32):

  force            -(rho_g * (f / 3))                  = -rho g integral(d n dA)
  torque           -(rho_g * (tq / 12))                = -rho g integral(d (r x n) dA), about the body origin t
  submerged_volume V = -(f.y / 3)                      = -integral(d n_y dA)
  center_offset    (-(q / 12)) / V, 0 unless V > 0     = S1 / V, S1 = -integral((d r + y d^2 / 2) n_y dA)
  max_residual, unconverged   over the body's world vertices, as buoyancy.py's
  drag.force       half_rho * g,   drag.torque  half_rho * gt,   wetted_drag_area  area,   max_relative_speed  speed

A body whose mesh has no vertices gets all-zero records.

Why these integrals.  d = eta - y is linear over a piece where the surface is flat, and so are r and u (they are linear in
the corners).  For f, g linear over a triangle of area A and unit normal n, integral(f n dA) = a (f0 + f1 + f2) / 3 and
integral(f g n dA) = a (sum f_i g_i + sum f sum g) / 12, with a = A n: the pressure force needs the first and the torque
(d r) x n, V and S1 the second (d^2 = d d), so no square root enters the hydrostatic record.  Take a closed hull on flat water
eta = const and let W be its submerged part, bounded by the wet hull and the waterplane cap, where d = 0.  The divergence
theorem gives, with the outward normal and the cap contributing nothing (its integrands carry a factor d):
  grad d = -y:              integral over dW of d n dA = integral over W of grad d dV = -V y,  so force = rho g V y
  div(d y) = -1:            -integral(d n_y dA) = V
  div(r_k d y) = d [k=y] - r_k:   -integral(r_k d n_y dA) = V c_k - [k=y] integral(d dV)
  div(d^2/2 y) = -d:        integral(d^2/2 n_y dA) = -integral(d dV)
so S1 = -integral((d r + y d^2/2) n_y dA) = V c exactly: V and t + S1 / V are the displaced volume and the centre of
buoyancy, and the torque -rho g integral(d r x n dA) = c x (rho g V y), at any heel.  On a wave the same integrals give the
pressure force normal to the hull, with a horizontal part on a slope.

Drag.  A piece moving through the water at relative velocity -dc (dc the water's velocity relative to it) feels normal
pressure drag 1/2 rho C_n A dn^2 on its front only (dn < 0: the water flows into the face) and tangential friction
1/2 rho C_t A |dt| dt; a box moving face-on at U then feels exactly 1/2 rho C_n A_face U^2.  The Jacobian of either term
with respect to the body velocity has norm at most rho C A |dc|, so c_v = density * wetted_drag_area * max_relative_speed
bounds it as bodies.py's step assumes, and since clip points lie on triangle edges, |r| <= max |p| keeps c_w = c_v r2 a bound.

Limits: one warp per body on the device; the SURFACE water velocity at every depth; no added mass, slamming or wave-making
terms; pieces are integrated on their flat corners, so a wave shorter than a triangle is seen only at the corners.

Numeric policy (as oracle/drag.py): every operation binary32, rounded once, in the order written, no contraction; divisions
and square roots IEEE.  The CUDA kernels (ocean_hull.cu, ocean_bodies.cu, -fmad=false) reproduce this bit for bit.
"""
from __future__ import annotations

import numpy as np

from . import bodies as bo
from . import buoyancy as bu
from . import drag as dr
from . import surface as su
from . import wake_coupling as wc
from .sampling import F

MESH = np.dtype([("first_vertex", np.int32), ("num_vertices", np.int32), ("first_triangle", np.int32), ("num_triangles", np.int32),
                 ("normal_drag", np.float32), ("tangential_drag", np.float32)])                                 # 24 B
BODY = np.dtype([("transform", np.float32, 12), ("mesh", np.int32), ("reserved", np.int32)])                    # 56 B
FLOATING = np.dtype([("mass", np.float32), ("inertia", np.float32, 3), ("mesh", np.int32)])                     # 20 B
LANES = bu.LANES


def volumes(meshes, vertices, triangles) -> np.ndarray:
    """The signed volume of each mesh, sum of p0 . (p2 x p1) / 6 over its triangles in binary64, as float32 [M]: positive for a
    closed mesh in Godot's winding, negative for one wound the other way (ocean_hull_set_meshes' volumes)."""
    meshes = np.ascontiguousarray(meshes, MESH).reshape(-1)
    v = np.asarray(vertices, np.float64).reshape(-1, 3)
    t = np.asarray(triangles, np.int64).reshape(-1, 3)
    out = np.zeros(len(meshes), np.float32)
    for m, h in enumerate(meshes):
        tri = t[h["first_triangle"]:h["first_triangle"] + h["num_triangles"]] + int(h["first_vertex"])
        a, b, c = v[tri[:, 0]], v[tri[:, 1]], v[tri[:, 2]]
        out[m] = np.float32(np.sum(np.einsum("ij,ij->i", a, np.cross(c, b))) / 6.0)
    return out


def world_vertices(bodies, meshes, vertices):
    """The world vertices in body-major order: (body index [n], j [n], r [n][3], wy [n], Q [n][2]), float32."""
    counts = meshes["num_vertices"].astype(np.int64)[bodies["mesh"]]
    body = np.repeat(np.arange(len(bodies)), counts)
    j = np.arange(int(counts.sum()), dtype=np.int64) - np.repeat(np.cumsum(counts) - counts, counts)
    p = np.asarray(vertices, np.float32).reshape(-1, 3)[meshes["first_vertex"].astype(np.int64)[bodies["mesh"]][body] + j]
    T = bodies["transform"].astype(np.float32)[body].reshape(-1, 3, 4)
    r = np.empty((len(body), 3), np.float32)
    with np.errstate(all="ignore"):
        for k in range(3):
            r[:, k] = (T[:, k, 0] * p[:, 0] + T[:, k, 1] * p[:, 1]) + T[:, k, 2] * p[:, 2]
        wy = r[:, 1] + T[:, 1, 3]
        Q = np.stack([r[:, 0] + T[:, 0, 3], r[:, 2] + T[:, 2, 3]], 1)
    return body, j, r, wy, Q


def _clip(ra, da, ua, rb, db, ub):
    t = da / (da - db)
    return ra + t[:, None] * (rb - ra), np.zeros_like(da), ua + t[:, None] * (ub - ua)


def _piece(r0, d0, u0, r1, d1, u1, r2, d2, u2, lin, ang, cn, ct, cnt):
    """One piece's sums per row: float32 [n][17] (f, tq, q, g, gt, area, speed; speed NaN where the piece has no drag)."""
    a = F(0.5) * dr.cross(r2 - r0, r1 - r0)
    sd = (d0 + d1) + d2
    sdd = (d0 * d0 + d1 * d1) + d2 * d2
    m = ((d0[:, None] * r0 + d1[:, None] * r1) + d2[:, None] * r2) + sd[:, None] * ((r0 + r1) + r2)
    my = m[:, 1] + F(0.5) * (sdd + sd * sd)
    f = a * sd[:, None]
    tq = dr.cross(m, a)
    q = np.stack([a[:, 1] * m[:, 0], a[:, 1] * my, a[:, 1] * m[:, 2]], 1)
    A = np.sqrt((a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1]) + a[:, 2] * a[:, 2])
    e0, e1, e2 = (u - (lin + dr.cross(ang, r)) for u, r in ((u0, r0), (u1, r1), (u2, r2)))
    dc = ((e0 + e1) + e2) / F(3.0)
    n = a / A[:, None]
    dn = (dc[:, 0] * n[:, 0] + dc[:, 1] * n[:, 1]) + dc[:, 2] * n[:, 2]
    dt = dc - dn[:, None] * n
    st = np.sqrt((dt[:, 0] * dt[:, 0] + dt[:, 1] * dt[:, 1]) + dt[:, 2] * dt[:, 2])
    kt = (ct * A) * st
    kn = np.where(dn < F(0.0), (cn * A) * (dn * dn), F(0.0)).astype(np.float32)
    G = kt[:, None] * dt - kn[:, None] * n
    rc = ((r0 + r1) + r2) / F(3.0)
    gt = dr.cross(rc, G)
    speed = np.sqrt((dc[:, 0] * dc[:, 0] + dc[:, 1] * dc[:, 1]) + dc[:, 2] * dc[:, 2])
    has = A > F(0.0)
    drag = np.concatenate([G, gt, (cnt * A)[:, None]], 1)
    drag[~has] = F(0.0)
    speed = np.where(has, speed, F(np.nan)).astype(np.float32)
    return np.concatenate([f, tq, q, drag, speed[:, None]], 1).astype(np.float32)


def triangle_sums(r, d, u, lin, ang, cn, ct):
    """The sums of each triangle, corners r [n][3][3], d [n][3], u [n][3][3] in winding order, the body's velocity lin, ang
    [n][3] and the mesh's C_n, C_t [n]: (float32 [n][17] as _piece's, kept [n] bool: False where a NaN depth drops the
    triangle or no corner is wet)."""
    r, d, u = (np.asarray(x, np.float32) for x in (r, d, u))
    lin, ang = np.asarray(lin, np.float32), np.asarray(ang, np.float32)
    cn, ct = np.asarray(cn, np.float32), np.asarray(ct, np.float32)
    cnt = cn + ct
    with np.errstate(all="ignore"):
        wet = d > F(0.0)
        count = wet.sum(1)
        kept = ~np.isnan(d).any(1) & (count > 0)
        shift = np.where(((count == 1) & wet[:, 1]) | ((count == 2) & ~wet[:, 0]), 1,
                         np.where(((count == 1) & wet[:, 2]) | ((count == 2) & ~wet[:, 1]), 2, 0))
        idx = (np.arange(3)[None, :] + shift[:, None]) % 3
        rows = np.arange(len(d))[:, None]
        r, d, u = r[rows, idx], d[rows, idx], u[rows, idx]
        c = [(r[:, k], d[:, k], u[:, k]) for k in range(3)]
        x01, x02 = _clip(*c[0], *c[1]), _clip(*c[0], *c[2])
        x12, x20 = _clip(*c[1], *c[2]), _clip(*c[0], *c[2])

        def pick(*choices):
            """Per row the corner of the first choice whose mask holds: choices are (mask, corner) pairs."""
            out = [np.array(v, copy=True) for v in choices[-1][1]]
            for mask, corner in reversed(choices[:-1]):
                for o, v in zip(out, corner):
                    o[mask] = v[mask]
            return out

        three, one = count == 3, count == 1
        b1 = pick((three, c[1]), (one, x01), (np.ones_like(one), c[1]))
        b2 = pick((three, c[2]), (one, x02), (np.ones_like(one), x12))
        p1 = _piece(*c[0], *b1, *b2, lin, ang, cn, ct, cnt)
        p2 = _piece(*c[0], *x12, *x20, lin, ang, cn, ct, cnt)
        sums = F(0.0) + p1[:, :16]
        two = count == 2
        sums[two] = sums[two] + p2[two, :16]
        speed = np.where(two, np.fmax(p1[:, 16], p2[:, 16]), p1[:, 16])
    return np.concatenate([sums, speed[:, None]], 1).astype(np.float32), kept


def hull_forces(displacement, normal, velocity, bodies, velocities, meshes, vertices, triangles, map_scales, density=1025.0,
                tolerance=1e-3, max_iterations=8, return_samples=False, wake: wc.Coupling | None = None):
    """displacement, normal, velocity: [C][N][N][4] float16; bodies: BODY [B]; velocities: drag.VELOCITY [B]; meshes: MESH [M];
    vertices [V][3] float32; triangles [T][3] int32; map_scales [C][4] float32.  Returns (buoyancy.RESULT [B], drag.RESULT [B]),
    and with return_samples also the surface records of the world vertices."""
    bodies = np.ascontiguousarray(bodies, BODY).reshape(-1)
    velocities = np.ascontiguousarray(velocities, dr.VELOCITY).reshape(-1)
    meshes = np.ascontiguousarray(meshes, MESH).reshape(-1)
    tris = np.asarray(triangles, np.int64).reshape(-1, 3)
    B = len(bodies)
    body, j, r, wy, Q = world_vertices(bodies, meshes, vertices)
    if len(body):
        with np.errstate(all="ignore"):
            samples = wc.query_surface(displacement, normal, Q, map_scales, tolerance, max_iterations, wake)
            d = samples["displacement"][:, 1] - wy
            u = dr.water_velocity(velocity, np.stack([samples["source_x"], samples["source_z"]], 1), map_scales)
            if wc.live(wake):
                u[:, 1] = u[:, 1] + wc.vertical_velocity(Q, wake, wake.cell_size)
    else:
        samples, d, u = np.zeros(0, su.RECORD), np.zeros(0, np.float32), np.zeros((0, 3), np.float32)
    # the triangles, body-major: corner k of triangle tj of body b is world vertex base[b] + tris[first_triangle + tj][k]
    vcounts = meshes["num_vertices"].astype(np.int64)[bodies["mesh"]]
    base = np.cumsum(vcounts) - vcounts
    tcounts = meshes["num_triangles"].astype(np.int64)[bodies["mesh"]]
    tbody = np.repeat(np.arange(B), tcounts)
    tj = np.arange(int(tcounts.sum()), dtype=np.int64) - np.repeat(np.cumsum(tcounts) - tcounts, tcounts)
    mesh = meshes[bodies["mesh"][tbody]]
    corner = tris[mesh["first_triangle"].astype(np.int64) + tj] + base[tbody][:, None]
    vel = velocities[tbody]
    sums, kept = triangle_sums(r[corner], d[corner], u[corner], vel["linear"], vel["angular"], mesh["normal_drag"], mesh["tangential_drag"])
    tb, tj, sums = tbody[kept], tj[kept], sums[kept]
    S = bu.lane_tree_sum(sums[:, :16], tb, tj, B) if len(tb) else np.zeros((B, 16), np.float32)
    speed = np.zeros(B, np.float32)
    np.fmax.at(speed, tb, sums[:, 16])
    rho_g = F(density) * bu.G
    half_rho = F(0.5) * F(density)
    hyd = np.zeros(B, bu.RESULT)
    drg = np.zeros(B, dr.RESULT)
    with np.errstate(all="ignore"):
        fk = S[:, 0:3] / F(3.0)
        hyd["force"] = -(rho_g * fk)
        hyd["torque"] = -(rho_g * (S[:, 3:6] / F(12.0)))
        V = -fk[:, 1]
        hyd["submerged_volume"] = V
        pos = V > F(0.0)
        hyd["center_offset"][pos] = (-(S[pos, 6:9] / F(12.0))) / V[pos, None]
        drg["force"] = half_rho * S[:, 9:12]
        drg["torque"] = half_rho * S[:, 12:15]
    drg["wetted_drag_area"] = S[:, 15]
    drg["max_relative_speed"] = speed
    max_res = np.full(B, np.nan, np.float32)
    np.fmax.at(max_res, body, samples["residual"])
    hyd["max_residual"] = max_res
    missed = (~(samples["residual"] <= F(tolerance))).astype(np.float64)
    hyd["unconverged"] = np.bincount(body, weights=missed, minlength=B).astype(np.uint32)
    empty = vcounts == 0
    hyd[empty] = np.zeros(1, bu.RESULT)
    drg[empty] = np.zeros(1, dr.RESULT)
    return (hyd, drg, samples) if return_samples else (hyd, drg)


def radius2(bodies, meshes, vertices) -> np.ndarray:
    """r2 of bodies.py over each body's mesh vertices: float32 [B]."""
    bodies = np.ascontiguousarray(bodies, FLOATING).reshape(-1)
    meshes = np.ascontiguousarray(meshes, MESH).reshape(-1)
    p = np.asarray(vertices, np.float32).reshape(-1, 3)
    out = np.zeros(len(bodies), np.float32)
    with np.errstate(all="ignore"):
        for b, m in enumerate(bodies["mesh"]):
            q = p[meshes["first_vertex"][m]:meshes["first_vertex"][m] + meshes["num_vertices"][m]]
            if len(q):
                out[b] = np.fmax.reduce(np.concatenate([[F(0.0)], (q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]]))
    return out


def pose(bodies, states):
    """The hull-forces inputs of one sub-step: (BODY [B], drag.VELOCITY [B])."""
    bodies = np.ascontiguousarray(bodies, FLOATING).reshape(-1)
    table = np.zeros(len(bodies), BODY)
    table["transform"] = bo.transforms(states)
    table["mesh"] = bodies["mesh"]
    _, vel = bo.pose(np.zeros(len(bodies), bo.BODY), states)
    return table, vel


def simulate(displacement, normal, velocity, bodies, states, meshes, vertices, triangles, map_scales, density=1025.0, dt=1.0 / 60.0,
             substeps=1, tolerance=1e-3, max_iterations=8, wake: wc.Coupling | None = None):
    """bodies.simulate on hull meshes: bodies FLOATING [B], states bodies.STATE [B].  Every sub-step takes hull_forces at the
    pose it starts from, then bodies.step with r2 = radius2.  Returns (STATE [B], buoyancy.RESULT [B], drag.RESULT [B],
    float32 [B][12])."""
    bodies = np.ascontiguousarray(bodies, FLOATING).reshape(-1)
    meshes = np.ascontiguousarray(meshes, MESH).reshape(-1)
    s = np.array(states, bo.STATE, copy=True).reshape(-1)
    h = F(dt) / F(substeps)
    r2 = radius2(bodies, meshes, vertices)
    rows = np.zeros(len(bodies), bo.BODY)
    rows["mass"], rows["inertia"] = bodies["mass"], bodies["inertia"]
    hyd, drg = np.zeros(len(bodies), bu.RESULT), np.zeros(len(bodies), dr.RESULT)
    for _ in range(substeps):
        table, vel = pose(bodies, s)
        with np.errstate(all="ignore"):
            hyd, drg = hull_forces(displacement, normal, velocity, table, vel, meshes, vertices, triangles, map_scales, density, tolerance,
                                   max_iterations, wake=wake)
        s = bo.step(rows, s, r2, hyd, drg, density, h)
    return s, hyd, drg, bo.transforms(s)
