"""CPU specification of the drifter op (ocean_drift): Lagrangian labels that drift with the Stokes drift, a current and
windage, rendered on the displaced surface as MultiMesh instances.

TEST INFRASTRUCTURE ONLY -- the product path (godotoceanwaves_b200/csrc) never imports or calls this module.

DRIFT   (dt > 0) us = sum over the cascades in order of (s s) u_s,i from +0 (s = (double)map_scales[i][2], u_s,i the
        cascade's Stokes moments, oracle/sea_state.py), then in binary64, each operation rounded once:
          u = ((stokes_scale us) + current) + (windage wind);  x = x + dt u.x;  z = z + dt u.z
          yaw = (float)((double)yaw + dt (double)yaw_rate)
WRAP    (dt > 0, WRAP) r = x - x0;  x = x0 + (r - W floor(r / W));  z likewise with (z0, D)
RENDER  D, g = oracle/sampling.py's sample_maps at ((float)x, (float)z);  X.x = (float)(x + D.x), X.z = (float)(z + D.z);
        with the wake: (hw, hgx, hgz) = oracle/wake.py's sample of h at (X.x, X.z), y = (double)D.y + hw (binary64),
        g.x += hgx, g.y += hgz (binary32);  X.y = (float)(y + offset);
        normalize(v) = v / sqrt((v.x v.x + v.y v.y) + v.z v.z), binary32;  n = normalize(-g.x, 1, -g.y);
        ny = normalize(0 + tilt (n.x - 0), 1 + tilt (n.y - 1), 0 + tilt (n.z - 0));  (sn, cs) = DETMATH sincos(yaw);
        f.n = (sn ny.x + 0 ny.y) + cs ny.z;  nz = normalize(sn - f.n ny.x, 0 - f.n ny.y, cs - f.n ny.z);  nx = ny x nz
        (x = y.y z.z - y.z z.y, y = y.z z.x - y.x z.z, z = y.x z.y - y.y z.x);  instance = 12 floats, 3 x 4 row-major
        [nx | ny | nz | X] with each basis component times scale.
"""
from __future__ import annotations

import numpy as np

from . import pyoracle as po
from . import wake as wk
from .sampling import sample_maps

F = np.float32
DRIFTER = np.dtype([("x", np.float64), ("z", np.float64), ("yaw", np.float32), ("yaw_rate", np.float32), ("windage", np.float32),
                    ("tilt", np.float32), ("offset", np.float32), ("scale", np.float32)])       # struct ocean_drifter
PARAMS = np.dtype([("current", np.float32, 2), ("wind", np.float32, 2), ("stokes_scale", np.float32), ("flags", np.uint32),
                   ("box", np.float64, 4)])                                                     # struct ocean_drift_params
WRAP, READ_WAKE = 1, 2


def stokes_total(moments, map_scales):
    """(us.x, us.z): sum over the cascades in order of (s s) u_s,i from +0."""
    sc = np.asarray(map_scales, np.float32).reshape(-1, 4)
    ux = uz = 0.0
    for m, s in zip(moments, sc[:, 2].astype(np.float64)):
        ux = ux + (s * s) * float(m[8])
        uz = uz + (s * s) * float(m[9])
    return ux, uz


def advance(drifters: np.ndarray, dt: float, params, us) -> np.ndarray:
    """DRIFT and WRAP of a DRIFTER array (a new array; unchanged when dt == 0)."""
    d = np.array(drifters, DRIFTER, copy=True).reshape(-1)
    p = np.asarray(params, PARAMS).reshape(())
    if not dt > 0.0:
        return d
    ss = float(p["stokes_scale"])
    wg = d["windage"].astype(np.float64)
    with np.errstate(all="ignore"):
        ux = ((ss * us[0]) + float(p["current"][0])) + wg * float(p["wind"][0])
        uz = ((ss * us[1]) + float(p["current"][1])) + wg * float(p["wind"][1])
        d["x"] = d["x"] + dt * ux
        d["z"] = d["z"] + dt * uz
        d["yaw"] = (d["yaw"].astype(np.float64) + dt * d["yaw_rate"].astype(np.float64)).astype(np.float32)
        if int(p["flags"]) & WRAP:
            x0, z0, W, D = (float(v) for v in p["box"])
            rx = d["x"] - x0
            rz = d["z"] - z0
            d["x"] = x0 + (rx - W * np.floor(rx / W))
            d["z"] = z0 + (rz - D * np.floor(rz / D))
    return d


def _normalize(x, y, z):
    l = np.sqrt((x * x + y * y) + z * z)
    return x / l, y / l, z / l


def render(drifters: np.ndarray, displacement: np.ndarray, normal: np.ndarray, map_scales, wake=None) -> np.ndarray:
    """[n][12] float32 instances.  displacement, normal: [C][N][N][4] float16 of the cascades used; wake = (h, cell_size,
    origin) of the layer the render reads, or None."""
    d = np.asarray(drifters, DRIFTER).reshape(-1)
    with np.errstate(all="ignore"):
        P = np.stack([d["x"].astype(np.float32), d["z"].astype(np.float32)], axis=-1)
        D, g = sample_maps(displacement, normal, P, map_scales)
        X = (d["x"] + D[:, 0].astype(np.float64)).astype(np.float32)
        Z = (d["z"] + D[:, 2].astype(np.float64)).astype(np.float32)
        y = D[:, 1].astype(np.float64)
        gx, gz = g[:, 0].copy(), g[:, 1].copy()
        if wake is not None:
            h, cell, origin = wake
            s = wk.sample(h, cell, origin, np.stack([X, Z], axis=-1))
            y = y + s[:, 0].astype(np.float64)
            gx = gx + s[:, 1]
            gz = gz + s[:, 2]
        Y = (y + d["offset"].astype(np.float64)).astype(np.float32)
        nx, ny, nz = _normalize(-gx, np.ones_like(gx), -gz)
        t = d["tilt"]
        yx, yy, yz = _normalize(F(0.0) + t * (nx - F(0.0)), F(1.0) + t * (ny - F(1.0)), F(0.0) + t * (nz - F(0.0)))
        sc = po.math_batch(po.MATH_SINCOS, d["yaw"])
        sn, cs = sc[:, 0], sc[:, 1]
        fn = (sn * yx + F(0.0) * yy) + cs * yz
        zx, zy, zz = _normalize(sn - fn * yx, F(0.0) - fn * yy, cs - fn * yz)
        xx = yy * zz - yz * zy
        xy = yz * zx - yx * zz
        xz = yx * zy - yy * zx
        s = d["scale"]
        out = np.stack([xx * s, yx * s, zx * s, X, xy * s, yy * s, zy * s, Y, xz * s, yz * s, zz * s, Z], axis=-1)
    return out.astype(np.float32)


def drift(drifters, dt: float, params, moments, displacement, normal, map_scales, wake=None, render_instances=True):
    """One ocean_drift call: (new drifters, instances or None).  moments: the MOMENTS of each cascade used (oracle/sea_state.py);
    wake as for render(), read only with READ_WAKE."""
    p = np.asarray(params, PARAMS).reshape(())
    d = advance(drifters, dt, p, stokes_total(moments, map_scales))
    if not render_instances:
        return d, None
    return d, render(d, displacement, normal, map_scales, wake if int(p["flags"]) & READ_WAKE else None)
