"""CPU tests of the wake readers' specification (oracle/wake_readers.py; include/ocean.h, "Wake layer", Readers): the ray cast
and spray reading the wake layer.  The `wake` keywords of oracle/raycast.py, spray.py and spray_particles.py change nothing
when absent or zero; the coupled ray cast against a binary64 bilinear model of e (hits on the surface, no earlier crossing);
the slab's soundness over random e; the spray spawn test against a binary64 evaluation; and the ABI's argument checks that
run without a device."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest

from oracle import raycast as rc
from oracle import spray as sp
from oracle import spray_particles as spp
from oracle import wake as wk
from oracle import wake_coupling as wc
from oracle import wake_readers as wr

f32 = np.float32
INVALID = 1                                                       # OCEAN_ERR_INVALID_ARGUMENT


def _maps(rng, C=2, N=32, amp=0.3):
    d = np.zeros((C, N, N, 4), np.float16)
    nm = np.zeros((C, N, N, 4), np.float16)
    if amp:
        d[..., :3] = (amp * rng.standard_normal((C, N, N, 3))).astype(np.float16)
        nm[..., :2] = (0.2 * rng.standard_normal((C, N, N, 2))).astype(np.float16)
        nm[..., 3] = rng.uniform(0, 1.2, (C, N, N)).astype(np.float16)
    scales = np.zeros((C, 4), np.float32)
    for c in range(C):
        scales[c] = (1.0 / (40.0 + 23.0 * c), 1.0 / (40.0 + 23.0 * c), 1.0, 1.0)
    return d, nm, scales


def _coupling(e, origin, cell):
    cp = wc.Coupling(e.shape[0], cell)
    cp.e = np.asarray(e, np.float32)
    cp.e_old = cp.e.copy()
    cp.origin_e = cp.origin_old = origin
    cp.T = f32(0.1)
    cp.primed = True
    return cp


def _rays(rng, n, centre, extent, y=(2.0, 6.0)):
    r = np.zeros(n, rc.RAY)
    r["origin"][:, 0] = rng.uniform(centre[0] - extent, centre[0] + extent, n)
    r["origin"][:, 2] = rng.uniform(centre[1] - extent, centre[1] + extent, n)
    r["origin"][:, 1] = rng.uniform(*y, n)
    d = rng.standard_normal((n, 3))
    d[:, 1] = -np.abs(d[:, 1]) - 0.05
    r["direction"] = d / np.linalg.norm(d, axis=1, keepdims=True)
    r["t_max"] = 60.0
    return r


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _hump(n, cell, origin, centre, radius, height):
    x0, z0 = (float(v) for v in wk.world_origin(origin, cell))
    c = (np.arange(n) + 0.5) * cell
    X, Z = np.meshgrid(x0 + c, z0 + c)
    return (height * np.exp(-((X - centre[0]) ** 2 + (Z - centre[1]) ** 2) / radius ** 2)).astype(np.float32)


def _sample64(f, cell, origin, x, z):
    """binary64 bilinear sample of f ([N][N]) and of its central differences, 0 outside the window and at cells outside it."""
    f = np.asarray(f, np.float64)
    n = f.shape[0]
    dx = float(f32(cell))
    x0, z0 = (float(v) for v in wk.world_origin(origin, cell))
    p = np.zeros((n + 4, n + 4))
    p[2:-2, 2:-2] = f
    gx = np.zeros_like(p)
    gz = np.zeros_like(p)
    gx[2:-2, 2:-2] = (p[2:-2, 3:-1] - p[2:-2, 1:-3]) / (2 * dx)
    gz[2:-2, 2:-2] = (p[3:-1, 2:-2] - p[1:-3, 2:-2]) / (2 * dx)
    x = np.asarray(x, np.float64)
    z = np.asarray(z, np.float64)
    out = np.zeros((len(x), 3))
    inside = (x >= x0) & (x < x0 + n * dx) & (z >= z0) & (z < z0 + n * dx)
    u = (x[inside] - x0) / dx - 0.5
    v = (z[inside] - z0) / dx - 0.5
    i, j = np.floor(u).astype(int), np.floor(v).astype(int)
    a, b = u - i, v - j
    for m, g in enumerate((p, gx, gz)):
        def at(ii, jj):
            return g[jj + 2, ii + 2]
        out[inside, m] = (1 - b) * ((1 - a) * at(i, j) + a * at(i + 1, j)) + b * ((1 - a) * at(i, j + 1) + a * at(i + 1, j + 1))
    return out


# ---- off and zero change nothing ----

def test_no_wake_is_byte_identical():
    rng = np.random.default_rng(1)
    d, nm, sc = _maps(rng)
    rays = _rays(rng, 64, (0, 0), 30)
    ref, tr = rc.raycast(d, nm, rays, sc, trace=True)
    for cp, read in ((None, True), (wc.Coupling(64, 0.5), True), (_coupling(np.ones((64, 64)), (0, 0), 0.5), False)):
        out, tr2 = wr.raycast(d, nm, rays, sc, trace=True, coupling=cp, read=read)
        assert np.array_equal(_bytes(out), _bytes(ref)) and np.array_equal(_bytes(tr2), _bytes(tr))
    pts = sp.spray_grid(400, 8 * np.eye(3, 4))
    assert np.array_equal(_bytes(wr.spray_candidates(nm, pts, sc, (20, 8.5, 20))), _bytes(sp.spray_candidates(nm, pts, sc, (20, 8.5, 20))))


def test_restated_ops_without_a_wake_are_the_originals_bytes():
    """The march, slab, spawn test and particle process restated in wake_readers.py give raycast.py's, spray.py's and
    spray_particles.py's bytes when no wake is read."""
    rng = np.random.default_rng(4)
    d, nm, sc = _maps(rng)
    rays = np.concatenate([_rays(rng, 96, (0, 0), 30), _rays(rng, 32, (0, 0), 30, y=(-3.0, 0.5))])
    rays["direction"][-32:, 1] *= -1
    rays["t_max"][::7] = np.inf
    rays["origin"][5, 0] = np.nan
    for iters in (8, 0):
        ref, tr = rc.raycast(d, nm, rays, sc, 0.5, 64, 1e-3, iters, trace=True)
        out, tr2 = wr._raycast(d, nm, rays, sc, 0.5, 64, 1e-3, iters, True, None)
        assert np.array_equal(_bytes(out), _bytes(ref)) and np.array_equal(_bytes(tr2), _bytes(tr))
    lo, hi, _, _, rho = rc.slab(d, sc, f32(1e-3))
    assert (lo, hi, rho) == wr.slab(d, sc, f32(1e-3))
    pts = sp.spray_grid(1600, 6 * np.eye(3, 4))
    assert np.array_equal(_bytes(wr._spray_candidates(nm, pts, sc, (20, 8.5, 20), None)),
                          _bytes(sp.spray_candidates(nm, pts, sc, (20, 8.5, 20))))
    em = spp.default_emitter()
    em["amount"] = em["num_particles"] = 1024
    s1 = s2 = np.zeros(1024, spp.PARTICLE)
    for k in range(5):
        s1, i1, c1 = spp.frame(s1, em, 0.5 * k, 0.5 * k + 0.5, d, nm, sc, 700)
        s2, i2, c2 = wr._frame(s2, em, 0.5 * k, 0.5 * k + 0.5, d, nm, sc, 700, None)
        assert c1 == c2 and np.array_equal(_bytes(i1), _bytes(i2)) and np.array_equal(_bytes(s1), _bytes(s2))


def test_zero_wake_equals_uncoupled_field_by_field():
    rng = np.random.default_rng(2)
    d, nm, sc = _maps(rng)
    n, cell = 64, 0.5
    rays = _rays(rng, 96, (0, 0), 20)
    ref = rc.raycast(d, nm, rays, sc)
    out = wr.raycast(d, nm, rays, sc, coupling=_coupling(np.zeros((n, n)), (-32, -32), cell))
    for f in rc.HIT.names:
        assert np.array_equal(out[f], ref[f], equal_nan=out[f].dtype.kind == "f"), f
    layer = wk.Layer(np.array((n, 8, cell, 0.1, 1.0), wk.PARAMS))
    layer.origin = (-32, -32)
    layer.foam = np.zeros((n, n), np.float32)
    pts = sp.spray_grid(900, 6 * np.eye(3, 4))
    a = sp.spray_candidates(nm, pts, sc, (20, 8.5, 20))
    for foam_on in (False, True):
        b = wr.spray_candidates(nm, pts, sc, (20, 8.5, 20), layer=layer, foam_on=foam_on)
        assert len(a) == len(b) > 0
        for f in sp.RECORD.names:
            assert np.array_equal(a[f], b[f]), f
    em = spp.default_emitter()
    em["amount"] = em["num_particles"] = 1024
    st = np.zeros(1024, spp.PARTICLE)
    s1, s2 = st, st
    for k in range(4):
        s1, i1, c1 = spp.frame(s1, em, 0.5 * k, 0.5 * k + 0.5, d, nm, sc)
        s2, i2, c2 = wr.frame(s2, em, 0.5 * k, 0.5 * k + 0.5, d, nm, sc, layer=layer, foam_on=True)
        assert c1 == c2 and np.array_equal(i1, i2)
        for f in spp.PARTICLE.names:
            assert np.array_equal(s1[f], s2[f], equal_nan=s1[f].dtype.kind == "f"), f


# ---- the coupled ray cast against a binary64 model of e ----

def test_raycast_hits_the_wake_hump_first():
    n, cell, origin = 128, 0.5, (-64, -64)
    e = _hump(n, cell, origin, (3.0, -2.0), 8.0, 1.5)
    d, nm, sc = _maps(None, amp=0)
    rng = np.random.default_rng(3)
    rays = _rays(rng, 400, (3.0, -2.0), 25, y=(1.0, 5.0))
    tol, step = 1e-3, 0.5
    out = wr.raycast(d, nm, rays, sc, step=step, tolerance=tol, coupling=_coupling(e, origin, cell))
    hit = (out["status"] == rc.HIT_FROM_ABOVE)
    assert hit.sum() > 100
    assert not (out["status"] == rc.HIT_FROM_BELOW).any()
    pos = out["position"].astype(np.float64)
    s = _sample64(e, cell, origin, pos[:, 0], pos[:, 2])
    conv = hit & (np.abs(out["gap"]) <= tol)
    assert conv.sum() == hit.sum()                                 # a smooth hump: every crossing resolves
    assert np.all(np.abs(pos[conv, 1] - s[conv, 0]) <= tol + 4e-6)
    # the record carries the coupled height and slopes; gap == position.y - displacement[1]
    assert np.all(np.abs(out["displacement"][hit, 1] - s[hit, 0]) <= 4e-6)
    assert np.all(np.abs(out["gradient_foam"][hit, 0] - s[hit, 1]) <= 4e-6)
    assert np.all(np.abs(out["gradient_foam"][hit, 1] - s[hit, 2]) <= 4e-6)
    assert np.array_equal(out["gap"][hit], out["position"][hit, 1] - out["displacement"][hit, 1])
    # a dense binary64 scan (step / 16 of horizontal travel) finds no earlier crossing
    for k in np.flatnonzero(hit):
        o = rays["origin"][k].astype(np.float64)
        dv = rays["direction"][k].astype(np.float64)
        hs = np.hypot(dv[0], dv[2])
        t = np.arange(0.0, float(out["t"][k]), step / 16 / hs)
        p = o[None, :] + t[:, None] * dv[None, :]
        g = p[:, 1] - _sample64(e, cell, origin, p[:, 0], p[:, 2])[:, 0]
        assert np.all(g > -(tol + 1e-5)), k


def test_horizontal_ray_below_the_crest_misses_uncoupled_and_hits_coupled():
    n, cell, origin = 128, 0.5, (-64, -64)
    e = _hump(n, cell, origin, (0.0, 0.0), 6.0, 0.5)
    d, nm, sc = _maps(None, amp=0)
    r = np.zeros(1, rc.RAY)
    r["origin"] = (-25.0, 0.2, 0.3)
    r["direction"] = (1.0, 0.0, 0.0)
    r["t_max"] = 60.0
    assert rc.raycast(d, nm, r, sc)["status"][0] == rc.MISS
    out = wr.raycast(d, nm, r, sc, coupling=_coupling(e, origin, cell))
    assert out["status"][0] == rc.HIT_FROM_ABOVE
    assert abs(out["gap"][0]) <= 1e-3 and out["position"][0, 1] == f32(0.2)
    x = float(out["position"][0, 0])
    assert -25.0 < x < 0.0 and abs(_sample64(e, cell, origin, [x], [0.3])[0, 0] - 0.2) <= 1e-3 + 1e-6


@pytest.mark.parametrize("kind", ["mixed", "negative", "positive", "signed-zero", "nan-cell"])
def test_slab_holds_every_evaluated_height(kind):
    rng = np.random.default_rng(hash(kind) % 2 ** 32)
    n, cell, origin = 64, 0.5, (-40, -20)
    d, nm, sc = _maps(rng)
    e = rng.standard_normal((n, n)).astype(np.float32) * f32(0.8)
    if kind == "negative":
        e = -np.abs(e) - f32(0.1)
    elif kind == "positive":
        e = np.abs(e) + f32(0.1)
    elif kind == "signed-zero":
        e = np.where(rng.random((n, n)) < 0.5, f32(0.0), f32(-0.0)).astype(np.float32)
    elif kind == "nan-cell":
        e[10, 12] = np.nan
    cp = _coupling(e, origin, cell)
    rays = _rays(rng, 200, (-4, 0), 20, y=(-3.0, 4.0))
    rays["direction"][::3, 1] *= -1                                  # some from below
    out, tr = wr.raycast(d, nm, rays, sc, trace=True, coupling=cp)
    lo, hi, _ = wr.slab(d, sc, f32(1e-3), wr.bounds(e))
    layers = d.astype(np.float32)
    with np.errstate(all="ignore"):
        eta = rc._height(layers, sc, tr["source_x"], tr["source_z"]) + wr.sample(e, cell, origin, tr["position"][:, 0],
                                                                                tr["position"][:, 2], False)[:, 0]
    ok = ~np.isnan(eta)
    assert ok.sum() > 500
    assert np.all((eta[ok] >= lo) & (eta[ok] <= hi))
    assert np.array_equal(tr["gap"][ok], (tr["position"][:, 1] - eta)[ok])     # the trace carries the coupled gap
    if kind == "nan-cell":
        assert (out["status"] == rc.INVALID).any() or not (~ok).any()


# ---- spray against a binary64 evaluation of the spawn inequalities ----

def test_spray_active_set_matches_binary64():
    n, cell, origin = 128, 0.25, (-64, -64)
    rng = np.random.default_rng(5)
    layer = wk.Layer(np.array((n, 8, cell, 0.1, 1.0), wk.PARAMS))
    layer.origin = origin
    layer.h = _hump(n, cell, origin, (1.0, 2.0), 4.0, 0.6) - _hump(n, cell, origin, (-6.0, -3.0), 3.0, 0.4)
    F = np.zeros((n, n), np.float32)
    F[40:90, 30:100] = rng.uniform(0.6, 1.0, (50, 70)).astype(np.float32)
    layer.foam = F
    d, nm, sc = _maps(None, amp=0)
    pts = rng.uniform(-18, 18, (20000, 2)).astype(np.float32)
    got = wr.spray_candidates(nm, pts, sc, (20, 8.5, 20), layer=layer, foam_on=True)
    s = _sample64(layer.h, cell, origin, pts[:, 0], pts[:, 1])
    fw = _sample64(F, cell, origin, pts[:, 0], pts[:, 1])[:, 0]
    ny = 1.0 / np.sqrt(s[:, 1] ** 2 + 1.0 + s[:, 2] ** 2)
    ny_lo = 0.92 - (0.99 - 0.92) / 3.0                              # normal_factor >= 0
    active = (ny >= ny_lo) & (fw > 0.9)
    clear = (np.abs(ny - ny_lo) > 1e-5) & (np.abs(fw - 0.9) > 1e-5)
    mask = np.zeros(len(pts), bool)
    mask[got["index"]] = True
    assert active[clear].sum() > 200 and (~active[clear]).sum() > 2000
    assert np.array_equal(mask[clear], active[clear])
    assert np.all(np.abs(got["foam"].astype(np.float64) - fw[got["index"]]) <= 4e-6)
    # foam off: F reads +0, so nothing is active on zero maps
    assert len(wr.spray_candidates(nm, pts, sc, (20, 8.5, 20), layer=layer, foam_on=False)) == 0


def test_spray_particle_height_follows_h():
    n, cell, origin = 128, 0.5, (-64, -64)
    layer = wk.Layer(np.array((n, 8, cell, 0.1, 1.0), wk.PARAMS))
    layer.origin = origin
    layer.h = _hump(n, cell, origin, (0.0, 0.0), 10.0, 0.7)
    layer.foam = np.ones((n, n), np.float32)
    d, nm, sc = _maps(None, amp=0)
    em = spp.default_emitter()
    em["amount"] = em["num_particles"] = 1024
    em["emission_transform"] = (1.5 * np.eye(3, 4)).reshape(12)
    a = b = np.zeros(1024, spp.PARTICLE)
    live = 0
    for k in range(6):
        a, _, _ = wr.frame(a, em, 0.5 * k, 0.5 * k + 0.5, d, nm, sc, layer=layer, foam_on=True)
        b, _, _ = wr.frame(b, em, 0.5 * k, 0.5 * k + 0.5, d, nm, sc, layer=wk.Layer(layer.params), foam_on=False)
        on = ((a["flags"] & spp.ACTIVE) != 0) & (a["userdata3"][:, 3] != 0)
        live += on.sum()
        sx, sz = a["userdata1"][on, 0], a["userdata1"][on, 2]
        hw = _sample64(layer.h, cell, origin, sx, sz)[:, 0]
        # the same particles without the wake's height (flat h = 0, F = 0 after the spawn: compare y only where both are live)
        both = on & ((b["flags"] & spp.ACTIVE) != 0) & (b["userdata3"][:, 3] != 0)
        if both.any():
            dy = a["transform"][both, 7].astype(np.float64) - b["transform"][both, 7]
            assert np.all(np.abs(dy - _sample64(layer.h, cell, origin, a["userdata1"][both, 0], a["userdata1"][both, 2])[:, 0]) <= 1e-5)
        assert np.all(hw >= 0)
    assert live > 0


# ---- the ABI without a device ----

def test_set_readers_rejects_a_null_generator():
    from godotoceanwaves_b200.native import load_library
    lib = load_library()
    for readers in (0, 1, 2, 3, 4):
        assert lib.ocean_wake_set_readers(None, ctypes.c_uint32(readers)) == INVALID
        assert b"NULL" in lib.ocean_last_error()
