"""GPU tests of the hull-mesh ops (include/ocean.h, "Hull meshes"): ocean_hull_forces and ocean_simulate_hull_bodies
byte-identical to oracle/hull.py on random welded and soup meshes (shared and empty ones), with the wake coupling off and on;
host and device forms; the flat-water closed forms on maps made from a zero spectrum; NaN isolation; launch counts; invalid
calls; a 2^16-triangle hull beside 2^12 small ones; and mesh sets that are rejected or released."""
import numpy as np
import pytest
from scipy.spatial import ConvexHull

from oracle import bodies as bo
from oracle import hull as oh
from oracle import wake as wk
from oracle import wake_coupling as wc
from test_gpu_sampling import _gen
from test_gpu_wake_coupling import _flat, _init, _params, _same
from test_oracle_hull import box

pytestmark = pytest.mark.gpu

RHO = 1025.0


def _convex(rng, k=24):
    """A random convex hull, welded: (vertices [V][3] float32, triangles [T][3] in Godot's winding)."""
    pts = (rng.normal(size=(k, 3)) * rng.uniform(0.5, 2.5, 3)).astype(np.float32)
    ch = ConvexHull(pts.astype(np.float64))
    v = pts[ch.vertices]
    remap = np.full(len(pts), -1)
    remap[ch.vertices] = np.arange(len(ch.vertices))
    t = remap[ch.simplices].astype(np.int32)
    a, b, c = (v[t[:, i]].astype(np.float64) for i in range(3))
    flip = np.einsum("ij,ij->i", np.cross(c - a, b - a), a - v.mean(0)) < 0
    t[flip] = t[flip][:, [0, 2, 1]]
    return v, t


def _mesh_set(rng, n=5):
    """Welded hulls, the soup of one of them, a box, an empty mesh: (MESH [M], vertices, triangles)."""
    parts = [_convex(rng, int(rng.integers(8, 40))) for _ in range(n)]
    v0, t0 = parts[0]
    parts.append((v0[t0].reshape(-1, 3), np.arange(3 * len(t0), dtype=np.int32).reshape(-1, 3)))     # soup
    bv, bt, _ = box(3.0, 1.0, 1.5)
    parts.append((bv, bt))
    parts.append((np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32)))                            # empty
    meshes = np.zeros(len(parts), oh.MESH)
    fv = ft = 0
    for k, (v, t) in enumerate(parts):
        meshes[k] = (fv, len(v), ft, len(t), rng.uniform(0.0, 1.5), rng.uniform(0.0, 0.2))
        fv, ft = fv + len(v), ft + len(t)
    return meshes, np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


def _bodies(rng, B, meshes, span=30.0):
    q = rng.normal(size=(B, 4)).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    s = np.zeros(B, bo.STATE)
    s["orientation"] = q
    s["position"] = np.stack([rng.uniform(-span, span, B), rng.uniform(-2.0, 2.0, B), rng.uniform(-span, span, B)], 1)
    s["linear_velocity"] = rng.normal(size=(B, 3)) * 2
    s["angular_velocity"] = rng.normal(size=(B, 3)) * 0.5
    fb = np.zeros(B, oh.FLOATING)
    fb["mesh"] = rng.integers(0, len(meshes), B)
    fb["mass"] = rng.uniform(200.0, 3000.0, B)
    fb["inertia"] = rng.uniform(100.0, 2000.0, (B, 3))
    return fb, s


def _launches(g):
    return g.info().kernel_launches


@pytest.mark.parametrize("N,C,scale,maxit,wake", [(128, 2, 1.0, 8, False), (256, 4, 2.0, 8, True), (512, 8, 1.0, 0, False),
                                                  (1024, 3, 2.0, 8, False), (256, 2, 1.0, 0, True)])
def test_forces_parity_with_the_specification(N, C, scale, maxit, wake):
    gow, g, params = _gen(N, C)
    scales = np.ascontiguousarray(gow.WaveGenerator.map_scales(params), np.float32)
    scales[:, 2] *= scale                                       # twice the displacement: steeper crests to straddle
    rng = np.random.default_rng(N + C)
    meshes, v, t = _mesh_set(rng)
    vols = g.set_hull_meshes(meshes, v, t)
    np.testing.assert_allclose(vols, oh.volumes(meshes, v, t), rtol=1e-6)
    assert (vols[:-1] > 0).all() and vols[-1] == 0
    cp = None
    if wake:
        dx, n = 0.5, 128
        p = _params(n, dx, damping=0.02, sponge_cells=16)
        _init(g, p)
        L, cp = wk.Layer(p), wc.Coupling(n, dx)
        g.wake_set_coupling(True)
        src = np.zeros(3, wk.SOURCE)
        src["x"], src["z"], src["vx"], src["radius"], src["head"], src["body"] = (10.0, 20.0, 30.0), (15.0, 30.0, 40.0), 2.0, 3.0, 0.4, -1
        for _ in range(2):
            g.wake_step(1.0 / 60.0, 2, (0, 0), src)
            wc.step(L, cp, 1.0 / 60.0, 2, (0, 0), src, None)
    fb, s = _bodies(rng, 24 if N < 1024 else 10, meshes, span=30.0)
    if wake:
        s["position"][:, [0, 2]] = rng.uniform(5.0, 60.0, (len(s), 2))
    table, vel = oh.pose(fb, s)
    g.update_velocity()
    d16, n16 = g.maps_to_host(0, C)
    velocity = g.velocity_to_host(0, C)
    before = _launches(g)
    hyd, drg, smp = g.hull_forces(table, vel, scales, RHO, 1e-3, maxit, return_samples=True)
    assert _launches(g) - before == (6 if maxit else 4) + (1 if wake else 0)
    with np.errstate(all="ignore"):
        rh, rd, rs = oh.hull_forces(d16, n16, velocity, table, vel, meshes, v, t, scales, RHO, 1e-3, maxit, True, wake=cp)
    assert _same(smp, rs) and _same(hyd, rh) and _same(drg, rd)
    assert (rh["submerged_volume"] > 0).sum() >= 3 and (rd["wetted_drag_area"] > 0).sum() >= 3
    assert not np.frombuffer(rh[fb["mesh"] == len(meshes) - 1].tobytes(), np.uint8).any()
    # the device form gives the same bytes
    import torch
    from godotoceanwaves_b200.native import check, load_library
    dev = torch.device("cuda", g.device)
    hd = torch.zeros(len(fb) * 12, dtype=torch.int32, device=dev)
    dd = torch.zeros(len(fb) * 8, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    check(load_library().ocean_hull_forces_device(g.context, len(fb), table.ctypes.data, vel.ctypes.data, C, scales.ctypes.data, RHO, 1e-3,
                                                  maxit, hd.data_ptr(), dd.data_ptr(), None))
    g.synchronize()
    assert _same(hd.cpu().numpy(), rh) and _same(dd.cpu().numpy(), rd)
    g.free()


@pytest.mark.parametrize("S", [1, 4, 16])
def test_integrator_parity_host_and_device(S):
    import torch
    from godotoceanwaves_b200.native import check, load_library
    N, C = 256, 3
    gow, g, params = _gen(N, C)
    scales = np.ascontiguousarray(gow.WaveGenerator.map_scales(params), np.float32)
    rng = np.random.default_rng(S)
    meshes, v, t = _mesh_set(rng, 3)
    g.set_hull_meshes(meshes, v, t)
    fb, s0 = _bodies(rng, 12, meshes, span=20.0)
    g.update_velocity()
    d16, n16 = g.maps_to_host(0, C)
    velocity = g.velocity_to_host(0, C)
    before = _launches(g)
    s1, hyd, drg, T = g.simulate_hull_bodies(fb, s0, scales, 1.0 / 30.0, S, RHO, return_records=True, return_transforms=True)
    assert _launches(g) - before == 1 + 7 * S
    with np.errstate(all="ignore"):
        rs, rh, rd, rT = oh.simulate(d16, n16, velocity, fb, s0, meshes, v, t, scales, RHO, 1.0 / 30.0, S)
    assert _same(s1, rs) and _same(hyd, rh) and _same(drg, rd) and _same(T, rT)
    dev = torch.device("cuda", g.device)
    st = torch.from_numpy(s0.view(np.uint8).copy()).to(dev)
    Td = torch.zeros(len(fb) * 12, dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    check(load_library().ocean_simulate_hull_bodies_device(g.context, len(fb), fb.ctypes.data, st.data_ptr(), C, scales.ctypes.data, RHO,
                                                           1.0 / 30.0, S, 1e-3, 8, None, None, Td.data_ptr()))
    g.synchronize()
    assert _same(np.frombuffer(st.cpu().numpy().tobytes(), bo.STATE), rs) and _same(Td.cpu().numpy(), rT)
    g.free()


def test_flat_maps_closed_forms():
    """On maps made from a zero spectrum: an upright box displaces its wet volume with its centre of buoyancy at half the draft,
    a box moving along x feels 1/2 rho C A U^2 on its front and sides, and a half-density box settles at half its height."""
    gow, g, params = _flat(256, 2)
    scales = gow.WaveGenerator.map_scales(params)
    lx, ly, lz, cn, ct, U = 2.0, 1.0, 3.0, 1.2, 0.05, 1.5
    bv, bt, mesh = box(lx, ly, lz, cn, ct)
    g.set_hull_meshes(mesh, bv, bt)
    drafts = [0.0, 0.25, 0.5, 0.75, 1.0]
    s = np.zeros(len(drafts), bo.STATE)
    s["orientation"] = (0, 0, 0, 1)
    s["position"][:, 0], s["position"][:, 1] = 37.0, [ly / 2 - d for d in drafts]
    s["linear_velocity"][:, 0] = U
    fb = np.zeros(len(drafts), oh.FLOATING)
    table, vel = oh.pose(fb, s)
    hyd, drg = g.hull_forces(table, vel, scales, RHO)
    np.testing.assert_allclose(hyd["submerged_volume"], [lx * lz * d for d in drafts], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(hyd["center_offset"][1:, 1], [-ly / 2 + d / 2 for d in drafts[1:]], rtol=1e-5, atol=1e-5)
    half = 0.5 * RHO
    d = 0.5
    want = -half * U * U * (cn * d * lz + ct * (2 * lx * d + lx * lz))
    assert drg["force"][2, 0] == pytest.approx(want, rel=1e-5)
    fb = np.zeros(1, oh.FLOATING)
    fb["mass"] = 0.5 * RHO * lx * ly * lz
    fb["inertia"] = 1000.0
    st = np.zeros(1, bo.STATE)
    st["orientation"], st["position"] = (0, 0, 0, 1), (5.0, 1.0, -3.0)
    ys = []
    for _ in range(60):
        st = g.simulate_hull_bodies(fb, st, scales, 1.0 / 3.0, 20, RHO)
        ys.append(float(st["position"][0, 1]))
    assert np.mean(ys[-12:]) == pytest.approx(0.0, abs=3e-3)
    g.free()


def test_nan_pose_is_isolated_and_invalid_calls_launch_nothing():
    gow, g, params = _gen(256, 2)
    scales = gow.WaveGenerator.map_scales(params)
    rng = np.random.default_rng(7)
    fb = np.zeros(4, oh.FLOATING)
    _, s = _bodies(rng, 4, np.zeros(1, oh.MESH))
    table, vel = oh.pose(fb, s)
    vel_bad = vel.copy()
    with pytest.raises(Exception):
        g.hull_forces(table, vel, scales)                      # no meshes registered
    meshes, v, t = _mesh_set(rng, 2)
    g.set_hull_meshes(meshes, v, t)
    table["mesh"] = (0, 1, 2, 3)
    ref = g.hull_forces(table, vel, scales, RHO)
    bad = table.copy()
    bad["transform"][1, 7] = np.nan
    vel_bad["angular"][2] = np.nan
    out = g.hull_forces(bad, vel_bad, scales, RHO)
    for a, b in zip(out, ref):
        assert a[[0, 3]].tobytes() == b[[0, 3]].tobytes()
    assert not out[0]["force"][1].any()                        # every depth of body 1 is NaN: every triangle is dropped
    fbh = np.zeros(4, oh.FLOATING)
    fbh["mass"], fbh["inertia"], fbh["mesh"] = 100.0, 10.0, (0, 1, 2, 3)
    before = _launches(g)
    for call in [lambda: g.hull_forces(_bad_mesh(table, len(meshes)), vel, scales),
                 lambda: g.simulate_hull_bodies(fbh, s, scales, 0.0, 1),
                 lambda: g.simulate_hull_bodies(fbh, s, scales, 1.0 / 60.0, 0),
                 lambda: g.simulate_hull_bodies(fbh, s, scales, 1.0 / 60.0, 65),
                 lambda: g.hull_forces(table, vel, scales, -1.0)]:
        with pytest.raises(Exception):
            call()
    assert _launches(g) == before
    # a rejected set keeps the previous one; an empty set releases it
    m2 = meshes.copy()
    m2["tangential_drag"][0] = -1.0
    with pytest.raises(Exception):
        g.set_hull_meshes(m2, v, t)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(g.hull_forces(table, vel, scales, RHO), ref))
    g.set_hull_meshes(np.zeros(0, oh.MESH), np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
    with pytest.raises(Exception):
        g.hull_forces(table, vel, scales)
    g.free()


def _bad_mesh(table, M):
    b = table.copy()
    b["mesh"][2] = M
    return b


def test_large_hull_beside_small_ones():
    """One hull of 2^16 triangles (a welded sphere grid) beside 2^12 tetrahedra, byte-identical to the specification."""
    gow, g, params = _gen(256, 2)
    scales = np.ascontiguousarray(gow.WaveGenerator.map_scales(params), np.float32)
    nu, nv = 256, 128                                           # 2 * 256 * 128 = 2^16 triangles on a (u, v) grid, poles pinched
    th = np.linspace(0, np.pi, nv + 1)
    ph = np.linspace(0, 2 * np.pi, nu, endpoint=False)
    grid = np.stack([np.outer(np.sin(th), np.cos(ph)), np.outer(np.cos(th), np.ones(nu)), np.outer(np.sin(th), np.sin(ph))], 2)
    sv = (grid.reshape(-1, 3) * (6.0, 2.0, 3.0)).astype(np.float32)
    idx = np.arange((nv + 1) * nu).reshape(nv + 1, nu)
    a, b = idx[:-1], np.roll(idx[:-1], -1, 1)
    c, d = idx[1:], np.roll(idx[1:], -1, 1)
    st = np.concatenate([np.stack([a, c, b], -1).reshape(-1, 3), np.stack([b, c, d], -1).reshape(-1, 3)]).astype(np.int32)
    tv = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32) - 0.25
    tt = np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]], np.int32)
    meshes = np.zeros(2, oh.MESH)
    meshes[0] = (0, len(sv), 0, len(st), 1.0, 0.05)
    meshes[1] = (len(sv), 4, len(st), 4, 1.0, 0.05)
    assert meshes["num_triangles"][0] == 2 ** 16
    v, t = np.concatenate([sv, tv]), np.concatenate([st, tt])
    vols = g.set_hull_meshes(meshes, v, t)
    assert vols[0] > 0 and vols[1] > 0                          # both wound outward
    rng = np.random.default_rng(11)
    fb = np.zeros(1 + 2 ** 12, oh.FLOATING)
    fb["mesh"][1:] = 1
    _, s = _bodies(rng, len(fb), meshes, span=40.0)
    s["position"][0] = (0.0, 0.0, 0.0)
    table, vel = oh.pose(fb, s)
    g.update_velocity()
    d16, n16 = g.maps_to_host(0, 2)
    velocity = g.velocity_to_host(0, 2)
    hyd, drg = g.hull_forces(table, vel, scales, RHO)
    with np.errstate(all="ignore"):
        rh, rd = oh.hull_forces(d16, n16, velocity, table, vel, meshes, v, t, scales, RHO)
    assert _same(hyd, rh) and _same(drg, rd)
    assert rh["submerged_volume"][0] > 0.1 * vols[0] and (rh["submerged_volume"][1:] > 0).any()
    g.free()
