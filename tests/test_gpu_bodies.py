"""GPU parity of the floating-body integrator (ocean_simulate_bodies) against its numpy specification oracle/bodies.py on
the generator's own maps and velocity maps: byte-identical 52-byte states, buoyancy and drag records and transforms after
several calls of several sub-steps; the records against ocean_body_forces; composition, isolation of bad bodies, rest on
flat water, launch counts, side effects and arguments."""
import numpy as np
import pytest

from conftest import demo_params
from oracle import bodies as ob
from oracle import buoyancy as bu
from oracle import drag as dr
from test_gpu_buoyancy import _scene
from test_gpu_sampling import _gen, _same_or_both_nan
from test_gpu_surface import _crc, _scales
from test_oracle_buoyancy import _box

pytestmark = pytest.mark.gpu

RHO = 1025.0
INVALID = 1   # OCEAN_ERR_INVALID_ARGUMENT
DT = 1.0 / 60.0


def _bodies(seed, sizes, share_every=3):
    """test_gpu_buoyancy._scene's hulls and ranges (shared hulls, empty bodies) as floating bodies of density 200 to 900 kg/m^3
    of their hull volume, with random unit quaternions, positions within 1 m of the surface, velocities and drag areas."""
    tbl, hull = _scene(seed, sizes, share_every)
    rng = np.random.default_rng(seed + 1)
    n = len(tbl)
    b = np.zeros(n, ob.BODY)
    b["first_point"], b["num_points"] = tbl["first_point"], tbl["num_points"]
    vol = np.array([hull["volume"][f:f + c].astype(np.float64).sum() for f, c in zip(tbl["first_point"], tbl["num_points"])])
    b["mass"] = np.where(vol > 0, vol, 1.0) * rng.uniform(200, 900, n)
    b["inertia"] = b["mass"][:, None] * rng.uniform(0.5, 3.0, (n, 3))
    s = np.zeros(n, ob.STATE)
    s["position"] = tbl["transform"][:, [3, 7, 11]]
    q = rng.normal(size=(n, 4))
    s["orientation"] = q / np.linalg.norm(q, axis=1, keepdims=True)
    s["linear_velocity"] = rng.uniform(-2, 2, (n, 3))
    s["angular_velocity"] = rng.uniform(-1, 1, (n, 3))
    return b, s, hull, rng.uniform(0.01, 0.6, len(hull)).astype(np.float32)


def _spec(g, C, bodies, states, hull, cda, scales, dt, substeps, maxit=8, density=RHO):
    d16, n16 = g.maps_to_host(0, C)
    with np.errstate(all="ignore"):
        return ob.simulate(d16, n16, g.velocity_to_host(0, C), bodies, states, hull, cda, scales, density, dt, substeps, 1e-3, maxit)


def _same(a, b):
    return a.tobytes() == b.tobytes()


@pytest.mark.parametrize("N,C", [(128, 3), (256, 4), (512, 2), (1024, 2)])
def test_simulate_bit_exact(N, C):
    gow, g, params = _gen(N, C)
    sizes = np.random.default_rng(N + 7).integers(0, 40, 300)
    bodies, s0, hull, cda = _bodies(300 + N, sizes)
    restarted = False
    for factor, maxit in ((1.0, 8), (2.0, 8), (1.0, 0)):       # twice the displacement: many more restarts
        scales = _scales(gow, params, C)
        scales[:, 2] *= np.float32(factor)
        table, vel = ob.pose(bodies, s0)
        _, _, smp = g.body_forces(table, vel, hull, cda, scales, RHO, 1e-3, maxit, return_samples=True)
        restarted |= bool(np.any(smp["iterations"] > 8))       # the first sub-step's query is this one
        s, r = s0, s0
        for _ in range(3):
            s, hyd, drg, T = g.simulate_bodies(bodies, s, hull, cda, scales, DT, 4, RHO, 1e-3, maxit, return_records=True,
                                               return_transforms=True)
            r, rh, rd, rT = _spec(g, C, bodies, r, hull, cda, scales, DT, 4, maxit)
            assert _same(s, r) and _same(hyd, rh) and _same(drg, rd) and _same(T, rT)
        moved = np.abs(s["position"] - s0["position"]).max(1)
        assert np.all(np.isfinite(s["position"])) and np.count_nonzero(moved) == len(s)
        assert np.count_nonzero(hyd["submerged_volume"]) > 100 and np.count_nonzero(drg["wetted_drag_area"]) > 100
        assert not hyd[bodies["num_points"] == 0].tobytes().strip(b"\0")
    assert restarted                                            # the restart kernel ran
    g.free()


def test_records_and_pose_tables_equal_body_forces():
    """With 1 sub-step the records are ocean_body_forces' on [R(q) | position] and the state's velocities (R(q) from the
    specification); with 2 they are ocean_body_forces' at the specification's state after the first sub-step, which the
    integrate kernel wrote into the device pose and velocity tables; the transforms are those of the final states."""
    import torch
    from godotoceanwaves_b200.native import check, load_library
    gow, g, params = _gen(256, 4)
    scales = _scales(gow, params, 4)
    bodies, s0, hull, cda = _bodies(401, np.random.default_rng(400).integers(0, 60, 500))
    table, vel = ob.pose(bodies, s0)
    dev = torch.device("cuda", g.device)
    hull_d = torch.from_numpy(hull.view(np.uint8).copy()).to(dev)
    cda_d = torch.from_numpy(cda).to(dev)
    hyd_d = torch.zeros(len(bodies) * 12, dtype=torch.int32, device=dev)
    drg_d = torch.zeros(len(bodies) * 8, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    check(load_library().ocean_body_forces_device(g.context, len(bodies), table.ctypes.data, vel.ctypes.data, len(hull), hull_d.data_ptr(),
                                                  cda_d.data_ptr(), 4, scales.ctypes.data, RHO, 1e-3, 8, hyd_d.data_ptr(), drg_d.data_ptr(),
                                                  None))
    g.synchronize()
    _, hyd, drg = g.simulate_bodies(bodies, s0, hull, cda, scales, DT, 1, RHO, return_records=True)
    assert hyd.tobytes() == hyd_d.cpu().numpy().tobytes() and drg.tobytes() == drg_d.cpu().numpy().tobytes()
    assert np.count_nonzero(drg["wetted_drag_area"]) > 100
    # the tables the integrate kernel writes for the second sub-step
    s1 = _spec(g, 4, bodies, s0, hull, cda, scales, np.float32(DT) / np.float32(2), 1)[0]
    t1, v1 = ob.pose(bodies, s1)
    h1, d1 = g.body_forces(t1, v1, hull, cda, scales, RHO)
    s2, hyd2, drg2, T2 = g.simulate_bodies(bodies, s0, hull, cda, scales, DT, 2, RHO, return_records=True, return_transforms=True)
    assert hyd2.tobytes() == h1.tobytes() and drg2.tobytes() == d1.tobytes()
    assert T2.tobytes() == ob.transforms(s2).tobytes()
    g.free()


def test_substeps_compose_on_the_device():
    gow, g, params = _gen(256, 3)
    scales = _scales(gow, params, 3)
    bodies, s0, hull, cda = _bodies(411, np.random.default_rng(410).integers(0, 50, 400))
    a, ha, da, Ta = g.simulate_bodies(bodies, s0, hull, cda, scales, DT, 6, RHO, return_records=True, return_transforms=True)
    c = s0
    for _ in range(6):
        c, hc, dc, Tc = g.simulate_bodies(bodies, c, hull, cda, scales, np.float32(DT) / np.float32(6), 1, RHO, return_records=True,
                                          return_transforms=True)
    assert _same(a, c) and _same(ha, hc) and _same(da, dc) and _same(Ta, Tc)
    g.free()


def test_bad_bodies_stay_isolated():
    """3000 bodies with a NaN orientation, an infinite position and a NaN velocity: NaN appears only in those bodies, and
    every other body is bit-identical to the specification."""
    gow, g, params = _gen(256, 4)
    scales = _scales(gow, params, 4)
    sizes = np.random.default_rng(420).integers(1, 40, 3000)
    sizes[10::97] = 0
    bodies, s0, hull, cda = _bodies(421, sizes, share_every=4)
    s0["orientation"][7, 1] = np.nan
    s0["position"][8, 0] = np.inf
    s0["linear_velocity"][6, 0] = np.nan
    s0["position"][6, 1] = -2.0                                 # under water: its drag sees the NaN
    s, hyd, drg, T = g.simulate_bodies(bodies, s0, hull, cda, scales, DT, 2, RHO, return_records=True, return_transforms=True)
    r, rh, rd, rT = _spec(g, 4, bodies, s0, hull, cda, scales, DT, 2)
    bad = np.zeros(len(bodies), bool)
    bad[[6, 7, 8]] = True
    assert _same(s[~bad], r[~bad]) and _same(hyd[~bad], rh[~bad]) and _same(drg[~bad], rd[~bad]) and _same(T[~bad], rT[~bad])
    for f in ob.STATE.names:
        assert _same_or_both_nan(s[bad][f], r[bad][f]), f
    assert np.isnan(s["linear_velocity"][6]).any() and np.isnan(s["orientation"][7]).all()
    good = s[~bad]
    for f in ob.STATE.names:
        assert np.isfinite(good[f]).all(), f
    assert np.isfinite(T[~bad]).all() and np.isfinite(hyd[~bad]["force"]).all() and np.isfinite(drg[~bad]["force"]).all()
    g.free()


def test_box_at_equilibrium_on_flat_water_stays_exactly_at_rest():
    import godotoceanwaves_b200 as gow
    N, Cn = 256, 2
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(Cn)
    params = [demo_params(gow.WaveCascadeParameters, c) for c in range(Cn)]
    g.update_all(0.02, params)
    for c in range(Cn):
        g.set_spectrum_amplitudes(c, np.zeros((N, N), np.complex64))
    g.update_all(0.02, params)
    hull = _box(2, 1, 2, 1.0)                                   # four 1 m columns; 1024 kg in water of 1024 kg/m^3: draft 0.25 m
    b = np.zeros(2, ob.BODY)
    b["mass"], b["inertia"], b["num_points"] = 1024.0, (400.0, 700.0, 400.0), len(hull)
    s0 = np.zeros(2, ob.STATE)
    s0["orientation"] = (0.0, 0.0, 0.0, 1.0)
    s0["position"] = [(37.0, 0.25, -91.5), (-12.0, 0.25, 3.0)]
    s = s0
    for _ in range(20):
        s = g.simulate_bodies(b, s, hull, np.ones(len(hull), np.float32), gow.WaveGenerator.map_scales(params), DT, 4, 1024.0)
    assert s.tobytes() == s0.tobytes()
    g.free()


def test_launch_counts_and_host_equals_device():
    import torch
    from godotoceanwaves_b200.native import check, load_library
    gow, g, params = _gen(256, 4)
    assert gow.WaveGenerator.FLOATING_BODY.itemsize == 24 and gow.WaveGenerator.BODY_STATE.itemsize == 52
    scales = _scales(gow, params, 4)
    bodies, s0, hull, cda = _bodies(431, np.random.default_rng(430).integers(0, 80, 600))
    g.update_velocity()
    for S, maxit, launches in ((1, 8, 8), (4, 8, 29), (4, 0, 21), (64, 8, 449)):
        before = g.info().kernel_launches
        g.simulate_bodies(bodies, s0, hull, cda, scales, DT, S, RHO, 1e-3, maxit)
        assert g.info().kernel_launches - before == launches, (S, maxit)
    empty = bodies.copy()
    empty["num_points"] = 0
    before = g.info().kernel_launches
    g.simulate_bodies(empty, s0, hull, cda, scales, DT, 4, RHO)
    assert g.info().kernel_launches - before == 1 + 3 * 4
    # the device entry point on device states equals the host entry point
    s, hyd, drg, T = g.simulate_bodies(bodies, s0, hull, cda, scales, DT, 3, RHO, return_records=True, return_transforms=True)
    dev = torch.device("cuda", g.device)
    st_d = torch.from_numpy(s0.view(np.uint8).copy()).to(dev)
    hull_d = torch.from_numpy(hull.view(np.uint8).copy()).to(dev)
    cda_d = torch.from_numpy(cda).to(dev)
    hyd_d = torch.zeros(len(bodies) * 12, dtype=torch.int32, device=dev)
    drg_d = torch.zeros(len(bodies) * 8, dtype=torch.int32, device=dev)
    T_d = torch.zeros(len(bodies) * 12, dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    check(load_library().ocean_simulate_bodies_device(g.context, len(bodies), bodies.ctypes.data, st_d.data_ptr(), len(hull), hull_d.data_ptr(),
                                                      cda_d.data_ptr(), 4, scales.ctypes.data, RHO, DT, 3, 1e-3, 8, hyd_d.data_ptr(),
                                                      drg_d.data_ptr(), T_d.data_ptr()))
    g.synchronize()
    assert st_d.cpu().numpy().tobytes() == s.tobytes()
    assert hyd_d.cpu().numpy().tobytes() == hyd.tobytes() and drg_d.cpu().numpy().tobytes() == drg.tobytes()
    assert T_d.cpu().numpy().tobytes() == T.tobytes()
    # records and transforms may be NULL
    st_d = torch.from_numpy(s0.view(np.uint8).copy()).to(dev)
    torch.cuda.synchronize()
    check(load_library().ocean_simulate_bodies_device(g.context, len(bodies), bodies.ctypes.data, st_d.data_ptr(), len(hull), hull_d.data_ptr(),
                                                      cda_d.data_ptr(), 4, scales.ctypes.data, RHO, DT, 3, 1e-3, 8, None, None, None))
    g.synchronize()
    assert st_d.cpu().numpy().tobytes() == s.tobytes()
    g.free()


def test_simulate_leaves_the_generator_alone_and_refreshes_stale_velocity():
    """Maps, foam, spectrum and the next update are byte-identical with and without integrator calls; a call after
    ocean_process refreshes the stale velocity layer once, and matches the specification on the refreshed maps."""
    import godotoceanwaves_b200 as gow
    N, Cn = 128, 3
    a = gow.WaveGenerator(); a.map_size = N; a.init_gpu(Cn)
    b = gow.WaveGenerator(); b.map_size = N; b.init_gpu(Cn)
    pa = [demo_params(gow.WaveCascadeParameters, c) for c in range(Cn)]
    pb = [demo_params(gow.WaveCascadeParameters, c) for c in range(Cn)]
    scales = gow.WaveGenerator.map_scales(pa)
    small, big = _bodies(441, [3, 4]), _bodies(442, np.full(500, 60))
    for k in range(3):
        a.update_all(1.0 / 50.0, pa)
        b.update_all(1.0 / 50.0, pb)
        for bodies, s0, hull, cda in (small, big) if k else (small,):
            a.simulate_bodies(bodies, s0, hull, cda, scales, DT, 3, return_records=True, return_transforms=True)
        da, na = a.maps_to_host(0, Cn)
        db, nb = b.maps_to_host(0, Cn)
        assert (_crc(da), _crc(na)) == (_crc(db), _crc(nb))
        for c in range(Cn):
            assert a.get_foam_state(c).tobytes() == b.get_foam_state(c).tobytes()
            assert a.spectrum_to_host(c).tobytes() == b.spectrum_to_host(c).tobytes()
    bodies, s0, hull, cda = big
    a.update_velocity()
    assert a.update_velocity() == 0                             # nothing stale: the integrator makes nothing stale
    a.simulate_bodies(bodies, s0, hull, cda, scales, DT, 2)
    assert a.update_velocity() == 0
    for _ in range(2):
        a.update(0.03, pa)
        a._process()                                            # one cascade's velocity layer is now stale
        before = a.info().kernel_launches
        s, hyd, drg = a.simulate_bodies(bodies, s0, hull, cda, scales, DT, 2, return_records=True)
        refresh = a.info().kernel_launches - before - (1 + 7 * 2)
        assert 0 < refresh <= 3                                 # the refresh ran once in the call ...
        assert a.update_velocity() == 0                         # ... and left nothing stale
        r, rh, rd, _ = _spec(a, Cn, bodies, s0, hull, cda, scales, DT, 2, 8, 1025.0)
        assert _same(s, r) and _same(hyd, rh) and _same(drg, rd)
    a.free(); b.free()


def test_simulate_arguments():
    """Every invalid argument returns OCEAN_ERR_INVALID_ARGUMENT and launches nothing (not even a velocity refresh), through
    both entry points."""
    from godotoceanwaves_b200.native import load_library
    gow, g, params = _gen(128, 2, frames=1)                     # the velocity layers are stale: a refresh would launch
    lib = load_library()
    scales = gow.WaveGenerator.map_scales(params)
    bodies, s0, hull, cda = _bodies(451, [4, 0, 6])
    bodies["num_points"][1] = 0
    hyd = np.zeros(len(bodies), bu.RESULT)
    drg = np.zeros(len(bodies), dr.RESULT)
    ok = dict(nb=len(bodies), b=bodies, st=s0.ctypes.data, np_=len(hull), p=hull.ctypes.data, a=cda.ctypes.data, nc=2, sc=scales.ctypes.data,
              rho=RHO, dt=DT, S=4, tol=1e-3, it=8)

    def body_edit(**kw):
        b = bodies.copy()
        for k, v in kw.items():
            b[k][0] = v
        return b

    big = bodies[:2].copy()
    big["first_point"], big["num_points"] = 0, 2 ** 31 - 1
    nan, inf = float("nan"), float("inf")
    bad = [dict(nb=-1), dict(np_=-1), dict(rho=0.0), dict(rho=nan), dict(rho=inf), dict(tol=0.0), dict(tol=nan), dict(it=-1), dict(it=65),
           dict(dt=0.0), dict(dt=-DT), dict(dt=nan), dict(dt=inf), dict(S=0), dict(S=65), dict(S=-1),
           dict(b=body_edit(mass=0.0)), dict(b=body_edit(mass=-1.0)), dict(b=body_edit(mass=nan)), dict(b=body_edit(mass=inf)),
           dict(b=body_edit(inertia=(1.0, 0.0, 1.0))), dict(b=body_edit(inertia=(1.0, 1.0, nan))), dict(b=body_edit(inertia=(-1.0, 1.0, 1.0))),
           dict(b=body_edit(inertia=(inf, 1.0, 1.0))),
           dict(b=body_edit(num_points=-1)), dict(b=body_edit(first_point=-1)), dict(b=body_edit(first_point=7)),
           dict(b=body_edit(first_point=2 ** 31 - 2)), dict(nb=2, b=big, np_=2 ** 31 - 1),
           dict(b=None), dict(st=None), dict(p=None), dict(a=None), dict(nc=0), dict(nc=3), dict(sc=None)]
    for fn in (lib.ocean_simulate_bodies, lib.ocean_simulate_bodies_device):
        for kw in bad:
            a = dict(ok)
            a.update(kw)
            before = g.info().kernel_launches
            rc = fn(g.context, a["nb"], None if a["b"] is None else a["b"].ctypes.data, a["st"], a["np_"], a["p"], a["a"], a["nc"], a["sc"],
                    a["rho"], a["dt"], a["S"], a["tol"], a["it"], hyd.ctypes.data, drg.ctypes.data, None)
            assert rc == INVALID, kw
            assert g.info().kernel_launches == before, kw
    # NULL is fine where no count needs the buffer
    empty = bodies[[1]]
    st = s0[[1]].copy()
    assert lib.ocean_simulate_bodies(g.context, 1, empty.ctypes.data, st.ctypes.data, 0, None, None, 2, scales.ctypes.data, RHO, DT, 1,
                                     1e-3, 8, None, None, None) == 0
    assert st["linear_velocity"][0, 1] < s0["linear_velocity"][1, 1]
    assert lib.ocean_simulate_bodies(g.context, 0, None, None, 0, None, None, 0, None, RHO, DT, 1, 1e-3, 8, None, None, None) == 0
    assert len(g.simulate_bodies(bodies[:0], s0[:0], hull, cda, scales, DT)) == 0
    with pytest.raises(ValueError):
        g.simulate_bodies(bodies, s0[:2], hull, cda, scales, DT)
    g.free()
