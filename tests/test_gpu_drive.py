"""GPU tests of the driven floating-body integrator (ocean_simulate_driven_bodies) against its numpy specification
oracle/drive.py: byte-identical states, hydrostatic, drag and drive records, tensions and transforms over random fleets with
shared hulls, many thrusters, foils and tethers per body (body to body and anchored), loads, and NaN / infinite actuators and
tethers; host form equals device form; launch counts; argument rejection with no launch; isolation from the plain integrator
and the maps; the closed-form steady states on flat water; and a thruster-driven boat that draws a Kelvin wedge."""
import math

import numpy as np
import pytest

from conftest import demo_params
from oracle import bodies as ob
from oracle import drive as od
from oracle import wake as wk
from oracle import wake_coupling as wc
from test_gpu_bodies import _bodies
from test_gpu_sampling import _gen
from test_gpu_surface import _crc, _scales
from test_gpu_wake_coupling import _flat, _init, _params, _same
from test_oracle_buoyancy import _box

pytestmark = pytest.mark.gpu

RHO = 1025.0
DT = 1.0 / 60.0
INVALID = 1   # OCEAN_ERR_INVALID_ARGUMENT


def _unit(rng, n):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _drive(rng, states, per_body=2, bad=True):
    """Random drive arguments for the bodies of `states`: per_body thrusters and foils per body on average, a tether per body
    (a quarter anchored), loads on every body; with bad, NaN and infinite actuators, tethers and a load on a few bodies.
    Returns (thrusters, foils, loads, tethers, the indices of the bodies a bad row touches)."""
    B = len(states)
    nt = nf = per_body * B
    th = np.zeros(nt, od.THRUSTER)
    th["body"] = rng.integers(0, B, nt)
    th["position"] = rng.uniform(-1.5, 1.5, (nt, 3))
    th["direction"] = _unit(rng, nt)
    th["thrust"] = rng.uniform(0, 3000, nt)
    th["half_height"] = np.where(rng.random(nt) < 0.2, 0.0, rng.uniform(0.05, 0.6, nt))
    fo = np.zeros(nf, od.FOIL)
    fo["body"] = rng.integers(0, B, nf)
    fo["position"] = rng.uniform(-1.5, 1.5, (nf, 3))
    fo["normal"] = _unit(rng, nf)
    fo["area"] = rng.uniform(0, 2, nf)
    fo["half_height"] = np.where(rng.random(nf) < 0.2, 0.0, rng.uniform(0.05, 0.6, nf))
    te = np.zeros(B, od.TETHER)
    te["body_a"] = rng.integers(0, B, B)
    other = (te["body_a"] + rng.integers(1, B, B)) % B
    te["body_b"] = np.where(rng.random(B) < 0.25, -1, other)
    te["point_a"] = rng.uniform(-1, 1, (B, 3))
    te["point_b"] = rng.uniform(-1, 1, (B, 3))
    anch = te["body_b"] < 0
    te["point_b"][anch] = states["position"][te["body_a"][anch]] + rng.uniform(-4, 4, (int(anch.sum()), 3))
    te["rest_length"] = rng.uniform(0, 4, B)
    te["stiffness"] = rng.uniform(0, 5e4, B)
    te["damping"] = rng.uniform(0, 2e3, B)
    ld = np.zeros(B, od.LOAD)
    ld["force"] = rng.uniform(-500, 500, (B, 3))
    ld["torque"] = rng.uniform(-200, 200, (B, 3))
    touched = set()
    if bad:
        th["thrust"][3] = np.nan
        th["direction"][5, 1] = np.inf
        fo["position"][4, 0] = np.nan
        fo["normal"][6, 2] = -np.inf
        te["point_a"][2, 1] = np.nan
        te["point_b"][6, 0] = np.inf
        ld["torque"][7, 0] = np.nan
        touched = {int(th["body"][3]), int(th["body"][5]), int(fo["body"][4]), int(fo["body"][6]), int(te["body_a"][2]),
                   int(te["body_b"][2]), int(te["body_a"][6]), int(te["body_b"][6]), 7} - {-1}
    return th, fo, ld, te, sorted(touched)


def _spec(g, C, bodies, states, hull, cda, scales, dt, substeps, maxit, th, fo, ld, te, wake=None):
    d16, n16 = g.maps_to_host(0, C)
    with np.errstate(all="ignore"):
        return od.simulate(d16, n16, g.velocity_to_host(0, C), bodies, states, hull, cda, scales, RHO, dt, substeps, 1e-3, maxit, th, fo, ld,
                           te, wake)


def _device(g, bodies, st_d, hull_d, cda_d, nh, C, scales, S, maxit, th, fo, ld, te, outs):
    from godotoceanwaves_b200.native import check, load_library
    import torch
    hyd_d, drg_d, drv_d, ten_d, T_d = outs
    ptr = lambda x: None if x is None else x.data_ptr()  # noqa: E731
    torch.cuda.synchronize()
    check(load_library().ocean_simulate_driven_bodies_device(
        g.context, len(bodies), bodies.ctypes.data, st_d.data_ptr(), nh, hull_d.data_ptr(), cda_d.data_ptr(), C, scales.ctypes.data, RHO, DT, S,
        1e-3, maxit, len(th), th.ctypes.data if len(th) else None, len(fo), fo.ctypes.data if len(fo) else None,
        None if ld is None else ld.ctypes.data, len(te), te.ctypes.data if len(te) else None, ptr(hyd_d), ptr(drg_d), ptr(drv_d), ptr(ten_d),
        ptr(T_d)))
    g.synchronize()


def _torch_outs(g, B, K):
    import torch
    dev = torch.device("cuda", g.device)
    return (torch.zeros(B * 12, dtype=torch.int32, device=dev), torch.zeros(B * 8, dtype=torch.int32, device=dev),
            torch.zeros(B * 8, dtype=torch.int32, device=dev), torch.zeros(max(K, 1), dtype=torch.float32, device=dev),
            torch.zeros(B * 12, dtype=torch.float32, device=dev))


def _host(outs, B, K):
    hyd_d, drg_d, drv_d, ten_d, T_d = outs
    return (np.frombuffer(hyd_d.cpu().numpy().tobytes(), ob.bu.RESULT), np.frombuffer(drg_d.cpu().numpy().tobytes(), ob.dr.RESULT),
            np.frombuffer(drv_d.cpu().numpy().tobytes(), od.RESULT), ten_d.cpu().numpy()[:K], T_d.cpu().numpy().reshape(B, 12))


@pytest.mark.parametrize("N,C,nb", [(128, 3, 300), (256, 4, 200), (512, 2, 120), (1024, 2, 60)])
def test_parity_with_the_specification(N, C, nb):
    """Device states across calls of S = 1 and 4 sub-steps with max_iterations 8 and 0: every output byte-identical to the
    specification (NaN only has to meet NaN), and the bad rows' NaN confined to the bodies they touch."""
    import torch
    gow, g, params = _gen(N, C)
    scales = _scales(gow, params, C)
    rng = np.random.default_rng(N)
    bodies, s0, hull, cda = _bodies(700 + N, rng.integers(0, 30, nb))
    th, fo, ld, te, touched = _drive(rng, s0)
    dev = torch.device("cuda", g.device)
    st_d = torch.from_numpy(s0.view(np.uint8).copy()).to(dev)
    hull_d = torch.from_numpy(hull.view(np.uint8).copy()).to(dev)
    cda_d = torch.from_numpy(cda).to(dev)
    outs = _torch_outs(g, len(bodies), len(te))
    r = s0
    for S, maxit in ((1, 8), (4, 8), (4, 0), (1, 0)):
        _device(g, bodies, st_d, hull_d, cda_d, len(hull), C, scales, S, maxit, th, fo, ld, te, outs)
        r, rh, rd, rdrv, rten, rT = _spec(g, C, bodies, r, hull, cda, scales, DT, S, maxit, th, fo, ld, te)
        s = np.frombuffer(st_d.cpu().numpy().tobytes(), ob.STATE)
        hyd, drg, drv, ten, T = _host(outs, len(bodies), len(te))
        assert _same(s, r) and _same(hyd, rh) and _same(drg, rd), (S, maxit)
        assert _same(drv, rdrv) and _same(ten, rten) and _same(T, rT), (S, maxit)
    good = np.setdiff1d(np.arange(len(bodies)), touched)
    for f in ob.STATE.names:
        assert np.isfinite(s[good][f]).all(), f
    assert np.isnan(s[7]["orientation"]).all()                     # the NaN load torque
    assert np.count_nonzero(drv["wetted_foil_area"]) > len(bodies) // 4 and np.count_nonzero(ten) > len(te) // 4
    assert np.count_nonzero(np.abs(drv["force"]).sum(1)) > len(bodies) // 2
    g.free()


@pytest.mark.parametrize("S", [1, 4])
def test_parity_with_the_wake_coupling(S):
    """The same on a coupled wake layer: the actuators' query points read the wake's height, and the foils its wv."""
    gow, g, params = _gen(256, 2)
    scales = gow.WaveGenerator.map_scales(params)
    n, dx = 256, 0.5
    p = _params(n, dx, damping=0.02, sponge_cells=24, sponge_damping=1.0)
    _init(g, p)
    L, cp = wk.Layer(p), wc.Coupling(n, dx)
    g.wake_set_coupling(True)
    rng = np.random.default_rng(50 + S)
    bodies, s0, hull, cda = _bodies(820 + S, rng.integers(1, 24, 24))
    ext = n * dx
    s0["position"][:, 0] = rng.uniform(0.2 * ext, 0.8 * ext, len(s0))
    s0["position"][:, 2] = rng.uniform(0.2 * ext, 0.8 * ext, len(s0))
    th, fo, ld, te, _ = _drive(rng, s0, 3, bad=False)
    src = np.zeros(len(bodies), wk.SOURCE)
    src["radius"], src["head"], src["body"] = 2.0, 0.3, np.arange(len(bodies))
    s = s0
    for call in range(3):
        g.wake_step(DT * 2, 2, (0, 0), src, s)
        wc.step(L, cp, DT * 2, 2, (0, 0), src, s)
        out = g.drive_bodies(bodies, s, hull, cda, scales, DT, S, RHO, 1e-3, 8, th, fo, ld, te, return_records=True, return_tensions=True,
                             return_transforms=True)
        ref = _spec(g, 2, bodies, s, hull, cda, scales, DT, S, 8, th, fo, ld, te, wake=cp)
        assert all(_same(a, b) for a, b in zip(out, ref)), call
        s = out[0]
    g.free()


def test_host_form_equals_device_form_and_launch_counts():
    import torch
    gow, g, params = _gen(256, 4)
    scales = _scales(gow, params, 4)
    rng = np.random.default_rng(3)
    bodies, s0, hull, cda = _bodies(431, rng.integers(0, 60, 400))
    th, fo, ld, te, _ = _drive(rng, s0, bad=False)
    g.update_velocity()
    host = g.drive_bodies(bodies, s0, hull, cda, scales, DT, 3, RHO, 1e-3, 8, th, fo, ld, te, return_records=True, return_tensions=True,
                          return_transforms=True)
    dev = torch.device("cuda", g.device)
    st_d = torch.from_numpy(s0.view(np.uint8).copy()).to(dev)
    hull_d = torch.from_numpy(hull.view(np.uint8).copy()).to(dev)
    cda_d = torch.from_numpy(cda).to(dev)
    outs = _torch_outs(g, len(bodies), len(te))
    _device(g, bodies, st_d, hull_d, cda_d, len(hull), 4, scales, 3, 8, th, fo, ld, te, outs)
    assert st_d.cpu().numpy().tobytes() == host[0].tobytes()
    for a, b in zip(_host(outs, len(bodies), len(te)), host[1:]):
        assert a.tobytes() == b.tobytes()
    st_d = torch.from_numpy(s0.view(np.uint8).copy()).to(dev)       # every output may be NULL
    _device(g, bodies, st_d, hull_d, cda_d, len(hull), 4, scales, 3, 8, th, fo, ld, te, (None,) * 5)
    assert st_d.cpu().numpy().tobytes() == host[0].tobytes()
    # 1 + S (7 + a + t + 1) with actuators and tethers; the header's other forms
    empty = np.zeros(0, od.THRUSTER), np.zeros(0, od.FOIL), np.zeros(0, od.TETHER)
    cases = [((th, fo, ld, te), 4, 8, 1 + 4 * 10), ((th, fo, ld, te), 4, 0, 1 + 4 * 8), ((th, empty[1], None, empty[2]), 2, 8, 1 + 2 * 9),
             ((empty[0], empty[1], None, te), 2, 8, 1 + 2 * 9), ((empty[0], empty[1], ld, empty[2]), 2, 8, 1 + 2 * 8),
             ((empty[0], empty[1], None, empty[2]), 4, 8, 1 + 4 * 7)]
    for (t, f, l, k), S, maxit, launches in cases:
        before = g.info().kernel_launches
        g.drive_bodies(bodies, s0, hull, cda, scales, DT, S, RHO, 1e-3, maxit, t, f, l, k)
        assert g.info().kernel_launches - before == launches, (S, maxit, len(t), len(f), l is None, len(k))
    ball = bodies.copy()
    ball["num_points"] = 0                                          # no world points, actuators only: 1 + S (3 + a + t + 1) ...
    before = g.info().kernel_launches
    g.drive_bodies(ball, s0, hull, cda, scales, DT, 2, RHO, 1e-3, 8, th, fo, ld, te)
    assert g.info().kernel_launches - before == 1 + 2 * (1 + 3 + 2 + 1 + 1 + 1)
    before = g.info().kernel_launches                               # ... and with no actuators either
    g.drive_bodies(ball, s0, hull, cda, scales, DT, 2, RHO, 1e-3, 8, None, None, ld, te)
    assert g.info().kernel_launches - before == 1 + 2 * (2 + 1 + 1 + 1)
    g.free()


def test_no_drive_is_simulate_bodies_and_leaves_the_generator_alone():
    """The call without drive arguments is ocean_simulate_bodies byte for byte (drive zeroed); maps, foam, spectrum,
    velocity and the wake layer are byte-identical with and without driven calls."""
    import godotoceanwaves_b200 as gow
    N, Cn = 128, 3
    a = gow.WaveGenerator(); a.map_size = N; a.init_gpu(Cn)
    b = gow.WaveGenerator(); b.map_size = N; b.init_gpu(Cn)
    pa = [demo_params(gow.WaveCascadeParameters, c) for c in range(Cn)]
    pb = [demo_params(gow.WaveCascadeParameters, c) for c in range(Cn)]
    scales = gow.WaveGenerator.map_scales(pa)
    rng = np.random.default_rng(9)
    bodies, s0, hull, cda = _bodies(441, rng.integers(0, 30, 200))
    th, fo, ld, te, _ = _drive(rng, s0, bad=False)
    for g in (a, b):
        _init(g, _params(128, 0.5))
    for k in range(3):
        a.update_all(1.0 / 50.0, pa)
        b.update_all(1.0 / 50.0, pb)
        plain = a.simulate_bodies(bodies, s0, hull, cda, scales, DT, 3, RHO, return_records=True, return_transforms=True)
        before = a.info().kernel_launches
        drv = a.drive_bodies(bodies, s0, hull, cda, scales, DT, 3, RHO, return_records=True, return_transforms=True)
        assert a.info().kernel_launches - before == 1 + 7 * 3
        assert all(x.tobytes() == y.tobytes() for x, y in zip(plain, drv[:3] + drv[4:]))
        assert not drv[3].tobytes().strip(b"\0")
        a.drive_bodies(bodies, s0, hull, cda, scales, DT, 2, RHO, 1e-3, 8, th, fo, ld, te)
        da, na = a.maps_to_host(0, Cn)
        db, nb = b.maps_to_host(0, Cn)
        assert (_crc(da), _crc(na)) == (_crc(db), _crc(nb))
        assert a.velocity_to_host(0, Cn).tobytes() == b.velocity_to_host(0, Cn).tobytes()
        for c in range(Cn):
            assert a.get_foam_state(c).tobytes() == b.get_foam_state(c).tobytes()
            assert a.spectrum_to_host(c).tobytes() == b.spectrum_to_host(c).tobytes()
        wa, wb = a.wake_state(), b.wake_state()
        assert wa[0].tobytes() == wb[0].tobytes() and wa[1].tobytes() == wb[1].tobytes() and tuple(wa[2]) == tuple(wb[2])
    a.free(); b.free()


def test_arguments():
    """Every invalid drive argument returns OCEAN_ERR_INVALID_ARGUMENT through both entry points and launches nothing."""
    from godotoceanwaves_b200.native import load_library
    gow, g, params = _gen(128, 2, frames=1)                         # stale velocity layers: a refresh would launch
    lib = load_library()
    scales = gow.WaveGenerator.map_scales(params)
    bodies, s0, hull, cda = _bodies(451, [4, 3, 6])
    rng = np.random.default_rng(1)
    th, fo, ld, te, _ = _drive(rng, s0, bad=False)
    te["body_b"][0] = -1

    def edit(rows, field, value, i=0):
        r = rows.copy()
        r[field][i] = value
        return r
    nan, inf = float("nan"), float("inf")
    bad = [dict(nt=-1), dict(nf=-1), dict(nk=-1), dict(th=None), dict(fo=None), dict(te=None),
           dict(th=edit(th, "body", 3)), dict(th=edit(th, "body", -1)), dict(fo=edit(fo, "body", 3)), dict(fo=edit(fo, "body", -2)),
           dict(te=edit(te, "body_a", 3)), dict(te=edit(te, "body_a", -1)), dict(te=edit(te, "body_b", 3, 1)),
           dict(te=edit(te, "body_b", -2, 1)), dict(te=edit(te, "body_b", int(te["body_a"][1]), 1)),
           dict(fo=edit(fo, "area", -1.0)), dict(fo=edit(fo, "area", nan)), dict(fo=edit(fo, "area", inf)),
           dict(te=edit(te, "rest_length", -0.5)), dict(te=edit(te, "rest_length", nan)), dict(te=edit(te, "stiffness", inf)),
           dict(te=edit(te, "stiffness", -1.0)), dict(te=edit(te, "damping", nan)), dict(te=edit(te, "damping", -1.0)),
           dict(np_=-1), dict(S=0), dict(rho=nan)]
    hyd = np.zeros(3, ob.bu.RESULT)
    for fn in (lib.ocean_simulate_driven_bodies, lib.ocean_simulate_driven_bodies_device):
        for kw in bad:
            a = dict(nt=len(th), th=th, nf=len(fo), fo=fo, nk=len(te), te=te, np_=len(hull), S=2, rho=RHO)
            a.update(kw)
            p = lambda x: None if x is None else x.ctypes.data  # noqa: E731
            before = g.info().kernel_launches
            rc = fn(g.context, 3, bodies.ctypes.data, s0.ctypes.data, a["np_"], hull.ctypes.data, cda.ctypes.data, 2, scales.ctypes.data,
                    a["rho"], DT, a["S"], 1e-3, 8, a["nt"], p(a["th"]), a["nf"], p(a["fo"]), ld.ctypes.data, a["nk"], p(a["te"]),
                    hyd.ctypes.data, None, None, None, None)
            assert rc == INVALID, kw
            assert g.info().kernel_launches == before, kw
    # NULL arrays are fine with zero counts, and positions, thrust and loads are not validated
    assert g.drive_bodies(bodies, s0, hull, cda, scales, DT, 1, RHO, thrusters=edit(th, "thrust", nan), loads=ld).shape == (3,)
    g.free()


def _boat(g, params, U=None, positions=((0.0, 0.25, 0.0),)):
    """_flat's generator and test_oracle_drive's raft: four 1 m columns, 1025 kg floating at draft 0.25 m."""
    hull = _box(2, 1, 2, 1.0)
    n = len(positions)
    b = np.zeros(n, ob.BODY)
    b["mass"], b["inertia"], b["num_points"] = 1025.0, (400.0, 700.0, 400.0), len(hull)
    s = np.zeros(n, ob.STATE)
    s["orientation"] = (0.0, 0.0, 0.0, 1.0)
    s["position"] = positions
    if U is not None:
        s["linear_velocity"][:, 0] = U
    return b, s, hull, np.ones(len(hull), np.float32)


def _thruster(body, thrust, half_height=1.0):
    t = np.zeros(1, od.THRUSTER)
    t["body"], t["direction"], t["thrust"], t["half_height"] = body, (1.0, 0.0, 0.0), thrust, half_height
    return t


def test_closed_forms_on_the_device():
    """test_oracle_drive's four steady states, run by the device on flat maps."""
    gow, g, params = _flat()
    sc = gow.WaveGenerator.map_scales(params)

    def run(b, s, hull, cda, steps, **kw):
        for _ in range(steps):
            s, hyd, drg, drv, ten = g.drive_bodies(b, s, hull, cda, sc, 1.0 / 30.0, 1, RHO, return_records=True, return_tensions=True, **kw)
        return s, hyd, drg, drv, ten
    # thruster: |drive force| = 1/2 rho A_w U^2
    b, s, hull, cda = _boat(g, params)
    s, hyd, drg, drv, ten = run(b, s, hull, cda, 600, thrusters=_thruster(0, 5000.0))
    U = float(np.linalg.norm(s["linear_velocity"][0].astype(np.float64)))
    Fd = float(np.linalg.norm(drv["force"][0].astype(np.float64)))
    assert U == pytest.approx(math.sqrt(Fd / (0.5 * RHO * float(drg["wetted_drag_area"][0]))), rel=1e-3)
    # keel under a lateral load: F = 1/2 rho (A_w + wetted_foil_area) U^2
    b, s, hull, cda = _boat(g, params)
    fo = np.zeros(1, od.FOIL)
    fo["normal"], fo["area"], fo["half_height"] = (0.0, 0.0, 1.0), 4.0, 1.0
    ld = np.zeros(1, od.LOAD)
    ld["force"] = (0.0, 0.0, 3000.0)
    s, hyd, drg, drv, ten = run(b, s, hull, cda, 600, foils=fo, loads=ld)
    U = float(np.linalg.norm(s["linear_velocity"][0].astype(np.float64)))
    assert U == pytest.approx(math.sqrt(3000.0 / (0.5 * RHO * (float(drg["wetted_drag_area"][0]) + float(drv["wetted_foil_area"][0])))),
                              rel=1e-3)
    # mooring: extension F / k
    b, s, hull, cda = _boat(g, params)
    te = np.zeros(1, od.TETHER)
    te["body_b"], te["point_b"], te["rest_length"], te["stiffness"], te["damping"] = -1, (6.0, 0.25, 0.0), 6.0, 4000.0, 2000.0
    ld["force"] = (-2000.0, 0.0, 0.0)
    s, hyd, drg, drv, ten = run(b, s, hull, cda, 900, tethers=te, loads=ld)
    assert -float(s["position"][0, 0]) == pytest.approx(2000.0 / 4000.0, rel=1e-3)
    # tow line: tension = 1/2 rho A_w,follower U^2
    b, s, hull, cda = _boat(g, params, positions=[(0.0, 0.25, 0.0), (-8.0, 0.25, 0.0)])
    te["body_a"], te["body_b"], te["point_b"], te["stiffness"], te["damping"] = 0, 1, (0.0, 0.0, 0.0), 2e4, 5e3
    s, hyd, drg, drv, ten = run(b, s, hull, cda, 900, thrusters=_thruster(0, 6000.0), tethers=te)
    U = float(s["linear_velocity"][1, 0])
    assert float(ten[0]) == pytest.approx(0.5 * RHO * float(drg["wetted_drag_area"][1]) * U * U, rel=1e-3)
    g.free()


def test_thruster_driven_boat_draws_a_kelvin_wedge():
    """A boat trimmed by the terminal-speed formula to U = 2.5 m/s under its own thruster, with a body-attached wake source
    (radius 4 m, dx = 0.5 m, coupling off): the wedge's half-angle, measured as test_gpu_wake.test_kelvin_wedge measures it,
    lies within 3 degrees of 19.47."""
    from scipy.ndimage import maximum_filter1d
    gow, g, params = _flat()
    sc = gow.WaveGenerator.map_scales(params)
    U, r, n, dx = 2.5, 4.0, 1024, 0.5
    b, s, hull, cda = _boat(g, params, U=U)
    _, _, drg = g.drive_bodies(b, s, hull, cda, sc, 1.0 / 30.0, 1, RHO, return_records=True)[:3]
    f = 0.375                                                       # the thruster's immersion at the boat's draft
    thrust = 0.5 * RHO * float(drg["wetted_drag_area"][0]) * U * U / f
    th = _thruster(0, thrust)
    _init(g, _params(n, dx, damping=0.0, sponge_cells=48, sponge_damping=3.0))
    src = np.zeros(1, wk.SOURCE)
    src["radius"], src["head"], src["body"] = r, 0.2, 0
    T = 60.0
    for _ in range(int(T)):
        ox = int(np.floor(float(s["position"][0, 0]) / dx)) - 768
        g.wake_step(1.0, 30, (ox, -512), src, s)
        s = g.drive_bodies(b, s, hull, cda, sc, 1.0, 30, RHO, thrusters=th)
    assert float(s["linear_velocity"][0, 0]) == pytest.approx(U, rel=1e-3) and abs(float(s["position"][0, 2])) < 0.01
    h, _, origin = g.wake_state()
    xs = float(s["position"][0, 0])
    x0, z0 = origin[0] * dx, origin[1] * dx
    offsets = {1: [], -1: []}
    dists = np.arange(20.0, 60.5, 2.0)
    for d in dists:
        i = int(round((xs - d - x0) / dx - 0.5))
        col = maximum_filter1d(np.abs(h[:, i - 1:i + 2]).max(1), size=int(2.0 / dx) * 2 + 1)
        zc = (np.arange(n) + 0.5) * dx + z0
        for side in (1, -1):
            m = (side * zc > 1.0) & (side * zc < d)
            offsets[side].append(abs(zc[m][np.argmax(col[m])]))
    angles = [np.degrees(np.arctan((dists @ np.array(offsets[side])) / (dists @ dists))) for side in (1, -1)]
    angle = float(np.mean(angles))
    print(f"Kelvin half-angle behind the driven boat {angle:.2f} deg (sides {angles[0]:.2f}, {angles[1]:.2f})")
    assert abs(angle - 19.47) <= 3.0, angles
    g.free()
