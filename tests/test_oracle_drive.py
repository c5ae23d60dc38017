"""The driven floating-body integrator's specification (oracle/drive.py) against oracle/bodies.py and closed forms: no drive
is bodies.simulate byte for byte, a body with nothing attached keeps the plain step's bits, slack tethers and dry thrusters add
nothing, and on flat water the terminal speed under thrust, the side speed of a keel, the extension of a mooring and the tension
of a tow line match their formulas; stiff tethers stay bounded and a rudder turns the boat to its side."""
import math

import numpy as np
import pytest

from oracle import bodies as ob
from oracle import drive as od
from test_oracle_bodies import _maps
from test_oracle_buoyancy import _box

F = np.float32
RHO = 1024.0


def _boats(n, positions=None):
    """n copies of a flat 2 x 2 raft of 1 m columns in the centre of mass's plane: 1024 kg floats at draft 0.25 m on still water
    of 1024 kg/m^3, each column wet to f = 0.25."""
    hull = _box(2, 1, 2, 1.0)
    b = np.zeros(n, ob.BODY)
    b["mass"], b["inertia"], b["first_point"], b["num_points"] = 1024.0, (400.0, 700.0, 400.0), 0, len(hull)
    s = np.zeros(n, ob.STATE)
    s["orientation"] = (0.0, 0.0, 0.0, 1.0)
    s["position"] = positions if positions is not None else [(10.0 * i, 0.25, 0.0) for i in range(n)]
    return b, s, hull, np.ones(len(hull), np.float32)


def _thruster(body, thrust, position=(0.0, 0.0, 0.0), direction=(1.0, 0.0, 0.0), half_height=1.0):
    t = np.zeros(1, od.THRUSTER)
    t["body"], t["position"], t["direction"], t["thrust"], t["half_height"] = body, position, direction, thrust, half_height
    return t


def _foil(body, area, normal=(0.0, 0.0, 1.0), position=(0.0, 0.0, 0.0), half_height=1.0):
    f = np.zeros(1, od.FOIL)
    f["body"], f["position"], f["normal"], f["area"], f["half_height"] = body, position, normal, area, half_height
    return f


def _tether(a, b, rest, k, c, pa=(0.0, 0.0, 0.0), pb=(0.0, 0.0, 0.0)):
    t = np.zeros(1, od.TETHER)
    t["body_a"], t["body_b"], t["point_a"], t["point_b"] = a, b, pa, pb
    t["rest_length"], t["stiffness"], t["damping"] = rest, k, c
    return t


def _wavy(seed, N=32):
    """Random rough maps: displacement up to 0.3 m, normals, and velocities up to 1 m/s."""
    rng = np.random.default_rng(seed)
    disp = np.zeros((1, N, N, 4), np.float16)
    disp[0, :, :, :3] = rng.uniform(-0.3, 0.3, (N, N, 3))
    nrm = np.zeros((1, N, N, 4), np.float16)
    nrm[0, :, :, :2] = rng.uniform(-0.2, 0.2, (N, N, 2))
    vel = np.zeros((1, N, N, 4), np.float16)
    vel[0, :, :, :3] = rng.uniform(-1, 1, (N, N, 3))
    return disp, nrm, vel, np.array([[1.0 / 16.0, 1.0 / 16.0, 1.0, 1.0]], np.float32)


def _run(maps, bodies, states, hull, cda, steps, dt=1.0 / 30.0, substeps=1, **drive):
    disp, nrm, vel, sc = maps
    for _ in range(steps):
        out = od.simulate(disp, nrm, vel, bodies, states, hull, cda, sc, RHO, dt, substeps, **drive)
        states = out[0]
    return out


def _fleet(seed, n=40):
    rng = np.random.default_rng(seed)
    b, s, hull, cda = _boats(n, [(rng.uniform(0, 30), rng.uniform(-0.3, 0.6), rng.uniform(0, 30)) for _ in range(n)])
    q = rng.normal(size=(n, 4)) * [0.1, 1.0, 0.1, 1.0]
    s["orientation"] = q / np.linalg.norm(q, axis=1, keepdims=True)
    s["linear_velocity"] = rng.uniform(-2, 2, (n, 3))
    s["angular_velocity"] = rng.uniform(-0.5, 0.5, (n, 3))
    return b, s, hull, cda * rng.uniform(0.2, 1.0, len(hull)).astype(np.float32)


def test_layouts_match_the_bindings():
    from godotoceanwaves_b200.wave_generator import WaveGenerator as W
    for spec, bound, size in [(od.THRUSTER, W.THRUSTER, 36), (od.FOIL, W.FOIL, 36), (od.LOAD, W.BODY_LOAD, 24),
                              (od.TETHER, W.TETHER, 44), (od.RESULT, W.DRIVE_RESULT, 32)]:
        assert spec == bound and spec.itemsize == size


def test_no_drive_is_bodies_simulate():
    disp, nrm, vel, sc = _wavy(1)
    b, s, hull, cda = _fleet(2)
    ref = ob.simulate(disp, nrm, vel, b, s, hull, cda, sc, RHO, 1.0 / 60.0, 3)
    for kw in (dict(), dict(thrusters=np.zeros(0, od.THRUSTER), foils=np.zeros(0, od.FOIL), tethers=np.zeros(0, od.TETHER))):
        out = od.simulate(disp, nrm, vel, b, s, hull, cda, sc, RHO, 1.0 / 60.0, 3, **kw)
        assert all(x.tobytes() == y.tobytes() for x, y in zip((out[0], out[1], out[2], out[5]), ref))
        assert not out[3].tobytes().strip(b"\0") and len(out[4]) == 0


def test_bodies_with_nothing_attached_keep_the_plain_step():
    """Half the fleet carries thrusters, foils and tethers (one anchored): the other half is bodies.simulate's bit for bit, and
    so is a body whose only tether is slack, and one whose only thruster is dry."""
    disp, nrm, vel, sc = _wavy(3)
    b, s, hull, cda = _fleet(4, 40)
    rng = np.random.default_rng(5)
    th = np.concatenate([_thruster(i, rng.uniform(100, 3000), rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3)) for i in range(0, 20, 2)])
    fo = np.concatenate([_foil(i, rng.uniform(0.1, 2), rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3)) for i in range(1, 20, 2)])
    te = np.concatenate([_tether(i, i + 1, 0.5, 5e4, 300.0, rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3)) for i in range(0, 18, 3)] +
                        [_tether(19, -1, 1.0, 1e4, 100.0, (0.5, 0, 0), (0.0, 0.0, 0.0))] +
                        [_tether(30, -1, 1e3, 1e4, 0.0, (0, 0, 0), (5.0, 0.0, 5.0))] +                 # slack
                        [_tether(31, 32, 1e3, 1e4, 0.0)])                                               # slack
    dry = _thruster(33, 5000.0, (0.0, 50.0, 0.0))                                                      # 50 m up: dry
    ref = ob.simulate(disp, nrm, vel, b, s, hull, cda, sc, RHO, 1.0 / 60.0, 2)
    out = od.simulate(disp, nrm, vel, b, s, hull, cda, sc, RHO, 1.0 / 60.0, 2, thrusters=np.concatenate([th, dry]), foils=fo, tethers=te)
    free = np.arange(20, 40)
    assert out[0][free].tobytes() == ref[0][free].tobytes() and out[5][free].tobytes() == ref[3][free].tobytes()
    assert out[1][free].tobytes() == ref[1][free].tobytes() and out[2][free].tobytes() == ref[2][free].tobytes()
    driven = np.arange(0, 20)
    assert np.all(np.any(out[0][driven]["linear_velocity"] != ref[0][driven]["linear_velocity"], 1))
    assert np.all(out[4][:-2] > 0) and np.all(out[4][-2:] == 0)
    assert not out[3][free].tobytes().strip(b"\0")


def test_slack_tether_and_dry_thruster_add_nothing():
    maps = _maps()
    b, s, hull, cda = _boats(2)
    s["linear_velocity"][0] = (1.0, 0.0, -0.5)
    base = _run(maps, b, s, hull, cda, 3, thrusters=_thruster(1, 0.0))
    slack = _run(maps, b, s, hull, cda, 3, thrusters=_thruster(1, 0.0), tethers=np.concatenate([_tether(0, 1, 20.0, 1e5, 1e3),
                                                                                               _tether(0, -1, 50.0, 1e5, 0.0)]))
    assert slack[0].tobytes() == base[0].tobytes() and slack[3].tobytes() == base[3].tobytes() and not slack[4].any()
    for y in (0.25 + 1.0 + 1e-3, 30.0):                         # more than half_height above the water (body at 0.25)
        dry = _run(maps, b, s, hull, cda, 3, thrusters=np.concatenate([_thruster(1, 0.0), _thruster(0, 4000.0, (0.0, y - 0.25, 0.0))]))
        assert dry[0].tobytes() == base[0].tobytes() and dry[3].tobytes() == base[3].tobytes()
    # centred on the water line: half the thrust (f = 0.5 exactly)
    half = _run(maps, b, s, hull, cda, 1, thrusters=_thruster(0, 4000.0, (0.0, -0.25, 0.0), (0.0, 0.0, 1.0), 0.5))
    assert half[3]["force"][0].tolist() == [0.0, 0.0, 2000.0]
    assert half[3]["torque"][0].tolist() == [-500.0, 0.0, 0.0]    # r x F, r = (0, -0.25, 0)


def _speed(states):
    return float(np.linalg.norm(states["linear_velocity"][0].astype(np.float64)))


def test_thruster_terminal_speed():
    """|drive force| = 1/2 rho A_w U^2 with A_w the drag record's wetted area."""
    maps = _maps()
    b, s, hull, cda = _boats(1)
    s, hyd, drg, drv, _, _ = _run(maps, b, s, hull, cda, 600, thrusters=_thruster(0, 5000.0))
    U = _speed(s)
    Fd = float(np.linalg.norm(drv["force"][0].astype(np.float64)))
    assert Fd == pytest.approx(0.375 * 5000.0, rel=1e-6)
    assert U == pytest.approx(math.sqrt(Fd / (0.5 * RHO * float(drg["wetted_drag_area"][0]))), rel=1e-3)
    assert abs(float(s["position"][0, 1]) - 0.25) < 1e-4 and np.abs(s["angular_velocity"]).max() < 1e-6


def test_keel_side_speed():
    """A lateral load F across a keel: F = 1/2 rho (A_w + wetted_foil_area) U^2."""
    maps = _maps()
    b, s, hull, cda = _boats(1)
    load = np.zeros(1, od.LOAD)
    load["force"] = (0.0, 0.0, 3000.0)
    s, hyd, drg, drv, _, _ = _run(maps, b, s, hull, cda, 600, foils=_foil(0, 4.0), loads=load)
    U = _speed(s)
    area = float(drg["wetted_drag_area"][0]) + float(drv["wetted_foil_area"][0])
    assert float(drv["wetted_foil_area"][0]) == 0.375 * 4.0
    assert U == pytest.approx(math.sqrt(3000.0 / (0.5 * RHO * area)), rel=1e-3)
    assert float(drv["max_normal_speed"][0]) == pytest.approx(U, rel=1e-3)


def test_mooring_extension():
    """A body moored to a world anchor 6 m away under a steady load F away from it settles at extension F / k."""
    maps = _maps()
    b, s, hull, cda = _boats(1, [(0.0, 0.25, 0.0)])
    load = np.zeros(1, od.LOAD)
    load["force"] = (-2000.0, 0.0, 0.0)
    k = 4000.0
    s, hyd, drg, drv, ten, _ = _run(maps, b, s, hull, cda, 900, tethers=_tether(0, -1, 6.0, k, 2000.0, pb=(6.0, 0.25, 0.0)), loads=load)
    ext = (6.0 - float(s["position"][0, 0])) - 6.0
    assert ext == pytest.approx(2000.0 / k, rel=1e-3)
    assert float(ten[0]) == pytest.approx(2000.0, rel=1e-3)


def test_tow_line_tension():
    """A follower towed by a thrusting leader: the line carries 1/2 rho A_w,follower U^2."""
    maps = _maps()
    b, s, hull, cda = _boats(2, [(0.0, 0.25, 0.0), (-8.0, 0.25, 0.0)])
    s, hyd, drg, drv, ten, _ = _run(maps, b, s, hull, cda, 900, thrusters=_thruster(0, 6000.0), tethers=_tether(0, 1, 6.0, 2e4, 5e3))
    U = float(s["linear_velocity"][1, 0])
    assert float(s["linear_velocity"][0, 0]) == pytest.approx(U, rel=1e-4)
    assert float(ten[0]) == pytest.approx(0.5 * RHO * float(drg["wetted_drag_area"][1]) * U * U, rel=1e-3)


def _hanging(n, k_over_m, h, stretch=0.1, jitter=0.01):
    """n ballistic bodies (no hull points) of 100 kg hanging in a chain of 1 m lines from a world anchor at the origin, the last
    pulled down by a load that stretches every line by at least `stretch`, so that all stay taut; each starts at its
    equilibrium displaced by up to `jitter` per axis.  Returns (bodies, states, tethers, loads, equilibrium positions)."""
    m, G = 100.0, 9.81
    k = k_over_m * m / (h * h)
    b = np.zeros(n, ob.BODY)
    b["mass"], b["inertia"] = m, (10.0, 10.0, 10.0)
    loads = np.zeros(n, od.LOAD)
    loads["force"][-1] = (0.0, -k * stretch, 0.0)
    ext = (k * stretch + m * G * (n - np.arange(n))) / k           # line j carries the load and the bodies below it
    eq = np.zeros((n, 3))
    eq[:, 1] = -np.cumsum(1.0 + ext)
    s = np.zeros(n, ob.STATE)
    s["orientation"] = (0.0, 0.0, 0.0, 1.0)
    s["position"] = eq + np.random.default_rng(n).uniform(-jitter, jitter, (n, 3))
    te = np.concatenate([_tether(0, -1, 1.0, k, 0.0)] + [_tether(i, i - 1, 1.0, k, 0.0) for i in range(1, n)])
    return b, s, te, loads, eq


@pytest.mark.parametrize("n", [1, 32])
def test_stiff_tethers_stay_bounded(n):
    """10^4 sub-steps at h^2 k / m = 100 (explicit Euler diverges past h^2 k / m = 4): one body on an anchor, and a chain of
    32 hanging from one, undamped and taut throughout: only the step's bound keeps them, and the motion stays within a few
    times the initial displacement."""
    h = 1.0 / 60.0
    b, s, te, loads, eq = _hanging(n, 100.0, h)
    disp, nrm, vel, sc = _maps()
    worst = 0.0
    for _ in range(100):
        s, _, _, _, ten, _ = od.simulate(disp, nrm, vel, b, s, np.zeros(0, od.bu.POINT), np.zeros(0, np.float32), sc, RHO, 100 * h, 100,
                                         tethers=te, loads=loads)
        assert np.isfinite(s["position"]).all() and np.all(ten > 0)
        worst = max(worst, float(np.abs(s["position"] - eq).max()))
    assert worst < 0.1


def test_rudder_turns_the_boat_to_its_side():
    """A thrusting boat with a keel and a stern rudder at delta: the bow swings towards the side the rudder's trailing edge is
    deflected to (yaw rate of the opposite sign to delta about +y), faster for larger |delta|."""
    maps = _maps()
    rates = {}
    for deg in (-20, -10, -5, 5, 10, 20):
        d = math.radians(deg)
        b, s, hull, cda = _boats(1)
        fo = np.concatenate([_foil(0, 2.0), _foil(0, 1.0, (math.sin(d), 0.0, math.cos(d)), (-2.0, 0.0, 0.0))])
        out = _run(maps, b, s, hull, cda, 240, thrusters=_thruster(0, 3000.0), foils=fo)
        rates[deg] = float(out[0]["angular_velocity"][0, 1])
    for deg in (5, 10, 20):
        assert rates[deg] < 0 < rates[-deg]
    assert abs(rates[5]) < abs(rates[10]) < abs(rates[20])
    assert abs(rates[-5]) < abs(rates[-10]) < abs(rates[-20])
