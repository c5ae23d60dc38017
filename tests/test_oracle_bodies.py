"""The floating-body integrator's specification (oracle/bodies.py) against closed forms and physical properties: free fall,
torque-free spin, exact rest at equilibrium, settling and the heave period, self-righting, the stiff-drag bound, and
sub-step composition."""
import math

import numpy as np

from oracle import bodies as ob
from oracle import buoyancy as bu
from test_oracle_buoyancy import _box

F = np.float32
G = F(9.81)
RHO = 1024.0                                                    # a power of two: (rho G) V == (rho V) G for dyadic V


def _maps(N=64, current=None):
    """Flat, still maps (zero displacement and normal), and velocity maps of a uniform current (zero by default)."""
    disp = np.zeros((1, N, N, 4), np.float16)
    vel = np.zeros((1, N, N, 4), np.float16)
    if current is not None:
        vel[0, :, :, :3] = np.asarray(current, np.float16)
    return disp, disp.copy(), vel, np.array([[1.0 / 64.0, 1.0 / 64.0, 1.0, 1.0]], np.float32)


def _body(mass, inertia, first=0, count=0):
    b = np.zeros(1, ob.BODY)
    b["mass"], b["inertia"], b["first_point"], b["num_points"] = mass, inertia, first, count
    return b


def _state(position=(0.0, 0.0, 0.0), orientation=(0.0, 0.0, 0.0, 1.0), linear=(0.0, 0.0, 0.0), angular=(0.0, 0.0, 0.0)):
    s = np.zeros(1, ob.STATE)
    s["position"], s["orientation"], s["linear_velocity"], s["angular_velocity"] = position, orientation, linear, angular
    return s


def _run(maps, bodies, states, hull, cda, dt, substeps, calls, density=RHO):
    disp, nrm, vel, sc = maps
    out = []
    for _ in range(calls):
        states, hyd, drg, T = ob.simulate(disp, nrm, vel, bodies, states, hull, cda, sc, density, dt, substeps)
        out.append(states.copy())
    return states, out


def test_layouts_match_the_bindings():
    from godotoceanwaves_b200.wave_generator import WaveGenerator
    for dt, wg, size in [(ob.BODY, WaveGenerator.FLOATING_BODY, 24), (ob.STATE, WaveGenerator.BODY_STATE, 52)]:
        assert dt.itemsize == wg.itemsize == size
        assert dt.names == wg.names
        for name in dt.names:
            assert dt.fields[name][1] == wg.fields[name][1], name
    assert WaveGenerator.FLOATING_BODY == ob.BODY and WaveGenerator.BODY_STATE == ob.STATE


def test_rotation_is_the_unit_quaternion_rotation():
    rng = np.random.default_rng(1)
    q = rng.normal(size=(200, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    R = ob.rotation(q.astype(np.float32)).astype(np.float64)
    x, y, z, w = q.T
    ref = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                    2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                    2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    assert np.abs(R - ref).max() < 1e-6
    assert np.abs(R @ R.transpose(0, 2, 1) - np.eye(3)).max() < 1e-6


def test_free_fall_is_the_binary32_recurrence_and_the_closed_form():
    maps = _maps()
    hull = _box(1, 1, 1)                                        # unused: the body has no hull points
    b = _body(2.5, (1.0, 1.0, 1.0))
    s0 = _state(position=(3.0, 500.0, -2.0))
    s, _ = _run(maps, b, s0, hull, np.zeros(len(hull), np.float32), 1.0, 60, 10)   # 600 sub-steps of 1/60 s
    h = F(1.0) / F(60)
    m = F(2.5)
    vy, py = F(0.0), F(500.0)
    for _ in range(600):
        vy = vy + (h / m) * (F(0.0) - m * G)
        py = py + h * vy
    assert s["linear_velocity"][0, 1] == vy and s["position"][0, 1] == py
    assert s["linear_velocity"][0, 0] == 0 and s["linear_velocity"][0, 2] == 0
    assert s["position"][0, 0] == F(3.0) and s["position"][0, 2] == F(-2.0)
    assert abs(float(vy) + 9.81 * 10.0) <= 1e-4 * 9.81 * 10.0
    assert s["orientation"].tolist() == [[0.0, 0.0, 0.0, 1.0]]


def test_torque_free_spin_about_a_principal_axis():
    """w' = R (R^T w) is not exact in binary32: |w| within 1e-4, the quaternion norm within 1e-6 of 1, and the angle within
    the quaternion update's truncation bound n (h |w|)^3 / 12 of |w| t."""
    maps = _maps()
    hull = _box(1, 1, 1)
    b = _body(3.0, (1.0, 2.0, 3.0))
    wmag = 2.0
    s = _state(angular=(0.0, wmag, 0.0))
    h = float(F(0.1) / F(50))
    n = 0
    for _ in range(200):                                       # 10^4 sub-steps
        s, _ = _run(maps, b, s, hull, np.zeros(len(hull), np.float32), 0.1, 50, 1)
        n += 50
    w = s["angular_velocity"][0].astype(np.float64)
    q = s["orientation"][0].astype(np.float64)
    assert abs(np.linalg.norm(w) - wmag) <= 1e-4 * wmag
    assert abs(np.linalg.norm(q) - 1.0) <= 1e-6
    assert abs(w[0]) < 1e-4 and abs(w[2]) < 1e-4
    angle = 2.0 * math.atan2(q[1], q[3])                        # about +y
    expected = wmag * h * n
    err = (angle - expected + math.pi) % (2 * math.pi) - math.pi
    assert abs(err) <= n * (h * wmag) ** 3 / 12 + 1e-4
    assert s["position"].tolist() != [[0.0, 0.0, 0.0]]          # gravity acts on a ballistic body too


def _float_box():
    """A 2 m x 1 m x 2 m box of four 1 m columns; at mass 1024 kg in water of density 1024 its draft is 0.25 m, with the
    origin (its centre) at y = 0.25."""
    hull = _box(2, 1, 2, 1.0)
    b = _body(1024.0, (1024.0 * 5 / 12, 1024.0 * 8 / 12, 1024.0 * 5 / 12), 0, len(hull))
    return b, hull


def test_box_at_equilibrium_stays_exactly_at_rest():
    maps = _maps()
    b, hull = _float_box()
    s0 = _state(position=(10.0, 0.25, -7.0))
    s, _ = _run(maps, b, s0, hull, np.full(len(hull), 1.0, np.float32), 1.0 / 60.0, 4, 30)
    assert s.tobytes() == s0.tobytes()


def test_settling_and_heave_period():
    maps = _maps()
    b, hull = _float_box()
    # released 0.3 m high, heavily damped: it settles at the draft m / (rho A)
    s, hist = _run(maps, b, _state(position=(0.0, 0.55, 0.0)), hull, np.full(len(hull), 8.0, np.float32), 1.0 / 60.0, 1, 1200)
    draft = 1024.0 / (RHO * 4.0)
    assert abs(float(s["position"][0, 1]) - (0.5 - draft)) < 0.01
    assert abs(float(s["linear_velocity"][0, 1])) < 0.05
    # small-amplitude heave without drag, 8 sub-steps of 1/60 s: the period is 2 pi sqrt(m / (rho G A))
    s, hist = _run(maps, b, _state(position=(0.0, 0.27, 0.0)), hull, np.zeros(len(hull), np.float32), 1.0 / 60.0, 8, 240)
    y = np.array([float(h["position"][0, 1]) for h in hist]) - 0.25
    ups = [i + y[i] / (y[i] - y[i + 1]) for i in range(len(y) - 1) if y[i] > 0 >= y[i + 1]]
    assert len(ups) >= 3
    period = float(np.mean(np.diff(ups))) / 60.0
    expected = 2 * math.pi * math.sqrt(1024.0 / (RHO * 9.81 * 4.0))
    assert abs(period - expected) <= 0.02 * expected


def test_rolled_wide_box_rights_itself():
    maps = _maps()
    hull = _box(8, 2, 4, 0.5)                                  # 4 m wide, 1 m high, 2 m deep
    m = 2048.0                                                  # draft 0.25 m
    b = _body(m, (m * 5 / 12, m * 20 / 12, m * 17 / 12), 0, len(hull))
    a = 0.3
    s0 = _state(position=(0.0, 0.25, 0.0), orientation=(0.0, 0.0, math.sin(a / 2), math.cos(a / 2)))   # rolled about z
    s, hist = _run(maps, b, s0, hull, np.full(len(hull), 0.25, np.float32), 1.0 / 60.0, 4, 300)
    roll = np.array([2 * math.atan2(float(h["orientation"][0, 2]), float(h["orientation"][0, 3])) for h in hist])
    assert np.all(np.isfinite(roll))
    assert roll.min() < 0.1                                     # it swings back through upright
    assert np.abs(roll[-60:]).max() < 0.5 * a                   # and the swing decays over the 5 s
    assert np.abs(roll[-60:]).max() < np.abs(roll[60:120]).max()


def test_stiff_drag_never_overshoots_the_current():
    """A 0.05 kg neutrally buoyant point body with C_d A 0.5 m^2, fully submerged in a 1 m/s current, 1 sub-step of 1/30 s:
    explicit Euler would overshoot the current 170-fold on the first step; the bounded step approaches it monotonically."""
    u = 1.0
    maps = _maps(current=(u, 0.0, 0.0))
    hull = np.zeros(1, bu.POINT)
    hull["volume"] = F(0.05) / F(RHO)                           # mass = rho V exactly: no net vertical force
    hull["half_height"] = 0.5
    b = _body(0.05, (1e-3, 1e-3, 1e-3), 0, 1)
    cda = np.full(1, 0.5, np.float32)
    s0 = _state(position=(0.0, -5.0, 0.0))
    s, hist = _run(maps, b, s0, hull, cda, 1.0 / 30.0, 1, 90)
    vx = np.array([float(h["linear_velocity"][0, 0]) for h in hist])
    assert np.all(np.diff(np.concatenate([[0.0], vx])) >= 0) and np.all(vx <= u)
    assert u - vx[-1] <= 1e-3
    assert all(float(h["linear_velocity"][0, 1]) == 0.0 for h in hist)
    # the same first step explicitly: F = 1/2 rho C_d A |u| u
    force = 0.5 * RHO * 0.5 * u * u
    explicit = 0.0 + (1.0 / 30.0) / 0.05 * force
    assert explicit > 100 * u
    assert 0 < vx[0] < u


def test_substeps_compose_bit_for_bit():
    """S sub-steps of dt equal S calls of (dt / S in binary32, 1 sub-step), on a scene with wet, dry and ballistic bodies."""
    maps = _maps(current=(0.5, 0.0, -0.25))
    hull = _box(4, 2, 2, 0.5)
    rng = np.random.default_rng(5)
    n = 6
    b = np.zeros(n, ob.BODY)
    b["mass"] = rng.uniform(200, 900, n) * 2.0
    b["inertia"] = rng.uniform(100, 400, (n, 3))
    b["num_points"] = len(hull)
    b["num_points"][2] = 0
    s = np.zeros(n, ob.STATE)
    s["position"] = np.stack([rng.uniform(-20, 20, n), rng.uniform(-0.5, 0.8, n), rng.uniform(-20, 20, n)], 1)
    q = rng.normal(size=(n, 4)) * np.array([0.1, 0.1, 0.1, 1.0])
    s["orientation"] = q / np.linalg.norm(q, axis=1, keepdims=True)
    s["linear_velocity"] = rng.uniform(-1, 1, (n, 3))
    s["angular_velocity"] = rng.uniform(-0.5, 0.5, (n, 3))
    cda = rng.uniform(0.05, 0.3, len(hull)).astype(np.float32)
    disp, nrm, vel, sc = maps
    a, ha, da, Ta = ob.simulate(disp, nrm, vel, b, s, hull, cda, sc, RHO, 1.0 / 60.0, 5)
    c = s
    for _ in range(5):
        c, hc, dc, Tc = ob.simulate(disp, nrm, vel, b, c, hull, cda, sc, RHO, F(1.0 / 60.0) / F(5), 1)
    assert a.tobytes() == c.tobytes() and ha.tobytes() == hc.tobytes() and da.tobytes() == dc.tobytes() and Ta.tobytes() == Tc.tobytes()
    assert Ta.tobytes() == ob.transforms(a).tobytes()
    assert np.count_nonzero(ha["submerged_volume"]) >= 3 and not ha[2].tobytes().strip(b"\0")
