"""CPU checks of the wake coupling's specification (oracle/wake_coupling.py): a zero wake changes no record, a body at rest
over its own depression feels exactly nothing of the wake, the priming rule, and each snapshot sampled in its own window."""
import numpy as np

from oracle import bodies as ob
from oracle import buoyancy as bu
from oracle import drag as dr
from oracle import wake as wk
from oracle import wake_coupling as wc

f32 = np.float32


def _maps(seed, N=64, C=2, amp=0.6):
    rng = np.random.default_rng(seed)
    d = (rng.normal(size=(C, N, N, 4)) * amp).astype(np.float16)
    n = (rng.normal(size=(C, N, N, 4)) * 0.2).astype(np.float16)
    v = (rng.normal(size=(C, N, N, 4)) * 0.5).astype(np.float16)
    sc = np.array([[1 / 37.0, 1 / 37.0, 1.0, 1.0], [1 / 13.0, 1 / 13.0, 0.5, 1.0]][:C], np.float32)
    return d, n, v, sc


def _params(n, dx, damping=0.0, sponge_cells=16, sponge_damping=1.0):
    p = np.zeros((), wk.PARAMS)
    p["size"], p["cell_size"], p["damping"], p["sponge_cells"], p["sponge_damping"] = n, dx, damping, sponge_cells, sponge_damping
    return p


def _box_hull(side=2.0, cells=4, height=1.0):
    """cells x cells vertical columns of a side x side box, each reaching height / 2 above and below the body origin."""
    c = (np.arange(cells) + 0.5) * (side / cells) - side / 2
    X, Z = np.meshgrid(c, c, indexing="ij")
    p = np.zeros(X.size, bu.POINT)
    p["position"][:, 0], p["position"][:, 2] = X.ravel(), Z.ravel()
    p["volume"] = (side / cells) ** 2 * height
    p["half_height"] = height / 2
    return p


def _equal(a, b):
    """Field by field ==, a NaN meeting a NaN (so +0 and -0 match)."""
    a, b = np.asarray(a), np.asarray(b)
    for name in a.dtype.names or (None,):
        x = (a[name] if name else a).astype(np.float64)
        y = (b[name] if name else b).astype(np.float64)
        if not np.all((x == y) | (np.isnan(x) & np.isnan(y))):
            return False
    return True


def _scene(seed, B=6):
    rng = np.random.default_rng(seed)
    hull = _box_hull()
    tbl = np.zeros(B, bu.BODY)
    tbl["transform"] = np.tile(np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], np.float32), (B, 1))
    tbl["transform"][:, 3] = rng.uniform(-20, 80, B)
    tbl["transform"][:, 7] = rng.uniform(-0.5, 0.5, B)
    tbl["transform"][:, 11] = rng.uniform(-20, 80, B)
    tbl["num_points"] = len(hull)
    tbl["num_points"][-1] = 0
    vel = np.zeros(B, dr.VELOCITY)
    vel["linear"] = rng.uniform(-1, 1, (B, 3))
    vel["angular"] = rng.uniform(-0.5, 0.5, (B, 3))
    return tbl, vel, hull, np.full(len(hull), 0.3, np.float32)


def test_zero_wake_changes_no_record():
    d, n, v, sc = _maps(1)
    tbl, vel, hull, cda = _scene(2)
    cp = wc.Coupling(128, 0.5)
    cp.primed, cp.T = True, f32(1 / 60)                     # primed, e = e_old = 0
    pts = np.random.default_rng(3).uniform(-30, 90, (200, 2)).astype(np.float32)
    pts[:3] = [[np.nan, 1.0], [np.inf, 0.0], [5.0, -np.inf]]
    assert _equal(wc.query_surface(d, n, pts, sc, wake=cp), wc.query_surface(d, n, pts, sc))
    h1, s1 = wc.buoyancy(d, n, tbl, hull, sc, return_samples=True, wake=cp)
    h0, s0 = bu.buoyancy(d, n, tbl, hull, sc, return_samples=True)
    assert _equal(h1, h0) and _equal(s1, s0)
    a1 = wc.body_forces(d, n, v, tbl, vel, hull, cda, sc, return_samples=True, wake=cp)
    a0 = dr.body_forces(d, n, v, tbl, vel, hull, cda, sc, return_samples=True)
    assert all(_equal(x, y) for x, y in zip(a1, a0))
    fb = np.zeros(len(tbl), ob.BODY)
    fb["mass"], fb["inertia"], fb["num_points"] = 1500.0, (900.0, 1200.0, 900.0), tbl["num_points"]
    st = np.zeros(len(tbl), ob.STATE)
    st["position"] = tbl["transform"][:, [3, 7, 11]]
    st["orientation"] = (0.0, 0.0, 0.0, 1.0)
    st["linear_velocity"] = vel["linear"]
    r1 = wc.simulate(d, n, v, fb, st, hull, cda, sc, substeps=3, wake=cp)
    r0 = ob.simulate(d, n, v, fb, st, hull, cda, sc, substeps=3)
    assert all(_equal(x, y) for x, y in zip(r1, r0))


def _rest_layer(n=128, dx=0.5, at=(32.0, 32.0)):
    """A layer at rest under a stationary body-attached source (damping 0): h = h_prev = -phi."""
    p = _params(n, dx, damping=0.0, sponge_cells=16, sponge_damping=1.0)
    L = wk.Layer(p)
    src = np.zeros(1, wk.SOURCE)
    src["radius"], src["head"], src["body"] = 2.0, 0.5, 0
    st = np.zeros(1, wk.STATE)
    st["position"] = (at[0], 0.0, at[1])
    st["orientation"] = (0.0, 0.0, 0.0, 1.0)
    phi = wk.rasterise(n, dx, (0, 0), src, st, 0.0)
    L.h, L.h_prev = -phi, -phi.copy()
    return L, src, st, phi


def test_rest_state_reads_nothing_of_the_wake():
    L, src, st, phi = _rest_layer()
    assert phi.max() > 0.45
    h0 = L.h.copy()
    cp = wc.Coupling(L.n, L.cell_size)
    for _ in range(3):
        wc.step(L, cp, 1 / 60, 2, (0, 0), src, st)
    assert np.array_equal(L.h, h0) and np.array_equal(L.h_prev, h0)       # the layer does not move (-0 where phi = 0 becomes +0)
    assert np.all(cp.e == 0.0) and np.all(cp.e_old == 0.0)
    # the body that carries the source: flat maps, coupled forces equal the uncoupled ones
    N, C = 64, 2
    d = np.zeros((C, N, N, 4), np.float16)
    nm = np.zeros((C, N, N, 4), np.float16)
    v = np.zeros((C, N, N, 4), np.float16)
    sc = np.array([[1 / 37.0, 1 / 37.0, 1.0, 1.0], [1 / 13.0, 1 / 13.0, 0.5, 1.0]], np.float32)
    hull = _box_hull()
    tbl = np.zeros(1, bu.BODY)
    tbl["transform"] = [1, 0, 0, 32.0, 0, 1, 0, 0.1, 0, 0, 1, 32.0]
    tbl["num_points"] = len(hull)
    vel = np.zeros(1, dr.VELOCITY)
    vel["linear"] = (0.0, -0.3, 0.0)
    cda = np.full(len(hull), 0.25, np.float32)
    a1 = wc.body_forces(d, nm, v, tbl, vel, hull, cda, sc, return_samples=True, wake=cp)
    a0 = dr.body_forces(d, nm, v, tbl, vel, hull, cda, sc, return_samples=True)
    assert all(_equal(x, y) for x, y in zip(a1, a0))
    w = bu.world_points(tbl, hull)[3]
    Q = np.stack([w[:, 0], w[:, 2]], 1)
    assert np.all(wc.vertical_velocity(Q, cp, cp.cell_size) == 0.0)
    # reading h instead would see the depression under the hull
    assert wk.sample(L.h, L.cell_size, L.origin, Q)[:, 0].max() < -0.1


def test_priming_rule():
    p = _params(128, 0.5)
    L = wk.Layer(p)
    cp = wc.Coupling(128, 0.5)
    src = np.zeros(2, wk.SOURCE)
    src["x"], src["z"], src["vx"], src["radius"], src["head"], src["body"] = (20, 40), (30, 35), (2.5, -1.0), 3.0, (0.3, -0.2), -1
    assert not wc.live(cp) and np.all(cp.e == 0) and np.all(cp.e_old == 0) and cp.T == 0
    rng = np.random.default_rng(5)
    Q = rng.uniform(0, 64, (300, 2)).astype(np.float32)
    for rounds in range(2):
        wc.step(L, cp, 0.05, 2, (0, 0), src)
        assert wc.live(cp) and cp.T == f32(2) * wk.substep(0.05, 2)
        assert cp.e.tobytes() == cp.e_old.tobytes() and np.abs(cp.e).max() > 0
        assert np.all(wc.vertical_velocity(Q, cp, cp.cell_size) == 0.0)
        wc.step(L, cp, 0.05, 2, (0, 0), src)
        assert np.abs(wc.vertical_velocity(Q, cp, cp.cell_size)).max() > 0
        cp.reset()                                          # ocean_wake_set_state: unprimed again
        L.h, L.h_prev = L.h.copy(), L.h_prev.copy()
        assert not wc.live(cp) and np.all(cp.e == 0) and cp.T == 0


def test_scroll_samples_e_old_in_its_own_window():
    p = _params(128, 0.5)
    L = wk.Layer(p)
    cp = wc.Coupling(128, 0.5)
    src = np.zeros(1, wk.SOURCE)
    src["x"], src["z"], src["vx"], src["radius"], src["head"], src["body"] = 30.0, 30.0, 2.0, 4.0, 0.4, -1
    wc.step(L, cp, 0.1, 2, (0, 0), src)
    wc.step(L, cp, 0.1, 2, (10, -6), src)
    assert cp.origin_old == (0, 0) and cp.origin_e == (10, -6)
    rng = np.random.default_rng(9)
    Q = rng.uniform(-10, 75, (400, 2)).astype(np.float32)
    a = wk.sample(cp.e, 0.5, (10, -6), Q)[:, 0]
    b = wk.sample(cp.e_old, 0.5, (0, 0), Q)[:, 0]
    wv = wc.vertical_velocity(Q, cp, cp.cell_size)
    assert wv.tobytes() == ((a - b) / cp.T).tobytes()
    # points inside e's window but outside e_old's read 0 from e_old
    only_new = (Q[:, 0] >= 64.0) & (Q[:, 0] < 69.0) & (Q[:, 1] >= -3.0) & (Q[:, 1] < 61.0)
    assert only_new.any() and np.all(b[only_new] == 0.0)
    assert wv.tobytes() != (wc.vertical_velocity(Q, _same_window(cp), cp.cell_size)).tobytes()


def _same_window(cp):
    """cp with e_old read in e's window, as a coupling that ignored the scroll would."""
    c = wc.Coupling(cp.n, cp.cell_size)
    c.e, c.e_old, c.origin_e, c.origin_old, c.T, c.primed = cp.e, cp.e_old, cp.origin_e, cp.origin_e, cp.T, True
    return c


def test_a_body_reading_h_would_sink_into_its_own_wake():
    """The self-wake scene of test_gpu_wake_coupling on the specification, with a coupling whose e is h instead of h + phi:
    flat sea, a 2 m x 2 m box of 0.5 m draft carrying its own source (radius 2 m, head 0.5 m), a 256-cell window of 0.5 m,
    damping 0 and a 48-cell sponge ramping to 1 / s, released 0.1 m above its equilibrium (height 0) and run 30 s of
    body-then-wake ticks at 1 / 60 s.  The body sinks into the depression of its own source; the coupled library keeps its
    mean height within 1 cm of the uncoupled run's, so that check tells the two apart."""
    dt = 1.0 / 60.0
    L = wk.Layer(_params(256, 0.5, damping=0.0, sponge_cells=48, sponge_damping=1.0))
    src = np.zeros(1, wk.SOURCE)
    src["radius"], src["head"], src["body"] = 2.0, 0.5, 0
    hull = _box_hull(2.0, 4, 1.0)
    fb = np.zeros(1, ob.BODY)
    fb["mass"] = 1025.0 * 2.0 * 2.0 * 0.5
    fb["inertia"] = fb["mass"] * np.array([5.0, 8.0, 5.0]) / 12.0
    fb["num_points"] = len(hull)
    s = np.zeros(1, ob.STATE)
    s["position"], s["orientation"] = (64.0, 0.1, 64.0), (0.0, 0.0, 0.0, 1.0)
    cda = np.full(len(hull), 0.5 * 0.25, np.float32)
    flat = np.zeros((2, 64, 64, 4), np.float16)
    sc = np.array([[1 / 37.0, 1 / 37.0, 1.0, 1.0], [1 / 13.0, 1 / 13.0, 0.5, 1.0]], np.float32)
    cp = wc.Coupling(256, 0.5)
    ys = []
    for _ in range(int(round(30.0 / dt))):
        with np.errstate(all="ignore"):
            s = wc.simulate(flat, flat, flat, fb, s, hull, cda, sc, 1025.0, dt, 1, wake=cp)[0]
        L.step(dt, 1, (0, 0), src, s)
        cp.e_old, cp.origin_old = (cp.e if cp.primed else L.h.copy()), L.origin
        cp.e, cp.origin_e, cp.T, cp.primed = L.h.copy(), L.origin, f32(dt), True
        ys.append(float(s["position"][0, 1]))
    mean = float(np.mean(ys[-600:]))
    print(f"reading h: mean height over the last 10 s {mean:+.4f} m (equilibrium 0, head 0.5 m)")
    assert np.all(np.isfinite(ys)) and mean < -0.1
