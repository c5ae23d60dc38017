"""GPU tests of the wake coupling (include/ocean.h, "Wake layer", ocean_wake_set_coupling): the surface query, buoyancy, body
forces and the body integrator byte-identical to the specification oracle/wake_coupling.py on coupled wake layers, with
body-attached sources driven by device states and scrolled windows; off means off; launch counts, device memory and
arguments; isolation from the cascades; and two physics checks, a body over its own wake and a body in a passing wake."""
import ctypes

import numpy as np
import pytest

from oracle import bodies as ob
from oracle import buoyancy as bu
from oracle import wake as wk
from oracle import wake_coupling as wc
from test_gpu_bodies import _bodies
from test_gpu_sampling import _gen

pytestmark = pytest.mark.gpu

INVALID, STATE = 1, 4
RHO = 1025.0
DT = 1.0 / 60.0


def _params(n, dx, damping=0.0, sponge_cells=16, sponge_damping=1.0):
    p = np.zeros((), wk.PARAMS)
    p["size"], p["cell_size"], p["damping"], p["sponge_cells"], p["sponge_damping"] = n, dx, damping, sponge_cells, sponge_damping
    return p


def _init(g, p):
    g.wake_init(int(p["size"]), float(p["cell_size"]), float(p["damping"]), int(p["sponge_cells"]), float(p["sponge_damping"]))


def _same(a, b):
    """Byte-identical, except that a NaN only has to meet a NaN (compared as float32 words)."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.tobytes() == b.tobytes():
        return True
    wa, wb = np.frombuffer(a.tobytes(), np.float32), np.frombuffer(b.tobytes(), np.float32)
    na, nb = np.isnan(wa), np.isnan(wb)
    return bool(wa.size == wb.size and np.array_equal(na, nb) and wa[~na].tobytes() == wb[~nb].tobytes())


def _points(rng, origin, n, dx, k=400):
    """World points inside, outside and straddling the window's edges, and non-finite ones."""
    x0, z0 = wk.world_origin(origin, dx)
    ext = float(np.float32(n) * np.float32(dx))
    pts = np.stack([rng.uniform(x0 - 0.1 * ext, x0 + 1.1 * ext, k), rng.uniform(z0 - 0.1 * ext, z0 + 1.1 * ext, k)], 1).astype(np.float32)
    edge = np.float32(x0 + np.float32(ext))
    extra = [[x0, z0 + 3.0], [np.nextafter(x0, np.float32(-1e9)), z0 + 3.0], [edge, z0 + 5.0], [np.nextafter(edge, np.float32(-1e9)), z0 + 5.0],
             [x0 + 0.25 * dx, z0 + 0.25 * dx], [np.nan, z0 + 1.0], [x0 + 1.0, np.inf], [-np.inf, np.nan]]
    return np.concatenate([pts, np.array(extra, np.float32)])


def _flat(N=256, C=2):
    """A generator whose maps are flat: every cascade's amplitudes set to 0, then one update."""
    gow, g, params = _gen(N, C, frames=1)
    for c in range(C):
        g.set_spectrum_amplitudes(c, np.zeros((N, N), np.complex64))
    g.update_all(1.0 / 50.0, params)
    return gow, g, params


@pytest.mark.parametrize("N,C,n", [(256, 4, 256), (1024, 3, 1024)])
def test_parity_with_the_specification(N, C, n):
    """Body-then-wake ticks through the device entry points (states never leave the device), with sub-steps S = 1 and 4 and
    the window scrolled between calls; after every call the states, records and transforms of ocean_simulate_bodies_device,
    the snapshots of ocean_wake_get_coupling and the records of ocean_query_surface (host and device), ocean_buoyancy and
    ocean_body_forces (with their samples) are byte-identical to the specification."""
    import torch
    from godotoceanwaves_b200.native import check, load_library
    lib = load_library()
    gow, g, params = _gen(N, C)
    scales = gow.WaveGenerator.map_scales(params)
    g.update_velocity()
    d16, n16 = g.maps_to_host(0, C)
    vel = g.velocity_to_host(0, C)
    dx = 0.5
    p = _params(n, dx, damping=0.02, sponge_cells=24, sponge_damping=1.0)
    _init(g, p)
    L = wk.Layer(p)
    cp = wc.Coupling(n, dx)
    g.wake_set_coupling(True)
    rng = np.random.default_rng(N + n)
    fb, s0, hull, cda = _bodies(900 + N, rng.integers(0, 24, 10))
    ext = n * dx
    s0["position"][:, 0] = rng.uniform(0.2 * ext, 0.8 * ext, len(s0))
    s0["position"][:, 2] = rng.uniform(0.2 * ext, 0.8 * ext, len(s0))
    # body 0 lies just past the first window's +x edge: once the window scrolls by +7 cells its hull is inside e's window but
    # outside e_old's, where the drag's wv reads 0 from e_old
    edge_body = int(np.argmax(fb["num_points"]))
    s0["position"][edge_body, 0] = ext + 1.0
    s0["linear_velocity"][edge_body] = 0.0
    s0["angular_velocity"][edge_body] = 0.0
    edge_reads = 0
    src = np.zeros(len(fb) + 3, wk.SOURCE)
    src["radius"], src["head"], src["body"] = 2.0, 0.25, -1
    src["body"][:len(fb)] = np.arange(len(fb))
    src["x"][len(fb):], src["z"][len(fb):] = rng.uniform(0.3 * ext, 0.7 * ext, 3), rng.uniform(0.3 * ext, 0.7 * ext, 3)
    src["vx"][len(fb):], src["vz"][len(fb):], src["radius"][len(fb):] = (2.5, -1.0, 0.5), (0.0, 2.0, -1.5), (4.0, 3.0, 2.5)
    dev = torch.device("cuda", g.device)
    st_d = torch.from_numpy(s0.view(np.uint8).copy()).to(dev)
    hull_d = torch.from_numpy(hull.view(np.uint8).copy()).to(dev)
    cda_d = torch.from_numpy(cda).to(dev)
    src_d = torch.from_numpy(src.view(np.uint8).copy()).to(dev)
    B = len(fb)
    hyd_d = torch.zeros(B * 12, dtype=torch.int32, device=dev)
    drg_d = torch.zeros(B * 8, dtype=torch.int32, device=dev)
    T_d = torch.zeros(B * 12, dtype=torch.float32, device=dev)
    sc = np.ascontiguousarray(scales, np.float32)

    def states():
        g.synchronize()
        return np.frombuffer(st_d.cpu().numpy().tobytes(), ob.STATE).copy()

    plan = [(1, 2, (0, 0)), (4, 1, (0, 0)), (1, 3, (7, -5)), (4, 2, (7, -5)), (4, 1, (-30, 21))]
    if N == 1024:                                               # the specification's surface query is slow on 1024^2 maps
        plan = [plan[0], plan[3], plan[4]]
    for call, (S, Sw, origin) in enumerate(plan):
        before = states()
        if wc.live(cp):
            table, _ = ob.pose(fb, before)
            body, _, _, w = bu.world_points(table, hull)
            q = w[body == edge_body][:, [0, 2]].astype(np.float64)

            def inside(o):
                x0, z0 = wk.world_origin(o, dx)
                return (q[:, 0] >= x0) & (q[:, 0] < x0 + ext) & (q[:, 1] >= z0) & (q[:, 1] < z0 + ext)
            edge_reads += int(np.count_nonzero(inside(cp.origin_e) & ~inside(cp.origin_old)))
        torch.cuda.synchronize()
        check(lib.ocean_simulate_bodies_device(g.context, B, fb.ctypes.data, st_d.data_ptr(), len(hull), hull_d.data_ptr(), cda_d.data_ptr(),
                                               C, sc.ctypes.data, RHO, DT, S, 1e-3, 8, hyd_d.data_ptr(), drg_d.data_ptr(), T_d.data_ptr()))
        with np.errstate(all="ignore"):
            rs, rh, rd, rT = wc.simulate(d16, n16, vel, fb, before, hull, cda, scales, RHO, DT, S, 1e-3, 8, wake=cp)
        after = states()
        assert _same(after, rs), (call, S)
        assert _same(hyd_d.cpu().numpy(), rh) and _same(drg_d.cpu().numpy(), rd) and _same(T_d.cpu().numpy(), rT), call
        check(lib.ocean_wake_step_device(g.context, DT * Sw, Sw, origin[0], origin[1], len(src), src_d.data_ptr(), B, st_d.data_ptr()))
        wc.step(L, cp, DT * Sw, Sw, origin, src, after)
        e, e_old, origins, T = g.wake_coupling()
        assert _same(e, cp.e) and _same(e_old, cp.e_old) and origins == (cp.origin_e, cp.origin_old) and T == cp.T, call
        assert np.abs(e).max() > 0
        # the ops on the coupled layer
        pts = _points(rng, origin, n, dx)
        with np.errstate(all="ignore"):
            ref = wc.query_surface(d16, n16, pts, scales, wake=cp)
        assert _same(g.query_surface(pts, scales), ref), call
        pts_d = torch.from_numpy(pts).to(dev)
        out_d = torch.zeros(len(pts) * 10, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        check(lib.ocean_query_surface_device(g.context, len(pts), pts_d.data_ptr(), C, sc.ctypes.data, 1e-3, 8, out_d.data_ptr()))
        g.synchronize()
        assert _same(out_d.cpu().numpy(), ref), call
        table, velo = ob.pose(fb, after)
        with np.errstate(all="ignore"):
            rb, rbs = wc.buoyancy(d16, n16, table, hull, scales, RHO, return_samples=True, wake=cp)
            rf = wc.body_forces(d16, n16, vel, table, velo, hull, cda, scales, RHO, return_samples=True, wake=cp)
        gb, gbs = g.buoyancy(table, hull, scales, RHO, return_samples=True)
        assert _same(gb, rb) and _same(gbs, rbs), call
        gf = g.body_forces(table, velo, hull, cda, scales, RHO, return_samples=True)
        assert all(_same(x, y) for x, y in zip(gf, rf)), call
    assert edge_reads > 0                                       # the simulate calls read wv where e_old's window ends
    g.free()


def _ops(g, scales, scene, pts):
    fb, s0, hull, cda = scene
    table, velo = ob.pose(fb, s0)
    out = [g.query_surface(pts, scales), *g.buoyancy(table, hull, scales, RHO, return_samples=True),
           *g.body_forces(table, velo, hull, cda, scales, RHO, return_samples=True)]
    out += list(g.simulate_bodies(fb, s0, hull, cda, scales, DT, 4, RHO, return_records=True, return_transforms=True))
    return [np.ascontiguousarray(x).tobytes() for x in out]


def test_off_means_off():
    """With the coupling off, after wake steps with sources, every record of the coupled ops is byte-identical to a generator
    without a wake layer; likewise after the coupling is enabled, stepped and disabled again."""
    gow, a, pa = _gen(256, 3)
    gow, b, pb = _gen(256, 3)
    scales = gow.WaveGenerator.map_scales(pa)
    rng = np.random.default_rng(21)
    scene = _bodies(311, rng.integers(1, 20, 8))
    scene[1]["position"][:, [0, 2]] = rng.uniform(10, 110, (len(scene[1]), 2))
    pts = _points(rng, (0, 0), 256, 0.5)
    _init(a, _params(256, 0.5))
    src = np.zeros(len(scene[0]), wk.SOURCE)
    src["radius"], src["head"], src["body"] = 2.0, 0.3, np.arange(len(scene[0]))
    a.wake_step(0.1, 3, (0, 0), src, scene[1])
    ref = _ops(b, scales, scene, pts)
    assert _ops(a, scales, scene, pts) == ref
    a.wake_set_coupling(True)
    a.wake_step(0.1, 3, (0, 0), src, scene[1])
    assert _ops(a, scales, scene, pts) != ref                   # the coupling reads the wake ...
    a.wake_set_coupling(False)
    a.wake_step(0.1, 3, (0, 0), src, scene[1])
    assert _ops(a, scales, scene, pts) == ref                   # ... and off it reads nothing
    a.free()
    b.free()


def test_launch_counts_and_device_memory():
    gow, g, params = _gen(256, 4)
    scales = gow.WaveGenerator.map_scales(params)
    rng = np.random.default_rng(5)
    fb, s0, hull, cda = _bodies(431, rng.integers(1, 40, 50))
    s0["position"][:, [0, 2]] = rng.uniform(10, 110, (len(s0), 2))
    table, velo = ob.pose(fb, s0)
    pts = _points(rng, (0, 0), 256, 0.5)
    n = 256
    _init(g, _params(n, 0.5))
    src = np.zeros(3, wk.SOURCE)
    src["x"], src["z"], src["radius"], src["head"], src["body"] = 40.0, 60.0, 3.0, 0.3, -1
    g.update_velocity()

    def counts(step=True, S=2):
        ops = [lambda: g.wake_step(0.05 * S, S, (0, 0), src)] if step else []
        ops += [lambda: g.query_surface(pts, scales), lambda: g.buoyancy(table, hull, scales),
                lambda: g.body_forces(table, velo, hull, cda, scales), lambda: g.simulate_bodies(fb, s0, hull, cda, scales, DT, 3)]
        out = []
        for op in ops:
            before = g.info().kernel_launches
            op()
            out.append(g.info().kernel_launches - before)
        return out

    off = [2, 3, 5, 6, 1 + 7 * 3]
    assert counts() == off
    base = g.info().device_bytes
    g.wake_set_coupling(True)
    assert g.info().device_bytes == base + 2 * 4 * n * n
    g.wake_set_coupling(True)                                   # enabling again changes nothing
    assert g.info().device_bytes == base + 2 * 4 * n * n
    assert counts(step=False) == off[1:]                        # unprimed: nothing extra
    assert counts() == [3, 4, 6, 7, 1 + 8 * 3]                  # the step primes; one more kernel per step, query and sub-step
    assert counts() == [3, 4, 6, 7, 1 + 8 * 3]
    g.set_wake_state(*g.wake_state()[:2])                       # unprimed again
    e, e_old, origins, T = g.wake_coupling()
    assert not e.any() and not e_old.any() and origins == ((0, 0), (0, 0)) and T == 0
    assert counts(step=False) == off[1:]
    g.wake_set_coupling(False)
    assert g.info().device_bytes == base
    g.wake_set_coupling(True)
    counts()
    _init(g, _params(n, 0.5))                                   # ocean_wake_init turns the coupling off
    assert g.info().device_bytes == base
    assert counts() == off
    g.free()


def test_invalid_arguments_launch_nothing_and_change_nothing():
    from godotoceanwaves_b200.native import load_library
    lib = load_library()
    gow, g, params = _gen(256, 2)
    assert lib.ocean_wake_set_coupling(g.context, 1) == STATE                  # no layer
    buf = np.zeros(4, np.int64)
    assert lib.ocean_wake_get_coupling(g.context, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data) == STATE
    _init(g, _params(256, 0.5))
    assert lib.ocean_wake_get_coupling(g.context, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data) == STATE  # off
    before, mem = g.info().kernel_launches, g.info().device_bytes
    for bad in (2, -1, 7):
        assert lib.ocean_wake_set_coupling(g.context, bad) == INVALID
    assert g.info().device_bytes == mem and g.info().kernel_launches == before
    g.wake_set_coupling(True)
    src = np.zeros(1, wk.SOURCE)
    src["x"], src["z"], src["radius"], src["head"], src["body"] = 30.0, 30.0, 3.0, 0.3, -1
    g.wake_step(0.1, 2, (1, 2), src)
    snap = g.wake_coupling()
    mem, before = g.info().device_bytes, g.info().kernel_launches
    for bad in (2, -1):
        assert lib.ocean_wake_set_coupling(g.context, bad) == INVALID
    n = 256
    e = np.zeros((n, n), np.float32)
    P = ctypes.c_void_p
    o, t = np.zeros(4, np.int64), np.zeros(1, np.float32)
    for args in ((None, e.ctypes.data, o.ctypes.data, t.ctypes.data), (e.ctypes.data, None, o.ctypes.data, t.ctypes.data),
                 (e.ctypes.data, e.ctypes.data, None, t.ctypes.data), (e.ctypes.data, e.ctypes.data, o.ctypes.data, None)):
        assert lib.ocean_wake_get_coupling(g.context, *[None if a is None else P(a) for a in args]) == INVALID
    scales = gow.WaveGenerator.map_scales(params)
    assert lib.ocean_query_surface(g.context, 3, None, 2, scales.ctypes.data, 1e-3, 8, None) == INVALID
    assert lib.ocean_wake_step(g.context, -1.0, 1, 0, 0, 0, None, 0, None) == INVALID
    assert g.info().kernel_launches == before and g.info().device_bytes == mem
    now = g.wake_coupling()
    assert all(_same(x, y) for x, y in zip(now[:2], snap[:2])) and now[2:] == snap[2:]
    g.free()


def test_isolation_from_the_cascades():
    """Maps, foam, spectrum, velocity maps and the next update are byte-identical with the coupling on or off."""
    rng = np.random.default_rng(8)
    gow, a, pa = _gen(256, 3)
    gow, b, pb = _gen(256, 3)
    scales = gow.WaveGenerator.map_scales(pa)
    scene = _bodies(77, rng.integers(1, 20, 6))
    scene[1]["position"][:, [0, 2]] = rng.uniform(10, 110, (len(scene[1]), 2))
    src = np.zeros(len(scene[0]), wk.SOURCE)
    src["radius"], src["head"], src["body"] = 2.0, 0.3, np.arange(len(scene[0]))
    pts = _points(rng, (0, 0), 256, 0.5)
    for g, on in ((a, False), (b, True)):
        _init(g, _params(256, 0.5))
        g.wake_set_coupling(on)
        for _ in range(2):
            g.wake_step(0.1, 3, (0, 0), src, scene[1])
            _ops(g, scales, scene, pts)
    for g, p in ((a, pa), (b, pb)):
        g.update_all(1.0 / 50.0, p)
    da, na = a.maps_to_host()
    db, nb = b.maps_to_host()
    assert da.tobytes() == db.tobytes() and na.tobytes() == nb.tobytes()
    for c in range(3):
        assert a.get_foam_state(c).tobytes() == b.get_foam_state(c).tobytes()
        assert a.spectrum_to_host(c).tobytes() == b.spectrum_to_host(c).tobytes()
    assert a.velocity_to_host(0, 3).tobytes() == b.velocity_to_host(0, 3).tobytes()
    a.free()
    b.free()


def _box(side, cells, height):
    """cells x cells vertical columns of a side x side box, each reaching height / 2 above and below the body origin."""
    c = (np.arange(cells) + 0.5) * (side / cells) - side / 2
    X, Z = np.meshgrid(c, c, indexing="ij")
    p = np.zeros(X.size, bu.POINT)
    p["position"][:, 0], p["position"][:, 2] = X.ravel(), Z.ravel()
    p["volume"] = (side / cells) ** 2 * height
    p["half_height"] = height / 2
    return p


def _floating_box(side, draft, height, at):
    hull = _box(side, 4, height)
    fb = np.zeros(1, ob.BODY)
    fb["mass"] = RHO * side * side * draft
    fb["inertia"] = fb["mass"] * np.array([side * side + height * height, 2 * side * side, side * side + height * height]) / 12.0
    fb["num_points"] = len(hull)
    st = np.zeros(1, ob.STATE)
    st["position"] = (at[0], height / 2 - draft, at[1])            # equilibrium on flat water
    st["orientation"] = (0.0, 0.0, 0.0, 1.0)
    return fb, st, hull, np.full(len(hull), 0.5 * (side / 4) ** 2, np.float32)


def test_self_wake_keeps_a_body_at_its_own_height():
    """Flat sea.  A 2 m x 2 m box of 0.5 m draft carries its own source (radius 2 m, head 0.5 m) on a 256-cell window of
    0.5 m with damping 0 and a 48-cell sponge ramping to 1 / s.  Released 0.1 m above its equilibrium, it runs 30 s of
    body-then-wake ticks at 1 / 60 s, coupled and uncoupled.  The coupled body reads e = h + phi, which is 0 at rest under its
    own source, so its mean height over the last 10 s stays within 1 cm of the uncoupled run's; a body that read h would
    sink by a large fraction of the head (test_oracle_wake_coupling shows that on the specification)."""
    gow, g, params = _flat(256, 2)
    scales = gow.WaveGenerator.map_scales(params)
    fb, st0, hull, cda = _floating_box(2.0, 0.5, 1.0, (64.0, 64.0))
    st0["position"][0, 1] += 0.1
    src = np.zeros(1, wk.SOURCE)
    src["radius"], src["head"], src["body"] = 2.0, 0.5, 0
    ticks = int(round(30.0 / DT))
    mean = {}
    for coupled in (False, True):
        _init(g, _params(256, 0.5, damping=0.0, sponge_cells=48, sponge_damping=1.0))
        g.wake_set_coupling(coupled)
        s = st0.copy()
        ys = []
        for _ in range(ticks):
            s = g.simulate_bodies(fb, s, hull, cda, scales, DT, 1, RHO)
            g.wake_step(DT, 1, (0, 0), src, s)
            ys.append(float(s["position"][0, 1]))
        ys = np.array(ys)
        assert np.all(np.isfinite(ys))
        mean[coupled] = ys[-int(round(10.0 / DT)):].mean()
        print(f"self-wake: coupled={coupled}: mean height over the last 10 s {mean[coupled]:+.5f} m, "
              f"range over the last 10 s {np.ptp(ys[-600:]):.5f} m")
    gap = mean[True] - mean[False]
    print(f"self-wake: coupled minus uncoupled mean height {100 * gap:+.3f} cm")
    assert abs(gap) <= 0.01
    g.free()


def test_passing_wake_lifts_a_floating_box():
    """Flat sea.  A free source at 2.5 m/s (radius 4 m, head 0.3 m; the Kelvin case of the wake layer, dx = 0.5 m) passes
    15 m abeam of a floating 1 m x 1 m box of 0.1 m draft, whose heave period (0.63 s) is shorter than the Kelvin wave's
    (1.6 s).  Uncoupled the box does not move (< 1 mm); coupled its height follows e at its centre over the passage:
    correlation >= 0.8 and a ratio of standard deviations in [0.5, 2]."""
    gow, g, params = _flat(256, 2)
    scales = gow.WaveGenerator.map_scales(params)
    n, dx, U = 512, 0.5, 2.5
    box = (128.0, 128.0)
    fb, st0, hull, cda = _floating_box(1.0, 0.1, 0.4, box)
    src = np.zeros(1, wk.SOURCE)
    src["x"], src["z"], src["vx"], src["radius"], src["head"], src["body"] = 40.0, box[1] - 15.0, U, 4.0, 0.3, -1
    T_run = (230.0 - 40.0) / U
    ticks = int(round(T_run / DT))
    abeam = int(round((box[0] - 40.0) / U / DT))
    centre = np.array([box], np.float32)
    runs = {}
    for coupled in (False, True):
        _init(g, _params(n, dx, damping=0.0, sponge_cells=48, sponge_damping=1.0))
        g.wake_set_coupling(coupled)
        s = st0.copy()
        ys, es = [], []
        for k in range(ticks):
            s = g.simulate_bodies(fb, s, hull, cda, scales, DT, 1, RHO)
            src["x"] = np.float32(40.0 + U * k * DT)
            g.wake_step(DT, 1, (0, 0), src)
            ys.append(float(s["position"][0, 1]))
            es.append(float(g.query_surface(centre, scales)["displacement"][0, 1]))
        runs[coupled] = (np.array(ys), np.array(es))
    y0 = float(st0["position"][0, 1])
    still = np.abs(runs[False][0] - y0).max()
    y, e = runs[True][0][abeam:], runs[True][1][abeam:]
    corr = float(np.corrcoef(y - y.mean(), e - e.mean())[0, 1])
    ratio = float(y.std() / e.std())
    print(f"passing wake: uncoupled motion {1000 * still:.4f} mm; coupled: correlation {corr:.4f}, std ratio {ratio:.4f}, "
          f"std of e {100 * e.std():.3f} cm, max |e| {100 * np.abs(e).max():.3f} cm")
    assert still < 1e-3
    assert np.abs(e).max() > 0.005
    assert corr >= 0.8 and 0.5 <= ratio <= 2.0
    g.free()
