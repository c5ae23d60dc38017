"""GPU tests of the wake layer's foam (include/ocean.h, "Wake layer", ocean_wake_set_foam): F, h, h_prev and the render map
byte-identical to the specification oracle/wake_foam.py after every call, with scrolls, invalid sources, a crowded scene
and body-attached sources on device states; off means off; launch counts, device memory and arguments; and the physics on
the device: the stirred trail's cross-track profile and breaking foam inside the Kelvin wedge."""

import numpy as np
import pytest

from oracle import bodies as ob
from oracle import wake as wk
from oracle import wake_foam as wf
from test_gpu_bodies import _bodies
from test_gpu_sampling import _gen
from test_oracle_wake_foam import _trail, trail_profile_check

pytestmark = pytest.mark.gpu

INVALID, STATE = 1, 4
RHO = 1025.0
DT = 1.0 / 60.0
BREAKING = dict(whitecap=0.02, grow_rate=4.0, stir_rate=0.0, decay_rate=0.3)
STIRRING = dict(whitecap=0.0, grow_rate=0.0, stir_rate=0.02, decay_rate=0.2)
BOTH = dict(whitecap=0.03, grow_rate=3.0, stir_rate=0.01, decay_rate=0.5)

def _params(n, dx, damping=0.0, sponge_cells=16, sponge_damping=1.0):
    p = np.zeros((), wk.PARAMS)
    p["size"], p["cell_size"], p["damping"], p["sponge_cells"], p["sponge_damping"] = n, dx, damping, sponge_cells, sponge_damping
    return p

def _init(g, p):
    g.wake_init(int(p["size"]), float(p["cell_size"]), float(p["damping"]), int(p["sponge_cells"]), float(p["sponge_damping"]))

def _set_foam(g, L, kw):
    g.wake_set_foam(**kw)
    L.foam_params = wf.foam_params(**kw)

def _same(a, b):
    """Byte-identical, except that a NaN only has to meet a NaN."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.tobytes() == b.tobytes():
        return True
    na, nb = np.isnan(a.astype(np.float32)), np.isnan(b.astype(np.float32))
    return bool(np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes())

def _sources(rng, k, extent, n_states=0):
    s = np.zeros(k, wk.SOURCE)
    s["x"], s["z"] = rng.uniform(-0.1 * extent, 1.1 * extent, k), rng.uniform(-0.1 * extent, 1.1 * extent, k)
    s["vx"], s["vz"] = rng.uniform(-4, 4, k), rng.uniform(-4, 4, k)
    s["radius"] = rng.uniform(0.5, 0.06 * extent, k)
    s["head"] = rng.uniform(-0.3, 0.3, k)
    s["body"] = -1
    if n_states:
        att = rng.random(k) < 0.4
        s["body"][att] = rng.integers(0, n_states, att.sum())
        s["x"][att], s["z"][att] = rng.uniform(-2, 2, att.sum()), rng.uniform(-2, 2, att.sum())
    return s

def _check(g, L):
    h, hp, origin = g.wake_state()
    assert origin == L.origin
    assert _same(h, L.h) and _same(hp, L.h_prev)
    assert _same(g.wake_foam(), L.foam)
    m, _ = g.wake_map()
    assert _same(m, L.render_map())

@pytest.mark.parametrize("n", [256, 512, 1024])
@pytest.mark.parametrize("dx", [0.25, 1.0])
def test_parity_with_the_specification(n, dx):
    """Breaking and stirring alone and together, S = 1 and 4, scrolls by (3, -2), by a negative offset and by N or more
    cells, and non-finite and degenerate sources beside ordinary ones; every call checked."""
    gow, g, _ = _gen(128, 2)
    rng = np.random.default_rng(n + int(dx * 8))
    p = _params(n, dx, damping=0.05, sponge_cells=24, sponge_damping=3.0)
    _init(g, p)
    L = wf.Layer(p)
    st = np.zeros(6, wk.STATE)
    st["position"] = rng.uniform(0, n * dx, (6, 3))
    st["linear_velocity"] = rng.uniform(-3, 3, (6, 3))
    h_max = np.sqrt(dx / wk.G)
    k = 24 if n < 1024 else 8
    plan = [(1, (0, 0), BREAKING), (4, (3, -2), BREAKING), (1, (3, -2), STIRRING), (4, (-7, 5), STIRRING),
            (1, (-7, 5), BOTH), (4, (-7 + n, 5), BOTH), (4, (40, 41), BOTH)]
    if n == 1024:                                           # the specification is slow on 1024^2 windows
        plan = [plan[0], plan[3], plan[4], plan[5]]
    for call, (S, origin, kw) in enumerate(plan):
        _set_foam(g, L, kw)
        s = _sources(rng, k, n * dx, len(st))
        if call == 2:                                       # non-finite and degenerate sources beside ordinary ones
            s["head"][0], s["x"][1], s["radius"][2], s["radius"][3], s["vz"][4] = np.nan, np.inf, 0.0, -2.0, np.inf
            s["vx"][5] = 3e20                               # a finite centre at tau = 0 whose |v|^2 overflows
        dt = 0.9 * h_max * S
        g.wake_step(dt, S, origin, s, st)
        L.step(dt, S, origin, s, st)
        _check(g, L)
        if call <= 1:
            assert L.foam.max() > 0
    g.free()

def test_many_overlapping_sources_keep_index_order():
    """The crowded 700-source scene of test_gpu_wake (three 256-source cull chunks, repeats and invalid sources in later
    warps and chunks) through ocean_wake_step_device, with breaking and stirring."""
    import torch
    from godotoceanwaves_b200.native import check, load_library
    lib = load_library()
    gow, g, _ = _gen(128, 2)
    n, dx = 256, 0.5
    p = _params(n, dx, damping=0.05, sponge_cells=24, sponge_damping=1.0)
    _init(g, p)
    L = wf.Layer(p)
    _set_foam(g, L, dict(whitecap=0.01, grow_rate=2.0, stir_rate=0.01, decay_rate=0.1))
    rng = np.random.default_rng(700)
    k = 700
    st = np.zeros(4, wk.STATE)
    st["position"] = rng.uniform(25, 45, (4, 3))
    st["linear_velocity"] = rng.uniform(-2, 2, (4, 3))
    dev = torch.device("cuda", g.device)
    st_d = torch.from_numpy(st.view(np.uint8).copy()).to(dev)
    for call, (S, origin) in enumerate([(2, (0, 0)), (1, (5, -3)), (3, (5, -3))]):
        s = np.zeros(k, wk.SOURCE)
        s["x"], s["z"] = rng.uniform(20, 60, k), rng.uniform(20, 60, k)
        s["vx"], s["vz"] = rng.uniform(-3, 3, k), rng.uniform(-3, 3, k)
        s["radius"] = rng.uniform(1.0, 6.0, k)
        s["head"] = rng.uniform(-0.05, 0.05, k)
        s["body"] = -1
        att = rng.random(k) < 0.2
        s["body"][att] = rng.integers(0, len(st), att.sum())
        s["x"][att], s["z"][att] = rng.uniform(-3, 3, att.sum()), rng.uniform(-3, 3, att.sum())
        s[300:312] = s[299]
        s[510:520] = s[3]
        s["head"][40], s["x"][97], s["radius"][130], s["radius"][260] = np.nan, np.inf, 0.0, -1.0
        s["vz"][390], s["radius"][520] = np.inf, np.inf
        s["body"][[200, 450, 650]] = len(st)
        src_d = torch.from_numpy(s.view(np.uint8).copy()).to(dev)
        dt = 0.05 * S
        torch.cuda.synchronize()
        check(lib.ocean_wake_step_device(g.context, dt, S, origin[0], origin[1], k, src_d.data_ptr(), len(st), st_d.data_ptr()))
        g.synchronize()
        L.step(dt, S, origin, s, st)
        _check(g, L)
        assert L.foam.max() > 0
    g.free()

def test_body_sources_on_device_states():
    """Body-then-wake ticks: ocean_simulate_bodies_device writes the states, ocean_wake_step_device reads them, with foam."""
    import torch
    from godotoceanwaves_b200.native import check, load_library
    lib = load_library()
    gow, g, params = _gen(256, 2)
    scales = np.ascontiguousarray(gow.WaveGenerator.map_scales(params), np.float32)
    n, dx = 256, 0.5
    p = _params(n, dx, damping=0.02, sponge_cells=24)
    _init(g, p)
    L = wf.Layer(p)
    _set_foam(g, L, BOTH)
    rng = np.random.default_rng(17)
    fb, s0, hull, cda = _bodies(613, rng.integers(1, 16, 8))
    s0["position"][:, 0] = rng.uniform(30, 100, len(s0))
    s0["position"][:, 2] = rng.uniform(30, 100, len(s0))
    s0["linear_velocity"][:, [0, 2]] = rng.uniform(-3, 3, (len(s0), 2))
    src = np.zeros(len(fb), wk.SOURCE)
    src["radius"], src["head"], src["body"] = 3.0, 0.3, np.arange(len(fb))
    dev = torch.device("cuda", g.device)
    st_d = torch.from_numpy(s0.view(np.uint8).copy()).to(dev)
    hull_d = torch.from_numpy(hull.view(np.uint8).copy()).to(dev)
    cda_d = torch.from_numpy(cda).to(dev)
    src_d = torch.from_numpy(src.view(np.uint8).copy()).to(dev)
    B = len(fb)
    for call, (S, origin) in enumerate([(1, (0, 0)), (4, (2, 1)), (2, (2, 1))]):
        torch.cuda.synchronize()
        check(lib.ocean_simulate_bodies_device(g.context, B, fb.ctypes.data, st_d.data_ptr(), len(hull), hull_d.data_ptr(),
                                               cda_d.data_ptr(), 2, scales.ctypes.data, RHO, DT, 2, 1e-3, 8, None, None, None))
        check(lib.ocean_wake_step_device(g.context, DT * S, S, origin[0], origin[1], len(src), src_d.data_ptr(), B, st_d.data_ptr()))
        g.synchronize()
        states = np.frombuffer(st_d.cpu().numpy().tobytes(), ob.STATE).copy()
        assert np.abs(states["linear_velocity"][:, [0, 2]]).max() > 0.1
        L.step(DT * S, S, origin, src, states)
        _check(g, L)
    assert L.foam.max() > 0
    g.free()

def _run(g, coupled, foam, scene, src, scales, pts):
    """Body-then-wake ticks; returns everything foam must not change."""
    fb, s0, hull, cda = scene
    _init(g, _params(256, 0.5))
    g.wake_set_coupling(coupled)
    out = []
    s = s0.copy()
    for tick in range(4):
        if foam == "on" or (foam == "on-off" and tick == 1):
            g.wake_set_foam(**BOTH)
        if foam == "on-off" and tick == 3:
            g.wake_set_foam(None)
        s = g.simulate_bodies(fb, s, hull, cda, scales, DT, 2, RHO)
        g.wake_step(0.1, 3, (tick, -tick), src, s)
        h, hp, origin = g.wake_state()
        m, rect = g.wake_map()
        item = [s, h, hp, np.array(origin), m[..., :3], rect, g.sample_wake(pts), g.query_surface(pts, scales)]
        if coupled:
            e, e_old, origins, T = g.wake_coupling()
            item += [e, e_old, np.array(origins), np.array(T)]
        out.append([np.ascontiguousarray(x).tobytes() for x in item])
        out[-1].append(m[..., 3].tobytes())
    return out

def test_off_means_off():
    """A generator that never enabled foam, one that enabled it and then disabled it, and one with foam on give the same
    states, h, h_prev, render map heights and slopes, samples, surface records and, coupled, snapshots; the render map's
    fourth channel is 0 while foam is off."""
    gow, g, params = _gen(256, 2)
    scales = gow.WaveGenerator.map_scales(params)
    rng = np.random.default_rng(31)
    scene = _bodies(311, rng.integers(1, 20, 6))
    scene[1]["position"][:, [0, 2]] = rng.uniform(20, 100, (len(scene[1]), 2))
    scene[1]["linear_velocity"][:, [0, 2]] = rng.uniform(-2, 2, (len(scene[1]), 2))
    src = np.zeros(len(scene[0]) + 1, wk.SOURCE)
    src["radius"], src["head"], src["body"] = 2.5, 0.3, -1
    src["body"][:len(scene[0])] = np.arange(len(scene[0]))
    src["x"][-1], src["z"][-1], src["vx"][-1] = 60.0, 60.0, 3.0
    pts = rng.uniform(0, 128, (300, 2)).astype(np.float32)
    for coupled in (False, True):
        never = _run(g, coupled, "never", scene, src, scales, pts)
        on_off = _run(g, coupled, "on-off", scene, src, scales, pts)
        on = _run(g, coupled, "on", scene, src, scales, pts)
        for tick in range(4):
            assert on[tick][:-1] == never[tick][:-1] and on_off[tick][:-1] == never[tick][:-1], (coupled, tick)
            assert not np.frombuffer(never[tick][-1], np.float16).any()
        assert on_off[0][-1] == on_off[3][-1] == never[0][-1]     # the fourth channel is 0 before enabling and after disabling
        assert np.frombuffer(on[-1][-1], np.float16).any()
    g.free()

def test_launch_counts_and_device_memory():
    gow, g, _ = _gen(128, 2)
    base = g.info().device_bytes
    n = 256
    _init(g, _params(n, 0.5))
    src = np.zeros(2, wk.SOURCE)
    src["x"], src["z"], src["vx"], src["radius"], src["head"], src["body"] = 40.0, 60.0, 2.0, 3.0, 0.3, -1

    def counts(S=3):
        out = []
        for op in (lambda: g.wake_step(0.05 * S, S, (1, 0), src), lambda: g.wake_map()):
            before = g.info().kernel_launches
            op()
            out.append(g.info().kernel_launches - before)
        return out

    assert counts() == [3, 1]
    layer = g.info().device_bytes                       # the layer and the host entry point's source staging
    g.wake_set_foam(**BOTH)
    assert g.info().device_bytes == layer + 2 * 4 * n * n
    assert counts() == [3, 1]
    g.wake_set_foam(**STIRRING)                         # changing the parameters keeps F and allocates nothing
    assert g.info().device_bytes == layer + 2 * 4 * n * n
    g.wake_set_coupling(True)
    assert counts() == [4, 1] and counts(5) == [6, 1]
    g.wake_set_coupling(False)
    g.wake_set_foam(None)
    assert g.info().device_bytes == layer
    g.wake_set_foam(**BOTH)
    assert not g.wake_foam().any()                      # enabling zeroes F
    counts()
    _init(g, _params(n, 0.5))                           # ocean_wake_init turns foam off
    assert g.info().device_bytes == layer
    from godotoceanwaves_b200.native import load_library
    buf = np.zeros((n, n), np.float32)
    assert load_library().ocean_wake_get_foam_state(g.context, buf.ctypes.data) == STATE
    g.wake_set_foam(**BOTH)
    _init(g, _params(0, 0.5))
    assert g.info().device_bytes == base
    g.free()

def test_invalid_arguments_launch_nothing_and_change_nothing():
    from godotoceanwaves_b200.native import load_library
    lib = load_library()
    gow, g, _ = _gen(128, 2)
    n = 256
    buf = np.zeros((n, n), np.float32)
    fp = np.array((0.1, 1.0, 1.0, 1.0), wf.FOAM_PARAMS)
    assert lib.ocean_wake_set_foam(g.context, fp.ctypes.data) == STATE                   # no layer
    assert lib.ocean_wake_get_foam_state(g.context, buf.ctypes.data) == STATE
    _init(g, _params(n, 0.5))
    assert lib.ocean_wake_get_foam_state(g.context, buf.ctypes.data) == STATE            # foam off
    assert lib.ocean_wake_set_foam_state(g.context, buf.ctypes.data) == STATE
    g.wake_set_foam(**BOTH)
    src = np.zeros(1, wk.SOURCE)
    src["x"], src["z"], src["vx"], src["radius"], src["head"], src["body"] = 30.0, 30.0, 3.0, 3.0, 0.3, -1
    g.wake_step(0.1, 2, (1, 2), src)
    F0 = g.wake_foam()
    assert F0.any()
    mem, before = g.info().device_bytes, g.info().kernel_launches
    bad = [(np.nan, 1, 1, 1), (np.inf, 1, 1, 1), (0.1, -1, 1, 1), (0.1, 1, -1e-30, 1), (0.1, 1, 1, -2), (0.1, np.inf, 1, 1),
           (0.1, 1, np.nan, 1), (0.1, 1, 1, np.inf)]
    for b in bad:
        assert lib.ocean_wake_set_foam(g.context, np.array(b, wf.FOAM_PARAMS).ctypes.data) == INVALID, b
    assert lib.ocean_wake_get_foam_state(g.context, None) == INVALID
    assert lib.ocean_wake_set_foam_state(g.context, None) == INVALID
    assert g.info().device_bytes == mem and g.info().kernel_launches == before
    assert g.wake_foam().tobytes() == F0.tobytes()
    # the parameters did not change either: the next call matches the specification with BOTH
    h, hp, origin = g.wake_state()
    L = wf.Layer(_params(n, 0.5), wf.foam_params(**BOTH))
    L.h, L.h_prev, L.origin, L.foam = h, hp, origin, F0
    g.wake_step(0.1, 2, (1, 2), src)
    L.step(0.1, 2, (1, 2), src)
    assert _same(g.wake_foam(), L.foam)
    # set and get round trip, and set_state leaves F untouched
    F1 = np.random.default_rng(2).uniform(0, 1, (n, n)).astype(np.float32)
    g.set_wake_foam(F1)
    g.set_wake_state(*g.wake_state()[:2])
    assert g.wake_foam().tobytes() == F1.tobytes()
    g.free()

def test_stirred_trail_on_the_device():
    """The cross-track profile of a straight stirred trail, as test_oracle_wake_foam checks it on the specification."""
    gow, g, _ = _gen(128, 2)
    n, dx, U, r, h_sub, stir = 256, 0.5, 3.0, 3.0, 0.03, 0.04
    _init(g, _params(n, dx, sponge_cells=24))
    g.wake_set_foam(whitecap=0.0, grow_rate=0.0, stir_rate=stir, decay_rate=0.0)
    _trail(lambda dt, S, src: g.wake_step(dt, S, (0, 0), src), n, dx, U, r, 64.1, 10.0, 118.0, h_sub, stir)
    F = g.wake_foam()
    worst = trail_profile_check(F, n, dx, U, r, 64.1, 10.0, 118.0, h_sub, stir)
    print(f"stirred trail: peak {F.max():.5f} (closed form {stir * 16 / 15 * r * U:.5f}), largest error {worst:.3f} of its bound")
    assert worst <= 1.0
    g.free()

def test_breaking_foam_lies_in_the_kelvin_wedge():
    """The Kelvin scene of test_gpu_wake (U = 2.5 m/s, r = 4 m, head 0.2 m, dx = 0.5 m, damping 0, a 48-cell sponge) on a
    fixed 1024-cell window, 60 s of 1 / 30 s sub-steps, breaking only (decay 0, so F marks every cell that ever broke).
    Run 1 recovers every sub-step's beta from the states, c = (a1 h - a2 h_prev - h_new) / a3, and its maximum over the
    run.  Run 2, at whitecap = 0.4 of that maximum: every foamy cell lies inside the wedge of half-angle 22.5 degrees
    behind the source (apex 2 r ahead of its final centre), under the source's path (within r + 1 m of the track), or
    within 30 m of its start.  Run 3, at whitecap just above the maximum: no foam at all."""
    gow, g, _ = _gen(128, 2)
    n, dx, U, r, hs, T = 1024, 0.5, 2.5, 4.0, 1.0 / 30.0, 60.0
    p = _params(n, dx, damping=0.0, sponge_cells=48, sponge_damping=3.0)
    steps = int(round(T / hs))
    x_start, z_src = 60.0, 256.0
    src = np.zeros(1, wk.SOURCE)
    src["x"], src["z"], src["vx"], src["radius"], src["head"], src["body"] = x_start, z_src, U, r, 0.2, -1
    a1, a2, a3 = wk.coefficients(p, wk.substep(hs, 1))
    rg = wk.ring(n, 48)
    a1, a2, a3 = a1[rg].astype(np.float64), a2[rg].astype(np.float64), a3[rg].astype(np.float64)

    def run(whitecap, track=False):
        _init(g, p)
        g.wake_set_foam(whitecap=whitecap, grow_rate=1.0, stir_rate=0.0, decay_rate=0.0)
        beta_max = 0.0
        h, hp, _ = g.wake_state()
        for k in range(steps):
            src["x"] = np.float32(x_start + U * k * hs)
            g.wake_step(hs, 1, (0, 0), src)
            if track:
                hn, _, _ = g.wake_state()
                c = (a1 * h - a2 * hp - hn) / a3
                beta_max = max(beta_max, float((c / dx).max()))
                hp, h = h, hn
        return g.wake_foam(), beta_max

    F, beta_max = run(3e38, track=True)
    assert not F.any()
    print(f"Kelvin scene: largest beta {beta_max:.5f}")
    assert beta_max > 0
    F, _ = run(0.4 * beta_max)
    j, i = np.nonzero(F)
    assert len(i) > 0
    x, z = (i + 0.5) * dx, (j + 0.5) * dx
    x_end = x_start + U * T
    inside = (x <= x_end + 2 * r) & (np.abs(z - z_src) <= np.tan(np.radians(22.5)) * (x_end + 2 * r - x))
    inside |= (x >= x_start - r - 1.0) & (x <= x_end + r + 1.0) & (np.abs(z - z_src) <= r + 1.0)
    near_start = np.hypot(x - x_start, z - z_src) <= 30.0
    out = ~(inside | near_start)
    far = np.hypot(x - x_start, z - z_src)[~inside]
    print(f"Kelvin scene at whitecap {0.4 * beta_max:.5f}: {len(i)} foamy cells, {np.count_nonzero(~inside)} outside the wedge "
          f"(farthest {far.max() if len(far) else 0.0:.1f} m from the start), {np.count_nonzero(out)} outside both; "
          f"largest lateral angle {np.degrees(np.arctan2(np.abs(z - z_src), x_end + 2 * r - x)[~near_start].max()):.2f} deg")
    assert not out.any()
    F, _ = run(beta_max * (1 + 1e-3) + 1e-6)
    assert not F.any()
    g.free()
