"""GPU tests of the wake layer's obstacles (include/ocean.h, "Wake layer", ocean_wake_set_obstacles): h, h_prev, the render
map, samples, F, the coupling's snapshots and the coupled records byte-identical to the specification oracle/wake_obstacles.py
after every call; off means off; the physics on the device (window-edge equivalence, the 6-cell barrier, stability in a
basin, reflection from a straight wall); launch counts, device memory, invalid arguments and isolation from the cascades."""

import numpy as np
import pytest

from oracle import bodies as ob
from oracle import buoyancy as bu
from oracle import wake as wk
from oracle import wake_coupling as wc
from oracle import wake_foam as wf
from oracle import wake_obstacles as wo
from test_gpu_bodies import _bodies
from test_gpu_sampling import _gen
from test_oracle_wake_obstacles import (FOAM, REFLECTION, REFLECTION_BOUND, barrier_masks, barrier_run, checkerboard, coastline,
                                        islands, reflection_fields, reflection_runs, single_cells, thin_walls,
                                        window_edge_scene)

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


def _check(g, L, rng, coupling=None):
    h, hp, origin = g.wake_state()
    assert origin == L.origin
    assert _same(h, L.h) and _same(hp, L.h_prev)
    m, _ = g.wake_map()
    assert _same(m, L.render_map())
    if L.foam_on:
        assert _same(g.wake_foam(), L.foam)
    x0, z0 = wk.world_origin(L.origin, L.cell_size)
    ext = float(L.n * L.cell_size)
    pts = np.stack([rng.uniform(x0 - 0.05 * ext, x0 + 1.05 * ext, 500), rng.uniform(z0 - 0.05 * ext, z0 + 1.05 * ext, 500)], 1)
    pts = pts.astype(np.float32)
    assert _same(g.sample_wake(pts), L.sample(pts))
    if coupling is not None:
        e, e_old, origins, T = g.wake_coupling()
        assert _same(e, coupling.e) and _same(e_old, coupling.e_old) and T == coupling.T
        assert origins == (coupling.origin_e, coupling.origin_old)


MASKS = {"coastline": coastline, "islands": islands, "single cells": single_cells, "checkerboard": checkerboard,
         "thin walls": thin_walls}


@pytest.mark.parametrize("n", [256, 512, 1024])
@pytest.mark.parametrize("dx", [0.25, 1.0])
def test_parity_with_the_specification(n, dx):
    """Every mask kind, plain, foam and coupled calls, S = 1 and 4, scrolls by (3, -2), by a negative offset and by N or more
    cells across the mask's edge, and the mask replaced between calls; every call checked."""
    gow, g, _ = _gen(128, 2)
    rng = np.random.default_rng(n + int(dx * 8))
    p = _params(n, dx, damping=0.05, sponge_cells=24, sponge_damping=3.0)
    _init(g, p)
    L = wo.Layer(p, wf.foam_params(**FOAM))
    L.foam_on = False
    st = np.zeros(6, wk.STATE)
    st["position"] = rng.uniform(0, n * dx, (6, 3))
    st["linear_velocity"] = rng.uniform(-3, 3, (6, 3))
    h_max = np.sqrt(dx / wk.G)
    k = 24 if n < 1024 else 8
    mo = (-n // 4, n // 8)                                          # the mask's origin: it covers part of every window
    plan = [(1, (0, 0), "coastline", "plain"), (4, (3, -2), "islands", "foam"), (1, (3, -2), "single cells", "coupled"),
            (4, (-7, 5), "checkerboard", "foam"), (1, (-7, 5), "thin walls", "plain"), (4, (-7 + n, 5), "coastline", "coupled"),
            (4, (40, 41), "islands", "plain")]
    if n == 1024:                                                   # the specification is slow on 1024^2 windows
        plan = [plan[0], plan[1], plan[2], plan[5]]
    cp = None
    for call, (S, origin, kind, mode) in enumerate(plan):
        mask = MASKS[kind](n + n // 2, n + n // 3, seed=call) if kind in ("coastline", "islands", "single cells") \
            else MASKS[kind](n + n // 2, n + n // 3)
        g.wake_set_obstacles(mask, mo)
        L.set_obstacles(mask, mo)
        if mode == "foam" and not L.foam_on:
            g.wake_set_foam(**FOAM)
            L.foam_on, L.foam = True, np.zeros_like(L.h)
        if mode == "coupled" and cp is None:
            g.wake_set_coupling(True)
            cp = wc.Coupling(n, dx)
        s = _sources(rng, k, n * dx, len(st))
        dt = 0.9 * h_max * S
        g.wake_step(dt, S, origin, s, st)
        wo.step(L, cp, dt, S, origin, s, st)
        _check(g, L, rng, cp)
        assert L.blocked().any() and not L.blocked().all()
    g.free()


def test_many_overlapping_sources_keep_index_order():
    """The crowded 700-source scene of test_gpu_wake through ocean_wake_step_device, over islands, with foam."""
    import torch
    from godotoceanwaves_b200.native import check, load_library
    lib = load_library()
    gow, g, _ = _gen(128, 2)
    n, dx = 256, 0.5
    p = _params(n, dx, damping=0.05, sponge_cells=24, sponge_damping=1.0)
    _init(g, p)
    L = wo.Layer(p, wf.foam_params(**FOAM))
    g.wake_set_foam(**FOAM)
    mask = islands(n, n, seed=7, count=30)
    g.wake_set_obstacles(mask, (0, 0))
    L.set_obstacles(mask, (0, 0))
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
        s["head"][40], s["x"][97], s["radius"][130], s["radius"][260] = np.nan, np.inf, 0.0, -1.0
        s["body"][[200, 450, 650]] = len(st)
        src_d = torch.from_numpy(s.view(np.uint8).copy()).to(dev)
        dt = 0.05 * S
        torch.cuda.synchronize()
        check(lib.ocean_wake_step_device(g.context, dt, S, origin[0], origin[1], k, src_d.data_ptr(), len(st), st_d.data_ptr()))
        g.synchronize()
        L.step(dt, S, origin, s, st)
        _check(g, L, rng)
    g.free()


def test_coupled_bodies_at_a_quay():
    """Bodies moored beside a quay and drifting into it, body-attached sources on the device states of
    ocean_simulate_bodies_device: after every call the states and records of simulate, the snapshots and the records of
    the surface query, buoyancy and body forces are byte-identical to the specification."""
    import torch
    from godotoceanwaves_b200.native import check, load_library
    lib = load_library()
    N, C, n, dx = 256, 2, 256, 0.5
    gow, g, params = _gen(N, C)
    scales = gow.WaveGenerator.map_scales(params)
    g.update_velocity()
    d16, n16 = g.maps_to_host(0, C)
    vel = g.velocity_to_host(0, C)
    p = _params(n, dx, damping=0.02, sponge_cells=24)
    _init(g, p)
    L = wo.Layer(p)
    cp = wc.Coupling(n, dx)
    g.wake_set_coupling(True)
    quay = np.zeros((n, n), np.uint8)
    quay[:, 150:] = 1                                               # the quay face at x = 75 m
    g.wake_set_obstacles(quay, (0, 0))
    L.set_obstacles(quay, (0, 0))
    rng = np.random.default_rng(77)
    fb, s0, hull, cda = _bodies(977, rng.integers(1, 16, 8))
    s0["position"][:, 0] = rng.uniform(68, 74, len(s0))            # beside the quay face
    s0["position"][:, 2] = rng.uniform(20, 100, len(s0))
    s0["linear_velocity"][:, [0, 2]] = 0.0
    s0["linear_velocity"][::2, 0] = 2.0                             # every other one drifts into it
    src = np.zeros(len(fb), wk.SOURCE)
    src["radius"], src["head"], src["body"] = 2.0, 0.25, np.arange(len(fb))
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
    for call, (S, Sw, origin) in enumerate([(1, 2, (0, 0)), (4, 1, (0, 0)), (1, 4, (3, -2))]):
        g.synchronize()
        before = np.frombuffer(st_d.cpu().numpy().tobytes(), ob.STATE).copy()
        torch.cuda.synchronize()
        check(lib.ocean_simulate_bodies_device(g.context, B, fb.ctypes.data, st_d.data_ptr(), len(hull), hull_d.data_ptr(), cda_d.data_ptr(),
                                               C, sc.ctypes.data, RHO, DT, S, 1e-3, 8, hyd_d.data_ptr(), drg_d.data_ptr(), T_d.data_ptr()))
        with np.errstate(all="ignore"):
            rs, rh, rd, rT = wc.simulate(d16, n16, vel, fb, before, hull, cda, scales, RHO, DT, S, 1e-3, 8, wake=cp)
        g.synchronize()
        after = np.frombuffer(st_d.cpu().numpy().tobytes(), ob.STATE).copy()
        assert _same(after, rs) and _same(hyd_d.cpu().numpy(), rh) and _same(drg_d.cpu().numpy(), rd), call
        assert _same(T_d.cpu().numpy(), rT), call
        check(lib.ocean_wake_step_device(g.context, DT * Sw, Sw, origin[0], origin[1], len(src), src_d.data_ptr(), B, st_d.data_ptr()))
        wo.step(L, cp, DT * Sw, Sw, origin, src, after)
        _check(g, L, rng, cp)
        assert np.abs(cp.e).max() > 0 and not cp.e[L.blocked()].any()
        pts = np.stack([rng.uniform(40, 100, 400), rng.uniform(0, 128, 400)], 1).astype(np.float32)
        with np.errstate(all="ignore"):
            ref = wc.query_surface(d16, n16, pts, scales, wake=cp)
        assert _same(g.query_surface(pts, scales), ref), call
        table, velo = ob.pose(fb, after)
        with np.errstate(all="ignore"):
            rb, rbs = wc.buoyancy(d16, n16, table, hull, scales, RHO, return_samples=True, wake=cp)
            rf = wc.body_forces(d16, n16, vel, table, velo, hull, cda, scales, RHO, return_samples=True, wake=cp)
        gb, gbs = g.buoyancy(table, hull, scales, RHO, return_samples=True)
        assert _same(gb, rb) and _same(gbs, rbs), call
        gf = g.body_forces(table, velo, hull, cda, scales, RHO, return_samples=True)
        assert all(_same(x, y) for x, y in zip(gf, rf)), call
    g.free()


def _run(g, coupled, foam, how, scene, src, scales, pts):
    """Body-then-wake ticks on a fresh layer whose mask is set as `how` says; returns every field and record as bytes."""
    fb, s0, hull, cda = scene
    _init(g, _params(256, 0.5))
    g.wake_set_coupling(coupled)
    if foam:
        g.wake_set_foam(**FOAM)
    if how == "set-and-cleared":
        g.wake_set_obstacles(coastline(300, 300), (0, 0))
        g.wake_set_obstacles(None)
    elif how == "misses the window":
        g.wake_set_obstacles(coastline(300, 300), (256 + 10 + 6, 0))   # beyond the farthest window plus its halo
    elif how == "all zero":
        g.wake_set_obstacles(np.zeros((400, 400), np.uint8), (-100, -100))
    out = []
    s = s0.copy()
    for tick in range(4):
        s = g.simulate_bodies(fb, s, hull, cda, scales, DT, 2, RHO)
        g.wake_step(0.1, 3, (tick, -tick), src, s)
        h, hp, origin = g.wake_state()
        m, rect = g.wake_map()
        item = [s, h, hp, np.array(origin), m, rect, g.sample_wake(pts), g.query_surface(pts, scales)]
        if coupled:
            e, e_old, origins, T = g.wake_coupling()
            item += [e, e_old, np.array(origins), np.array(T)]
        if foam:
            item.append(g.wake_foam())
        out.append([np.ascontiguousarray(x).tobytes() for x in item])
    return out


def test_off_means_off():
    """Never set, set and cleared, a mask that blocks nothing in the window and an all-zero mask: every field and record
    byte-identical, with foam and the coupling on and off."""
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
        for foam in (False, True):
            runs = [_run(g, coupled, foam, how, scene, src, scales, pts)
                    for how in ("never", "set-and-cleared", "misses the window", "all zero")]
            assert runs[1] == runs[0] and runs[2] == runs[0] and runs[3] == runs[0], (coupled, foam)
    g.free()


def test_window_edge_equivalence_and_the_barrier_on_the_device():
    """The specification's window-edge equivalence, on the device: the 256-cell window blocked but for [0, 128)^2 matches a
    128-cell window on the quadrant, with foam and the coupling, and is +0 elsewhere; and 2000 sub-steps of forcing leave
    the far side of 6-cell walls exactly +0 and reach past 5-cell ones."""
    gow, a, _ = _gen(128, 2)
    gow, b, _ = _gen(128, 2)
    _init(a, _params(256, 0.5, damping=0.02, sponge_cells=0))
    _init(b, _params(128, 0.5, damping=0.02, sponge_cells=0))
    mask = np.ones((256, 256), np.uint8)
    mask[:128, :128] = 0
    a.wake_set_obstacles(mask, (7, -3))
    for g in (a, b):
        g.wake_set_foam(**FOAM)
        g.wake_set_coupling(True)
    s = window_edge_scene()
    q = (slice(0, 128), slice(0, 128))
    rest = mask != 0
    for S in (1, 4, 2, 3):
        a.wake_step(0.1 * S, S, (7, -3), s)
        b.wake_step(0.1 * S, S, (7, -3), s)
        (ha, hpa, _), (hb, hpb, _) = a.wake_state(), b.wake_state()
        Fa, Fb = a.wake_foam(), b.wake_foam()
        ea, eoa, _, _ = a.wake_coupling()
        eb, eob, _, _ = b.wake_coupling()
        assert _same(ha[q], hb) and _same(hpa[q], hpb) and _same(Fa[q], Fb) and _same(ea[q], eb) and _same(eoa[q], eob)
        for f in (ha, Fa, ea):
            assert not f[rest].any() and not np.signbit(f[rest]).any()
    assert np.abs(hb).max() > 0
    a.free()
    b.free()
    gow, g, _ = _gen(128, 2)
    for name, m, far in barrier_masks(128):
        _init(g, _params(128, 0.5, sponge_cells=0))
        g.wake_set_obstacles(m, (0, 0))
        barrier_run(lambda dt, S, src: g.wake_step(dt, S, (0, 0), src), 128)
        h, hp, _ = g.wake_state()
        if name.endswith("6"):
            assert not h[far].any() and not np.signbit(h[far]).any() and not hp[far].any(), name
        else:
            assert np.abs(h[far]).max() > 0, name
    g.free()


def test_stability_in_a_basin_at_the_largest_sub_step():
    """10^4 sub-steps of a random field at the largest accepted sub-step, no damping and no sponge, in a basin closed by a
    border wall with random islands, 1-cell walls and single blocked cells inside: bounded."""
    gow, g, _ = _gen(128, 2)
    n, dx = 256, 0.5
    _init(g, _params(n, dx, damping=0.0, sponge_cells=0, sponge_damping=0.0))
    h = np.float32(np.sqrt(dx / wk.G))
    while not wk.stable(dx, h):
        h = np.nextafter(h, np.float32(0))
    mask = islands(n, n, seed=3, count=10) | thin_walls(n, n) | single_cells(n, n, seed=4, count=200)
    mask[:8], mask[-8:], mask[:, :8], mask[:, -8:] = 1, 1, 1, 1
    g.wake_set_obstacles(mask, (0, 0))
    rng = np.random.default_rng(11)
    h0 = rng.uniform(-1, 1, (n, n)).astype(np.float32)
    g.set_wake_state(h0, h0)
    for _ in range(40):
        g.wake_step(float(h) * 250, 250, (0, 0))
    hh, hp, _ = g.wake_state()
    print(f"basin: largest |h| after 10^4 sub-steps {np.abs(hh).max():.3f}")
    assert np.all(np.isfinite(hh)) and np.abs(hh).max() < 50.0, np.abs(hh).max()
    assert not hh[mask != 0].any()
    g.free()


def test_a_straight_wall_reflects_like_the_method_of_images():
    """test_oracle_wake_obstacles' reflection measurement on the device (bit-identical to the specification's)."""
    gow, gw, _ = _gen(128, 2)
    gow, gi, _ = _gen(128, 2)
    n, dx = REFLECTION["n"], REFLECTION["dx"]
    mask, pulse, images = reflection_fields(**REFLECTION)
    for g in (gw, gi):
        _init(g, _params(n, dx, sponge_cells=0, sponge_damping=0.0))
    gw.wake_set_obstacles(mask, (0, 0))
    gw.set_wake_state(pulse, pulse)
    gi.set_wake_state(images, images)

    def step(g):
        def f(dt, S):
            g.wake_step(dt, S, (0, 0))
            return g.wake_state()[0]
        return f

    ratio, t = reflection_runs(step(gw), step(gi), **REFLECTION)
    print(f"straight wall against the method of images: {t:.0f} s compared, RMS difference {100 * ratio:.2f} % of the image run's")
    assert t >= 20.0 and ratio < REFLECTION_BOUND
    gw.free()
    gi.free()


def test_launch_counts_and_device_memory():
    gow, g, _ = _gen(128, 2)
    base = g.info().device_bytes
    n = 256
    _init(g, _params(n, 0.5))
    src = np.zeros(2, wk.SOURCE)
    src["x"], src["z"], src["vx"], src["radius"], src["head"], src["body"] = 40.0, 60.0, 2.0, 3.0, 0.3, -1

    def counts(S=3):
        before = g.info().kernel_launches
        g.wake_step(0.05 * S, S, (1, 0), src)
        return g.info().kernel_launches - before

    assert counts() == 3
    layer = g.info().device_bytes
    g.wake_set_obstacles(coastline(300, 200), (-10, -10))
    assert g.info().device_bytes == layer + 300 * 200                   # one byte per mask cell
    assert counts() == 3
    g.wake_set_obstacles(islands(300, 200), (5, 5))                      # same size: the block is reused
    assert g.info().device_bytes == layer + 300 * 200
    g.wake_set_obstacles(islands(64, 50), (5, 5))
    assert g.info().device_bytes == layer + 64 * 50
    g.wake_set_foam(**FOAM)
    g.wake_set_coupling(True)
    assert counts() == 4 and counts(5) == 6
    g.wake_set_coupling(False)
    g.wake_set_foam(None)
    g.wake_set_obstacles(None)
    assert g.info().device_bytes == layer
    g.wake_set_obstacles(coastline(100, 100))
    _init(g, _params(n, 0.5))                                           # ocean_wake_init releases the mask
    assert g.info().device_bytes == layer
    assert counts() == 3
    h, _, _ = g.wake_state()
    assert h.any()                                                       # nothing blocked after the re-create
    g.wake_set_obstacles(coastline(100, 100))
    _init(g, _params(0, 0.5))
    assert g.info().device_bytes == base
    g.free()


def test_invalid_arguments_launch_nothing_and_keep_the_mask():
    from godotoceanwaves_b200.native import load_library
    lib = load_library()
    gow, g, _ = _gen(128, 2)
    n = 256
    m = np.ones((4, 4), np.uint8)
    assert lib.ocean_wake_set_obstacles(g.context, m.ctypes.data, 4, 4, 0, 0) == STATE     # no layer
    p = _params(n, 0.5)
    _init(g, p)
    mask = coastline(n, n)
    g.wake_set_obstacles(mask, (0, 0))
    mem, before = g.info().device_bytes, g.info().kernel_launches
    I64_MAX = 2 ** 63 - 1
    big = np.zeros(1, np.uint8)
    bad = [(None, 4, 4, 0, 0), (m, 0, 4, 0, 0), (m, 4, 0, 0, 0), (m, -1, 4, 0, 0), (m, 4, -3, 0, 0), (None, 0, 4, 0, 0),
           (big, 16385, 16384, 0, 0), (big, 1 << 28, 2, 0, 0), (m, 4, 4, I64_MAX - 3, 0), (m, 4, 4, 0, I64_MAX)]
    for arr, w, d, ox, oz in bad:
        ptr = None if arr is None else arr.ctypes.data
        assert lib.ocean_wake_set_obstacles(g.context, ptr, w, d, ox, oz) == INVALID, (w, d, ox, oz)
    assert g.info().device_bytes == mem and g.info().kernel_launches == before
    # the previous mask is still in force: the next call matches the specification with it
    L = wo.Layer(p).set_obstacles(mask, (0, 0))
    src = np.zeros(1, wk.SOURCE)
    src["x"], src["z"], src["vx"], src["radius"], src["head"], src["body"] = 30.0, 30.0, 3.0, 3.0, 0.3, -1
    g.wake_step(0.1, 2, (1, 2), src)
    L.step(0.1, 2, (1, 2), src)
    h, hp, _ = g.wake_state()
    assert _same(h, L.h) and _same(hp, L.h_prev) and L.blocked().any()
    # the largest accepted origin: origin + size just representable
    assert lib.ocean_wake_set_obstacles(g.context, m.ctypes.data, 4, 4, I64_MAX - 4, I64_MAX - 4) == 0
    g.free()


def test_isolation_from_the_cascades():
    """Maps, foam, spectrum, velocity staleness and the next update are byte-identical with and without obstacle calls."""
    a, pa = _gen(256, 3)[1:]
    b, pb = _gen(256, 3)[1:]
    for g, p in ((a, pa), (b, pb)):
        g.update_all(1.0 / 50.0, p)
    _init(b, _params(512, 0.5))
    b.wake_set_obstacles(coastline(600, 600), (-20, -20))
    b.wake_step(0.1, 4, (3, 3), _sources(np.random.default_rng(2), 50, 256.0))
    b.wake_map()
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
