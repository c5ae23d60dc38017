"""GPU tests of the wake layer across the whole range include/ocean.h accepts (window sizes 128 and 2048, sponge widths 0 to
min(64, N/2), 256 sub-steps at the largest accepted sub-step, ~10^4 sources on one tile and 2^16 over a 2048 window, origins
near +-2^31, +-2^40 and the int64 ends, cell sizes 1e-3 and 1e20): after every call h, h_prev, the render map (four
channels), 500 wake samples, F and the coupling's snapshots with their origins and T are byte-identical to the specification
(oracle/wake*.py), a NaN only meeting a NaN; and for one call per window size the device's h and F are within the a-priori
bound of tests/test_oracle_wake_model64.py of the binary64 model written from the header."""
import time

import numpy as np
import pytest

from oracle import wake as wk
from oracle import wake_coupling as wc
from oracle import wake_foam as wf
from oracle import wake_model64 as m64
from oracle import wake_obstacles as wo
from test_gpu_sampling import _gen
from test_oracle_wake_model64 import largest_substep, model_call

pytestmark = pytest.mark.gpu

INVALID = 1
I64_MAX, I64_MIN = 2 ** 63 - 1, -2 ** 63
FOAM = dict(whitecap=0.05, grow_rate=2.0, stir_rate=0.3, decay_rate=0.5)


def _params(n, dx, damping=0.05, sponge_cells=16, sponge_damping=1.0):
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


def _points(L, rng, k=500):
    """k points: random over the window and 5 % around it, plus points on and one binary32 step beyond all four edges (the
    window's binary32 corner and x0 + N dx); when the corner is not finite, points spread over the binary32 range."""
    x0, z0 = wk.world_origin(L.origin, L.cell_size)
    ext = np.float32(L.n) * L.cell_size
    if not (np.isfinite(x0) and np.isfinite(z0)):
        return rng.uniform(-3e38, 3e38, (k, 2)).astype(np.float32)
    with np.errstate(all="ignore"):
        x1, z1 = x0 + ext, z0 + ext
    lo, hi = np.float32(-np.inf), np.float32(np.inf)
    mid_x, mid_z = np.float32(float(x0) + 0.37 * float(ext)), np.float32(float(z0) + 0.61 * float(ext))
    edges = [(x0, mid_z), (np.nextafter(x0, lo), mid_z), (x1, mid_z), (np.nextafter(x1, lo), mid_z),
             (mid_x, z0), (mid_x, np.nextafter(z0, lo)), (mid_x, z1), (mid_x, np.nextafter(z1, lo)),
             (x0, z0), (np.nextafter(x1, lo), np.nextafter(z1, lo)), (np.nextafter(x0, hi), np.nextafter(z0, hi))]
    r = rng.uniform(-0.05, 1.05, (k - len(edges), 2))
    pts = np.stack([float(x0) + r[:, 0] * float(ext), float(z0) + r[:, 1] * float(ext)], 1)
    return np.concatenate([np.array(edges, np.float64), pts]).astype(np.float32)


def _check(g, L, rng, cp=None):
    h, hp, origin = g.wake_state()
    assert origin == L.origin
    assert _same(h, L.h) and _same(hp, L.h_prev)
    m, rect = g.wake_map()
    assert _same(m, L.render_map())
    x0, z0 = wk.world_origin(L.origin, L.cell_size)
    assert _same(rect[:2], np.array([x0, z0], np.float32))
    if L.foam_on:
        assert _same(g.wake_foam(), L.foam)
    pts = _points(L, rng)
    assert _same(g.sample_wake(pts), L.sample(pts))
    if cp is not None:
        e, e_old, origins, T = g.wake_coupling()
        assert _same(e, cp.e) and _same(e_old, cp.e_old) and T == cp.T
        assert origins == (cp.origin_e, cp.origin_old)


def _sources(rng, k, L, origin, n_states=0, spread=1.0):
    """k sources over the window at `origin` and straddling its edges; some moving, some on bodies, a few invalid."""
    s = np.zeros(k, wk.SOURCE)
    dx = float(L.cell_size)
    x0, z0 = (float(v) for v in wk.world_origin(origin, dx))
    ext = L.n * dx
    s["x"] = x0 + rng.uniform(-0.05, 1.05, k) * ext * spread
    s["z"] = z0 + rng.uniform(-0.05, 1.05, k) * ext * spread
    s["vx"], s["vz"] = rng.uniform(-3, 3, k), rng.uniform(-3, 3, k)
    s["radius"] = rng.uniform(1.5, 10, k) * dx
    s["head"] = rng.uniform(-0.3, 0.3, k)
    s["body"] = -1
    if n_states:
        att = rng.random(k) < 0.3
        s["body"][att] = rng.integers(0, n_states, att.sum())
        s["x"][att], s["z"][att] = rng.uniform(-2, 2, att.sum()) * dx, rng.uniform(-2, 2, att.sum()) * dx
    if k > 8:
        s["head"][3], s["radius"][5], s["x"][7] = np.nan, 0.0, np.inf
    return s


def _states(rng, L, origin, k=4):
    st = np.zeros(k, wk.STATE)
    dx = float(L.cell_size)
    x0, z0 = (float(v) for v in wk.world_origin(origin, dx))
    st["position"][:, 0] = x0 + rng.uniform(0, L.n * dx, k)
    st["position"][:, 2] = z0 + rng.uniform(0, L.n * dx, k)
    st["linear_velocity"] = rng.uniform(-2, 2, (k, 3))
    return st


def _launches(g, fn):
    before = g.info().kernel_launches
    fn()
    return g.info().kernel_launches - before


@pytest.mark.parametrize("n", [128, 2048])
def test_window_sizes_every_kernel_form(n):
    """Plain, foam, obstacles and foam + obstacles, the coupling on from the third call; S = 1 and 2 at the largest sub-step;
    scrolls by (3, -2) and by N cells or more; samples on and beyond the four edges."""
    t0 = time.time()
    _, g, _ = _gen(128, 2)
    dx = 0.5
    p = _params(n, dx, damping=0.05, sponge_cells=24 if n == 128 else 64, sponge_damping=2.0)
    _init(g, p)
    L = wo.Layer(p, wf.foam_params(**FOAM))
    L.foam_on = False
    rng = np.random.default_rng(n)
    h = float(largest_substep(dx))
    k = 40 if n == 128 else 8
    mask = (rng.random((n + n // 2, n + n // 3)) < 0.02).astype(np.uint8)
    mask[n // 3:n // 3 + 7, :] = 1
    mo = (-n // 4, n // 8)
    cp = None
    plan = [(1, (0, 0), "plain"), (2, (3, -2), "obstacles"), (1, (3 - n, -2), "foam"), (2, (6, n // 2), "foam+obstacles")]
    for call, (S, origin, form) in enumerate(plan):
        if "foam" in form and not L.foam_on:
            g.wake_set_foam(**FOAM)
            L.foam_on, L.foam = True, np.zeros_like(L.h)
        if ("obstacles" in form) != (L.mask is not None):
            g.wake_set_obstacles(mask if "obstacles" in form else None, mo)
            L.set_obstacles(mask if "obstacles" in form else None, mo)
        if call == 2:
            g.wake_set_coupling(True)
            cp = wc.Coupling(n, dx)
        st = _states(rng, L, origin)
        s = _sources(rng, k, L, origin, len(st))
        launches = _launches(g, lambda: g.wake_step(h * S, S, origin, s, st))
        assert launches == S + (cp is not None)
        wo.step(L, cp, h * S, S, origin, s, st)
        _check(g, L, rng, cp)
        if "obstacles" in form:
            assert L.blocked().any() and not L.blocked().all()
    assert np.abs(L.h).max() > 0 and L.foam.max() > 0
    g.free()
    print(f"window {n}: {time.time() - t0:.1f} s")


def test_the_sub_step_cap():
    """One call of S = 256 at exactly the largest accepted sub-step, with the coupling (257 launches) and without (256); the
    next binary32 dt is rejected with no launch and no change."""
    _, g, _ = _gen(128, 2)
    n, dx = 128, 0.5
    p = _params(n, dx, damping=0.0, sponge_cells=32, sponge_damping=1.0)
    _init(g, p)
    L = wo.Layer(p)
    rng = np.random.default_rng(256)
    h = largest_substep(dx)
    dt = float(h) * 256                                         # exact: a binary32 times a power of two
    s = _sources(rng, 12, L, (0, 0))
    assert _launches(g, lambda: g.wake_step(dt, 256, (0, 0), s)) == 256
    wo.step(L, None, dt, 256, (0, 0), s)
    _check(g, L, rng)
    g.wake_set_coupling(True)
    cp = wc.Coupling(n, dx)
    assert _launches(g, lambda: g.wake_step(dt, 256, (2, -1), s)) == 257
    wo.step(L, cp, dt, 256, (2, -1), s)
    _check(g, L, rng, cp)
    from godotoceanwaves_b200.native import load_library
    lib = load_library()
    bad = float(np.nextafter(np.float32(dt), np.float32(np.inf)))
    before = g.wake_state()
    rcs = []
    assert _launches(g, lambda: rcs.extend(lib.ocean_wake_step(g.context, t, S, 2, -1, 0, None, 0, None)
                                           for t, S in ((bad, 256), (dt, 257)))) == 0
    assert rcs == [INVALID, INVALID]
    after = g.wake_state()
    assert _same(before[0], after[0]) and _same(before[1], after[1])
    g.free()


@pytest.mark.parametrize("sponge_cells", [0, 1, 63, 64])
def test_sponge_extremes(sponge_cells):
    """sponge_cells 0, 1, 63 and 64 at N = 128 (64: every cell is in the sponge, the table's last slot is the centre's),
    damping above and below sponge_damping, with foam; and 64 at N = 2048 once."""
    _, g, _ = _gen(128, 2)
    rng = np.random.default_rng(sponge_cells)
    for damping, sponge_damping in ((0.05, 3.0), (2.0, 0.2)):
        p = _params(128, 0.25, damping, sponge_cells, sponge_damping)
        _init(g, p)
        g.wake_set_foam(**FOAM)
        L = wo.Layer(p, wf.foam_params(**FOAM))
        h0 = rng.standard_normal((128, 128)).astype(np.float32) * np.float32(0.05)
        g.set_wake_state(h0, h0)
        L.h, L.h_prev = h0.copy(), h0.copy()
        h = float(largest_substep(0.25))
        for S, origin in ((1, (0, 0)), (3, (-5, 4))):
            s = _sources(rng, 16, L, origin)
            g.wake_step(h * S, S, origin, s)
            wo.step(L, None, h * S, S, origin, s)
            _check(g, L, rng)
    g.free()


def test_crowded_sources():
    """~10^4 sources over one 32 x 32 tile at N = 128 (40 cull chunks) with invalid sources at chunk and warp boundaries
    and body indices num_states - 1 and num_states through ocean_wake_step_device, with foam; then 2^16 sources over a 2048
    window."""
    import torch
    from godotoceanwaves_b200.native import check, load_library
    lib = load_library()
    _, g, _ = _gen(128, 2)
    n, dx = 128, 0.5
    p = _params(n, dx, damping=0.05, sponge_cells=16)
    _init(g, p)
    g.wake_set_foam(**FOAM)
    L = wo.Layer(p, wf.foam_params(**FOAM))
    rng = np.random.default_rng(10000)
    k = 10000
    st = np.zeros(3, wk.STATE)
    st["position"][:, [0, 2]] = rng.uniform(20, 28, (3, 2))
    st["linear_velocity"][:, [0, 2]] = rng.uniform(-1, 1, (3, 2))
    s = np.zeros(k, wk.SOURCE)
    s["x"], s["z"] = rng.uniform(16, 32, k), rng.uniform(16, 32, k)      # cells 32..63: one tile
    s["vx"], s["vz"] = rng.uniform(-1, 1, k), rng.uniform(-1, 1, k)
    s["radius"] = rng.uniform(0.3, 2.0, k)
    s["head"] = rng.uniform(-0.01, 0.01, k)
    s["body"] = -1
    att = rng.random(k) < 0.1
    s["body"][att] = rng.integers(0, len(st), att.sum())
    s["x"][att], s["z"][att] = rng.uniform(-3, 3, att.sum()), rng.uniform(-3, 3, att.sum())
    edges = [31, 32, 255, 256, 257, 511, 512, 4095, 4096, 8191, 8192, 9983, 9984, 9999]
    s["head"][edges[0::3]] = np.nan
    s["radius"][edges[1::3]] = -1.0
    s["body"][edges[2::3]] = len(st)                                        # not below num_states: nothing
    s["body"][[100, 6000]] = len(st) - 1
    dev = torch.device("cuda", g.device)
    src_d = torch.from_numpy(s.view(np.uint8).copy()).to(dev)
    st_d = torch.from_numpy(st.view(np.uint8).copy()).to(dev)
    torch.cuda.synchronize()
    for S, origin in ((2, (0, 0)), (1, (3, -2))):
        check(lib.ocean_wake_step_device(g.context, 0.05 * S, S, origin[0], origin[1], k, src_d.data_ptr(), len(st), st_d.data_ptr()))
        g.synchronize()
        L.step(0.05 * S, S, origin, s, st)
        _check(g, L, rng)
    assert np.abs(L.h[10:40, 30:70]).max() > 0 and L.foam.max() > 0
    # 2^16 sources spread over a 2048 window
    n = 2048
    p = _params(n, 0.5, damping=0.05, sponge_cells=64)
    _init(g, p)
    L = wo.Layer(p)
    s = _sources(rng, 1 << 16, L, (-7, 11))
    s["radius"] = rng.uniform(0.5, 3.0, len(s))
    g.wake_step(0.1, 1, (-7, 11), s)
    L.step(0.1, 1, (-7, 11), s)
    _check(g, L, rng)
    g.free()


FAR = [(2 ** 31 + 3, -(2 ** 31) - 2), (-(2 ** 31) + 5, 2 ** 31 - 7), (2 ** 40, -(2 ** 40)), (I64_MAX - 100, I64_MIN + 5)]


@pytest.mark.parametrize("dx", [0.5, 1e-3, 1e20])
def test_far_origins(dx):
    """Windows near +-2^31, +-2^40 and within N of the int64 ends, with foam, obstacles and the coupling; a scroll from one
    int64 end to the other; a mask at the opposite end (the +-2^30 offset clamp) and one the window steps across; cell
    sizes 1e-3 and 1e20 (the corner inexact, or +-inf)."""
    _, g, _ = _gen(128, 2)
    n = 128
    p = _params(n, dx, damping=0.05, sponge_cells=8)
    _init(g, p)
    L = wo.Layer(p, wf.foam_params(**FOAM))
    g.wake_set_foam(**FOAM)
    g.wake_set_coupling(True)
    cp = wc.Coupling(n, dx)
    rng = np.random.default_rng(int(np.log10(dx) + 40))
    h = float(largest_substep(dx))
    mask = np.ones((40, 300), np.uint8)
    mask[:, 100:110] = 0
    plan = [(o, 1) for o in FAR] + [((I64_MIN + 2, I64_MAX - 200), 2), ((I64_MAX - 127, I64_MIN), 1)]
    for origin, S in plan:
        if origin[0] == I64_MIN + 2:                                  # a mask at the far end of the x axis: clamped away
            g.wake_set_obstacles(mask, (I64_MAX - 400, I64_MAX - 240))
            L.set_obstacles(mask, (I64_MAX - 400, I64_MAX - 240))
        if origin[0] == I64_MAX - 127:                                 # the window's cells reach past the mask's edge
            g.wake_set_obstacles(mask, (I64_MAX - 350, I64_MIN + 60))
            L.set_obstacles(mask, (I64_MAX - 350, I64_MIN + 60))
        st = _states(rng, L, origin) if np.isfinite(wk.world_origin(origin, dx)[0]) else None
        s = _sources(rng, 24, L, origin, 0 if st is None else len(st)) if st is not None else _sources(rng, 24, L, (0, 0))
        with np.errstate(all="ignore"):
            g.wake_step(h * S, S, origin, s, st)
            wo.step(L, cp, h * S, S, origin, s, st)
            _check(g, L, rng, cp)
    # a step across the mask's edge: the window one cell further on each call
    for d in (1, 2, 3):
        origin = (I64_MAX - 127 - 60 * d, I64_MIN + 30 * d)
        s = _sources(rng, 12, L, (0, 0))
        with np.errstate(all="ignore"):
            g.wake_step(h, 1, origin, s)
            wo.step(L, cp, h, 1, origin, s)
            _check(g, L, rng, cp)
        assert L.blocked().any() and not L.blocked().all()
    g.free()


def test_far_origin_centres_against_the_exact_ones():
    """How far the binary32 cell centres x0 + (i + 1/2) dx, which phi and the samples use, lie from the exact centres
    (ox + i + 1/2) dx, in cells, at growing distances from the world origin (host arithmetic: the device is bit-identical to
    the specification, which the other tests check).  The header states the limit: about 2^-24 |x0| / dx cells, so a
    window more than 2^22 cells out places sources to within a quarter cell or worse."""
    for dx in (0.5, 1.0, 0.1):
        for e in (16, 22, 24, 31, 40):
            ox = 2 ** e + 3
            px, _ = m64.cell_centres(128, dx, (ox, 0))
            x0 = np.float32(m64.corner((ox, 0), dx)[0])
            p32 = (x0 + (np.arange(128, dtype=np.float32) + np.float32(0.5)) * np.float32(dx)).astype(np.float64)
            err = np.abs(p32 - px).max() / float(np.float32(dx))
            print(f"dx {dx}: ox 2^{e}: centres off by up to {err:.3g} cells (2^-24 |x0| / dx = {2.0 ** -24 * abs(float(x0)) / float(np.float32(dx)):.3g})")
            assert err <= 2.0 ** -23 * abs(float(x0)) / float(np.float32(dx)) + 1e-6


@pytest.mark.parametrize("n", [128, 2048])
def test_device_against_the_binary64_model(n):
    """One call per window size from a random start state with foam and sources: the device's h and F against the binary64
    model started from the device's own state (ocean_wake_get_state, ocean_wake_get_foam_state), within the a-priori bound."""
    _, g, _ = _gen(128, 2)
    dx = 0.25
    p = _params(n, dx, damping=0.1, sponge_cells=48, sponge_damping=2.0)
    _init(g, p)
    g.wake_set_foam(**FOAM)
    rng = np.random.default_rng(64 + n)
    h0 = rng.standard_normal((n, n)).astype(np.float32) * np.float32(0.05)
    g.set_wake_state(h0, h0 * np.float32(0.9))
    g.set_wake_foam(rng.uniform(0, 1, (n, n)).astype(np.float32))
    dh, dhp, origin = g.wake_state()
    dF = g.wake_foam()
    M = m64.Model(p, (FOAM["whitecap"], FOAM["grow_rate"], FOAM["stir_rate"], FOAM["decay_rate"]))
    M.h, M.h_prev, M.F, M.origin = dh.astype(np.float64), dhp.astype(np.float64), dF.astype(np.float64), origin
    L = wo.Layer(p)
    s = _sources(rng, 8, L, (3, -2))
    h = float(largest_substep(dx))
    g.wake_step(h, 1, (3, -2), s)
    eh, ef, _ = model_call(M, h, 1, (3, -2), s, None)
    gh, _, _ = g.wake_state()
    gF = g.wake_foam()
    err, errf = np.abs(gh - M.h), np.abs(gF - M.F)
    print(f"device against the binary64 model at {n}: h error / bound max {np.max(err / eh):.3f}, F {np.max(errf / np.maximum(ef, 1e-300)):.3f}")
    assert np.all(err <= eh) and np.all(errf <= ef)
    assert eh.max() <= 1e-3 * np.abs(M.h).max()
    g.free()
