"""GPU tests of the wake layer (include/ocean.h, "Wake layer"): h, h_prev, the render map and samples byte-identical to
the specification oracle/wake.py after every call; sources attached to body states written by ocean_simulate_bodies_device;
scrolls; the Kelvin wedge, the rest state under a stationary source, the sponge and the stability bound; the device entry
points, launch counts, argument checks, device memory and isolation from the rest of the generator."""
import ctypes

import numpy as np
import pytest

from conftest import demo_params
from oracle import wake as wk

pytestmark = pytest.mark.gpu

INVALID, STATE = 1, 4


def _gen(N=128, C=2, updates=1):
    import godotoceanwaves_b200 as gow
    g = gow.WaveGenerator()
    g.map_size = N
    g.init_gpu(C)
    params = [demo_params(gow.WaveCascadeParameters, c) for c in range(C)]
    for _ in range(updates):
        g.update_all(1.0 / 50.0, params)
    return g, params


def _params(n, dx, damping=0.0, sponge_cells=16, sponge_damping=4.0):
    p = np.zeros((), wk.PARAMS)
    p["size"], p["cell_size"], p["damping"], p["sponge_cells"], p["sponge_damping"] = n, dx, damping, sponge_cells, sponge_damping
    return p


def _init(g, p):
    g.wake_init(int(p["size"]), float(p["cell_size"]), float(p["damping"]), int(p["sponge_cells"]), float(p["sponge_damping"]))


def _same(a, b):
    """Byte-identical, except that a NaN only has to meet a NaN."""
    a, b = np.asarray(a), np.asarray(b)
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


def _check(g, L, rng):
    h, hp, origin = g.wake_state()
    assert origin == L.origin
    assert _same(h, L.h) and _same(hp, L.h_prev)
    m, rect = g.wake_map()
    assert _same(m, L.render_map())
    x0, z0 = wk.world_origin(L.origin, L.cell_size)
    assert rect.tolist() == [x0, z0, np.float32(L.n) * L.cell_size, np.float32(L.n) * L.cell_size]
    ext = float(L.n * L.cell_size)
    pts = np.stack([rng.uniform(x0 - 0.1 * ext, x0 + 1.1 * ext, 500), rng.uniform(z0 - 0.1 * ext, z0 + 1.1 * ext, 500)], 1).astype(np.float32)
    assert _same(g.sample_wake(pts), L.sample(pts))


@pytest.mark.parametrize("n", [256, 512, 1024])
@pytest.mark.parametrize("dx", [0.25, 1.0])
def test_bit_exact_against_the_specification(n, dx):
    g, _ = _gen()
    rng = np.random.default_rng(n + int(dx * 8))
    p = _params(n, dx, damping=0.05, sponge_cells=24, sponge_damping=3.0)
    _init(g, p)
    L = wk.Layer(p)
    st = np.zeros(6, wk.STATE)
    st["position"] = rng.uniform(0, n * dx, (6, 3))
    st["linear_velocity"] = rng.uniform(-3, 3, (6, 3))
    h_max = np.sqrt(dx / wk.G)
    k = 24 if n < 1024 else 8
    plan = [(1, (0, 0)), (4, (3, -2)), (1, (-7, 5)), (4, (-7, 5)), (1, (-7 + n, 5)), (4, (40, 41))]
    for call, (S, origin) in enumerate(plan):
        s = _sources(rng, k, n * dx, len(st))
        if call == 2:                                   # non-finite and degenerate sources beside ordinary ones
            s["head"][0], s["x"][1], s["radius"][2], s["radius"][3], s["vz"][4] = np.nan, np.inf, 0.0, -2.0, np.inf
        if call == 4:
            s[:] = s[0]                                 # several identical sources: the order of their sum matters
        dt = 0.9 * h_max * S
        g.wake_step(dt, S, origin, s, st)
        L.step(dt, S, origin, s, st)
        _check(g, L, rng)
        if call == 0:
            assert np.abs(L.h).max() > 0
    g.free()


def test_many_overlapping_sources_keep_index_order():
    """700 sources crowded onto a few tiles: every warp of the cull keeps sources and the cull runs three 256-source chunks,
    so phi's sum order depends on the prefix over the warps and on the order across chunks.  Repeated identical sources and
    invalid ones (non-finite, radius <= 0, a body index not below num_states: device sources are not validated) sit in
    warps other than warp 0 and in later chunks.  Device entry point, byte-identical to the specification after every call."""
    import torch
    from godotoceanwaves_b200.native import check, load_library
    lib = load_library()
    g, _ = _gen()
    n, dx = 256, 0.5
    p = _params(n, dx, damping=0.05, sponge_cells=24, sponge_damping=1.0)
    _init(g, p)
    L = wk.Layer(p)
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
        s[300:312] = s[299]                              # repeats across warps 1..2 of chunk 1
        s[510:520] = s[3]                                # and of a warp-0 source into chunk 1's last warps
        s["head"][40], s["x"][97], s["radius"][130], s["radius"][260] = np.nan, np.inf, 0.0, -1.0
        s["vz"][390], s["radius"][520] = np.inf, np.inf
        s["body"][[200, 450, 650]] = len(st)             # not below num_states: contributes nothing
        src_d = torch.from_numpy(s.view(np.uint8).copy()).to(dev)
        dt = 0.05 * S
        torch.cuda.synchronize()
        check(lib.ocean_wake_step_device(g.context, dt, S, origin[0], origin[1], k, src_d.data_ptr(), len(st), st_d.data_ptr()))
        g.synchronize()
        L.step(dt, S, origin, s, st)
        _check(g, L, rng)
        if call == 0:
            # the crowding this test is about: every warp of the cull keeps sources on some tile, in every chunk
            cx, cz, r2, _, valid = wk.centres(s, st, 0.0)
            tile = (slice(96, 128), slice(96, 128))     # window cells 96..127 lie at 48..64 m
            lo, hi = (96 - 7 + 0.5) * dx, (128 + 7 + 0.5) * dx
            r = np.sqrt(r2)
            near = valid & (cx + r >= lo) & (cx - r <= hi) & (cz + r >= lo) & (cz - r <= hi)
            kept = np.flatnonzero(near)
            assert len(set(kept // 32)) >= 20 and len(set(kept // 256)) == 3
            assert np.count_nonzero(L.h[tile]) > 1000
    g.free()


def _body_scene(rng, n_bodies=5):
    """Bodies floating on the generator's maps; returns the FLOATING_BODY rows, states, points and drag areas."""
    from test_gpu_bodies import _bodies
    bodies, s0, hull, cda = _bodies(501, rng.integers(4, 20, n_bodies))
    return bodies, s0, hull, cda


def test_body_sources_follow_device_states():
    """States advanced by ocean_simulate_bodies_device stay on the device and drive the wake step through
    ocean_wake_step_device; the result equals the specification on those states copied back, and equals the host entry."""
    import torch
    import godotoceanwaves_b200 as gow
    from godotoceanwaves_b200.native import check, load_library
    lib = load_library()
    g, params = _gen(256, 3, updates=2)
    g2, _ = _gen(256, 3, updates=2)
    scales = gow.WaveGenerator.map_scales(params)
    rng = np.random.default_rng(77)
    bodies, s0, hull, cda = _body_scene(rng)
    s0["position"][:, 0] = rng.uniform(20, 100, len(s0))
    s0["position"][:, 2] = rng.uniform(20, 100, len(s0))
    s0["linear_velocity"][:, [0, 2]] = rng.uniform(-3, 3, (len(s0), 2))
    dev = torch.device("cuda", g.device)
    st_d = torch.from_numpy(s0.view(np.uint8).copy()).to(dev)
    hull_d = torch.from_numpy(hull.view(np.uint8).copy()).to(dev)
    cda_d = torch.from_numpy(cda).to(dev)
    p = _params(256, 0.5, damping=0.02)
    _init(g, p)
    _init(g2, p)
    L = wk.Layer(p)
    src = np.zeros(len(bodies), wk.SOURCE)
    src["radius"], src["head"], src["body"] = 2.0, 0.2, np.arange(len(bodies))
    src_d = torch.from_numpy(src.view(np.uint8).copy()).to(dev)
    sc = np.ascontiguousarray(scales, np.float32)
    for call in range(3):
        torch.cuda.synchronize()
        check(lib.ocean_simulate_bodies_device(g.context, len(bodies), bodies.ctypes.data, st_d.data_ptr(), len(hull), hull_d.data_ptr(),
                                               cda_d.data_ptr(), 3, sc.ctypes.data, 1025.0, 1.0 / 60.0, 2, 1e-3, 8, None, None, None))
        check(lib.ocean_wake_step_device(g.context, 1.0 / 60.0, 2, 0, 0, len(src), src_d.data_ptr(), len(bodies), st_d.data_ptr()))
        g.synchronize()
        states = np.frombuffer(st_d.cpu().numpy().tobytes(), wk.STATE)
        g2.wake_step(1.0 / 60.0, 2, (0, 0), src, states)
        L.step(1.0 / 60.0, 2, (0, 0), src, states)
        h, hp, _ = g.wake_state()
        h2, hp2, _ = g2.wake_state()
        assert _same(h, L.h) and _same(hp, L.h_prev) and h.tobytes() == h2.tobytes() and hp.tobytes() == hp2.tobytes()
    assert np.count_nonzero(L.h) > 100
    # the device sample equals the host sample
    pts = rng.uniform(0, 128, (300, 2)).astype(np.float32)
    out_d = torch.zeros(900, dtype=torch.float32, device=dev)
    pts_d = torch.from_numpy(pts).to(dev)
    check(lib.ocean_sample_wake_device(g.context, len(pts), pts_d.data_ptr(), out_d.data_ptr()))
    g.synchronize()
    assert out_d.cpu().numpy().tobytes() == g.sample_wake(pts).tobytes()
    g.free()
    g2.free()


def test_launch_counts_and_invalid_arguments():
    from godotoceanwaves_b200.native import load_library
    lib = load_library()
    g, _ = _gen()
    n = 256
    assert lib.ocean_wake_step(g.context, 0.01, 1, 0, 0, 0, None, 0, None) == STATE          # no layer yet
    _init(g, _params(n, 0.5))
    rng = np.random.default_rng(3)
    h0 = rng.normal(size=(n, n)).astype(np.float32)
    g.set_wake_state(h0, h0 * 0.5, (5, 6))
    s = _sources(rng, 10, 128.0, 2)
    st = np.zeros(2, wk.STATE)
    for S in (1, 3, 7):
        before = g.info().kernel_launches
        g.wake_step(0.05 * S, S, (5, 6), s, st)
        assert g.info().kernel_launches - before == S
    before = g.info().kernel_launches
    g.wake_map()
    g.sample_wake(np.zeros((5, 2), np.float32))
    assert g.info().kernel_launches - before == 2
    h, hp, o = g.wake_state()
    h_max = np.sqrt(0.5 / wk.G)
    big = np.float32(h_max)
    while big * big * 9.81 / 0.5 * 4 <= 4.0:
        big = np.nextafter(big, np.float32(1))
    bad_body = s.copy()
    bad_body["body"][0] = 2
    P = ctypes.c_void_p
    cases = [
        (0.0, 1, s, st), (np.nan, 1, s, st), (np.inf, 1, s, st), (-0.1, 1, s, st), (0.05, 0, s, st), (0.05, 257, s, st),
        (float(big), 1, s, st), (0.05, 1, bad_body, st), (0.05, 1, s, st[:0]),
    ]
    before = g.info().kernel_launches
    for dt, S, src, sts in cases:
        rc = lib.ocean_wake_step(g.context, dt, S, 9, 9, len(src), src.ctypes.data, len(sts), sts.ctypes.data if len(sts) else None)
        assert rc == INVALID, (dt, S)
    assert lib.ocean_wake_step(g.context, 0.05, 1, 9, 9, 3, None, 0, None) == INVALID
    assert lib.ocean_wake_step(g.context, 0.05, 1, 9, 9, -1, None, 0, None) == INVALID
    assert lib.ocean_wake_step_device(g.context, float(big), 1, 9, 9, 0, None, 0, None) == INVALID
    assert lib.ocean_wake_render_map(g.context, None, None) == INVALID
    assert lib.ocean_sample_wake(g.context, -1, None, None) == INVALID
    assert lib.ocean_sample_wake(g.context, 3, None, None) == INVALID
    for bad in [(100, 16, 0.5, 0.0, 1.0), (4096, 16, 0.5, 0.0, 1.0), (256, 65, 0.5, 0.0, 1.0), (128, 65, 0.5, 0.0, 1.0),
                (256, 16, 0.0, 0.0, 1.0), (256, 16, np.nan, 0.0, 1.0), (256, 16, 0.5, -1.0, 1.0), (256, 16, 0.5, 0.0, np.inf),
                (256, -1, 0.5, 0.0, 1.0)]:
        p = np.array(bad, g.WAKE_PARAMS)
        assert lib.ocean_wake_init(g.context, p.ctypes.data) == INVALID, bad
    assert g.info().kernel_launches == before
    h2, hp2, o2 = g.wake_state()
    assert h2.tobytes() == h.tobytes() and hp2.tobytes() == hp.tobytes() and o2 == o
    # the largest accepted sub-step is accepted
    ok = np.nextafter(big, np.float32(0))
    assert lib.ocean_wake_step(g.context, float(ok), 1, 9, 9, 0, None, 0, None) == 0
    g.free()


def test_stability_at_the_largest_sub_step():
    """10^4 sub-steps of a random field at the largest accepted sub-step, no damping and no sponge, stay bounded."""
    g, _ = _gen()
    n, dx = 256, 0.5
    _init(g, _params(n, dx, damping=0.0, sponge_cells=0, sponge_damping=0.0))
    h = np.float32(np.sqrt(dx / wk.G))
    while not wk.stable(dx, h):
        h = np.nextafter(h, np.float32(0))
    assert not wk.stable(dx, np.nextafter(h, np.float32(1)))
    rng = np.random.default_rng(11)
    h0 = rng.uniform(-1, 1, (n, n)).astype(np.float32)
    g.set_wake_state(h0, h0)
    for _ in range(40):
        g.wake_step(float(h) * 250, 250, (0, 0))
    hh, hp, _ = g.wake_state()
    assert np.all(np.isfinite(hh)) and np.abs(hh).max() < 50.0, np.abs(hh).max()
    g.free()


def test_device_memory_is_exact():
    g, _ = _gen()
    base = g.info().device_bytes
    _init(g, _params(256, 0.5))
    assert g.info().device_bytes == base + 4 * 4 * 256 * 256
    g.wake_step(0.05, 1, (0, 0), _sources(np.random.default_rng(1), 300, 128.0))
    staged = g.info().device_bytes
    _init(g, _params(1024, 0.5))
    assert g.info().device_bytes == staged + 4 * 4 * (1024 * 1024 - 256 * 256)
    g.sample_wake(np.random.default_rng(2).uniform(0, 512, (100, 2)))    # its staging goes with the layer too
    _init(g, _params(0, 0.5))
    assert g.info().device_bytes == base
    g.free()


def test_isolation_from_the_cascades():
    """Maps, foam, spectrum, velocity staleness and the next update are byte-identical with and without wake calls."""
    import godotoceanwaves_b200 as gow
    a, pa = _gen(256, 3, updates=2)
    b, pb = _gen(256, 3, updates=2)
    _init(b, _params(512, 0.5))
    b.wake_step(0.1, 4, (3, 3), _sources(np.random.default_rng(2), 50, 256.0))
    b.wake_map()
    b.sample_wake(np.zeros((10, 2), np.float32))
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


def test_kelvin_wedge():
    """A source moving along +x at U = 2.5 m/s with radius 4 m (Froude number U / sqrt(g radius) = 0.40) on dx = 0.5 m
    (the Kelvin wavelength 2 pi U^2 / g = 4.0 m is 8 cells, inside the stencil's band); the window follows the source.
    Method: for each cross-section 20-60 m behind the source, the lateral offset of the largest |h| on each side (|h| first
    smoothed by a maximum over 2 m along the section, which removes the wave phase) is taken; a line through the origin fitted
    to (distance, offset) gives the half-angle atan(slope), averaged over the two sides."""
    g, _ = _gen()
    n, dx, U, r = 1024, 0.5, 2.5, 4.0
    _init(g, _params(n, dx, damping=0.0, sponge_cells=48, sponge_damping=3.0))
    h_sub = 1.0 / 30.0
    T = 60.0
    steps = int(round(T / h_sub))
    src = np.zeros(1, wk.SOURCE)
    src["radius"], src["head"], src["body"] = r, 0.2, -1
    # the source sits at cell (768, 512) of the window; its world x at time t is U t
    for k in range(0, steps, 30):
        t0 = k * h_sub
        src["x"], src["z"], src["vx"] = U * t0, 0.0, U
        ox = int(np.floor(U * t0 / dx)) - 768
        g.wake_step(h_sub * 30, 30, (ox, -512), src)
    h, _, origin = g.wake_state()
    xs = U * T
    x0, z0 = origin[0] * dx, origin[1] * dx
    from scipy.ndimage import maximum_filter1d
    offsets = {1: [], -1: []}
    dists = np.arange(20.0, 60.5, 2.0)
    for d in dists:
        i = int(round((xs - d - x0) / dx - 0.5))
        col = maximum_filter1d(np.abs(h[:, i - 1:i + 2]).max(1), size=int(2.0 / dx) * 2 + 1)
        zc = (np.arange(n) + 0.5) * dx + z0
        for side in (1, -1):
            m = (side * zc > 1.0) & (side * zc < d)
            offsets[side].append(abs(zc[m][np.argmax(col[m])]))
    angles = []
    for side in (1, -1):
        o = np.array(offsets[side])
        slope = (dists @ o) / (dists @ dists)
        angles.append(np.degrees(np.arctan(slope)))
    angle = float(np.mean(angles))
    print(f"Kelvin half-angle {angle:.2f} deg (sides {angles[0]:.2f}, {angles[1]:.2f})")
    assert abs(angle - 19.47) <= 3.0, angles
    g.free()


def test_stationary_source_settles_to_the_depression():
    """A stationary source with damping alpha = 0.002 / s: the rest state of the scheme solves G(h + phi) =
    -(2 alpha dx / (g h_sub)) h, a relative deviation of about 2 alpha / (g h_sub |k|) ~ 1.4 % for this 10 m patch
    (|k| ~ 1 / radius) at h_sub = 0.3 s; 6000 s of simulated time leave exp(-6) of the start-up transient (modes decay
    at alpha / 2, the sponge takes the radiated waves).  Tolerance: 5 % of the head at the centre, 10 % of phi's RMS
    under the patch."""
    g, _ = _gen()
    n, dx = 256, 1.0
    _init(g, _params(n, dx, damping=0.002, sponge_cells=48, sponge_damping=1.0))
    src = np.zeros(1, wk.SOURCE)
    src["x"], src["z"], src["radius"], src["head"], src["body"] = 128.0, 128.0, 10.0, 0.3, -1
    for _ in range(80):
        g.wake_step(0.3 * 250, 250, (0, 0), src)
    h, _, _ = g.wake_state()
    phi = wk.rasterise(n, dx, (0, 0), src, None, 0.0)
    centre = h[128, 128] + phi[128, 128]
    patch = phi != 0
    rms = np.sqrt(np.mean((h[patch] + phi[patch]) ** 2)) / np.sqrt(np.mean(phi[patch] ** 2))
    print(f"rest state: centre deviation {centre / 0.3:+.4f} of the head, RMS deviation {rms:.4f} of phi")
    assert abs(centre) <= 0.05 * 0.3 and rms <= 0.10
    g.free()


def test_sponge_absorbs_outgoing_waves():
    """A pulse on a 256-cell window and, centred on the same cells, on a 1024-cell window, both with a 48-cell sponge ramping
    to 1 / s.  Until a wave at the scheme's largest group velocity could have gone from the small window's edge to the large
    window's sponge and back (and for at most 60 s), the large run is the unbounded answer on the small window's interior
    (inside its sponge), so the difference there is what the small window's sponge and edge reflect.  The pulse is a ring,
    0.2 cos(|r| / dx) exp(-|r|^2 / (2 (6 dx)^2)), whose energy lies in the stencil's band (wavelength 6.3 cells); waves
    longer than the band are also slower than deep water and are not what the sponge is sized for.  Measure: the RMS of the
    difference over all snapshots (one per second) over the RMS of the large run, below 5 %."""
    gs, _ = _gen()
    gl, _ = _gen()
    dx, sc, h_sub = 0.5, 48, 0.2
    _init(gs, _params(256, dx, 0.0, sc, 1.0))
    _init(gl, _params(1024, dx, 0.0, sc, 1.0))
    i = np.arange(256)
    r2 = (i[None, :] - 128.0) ** 2 + (i[:, None] - 128.0) ** 2
    pulse = (0.2 * np.cos(np.sqrt(r2)) * np.exp(-r2 / (2 * 6.0 ** 2))).astype(np.float32)
    big = np.zeros((1024, 1024), np.float32)
    big[384:640, 384:640] = pulse
    gs.set_wake_state(pulse, pulse, (0, 0))
    gl.set_wake_state(big, big, (-384, -384))
    # the largest group velocity of the discrete dispersion, binary64 on a fine grid of |k| dx along an axis and the diagonal
    g = wk.taps()
    k = np.linspace(1e-3, np.pi, 4000)
    a3 = wk.G * h_sub * h_sub / dx
    cg = 0.0
    for th in (0.0, np.pi / 4):
        w = np.arccos(np.clip(1.0 - a3 * wk.symbol(g, k * np.cos(th), k * np.sin(th)) / 2.0, -1, 1)) / h_sub
        cg = max(cg, float(np.max(np.diff(w) / np.diff(k / dx))))
    t_end = min(60.0, 2 * (384 - sc) * dx / cg)
    core = slice(sc, 256 - sc)
    num = den = 0.0
    t = 0.0
    while t + 1.0 <= t_end + 1e-9:
        gs.wake_step(1.0, 5, (0, 0))
        gl.wake_step(1.0, 5, (-384, -384))
        t += 1.0
        hs = gs.wake_state()[0][core, core].astype(np.float64)
        hl = gl.wake_state()[0][384:640, 384:640][core, core].astype(np.float64)
        num += np.sum((hs - hl) ** 2)
        den += np.sum(hl ** 2)
    ratio = np.sqrt(num / den)
    print(f"sponge: {t:.0f} s compared (largest group velocity {cg:.2f} m/s), reflected RMS {100 * ratio:.2f} % of the large run's")
    assert t >= 30.0 and ratio < 0.05
    gs.free()
    gl.free()
