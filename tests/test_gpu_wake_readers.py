"""GPU tests of the wake readers (include/ocean.h, "Wake layer", Readers; ocean_wake_set_readers): the ray cast on the coupled
surface and spray from the wake layer, byte-identical to the specification oracle/wake_readers.py over moving and
body-attached sources, a scrolled window, an obstacle mask and foam; readers 0 (and the ray cast bit on an uncoupled or
unprimed layer) byte-identical to a generator without a layer, with no extra launch; the visible effects (a ray hits a wake
crest it misses uncoupled, spray on a stirred trail, particle heights on h); validation; and a 2048^2 layer with 2^20 rays."""
import numpy as np
import pytest

from oracle import raycast as rc
from oracle import spray as sp
from oracle import spray_particles as spp
from oracle import wake as wk
from oracle import wake_coupling as wc
from oracle import wake_foam as wf
from oracle import wake_obstacles as wo
from oracle import wake_readers as wr
from test_gpu_raycast import _extreme_rays, _records_match
from test_gpu_sampling import _gen, _same_or_both_nan
from test_gpu_surface import _scales
from test_oracle_raycast import grazing, ray_mix
from test_oracle_wake_obstacles import FOAM, islands

pytestmark = pytest.mark.gpu

INVALID, STATE = 1, 4
RAYCAST, SPRAY = 1, 2
PS = (20.0, 8.5, 20.0)


def _params(n, dx, damping=0.05, sponge_cells=16, sponge_damping=1.0):
    p = np.zeros((), wk.PARAMS)
    p["size"], p["cell_size"], p["damping"], p["sponge_cells"], p["sponge_damping"] = n, dx, damping, sponge_cells, sponge_damping
    return p


def _init(g, p):
    g.wake_init(int(p["size"]), float(p["cell_size"]), float(p["damping"]), int(p["sponge_cells"]), float(p["sponge_damping"]))


def _launches(g, fn):
    before = g.info().kernel_launches
    out = fn()
    return g.info().kernel_launches - before, out


def _cast(g, rays, scales):
    """(launches, record bytes) of one ray cast"""
    k, rec = _launches(g, lambda: g.raycast(rays, scales))
    return k, rec.tobytes()


def _emitter(amount=32768, transform=15 * np.eye(3, 4)):
    e = spp.default_emitter()
    e["amount"] = e["num_particles"] = amount
    e["emission_transform"] = np.asarray(transform, np.float32).reshape(12)
    return e


def _edge_rays(x0, z0, ext, n, seed):
    """camera rays aimed across the edges of the wake window (x = x0, x0 + ext; z likewise)"""
    rng = np.random.default_rng(seed)
    r = np.zeros(n, rc.RAY)
    side = rng.integers(0, 4, n)
    along = rng.uniform(0, ext, n)
    ex = np.where(side == 0, x0, np.where(side == 1, x0 + ext, x0 + along))
    ez = np.where(side == 2, z0, np.where(side == 3, z0 + ext, z0 + along))
    o = np.stack([ex + rng.uniform(-6, 6, n), rng.uniform(0.5, 6.0, n), ez + rng.uniform(-6, 6, n)], 1)
    tgt = np.stack([ex, np.zeros(n), ez], 1)
    r["origin"] = o
    r["direction"] = (tgt - o) / np.linalg.norm(tgt - o, axis=1, keepdims=True)
    r["t_max"] = 40.0
    return r


def _check_spray(g, scales, L, foam_on, pts, em, states, frames, t0):
    """extract_spray and `frames` particle frames from t0 against the specification; returns the device states"""
    d16, n16 = g.maps_to_host(0, len(scales))
    rec, count = g.extract_spray(pts, scales, PS)
    ref = wr.spray_candidates(n16, pts, scales, PS, layer=L, foam_on=foam_on)
    assert count == len(ref) and rec.tobytes() == ref.tobytes()
    s_dev, s_ref = states, states
    for k in range(frames):
        a, b = t0 + 0.1 * k, t0 + 0.1 * (k + 1)
        s_dev, inst, cnt = g.spray_particles(em, s_dev, a, b, scales)
        s_ref, inst_ref, cnt_ref = wr.frame(s_ref, em, a, b, d16, n16, scales, layer=L, foam_on=foam_on)
        assert cnt == cnt_ref and _same_or_both_nan(inst, inst_ref) and _same_or_both_nan(s_dev.view(np.float32), s_ref.view(np.float32))
    return s_dev, count


def test_parity_with_the_specification():
    """4 x 256^2 cascades, a 256^2 coupled layer with foam on and an obstacle mask; four step calls with moving and
    body-attached sources and a scrolled window.  After each: the ray cast (host and device entry points; rays from above,
    below, grazing, across the window edge, max_iterations 0, non-finite) and spray (candidates, particle frames)."""
    import torch
    from godotoceanwaves_b200.native import check, load_library
    lib = load_library()
    gow, g, params = _gen(256, 4)
    C = 4
    scales = _scales(gow, params, C)
    d16, n16 = g.maps_to_host(0, C)
    n, dx = 256, 0.5
    p = _params(n, dx)
    _init(g, p)
    g.wake_set_foam(**FOAM)
    g.wake_set_coupling(True)
    mask = islands(n + 64, n + 64, seed=3, count=6)
    g.wake_set_obstacles(mask, (-160, -160))
    g.wake_set_readers(raycast=True, spray=True)
    L = wo.Layer(p, wf.foam_params(**FOAM))
    L.foam_on, L.foam = True, np.zeros((n, n), np.float32)
    L.set_obstacles(mask, (-160, -160))
    cp = wc.Coupling(n, dx)
    rng = np.random.default_rng(7)
    st = np.zeros(3, wk.STATE)
    st["position"][:, [0, 2]] = rng.uniform(-30, 30, (3, 2))
    st["linear_velocity"][:, [0, 2]] = rng.uniform(-5, 5, (3, 2))
    src = np.zeros(8, wk.SOURCE)
    src["x"], src["z"] = rng.uniform(-40, 40, 8), rng.uniform(-40, 40, 8)
    src["vx"], src["vz"] = rng.uniform(-6, 6, 8), rng.uniform(-6, 6, 8)
    src["radius"], src["head"], src["body"] = rng.uniform(1.0, 3.0, 8), rng.uniform(0.1, 0.4, 8), [-1, -1, -1, -1, -1, 0, 1, 2]
    src["x"][5:], src["z"][5:] = 0.0, 0.0
    em = _emitter()
    pts = sp.spray_grid(32768, 15 * np.eye(3, 4))
    states = np.zeros(32768, spp.PARTICLE)
    dev = torch.device("cuda", g.device)
    statuses = set()
    for call, (origin, S) in enumerate([((-128, -128), 2), ((-125, -130), 3), ((-125, -130), 1), ((-120, -126), 2)]):
        dt = 0.9 * float(np.sqrt(dx / wk.G)) * S
        g.wake_step(dt, S, origin, src, st)
        wo.step(L, cp, dt, S, origin, src, st)
        st["position"] = st["position"] + st["linear_velocity"] * np.float32(dt)
        x0, z0 = (float(v) for v in wk.world_origin(L.origin, dx))
        rays = np.concatenate([ray_mix(240, 80 + call, 90.0), grazing(24, 90 + call, 60.0), _edge_rays(x0, z0, n * dx, 60, call),
                               _extreme_rays(100 + call)])
        for iters in (8, 0):
            k, rec = _launches(g, lambda: g.raycast(rays, scales, 0.5, 256, 1e-3, iters))
            ref = wr.raycast(d16, n16, rays, scales, 0.5, 256, 1e-3, iters, coupling=cp)
            assert k == 3 and _records_match(rec, ref), (call, iters)
            statuses |= set(np.unique(rec["status"]).tolist())
        # the device entry point
        rays_d = torch.from_numpy(rays.view(np.uint8).copy()).to(dev)
        out_d = torch.zeros(len(rays) * 18, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        check(lib.ocean_raycast_device(g.context, len(rays), rays_d.data_ptr(), C, scales.ctypes.data, 0.5, 256, 1e-3, 0, out_d.data_ptr()))
        g.synchronize()
        assert out_d.cpu().numpy().tobytes() == rec.tobytes()
        states, count = _check_spray(g, scales, L, True, pts, em, states, 2, 0.2 * call)
    assert {rc.MISS, rc.HIT_FROM_ABOVE, rc.HIT_FROM_BELOW, rc.INVALID} <= statuses
    g.free()


def _ops(g, scales, rays, pts, em):
    states = None
    out = [g.raycast(rays, scales).tobytes(), g.extract_spray(pts, scales, PS)[0].tobytes()]
    for k in range(3):
        states, inst, cnt = g.spray_particles(em, states, 0.2 * k, 0.2 * (k + 1), scales)
        out += [states.tobytes(), inst.tobytes(), cnt]
    return out


def test_readers_off_and_unlive_change_nothing():
    """Readers 0 with coupling and foam on, and the ray cast bit while the coupling is off or unprimed, give the outputs of a
    generator without a layer, with no extra launch."""
    gow, ref_g, params = _gen(256, 4)
    _, g, _ = _gen(256, 4)
    scales = _scales(gow, params, 4)
    rays = np.concatenate([ray_mix(400, 5, 90.0), grazing(40, 6, 60.0)])
    pts = sp.spray_grid(32768, 15 * np.eye(3, 4))
    em = _emitter()
    ref = _ops(ref_g, scales, rays, pts, em)
    k_ref = _launches(ref_g, lambda: _ops(ref_g, scales, rays, pts, em))[0]
    n, dx = 256, 0.5
    _init(g, _params(n, dx))
    g.wake_set_foam(**FOAM)
    src = np.zeros(3, wk.SOURCE)
    src["x"], src["z"], src["vx"], src["radius"], src["head"], src["body"] = [0, 10, -20], [0, -15, 5], [4, -3, 5], 2.0, 0.3, -1
    g.wake_set_readers(raycast=True)                     # coupling off: the bit does nothing
    g.wake_step(0.1, 2, (-128, -128), src)
    assert _launches(g, lambda: _ops(g, scales, rays, pts, em)) == (k_ref, ref)
    g.wake_set_coupling(True)                            # on but unprimed
    assert _launches(g, lambda: _ops(g, scales, rays, pts, em)) == (k_ref, ref)
    g.wake_set_readers()                                 # readers 0, coupled, primed, foam on
    for _ in range(3):
        g.wake_step(0.1, 2, (-128, -128), src)
    assert _launches(g, lambda: _ops(g, scales, rays, pts, em)) == (k_ref, ref)
    g.wake_set_readers(raycast=True, spray=True)
    assert _ops(g, scales, rays, pts, em) != ref         # ... and the readers do read it
    ref_g.free()
    g.free()


def _flat(N=128, C=2):
    gow, g, params = _gen(N, C)
    for c in range(C):
        g.set_spectrum_amplitudes(c, np.zeros((N, N), np.complex64))
    g.update_all(1.0 / 50.0, params)
    assert not g.maps_to_host(0, C)[0].astype(np.float32).any()
    return gow, g, gow.WaveGenerator.map_scales(params)


def test_a_ray_hits_a_wake_crest_it_misses_uncoupled():
    gow, g, scales = _flat()
    n, dx = 256, 0.5
    _init(g, _params(n, dx, damping=0.0))
    c = (np.arange(n) + 0.5) * dx - 64.0
    X, Z = np.meshgrid(c, c)
    hump = (0.6 * np.exp(-(X ** 2 + Z ** 2) / 36.0)).astype(np.float32)
    g.set_wake_state(hump, hump, (-128, -128))
    g.wake_set_coupling(True)
    g.wake_step(0.05, 1, (-128, -128))
    e = g.wake_coupling()[0]
    assert e.max() > 0.4
    r = np.zeros(3, rc.RAY)
    r["origin"] = [(-40.0, 0.2, 0.3), (0.4, -40.0 + 0.0, 35.0), (-30.0, 5.0, -1.0)]
    r["direction"] = [(1.0, 0.0, 0.0), (0.0, 0.0, -1.0), (1.0, -0.2, 0.05)]
    r["origin"][1] = (0.4, 0.25, 35.0)
    r["t_max"] = 80.0
    off = g.raycast(r, scales)
    g.wake_set_readers(raycast=True)
    on = g.raycast(r, scales)
    assert off["status"][0] == rc.MISS and off["status"][1] == rc.MISS
    assert on["status"][0] == rc.HIT_FROM_ABOVE and on["status"][1] == rc.HIT_FROM_ABOVE
    assert np.all(np.abs(on["gap"]) <= 1e-3)
    cp = wc.Coupling(n, dx)
    cp.e, cp.origin_e, cp.primed = e, (-128, -128), True
    ref = wr.raycast(*g.maps_to_host(0, 2), r, scales, coupling=cp)
    assert _records_match(on, ref)
    # the crest is where the surface query says it is
    q = g.query_surface(on["position"][:, [0, 2]].copy(), scales)
    assert np.all(np.abs(q["displacement"][:, 1] - on["displacement"][:, 1]) == 0)
    g.free()


def test_a_moving_source_throws_spray_on_its_trail():
    """Stir foam on the trail of a moving source: active candidates and live particles with the spray bit, none without;
    the live particles' heights carry h at their start positions."""
    gow, g, scales = _flat()
    n, dx = 256, 0.5
    p = _params(n, dx)
    _init(g, p)
    g.wake_set_foam(whitecap=0.05, grow_rate=1.0, stir_rate=1.0, decay_rate=0.2)
    src = np.zeros(1, wk.SOURCE)
    src["x"], src["z"], src["vx"], src["radius"], src["head"], src["body"] = -40.0, 0.0, 6.0, 2.0, 0.3, -1
    L = wk.Layer(p)
    for k in range(12):
        s = src.copy()
        s["x"] = -40.0 + 6.0 * 0.1 * k
        g.wake_step(0.1, 2, (-128, -128), s)
    h, _, origin = g.wake_state()
    L.h, L.origin, L.foam = h, origin, g.wake_foam()
    assert L.foam.max() > 0.95
    E = np.array([[4, 0, 0, -36], [0, 1, 0, 0], [0, 0, 4, 0]], np.float32)     # a 40 m square around the trail
    pts = sp.spray_grid(32768, E)
    em = _emitter(transform=E)

    def on_trail(x, z):                             # the maps keep some cascade foam of their earlier updates elsewhere
        return (np.abs(z) < 6.0) & (x > -45.0) & (x < -28.0)

    rec, _ = g.extract_spray(pts, scales, PS)
    assert not on_trail(rec["start_x"], rec["start_z"]).any()
    states = None
    for k in range(10):
        states, _, _ = g.spray_particles(em, states, 0.3 * k, 0.3 * (k + 1), scales)
        on = ((states["flags"] & spp.ACTIVE) != 0) & (states["userdata3"][:, 3] != 0)
        assert not on_trail(states["userdata1"][on, 0], states["userdata1"][on, 2]).any()
    g.wake_set_readers(spray=True)
    rec, _ = g.extract_spray(pts, scales, PS)
    assert on_trail(rec["start_x"], rec["start_z"]).sum() > 100
    d16, n16 = g.maps_to_host(0, 2)

    class NoHeight(wr.SprayLayer):
        def spray(self, x, z):
            hw, gx, gz, fw = super().spray(x, z)
            return np.zeros_like(hw), gx, gz, fw

    states, s_ref, total = None, None, 0
    for k in range(10):
        states, inst, live = g.spray_particles(em, states, 0.3 * k, 0.3 * (k + 1), scales)
        s_ref, _, _ = wr.frame(s_ref if s_ref is not None else np.zeros(em["amount"], spp.PARTICLE), em, 0.3 * k, 0.3 * (k + 1),
                               d16, n16, scales, wake=NoHeight(L, True))
        on = ((states["flags"] & spp.ACTIVE) != 0) & (states["userdata3"][:, 3] != 0)
        total += int(on_trail(states["userdata1"][on, 0], states["userdata1"][on, 2]).sum())
        if on.any():
            hw = L.sample(np.stack([states["userdata1"][on, 0], states["userdata1"][on, 2]], 1))[:, 0]
            dy = states["transform"][on, 7].astype(np.float64) - s_ref["transform"][on, 7]
            assert np.all(np.abs(dy - hw) <= 1e-5 + 1e-6 * np.abs(hw))
    assert total > 0
    g.free()


def test_readers_arguments_and_lifetime():
    from godotoceanwaves_b200.native import load_library
    lib = load_library()
    gow, g, params = _gen(128, 2)
    scales = _scales(gow, params, 2)
    assert lib.ocean_wake_set_readers(g.context, 1) == STATE                  # no layer
    n = 256
    _init(g, _params(n, 0.5))
    g.wake_set_coupling(True)
    src = np.zeros(1, wk.SOURCE)
    src["x"], src["z"], src["vx"], src["radius"], src["head"], src["body"] = 5.0, 5.0, 3.0, 3.0, 0.4, -1
    g.wake_step(0.1, 2, (-128, -128), src)
    rays = np.concatenate([ray_mix(300, 12, 60.0), grazing(30, 13, 40.0)])
    base = _cast(g, rays, scales)
    before = g.info()
    for bad in (4, 8, 5, 7, 1 << 31, 0xFFFFFFFF):
        assert lib.ocean_wake_set_readers(g.context, bad) == INVALID
    assert g.info().kernel_launches == before.kernel_launches and g.info().device_bytes == before.device_bytes
    assert _cast(g, rays, scales) == base                                       # nothing changed
    g.wake_set_readers(raycast=True)
    k, on = _cast(g, rays, scales)
    assert k == 3 and on != base[1]
    g.wake_set_coupling(False)                                                  # off: the bit stays, reads nothing
    assert _cast(g, rays, scales) == base
    g.wake_set_coupling(True)
    g.wake_step(0.1, 2, (-128, -128), src)
    assert _cast(g, rays, scales)[0] == 3               # set_coupling left the readers set
    _init(g, _params(n, 0.5))                                                   # ocean_wake_init clears them
    g.wake_set_coupling(True)
    g.wake_step(0.1, 2, (-128, -128), src)
    assert _cast(g, rays, scales)[0] == 2
    g.wake_set_readers(raycast=True)
    _init(g, _params(0, 0.5))                                                   # release, then re-create: still clear
    _init(g, _params(n, 0.5))
    g.wake_set_coupling(True)
    g.wake_step(0.1, 2, (-128, -128), src)
    assert _cast(g, rays, scales)[0] == 2
    g.free()


def test_largest_layer_with_a_million_rays():
    """A 2048^2 coupled layer and 2^20 rays complete; a seeded subset matches the specification on the device's e."""
    gow, g, params = _gen(256, 4)
    C = 4
    scales = _scales(gow, params, C)
    n, dx = 2048, 0.25
    _init(g, _params(n, dx, sponge_cells=64))
    g.wake_set_coupling(True)
    g.wake_set_readers(raycast=True, spray=True)
    rng = np.random.default_rng(11)
    src = np.zeros(64, wk.SOURCE)
    src["x"], src["z"] = rng.uniform(-200, 200, 64), rng.uniform(-200, 200, 64)
    src["vx"], src["vz"] = rng.uniform(-6, 6, 64), rng.uniform(-6, 6, 64)
    src["radius"], src["head"], src["body"] = rng.uniform(1, 4, 64), rng.uniform(0.1, 0.5, 64), -1
    h_max = float(np.sqrt(dx / wk.G))
    for _ in range(3):
        g.wake_step(0.9 * h_max * 4, 4, (-1024, -1024), src)
    e, _, origins, _ = g.wake_coupling()
    cp = wc.Coupling(n, dx)
    cp.e, cp.origin_e, cp.primed = e, origins[0], True
    rays = np.concatenate([ray_mix((1 << 20) - 4096, 21, 300.0), grazing(4096, 22, 250.0)])
    rec = g.raycast(rays, scales, 0.5, 1024, 1e-3, 8)
    assert len(rec) == 1 << 20 and (rec["status"] == rc.HIT_FROM_ABOVE).sum() > 1 << 16
    pick = np.sort(rng.choice(len(rays), 2500, replace=False))
    d16, n16 = g.maps_to_host(0, C)
    ref = wr.raycast(d16, n16, rays[pick], scales, 0.5, 1024, 1e-3, 8, coupling=cp)
    # the slab is the whole e's: the subset's records are those of the full call
    assert _records_match(rec[pick], ref)
    g.free()
