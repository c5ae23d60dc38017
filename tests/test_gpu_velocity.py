"""GPU velocity maps (ocean_update_velocity and friends; ocean_velocity.cu) against the oracle's specification
(oracle_velocity_update, oracle/velocity_oracle.c): the half maps and the binary32 tap bit for bit, signed zeros included, through every path that
writes the maps; staleness tracking, sampling, properties of the derivative, isolation from the update path, arguments."""
import ctypes as C
import math

import numpy as np
import pytest

from conftest import demo_params
from oracle import pyoracle as po
from oracle import sampling as sp
from oracle import velocity as ov
from test_gpu_parity import _bits_equal, _pair
from test_gpu_sampling import _extreme_points, _points, _same_or_both_nan

pytestmark = pytest.mark.gpu

INVALID = 1   # OCEAN_ERR_INVALID_ARGUMENT


def _gow():
    import godotoceanwaves_b200 as gow
    return gow


@pytest.fixture(autouse=True)
def _modes():
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    yield
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)


def _generator(N, C, taps=True):
    g = _gow().WaveGenerator()
    g.map_size = N
    g.init_gpu(C)
    if taps:
        g.enable_f32_taps(True)
    return g


def _oracle(N):
    o = ov.OracleWaveGenerator(N)
    o.keep_f32 = False
    return o


def _check_velocity(g, o, C, taps=True, what=""):
    v = g.velocity_to_host(0, C)
    for c in range(C):
        ov, of = o.velocity(c)
        assert _bits_equal(v[c].view(np.uint16), ov), f"{what}: velocity map of cascade {c}"
        if taps:
            assert _bits_equal(g.velocity_f32_to_host(c), of), f"{what}: binary32 velocity of cascade {c}"


@pytest.mark.parametrize("tiles", ["distinct", "shared"])
@pytest.mark.parametrize("N", [128, 256, 512, 1024])
def test_velocity_bit_exact(N, tiles):
    """update_all, then update + one _process (the cascades' maps at different times), then a parameter edit (new spectrum,
    new dispersion-table slot): after each, every cascade's velocity equals the oracle's."""
    gow = _gow()
    C = 2 if N == 1024 else 3
    over = {} if tiles == "distinct" else dict(tile_length=(57.0, 57.0))
    pg, pc = _pair(gow.WaveCascadeParameters, C, **over)
    g, o = _generator(N, C), _oracle(N)
    g.update_all(0.02, pg)
    o.update_all(0.02, pc)
    assert g.update_velocity() == C
    _check_velocity(g, o, C, what="update_all")
    g.update(0.031, pg)
    o.update(0.031, pc)
    g._process()
    o.process()
    _check_velocity(g, o, C, what="partial _process")
    for p in (pg[0], pc[0]):
        p.tile_length = (61.0, 47.0)
        p.wind_speed = 7.5
        p.should_generate_spectrum = True
    g.update_all(0.02, pg)
    o.update_all(0.02, pc)
    _check_velocity(g, o, C, what="parameter edit")
    g.free()


def test_velocity_after_fused_frames():
    """ocean_update_frames: the velocity describes the last frame of the fused launch (half maps, no taps: the production
    persistent kernel)."""
    gow = _gow()
    N, C = 256, 3
    pg, pc = _pair(gow.WaveCascadeParameters, C)
    g, o = _generator(N, C, taps=False), _oracle(N)
    g.update_frames(0.02, pg, 5)
    for _ in range(5):
        o.update_all(0.02, pc)
    assert g.update_velocity() == C
    _check_velocity(g, o, C, taps=False, what="fused frames")
    g.free()


@pytest.mark.parametrize("taps", [False, True], ids=["untapped", "taps"])
def test_velocity_two_kernel_pipeline(taps):
    gow = _gow()
    N, C = 512, 4
    pg, pc = _pair(gow.WaveCascadeParameters, C)
    g, o = _generator(N, C, taps=taps), _oracle(N)
    g.set_profiling(True)
    for delta in (0.02, 0.025):
        g.update_all(delta, pg)
        o.update_all(delta, pc)
    _check_velocity(g, o, C, taps=taps, what="split pipeline")
    g.free()


def _water(N, C, rate):
    gow = _gow()
    w = gow.Water(map_size=N, updates_per_second=rate)
    w.parameters = [demo_params(gow.WaveCascadeParameters, c) for c in range(C)]
    return w


def test_staleness_follows_the_frame_scheduler():
    """Water frames at 60 Hz with updates at 10 Hz: one cascade is processed per frame and the pass drains before the next
    update.  A velocity call per frame recomputes exactly the cascades processed since the previous call; the end result
    equals that of a generator that computed its velocity once, at the end; a second call recomputes nothing and changes
    no byte."""
    N, C = 256, 3
    a, b = _water(N, C, 10.0), _water(N, C, 10.0)
    recomputed = []
    for _ in range(20):
        before = a.wave_generator.info().cascade_updates
        a.process(1.0 / 60.0)
        b.process(1.0 / 60.0)
        processed = a.wave_generator.info().cascade_updates - before
        n = a.wave_generator.update_velocity()
        assert n == processed
        recomputed.append(n)
    assert sum(recomputed) >= 2 * C and max(recomputed) == 1
    va = a.wave_generator.velocity_to_host(0, C)
    assert b.wave_generator.update_velocity() == C
    vb = b.wave_generator.velocity_to_host(0, C)
    assert _bits_equal(va, vb)
    assert a.wave_generator.update_velocity() == 0
    assert _bits_equal(a.wave_generator.velocity_to_host(0, C), va)
    a.free(); b.free()


def test_sampling_bit_exact_and_refreshing():
    """ocean_sample_velocity == oracle/sampling.py's displacement sum on the velocity maps, at the sampling tests' points,
    with extreme and non-finite coordinates; the device entry point equals the host one; sampling brings stale layers up
    to date by itself."""
    import torch
    from godotoceanwaves_b200.native import check, load_library
    gow = _gow()
    N, C = 256, 4
    pa, _ = _pair(gow.WaveCascadeParameters, C)
    pb, _ = _pair(gow.WaveCascadeParameters, C)
    a, b = _generator(N, C, taps=False), _generator(N, C, taps=False)
    for _ in range(2):
        a.update_all(0.02, pa)
        b.update_all(0.02, pb)
    scales = gow.WaveGenerator.map_scales(pa)
    scales[:, 2] = [1.0, -0.75, 0.0, 0.5]
    pts = _points(20000, 71, 300.0)
    v = a.sample_velocity(pts, scales)                          # no explicit update: the layers are refreshed first
    assert b.update_velocity() == C
    assert v.tobytes() == b.sample_velocity(pts, scales).tobytes()
    maps = a.velocity_to_host(0, C)
    ref, _ = sp.sample_maps(maps, maps, pts, scales)
    assert np.array_equal(v.view(np.uint32), ref.view(np.uint32))
    v1 = a.sample_velocity(pts[:1000], scales[:1])
    ref1, _ = sp.sample_maps(maps[:1], maps[:1], pts[:1000], scales[:1])
    assert np.array_equal(v1.view(np.uint32), ref1.view(np.uint32))
    ext, mask = _extreme_points(4000, 43)
    ve = a.sample_velocity(ext, scales)
    with np.errstate(all="ignore"):
        ref_e, _ = sp.sample_maps(maps, maps, ext, scales)
    assert _same_or_both_nan(ve, ref_e)
    assert np.isnan(ve[~np.isfinite(ext).all(1)]).all()
    dev = torch.device("cuda", a.device)
    pts_d = torch.from_numpy(pts).to(dev)
    out_d = torch.zeros(pts.shape[0] * 3, dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    check(load_library().ocean_sample_velocity_device(a.context, pts.shape[0], pts_d.data_ptr(), C, scales.ctypes.data, out_d.data_ptr()))
    a.synchronize()
    assert out_d.cpu().numpy().tobytes() == v.tobytes()
    a.free(); b.free()


def test_zero_spectrum_and_power_of_two_scaling():
    """A zero spectrum gives an all-zero map; doubling every amplitude doubles every binary32 velocity exactly."""
    gow = _gow()
    N = 256
    p0 = demo_params(gow.WaveCascadeParameters, 0)
    g = _generator(N, 3)
    g.update_all(0.02, [p0])
    tex = g.spectrum_to_host(0)
    amp = (tex[..., 0] + 1j * tex[..., 1]).astype(np.complex64)
    params = [demo_params(gow.WaveCascadeParameters, 0) for _ in range(3)]
    for p in params:
        p.should_generate_spectrum = False
    g.set_spectrum_amplitudes(0, np.zeros_like(amp))
    g.set_spectrum_amplitudes(1, amp)
    g.set_spectrum_amplitudes(2, amp * np.float32(2.0))
    g.update_all(0.02, params)
    v = g.velocity_to_host(0, 3)
    assert not (v[0].view(np.uint16) & 0x7FFF).any()
    assert np.all(g.velocity_f32_to_host(0) == 0)
    v1, v2 = g.velocity_f32_to_host(1), g.velocity_f32_to_host(2)
    assert np.isfinite(v1).all() and np.abs(v1).max() > 0
    assert np.array_equal(v2, v1 * np.float32(2.0))
    g.free()


@pytest.mark.parametrize("x,y,tile", [(131, 120, 50.0), (3, 250, 88.0)])
def test_single_wave_quarter_period_identity(x, y, tile):
    """One wave: v(t) = w D(t + pi / (2 w)) on the binary32 taps, within 1e-5 of the map's maximum (tests/test_oracle_velocity.py
    states why the bound is over the three fields)."""
    gow = _gow()
    N = 256
    amp = np.zeros((N, N), np.complex64)
    amp[y, x] = np.complex64(0.3 - 0.7j)
    kvx = (np.float32(x) - np.float32(N / 2)) * np.float32(2.0) * np.float32(math.pi) / np.float32(tile)
    kvy = (np.float32(y) - np.float32(N / 2)) * np.float32(2.0) * np.float32(math.pi) / np.float32(tile)
    k = float(np.sqrt(kvx * kvx + kvy * kvy) + np.float32(1e-6))
    w = math.sqrt(po.G * k * math.tanh(k * po.DEPTH))

    def run(time):
        g = _generator(N, 2)
        params = [gow.WaveCascadeParameters(tile_length=(tile, tile)) for _ in range(2)]
        for p in params:
            p.time = time
            p.should_generate_spectrum = False
        g.set_spectrum_amplitudes(0, amp)
        g.update_all(0.0, params)
        v, d = g.velocity_f32_to_host(0), g.f32_maps_to_host(0)[0]
        g.free()
        return v, d

    v, _ = run(0.75)
    _, d = run(0.75 + math.pi / (2.0 * w))
    m = np.max(np.abs(v[..., :3]))
    for ch in range(3):
        assert np.max(np.abs(v[..., ch])) > 0
        assert np.max(np.abs(v[..., ch] - w * d[..., ch].astype(np.float64))) <= 1e-5 * m, ch


def test_isolation_from_the_update_path():
    """Maps, foam, spectrum and the next update's maps are byte-identical with and without velocity calls; a cascade that was
    never updated has a zero velocity layer."""
    gow = _gow()
    N, C = 256, 3
    pa, _ = _pair(gow.WaveCascadeParameters, C)
    pb, _ = _pair(gow.WaveCascadeParameters, C)
    a, b = _generator(N, C, taps=False), _generator(N, C, taps=False)
    a.update(0.02, pa)
    b.update(0.02, pb)
    a._process()                                               # only cascade C-1 has maps now
    b._process()
    v = a.velocity_to_host(0, C)
    assert not v[:C - 1].view(np.uint16).any() and v[C - 1].view(np.uint16).any()
    for _ in range(3):
        a.update_all(0.02, pa)
        b.update_all(0.02, pb)
        a.update_velocity()
        a.sample_velocity(_points(1000, 5, 100.0), gow.WaveGenerator.map_scales(pa))
        da, na = a.maps_to_host(0, C)
        db, nb = b.maps_to_host(0, C)
        assert _bits_equal(da, db) and _bits_equal(na, nb)
        for c in range(C):
            assert _bits_equal(a.get_foam_state(c), b.get_foam_state(c))
            assert _bits_equal(a.spectrum_to_host(c), b.spectrum_to_host(c))
    a.free(); b.free()


def test_log0_hazard_seed():
    """The spectrum seed that reaches the reference's log(0): the velocity is non-finite exactly where the oracle's is, and the
    neighbouring cascade's layer is the oracle's bit for bit."""
    gow = _gow()
    N = 128
    idx, idy = N // 2 + 3, N // 2 + 5
    over = dict(spectrum_seed=po.hash_seed_for(idx, idy, 0))
    pg = [demo_params(gow.WaveCascadeParameters, 0, **over), demo_params(gow.WaveCascadeParameters, 1)]
    pc = [demo_params(po.CascadeParams, 0, **over), demo_params(po.CascadeParams, 1)]
    g, o = _generator(N, 2), _oracle(N)
    for delta in (0.02, 0.02):
        g.update_all(delta, pg)
        o.update_all(delta, pc)
    v = g.velocity_to_host(0, 2)
    ov0, of0 = o.velocity(0)
    assert not np.isfinite(of0[..., :3]).all()
    assert np.array_equal(np.isfinite(v[0]), np.isfinite(ov0.view(np.float16)))
    assert np.array_equal(np.isfinite(g.velocity_f32_to_host(0)), np.isfinite(of0))
    ov1, of1 = o.velocity(1)
    assert _bits_equal(v[1].view(np.uint16), ov1) and _bits_equal(g.velocity_f32_to_host(1), of1)
    g.free()


def test_arguments():
    gow = _gow()
    from godotoceanwaves_b200.native import load_library
    lib = load_library()
    g = _generator(128, 2, taps=False)
    params = [demo_params(gow.WaveCascadeParameters, c) for c in range(2)]
    g.update_all(0.02, params)
    scales = gow.WaveGenerator.map_scales(params)
    pts = np.zeros((4, 2), np.float32)
    out = np.zeros((4, 3), np.float32)
    host = np.zeros((128, 128, 4), np.float32)
    h = g.context
    launches = g.info().kernel_launches
    cases = [
        lambda: lib.ocean_update_velocity(None, None),
        lambda: lib.ocean_get_velocity_map(None, None, None),
        lambda: lib.ocean_copy_velocity_to_host(h, -1, 1, host.ctypes.data),
        lambda: lib.ocean_copy_velocity_to_host(h, 1, 2, host.ctypes.data),
        lambda: lib.ocean_copy_velocity_to_host(h, 0, 1, None),
        lambda: lib.ocean_copy_f32_velocity_to_host(h, 2, host.ctypes.data),
        lambda: lib.ocean_copy_f32_velocity_to_host(h, -1, host.ctypes.data),
        lambda: lib.ocean_copy_f32_velocity_to_host(h, 0, None),
        lambda: lib.ocean_sample_velocity(h, -1, pts.ctypes.data, 2, scales.ctypes.data, out.ctypes.data),
        lambda: lib.ocean_sample_velocity(h, 4, None, 2, scales.ctypes.data, out.ctypes.data),
        lambda: lib.ocean_sample_velocity(h, 4, pts.ctypes.data, 2, scales.ctypes.data, None),
        lambda: lib.ocean_sample_velocity(h, 4, pts.ctypes.data, 0, scales.ctypes.data, out.ctypes.data),
        lambda: lib.ocean_sample_velocity(h, 4, pts.ctypes.data, 3, scales.ctypes.data, out.ctypes.data),
        lambda: lib.ocean_sample_velocity(h, 4, pts.ctypes.data, 2, None, out.ctypes.data),
        lambda: lib.ocean_sample_velocity_device(h, -1, pts.ctypes.data, 2, scales.ctypes.data, out.ctypes.data),
        lambda: lib.ocean_sample_velocity_device(h, 4, None, 2, scales.ctypes.data, out.ctypes.data),
        lambda: lib.ocean_sample_velocity_device(h, 4, pts.ctypes.data, 2, scales.ctypes.data, None),
        lambda: lib.ocean_sample_velocity_device(h, 4, pts.ctypes.data, 0, scales.ctypes.data, out.ctypes.data),
        lambda: lib.ocean_sample_velocity_device(h, 4, pts.ctypes.data, 3, scales.ctypes.data, out.ctypes.data),
        lambda: lib.ocean_sample_velocity_device(h, 4, pts.ctypes.data, 2, None, out.ctypes.data),
    ]
    for k, call in enumerate(cases):
        assert call() == INVALID, k
    assert g.info().kernel_launches == launches                 # nothing was launched
    # the binary32 tap needs the taps; empty requests succeed
    assert lib.ocean_copy_f32_velocity_to_host(h, 0, host.ctypes.data) == 4   # OCEAN_ERR_STATE
    assert lib.ocean_sample_velocity(h, 0, None, 2, scales.ctypes.data, None) == 0
    assert lib.ocean_copy_velocity_to_host(h, 0, 0, None) == 0
    ptr, size = C.c_void_p(), C.c_size_t()
    assert lib.ocean_get_velocity_map(h, C.byref(ptr), C.byref(size)) == 0 and ptr.value and size.value == 128 * 128 * 8
    g.free()
