"""GPU sea state (ocean_get_sea_state; ocean_drift.cu) against oracle/sea_state.py: the cached moments bit for bit from the
spectrum as stored, the scaled total and derived fields, the staleness of the cache and the call's validation."""
import numpy as np
import pytest

from conftest import demo_params
from oracle import pyoracle as po
from oracle import sea_state as ss

pytestmark = pytest.mark.gpu

INVALID = 1   # OCEAN_ERR_INVALID_ARGUMENT
MOMENT_FIELDS = ("m_minus1", "m0", "m1", "m2", "direction", "slope", "stokes")


@pytest.fixture(autouse=True)
def _modes():
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    yield
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)


def _gow():
    import godotoceanwaves_b200 as gow
    return gow


def _generator(N, params):
    g = _gow().WaveGenerator()
    g.map_size = N
    g.init_gpu(len(params))
    g.update_all(0.02, params)
    return g


def _moments(rec):
    return np.concatenate([np.atleast_1d(rec[f]).astype(np.float64) for f in MOMENT_FIELDS])


def _expected(g, params, C):
    return [ss.cascade_moments(g.spectrum_to_host(c), params[c].tile_length) for c in range(C)]


def _check(g, params, C, what=""):
    sc = g.map_scales(params[:C])
    total, per = g.sea_state(sc)
    want = _expected(g, params, C)
    for c in range(C):
        assert np.array_equal(_moments(per[c]).view(np.uint64), want[c].view(np.uint64)), f"{what}: moments of cascade {c}"
        exp = ss.record(want[c])
        for f in ss.SEA_STATE.names:
            np.testing.assert_allclose(per[c][f], exp[f], rtol=1e-14, atol=0, err_msg=f"{what}: {f} of cascade {c}")
    tm = ss.total_moments(want, sc)
    assert np.array_equal(_moments(total).view(np.uint64), tm.view(np.uint64)), f"{what}: total moments"
    exp = ss.record(tm)
    for f in ss.SEA_STATE.names:
        np.testing.assert_allclose(total[f], exp[f], rtol=1e-14, atol=0, err_msg=f"{what}: total {f}")
    return total, per


@pytest.mark.parametrize("N,C", [(128, 1), (128, 8), (256, 4), (512, 3), (1024, 8)])
def test_sea_state_bit_exact_demo(N, C):
    """The reference's demo parameters cycled over C cascades: every cascade's moments bit for bit, the derived fields and
    the displacement-scaled total."""
    gow = _gow()
    params = [demo_params(gow.WaveCascadeParameters, c) for c in range(C)]
    g = _generator(N, params)
    total, _ = _check(g, params, C, what=f"{N}x{C}")
    assert total["significant_wave_height"] > 0 and np.isfinite(total["stokes_speed"])


@pytest.mark.parametrize("N", [128, 256, 1024])
def test_sea_state_injected_spectra(N):
    """Injected amplitudes (random sparse, a single wave, signed zeros, huge values) through ocean_set_spectrum_amplitudes."""
    gow = _gow()
    params = [demo_params(gow.WaveCascadeParameters, c, tile_length=(37.0 + 11 * c, 53.0)) for c in range(3)]
    g = _generator(N, params)
    rng = np.random.default_rng(N)
    amps = []
    a = np.zeros((N, N, 2), np.float32)
    mask = rng.random((N, N)) < 0.05
    a[mask] = rng.normal(size=(int(mask.sum()), 2)).astype(np.float32)
    amps.append(a)
    b = np.zeros((N, N, 2), np.float32)
    b[N // 2 + 3, N // 2 - 5] = (0.75, -0.25)
    b[N // 2, N // 2] = (9.0, 9.0)          # the DC texel contributes nothing
    b[7, 9] = (-0.0, 0.0)
    amps.append(b)
    c = (rng.normal(size=(N, N, 2)) * 1e15).astype(np.float32)
    amps.append(c)
    for i, a in enumerate(amps):
        g.set_spectrum_amplitudes(i, (a[..., 0] + 1j * a[..., 1]).astype(np.complex64))
    _check(g, params, 3, what="injected")


def _launches(g):
    return g.info().kernel_launches


def test_sea_state_recomputes_only_after_spectrum_writes():
    """0 launches while no spectrum or table changed; 2 (one launch sequence) after a regeneration, an injection or a new
    tile; a generator whose cascades were never updated has zero moments."""
    gow = _gow()
    g = gow.WaveGenerator()
    g.map_size = 128
    g.init_gpu(3)
    params = [demo_params(gow.WaveCascadeParameters, c) for c in range(3)]
    start = _launches(g)
    total, per = g.sea_state(g.map_scales(params))
    assert _launches(g) == start and total["m0"] == 0 and total["significant_wave_height"] == 0 and np.all(per["m0"] == 0)
    g.update_all(0.02, params)
    n0 = _launches(g)
    _check(g, params, 3, "first")
    assert _launches(g) - n0 == 2
    for _ in range(3):                                  # map updates without spectrum writes: nothing to recompute
        g.update_all(0.02, params)
    n1 = _launches(g)
    _check(g, params, 3, "steady")
    assert _launches(g) == n1
    params[1].wind_speed = 7.0
    params[1].should_generate_spectrum = True
    g.update_all(0.02, params)
    n2 = _launches(g)
    _check(g, params, 3, "regenerated")
    assert _launches(g) - n2 == 2
    g.set_spectrum_amplitudes(2, np.full((128, 128), 0.01, np.complex64))
    n3 = _launches(g)
    _check(g, params, 3, "injected")
    assert _launches(g) - n3 == 2
    params[0].tile_length = (77.0, 31.0)                # a new dispersion table, same spectrum
    g.update_all(0.02, params)
    n4 = _launches(g)
    _check(g, params, 3, "new tile")
    assert _launches(g) - n4 == 2
    assert _launches(g) == n4 + 2
    g.sea_state(g.map_scales(params))
    assert _launches(g) == n4 + 2


def test_sea_state_memory_is_counted_on_first_use():
    gow = _gow()
    params = [demo_params(gow.WaveCascadeParameters, c) for c in range(2)]
    g = _generator(256, params)
    before = g.info().device_bytes
    g.sea_state(g.map_scales(params))
    assert g.info().device_bytes > before


def test_sea_state_validation():
    gow = _gow()
    params = [demo_params(gow.WaveCascadeParameters, c) for c in range(2)]
    g = _generator(128, params)
    lib = gow.native.load_library()
    sc = g.map_scales(params)
    total = np.zeros((), ss.SEA_STATE)
    n0 = _launches(g)
    assert lib.ocean_get_sea_state(g.context, 0, sc.ctypes.data, None, total.ctypes.data) == INVALID
    assert lib.ocean_get_sea_state(g.context, 3, sc.ctypes.data, None, total.ctypes.data) == INVALID
    assert lib.ocean_get_sea_state(g.context, 2, None, None, total.ctypes.data) == INVALID
    assert lib.ocean_get_sea_state(g.context, 2, sc.ctypes.data, None, None) == INVALID
    assert _launches(g) == n0
    assert lib.ocean_get_sea_state(g.context, 2, sc.ctypes.data, None, total.ctypes.data) == 0
