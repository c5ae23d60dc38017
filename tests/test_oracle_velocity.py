"""The velocity-map specification (oracle_velocity_update, oracle/velocity_oracle.c): the time derivative of the displacement map,
checked against the independent float64 numpy model and against identities of the analytic derivative.  CPU only."""
import math

import numpy as np
import pytest

from conftest import demo_params
from oracle import pyoracle as po
from oracle import velocity as ov


@pytest.fixture(autouse=True)
def _modes():
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    yield
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)


def _oracle_after_update(N, params, delta=1.0 / 50.0):
    g = ov.OracleWaveGenerator(N)
    g.update_all(delta, params)
    return g


def _model_velocity(g, c, p):
    sp = g.spectrum[c].astype(np.float64)
    pcm = g.velocity_source[c]
    return ov.float64_velocity(sp[..., 0] + 1j * sp[..., 1], sp[..., 2] + 1j * sp[..., 3], g.map_size,
                       (pcm.tile_length[0], pcm.tile_length[1]), po.DEPTH, pcm.time)


def _close_per_field(f32, model, tol):
    for ch in range(3):
        m = np.max(np.abs(model[ch]))
        assert m > 0
        err = np.max(np.abs(f32[..., ch].astype(np.float64) - model[ch]))
        assert err <= tol * m, (ch, err / m)


@pytest.mark.parametrize("c", [0, 1, 2, 3])
def test_matches_float64_derivative_cfg2(c):
    """cfg2 (256^2, demo cascades 0-3): every field within 5e-6 of its maximum of the float64 derivative."""
    N = 256
    params = [demo_params(po.CascadeParams, i) for i in range(4)]
    g = _oracle_after_update(N, params)
    vel, f32 = g.velocity(c)
    _close_per_field(f32, _model_velocity(g, c, params[c]), 5e-6)
    assert np.array_equal(vel, f32.astype(np.float16).view(np.uint16))     # half = RTNE of the binary32 values
    assert np.all(f32[..., 3] == 0)


def test_matches_float64_derivative_1024_short_tile():
    """1024^2 at L = 16 m, t = 120 s: the steepest, fastest waves of the demo."""
    N = 1024
    p = demo_params(po.CascadeParams, 2, tile_length=(16.0, 16.0), time=120.0 - 1.0 / 50.0)
    g = _oracle_after_update(N, [p])
    assert g.velocity_source[0].time == np.float32(120.0)
    _, f32 = g.velocity(0)
    _close_per_field(f32, _model_velocity(g, 0, p), 5e-6)


def test_strict_and_fma_modes_agree():
    N = 256
    params = [demo_params(po.CascadeParams, i) for i in range(2)]
    g = _oracle_after_update(N, params)
    _, fma = g.velocity(1)
    po.set_modes(po.MATH_DET, po.CONTRACT_STRICT)
    _, strict = g.velocity(1)
    assert not np.array_equal(fma, strict)          # the velocity library follows the main oracle's contraction mode
    for ch in range(3):
        assert np.max(np.abs(fma[..., ch] - strict[..., ch])) <= 1e-6 * np.max(np.abs(fma[..., ch]))


def test_zero_spectrum_gives_exact_zeros():
    N = 128
    g = _oracle_after_update(N, [demo_params(po.CascadeParams, 0)])
    g.set_spectrum(0, np.zeros((N, N, 4), np.float32))
    vel, f32 = g.velocity(0)
    assert np.all(f32 == 0) and np.all((vel & 0x7FFF) == 0)


def test_never_updated_cascade_is_zero():
    g = ov.OracleWaveGenerator(128)
    g.init_gpu(2)
    vel, f32 = g.velocity(1)
    assert not vel.any() and not f32.any()


def _single_wave_texture(N, x, y, a):
    """The texture the library stores for one amplitude A(x, y) = a: texel (x, y) = (a, 0) and its mirror texel
    (N - x, N - y) = (0, conj a), so h0b = 0 where h0a != 0 and the other way round."""
    amp = np.zeros((N, N), np.complex64)
    amp[y, x] = a
    return po.spectrum_texture(amp)


@pytest.mark.parametrize("x,y,tile", [(131, 120, 50.0), (129, 140, 16.0), (3, 250, 88.0)])
def test_single_wave_quarter_period_identity(x, y, tile):
    """One wave: h(k) = a e^{i w t} and h(-k) = conj(a) e^{-i w t}, each texel with one of h0a, h0b zero.  Then
    dh/dt = w h(t + pi / (2 w)) at both texels, so v(t) = w D(t + pi / (2 w)) -- in binary32, within 1e-5 of the field's
    maximum over the three fields.  (The displacement's hz channel shares its packed layer with dhy_dx, whose binary32
    transform leaves rounding noise of |dhy_dx| in it; per field the bound would be that noise over |hz|.  With the mirror
    texel left out the packed layer 1 would carry the imaginary part of the dhy_dx transform into
    the hz channel of D, which the velocity layer does not pack.)"""
    N = 256
    a = np.complex64(0.3 - 0.7j)
    p = po.CascadeParams(tile_length=(tile, tile), time=0.75)
    g = ov.OracleWaveGenerator(N)
    g.update(0.0, [p])
    g.set_spectrum(0, _single_wave_texture(N, x, y, a))
    p.should_generate_spectrum = False
    g.process()
    _, v = g.velocity(0)
    kvx = (np.float32(x) - np.float32(N / 2)) * np.float32(2.0) * np.float32(math.pi) / np.float32(tile)
    kvy = (np.float32(y) - np.float32(N / 2)) * np.float32(2.0) * np.float32(math.pi) / np.float32(tile)
    k = float(np.sqrt(kvx * kvx + kvy * kvy) + np.float32(1e-6))
    w = math.sqrt(po.G * k * math.tanh(k * po.DEPTH))
    q = po.CascadeParams(tile_length=(tile, tile), time=0.75 + math.pi / (2.0 * w), should_generate_spectrum=False)
    h = ov.OracleWaveGenerator(N)
    h.update(0.0, [q])
    h.set_spectrum(0, _single_wave_texture(N, x, y, a))
    h.process()
    d = h.displacement_f32[0].astype(np.float64)
    m = np.max(np.abs(v[..., :3]))
    for ch in range(3):
        assert np.max(np.abs(v[..., ch])) > 0
        assert np.max(np.abs(v[..., ch] - w * d[..., ch])) <= 1e-5 * m, ch
