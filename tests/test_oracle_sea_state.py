"""oracle/sea_state.py against the float64 model of the maps (oracle/numpy_model.py): the variance and amplitude of a single
wave, its direction of travel and Stokes drift, Parseval on sparse spectra, the fixed summation order and the derived
fields."""
import math

import numpy as np
import pytest

from oracle import numpy_model as nm
from oracle import pyoracle as po
from oracle import sea_state as ss

N = 128
TILE = (50.0, 50.0)


@pytest.fixture(autouse=True)
def _modes():
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    yield
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)


def _height(texture, time):
    """The float64 height map [row z][column x] of a spectrum texture at `time`."""
    h0 = texture[..., 0].astype(np.float64) + 1j * texture[..., 1]
    h0m = texture[..., 2].astype(np.float64) + 1j * texture[..., 3]
    return nm.ifft_maps(nm.modulate(h0, h0m, N, TILE, ss.DEPTH, time, phase_fp32=False))[0].imag


def _single(ix, iy, a):
    amps = np.zeros((N, N), np.complex64)
    amps[iy, ix] = a
    return po.spectrum_texture(amps)


def _wave(ix, iy):
    """world wave vector (the transposed map), k and omega of texel (ix, iy), float64"""
    kvx = (ix - N / 2) * 2 * math.pi / TILE[0]
    kvy = (iy - N / 2) * 2 * math.pi / TILE[1]
    k = math.hypot(kvx, kvy)
    return np.array([kvy, kvx]), k, math.sqrt(9.81 * k * math.tanh(k * ss.DEPTH))


@pytest.mark.parametrize("ix,iy", [(N // 2 + 3, N // 2 - 5), (N // 2 - 7, N // 2 + 2), (N // 2 + 1, N // 2)])
def test_single_wave_variance_direction_and_stokes(ix, iy):
    a = 0.3 * np.exp(0.7j)
    tex = _single(ix, iy, a)
    m = ss.cascade_moments(tex, TILE)
    assert m[1] == pytest.approx(2 * abs(a) ** 2, rel=1e-6)
    h = _height(tex, 3.0)
    assert np.mean(h * h) == pytest.approx(m[1], rel=1e-9)
    assert np.max(np.abs(h)) == pytest.approx(2 * abs(a), rel=1e-2)
    kw, k, w = _wave(ix, iy)
    # phase of the wave on the world grid (x along the map's columns, z along its rows) at two times
    xs = np.arange(N) * TILE[0] / N
    zs = np.arange(N) * TILE[1] / N
    basis = np.exp(-1j * (kw[0] * xs[None, :] + kw[1] * zs[:, None]))
    dt = 0.01
    c0 = np.sum(_height(tex, 3.0) * basis)
    c1 = np.sum(_height(tex, 3.0 + dt) * basis)
    assert abs(c0) == pytest.approx(N * N * abs(a), rel=1e-6)      # the wave vector of the map is kw
    dpsi = np.angle(c1 / c0)
    assert dpsi == pytest.approx(w * dt, rel=1e-4)                  # cos(kw.x + w t + phi): crests travel along -kw
    d = -kw / k
    assert m[4:6] / m[1] == pytest.approx(d, abs=1e-5)
    F = math.cosh(2 * k * ss.DEPTH) / (2 * math.sinh(k * ss.DEPTH) ** 2)
    assert m[8:10] == pytest.approx(w * k * (2 * abs(a)) ** 2 * F * d, rel=1e-5, abs=1e-12)


def _sparse(rng, count):
    """random amplitudes on `count` texels, none on row or column 0, the DC texel, or both a texel and its mirror"""
    amps = np.zeros((N, N), np.complex64)
    used = set()
    while len(used) < count:
        x, y = (int(v) for v in rng.integers(1, N, 2))
        if (x, y) == (N // 2, N // 2) or (x, y) in used or (N - x, N - y) in used:
            continue
        used.add((x, y))
        amps[y, x] = rng.normal() + 1j * rng.normal()
    return po.spectrum_texture(amps)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_parseval_on_sparse_spectra(seed):
    rng = np.random.default_rng(seed)
    tex = _sparse(rng, 40)
    m0 = ss.cascade_moments(tex, TILE)[1]
    for t in (0.0, 1.7, 123.4):
        h = _height(tex, t)
        assert np.mean(h * h) == pytest.approx(m0, rel=1e-6)


def test_parseval_mean_over_time_with_mirrored_waves():
    """A texel and its mirror interfere (a standing component), so the variance oscillates; its mean over time is m0."""
    amps = np.zeros((N, N), np.complex64)
    amps[N // 2 + 4, N // 2 + 9] = 0.5
    amps[N // 2 - 4, N // 2 - 9] = 0.3j
    tex = po.spectrum_texture(amps)
    m0 = ss.cascade_moments(tex, TILE)[1]
    times = np.linspace(0.0, 200.0, 801)
    v = [np.mean(_height(tex, t) ** 2) for t in times]
    assert np.std(v) > 0.05 * m0
    assert np.mean(v) == pytest.approx(m0, rel=2e-2)


def test_fixed_order_matches_exact_sums():
    rng = np.random.default_rng(5)
    amps = (rng.normal(size=(N, N)) + 1j * rng.normal(size=(N, N))).astype(np.complex64) * np.float32(0.01)
    tex = po.spectrum_texture(amps)
    terms = ss.texel_terms(tex, TILE)
    got = ss.fixed_sum(terms)
    for j in range(ss.MOMENTS):
        exact = math.fsum(terms[:, j])
        scale = math.fsum(np.abs(terms[:, j]))
        assert abs(got[j] - exact) <= 1e-12 * scale, j


def test_derived_fields():
    rng = np.random.default_rng(9)
    m = ss.cascade_moments(_sparse(rng, 30), TILE)
    r = ss.record(m)
    assert r["significant_wave_height"] == 4 * math.sqrt(m[1])
    assert r["mean_period"] == 2 * math.pi * m[1] / m[2]
    assert r["zero_crossing_period"] == 2 * math.pi * math.sqrt(m[1] / m[3])
    assert r["energy_period"] == 2 * math.pi * m[0] / m[1]
    assert r["mean_square_slope"] == m[6] + m[7]
    assert r["stokes_speed"] == math.hypot(m[8], m[9])
    R = math.hypot(m[4], m[5]) / m[1]
    assert 0 <= R <= 1 and r["directional_spread"] == math.sqrt(2 * (1 - R))
    zero = ss.record(np.zeros(ss.MOMENTS))
    assert all(np.all(zero[f] == 0) for f in ss.SEA_STATE.names)


@pytest.mark.parametrize("wind_direction", [0.0, 30.0, -120.0, 75.0])
def test_mean_direction_follows_wind_direction(wind_direction):
    """The generated spectrum of a narrow wind sea peaks at spectrum_compute.glsl's theta = wind_direction: the mean direction
    reports it in the same degrees."""
    p = po.CascadeParams(wind_direction=wind_direction, wind_speed=10.0, fetch_length=100.0, spread=0.0, swell=0.0,
                         tile_length=(1000.0, 1000.0), spectrum_seed=(3, 4))      # the peak (about 60 m) well resolved
    o = po.OracleWaveGenerator(N)
    o.init_gpu(1)
    o.update_all(0.02, [p])
    r = ss.record(ss.cascade_moments(o.spectrum[0], p.tile_length))
    diff = (r["mean_direction"] - wind_direction + 180.0) % 360.0 - 180.0
    assert abs(diff) < 3.0
    assert r["significant_wave_height"] > 0
