"""CPU checks of the map-sampling restatement (oracle/sampling.py; water.gdshader:27-39,42-84)."""
import numpy as np
import pytest

from oracle import sampling as sp


def _tex(N, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((N, N, 4)).astype(np.float16)


def test_bilinear_hits_texel_centres_and_wraps():
    N = 128
    t = _tex(N, 1)
    xs, ys = np.meshgrid(np.arange(N), np.arange(N))
    u = ((xs.ravel() + 0.5) / N).astype(np.float32)
    v = ((ys.ravel() + 0.5) / N).astype(np.float32)
    out = sp.texture_bilinear(t, u, v)
    assert np.array_equal(out, t.astype(np.float32).reshape(-1, 4))
    # REPEAT addressing: whole-tile shifts (exact in binary32 for these dyadic coordinates) change nothing
    for shift in (1.0, -3.0, 64.0):
        assert np.array_equal(sp.texture_bilinear(t, u + np.float32(shift), v - np.float32(shift)), out)


def test_bilinear_wraps_beyond_the_int64_range():
    """At |u*N| >= 2^63 the texel index still follows REPEAT addressing (floor(u*N - 0.5) mod N, computed here with
    Python integers), without a RuntimeWarning from an out-of-range conversion; so does bilinear_slopes."""
    import warnings
    from oracle import surface as su
    N = 8
    t = _tex(N, 9)
    # x = u*N - 0.5 rounds to u*N at these magnitudes, all beyond 2^63 (3e37*8 near FLT_MAX); the saturating conversion
    # of the GPU would give INT64_MAX mod N = N - 1 for the positive ones, REPEAT gives texel 0
    big =np.array([1e20, -1e20, 2.0 ** 61, -(2.0 ** 61), 3e37, -3e37, 3.0 * 2.0 ** 61, 1e19], np.float32)
    v = np.full(big.size, np.float32(2.5 / N), np.float32)               # texel row 2, fy = 0
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        out = sp.texture_bilinear(t, big, v)
        du, dv = su.bilinear_slopes(t, big, v)
    x = big * np.float32(N) - np.float32(0.5)
    assert np.all(np.abs(x) >= 2.0 ** 63) and np.array_equal(x, np.floor(x))
    ix = [int(xi) % N for xi in x]                                          # exact: Python int of a binary32
    assert np.array_equal(out, t.astype(np.float32)[2, ix])
    # the same texels at an in-range coordinate: u = (ix + 0.5) / N
    u_in = ((np.array(ix) + 0.5) / N).astype(np.float32)
    assert np.array_equal(out, sp.texture_bilinear(t, u_in, v))
    du_in, dv_in = su.bilinear_slopes(t, u_in, v)
    assert np.array_equal(du, du_in) and np.array_equal(dv, dv_in)
    # NaN and infinities: index 0, NaN fields
    with np.errstate(invalid="ignore"):
        odd = sp.texture_bilinear(t, np.array([np.nan, np.inf, -np.inf], np.float32), v[:3])
    assert np.isnan(odd).all()


def test_bilinear_matches_scipy_grid_wrap():
    ndi = pytest.importorskip("scipy.ndimage")
    N = 128
    t = _tex(N, 2)
    rng = np.random.default_rng(3)
    u = rng.uniform(-2.0, 3.0, 4000).astype(np.float32)
    v = rng.uniform(-2.0, 3.0, 4000).astype(np.float32)
    out = sp.texture_bilinear(t, u, v)
    # the sample position as the filter sees it (binary32 u*N - 0.5), then exact interpolation in float64
    x = (u * np.float32(N) - np.float32(0.5)).astype(np.float64)
    y = (v * np.float32(N) - np.float32(0.5)).astype(np.float64)
    for ch in range(4):
        ref = ndi.map_coordinates(t[:, :, ch].astype(np.float64), [y, x], order=1, mode="grid-wrap")
        assert np.allclose(out[:, ch], ref, rtol=0, atol=5e-6)


def test_bicubic_is_the_uniform_b_spline():
    N = 128
    t = _tex(N, 4)
    rng = np.random.default_rng(5)
    u = rng.uniform(-1.0, 2.0, 2000).astype(np.float32)
    v = rng.uniform(-1.0, 2.0, 2000).astype(np.float32)
    out = sp.texture_bicubic(t, u, v)
    # direct 16-tap cubic B-spline in float64 at the same sample position (texel centres at integer + 0.5)
    x = u.astype(np.float64) * N - 0.5
    y = v.astype(np.float64) * N - 0.5
    x0, y0 = np.floor(x), np.floor(y)
    a, b = x - x0, y - y0

    def w(a):
        return np.stack([(1 - a) ** 3, 3 * a ** 3 - 6 * a ** 2 + 4, -3 * a ** 3 + 3 * a ** 2 + 3 * a + 1, a ** 3]) / 6.0

    wx, wy = w(a), w(b)
    tf = t.astype(np.float64)
    ref = np.zeros((u.size, 4))
    for j in range(4):
        for i in range(4):
            ix = np.mod(x0.astype(np.int64) - 1 + i, N)
            iy = np.mod(y0.astype(np.int64) - 1 + j, N)
            ref += (wx[i] * wy[j])[:, None] * tf[iy, ix]
    assert np.allclose(out, ref, rtol=0, atol=5e-4)          # binary32 weights, four-tap factorisation
    # partition of unity: a constant texture stays constant
    const = np.full((N, N, 4), 1.5, np.float16)
    assert np.allclose(sp.texture_bicubic(const, u, v), 1.5, rtol=0, atol=1e-6)


def test_sample_maps_sums_cascades_with_their_scales():
    N, C = 128, 3
    rng = np.random.default_rng(6)
    disp = rng.standard_normal((C, N, N, 4)).astype(np.float16)
    nrm = rng.standard_normal((C, N, N, 4)).astype(np.float16)
    pts = rng.uniform(-200.0, 200.0, (500, 2)).astype(np.float32)
    scales = np.array([[1 / 88.0, 1 / 88.0, 1.0, 1.0], [1 / 57.0, 1 / 57.0, 0.75, 1.0], [1 / 8.0, 1 / 8.0, 0.0, 0.25]], np.float32)
    d, g = sp.sample_maps(disp, nrm, pts, scales)
    assert d.dtype == np.float32 and d.shape == (500, 3) and g.shape == (500, 3)
    # cascade 2 has displacement_scale 0 (main.tscn:71-83): it contributes nothing to the displacement ...
    d2, _ = sp.sample_maps(disp[:2], nrm[:2], pts, scales[:2])
    assert np.array_equal(d, d2)
    # ... and the foam channel ignores normal_scale (vec3(scales.ww, 1.0), water.gdshader:83)
    s2 = scales.copy(); s2[:, 3] = 0.0
    _, g0 = sp.sample_maps(disp, nrm, pts, s2)
    assert np.all(g0[:, :2] == 0.0) and np.array_equal(g0[:, 2], g[:, 2])
    # high pixel density (ppm*0.1 >= 1) selects the plain bilinear filter
    u = pts[:, 0] * scales[2, 0]; v = pts[:, 1] * scales[2, 1]
    _, g_last = sp.sample_maps(disp[2:], nrm[2:], pts, scales[2:])
    assert N * scales[2, 0] * 0.1 >= 1.0
    assert np.array_equal(g_last[:, 2], (np.zeros(500, np.float32) + sp.texture_bilinear(nrm[2], u, v)[:, 3] * np.float32(1.0)))
