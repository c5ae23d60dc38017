"""CPU checks of the surface-query specification (oracle/surface.py): the surface at a world position, found by inverting
the horizontal displacement of the water shader (water.gdshader:28,37) and sampling the maps there."""
import numpy as np
import pytest

from conftest import demo_params
from oracle import sampling as sp
from oracle import surface as su

TOL = np.float32(1e-3)


@pytest.fixture(scope="module")
def demo_maps():
    """Demo 256^2 x 4 after two updates, from the CPU oracle, with map_scales as water.gd:102-110 builds them."""
    from oracle import pyoracle as po
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    gen = po.OracleWaveGenerator(256)
    gen.init_gpu(4)
    params = [demo_params(po.CascadeParams, c) for c in range(4)]
    for _ in range(2):
        gen.update_all(1.0 / 50.0, params)
    scales = np.array([[np.float32(1.0) / np.float32(p.tile_length[0]), np.float32(1.0) / np.float32(p.tile_length[1]),
                        p.displacement_scale, p.normal_scale] for p in params], np.float32)
    return gen.displacement_map[:4].view(np.float16).copy(), gen.normal_map[:4].view(np.float16).copy(), scales


def _points(n, seed):
    return np.random.default_rng(seed).uniform(-300.0, 300.0, (n, 2)).astype(np.float32)


def test_record_layout():
    assert su.RECORD.itemsize == 40
    assert list(su.RECORD.names) == ["source_x", "source_z", "displacement", "gradient_foam", "residual", "iterations"]


def test_zero_iterations_is_the_map_query(demo_maps):
    d16, n16, scales = demo_maps
    pts = _points(3000, 1)
    rec = su.query_surface(d16, n16, pts, scales, TOL, 0)
    d, g = sp.sample_maps(d16, n16, pts, scales)
    assert rec["displacement"].tobytes() == d.tobytes() and rec["gradient_foam"].tobytes() == g.tobytes()
    assert rec["source_x"].tobytes() == pts[:, 0].tobytes() and rec["source_z"].tobytes() == pts[:, 1].tobytes()
    assert np.all(rec["iterations"] == 0)


def test_zero_displacement_is_the_identity(demo_maps):
    _, n16, scales = demo_maps
    pts = _points(2000, 2)
    rec = su.query_surface(np.zeros((4, 256, 256, 4), np.float16), n16, pts, scales, TOL, 8)
    assert rec["source_x"].tobytes() == pts[:, 0].tobytes() and rec["source_z"].tobytes() == pts[:, 1].tobytes()
    assert np.all(rec["iterations"] == 0) and np.all(rec["residual"] == 0.0)


def test_bilinear_slopes_are_the_derivative_of_the_interpolant():
    rng = np.random.default_rng(3)
    N = 128
    tex = rng.standard_normal((N, N, 4)).astype(np.float16)
    # inside one texel cell the bilinear interpolant is linear along each axis: a central difference is exact up to rounding
    x0 = rng.integers(0, N, 500)
    y0 = rng.integers(0, N, 500)
    fx = rng.uniform(0.2, 0.8, 500)
    fy = rng.uniform(0.2, 0.8, 500)
    u = ((x0 + 0.5 + fx) / N).astype(np.float32)
    v = ((y0 + 0.5 + fy) / N).astype(np.float32)
    du, dv = su.bilinear_slopes(tex, u, v)
    h = np.float32(0.1 / N)
    num_u = (sp.texture_bilinear(tex, u + h, v).astype(np.float64) - sp.texture_bilinear(tex, u - h, v)) / (2.0 * np.float64(h))
    num_v = (sp.texture_bilinear(tex, u, v + h).astype(np.float64) - sp.texture_bilinear(tex, u, v - h)) / (2.0 * np.float64(h))
    assert np.allclose(du, num_u, rtol=0, atol=0.05) and np.allclose(dv, num_v, rtol=0, atol=0.05)


def test_single_gerstner_wave_matches_the_continuous_trochoid():
    """One trochoidal wave written straight into a displacement texture: D(P) = (-k^ A sin(k.P), A cos(k.P)).  The query's
    height at Q must match a float64 root solve of the continuous trochoid, Q = P - k^ A sin(k.P)."""
    N, L = 256, np.float32(64.0)
    kv = 2.0 * np.pi * np.array([2.0, 1.0]) / float(L)         # two and one wave lengths per tile along x, z: periodic
    kn = np.linalg.norm(kv)
    khat = kv / kn
    A = 0.5 / kn                                               # steepness A|k| = 0.5: no folds
    c = (np.arange(N) + 0.5) * (float(L) / N)                  # texel centres in metres
    X, Z = np.meshgrid(c, c)                                   # row = z, column = x
    ph = kv[0] * X + kv[1] * Z
    tex = np.zeros((1, N, N, 4), np.float16)
    tex[0, :, :, 0] = -khat[0] * A * np.sin(ph)
    tex[0, :, :, 1] = A * np.cos(ph)
    tex[0, :, :, 2] = -khat[1] * A * np.sin(ph)
    scales = np.array([[1.0 / L, 1.0 / L, 1.0, 1.0]], np.float32)
    pts = _points(20000, 4)
    rec = su.query_surface(tex, np.zeros_like(tex), pts, scales, TOL, 8)
    assert np.all(rec["residual"] <= TOL)

    # float64 root of s - A sin(|k| s) = k^.Q along the wave direction (monotone, A|k| < 1)
    q = khat[0] * pts[:, 0].astype(np.float64) + khat[1] * pts[:, 1].astype(np.float64)
    s = q.copy()
    for _ in range(50):
        s -= (s - A * np.sin(kn * s) - q) / (1.0 - A * kn * np.cos(kn * s))
    height = A * np.cos(kn * s)

    # bound: bilinear interpolation of a function with |f_xx| + |f_zz| <= A|k|^2 errs by at most h^2 A|k|^2 / 8, the half
    # texels by half an ulp, 2^-11 relative; the horizontal error and the residual tolerance move the source point by up to
    # sqrt(2) (e + tol) / (1 - A|k|), which changes the height by A|k| times that
    h = float(L) / N
    e = h * h * A * kn * kn / 8.0 + A * 2.0 ** -11
    bound = e + A * kn * np.sqrt(2.0) * (e + float(TOL)) / (1.0 - A * kn) + 1e-5
    err = np.abs(rec["displacement"][:, 1].astype(np.float64) - height)
    assert err.max() <= bound, (err.max(), bound)


@pytest.mark.parametrize("factor,bar", [(1.0, 0.999), (2.0, 0.99)])
def test_convergence_bar(demo_maps, factor, bar):
    d16, n16, scales = demo_maps
    sc = scales.copy()
    sc[:, 2] *= np.float32(factor)
    pts = _points(100000, 5)
    rec = su.query_surface(d16, n16, pts, sc, TOL, 8)
    conv = rec["residual"] <= TOL
    assert conv.mean() >= bar, conv.mean()
    # consistency: the map query at the source point puts its surface point back over the query
    k = np.nonzero(conv)[0]
    d, g = sp.sample_maps(d16, n16, np.stack([rec["source_x"][k], rec["source_z"][k]], 1), sc)
    assert d.tobytes() == rec["displacement"][k].tobytes() and g.tobytes() == rec["gradient_foam"][k].tobytes()
    ex = (rec["source_x"][k] + d[:, 0]) - pts[k, 0]
    ez = (rec["source_z"][k] + d[:, 2]) - pts[k, 1]
    assert np.all(np.fmax(np.abs(ex), np.abs(ez)) <= TOL)
    # the restarts ran (more steps than one start can take)
    assert np.any(rec["iterations"] > 8)
