"""oracle/drifters.py: labels that stay put without drift sources, closed orbits over whole periods, the mean drift rate,
the render against ocean_sample_maps' sampling and Godot's Basis(UP, yaw), consistency with the velocity maps, and the wrap."""
import math

import numpy as np
import pytest

from oracle import drifters as od
from oracle import numpy_model as nm
from oracle import pyoracle as po
from oracle import sampling as sp
from oracle import velocity as ov

N = 128
TILE = (50.0, 50.0)
SCALES = np.array([[1 / 50.0, 1 / 50.0, 1.0, 1.0]], np.float32)


@pytest.fixture(autouse=True)
def _modes():
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    yield
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)


def _single_wave(ix=N // 2 + 3, iy=N // 2 - 5, a=0.4):
    amps = np.zeros((N, N), np.complex64)
    amps[iy, ix] = a
    t = po.spectrum_texture(amps)
    return t[..., 0].astype(np.float64) + 1j * t[..., 1], t[..., 2].astype(np.float64) + 1j * t[..., 3]


def _maps(h0, h0m, time):
    """[1][N][N][4] float16 displacement and normal maps of the float64 model at `time` (foam 0)."""
    f = nm.ifft_maps(nm.modulate(h0, h0m, N, TILE, 20.0, time, phase_fp32=False))
    disp, normal, _ = nm.unpack(f, np.zeros((N, N)), 0.5, 0.0, 0.0)
    return disp[None].astype(np.float16), normal[None].astype(np.float16)


def _drifters(n, seed=0):
    rng = np.random.default_rng(seed)
    d = np.zeros(n, od.DRIFTER)
    d["x"] = rng.uniform(-40, 40, n)
    d["z"] = rng.uniform(-40, 40, n)
    d["yaw"] = rng.uniform(-3, 3, n)
    d["yaw_rate"] = rng.uniform(-1, 1, n)
    d["scale"] = 1.5
    return d


def _params(**kw):
    p = np.zeros((), od.PARAMS)
    for k, v in kw.items():
        p[k] = v
    return p


def test_no_drift_without_sources():
    d = _drifters(200)
    p = _params(stokes_scale=0.0)
    moments = [np.arange(10, dtype=np.float64)]
    out = d
    for _ in range(50):
        out = od.advance(out, 1.0 / 60.0, p, od.stokes_total(moments, SCALES))
    assert np.array_equal(out[["x", "z"]], d[["x", "z"]])


def test_closed_orbit_over_whole_periods():
    h0, h0m = _single_wave()
    kvx, kvy = 3 * 2 * math.pi / 50.0, -5 * 2 * math.pi / 50.0
    k = math.hypot(kvx, kvy)
    T = 2 * math.pi / math.sqrt(9.81 * k * math.tanh(20.0 * k))
    d = _drifters(100, seed=1)
    d["tilt"] = 1.0
    X0 = od.render(d, *_maps(h0, h0m, 7.0), SCALES)
    Xh = od.render(d, *_maps(h0, h0m, 7.0 + 0.5 * T), SCALES)
    X1 = od.render(d, *_maps(h0, h0m, 7.0 + 3 * T), SCALES)
    assert np.allclose(X1, X0, atol=2e-3)
    assert not np.allclose(Xh[:, 7], X0[:, 7], atol=0.1)   # half a period later the drifters are elsewhere on the orbit


def test_drift_rate_is_the_stokes_vector():
    d = _drifters(50, seed=2)
    moments = [np.r_[np.zeros(8), 0.03, -0.01], np.r_[np.zeros(8), 0.02, 0.05]]
    sc = np.array([[0.02, 0.02, 1.0, 1.0], [0.1, 0.1, 0.5, 1.0]], np.float32)
    us = od.stokes_total(moments, sc)
    assert us == pytest.approx((0.03 + 0.25 * 0.02, -0.01 + 0.25 * 0.05))
    out = d
    steps, dt = 600, 1.0 / 60.0
    for _ in range(steps):
        out = od.advance(out, dt, _params(stokes_scale=1.0), us)
    v = np.stack([out["x"] - d["x"], out["z"] - d["z"]], axis=-1) / (steps * dt)
    assert np.allclose(v, us, rtol=1e-9)


def test_render_at_tilt_zero_is_the_map_sample_and_godot_basis():
    rng = np.random.default_rng(4)
    disp = (rng.normal(size=(1, N, N, 4)) * 0.5).astype(np.float16)
    normal = (rng.normal(size=(1, N, N, 4)) * 0.2).astype(np.float16)
    d = _drifters(300, seed=4)
    inst = od.render(d, disp, normal, SCALES)
    P = np.stack([d["x"], d["z"]], axis=-1).astype(np.float32)
    D, _ = sp.sample_maps(disp, normal, P, SCALES)
    assert np.array_equal(inst[:, 3], (d["x"] + D[:, 0]).astype(np.float32))
    assert np.array_equal(inst[:, 7], D[:, 1])
    assert np.array_equal(inst[:, 11], (d["z"] + D[:, 2]).astype(np.float32))
    c, s = np.cos(d["yaw"].astype(np.float64)), np.sin(d["yaw"].astype(np.float64))
    z = np.zeros_like(c)
    godot = np.stack([c, z, s, z, z + 1, z, -s, z, c], axis=-1).reshape(-1, 3, 3) * 1.5   # Basis(UP, yaw) rows
    basis = inst.reshape(-1, 3, 4)[:, :, :3]
    assert np.allclose(basis, godot, atol=1e-6)


def test_label_motion_matches_the_velocity_maps():
    """(X(t + h) - X(t)) / h at a fixed label is the water velocity at the label (ocean_sample_velocity's)."""
    h0, h0m = _single_wave(a=0.2)
    d = _drifters(200, seed=5)
    t, h = 11.0, 1e-3
    f0 = nm.ifft_maps(nm.modulate(h0, h0m, N, TILE, 20.0, t, phase_fp32=False))
    f1 = nm.ifft_maps(nm.modulate(h0, h0m, N, TILE, 20.0, t + h, phase_fp32=False))
    vel = ov.float64_velocity(h0, h0m, N, TILE, 20.0, t, phase_fp32=False)
    # at texel centres the bilinear filter is exact: compare the fields there
    fd = (np.stack([f1[0].real, f1[0].imag, f1[1].real]) - np.stack([f0[0].real, f0[0].imag, f0[1].real])) / h
    assert np.allclose(fd, vel, atol=2e-3 * np.max(np.abs(vel)))
    # and through the render: X moves with the sampled velocity
    vmap = np.concatenate([np.moveaxis(vel, 0, -1), np.zeros((N, N, 1))], axis=-1)[None].astype(np.float16)
    X0 = od.render(d, *_maps(h0, h0m, t - 0.02), SCALES).astype(np.float64)
    X1 = od.render(d, *_maps(h0, h0m, t + 0.02), SCALES).astype(np.float64)
    P = np.stack([d["x"], d["z"]], axis=-1).astype(np.float32)
    v, _ = sp.sample_maps(vmap, vmap, P, SCALES)
    got = (X1[:, [3, 7, 11]] - X0[:, [3, 7, 11]]) / 0.04           # central difference: half-map rounding dominates
    assert np.allclose(got, v, atol=0.03 * np.max(np.abs(v)))


def test_wrap_keeps_labels_in_the_box_exactly():
    rng = np.random.default_rng(6)
    d = np.zeros(5000, od.DRIFTER)
    d["x"] = rng.uniform(-1e4, 1e4, d.size)
    d["z"] = rng.uniform(-1e4, 1e4, d.size)
    d["x"][:3] = (-1e-300, 250.0, -250.0)
    box = (-250.0, 100.0, 500.0, 300.0)
    p = _params(current=(1.5, -0.5), stokes_scale=0.0, flags=od.WRAP, box=box)
    out = od.advance(d, 0.5, p, (0.0, 0.0))
    free = od.advance(d, 0.5, _params(current=(1.5, -0.5), stokes_scale=0.0), (0.0, 0.0))
    assert np.all((out["x"] >= -250.0) & (out["x"] <= 250.0)) and np.all((out["z"] >= 100.0) & (out["z"] <= 400.0))
    nx = (free["x"] - out["x"]) / 500.0
    nz = (free["z"] - out["z"]) / 300.0
    assert np.allclose(nx, np.round(nx), atol=1e-9) and np.allclose(nz, np.round(nz), atol=1e-9)
    inside = (free["x"] >= -250.0) & (free["x"] < 250.0)
    assert np.array_equal(out["x"][inside], free["x"][inside])
