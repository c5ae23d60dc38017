"""The wake layer's specification (oracle/wake.py) on the CPU: the stencil's taps and their fit, the exact interior
evolution of lattice modes against the scheme's own discrete frequency and damping, the deep-water dispersion over the
stated band, scrolling, and the rasterisation of sources."""
import importlib.util
import os

import numpy as np
import pytest

from oracle import wake as wk

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K_LO, K_HI = 0.4, 2.0           # the band stated in include/ocean.h, in units of 1/dx


def _fit_script():
    spec = importlib.util.spec_from_file_location("fit_wake_kernel", os.path.join(ROOT, "tools", "fit_wake_kernel.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _zone(n):
    ax = np.linspace(-np.pi, np.pi, n)
    return np.meshgrid(ax, ax, indexing="ij")


def test_taps_are_the_fit_scripts_output():
    assert wk.taps().tobytes() == _fit_script().fit()[0].tobytes()


def test_taps_sum_sign_cap_and_band_error():
    g = wk.taps().astype(np.float64)
    counts = np.array([len(wk.orbit(a, b)) for a, b in wk.OFFSETS], float)
    assert counts @ g == 0.0                                    # exact: the k = 0 mode is neutral
    kx, kz = _zone(1201)
    gh = wk.symbol(g, kx, kz)
    assert gh.min() >= -1e-12 and gh.max() <= wk.CAP
    k = np.linspace(K_LO, K_HI, 200)
    for th in np.linspace(0.0, np.pi / 2, 19):
        rel = wk.symbol(g, k * np.cos(th), k * np.sin(th)) / k - 1.0
        assert np.abs(rel).max() <= 0.039


def test_stability_bound():
    dx = np.float32(0.5)
    h_max = np.sqrt(float(dx) / wk.G)
    assert wk.stable(dx, np.float32(h_max) if np.float32(h_max) <= h_max else np.nextafter(np.float32(h_max), np.float32(0)))
    assert not wk.stable(dx, np.nextafter(np.float32(h_max), np.float32(1)))


def _layer(n, dx, damping=0.0, sponge_cells=0, sponge_damping=0.0):
    p = np.zeros((), wk.PARAMS)
    p["size"], p["cell_size"], p["damping"], p["sponge_cells"], p["sponge_damping"] = n, dx, damping, sponge_cells, sponge_damping
    return wk.Layer(p)


def _mode(n, m, l):
    i = np.arange(n)
    kx, kz = 2 * np.pi * m / n, 2 * np.pi * l / n
    return np.cos(kx * i[None, :] + kz * i[:, None]), kx, kz


@pytest.mark.parametrize("m,l", [(24, 0), (20, 14), (40, 30)])
def test_lattice_mode_follows_the_discrete_frequency(m, l):
    """A lattice mode started with h_prev from omega_d = arccos(1 - a3 Ghat / 2) / h: after n sub-steps every cell farther
    than 6 n from the edge follows cos(omega_d t) (the stencil spreads 6 cells per sub-step)."""
    n, dx, steps = 256, np.float32(0.5), 16
    L = _layer(n, dx)
    h = wk.substep(0.8 * np.sqrt(0.5 / wk.G), 1)
    shape, kx, kz = _mode(n, m, l)
    a3 = float(wk.coefficients(L.params, h)[2, 0])
    w = np.arccos(1.0 - a3 * wk.symbol(wk.taps(), kx, kz) / 2.0) / float(h)
    L.h = shape.astype(np.float32)
    L.h_prev = (shape * np.cos(w * float(h))).astype(np.float32)
    core = slice(6 * steps, n - 6 * steps)
    for k in range(1, steps + 1):
        L.step(h, 1, (0, 0))
        assert np.abs(L.h[core, core] - shape[core, core] * np.cos(w * float(h) * k)).max() < 1e-5


def test_discrete_dispersion_is_deep_water_over_the_band():
    """omega_d against sqrt(g |k|) for |k| dx in the band, every direction, at a quarter of the largest sub-step (the
    figure DESIGN.md states); at the largest sub-step the time discretisation adds its own error at short waves."""
    dx = 0.5
    g = wk.taps()
    worst = 0.0
    for frac in (0.25,):
        h = float(np.float32(frac * np.sqrt(dx / wk.G)))
        a3 = wk.G * h * h / dx
        k = np.linspace(K_LO, K_HI, 100)
        for th in np.linspace(0.0, np.pi / 4, 10):
            w = np.arccos(1.0 - a3 * wk.symbol(g, k * np.cos(th), k * np.sin(th)) / 2.0) / h
            worst = max(worst, np.abs(w / np.sqrt(wk.G * k / dx) - 1.0).max())
    assert worst <= 0.025


def test_uniform_damping_decays_at_the_schemes_rate():
    """With uniform alpha the interior of a lattice mode follows the scalar recurrence e' = (a1 e - a2 e_prev) - a3 Ghat e,
    whose envelope shrinks by sqrt(a2) per sub-step."""
    n, dx, steps = 256, np.float32(0.5), 16
    L = _layer(n, dx, damping=0.5, sponge_cells=0)
    h = wk.substep(0.2, 1)
    shape, kx, kz = _mode(n, 20, 14)
    a1, a2, a3 = (float(c[0]) for c in wk.coefficients(L.params, h))
    gh = wk.symbol(wk.taps(), kx, kz)
    L.h = shape.astype(np.float32)
    L.h_prev = shape.astype(np.float32)
    e, ep = 1.0, 1.0
    core = slice(6 * steps, n - 6 * steps)
    for _ in range(steps):
        L.step(h, 1, (0, 0))
        e, ep = (a1 * e - a2 * ep) - a3 * gh * e, e
        assert np.abs(L.h[core, core] - shape[core, core] * e).max() < 1e-5
    # the envelope: |z|^2 = a2 for the complex roots of z^2 - (a1 - a3 Ghat) z + a2
    z = np.roots([1.0, -(a1 - a3 * gh), a2])
    assert np.allclose(np.abs(z), np.sqrt(a2))


@pytest.mark.parametrize("di,dj", [(0, 0), (3, 0), (-5, 7), (17, -128), (-200, 1), (256, 0), (0, -256), (10**12, 5)])
def test_scroll_is_a_shift_with_zero_fill(di, dj):
    n = 256
    f = np.random.default_rng(5).normal(size=(n, n)).astype(np.float32)
    out = wk.scroll(f, di, dj)
    ref = np.zeros_like(f)
    for j in range(n):
        for i in range(n):
            if 0 <= i + di < n and 0 <= j + dj < n:
                ref[j, i] = f[j + dj, i + di]
    assert out.tobytes() == ref.tobytes()


def _sources(rng, k, n_states):
    s = np.zeros(k, wk.SOURCE)
    s["x"], s["z"] = rng.uniform(-5, 70, k), rng.uniform(-5, 70, k)
    s["vx"], s["vz"] = rng.uniform(-3, 3, k), rng.uniform(-3, 3, k)
    s["radius"] = rng.uniform(0.3, 6, k)
    s["head"] = rng.uniform(-0.5, 0.5, k)
    s["body"] = np.where(rng.random(k) < 0.3, rng.integers(0, n_states, k), -1)
    return s


def test_rasterisation_matches_a_per_cell_loop():
    rng = np.random.default_rng(7)
    n, dx, origin, tau = 128, np.float32(0.5), (3, -2), np.float32(0.125)
    st = np.zeros(4, wk.STATE)
    st["position"] = rng.uniform(0, 40, (4, 3))
    st["linear_velocity"] = rng.uniform(-2, 2, (4, 3))
    s = _sources(rng, 24, 4)
    s["radius"][3] = 0.0
    s["radius"][4] = -1.0
    s["head"][5] = np.nan
    s["x"][6] = np.inf
    s["radius"][7] = np.inf
    s["body"][8] = 4                                           # not below num_states: nothing
    phi = wk.rasterise(n, dx, origin, s, st, tau)
    x0, z0 = wk.world_origin(origin, dx)
    ref = np.zeros((n, n), np.float32)
    f = np.float32
    for k in range(len(s)):
        r = s[k]
        cx, cz = r["x"] + r["vx"] * tau, r["z"] + r["vz"] * tau
        if r["body"] >= 0:
            if r["body"] >= len(st):
                continue
            b = st[r["body"]]
            cx, cz = cx + (b["position"][0] + b["linear_velocity"][0] * tau), cz + (b["position"][2] + b["linear_velocity"][2] * tau)
        r2 = r["radius"] * r["radius"]
        if not (np.isfinite([cx, cz, r["head"], r["radius"], r2]).all() and r["radius"] > 0):
            continue
        for j in range(n):
            pz = z0 + (f(j) + f(0.5)) * dx
            for i in range(n):
                px = x0 + (f(i) + f(0.5)) * dx
                d2 = (px - cx) * (px - cx) + (pz - cz) * (pz - cz)
                if d2 < r2:
                    w = f(1) - d2 / r2
                    ref[j, i] = ref[j, i] + r["head"] * (w * w)
    assert phi.tobytes() == ref.tobytes()
    assert np.count_nonzero(phi) > 1000
    bad = s[[3, 4, 5, 6, 7, 8]]
    assert not wk.rasterise(n, dx, origin, bad, st, tau).any()


def test_sample_matches_the_map_inside_and_is_zero_outside():
    n, dx = 128, np.float32(0.5)
    h = np.random.default_rng(8).normal(size=(n, n)).astype(np.float32)
    origin = (-40, 12)
    x0, z0 = wk.world_origin(origin, dx)
    gx, gz = wk.gradients(h, dx)
    centres = np.array([[x0 + (i + 0.5) * dx, z0 + (j + 0.5) * dx] for i, j in [(0, 0), (5, 9), (127, 127), (64, 3)]], np.float32)
    out = wk.sample(h, dx, origin, centres)
    for (i, j), o in zip([(0, 0), (5, 9), (127, 127), (64, 3)], out):
        assert (o == [h[j, i], gx[j, i], gz[j, i]]).all()
    far = np.array([[x0 - 0.01, z0 + 1], [x0 + n * dx, z0 + 1], [x0 + 1, z0 + n * dx + 3], [np.nan, z0 + 1]], np.float32)
    assert not wk.sample(h, dx, origin, far).any()
