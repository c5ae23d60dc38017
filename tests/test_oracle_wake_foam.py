"""CPU tests of the wake foam specification (oracle/wake_foam.py): it leaves the wake layer's h and h_prev exactly as
oracle/wake.py advances them; pure decay, a boat at rest, the stirred trail's cross-track profile, breaking on the crests
of a single wave, the scroll, and the clamp."""
import numpy as np

from oracle import wake as wk
from oracle import wake_foam as wf

f32 = np.float32
EPS = float(np.finfo(np.float32).eps)


def _params(n, dx, damping=0.0, sponge_cells=0, sponge_damping=0.0):
    p = np.zeros((), wk.PARAMS)
    p["size"], p["cell_size"], p["damping"], p["sponge_cells"], p["sponge_damping"] = n, dx, damping, sponge_cells, sponge_damping
    return p


def _sources(rng, k, extent, n_states=0):
    s = np.zeros(k, wk.SOURCE)
    s["x"], s["z"] = rng.uniform(0.1 * extent, 0.9 * extent, k), rng.uniform(0.1 * extent, 0.9 * extent, k)
    s["vx"], s["vz"] = rng.uniform(-4, 4, k), rng.uniform(-4, 4, k)
    s["radius"], s["head"], s["body"] = rng.uniform(1.0, 6.0, k), rng.uniform(-0.3, 0.3, k), -1
    if n_states:
        att = rng.random(k) < 0.5
        s["body"][att] = rng.integers(0, n_states, att.sum())
        s["x"][att], s["z"][att] = rng.uniform(-2, 2, att.sum()), rng.uniform(-2, 2, att.sum())
    return s


def test_h_and_h_prev_equal_the_wake_layer_bit_for_bit():
    rng = np.random.default_rng(3)
    n, dx = 128, 0.5
    p = _params(n, dx, damping=0.05, sponge_cells=16, sponge_damping=2.0)
    L, F = wk.Layer(p), wf.Layer(p, wf.foam_params(whitecap=0.01, grow_rate=2.0, stir_rate=0.05, decay_rate=0.3))
    st = np.zeros(3, wk.STATE)
    st["position"] = rng.uniform(10, 50, (3, 3))
    st["linear_velocity"] = rng.uniform(-2, 2, (3, 3))
    for S, origin in [(1, (0, 0)), (3, (3, -2)), (2, (-5, 4)), (1, (-5 + n, 4))]:
        s = _sources(rng, 6, n * dx, len(st))
        L.step(0.05 * S, S, origin, s, st)
        F.step(0.05 * S, S, origin, s, st)
        assert L.h.tobytes() == F.h.tobytes() and L.h_prev.tobytes() == F.h_prev.tobytes() and L.origin == F.origin
        if origin == (0, 0):
            assert F.foam.max() > 0
    assert 0 <= F.foam.min() and F.foam.max() <= 1


def test_pure_decay_is_the_binary32_recurrence():
    n, dx, decay, S, dt = 128, 1.0, 0.5, 8, 0.8
    F = wf.Layer(_params(n, dx), wf.foam_params(whitecap=0.1, grow_rate=3.0, stir_rate=2.0, decay_rate=decay))
    F0 = np.random.default_rng(1).uniform(0, 1, (n, n)).astype(np.float32)
    F.foam = F0.copy()
    F.step(dt, S, (0, 0))
    h = wk.substep(dt, S)
    d = wf.detmath_exp(-(f32(decay) * h))
    want = F0.copy()
    for _ in range(S):
        want = want * d
    assert F.foam.tobytes() == want.tobytes()
    exact = F0.astype(np.float64) * np.exp(-decay * S * float(h))
    assert np.abs(F.foam - exact).max() <= 1e-6


def test_a_source_at_rest_makes_no_foam():
    """alpha = 0 everywhere and h = h_prev = -phi under a stationary source: s = h + phi is exactly 0, so beta is 0 on
    every one of 1000 sub-steps, and the source's velocity is 0, so nothing is stirred."""
    n, dx = 128, 0.5
    F = wf.Layer(_params(n, dx), wf.foam_params(whitecap=0.0, grow_rate=10.0, stir_rate=10.0, decay_rate=0.0))
    s = np.zeros(1, wk.SOURCE)
    s["x"], s["z"], s["radius"], s["head"], s["body"] = 31.7, 30.2, 4.0, 0.5, -1
    phi = wk.rasterise(n, dx, (0, 0), s, None, 0.0)
    F.h, F.h_prev = -phi, -phi.copy()
    for _ in range(10):
        F.step(0.05 * 100, 100, (0, 0), s)
    assert np.array_equal(F.h, -phi)
    assert not F.foam.any()


def _trail(step, n, dx, U, r, z_src, x_start, x_end, h_sub, stir):
    """Drives a source of radius r along +x at U from x_start to x_end with stirring only (grow 0, decay 0) and returns F;
    step(dt, S, src) advances the layer under test by one call."""
    S = 100
    t, x = 0.0, x_start
    src = np.zeros(1, wk.SOURCE)
    src["z"], src["vx"], src["radius"], src["head"], src["body"] = z_src, U, r, 0.05, -1
    while x < x_end:
        src["x"] = np.float32(x)
        step(h_sub * S, S, src)
        t += h_sub * S
        x = x_start + U * t


def trail_profile_check(foam, n, dx, U, r, z_src, x_start, x_end, h_sub, stir):
    """The cross-track profile of every column the source passed over completely: F(y) against
    stir (16/15) r U (1 - y^2/r^2)^(5/2), the integral over time of stir w^2 U^2 with w = 1 - (x^2 + y^2) / r^2.
    The sub-steps sample that integral at spacing U h (a Riemann sum of f(x) = stir U (a^2 - x^2)^2 / r^4, a^2 = r^2 - y^2,
    whose value and slope vanish at x = +-a), so the error is at most (U h)^2 times the integral of |f''|, which is
    stir U 32 a^3 / (3 sqrt(3) r^4); binary32 sums add 1e-5 of the peak.  Returns the largest error relative to its bound."""
    zc = (np.arange(n) + 0.5) * dx
    y = zc - np.float64(np.float32(z_src))
    a2 = np.maximum(r * r - y * y, 0.0)
    want = stir * (16.0 / 15.0) * r * U * (a2 / (r * r)) ** 2.5
    bound = (U * h_sub) ** 2 * stir * U * 32.0 * a2 ** 1.5 / (3.0 * np.sqrt(3.0) * r ** 4) + 1e-5 * want.max()
    xc = (np.arange(n) + 0.5) * dx
    cols = np.flatnonzero((xc > x_start + r + 1.0) & (xc < x_end - r - 1.0))
    assert len(cols) > 10
    worst = 0.0
    for i in cols:
        err = np.abs(foam[:, i].astype(np.float64) - want)
        worst = max(worst, float((err / bound).max()))
    return worst


def test_stirred_trail_follows_the_closed_form():
    n, dx, U, r, h_sub, stir = 128, 0.5, 2.0, 4.0, 0.04, 0.05
    F = wf.Layer(_params(n, dx), wf.foam_params(whitecap=0.0, grow_rate=0.0, stir_rate=stir, decay_rate=0.0))
    _trail(lambda dt, S, src: F.step(dt, S, (0, 0), src), n, dx, U, r, 32.1, 6.0, 58.0, h_sub, stir)
    assert F.foam.max() > 0.1
    assert trail_profile_check(F.foam, n, dx, U, r, 32.1, 6.0, 58.0, h_sub, stir) <= 1.0


def test_breaking_forms_foam_on_the_crests_only():
    """A single wave of 8 cells along x (|k| dx = 0.79, in the stencil's band), amplitude 0.3 m (kA = 0.24), set as h and
    h_prev one sub-step apart, with alpha = 0: after one sub-step, in the interior, foam forms exactly where beta = c / dx
    exceeds whitecap, those cells lie on crests, and their beta equals -(h_new - 2 h + h_prev) / (g h^2) within rounding."""
    n, dx, A, wc, hs = 128, 1.0, 0.3, 0.15, 0.1
    k = 2 * np.pi / (8 * dx)
    w = np.sqrt(wk.G * k)
    x = (np.arange(n) + 0.5) * dx
    F = wf.Layer(_params(n, dx), wf.foam_params(whitecap=wc, grow_rate=1.0, stir_rate=0.0, decay_rate=0.0))
    F.h = np.tile(A * np.cos(k * x), (n, 1)).astype(np.float32)
    F.h_prev = np.tile(A * np.cos(k * x + w * hs), (n, 1)).astype(np.float32)
    h0, hp0 = F.h.copy(), F.h_prev.copy()
    F.record_beta = True
    F.step(hs, 1, (0, 0))
    beta = F.betas[0]
    inner = (slice(8, n - 8), slice(8, n - 8))
    foamy = F.foam[inner] > 0
    assert np.array_equal(foamy, beta[inner] > wc)
    assert 0 < foamy.mean() < 0.5
    assert np.all(h0[inner][foamy] > 0.5 * A)                  # on the crests
    h2 = f32(hs) * f32(hs)
    est = -(F.h.astype(np.float64) - 2.0 * h0 + hp0) / (wk.G * float(h2))
    tol = 8 * EPS * (np.abs(F.h) + 2 * np.abs(h0) + np.abs(hp0)) / (wk.G * float(h2)) + 1e-5 * np.abs(beta)
    assert np.all(np.abs(est - beta)[inner][foamy] <= tol[inner][foamy])


def test_scroll_moves_foam_as_it_moves_h():
    n = 128
    F0 = np.random.default_rng(5).uniform(0, 1, (n, n)).astype(np.float32)
    F = wf.Layer(_params(n, 0.5), wf.foam_params(whitecap=0.5))      # no growth and d = exp(0) = 1: F only moves
    F.foam = F0.copy()
    F.step(0.05, 1, (3, -2))
    assert F.foam.tobytes() == wk.scroll(F0, 3, -2).tobytes()
    F.step(0.05, 1, (-4, 5))
    assert F.foam.tobytes() == wk.scroll(wk.scroll(F0, 3, -2), -7, 7).tobytes()
    F.step(0.05, 1, (-4 + n, 5))
    assert not F.foam.any()


def test_clamp_at_one_and_nan_to_zero():
    foam = np.array([[0.9, np.nan, np.inf, -np.inf, -0.5, 0.25, 0.0, -0.0]], np.float32)
    c = np.zeros_like(foam)
    c[0, 0] = 100.0
    out = wf.update(foam, c, np.zeros_like(foam), 1.0, 0.1, f32(1.0), f32(0.5), f32(0.0))
    assert out.tolist() == [[1.0, 0.0, 1.0, 0.0, 0.0, 0.25, 0.0, 0.0]]
    assert not np.signbit(out).any()                            # -0 leaves as +0
    c[0, :] = np.nan                                            # a NaN beta grows nothing
    out = wf.update(foam, c, np.zeros_like(foam), 1.0, 0.1, f32(1.0), f32(0.5), f32(0.0))
    assert out.tolist() == [[f32(0.9), 0.0, 1.0, 0.0, 0.0, 0.25, 0.0, 0.0]]
    # through a step: NaN foam goes to 0 even under growth, foam pushed over 1 stays at 1
    F = wf.Layer(_params(128, 1.0), wf.foam_params(whitecap=-1.0, grow_rate=100.0))
    F.foam[0, 0], F.foam[5, 5] = np.nan, 0.99
    F.step(0.1, 1, (0, 0))
    assert F.foam[0, 0] == 0.0 and F.foam[5, 5] == 1.0 and np.count_nonzero(F.foam == 1.0) == F.foam.size - 1
    F = wf.Layer(_params(128, 1.0), wf.foam_params(whitecap=1.0, decay_rate=1.0))
    F.foam[3, 3] = np.nan
    F.step(0.1, 1, (0, 0))
    assert F.foam[3, 3] == 0.0 and not np.signbit(F.foam).any()
