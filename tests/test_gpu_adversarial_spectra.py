"""The update path against the CPU oracle on injected spectra, bit for bit, in the regimes the generated spectra never reach.

Every other parity test feeds the update kernels spectra that spectrum_compute makes from cascade parameters: smooth, dense,
of moderate size.  Here ocean_set_spectrum_amplitudes injects the spectrum of each cascade, the texture the GPU stores is
checked bit for bit (signed zeros included) against the host construction (A(id), conj A(mod(-id, N))), and the oracle runs
on exactly those bits (should_generate_spectrum = False).  Families, one cascade per case in one generator, at every N:

  * a magnitude ladder: one dense seeded spectrum scaled by powers of two, each rung asserted (from the oracle's own buffers)
    to reach its regime -- binary32 subnormals and exact underflow, gradient numerators straddling 2^-100 inside one
    thread's sixteen texels, half subnormals and half flush to +-0, half overflow beside finite binary32 maps, |dhx_dx| and
    |dhz_dz| above 2^20 and above 2^126, numerators above 2^100, binary32 overflow inside the FFT;
  * mixed magnitudes: a demo-sized spectrum with texels at 2^-60 and one wave whose slopes cross the fast path's 2^20 bound
    inside single threads, foam driven into both clamps;
  * structured sparse spectra: single texels at DC, on the axes, on the Nyquist row and column, in the self-mirrored rows,
    in column 0; one full row, one full column; Hermitian and anti-Hermitian spectra at t = 0 (h exactly 2 A resp. exactly
    zero); each case asserted to reach its structure, most of them with exact zeros of both signs in the maps;
  * the reference's own log(0) hazard through spectrum_compute: a seed solved in closed form so that the hash of one texel
    is 0 or 1 (u0 = 0), beside a normal cascade, then a clean seed.

Paths: the production persistent kernel without taps (k_update_persistent<N, false>), the taps kernel (binary32 maps and the
row pass compared too), and the two-kernel pipeline (profiling on); fused frames (ocean_update_frames) carry the
foam plane through the ladder and the mixed spectrum.

Comparison rule: equal bits wherever the oracle's value is not NaN, signed zeros included, NaN exactly where the oracle's
is; foam bit for bit everywhere.  Two exceptions, each stated where it is used: the row pass is compared up to the sign of
exact zeros, and one texel of dhx_dx may hold a zero of the other sign for two sparse spectra (KNOWN_ZERO_SIGN)."""
import math

import numpy as np
import pytest

from conftest import demo_params
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu

SIZES = [128, 256, 512, 1024]
PATHS = ["persistent", "taps", "split"]


@pytest.fixture(autouse=True)
def _modes():
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    yield
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)


def assert_match(got, ref, what, overflow=False, zero_sign=True, allow=None):
    """Equal bits where ref is not NaN -- signed zeros included -- and NaN exactly where ref is NaN (float16 or float32).
    zero_sign=False: a zero may have either sign (the row pass: its butterflies round -(a + b) where the reference rounds
    (-a) + (-b), and skip the product by (1, 0), so a zero sum can come out with the other sign).
    allow: texels where a zero may have either sign (KNOWN_ZERO_SIGN: the one map texel where such a zero survives).
    overflow: a binary32 intermediate overflowed, after which the unit-twiddle skip passes inf or finite values where the
    reference makes NaN (inf * 0); then values are compared where the oracle's are finite (callers check the non-finite
    texels of the half maps separately)."""
    got = np.ascontiguousarray(got)
    ref = np.ascontiguousarray(ref)
    assert got.shape == ref.shape and got.dtype == ref.dtype, what
    ui = np.uint16 if ref.dtype == np.float16 else np.uint32
    nan = ~np.isfinite(ref) if overflow else np.isnan(ref)
    differ = ~nan & (got.view(ui) != ref.view(ui))
    zeros = (got == 0) & (ref == 0)
    if not zero_sign:
        differ &= ~zeros
    elif allow is not None:
        differ &= ~(zeros & allow)
    bad = differ | (False if overflow else (np.isnan(got) != nan))
    if bad.any():
        idx = np.argwhere(bad)[:4]
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} differ, first at {idx.tolist()}: "
                             f"gpu {[got[tuple(i)] for i in idx]}, oracle {[ref[tuple(i)] for i in idx]}")


# ---- spectra ---------------------------------------------------------------------------------------------------------
def _dense(N, seed=5):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((N, N)) + 1j * rng.standard_normal((N, N))


def _scaled(a, e):
    """a * 2^e rounded once to complex64 (binary64 product: exact, then one rounding, subnormals included)"""
    return (np.asarray(a, np.complex128) * 2.0 ** e).astype(np.complex64)


# rung -> (exponent at N = 256, exponent change per doubling of N): the displacement grows like N (random walk over N^2
# texels), the gradients and slopes like N^2 (|k| grows with N too)
LADDER = {"underflow": (-146, 1), "straddle_2m100": (-110, 2), "half_flush": (-35, 1), "half_subnormal": (-22, 1),
          "half_overflow": (10, 1), "slope_2p20": (20, 2), "numerator_2p100": (90, 2), "slope_2p126": (114, 2),
          "f32_overflow": (120, 1)}


def ladder_cases(N):
    base = _dense(N)
    doublings = int(math.log2(N)) - 8
    return [(name, _scaled(base, e - k * doublings), {}) for name, (e, k) in LADDER.items()]


def mixed_cases(N):
    """demo-sized amplitudes (~1e-2), a few texels at 2^-60, and one wave at k = (3, 3) dk whose slope |dhx_dx| peaks at
    2^21 (|A| kvy^2 / |k| with tile 88 m): every texel of the map carries it, so |dhx_dx| and |dhz_dz| cross the fast path's
    2^20 bound between the sixteen texels of one column-pass thread, which then mix fast-path and fixed-up quotients.  A
    whitecap of 1 and a large foam amount drive foam to both clamps (1 where the Jacobian dips, 0 where it does not).  (A
    texel at 2^60 would not mix: a single texel reaches every output, so it puts every quotient out of range.)"""
    rng = np.random.default_rng(17)
    a = (_dense(N, 6) * 1e-2).astype(np.complex64)
    for _ in range(4):
        y, x = rng.integers(0, N, 2)
        a[y, x] = np.complex64(complex(rng.standard_normal(), rng.standard_normal()) * 2.0 ** -60)
    dk = 2 * math.pi / 88.0
    kvy, k = 3 * dk, math.hypot(3 * dk, 3 * dk)
    a[N // 2 + 3, N // 2 + 3] = np.complex64((0.8 + 0.6j) * 2.0 ** 21 * k / (kvy * kvy))
    return [("mixed", a, dict(whitecap=1.0, foam_amount=1000.0))]


def _single(N, y, x, v=1.5 - 0.75j):
    a = np.zeros((N, N), np.complex64)
    a[y, x] = v
    return a


def sparse_cases(N):
    h = N // 2
    rng = np.random.default_rng(23)
    cases = [("dc", _single(N, h, h), {}),
             ("axis_kx0", _single(N, h + 3, h), {}), ("axis_ky0", _single(N, h, h - 5), {}),
             ("nyquist_row", _single(N, 0, h + 7), {}), ("nyquist_col", _single(N, h - 9, 0), {}),
             ("row0_col0", _single(N, 0, 0), {}),
             ("row_half", _single(N, h, 11), {}), ("col0", _single(N, 13, 0), {})]
    row = np.zeros((N, N), np.complex64)
    row[h + 2] = (rng.standard_normal(N) + 1j * rng.standard_normal(N)).astype(np.complex64)
    col = np.zeros((N, N), np.complex64)
    col[:, 5] = (rng.standard_normal(N) + 1j * rng.standard_normal(N)).astype(np.complex64)
    cases += [("full_row", row, {}), ("full_col", col, {})]
    # A(mod(-id, N)) = conj A(id) (Hermitian) or -conj A(id) (anti-Hermitian): at t = 0 the packed h = A(id) + conj A(-id)
    # is then exactly 2 A resp. exactly zero everywhere (zeros of both signs)
    d = _dense(N, 29).astype(np.complex64)
    m = np.roll(d[::-1, ::-1], 1, axis=(0, 1))
    herm = ((d + np.conj(m)) * 0.5).astype(np.complex64)
    anti = ((d - np.conj(m)) * 0.5).astype(np.complex64)
    # time -0.02: the family's one update of 0.02 runs them at t = 0 exactly
    cases += [("hermitian_t0", herm, dict(time=-0.02)), ("antihermitian_t0", anti, dict(time=-0.02))]
    return cases


# ---- runs ------------------------------------------------------------------------------------------------------------
def _params(cls, over):
    return demo_params(cls, 0, **over)


_ORACLE = {}


def oracle_run(family, N, cases, deltas, frames):
    """the oracle's buffers after the updates of `deltas`, and after `frames` more updates of 0.02 (cached for the paths of
    one family and N, which run one after another)"""
    key = (family, N)
    if key in _ORACLE:
        return _ORACLE[key]
    _ORACLE.clear()                 # one (family, N) at a time: a 1024^2 family holds gigabytes of oracle buffers
    C = len(cases)
    o = po.OracleWaveGenerator(N)
    o.init_gpu(max(2, C))
    pc = []
    for c, (_, a, over) in enumerate(cases):
        o.set_spectrum(c, po.spectrum_texture(a))
        p = _params(po.CascadeParams, over)
        p.should_generate_spectrum = False
        pc.append(p)
    snaps = []
    steps = list(deltas) + [0.02] * frames
    for i, delta in enumerate(steps):
        o.update_all(delta, pc)
        if i == len(deltas) - 1 or i == len(steps) - 1:
            snaps.append(dict(disp=o.displacement_half()[:C].copy(), norm=o.normal_half()[:C].copy(),
                              d32=o.displacement_f32[:C].copy(), n32=o.normal_f32[:C].copy(),
                              rp=np.ascontiguousarray(np.swapaxes(o.fft_buffer[:C, 0], 2, 3)), h1=o.fft_buffer[:C, 1].copy()))
    _ORACLE[key] = snaps
    return snaps


def gpu_run(N, cases, deltas, frames, path):
    import godotoceanwaves_b200 as gow
    C = len(cases)
    g = gow.WaveGenerator()
    g.map_size = N
    g.init_gpu(max(2, C))
    if path == "split":
        g.set_profiling(True)
    if path == "taps":
        g.enable_f32_taps(True)
    pg = [_params(gow.WaveCascadeParameters, over) for _, _, over in cases]
    g.update_all(0.0, pg)                                      # spectrum and tables; delta 0 leaves time and foam (0) alone
    for c, (name, a, _) in enumerate(cases):
        g.set_spectrum_amplitudes(c, a)
        g.set_foam_state(c, np.zeros((N, N), np.float16))
        tex = g.spectrum_to_host(c)
        assert np.array_equal(tex.view(np.uint32), po.spectrum_texture(a).view(np.uint32)), f"stored spectrum of {name}"
    snaps = []
    for delta in deltas:
        g.update_all(delta, pg)
    snaps.append(_gpu_snapshot(g, C, path))
    if frames:
        g.update_frames(0.02, pg, frames)
        snaps.append(_gpu_snapshot(g, C, path))
    g.free()
    return snaps


def _gpu_snapshot(g, C, path):
    d16, n16 = g.maps_to_host(0, C)
    s = dict(disp=d16, norm=n16)
    if path == "taps":
        f = [g.f32_maps_to_host(c) for c in range(C)]
        s["d32"] = np.stack([x[0] for x in f])
        s["n32"] = np.stack([x[1] for x in f])
        s["rp"] = np.stack([g.rowpass_to_host(c) for c in range(C)])
    return s


OVERFLOWING = {"f32_overflow"}      # cases with a binary32 overflow inside the FFT (see assert_match)

# The only map texels where the sign of a zero differs from the oracle's: dhx_dx (normal channel 2) at row N-1, column N-2,
# for spectra whose dhx_dx layer is exactly zero everywhere after modulation (a single DC texel; anti-Hermitian at t = 0).
# The CUDA value is +0 and the oracle's -0: the column pass's u - p for the reference's u + l*(-tw) (fft_core.cuh).
KNOWN_ZERO_SIGN = {"dc", "antihermitian_t0"}


def _allowed(name, N, shape):
    m = np.zeros(shape, bool)
    if name in KNOWN_ZERO_SIGN:
        m[N - 1, N - 2, 2] = True
    return m


def compare(family, N, cases, deltas, frames, path):
    ref = oracle_run(family, N, cases, deltas, frames)
    got = gpu_run(N, cases, deltas, frames if path == "persistent" else 0, path)
    for k, s in enumerate(got):
        r = ref[k]
        for c, (name, _, _) in enumerate(cases):
            tag = f"{family} {name} N={N} {path} snapshot {k}"
            ov = name in OVERFLOWING
            allow = _allowed(name, N, (N, N, 4))
            assert_match(s["disp"][c], r["disp"][c], "displacement " + tag, ov)
            assert_match(s["norm"][c][..., :3], r["norm"][c][..., :3], "normal " + tag, ov, allow=allow[..., :3])
            if ov:
                assert np.array_equal(np.isfinite(s["disp"][c]), np.isfinite(r["disp"][c])), "non-finite displacement " + tag
                assert np.array_equal(np.isfinite(s["norm"][c]), np.isfinite(r["norm"][c])), "non-finite normal " + tag
            assert np.array_equal(s["norm"][c][..., 3].view(np.uint16), r["norm"][c][..., 3].view(np.uint16)), "foam " + tag
            if "d32" in s:
                assert_match(s["d32"][c], r["d32"][c], "binary32 displacement " + tag, ov)
                assert_match(s["n32"][c], r["n32"][c], "binary32 normal " + tag, ov, allow=allow)
                assert_match(s["rp"][c], r["rp"][c], "row pass " + tag, ov, zero_sign=False)
    return ref


# ---- regime assertions (the oracle's own buffers) ----------------------------------------------------------------------
TINY = np.float32(np.finfo(np.float32).tiny)


def _numerators(h1):
    """|dhy_dx|, |dhy_dz| before the sign shift: layer 1 imaginary and layer 2 real of the column-pass output"""
    return np.abs(np.stack([h1[1, ..., 1], h1[2, ..., 0]]))


def _denominator_terms(h1):
    """|dhx_dx|, |dhz_dz|: layer 2 imaginary and layer 3 real"""
    return np.abs(np.stack([h1[2, ..., 1], h1[3, ..., 0]]))


def _thread_groups(a, N):
    """a[..., y, x] regrouped as [..., y, t, 16]: the sixteen texels one column-pass thread writes are row y, x = t mod N/16"""
    return np.swapaxes(a.reshape(*a.shape[:-1], 16, N // 16), -1, -2)


def assert_ladder_regimes(N, snap):
    names = list(LADDER)
    with np.errstate(all="ignore"):
        for c, name in enumerate(names):
            h1, rp = snap["h1"][c], snap["rp"][c]
            d32, n32 = snap["d32"][c], snap["n32"][c]
            dh, nh = snap["disp"][c].astype(np.float32), snap["norm"][c].astype(np.float32)
            num, den = _numerators(h1), _denominator_terms(h1)
            fin = np.isfinite
            if name == "underflow":
                assert ((np.abs(rp) < TINY) & (rp != 0)).any() and (rp == 0).any(), name        # subnormals and exact zeros
                assert ((np.abs(d32) < TINY) & (d32 != 0)).any(), name
            elif name == "straddle_2m100":
                g = _thread_groups(num, N)
                mixed = (g < 2.0 ** -100).any(-1) & (g >= 2.0 ** -100).any(-1)
                assert mixed.any() and (num < 2.0 ** -100).any() and (num >= 2.0 ** -100).any(), name
            elif name == "half_flush":
                flushed = (d32[..., :3] != 0) & (dh[..., :3] == 0)
                assert flushed.mean() > 0.5 and np.signbit(dh[..., :3][flushed]).any() and (~np.signbit(dh[..., :3][flushed])).any(), name
            elif name == "half_subnormal":
                assert ((np.abs(dh[..., :3]) < 2.0 ** -14) & (dh[..., :3] != 0)).any(), name
            elif name == "half_overflow":
                assert fin(d32).all() and fin(n32).all() and np.isinf(dh).any() and np.isinf(nh).any(), name
            elif name == "slope_2p20":
                assert fin(n32).all() and (den > 2.0 ** 20).any(), name
            elif name == "numerator_2p100":
                assert fin(num).all() and (num > 2.0 ** 100).any(), name
            elif name == "slope_2p126":
                assert (den[fin(den)] > 2.0 ** 126).any(), name                                   # rcp.approx.ftz would flush
            elif name == "f32_overflow":
                assert (~fin(rp)).any() and np.isnan(n32).any(), name                             # inf inside the FFT


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("N", SIZES)
def test_magnitude_ladder(N, path):
    cases = ladder_cases(N)
    ref = compare("ladder", N, cases, (0.02,), 3, path)
    assert_ladder_regimes(N, ref[0])


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("N", SIZES)
def test_mixed_magnitudes(N, path):
    cases = mixed_cases(N)
    ref = compare("mixed", N, cases, (0.02, 0.02), 3, path)
    h1 = ref[0]["h1"][0]
    out = (_denominator_terms(h1) > 2.0 ** 20).any(0) | (_numerators(h1) < 2.0 ** -100).any(0)
    g = _thread_groups(out, N)
    assert (g.any(-1) & ~g.all(-1)).any()                                                  # threads that mix both
    foam = ref[-1]["norm"][0][..., 3].astype(np.float32)
    assert (foam == 1).any() and (foam == 0).any()                                        # both clamps


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("N", SIZES)
def test_structured_sparse_spectra(N, path):
    cases = sparse_cases(N)
    ref = compare("sparse", N, cases, (0.02,), 0, path)
    assert_sparse_regimes(N, cases, ref[0])


def _both_zero_signs(a):
    """every value an exact zero, and zeros of both signs among them"""
    return bool((a == 0).all() and np.signbit(a).any() and (~np.signbit(a)).any())


def _has_both_zeros(a):
    """exact zeros of both signs among the values"""
    z = a[a == 0]
    return bool(np.signbit(z).any() and (~np.signbit(z)).any())


def assert_sparse_regimes(N, cases, snap):
    """Each sparse case reaches the structure it is meant to, read from the texture and from the oracle's maps.  Channels:
    displacement (hx, hy, hz, 0), normal (gx = dhy_dx / (1 + |dhx_dx|), gy = dhy_dz / (1 + |dhz_dz|), dhx_dx, foam)."""
    h = N // 2
    for c, (name, a, _) in enumerate(cases):
        tex = po.spectrum_texture(a)
        nz = np.argwhere((tex != 0).any(-1))
        rows, cols = set(nz[:, 0].tolist()), set(nz[:, 1].tolist())
        d32, n32 = snap["d32"][c], snap["n32"][c]
        dh, nh = snap["disp"][c], snap["norm"][c]
        some_zeros = _has_both_zeros(dh[..., :3]) and _has_both_zeros(nh[..., :3])
        if name == "dc":               # k = 0: every term with a component of k is a zero (signed); only the height remains
            assert rows == cols == {h} and (d32[..., 1] != 0).all() and (n32[..., :3] == 0).all(), name
            for a_ in (dh[..., 0], dh[..., 2], nh[..., 0], nh[..., 1], nh[..., 2]):
                assert _both_zero_signs(a_), name
        elif name in ("axis_kx0", "axis_ky0"):      # on an axis: exact zeros of both signs wherever the wave has a node
            assert (cols if name == "axis_kx0" else rows) == {h} and some_zeros, name
        elif name in ("nyquist_row", "row_half"):   # texel and its mirror in the same (self-mirrored) row
            assert len(nz) == 2 and rows == ({0} if name == "nyquist_row" else {h}) and some_zeros, name
            if name == "nyquist_row":
                assert _both_zero_signs(dh[..., 0]), name
        elif name in ("nyquist_col", "col0"):       # the mirror partner of a column-0 texel is in column 0 too
            assert len(nz) == 2 and cols == {0} and some_zeros, name
        elif name == "row0_col0":      # the self-mirrored texel (0, 0) holds A and conj A of itself
            assert nz.tolist() == [[0, 0]] and tex[0, 0, 2] == tex[0, 0, 0] and tex[0, 0, 3] == -tex[0, 0, 1], name
            assert _both_zero_signs(dh[..., 0]) and _both_zero_signs(nh[..., 1]), name
        elif name == "full_row":
            assert rows == {h + 2, h - 2} and len(nz) == 2 * N, name
        elif name == "full_col":
            assert cols == {5, N - 5} and len(nz) == 2 * N, name
        elif name == "hermitian_t0":   # conj A(-k) == A(k) (as values: a self-mirrored texel's imaginary zero flips sign): h = 2 A
            assert np.array_equal(tex[..., 2:4], tex[..., 0:2]), name
        elif name == "antihermitian_t0":   # conj A(-k) == -A(k) bit for bit: at t = 0 h is a zero, every map a signed zero
            assert np.array_equal(tex[..., 2:4], -tex[..., 0:2]), name
            for ch in range(3):
                assert _both_zero_signs(dh[..., ch]) and _both_zero_signs(nh[..., ch]), (name, ch)


@pytest.mark.parametrize("N", SIZES)
@pytest.mark.parametrize("n", [0, 1])
def test_log_of_zero_hazard_through_spectrum_compute(N, n):
    """A seed that makes the hash of texel (N/2 + 3, N/2 + 5) exactly n (u0 = 0): gaussian() takes log(0), so h0 there is
    (inf, NaN) for n = 0 and (inf, inf) for n = 1.  Generated on the GPU beside a normal cascade: the normal cascade stays
    bit-identical, the hazard cascade's spectrum and foam are bit-identical (foam is finite on both sides), its other fields
    have the oracle's non-finite texels and its values elsewhere.  A clean seed then makes the next frames bit-identical again."""
    import godotoceanwaves_b200 as gow
    idx, idy = N // 2 + 3, N // 2 + 5
    seed = po.hash_seed_for(idx, idy, n)
    over = dict(spectrum_seed=seed)
    pg = [demo_params(gow.WaveCascadeParameters, 0, **over), demo_params(gow.WaveCascadeParameters, 1)]
    pc = [demo_params(po.CascadeParams, 0, **over), demo_params(po.CascadeParams, 1)]
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(2)
    o = po.OracleWaveGenerator(N)
    for delta in (0.02, 0.02):
        g.update_all(delta, pg)
        o.update_all(delta, pc)
    sp = g.spectrum_to_host(0)
    assert np.isinf(o.spectrum[0, idy, idx, 0]) and (np.isnan if n == 0 else np.isinf)(o.spectrum[0, idy, idx, 1])
    assert np.array_equal(sp.view(np.uint32)[np.isfinite(o.spectrum[0])], o.spectrum[0].view(np.uint32)[np.isfinite(o.spectrum[0])])
    assert np.array_equal(np.isnan(sp), np.isnan(o.spectrum[0])) and np.array_equal(np.isinf(sp), np.isinf(o.spectrum[0]))
    d16, n16 = g.maps_to_host(0, 2)
    od, on = o.displacement_half(), o.normal_half()
    assert np.array_equal(d16[1].view(np.uint16), od[1].view(np.uint16)) and np.array_equal(n16[1].view(np.uint16), on[1].view(np.uint16))
    assert np.array_equal(n16[0][..., 3].view(np.uint16), on[0][..., 3].view(np.uint16))           # foam
    assert not np.isfinite(od[0][..., :3]).all()
    assert_match(d16[0], od[0], "displacement of the hazard cascade", overflow=True)
    assert_match(n16[0], on[0], "normal of the hazard cascade", overflow=True)
    assert np.array_equal(np.isfinite(d16[0]), np.isfinite(od[0])) and np.array_equal(np.isfinite(n16[0]), np.isfinite(on[0]))
    # a clean seed: the spectrum is regenerated and the next frames agree bit for bit again
    pg[0].spectrum_seed = (7, 9)
    pc[0].spectrum_seed = (7, 9)
    pg[0].should_generate_spectrum = pc[0].should_generate_spectrum = True
    for delta in (0.02, 0.02):
        g.update_all(delta, pg)
        o.update_all(delta, pc)
    d16, n16 = g.maps_to_host(0, 2)
    assert np.array_equal(d16.view(np.uint16), o.displacement_map[:2]) and np.array_equal(n16.view(np.uint16), o.normal_map[:2])
    g.free()
