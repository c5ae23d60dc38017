"""GPU drifters (ocean_drift[_device]; ocean_drift.cu) against oracle/drifters.py bit for bit: drift, wrap, render with and
without the wake layer, NaN drifters and labels far from the origin, the device form, validation and a large batch."""
import numpy as np
import pytest

from conftest import demo_params
from oracle import drifters as od
from oracle import pyoracle as po
from test_gpu_parity import _bits_equal

pytestmark = pytest.mark.gpu

INVALID = 1   # OCEAN_ERR_INVALID_ARGUMENT


@pytest.fixture(autouse=True)
def _modes():
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    yield
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)


def _gow():
    import godotoceanwaves_b200 as gow
    return gow


def _setup(N, C):
    gow = _gow()
    params = [demo_params(gow.WaveCascadeParameters, c) for c in range(C)]
    g = gow.WaveGenerator()
    g.map_size = N
    g.init_gpu(C)
    g.update_all(0.02, params)
    return g, params


def _same(a, b):
    """bit-identical field by field, except that a NaN only has to meet a NaN (numpy keeps an input NaN's payload, the GPU
    returns the canonical one)"""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.dtype.names:
        return a.dtype == b.dtype and all(_same(a[f], b[f]) for f in a.dtype.names)
    nan = np.isnan(b)
    u = np.uint64 if a.dtype.itemsize == 8 else np.uint32
    return a.shape == b.shape and np.array_equal(np.isnan(a), nan) and np.array_equal(a[~nan].view(u), b[~nan].view(u))


def _drifters(n, seed=0, spread=400.0, center=(0.0, 0.0)):
    rng = np.random.default_rng(seed)
    d = np.zeros(n, od.DRIFTER)
    d["x"] = center[0] + rng.uniform(-spread, spread, n)
    d["z"] = center[1] + rng.uniform(-spread, spread, n)
    d["yaw"] = rng.uniform(-4, 4, n)
    d["yaw_rate"] = rng.uniform(-1, 1, n)
    d["windage"] = rng.uniform(0, 0.05, n)
    d["tilt"] = rng.uniform(0, 1, n)
    d["tilt"][::4] = 0.0
    d["offset"] = rng.uniform(-0.5, 0.5, n)
    d["scale"] = rng.uniform(0.5, 2, n)
    return d


def _expect(g, params, d, dt, p, wake=None):
    sc = g.map_scales(params)
    _, per = g.sea_state(sc)                             # the device cache's moments
    moments = [np.concatenate([np.atleast_1d(r[f]) for f in ("m_minus1", "m0", "m1", "m2", "direction", "slope", "stokes")])
               for r in per]
    disp, nrm = g.maps_to_host(0, len(params))
    return od.drift(d, dt, p, moments, disp, nrm, sc, wake=wake)


@pytest.mark.parametrize("wrap", [False, True])
@pytest.mark.parametrize("N,C", [(128, 2), (256, 4), (1024, 3)])
def test_drift_bit_exact(N, C, wrap):
    g, params = _setup(N, C)
    d = _drifters(4099, seed=N + C)
    d["x"][:5] = np.nan                                   # a NaN or infinite drifter affects only itself
    d["z"][5] = np.inf
    d["yaw"][6] = np.nan
    box = (-150.0, -80.0, 300.0, 160.0) if wrap else None
    p = g.drift_params(current=(0.3, -0.2), wind=(8.0, 3.0), stokes_scale=1.0, box=box)
    sc = g.map_scales(params)
    for dt in (1.0 / 60.0, 0.5, 0.0):
        want_d, want_i = _expect(g, params, d, dt, p)
        got_d, got_i = g.drift(d, dt, sc, p)
        assert _same(got_d, want_d), f"drifters, dt={dt}"
        assert _same(got_i, want_i), f"instances, dt={dt}"
        d = got_d
    finite = np.isfinite(d["x"]) & np.isfinite(d["z"])
    if wrap:
        assert np.all((d["x"][finite] >= -150.0) & (d["x"][finite] <= 150.0))
        assert np.all((d["z"][finite] >= -80.0) & (d["z"][finite] <= 80.0))


def test_drift_far_labels_and_device_form():
    """Labels about 1e5 m out keep millimetre steps (binary64), and the device form gives the host form's bytes."""
    import torch
    g, params = _setup(256, 3)
    d = _drifters(1000, seed=7, spread=50.0, center=(1.0e5, -1.2e5))
    p = g.drift_params(current=(0.001, 0.0), stokes_scale=0.0)
    sc = g.map_scales(params)
    want_d, want_i = _expect(g, params, d, 1.0, p)
    got_d, got_i = g.drift(d, 1.0, sc, p)
    assert _bits_equal(got_d, want_d) and _bits_equal(got_i, want_i)
    assert np.allclose(got_d["x"] - d["x"], 0.001, rtol=0, atol=1e-9)
    lib = _gow().native.load_library()
    dev = torch.from_numpy(d.view(np.uint8).copy()).cuda()
    inst = torch.zeros((len(d), 12), dtype=torch.float32, device="cuda")
    assert lib.ocean_drift_device(g.context, 1.0, p.ctypes.data, len(d), dev.data_ptr(), sc.shape[0], sc.ctypes.data, inst.data_ptr()) == 0
    g.synchronize()
    assert _bits_equal(dev.cpu().numpy().view(od.DRIFTER), want_d)
    assert _bits_equal(inst.cpu().numpy(), want_i)


def test_drift_without_sources_keeps_labels():
    g, params = _setup(128, 2)
    d = _drifters(500, seed=3)
    d["windage"] = 0.0
    p = g.drift_params(stokes_scale=0.0)
    sc = g.map_scales(params)
    got = d
    for _ in range(5):
        got, _ = g.drift(got, 0.25, sc, p, render=False)
    assert _bits_equal(got["x"], d["x"]) and _bits_equal(got["z"], d["z"])


def test_drift_reads_the_wake():
    """With READ_WAKE the render adds the wake's h and slopes (bit for bit); without it the bytes are those of a generator
    without a layer, and either way the call launches one kernel."""
    g, params = _setup(256, 2)
    g.wake_init(256, cell_size=0.5)
    src = np.zeros(1, g.WAKE_SOURCE)
    src[0] = (30.0, 30.0, 4.0, 0.0, 3.0, 0.4, -1)           # inside the window [0, 128)^2
    g.wake_step(0.05, 4, sources=src)
    g.synchronize()
    h, _, origin = g.wake_state()
    d = _drifters(3000, seed=11, spread=25.0, center=(30.0, 30.0))
    sc = g.map_scales(params)
    for read in (False, True):
        p = g.drift_params(read_wake=read)
        want_d, want_i = _expect(g, params, d, 0.0, p, wake=(h, 0.5, origin))
        g.sea_state(sc)
        n0 = g.info().kernel_launches
        got_d, got_i = g.drift(d, 0.0, sc, p)
        assert g.info().kernel_launches - n0 == 1
        assert _bits_equal(got_i, want_i), f"read_wake={read}"
    plain = g.drift(d, 0.0, sc, g.drift_params())[1]
    assert not _bits_equal(plain, got_i)                 # the wake moved some drifters


def test_drift_validation():
    g, params = _setup(128, 2)
    lib = _gow().native.load_library()
    sc = g.map_scales(params)
    d = _drifters(10)
    d0 = d.copy()
    inst = np.zeros((10, 12), np.float32)
    n0 = g.info().kernel_launches

    def call(dt=0.1, p=None, n=10, arr=d, nc=2, scales=sc):
        p = g.drift_params() if p is None else p
        return lib.ocean_drift(g.context, dt, p.ctypes.data, n, None if arr is None else arr.ctypes.data, nc,
                               None if scales is None else scales.ctypes.data, inst.ctypes.data)

    assert call(dt=-1.0) == INVALID
    assert call(dt=float("nan")) == INVALID
    assert call(dt=float("inf")) == INVALID
    for field, value in (("current", (np.nan, 0)), ("wind", (0, np.inf)), ("stokes_scale", np.nan), ("box", (0, 0, np.nan, 1))):
        p = g.drift_params()
        p[field] = value
        assert call(p=p) == INVALID, field
    assert call(p=g.drift_params(box=(0, 0, 0, 10))) == INVALID
    assert call(p=g.drift_params(box=(0, 0, 10, -1))) == INVALID
    p = g.drift_params()
    p["flags"] = 4
    assert call(p=p) == INVALID
    assert lib.ocean_drift(g.context, 0.1, None, 10, d.ctypes.data, 2, sc.ctypes.data, None) == INVALID
    assert call(nc=0) == INVALID and call(nc=3) == INVALID
    assert call(scales=None) == INVALID
    assert call(n=-1) == INVALID and call(arr=None) == INVALID
    assert g.info().kernel_launches == n0 and _bits_equal(d, d0)
    assert call(n=0, arr=None) == 0


def test_drift_large_batch():
    """2^20 drifters at N = 1024, C = 8 against the specification."""
    g, params = _setup(1024, 8)
    d = _drifters(1 << 20, seed=5, spread=2000.0)
    p = g.drift_params(current=(0.1, 0.1), wind=(5.0, -5.0), box=(-1000.0, -1000.0, 2000.0, 2000.0))
    want_d, want_i = _expect(g, params, d, 1.0 / 30.0, p)
    got_d, got_i = g.drift(d, 1.0 / 30.0, g.map_scales(params), p)
    assert _bits_equal(got_d, want_d) and _bits_equal(got_i, want_i)


def test_drift_refreshes_stale_sea_state_itself():
    """A drift call with dt > 0 brings stale cascades up to date on its own (2 kernels, then the drift kernel): after a
    regenerated and an injected spectrum, with no sea-state call in between, the labels move with the new Stokes drift.
    With nothing stale it launches the drift kernel alone."""
    from oracle import sea_state as ss
    g, params = _setup(256, 3)
    sc = g.map_scales(params)
    d = _drifters(2048, seed=13)
    p = g.drift_params(current=(0.2, 0.0), wind=(4.0, 1.0), stokes_scale=1.0)
    n0 = g.info().kernel_launches
    d, _ = g.drift(d, 1.0 / 60.0, sc, p)
    assert g.info().kernel_launches - n0 == 3             # first use: every cascade is stale
    params[1].wind_speed = 9.0
    params[1].should_generate_spectrum = True
    g.update_all(0.02, params)
    rng = np.random.default_rng(2)
    g.set_spectrum_amplitudes(2, (rng.normal(size=(256, 256)) * 0.05 + 1j * rng.normal(size=(256, 256)) * 0.05).astype(np.complex64))
    n1 = g.info().kernel_launches
    got_d, got_i = g.drift(d, 0.5, sc, p)
    assert g.info().kernel_launches - n1 == 3
    moments = [ss.cascade_moments(g.spectrum_to_host(c), params[c].tile_length) for c in range(3)]
    disp, nrm = g.maps_to_host(0, 3)
    want_d, want_i = od.drift(d, 0.5, p, moments, disp, nrm, sc)
    assert _bits_equal(got_d, want_d) and _bits_equal(got_i, want_i)
    n2 = g.info().kernel_launches
    g.drift(got_d, 0.5, sc, p)
    assert g.info().kernel_launches - n2 == 1
