"""GPU parity of the map-query op (ocean_sample_maps; water.gdshader:27-39,42-84) against oracle/sampling.py on the
generator's own RGBA16F maps: bit-identical binary32 results."""
import numpy as np
import pytest

from conftest import EDGE_CASES, demo_params
from oracle import sampling as sp

pytestmark = pytest.mark.gpu


def _gen(N, C, frames=2):
    import godotoceanwaves_b200 as gow
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(max(2, C))
    params = [demo_params(gow.WaveCascadeParameters, c) for c in range(C)]
    for _ in range(frames):
        g.update_all(1.0 / 50.0, params)
    return gow, g, params


def _points(n, seed, span):
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-span, span, (n, 2)).astype(np.float32)
    # texel centres, texel edges, the origin, whole tiles away: the corners of the addressing logic
    pts[:8] = np.array([[0, 0], [0.34375, 0.34375], [88.0, -88.0], [-0.0, 57.0], [1e-30, -1e-30], [16.0, 16.0], [-1234.5, 987.25],
                        [4096.0, -4096.0]], np.float32)
    return pts


def _aniso_gen(frames=2):
    """256^2 maps of cascades with non-square tiles, so that min(s.x, s.y) is the x scale for some cascades and the y
    scale for others, and signed scales: returns (gow, generator, map_scales).
      cascade 0: the anisotropic_tile corner, 93 x 41 m  ppm = 256/93  -> t = min(1, 0.1 ppm) = 0.275
      cascade 1: the axes the other way round, 41 x 93    ppm = 256/93  -> t = 0.275, displacement scale < 0
      cascade 2: 16 x 9 m                                 ppm = 256/16  -> t = 1,     normal scale < 0
      cascade 3: 30 x 70 m                                ppm = 256/70  -> t = 0.366"""
    import godotoceanwaves_b200 as gow
    N, C = 256, 4
    tiles = [EDGE_CASES["anisotropic_tile"]["tile_length"], (41.0, 93.0), (16.0, 9.0), (30.0, 70.0)]
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(C)
    params = [demo_params(gow.WaveCascadeParameters, c, tile_length=tiles[c]) for c in range(C)]
    for _ in range(frames):
        g.update_all(1.0 / 50.0, params)
    scales = gow.WaveGenerator.map_scales(params)
    scales[:, 2] = [1.0, -0.75, 0.5, 1.0]
    scales[:, 3] = [1.0, 1.0, -0.25, 0.5]
    ppm = N * np.minimum(scales[:, 0], scales[:, 1])
    assert np.any(ppm * 0.1 < 1) and np.any(ppm * 0.1 >= 1)
    assert np.any(scales[:, 0] < scales[:, 1]) and np.any(scales[:, 0] > scales[:, 1])
    return gow, g, scales


# coordinates where the float32 -> texel index conversion leaves the usual range: integer spacing (2^23, 2^24), beyond
# int32 (2^31, 2^40), beyond int64 once multiplied by N/tile (1e19, 1e20), u*N overflowing to inf (3e38), and non-finite
EXTREMES = [v for a in (2.0 ** 23, 2.0 ** 24, 2.0 ** 31, 2.0 ** 40, 1e19, 1e20, 3e38, np.inf) for v in (a, -a)] + [np.nan]


def _extreme_points(n, seed):
    """n ordinary points (_points) with every EXTREMES value placed in x, in z and in both, at random rows.
    Returns (points, mask of the rows that hold an extreme value)."""
    pts = _points(n, seed, 300.0)
    rng = np.random.default_rng(seed)
    rows = rng.choice(np.arange(8, n), 3 * len(EXTREMES), replace=False)
    for k, v in enumerate(EXTREMES):
        r = rows[3 * k:3 * k + 3]
        pts[r[0], 0] = v
        pts[r[1], 1] = v
        pts[r[2]] = v
    mask = np.zeros(n, bool)
    mask[rows] = True
    return pts, mask


def _same_or_both_nan(a, b):
    """bit-identical, except that a NaN only has to meet a NaN: numpy keeps the payload of an input NaN, the GPU returns
    the canonical one"""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    nan = np.isnan(b)
    return a.shape == b.shape and np.array_equal(np.isnan(a), nan) and np.array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32))


@pytest.mark.parametrize("N,C", [(128, 3), (256, 4), (512, 2), (1024, 2)])
def test_sample_maps_bit_exact(N, C):
    gow, g, params = _gen(N, C)
    d16, n16 = g.maps_to_host(0, C)
    scales = gow.WaveGenerator.map_scales(params)
    scales[:, 2] = [1.0, 0.75, 0.0, 0.5][:C]                   # displacement scales of main.tscn:43-83 (+ one more)
    scales[:, 3] = [1.0, 1.0, 0.25, 0.5][:C]
    pts = _points(20000, 11 + N, 300.0)
    d, gr = g.sample(pts, scales)
    d_ref, g_ref = sp.sample_maps(d16, n16, pts, scales)
    assert np.array_equal(d.view(np.uint32), d_ref.view(np.uint32))
    assert np.array_equal(gr.view(np.uint32), g_ref.view(np.uint32))
    # fewer cascades = a prefix sum
    d1, g1 = g.sample(pts[:1000], scales[:1])
    d1_ref, g1_ref = sp.sample_maps(d16[:1], n16[:1], pts[:1000], scales[:1])
    assert np.array_equal(d1.view(np.uint32), d1_ref.view(np.uint32)) and np.array_equal(g1.view(np.uint32), g1_ref.view(np.uint32))
    g.free()


def test_sample_maps_texel_centres_return_the_texels():
    gow, g, params = _gen(128, 2)
    d16, n16 = g.maps_to_host(0, 2)
    N = 128
    L = np.float32(64.0)                                        # dyadic tile: u = x/L is exact
    xs, ys = np.meshgrid(np.arange(N), np.arange(N))
    pts = np.stack([(xs.ravel() + 0.5) * (L / N), (ys.ravel() + 0.5) * (L / N)], 1).astype(np.float32)
    scales = np.array([[1 / L, 1 / L, 1.0, 1.0]], np.float32)
    d, gr = g.sample(pts, scales)
    assert np.array_equal(d, d16[0].astype(np.float32).reshape(-1, 4)[:, :3])
    # ppm = 128/64 = 2 -> t = 0.2: mostly bicubic, so only the oracle comparison applies to the gradient
    _, g_ref = sp.sample_maps(d16[:1], n16[:1], pts, scales)
    assert np.array_equal(gr.view(np.uint32), g_ref.view(np.uint32))
    g.free()


def test_sample_maps_anisotropic_signed_scales():
    gow, g, scales = _aniso_gen()
    d16, n16 = g.maps_to_host(0, 4)
    pts = _points(20000, 31, 300.0)
    d, gr = g.sample(pts, scales)
    d_ref, g_ref = sp.sample_maps(d16, n16, pts, scales)
    assert np.array_equal(d.view(np.uint32), d_ref.view(np.uint32))
    assert np.array_equal(gr.view(np.uint32), g_ref.view(np.uint32))
    g.free()


def test_sample_maps_extreme_coordinates():
    """Huge, overflowing and non-finite coordinates: finite queries are bit-identical to the specification (NaN where
    u*N overflows), non-finite ones give NaN in every field, and no query changes another's result."""
    gow, g, params = _gen(256, 4)
    d16, n16 = g.maps_to_host(0, 4)
    scales = gow.WaveGenerator.map_scales(params)
    pts, mask = _extreme_points(4000, 41)
    d, gr = g.sample(pts, scales)
    with np.errstate(all="ignore"):
        d_ref, g_ref = sp.sample_maps(d16, n16, pts, scales)
    assert _same_or_both_nan(d, d_ref) and _same_or_both_nan(gr, g_ref)
    bad = ~np.isfinite(pts).all(1)
    assert np.isnan(d[bad]).all() and np.isnan(gr[bad]).all()
    d_ord, g_ord = g.sample(pts[~mask], scales)
    assert np.array_equal(d[~mask].view(np.uint32), d_ord.view(np.uint32)) and np.array_equal(gr[~mask].view(np.uint32), g_ord.view(np.uint32))
    g.free()


def test_sample_maps_device_equals_host():
    import torch
    from godotoceanwaves_b200.native import check, load_library
    gow, g, params = _gen(256, 4)
    scales = gow.WaveGenerator.map_scales(params)
    pts = _points(50000, 12, 300.0)
    d_host, g_host = g.sample(pts, scales)
    dev = torch.device("cuda", g.device)
    pts_d = torch.from_numpy(pts).to(dev)
    d_d = torch.zeros(pts.shape[0] * 3, dtype=torch.float32, device=dev)
    g_d = torch.zeros(pts.shape[0] * 3, dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    check(load_library().ocean_sample_maps_device(g.context, pts.shape[0], pts_d.data_ptr(), 4, scales.ctypes.data, d_d.data_ptr(), g_d.data_ptr()))
    g.synchronize()
    assert d_d.cpu().numpy().tobytes() == d_host.tobytes() and g_d.cpu().numpy().tobytes() == g_host.tobytes()
    g.free()


def test_sample_maps_arguments():
    gow, g, params = _gen(128, 2, frames=1)
    scales = gow.WaveGenerator.map_scales(params)
    d, gr = g.sample(np.zeros((0, 2), np.float32), scales)       # empty batch
    assert d.shape == (0, 3) and gr.shape == (0, 3)
    with pytest.raises(gow.OceanError):
        g.sample(np.zeros((4, 2), np.float32), np.zeros((5, 4), np.float32))    # more cascades than layers
    with pytest.raises(gow.OceanError):
        g.sample(np.zeros((4, 2), np.float32), np.zeros((0, 4), np.float32))
    g.free()
