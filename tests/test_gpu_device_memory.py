"""ocean_info.device_bytes is the exact size of the generator's live device allocations: staging grown by a larger call
replaces the smaller block in the count, the binary32 taps return their bytes when they are switched off, and calls that
only need scratch leave the count as it was.  Every figure here is the generator's own count; device-wide free memory
(cudaMemGetInfo) also moves with other processes on the device and is never consulted."""
import ctypes

import numpy as np
import pytest

from conftest import demo_params

pytestmark = pytest.mark.gpu

N, C = 128, 2
SMALL, LARGE = 64, 5000
POINTS_PER_BODY = 4


def _gen():
    import godotoceanwaves_b200 as gow
    g = gow.WaveGenerator()
    g.map_size = N
    g.init_gpu(C)
    params = [demo_params(gow.WaveCascadeParameters, c) for c in range(C)]
    for _ in range(2):
        g.update_all(1.0 / 50.0, params)
    return g, params, gow.WaveGenerator.map_scales(params)


def _bytes(g):
    return g.info().device_bytes


def _points(n):
    return np.random.default_rng(n).uniform(-100, 100, (n, 2)).astype(np.float32)


def _rays(g, n):
    r = np.zeros(n, g.RAY)
    r["origin"][:, [0, 2]] = _points(n)
    r["origin"][:, 1] = 5.0
    r["direction"] = (0.3, -1.0, 0.2)
    r["t_max"] = 20.0
    return r


def _hull(g, n):
    """n bodies floating at y = 0 with POINTS_PER_BODY hull points each, and their drag areas."""
    pts = np.zeros(n * POINTS_PER_BODY, g.BUOYANCY_POINT)
    pts["position"] = np.random.default_rng(n).uniform(-1, 1, (len(pts), 3))
    pts["volume"] = 0.1
    pts["half_height"] = 0.2
    return pts, np.full(len(pts), 0.3, np.float32)


def _poses(g, n):
    b = np.zeros(n, g.BUOYANCY_BODY)
    b["transform"][:, [0, 5, 10]] = 1.0
    b["transform"][:, [3, 11]] = _points(n)
    b["first_point"] = np.arange(n) * POINTS_PER_BODY
    b["num_points"] = POINTS_PER_BODY
    return b


def _sample_maps(g, scales, n):
    g.sample(_points(n), scales)


def _sample_velocity(g, scales, n):
    g.sample_velocity(_points(n), scales)


def _query_surface(g, scales, n):
    g.query_surface(_points(n), scales)


def _raycast(g, scales, n):
    g.raycast(_rays(g, n), scales, max_samples=64)


def _extract_spray(g, scales, n):
    g.extract_spray(_points(n), scales)


def _buoyancy(g, scales, n):
    pts, _ = _hull(g, n)
    g.buoyancy(_poses(g, n), pts, scales, return_samples=True)


def _body_forces(g, scales, n):
    pts, cda = _hull(g, n)
    g.body_forces(_poses(g, n), np.zeros(n, g.BODY_VELOCITY), pts, cda, scales, return_samples=True)


def _simulate_bodies(g, scales, n):
    pts, cda = _hull(g, n)
    b = np.zeros(n, g.FLOATING_BODY)
    b["mass"] = 200.0
    b["inertia"] = 50.0
    b["first_point"] = np.arange(n) * POINTS_PER_BODY
    b["num_points"] = POINTS_PER_BODY
    s = np.zeros(n, g.BODY_STATE)
    s["position"][:, [0, 2]] = _points(n)
    s["orientation"][:, 3] = 1.0
    g.simulate_bodies(b, s, pts, cda, scales, 1.0 / 60.0, 2, return_records=True, return_transforms=True)


def _debug_device_math(g, scales, n):
    from godotoceanwaves_b200.native import check, load_library
    a = np.linspace(-10, 10, n, dtype=np.float32)
    out = np.empty((n, 2), np.float32)
    check(load_library().ocean_debug_device_math(g.context, 0, n, a.ctypes.data, a.ctypes.data, out.ctypes.data))   # OCEAN_MATH_SINCOS


OPS = [_sample_maps, _sample_velocity, _query_surface, _raycast, _extract_spray, _buoyancy, _body_forces, _simulate_bodies,
       _debug_device_math]


@pytest.mark.parametrize("op", OPS, ids=[op.__name__[1:] for op in OPS])
def test_growth_counts_only_the_live_block(op):
    """A small call and then a large one leave the count of one large call: the grown staging replaces the old block."""
    a, _, scales = _gen()
    b, _, _ = _gen()
    created = _bytes(b)
    assert _bytes(a) == created
    op(a, scales, SMALL)
    op(a, scales, LARGE)
    op(b, scales, LARGE)
    a.synchronize()
    b.synchronize()
    assert _bytes(b) > created
    assert _bytes(a) == _bytes(b)
    a.free()
    b.free()


def test_taps_return_their_bytes():
    g, _, scales = _gen()
    pts = _points(SMALL)
    g.sample_velocity(pts, scales)                              # allocates the velocity maps
    before = _bytes(g)
    layer = C * N * N * 16                                      # one float4 map set
    g.enable_f32_taps(True)
    assert _bytes(g) == before + 2 * layer
    g.sample_velocity(pts, scales)                              # allocates the binary32 velocity tap
    assert _bytes(g) == before + 3 * layer
    g.enable_f32_taps(False)
    assert _bytes(g) == before
    g.free()


def test_scratch_only_calls_keep_the_count():
    from godotoceanwaves_b200.native import check, load_library
    g, params, _ = _gen()
    before = _bytes(g)
    failures, tested = ctypes.c_uint64(), ctypes.c_uint64()
    check(load_library().ocean_selftest_math(g.context, ctypes.byref(failures), ctypes.byref(tested)))
    assert tested.value > 0
    assert _bytes(g) == before
    g.update_frames(0.02, params, 5)                            # builds and keeps the fused launch's item table
    cached = _bytes(g)
    g.update_frames(0.02, params, 5)                            # the same table again
    assert _bytes(g) == cached
    g.free()
