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
WAKE = 128                                                      # cells per side of the wake layer the wake ops run on
INVALID = 1                                                     # OCEAN_ERR_INVALID_ARGUMENT


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


def _floating(g, n):
    """n floating bodies over _hull(g, n), and their states."""
    b = np.zeros(n, g.FLOATING_BODY)
    b["mass"] = 200.0
    b["inertia"] = 50.0
    b["first_point"] = np.arange(n) * POINTS_PER_BODY
    b["num_points"] = POINTS_PER_BODY
    s = np.zeros(n, g.BODY_STATE)
    s["position"][:, [0, 2]] = _points(n)
    s["orientation"][:, 3] = 1.0
    return b, s


def _simulate_bodies(g, scales, n):
    pts, cda = _hull(g, n)
    b, s = _floating(g, n)
    g.simulate_bodies(b, s, pts, cda, scales, 1.0 / 60.0, 2, return_records=True, return_transforms=True)


def _drive_bodies(g, scales, n):
    """_simulate_bodies with one thruster, one foil and one load per body and a tether from each body to the next (the last one
    anchored), so that every drive array is staged."""
    pts, cda = _hull(g, n)
    b, s = _floating(g, n)
    k = np.arange(n)
    th = np.zeros(n, g.THRUSTER)
    th["body"], th["direction"], th["thrust"], th["half_height"] = k, (1.0, 0.0, 0.0), 50.0, 0.1
    fo = np.zeros(n, g.FOIL)
    fo["body"], fo["normal"], fo["area"], fo["half_height"] = k, (0.0, 0.0, 1.0), 0.5, 0.1
    te = np.zeros(n, g.TETHER)
    te["body_a"], te["body_b"] = k, np.where(k + 1 < n, k + 1, -1)
    te["rest_length"], te["stiffness"], te["damping"] = 5.0, 100.0, 10.0
    g.drive_bodies(b, s, pts, cda, scales, 1.0 / 60.0, 2, thrusters=th, foils=fo, loads=np.zeros(n, g.BODY_LOAD), tethers=te,
                   return_records=True, return_tensions=True, return_transforms=True)


def _hull_meshes(g):
    """Registers one closed unit box (8 vertices, 12 triangles); the same set again keeps the count."""
    v = np.array([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)], np.float32)
    t = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4],
                  [1, 5, 7], [1, 7, 3]], np.int32)
    m = np.zeros(1, g.HULL_MESH)
    m["num_vertices"], m["num_triangles"], m["normal_drag"], m["tangential_drag"] = len(v), len(t), 1.0, 0.1
    g.set_hull_meshes(m, v, t)


def _hull_poses(g, n):
    b = np.zeros(n, g.HULL_BODY)
    b["transform"][:, [0, 5, 10]] = 1.0
    b["transform"][:, [3, 11]] = _points(n)
    return b


def _floating_hulls(g, n):
    b = np.zeros(n, g.FLOATING_HULL)
    b["mass"] = 200.0
    b["inertia"] = 50.0
    s = np.zeros(n, g.BODY_STATE)
    s["position"][:, [0, 2]] = _points(n)
    s["orientation"][:, 3] = 1.0
    return b, s


def _hull_forces(g, scales, n):
    _hull_meshes(g)
    g.hull_forces(_hull_poses(g, n), np.zeros(n, g.BODY_VELOCITY), scales, return_samples=True)


def _simulate_hull_bodies(g, scales, n):
    _hull_meshes(g)
    b, s = _floating_hulls(g, n)
    g.simulate_hull_bodies(b, s, scales, 1.0 / 60.0, 2, return_records=True, return_transforms=True)


def _debug_device_math(g, scales, n):
    from godotoceanwaves_b200.native import check, load_library
    a = np.linspace(-10, 10, n, dtype=np.float32)
    out = np.empty((n, 2), np.float32)
    check(load_library().ocean_debug_device_math(g.context, 0, n, a.ctypes.data, a.ctypes.data, out.ctypes.data))   # OCEAN_MATH_SINCOS


def _wake_layer(g):
    g.wake_init(WAKE, 0.5)                                      # the same size again keeps the fields and the staging


def _wake_step(g, scales, n):
    """n sources, every other one attached to one of n body states, so that both arrays are staged."""
    _wake_layer(g)
    src = np.zeros(n, g.WAKE_SOURCE)
    src["x"], src["z"] = np.random.default_rng(n).uniform(0, 0.5 * WAKE, (2, n))
    src["vx"], src["radius"], src["head"] = 2.0, 1.5, 0.2
    src["body"] = np.where(np.arange(n) % 2 == 0, np.arange(n), -1)
    states = np.zeros(n, g.BODY_STATE)
    states["orientation"][:, 3] = 1.0
    g.wake_step(0.05, 1, (0, 0), src, states)


def _sample_wake(g, scales, n):
    _wake_layer(g)
    g.sample_wake(_points(n))


OPS = [_sample_maps, _sample_velocity, _query_surface, _raycast, _extract_spray, _buoyancy, _body_forces, _simulate_bodies,
       _drive_bodies, _hull_forces, _simulate_hull_bodies, _debug_device_math, _wake_step, _sample_wake]


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


def _invalid_call(op, g, scales):
    """One call of host entry point `op` with a NULL host buffer where a positive count needs one; returns its status."""
    from godotoceanwaves_b200.native import load_library
    lib, h, n = load_library(), g.context, 8
    pts, out = _points(n), np.zeros(16 * n, np.float32)        # inputs, and room for any output
    P, O, S = pts.ctypes.data, out.ctypes.data, scales.ctypes.data
    rays, ps, emitter = _rays(g, n), np.ones(3, np.float32), g.default_spray_emitter()
    poses, velocities, (hull, cda) = _poses(g, 2), np.zeros(2, g.BODY_VELOCITY), _hull(g, 2)
    bodies, states = _floating(g, 2)
    thrusters = np.zeros(2, g.THRUSTER)
    thrusters["body"] = (0, 1)
    hull_poses, (hulls, _) = _hull_poses(g, 2), _floating_hulls(g, 2)
    count = ctypes.c_int()
    calls = {
        "sample_maps": lambda: lib.ocean_sample_maps(h, n, P, C, S, None, O),
        "sample_velocity": lambda: lib.ocean_sample_velocity(h, n, P, C, S, None),
        "query_surface": lambda: lib.ocean_query_surface(h, n, P, C, S, 1e-3, 8, None),
        "raycast": lambda: lib.ocean_raycast(h, n, rays.ctypes.data, C, S, 0.5, 64, 1e-3, 8, None),
        "extract_spray": lambda: lib.ocean_extract_spray(h, n, P, C, S, ps.ctypes.data, n, None, ctypes.byref(count)),
        "spray_particles": lambda: lib.ocean_spray_particles(h, emitter.ctypes.data, 0.0, 0.02, C, S, None, n, O, ctypes.byref(count)),
        "buoyancy": lambda: lib.ocean_buoyancy(h, 2, poses.ctypes.data, len(hull), hull.ctypes.data, C, S, 1025.0, 1e-3, 8, None, None),
        "body_forces": lambda: lib.ocean_body_forces(h, 2, poses.ctypes.data, velocities.ctypes.data, len(hull), hull.ctypes.data,
                                                     cda.ctypes.data, C, S, 1025.0, 1e-3, 8, None, O, None),
        "simulate_bodies": lambda: lib.ocean_simulate_bodies(h, 2, bodies.ctypes.data, states.ctypes.data, len(hull), None, cda.ctypes.data,
                                                             C, S, 1025.0, 1.0 / 60.0, 1, 1e-3, 8, None, None, None),
        "drive_bodies": lambda: lib.ocean_simulate_driven_bodies(h, 2, bodies.ctypes.data, states.ctypes.data, len(hull), None,
                                                                 cda.ctypes.data, C, S, 1025.0, 1.0 / 60.0, 1, 1e-3, 8, 2,
                                                                 thrusters.ctypes.data, 0, None, None, 0, None, None, None, None, None, None),
        "hull_forces": lambda: lib.ocean_hull_forces(h, 2, hull_poses.ctypes.data, velocities.ctypes.data, C, S, 1025.0, 1e-3, 8, None, O,
                                                     None),
        "simulate_hull_bodies": lambda: lib.ocean_simulate_hull_bodies(h, 2, hulls.ctypes.data, None, C, S, 1025.0, 1.0 / 60.0, 1, 1e-3, 8,
                                                                       None, None, None),
        "debug_device_math": lambda: lib.ocean_debug_device_math(h, 0, n, P, P, None),
        "wake_step": lambda: lib.ocean_wake_step(h, 0.05, 1, 0, 0, n, None, 0, None),
        "sample_wake": lambda: lib.ocean_sample_wake(h, n, P, None),
    }
    return calls[op]()


HOST_OPS = ["sample_maps", "sample_velocity", "query_surface", "raycast", "extract_spray", "spray_particles", "buoyancy", "body_forces",
            "simulate_bodies", "drive_bodies", "hull_forces", "simulate_hull_bodies", "debug_device_math", "wake_step", "sample_wake"]


@pytest.mark.parametrize("op", HOST_OPS)
def test_invalid_host_call_stages_nothing(op):
    """A host entry point validates its arguments before it stages anything: an invalid call on a generator whose staging is
    still empty allocates nothing and launches nothing."""
    g, _, scales = _gen()
    if op in ("wake_step", "sample_wake"):
        _wake_layer(g)
    if op in ("hull_forces", "simulate_hull_bodies"):
        _hull_meshes(g)                                         # so that the NULL buffer, not a missing mesh set, is rejected
    before = _bytes(g), g.info().kernel_launches
    assert _invalid_call(op, g, scales) == INVALID
    assert (_bytes(g), g.info().kernel_launches) == before
    g.free()


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
