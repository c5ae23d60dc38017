"""The hull-mesh specification oracle/hull.py against independent computations on flat water: clipped boxes and convex hulls
against scipy's half-space intersection in float64, full immersion, inverted winding, each clip case by hand, the drag
closed forms of a box moving through still water, and the integrator's draft, heave period and stability."""
import numpy as np
import pytest
from scipy.optimize import linprog
from scipy.spatial import ConvexHull, HalfspaceIntersection

from oracle import bodies as bo
from oracle import drag as dr
from oracle import hull as oh

RHO = 1025.0
RHO_G = float(np.float32(RHO) * np.float32(9.81))
N, C = 16, 1
ZERO = np.zeros((C, N, N, 4), np.float16)
SCALES = np.array([[1.0 / 16.0, 1.0 / 16.0, 1.0, 1.0]], np.float32)


def box(lx, ly, lz, c_n=0.0, c_t=0.0):
    """(vertices [8][3], triangles [12][3] in Godot's winding, MESH [1]) of an axis-aligned box centred on the origin."""
    v = np.array([[x, y, z] for x in (-lx / 2, lx / 2) for y in (-ly / 2, ly / 2) for z in (-lz / 2, lz / 2)], np.float32)
    return (v, *_outward(v, ConvexHull(v.astype(np.float64)).simplices, c_n, c_t))


def _outward(v, simplices, c_n=0.0, c_t=0.0):
    """The triangles of a convex hull wound clockwise seen from outside (a = 0.5 (c - a) x (b - a) points out), and a MESH row."""
    v = v.astype(np.float64)
    centre = v.mean(0)
    tris = []
    for t in simplices:
        a, b, c = v[t]
        if np.dot(np.cross(c - a, b - a), a - centre) < 0:
            t = t[[0, 2, 1]]
        tris.append(t)
    tris = np.array(tris, np.int32)
    mesh = np.zeros(1, oh.MESH)
    mesh["num_vertices"], mesh["num_triangles"] = len(v), len(tris)
    mesh["normal_drag"], mesh["tangential_drag"] = c_n, c_t
    return tris, mesh


def rotation(axis, angle):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    q = np.concatenate([axis * np.sin(angle / 2), [np.cos(angle / 2)]]).astype(np.float32)
    return q


def pose(q, t):
    s = np.zeros(1, bo.STATE)
    s["orientation"], s["position"] = q, t
    body = np.zeros(1, oh.BODY)
    body["transform"] = bo.transforms(s)
    return body


def forces(body, mesh, v, tris, velocity=None, zero_velocity=ZERO):
    vel = np.zeros(len(body), dr.VELOCITY) if velocity is None else velocity
    with np.errstate(all="ignore"):
        return oh.hull_forces(ZERO, ZERO, zero_velocity, body, vel, mesh, v, tris, SCALES, RHO)


def submerged_float64(v, body):
    """Volume and centroid (world) of the hull below y = 0, by scipy's half-space intersection in float64."""
    T = body["transform"][0].reshape(3, 4).astype(np.float64)
    w = v.astype(np.float64) @ T[:, :3].T + T[:, 3]
    eq = np.concatenate([ConvexHull(w).equations, [[0.0, 1.0, 0.0, 0.0]]])
    # an interior point: the centre of the largest ball inside (Chebyshev centre)
    norm = np.linalg.norm(eq[:, :3], axis=1)
    res = linprog(np.r_[0, 0, 0, -1], A_ub=np.c_[eq[:, :3], norm], b_ub=-eq[:, 3], bounds=[(None, None)] * 3 + [(0, None)])
    assert res.status == 0 and res.x[3] > 1e-3
    pts = HalfspaceIntersection(eq, res.x[:3]).intersections
    ch = ConvexHull(pts)
    o = pts.mean(0)
    vol, mom = 0.0, np.zeros(3)
    for s in ch.simplices:
        tet = np.abs(np.linalg.det(pts[s] - o)) / 6.0
        vol += tet
        mom += tet * (pts[s].sum(0) + o) / 4.0
    return vol, mom / vol


def _straddle(v, q, rng, x, z):
    """A position that puts between 20 % and 80 % of the rotated hull's height under y = 0."""
    y = (v.astype(np.float64) @ bo.rotation(q)[0].T.astype(np.float64))[:, 1]
    return (x, -(y.min() + rng.uniform(0.2, 0.8) * (y.max() - y.min())), z)


def _check_flat(v, tris, mesh, q, t):
    body = pose(q, t)
    hyd, _ = forces(body, mesh, v, tris)
    vol, c = submerged_float64(v, body)
    h = hyd[0]
    size = float(np.abs(v).max())
    assert abs(h["submerged_volume"] - vol) <= 2e-5 * max(vol, size ** 3)
    centre = np.asarray(t, np.float64) + h["center_offset"]
    assert np.abs(centre - c).max() <= 2e-5 * size
    assert abs(h["force"][1] - RHO_G * vol) <= 2e-5 * RHO_G * max(vol, size ** 3)
    assert np.abs(h["force"][[0, 2]]).max() <= 2e-5 * RHO_G * size ** 3
    want = np.cross(h["center_offset"].astype(np.float64), h["force"].astype(np.float64))
    assert np.abs(h["torque"] - want).max() <= 5e-5 * RHO_G * size ** 4


def test_flat_water_box_matches_float64_clipping():
    rng = np.random.default_rng(1)
    v, tris, mesh = box(2.0, 1.0, 3.0)
    for _ in range(12):
        q = rotation(rng.normal(size=3), rng.uniform(0, np.pi))
        _check_flat(v, tris, mesh, q, _straddle(v, q, rng, rng.uniform(-5, 5), rng.uniform(-5, 5)))


def test_flat_water_convex_hulls_match_float64_clipping():
    rng = np.random.default_rng(2)
    for _ in range(10):
        pts = (rng.normal(size=(40, 3)) * rng.uniform(0.5, 2.0, 3)).astype(np.float32)
        ch = ConvexHull(pts.astype(np.float64))
        v = pts[ch.vertices]
        remap = np.full(len(pts), -1)
        remap[ch.vertices] = np.arange(len(ch.vertices))
        tris, mesh = _outward(v, remap[ch.simplices])
        q = rotation(rng.normal(size=3), rng.uniform(0, np.pi))
        _check_flat(v, tris, mesh, q, _straddle(v, q, rng, rng.uniform(-3, 3), rng.uniform(-3, 3)))


def test_volumes_match_convex_hull_and_flip_with_winding():
    v, tris, mesh = box(2.0, 1.0, 3.0)
    assert oh.volumes(mesh, v, tris)[0] == pytest.approx(6.0, rel=1e-6)
    assert oh.volumes(mesh, v, tris[:, [0, 2, 1]])[0] == pytest.approx(-6.0, rel=1e-6)


def test_fully_submerged_volume_is_the_mesh_volume_at_any_depth():
    rng = np.random.default_rng(3)
    pts = rng.normal(size=(30, 3)).astype(np.float32)
    ch = ConvexHull(pts.astype(np.float64))
    v = pts[ch.vertices]
    remap = np.full(len(pts), -1)
    remap[ch.vertices] = np.arange(len(ch.vertices))
    tris, mesh = _outward(v, remap[ch.simplices])
    vol = float(oh.volumes(mesh, v, tris)[0])
    q = rotation((1, 2, 3), 0.7)
    for depth in (5.0, 20.0, 80.0):
        hyd, _ = forces(pose(q, (1.0, -depth, 2.0)), mesh, v, tris)
        assert hyd["submerged_volume"][0] == pytest.approx(vol, rel=2e-5 * depth)
        assert hyd["force"][0, 1] == pytest.approx(RHO_G * vol, rel=2e-5 * depth)


def test_inverted_winding_flips_every_sign():
    v, tris, mesh = box(2.0, 1.0, 3.0)
    body = pose(rotation((1, 0, 1), 0.4), (0.3, 0.1, -0.2))
    a, _ = forces(body, mesh, v, tris)
    b, _ = forces(body, mesh, v, tris[:, [0, 2, 1]])
    for k in ("force", "torque", "submerged_volume"):
        np.testing.assert_allclose(b[k], -a[k], rtol=1e-5, atol=1e-3)
    assert a["submerged_volume"][0] > 0 and not b["center_offset"].any()      # V < 0: no centre of buoyancy


def _triangle(corners):
    """One open triangle as a mesh, at the identity pose: depth d = -y on flat water."""
    v = np.asarray(corners, np.float32)
    mesh = np.zeros(1, oh.MESH)
    mesh["num_vertices"], mesh["num_triangles"] = 3, 1
    return v, np.array([[0, 1, 2]], np.int32), mesh


@pytest.mark.parametrize("corners,integral", [
    ([(0, 1, 0), (0, 1, 2), (0, 2, 0)], 0.0),                  # 0 wet
    ([(0, 1, 0), (0, 1, 2), (0, -1, 0)], 1.0 / 6.0),           # 1 wet: the triangle (0,-1,0), (0,0,0), (0,0,1), mean depth 1/3
    ([(0, -1, 0), (0, -1, 2), (0, 1, 0)], 5.0 / 6.0),          # 2 wet: 2/3 over the whole triangle minus -1/6 over its dry part
    ([(0, -1, 0), (0, -1, 1), (0, -2, 0)], 2.0 / 3.0),         # 3 wet: area 1/2, mean depth 4/3
    ([(0, 0, 0), (0, 0, 1), (0, -1, 0)], 1.0 / 6.0),           # two corners at exactly d = 0: the whole triangle
    ([(0, 0, 0), (0, 0, 1), (0, 0, 2)], 0.0),                  # every corner at d = 0
])
def test_clip_cases_by_hand(corners, integral):
    """A triangle in the plane x = 0: the pressure force is rho g integral(d dA) along -n, n = +-x."""
    v, tris, mesh = _triangle(corners)
    for t in (tris, tris[:, [1, 2, 0]], tris[:, [2, 0, 1]], tris[:, [0, 2, 1]]):
        hyd, drg = forces(pose(rotation((0, 1, 0), 0.0), (0, 0, 0)), mesh, v, t)
        assert abs(hyd["force"][0, 0]) == pytest.approx(RHO_G * integral, rel=1e-6, abs=1e-9)
        assert not hyd["force"][0, 1:].any() and not hyd["submerged_volume"].any()


def test_zero_area_and_nan_depth_triangles_add_nothing():
    v, tris, mesh = _triangle([(0, -1, 0), (0, -2, 0), (0, -3, 0)])    # collinear, all wet
    vel = np.zeros(1, dr.VELOCITY)
    vel["linear"] = (1.0, 2.0, 3.0)
    mesh["normal_drag"], mesh["tangential_drag"] = 1.0, 0.5
    hyd, drg = forces(pose(rotation((0, 1, 0), 0.0), (0, 0, 0)), mesh, v, tris, vel)
    assert not np.isnan(hyd["force"]).any() and not hyd["force"].any()
    assert np.frombuffer(drg.tobytes(), np.uint8).sum() == 0
    r = np.zeros((2, 3, 3), np.float32)
    r[:, 1, 0], r[:, 2, 2] = 1.0, 1.0
    d = np.array([[1.0, np.nan, 1.0], [1.0, 1.0, 1.0]], np.float32)
    sums, kept = oh.triangle_sums(r, d, np.zeros((2, 3, 3), np.float32), np.zeros((2, 3)), np.zeros((2, 3)), np.ones(2), np.ones(2))
    assert kept.tolist() == [False, True]


def test_box_drag_closed_forms():
    """A box half under water moving along +x at U through still water: the front face feels 1/2 rho C_n A U^2, the faces along
    the motion 1/2 rho C_t A U^2, the lee face nothing."""
    lx, ly, lz, U, cn, ct = 2.0, 1.0, 3.0, 1.5, 1.2, 0.05
    v, tris, mesh = box(lx, ly, lz, cn, ct)
    vel = np.zeros(1, dr.VELOCITY)
    vel["linear"] = (U, 0.0, 0.0)
    body = pose(rotation((0, 1, 0), 0.0), (0.0, 0.0, 0.0))
    a = 0.5 * np.cross(v[tris[:, 2]] - v[tris[:, 0]], v[tris[:, 1]] - v[tris[:, 0]])
    n = a / np.linalg.norm(a, axis=1)[:, None]
    faces = {"front": n[:, 0] > 0.5, "lee": n[:, 0] < -0.5, "sides": np.abs(n[:, 2]) > 0.5, "bottom": n[:, 1] < -0.5}
    wet = {"front": ly / 2 * lz, "lee": ly / 2 * lz, "sides": 2 * lx * ly / 2, "bottom": lx * lz}
    half = 0.5 * RHO
    want = {"front": -half * cn * wet["front"] * U * U, "lee": 0.0, "sides": -half * ct * wet["sides"] * U * U,
            "bottom": -half * ct * wet["bottom"] * U * U}
    for face, sel in faces.items():
        m = mesh.copy()
        m["num_triangles"] = int(sel.sum())
        _, drg = forces(body, m, v, tris[sel], vel)
        assert drg["force"][0, 0] == pytest.approx(want[face], rel=1e-5, abs=1e-6), face
        assert np.abs(drg["force"][0, 1:]).max() <= 1e-5 * max(1.0, abs(want[face])), face
        assert drg["wetted_drag_area"][0] == pytest.approx((cn + ct) * wet[face], rel=1e-5)
    _, drg = forces(body, mesh, v, tris, vel)
    assert drg["force"][0, 0] == pytest.approx(sum(want.values()), rel=1e-5)
    assert drg["max_relative_speed"][0] == pytest.approx(U, rel=1e-6)


def _floating(v, tris, mesh, density_ratio):
    lx, ly, lz = (v.max(0) - v.min(0)).astype(np.float64)
    m = density_ratio * RHO * lx * ly * lz
    fb = np.zeros(1, oh.FLOATING)
    fb["mass"] = m
    fb["inertia"] = (m / 12 * (ly * ly + lz * lz), m / 12 * (lx * lx + lz * lz), m / 12 * (lx * lx + ly * ly))
    return fb


def _state(q, t):
    s = np.zeros(1, bo.STATE)
    s["orientation"], s["position"] = q, t
    return s


def _run(fb, s, v, tris, mesh, steps, dt, record=None):
    for _ in range(steps):
        s = oh.simulate(ZERO, ZERO, ZERO, fb, s, mesh, v, tris, SCALES, RHO, dt, 1)[0]
        if record is not None:
            record.append(s.copy())
    return s


def test_box_settles_at_its_draft():
    """Released 1 m above the water, a box of half the water's density ends with half its height under water (its centre
    at the waterline): averaged over the last 4 s, since quadratic drag damps the last centimetres slowly."""
    v, tris, mesh = box(1.0, 1.0, 1.0, 2.0, 0.5)
    fb = _floating(v, tris, mesh, 0.5)
    rec = []
    _run(fb, _state((0, 0, 0, 1), (0.0, 1.0, 0.0)), v, tris, mesh, 1200, 1.0 / 60.0, rec)
    y = np.array([r["position"][0, 1] for r in rec[-240:]])
    draft = 0.5 * 1.0
    assert y.mean() == pytest.approx(draft - 0.5, abs=3e-3)
    assert np.abs(y - y.mean()).max() < 1e-2


def test_undamped_heave_period():
    v, tris, mesh = box(1.0, 1.0, 1.0)
    fb = _floating(v, tris, mesh, 0.5)
    dt = 1.0 / 240.0
    rec = []
    eq = 0.5 * 1.0 - 0.5
    _run(fb, _state((0, 0, 0, 1), (0.0, eq - 0.05, 0.0)), v, tris, mesh, 1200, dt, rec)
    y = np.array([r["position"][0, 1] for r in rec]) - eq
    up = np.nonzero((y[:-1] < 0) & (y[1:] >= 0))[0]
    period = np.diff(up).mean() * dt
    want = 2 * np.pi * np.sqrt(float(fb["mass"][0]) / (RHO * 9.81 * 1.0))
    assert period == pytest.approx(want, rel=0.03)


def _roll(s):
    """The angle between the body's up axis and the world's, in degrees."""
    R = bo.rotation(s["orientation"])[0]
    return np.degrees(np.arccos(np.clip(R[1, 1], -1.0, 1.0)))


@pytest.mark.parametrize("shape,stable", [((2.0, 0.5, 2.0), True), ((0.4, 2.0, 2.0), False)])
def test_metacentric_stability(shape, stable):
    """A wide flat box (B^2 / 12 T > KG - T / 2) heeled 20 degrees rights itself; a tall narrow one capsizes."""
    v, tris, mesh = box(*shape, 2.0, 0.5)
    fb = _floating(v, tris, mesh, 0.5)
    T = 0.5 * shape[1]
    gm = shape[0] ** 2 / (12 * T) - (shape[1] / 2 - T / 2)
    assert (gm > 0) == stable
    q = rotation((0, 0, 1), np.radians(20.0))
    y = T - shape[1] / 2
    hyd, _ = forces(pose(q, (0.0, y, 0.0)), mesh, v, tris)
    assert (hyd["torque"][0, 2] < 0) == stable                    # restoring: against the +z heel
    rec = []
    _run(fb, _state(q, (0.0, y, 0.0)), v, tris, mesh, 1800, 1.0 / 60.0, rec)
    if stable:
        assert max(_roll(r) for r in rec[-120:]) < 4.0
    else:
        assert max(_roll(r) for r in rec) > 60.0


def test_body_without_vertices_gets_zero_records():
    v, tris, mesh = box(1.0, 1.0, 1.0, 1.0, 1.0)
    meshes = np.concatenate([mesh, np.zeros(1, oh.MESH)])
    bodies = np.concatenate([pose(rotation((0, 1, 0), 0.0), (0, 0, 0))] * 2)
    bodies["mesh"] = (0, 1)
    vel = np.zeros(2, dr.VELOCITY)
    vel["linear"] = (1.0, 0.0, 0.0)
    with np.errstate(all="ignore"):
        hyd, drg = oh.hull_forces(ZERO, ZERO, ZERO, bodies, vel, meshes, v, tris, SCALES, RHO)
    assert hyd["submerged_volume"][0] > 0 and drg["wetted_drag_area"][0] > 0
    assert not np.frombuffer(hyd[1:].tobytes(), np.uint8).any() and not np.frombuffer(drg[1:].tobytes(), np.uint8).any()
