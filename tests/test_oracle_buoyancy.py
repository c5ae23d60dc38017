"""CPU checks of the buoyancy specification (oracle/buoyancy.py): hydrostatic force and torque per body from hull points
on the displaced water surface, with a fixed per-body reduction order."""
import math

import numpy as np

from oracle import buoyancy as bu

F = np.float32
RHO = 1025.0
TOL = F(1e-3)


def _flat(N=128, C_=1):
    return np.zeros((C_, N, N, 4), np.float16), np.array([[1.0 / 64.0, 1.0 / 64.0, 1.0, 1.0]] * C_, np.float32)


def _box(nx, ny, nz, s=0.5):
    """An upright voxel box centred on the body origin: one point per voxel of side s, volume s^3, half height s / 2."""
    g = [(np.arange(n) + 0.5) * s - n * s / 2 for n in (nx, ny, nz)]
    X, Y, Z = np.meshgrid(*g, indexing="ij")
    p = np.zeros(X.size, bu.POINT)
    p["position"] = np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1)
    p["volume"] = s ** 3
    p["half_height"] = s / 2
    return p


def _transform(R=np.eye(3), t=(0.0, 0.0, 0.0)):
    return np.concatenate([np.asarray(R, np.float32), np.asarray(t, np.float32).reshape(3, 1)], 1).reshape(12)


def _bodies(transforms, ranges):
    b = np.zeros(len(transforms), bu.BODY)
    for i, (T, (first, n)) in enumerate(zip(transforms, ranges)):
        b[i]["transform"], b[i]["first_point"], b[i]["num_points"] = T, first, n
    return b


def _rot_y(a):
    c, s = math.cos(a), math.sin(a)
    return [[c, 0, s], [0, 1, 0], [-s, 0, c]]


def _rot_z(a):
    c, s = math.cos(a), math.sin(a)
    return [[c, -s, 0], [s, c, 0], [0, 0, 1]]


def _rot_x(a):
    c, s = math.cos(a), math.sin(a)
    return [[1, 0, 0], [0, c, -s], [0, s, c]]


def _random_rotations(rng, n):
    q = rng.standard_normal((n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], 1).reshape(n, 3, 3)


def _trochoid(N=256, L=64.0):
    """The single trochoidal wave of test_oracle_surface.py::test_single_gerstner_wave_matches_the_continuous_trochoid:
    (texture, map_scales, amplitude A, |k|, unit k, bound on the height error at a converged point)."""
    L = np.float32(L)
    kv = 2.0 * np.pi * np.array([2.0, 1.0]) / float(L)
    kn = np.linalg.norm(kv)
    khat = kv / kn
    A = 0.5 / kn
    c = (np.arange(N) + 0.5) * (float(L) / N)
    X, Z = np.meshgrid(c, c)
    ph = kv[0] * X + kv[1] * Z
    tex = np.zeros((1, N, N, 4), np.float16)
    tex[0, :, :, 0] = -khat[0] * A * np.sin(ph)
    tex[0, :, :, 1] = A * np.cos(ph)
    tex[0, :, :, 2] = -khat[1] * A * np.sin(ph)
    scales = np.array([[1.0 / L, 1.0 / L, 1.0, 1.0]], np.float32)
    h = float(L) / N
    e = h * h * A * kn * kn / 8.0 + A * 2.0 ** -11
    bound = e + A * kn * np.sqrt(2.0) * (e + float(TOL)) / (1.0 - A * kn) + 1e-5
    return tex, scales, A, kn, khat, bound


def _trochoid_height(A, kn, khat, x, z):
    """float64 height of the continuous trochoid over world (x, z): the root of s - A sin(|k| s) = k^.Q."""
    q = khat[0] * np.asarray(x, np.float64) + khat[1] * np.asarray(z, np.float64)
    s = q.copy()
    for _ in range(50):
        s -= (s - A * np.sin(kn * s) - q) / (1.0 - A * kn * np.cos(kn * s))
    return A * np.cos(kn * s)


def test_record_layouts_match_the_bindings():
    from godotoceanwaves_b200.wave_generator import WaveGenerator
    for dt, wg, size in [(bu.POINT, WaveGenerator.BUOYANCY_POINT, 20), (bu.BODY, WaveGenerator.BUOYANCY_BODY, 56),
                         (bu.RESULT, WaveGenerator.BUOYANCY_RESULT, 48)]:
        assert dt.itemsize == wg.itemsize == size
        assert dt.names == wg.names
        for name in dt.names:
            assert dt.fields[name][1] == wg.fields[name][1], name
    assert WaveGenerator.BUOYANCY_POINT == bu.POINT and WaveGenerator.BUOYANCY_BODY == bu.BODY
    assert WaveGenerator.BUOYANCY_RESULT == bu.RESULT


def test_flat_water_submerged_volume_is_exact():
    """4 x 4 x 4 voxels of 0.5 m: footprint A = 4 m^2, from y = -1 to 1 in the body.  At dyadic drafts every operation is exact."""
    d16, sc = _flat()
    hull = _box(4, 4, 4)
    drafts = [0.0, 0.125, 0.375, 0.5, 0.625, 1.0, 1.3125, 2.0]
    ty = [1.0 - d for d in drafts] + [1.5, -1.25, 40.0, -40.0]
    bodies = _bodies([_transform(t=(3.0, y, -7.5)) for y in ty], [(0, len(hull))] * len(ty))
    out = bu.buoyancy(d16, d16, bodies, hull, sc, RHO, TOL, 8)
    want = [4.0 * d for d in drafts] + [0.0, 8.0, 0.0, 8.0]
    assert out["submerged_volume"].tolist() == want
    assert out["force"][:, 1].tolist() == [F(F(RHO) * bu.G) * F(v) for v in want]
    assert not out["force"][:, [0, 2]].any() and not out["torque"].any()     # symmetric about the vertical axis
    assert not out["center_offset"][:, [0, 2]].any()
    assert np.all(out["max_residual"] == 0) and not out["unconverged"].any()


def test_zero_half_height_is_a_step():
    d16, sc = _flat()
    p = np.zeros(5, bu.POINT)
    p["position"][:, 1] = [-0.5, -2.0 ** -20, 0.0, 2.0 ** -20, 0.5]
    p["volume"] = [1.0, 2.0, 4.0, 8.0, 16.0]
    out = bu.buoyancy(d16, d16, _bodies([_transform()], [(0, 5)]), p, sc, RHO, TOL, 8)
    assert out["submerged_volume"][0] == 7.0                     # w.y <= eta = 0: the first three
    d16b = d16.copy()                                             # the surface at 0.25 m: the fourth point is below it too
    d16b[..., 1] = np.float16(0.25)
    out = bu.buoyancy(d16b, d16b, _bodies([_transform()], [(0, 5)]), p, sc, RHO, TOL, 8)
    assert out["submerged_volume"][0] == 15.0


def test_rotation_about_the_vertical_keeps_the_volume():
    d16, sc = _flat()
    hull = _box(6, 4, 2)
    angles = [0.0, 0.3, 1.0, 2.0, -2.5, math.pi / 2]
    bodies = _bodies([_transform(_rot_y(a), (0.0, 0.375, 0.0)) for a in angles], [(0, len(hull))] * len(angles))
    out = bu.buoyancy(d16, d16, bodies, hull, sc, RHO, TOL, 8)
    assert np.all(out["submerged_volume"] == out["submerged_volume"][0]) and out["submerged_volume"][0] == 3.0 * 1.0 * 0.625


def test_equilibrium_draft_by_bisection():
    d16, sc = _flat()
    hull = _box(4, 4, 4)                                          # A = 4 m^2, 0.5 m voxel layers
    mass = 3000.0                                                 # kg: m / (rho A) = 0.7317 m
    lo, hi = -1.0, 1.0                                            # body height ty; the volume falls as ty rises
    for _ in range(40):
        mid = 0.5 * (lo + hi)
        v = bu.buoyancy(d16, d16, _bodies([_transform(t=(0.0, mid, 0.0))], [(0, len(hull))]), hull, sc, RHO, TOL, 0)
        if float(v["force"][0, 1]) > mass * float(bu.G):
            lo = mid
        else:
            hi = mid
    draft = 1.0 - 0.5 * (lo + hi)
    want = mass / (RHO * 4.0)
    assert abs(draft - want) <= 0.5                               # within one voxel layer ...
    assert abs(draft - want) <= 1e-5                              # ... and, the columns being continuous, much closer


def test_roll_gives_a_restoring_torque():
    """A wide shallow box (8 m x 1 m x 4 m) floating at half its height, rolled by +-10 degrees about z and about x."""
    d16, sc = _flat()
    hull = _box(16, 2, 8)
    rolls = [10.0, -10.0]
    Rs = [_rot_z(math.radians(a)) for a in rolls] + [_rot_x(math.radians(a)) for a in rolls]
    out = bu.buoyancy(d16, d16, _bodies([_transform(R) for R in Rs], [(0, len(hull))] * 4), hull, sc, RHO, TOL, 8)
    tz, tx = out["torque"][:2, 2], out["torque"][2:, 0]
    assert np.all(np.sign(tz) == -np.sign(rolls)) and np.all(np.sign(tx) == -np.sign(rolls))
    assert np.all(np.abs(tz) > 1e4) and np.all(np.abs(tx) > 1e3)


def test_trochoid_heights_and_thin_column_volumes():
    """Thin columns (area a = 1/16 m^2, 2 m tall) over the single trochoidal wave, one body each, all sharing one hull point.
    The spec's height at every column matches the float64 trochoid within the surface test's bound, and the submerged volume
    the analytic a * clamp(eta - (y - h), 0, 2h) within that bound times a."""
    tex, sc, A, kn, khat, bound = _trochoid()
    rng = np.random.default_rng(11)
    n = 4000
    t = np.stack([rng.uniform(-300, 300, n), rng.uniform(-A - 1.5, A + 1.5, n), rng.uniform(-300, 300, n)], 1)
    a, h = 1.0 / 16.0, 1.0
    hull = np.zeros(1, bu.POINT)
    hull["volume"], hull["half_height"] = a * 2 * h, h
    bodies = _bodies([_transform(t=ti) for ti in t], [(0, 1)] * n)
    out, samples = bu.buoyancy(tex, np.zeros_like(tex), bodies, hull, sc, RHO, TOL, 8, return_samples=True)
    assert np.all(samples["residual"] <= TOL)
    w = t.astype(np.float32)
    eta = _trochoid_height(A, kn, khat, w[:, 0], w[:, 2])
    assert np.abs(samples["displacement"][:, 1] - eta).max() <= bound
    want = a * np.clip(eta - (w[:, 1].astype(np.float64) - h), 0.0, 2 * h)
    assert 0 < np.mean(want == 0) < 0.5 and 0 < np.mean(want == a * 2 * h) < 0.5      # dry, wet and partial columns
    assert np.abs(out["submerged_volume"] - want).max() <= bound * a + 1e-6


def _random_scene(rng, sizes):
    """Bodies of the given sizes, random rotations and positions near the surface, random hulls (one zero half height)."""
    hull = np.zeros(int(sum(sizes)), bu.POINT)
    hull["position"] = rng.uniform(-3, 3, (len(hull), 3))
    hull["volume"] = rng.uniform(0.01, 0.5, len(hull))
    hull["half_height"] = rng.uniform(0.05, 0.6, len(hull))
    hull["half_height"][::7] = 0.0
    R = _random_rotations(rng, len(sizes))
    t = np.stack([rng.uniform(-200, 200, len(sizes)), rng.uniform(-1, 1, len(sizes)), rng.uniform(-200, 200, len(sizes))], 1)
    starts = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    return _bodies([_transform(R[i], t[i]) for i in range(len(sizes))], list(zip(starts, sizes))), hull


def test_sums_match_fsum():
    tex, sc, *_ = _trochoid()
    rng = np.random.default_rng(12)
    sizes = [1, 31, 32, 33, 1000, 77, 500]
    bodies, hull = _random_scene(rng, sizes)
    out, samples = bu.buoyancy(tex, tex, bodies, hull, sc, RHO, TOL, 8, return_samples=True)
    body, j, r, w = bu.world_points(bodies, hull)
    p = hull[bodies["first_point"][body] + j]
    v = bu.submerged_fraction(samples["displacement"][:, 1], w[:, 1], p["half_height"]) * p["volume"]
    terms = np.stack([v, v * r[:, 0], v * r[:, 1], v * r[:, 2]], 1)
    S = bu.lane_tree_sum(terms, body, j, len(sizes))
    assert out["submerged_volume"].tobytes() == S[:, 0].tobytes()
    rg = F(RHO) * bu.G
    assert out["torque"][:, 0].tobytes() == (-(rg * S[:, 3])).tobytes() and out["torque"][:, 2].tobytes() == (rg * S[:, 1]).tobytes()
    assert np.count_nonzero(S[:, 0]) >= len(sizes) - 1
    for b in range(len(sizes)):
        k = body == b
        for c in range(4):
            exact = math.fsum(terms[k, c].astype(np.float64))
            scale = math.fsum(np.abs(terms[k, c]).astype(np.float64))
            assert abs(float(S[b, c]) - exact) <= 1e-6 * scale, (b, c)


def _restated(bodies, hull, samples, density, tol):
    """The record of every body by an explicit scalar loop: lane j mod 32, increasing j, the shuffle tree."""
    out = np.zeros(len(bodies), bu.RESULT)
    k = 0
    for b, body in enumerate(bodies):
        T = body["transform"].reshape(3, 4)
        lanes = np.zeros((32, 4), np.float32)
        mx, missed = F(np.nan), 0
        for j in range(body["num_points"]):
            p = hull[body["first_point"] + j]
            x, y, z = p["position"]
            r = [(T[i, 0] * x + T[i, 1] * y) + T[i, 2] * z for i in range(3)]
            wy = r[1] + T[1, 3]
            eta, res = samples[k]["displacement"][1], samples[k]["residual"]
            h = p["half_height"]
            if h > 0:
                f = np.fmin(np.fmax((eta - (wy - h)) / (h + h), F(0)), F(1))
            else:
                f = F(1) if wy <= eta else F(0)
            v = F(f) * p["volume"]
            lanes[j % 32] = [lanes[j % 32, 0] + v, lanes[j % 32, 1] + v * r[0], lanes[j % 32, 2] + v * r[1], lanes[j % 32, 3] + v * r[2]]
            mx = np.fmax(mx, res)
            missed += not (res <= tol)
            k += 1
        for o in (16, 8, 4, 2, 1):
            for l in range(o):
                lanes[l] = lanes[l] + lanes[l + o]
        s0, s1 = lanes[0, 0], lanes[0, 1:]
        if body["num_points"] == 0:
            continue
        rg = F(density) * bu.G
        out[b]["force"] = (0, rg * s0, 0)
        out[b]["torque"] = (-(rg * s1[2]), 0, rg * s1[0])
        out[b]["submerged_volume"] = s0
        out[b]["center_offset"] = s1 / s0 if s0 > 0 else (0, 0, 0)
        out[b]["max_residual"] = mx
        out[b]["unconverged"] = missed
    return out


def test_reduction_equals_an_explicit_lane_tree_restatement():
    tex, sc, *_ = _trochoid()
    rng = np.random.default_rng(13)
    sizes = [1, 31, 32, 33, 1000, 0, 64]
    bodies, hull = _random_scene(rng, sizes)
    bodies = np.concatenate([bodies, bodies[[4, 1]]])             # overlapping (shared) ranges
    bodies["transform"][-1] = _transform(_rot_x(0.4), (5.0, 0.25, -9.0))
    sc2 = sc.copy()
    sc2[:, 2] *= F(2.0)                                           # steeper than 0.5: some points do not converge
    for scales, maxit, tol in [(sc, 8, TOL), (sc2, 2, F(1e-5))]:
        out, samples = bu.buoyancy(tex, tex, bodies, hull, scales, RHO, tol, maxit, return_samples=True)
        assert out.tobytes() == _restated(bodies, hull, samples, RHO, tol).tobytes()
        assert out[5].tobytes() == bytes(48)                      # the empty body
    assert out["unconverged"].sum() > 0
