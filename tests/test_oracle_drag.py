"""CPU checks of the body-forces specification (oracle/drag.py): quadratic drag against the water velocity per body, next to
the unchanged buoyancy record, with the buoyancy op's fixed per-body reduction order."""
import math
import os
import re

import numpy as np

from oracle import buoyancy as bu
from oracle import drag as dr
from oracle import sampling as sp
from test_oracle_buoyancy import _box, _bodies, _random_rotations, _random_scene, _transform, _trochoid

F = np.float32
RHO = 1025.0
HALF_RHO = F(0.5) * F(RHO)                   # 512.5, exact
TOL = F(1e-3)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _flat(N=128, C_=1):
    return np.zeros((C_, N, N, 4), np.float16), np.array([[1.0 / 64.0, 1.0 / 64.0, 1.0, 1.0]] * C_, np.float32)


def _current(u, N=128, C_=1):
    """Velocity maps of a uniform current u (m/s) in cascade 0, zero in the others."""
    v = np.zeros((C_, N, N, 4), np.float16)
    v[0, :, :, :3] = np.asarray(u, np.float16)
    return v


def _velocities(linear, angular=None):
    linear = np.asarray(linear, np.float32).reshape(-1, 3)
    v = np.zeros(len(linear), dr.VELOCITY)
    v["linear"] = linear
    if angular is not None:
        v["angular"] = np.asarray(angular, np.float32).reshape(-1, 3)
    return v


def test_record_layouts_match_the_bindings_and_the_header():
    from godotoceanwaves_b200.wave_generator import WaveGenerator
    header = open(os.path.join(ROOT, "include", "ocean.h")).read()
    for dt, wg, size, name in [(dr.VELOCITY, WaveGenerator.BODY_VELOCITY, 24, "ocean_body_velocity"),
                               (dr.RESULT, WaveGenerator.DRAG_RESULT, 32, "ocean_drag_result")]:
        assert dt.itemsize == wg.itemsize == size
        assert dt.names == wg.names
        for field in dt.names:
            assert dt.fields[field][1] == wg.fields[field][1], field
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), header, re.S).group(1)
        fields = re.findall(r"float (\w+)(?:\[(\d)\])?;", body)
        assert [f for f, _ in fields] == list(dt.names)
        assert 4 * sum(int(n or 1) for _, n in fields) == size
    assert WaveGenerator.BODY_VELOCITY == dr.VELOCITY and WaveGenerator.DRAG_RESULT == dr.RESULT


def test_translating_box_in_still_water_is_the_closed_form():
    """A fully submerged 4 x 4 x 4 voxel box (C_d A = 1/4 m^2 per point, 16 m^2 in all), its hull centred on (1, -0.5, 2) in
    the body, moving at v = (3, 0, 4), |v| = 5, through flat still water: every operation is exact."""
    d16, sc = _flat()
    hull = _box(4, 4, 4)
    c = np.array([1.0, -0.5, 2.0], np.float32)
    hull["position"] += c
    cda = np.full(len(hull), 0.25, np.float32)
    v = np.array([3.0, 0.0, 4.0])
    bodies = _bodies([_transform(t=(3.0, -5.0, -7.5))], [(0, len(hull))])
    hydro, drag = dr.body_forces(d16, d16, np.zeros_like(d16), bodies, _velocities(v), hull, cda, sc, RHO, TOL, 8)
    want_f = -float(HALF_RHO) * 16.0 * 5.0 * v
    assert drag["force"][0].tolist() == want_f.tolist()
    Fp = -0.25 * 5.0 * v                                          # each point's F; the torque is (sum r) x F = 64 c x F
    want_t = float(HALF_RHO) * 64.0 * np.cross(c.astype(np.float64), Fp)
    assert drag["torque"][0].tolist() == want_t.tolist()
    assert drag["wetted_drag_area"][0] == 16.0 and drag["max_relative_speed"][0] == 5.0
    assert hydro.tobytes() == bu.buoyancy(d16, d16, bodies, hull, sc, RHO, TOL, 8).tobytes()


def test_spinning_body_torque_is_the_closed_form():
    """Points in the body's horizontal plane, in opposite pairs, spinning at W about the vertical in still water: the drag
    torque about y is -1/2 rho C_d A W^2 sum rho_i^3 (it opposes the spin) and the net force vanishes."""
    d16, sc = _flat()
    rng = np.random.default_rng(3)
    n = 48
    ang = rng.uniform(0, 2 * np.pi, n)
    rad = rng.uniform(0.5, 4.0, n)
    half = np.stack([rad * np.cos(ang), np.zeros(n), rad * np.sin(ang)], 1).astype(np.float32)
    hull = np.zeros(2 * n, bu.POINT)
    hull["position"] = np.concatenate([half, -half])
    hull["volume"], hull["half_height"] = 0.1, 0.25
    cda = np.full(len(hull), 0.375, np.float32)
    bodies = _bodies([_transform(t=(10.0, -3.0, 20.0))] * 2, [(0, len(hull))] * 2)
    for k, W in enumerate((0.8, -1.7)):
        _, drag = dr.body_forces(d16, d16, np.zeros_like(d16), bodies[:1], _velocities([0, 0, 0], [0, W, 0]), hull, cda, sc, RHO, TOL, 8)
        r = np.linalg.norm(hull["position"].astype(np.float64), axis=1)
        want = -math.copysign(1.0, W) * 0.5 * RHO * 0.375 * W * W * math.fsum(r ** 3)
        assert abs(float(drag["torque"][0, 1]) - want) <= 1e-6 * abs(want), (W, drag["torque"][0], want)
        scale = 0.5 * RHO * 0.375 * W * W * math.fsum(r ** 2)
        assert np.abs(drag["force"][0].astype(np.float64)).max() <= 1e-6 * scale
        assert abs(float(drag["torque"][0, 0])) <= 1e-6 * abs(want) and abs(float(drag["torque"][0, 2])) <= 1e-6 * abs(want)


def test_dry_body_has_an_all_zero_record():
    d16, sc = _flat()
    hull = _box(2, 2, 2)
    bodies = _bodies([_transform(t=(0.0, 40.0, 0.0)), _transform(t=(0.0, 0.0, 0.0))], [(0, len(hull)), (0, 0)])
    vel = _velocities([[7.0, -2.0, 1.0], [1.0, 1.0, 1.0]], [[0.5, 3.0, -1.0], [1.0, 0.0, 0.0]])
    hydro, drag = dr.body_forces(d16, d16, _current((1.0, 0.5, -2.0)), bodies, vel, hull, np.ones(len(hull), np.float32), sc, RHO, TOL, 8)
    assert drag.tobytes() == bytes(2 * 32)                           # the dry body and the empty body
    assert hydro["submerged_volume"].tolist() == [0.0, 0.0]


def test_uniform_current_drags_a_body_at_rest_and_not_one_moving_with_it():
    """Texel-centred points (the bilinear weights are 0 and 1) in a uniform current u = (0.75, 0, 1), |u| = 1.25."""
    d16, sc = _flat()
    u = np.array([0.75, 0.0, 1.0])
    hull = _box(4, 4, 4)
    cda = np.full(len(hull), 0.25, np.float32)
    bodies = _bodies([_transform(t=(3.0, -5.0, -7.5))] * 2, [(0, len(hull))] * 2)
    _, drag, smp = dr.body_forces(d16, d16, _current(u), bodies, _velocities([[0, 0, 0], u]), hull, cda, sc, RHO, TOL, 8,
                                  return_samples=True)
    x = smp["source_x"] * sc[0, 0] * F(128) - F(0.5)
    assert np.all(x == np.floor(x))                                  # texel centres
    assert drag["force"][0].tolist() == (float(HALF_RHO) * 16.0 * 1.25 * u).tolist()
    assert not drag["torque"][0].any()                               # the hull is centred on the origin
    assert not drag["force"][1].any() and not drag["torque"][1].any() and drag["max_relative_speed"][1] == 0.0
    assert drag["wetted_drag_area"].tolist() == [16.0, 16.0]


def test_drag_dissipates_energy_in_the_frame_of_the_current():
    """F . (u - v) - w . tau = sum_j k_j |d_j|^2 >= 0 for every body (float64 on the binary32 results)."""
    tex, sc, *_ = _trochoid()
    rng = np.random.default_rng(21)
    sizes = rng.integers(1, 60, 200)
    bodies, hull = _random_scene(rng, sizes)
    u = np.array([0.5, -0.125, 1.25])
    vel = _velocities(rng.uniform(-3, 3, (len(bodies), 3)), rng.uniform(-2, 2, (len(bodies), 3)))
    cda = rng.uniform(0.01, 0.6, len(hull)).astype(np.float32)
    vmap = _current(u, tex.shape[1])
    _, drag = dr.body_forces(tex, tex, vmap, bodies, vel, hull, cda, sc, RHO, TOL, 8)
    Fd = drag["force"].astype(np.float64)
    T = drag["torque"].astype(np.float64)
    rel = u - vel["linear"].astype(np.float64)
    w = vel["angular"].astype(np.float64)
    P = np.sum(Fd * rel, 1) - np.sum(w * T, 1)
    scale = np.linalg.norm(Fd, axis=1) * np.linalg.norm(rel, axis=1) + np.linalg.norm(w, axis=1) * np.linalg.norm(T, axis=1)
    assert np.all(P >= -1e-5 * scale)
    wet = drag["wetted_drag_area"] > 0
    assert wet.sum() > 100 and np.all(P[wet] > 0)


def _sources_velocity(vmap, smp, sc):
    """The water velocity at the records' source points through oracle/sampling.py's sample_maps (its displacement half)."""
    u, _ = sp.sample_maps(vmap, vmap, np.stack([smp["source_x"], smp["source_z"]], 1), sc)
    return u


def _restated(bodies, vel, hull, cda, smp, u, density):
    """The drag record of every body by an explicit scalar loop: lane j mod 32, increasing j, the shuffle tree."""
    out = np.zeros(len(bodies), dr.RESULT)
    k = 0
    for b, body in enumerate(bodies):
        T = body["transform"].reshape(3, 4)
        v, a = vel[b]["linear"], vel[b]["angular"]
        lanes = np.zeros((32, 7), np.float32)
        mx = F(0)
        for j in range(body["num_points"]):
            p = hull[body["first_point"] + j]
            x, y, z = p["position"]
            r = [(T[i, 0] * x + T[i, 1] * y) + T[i, 2] * z for i in range(3)]
            wy = r[1] + T[1, 3]
            eta, h = smp[k]["displacement"][1], p["half_height"]
            if h > 0:
                f = np.fmin(np.fmax((eta - (wy - h)) / (h + h), F(0)), F(1))
            else:
                f = F(1) if wy <= eta else F(0)
            uk = u[k]
            k += 1
            if not f > 0:
                continue
            vb = [v[0] + (a[1] * r[2] - a[2] * r[1]), v[1] + (a[2] * r[0] - a[0] * r[2]), v[2] + (a[0] * r[1] - a[1] * r[0])]
            d = [uk[i] - vb[i] for i in range(3)]
            s = np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
            fa = F(f) * cda[body["first_point"] + j]
            kk = fa * s
            Fp = [kk * d[i] for i in range(3)]
            Tp = [r[1] * Fp[2] - r[2] * Fp[1], r[2] * Fp[0] - r[0] * Fp[2], r[0] * Fp[1] - r[1] * Fp[0]]
            lanes[j % 32] = lanes[j % 32] + np.array(Fp + Tp + [fa], np.float32)
            mx = np.fmax(mx, s)
        for o in (16, 8, 4, 2, 1):
            for l in range(o):
                lanes[l] = lanes[l] + lanes[l + o]
        if body["num_points"] == 0:
            continue
        hr = F(0.5) * F(density)
        out[b]["force"] = hr * lanes[0, 0:3]
        out[b]["torque"] = hr * lanes[0, 3:6]
        out[b]["wetted_drag_area"] = lanes[0, 6]
        out[b]["max_relative_speed"] = mx
    return out


def _random_velocity_map(rng, shape):
    v = np.zeros(shape, np.float16)
    v[..., :3] = rng.uniform(-1.5, 1.5, shape[:-1] + (3,))
    return v


def test_reduction_equals_fsum_and_an_explicit_lane_tree_restatement():
    tex, sc, *_ = _trochoid()
    rng = np.random.default_rng(23)
    sizes = [1, 31, 32, 33, 1000, 0, 77, 500, 64]
    bodies, hull = _random_scene(rng, sizes)
    bodies = np.concatenate([bodies, bodies[[4, 1]]])                # overlapping (shared) ranges
    vel = _velocities(rng.uniform(-2, 2, (len(bodies), 3)), rng.uniform(-1, 1, (len(bodies), 3)))
    cda = rng.uniform(0.01, 0.6, len(hull)).astype(np.float32)
    vmap = _random_velocity_map(rng, tex.shape)
    hydro, drag, smp = dr.body_forces(tex, tex, vmap, bodies, vel, hull, cda, sc, RHO, TOL, 8, return_samples=True)
    ref_h, ref_s = bu.buoyancy(tex, tex, bodies, hull, sc, RHO, TOL, 8, return_samples=True)
    assert hydro.tobytes() == ref_h.tobytes() and smp.tobytes() == ref_s.tobytes()
    u = _sources_velocity(vmap, smp, sc)
    assert drag.tobytes() == _restated(bodies, vel, hull, cda, smp, u, RHO).tobytes()
    assert drag[5].tobytes() == bytes(32)                            # the empty body
    # the per-point terms in float32, their sums against math.fsum
    body, j, r, w = bu.world_points(bodies, hull)
    kp = bodies["first_point"][body] + j
    f = bu.submerged_fraction(smp["displacement"][:, 1], w[:, 1], hull["half_height"][kp])
    assert 0 < np.mean(f > 0) < 1 and np.mean((f > 0) & (f < 1)) > 0.05
    vb = vel["linear"][body] + dr.cross(vel["angular"][body], r)
    d = u - vb
    s = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    a = f * cda[kp]
    Fp = (a * s)[:, None] * d
    terms = np.concatenate([Fp, dr.cross(r, Fp), a[:, None]], 1)
    terms[~(f > 0)] = 0.0
    for b in range(len(bodies)):
        m = body == b
        for c in range(7):
            exact = math.fsum(terms[m, c].astype(np.float64))
            scale = math.fsum(np.abs(terms[m, c]).astype(np.float64))
            got = float(drag[b]["wetted_drag_area"]) if c == 6 else float(((drag[b]["force"], drag[b]["torque"])[c // 3][c % 3]) / HALF_RHO)
            assert abs(got - exact) <= 1e-6 * scale + 1e-7 * abs(exact), (b, c)
    assert np.count_nonzero(drag["wetted_drag_area"]) >= len(bodies) - 2


def test_hydrostatic_record_is_the_buoyancy_op():
    tex, sc, *_ = _trochoid()
    rng = np.random.default_rng(29)
    bodies, hull = _random_scene(rng, rng.integers(0, 50, 120))
    vel = _velocities(rng.uniform(-2, 2, (len(bodies), 3)), rng.uniform(-1, 1, (len(bodies), 3)))
    cda = rng.uniform(0.01, 0.6, len(hull)).astype(np.float32)
    sc2 = sc.copy()
    sc2[:, 2] *= F(2.0)                                             # steeper: some points do not converge
    for scales, maxit in [(sc, 8), (sc2, 2), (sc, 0)]:
        hydro, _, smp = dr.body_forces(tex, tex, _random_velocity_map(rng, tex.shape), bodies, vel, hull, cda, scales, RHO, TOL, maxit,
                                       return_samples=True)
        ref, rsmp = bu.buoyancy(tex, tex, bodies, hull, scales, RHO, TOL, maxit, return_samples=True)
        assert hydro.tobytes() == ref.tobytes() and smp.tobytes() == rsmp.tobytes()
