"""CPU checks of the ray-cast specification (oracle/raycast.py): the first crossing of a ray with the displaced water
surface, on flat water, on a single trochoid wave with a float64 root, and on demo maps."""

import numpy as np
import pytest

from conftest import demo_params
from oracle import raycast as rc
from oracle import sampling as sp
from oracle import surface as su

TOL = np.float32(1e-3)


@pytest.fixture(scope="module")
def demo_maps():
    """Demo 256^2 x 4 after two updates, from the CPU oracle, with map_scales as water.gd:102-110 builds them."""
    from oracle import pyoracle as po
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    gen = po.OracleWaveGenerator(256)
    gen.init_gpu(4)
    params = [demo_params(po.CascadeParams, c) for c in range(4)]
    for _ in range(2):
        gen.update_all(1.0 / 50.0, params)
    scales = np.array([[np.float32(1.0) / np.float32(p.tile_length[0]), np.float32(1.0) / np.float32(p.tile_length[1]),
                        p.displacement_scale, p.normal_scale] for p in params], np.float32)
    return gen.displacement_map[:4].view(np.float16).copy(), gen.normal_map[:4].view(np.float16).copy(), scales


def trochoid(N=256, L=64.0, steepness=0.5):
    """One trochoidal wave written into a displacement texture, D(P) = (-k^ A sin(k.P), A cos(k.P)): (tex, scales, kv, A)."""
    L = np.float32(L)
    kv = 2.0 * np.pi * np.array([2.0, 1.0]) / float(L)
    kn = np.linalg.norm(kv)
    khat = kv / kn
    A = steepness / kn
    c = (np.arange(N) + 0.5) * (float(L) / N)
    X, Z = np.meshgrid(c, c)
    ph = kv[0] * X + kv[1] * Z
    tex = np.zeros((1, N, N, 4), np.float16)
    tex[0, :, :, 0] = -khat[0] * A * np.sin(ph)
    tex[0, :, :, 1] = A * np.cos(ph)
    tex[0, :, :, 2] = -khat[1] * A * np.sin(ph)
    return tex, np.array([[1.0 / L, 1.0 / L, 1.0, 1.0]], np.float32), kv, A


def _dirs(pitch_deg, yaw):
    p = np.radians(pitch_deg)
    return np.stack([np.cos(p) * np.cos(yaw), np.sin(p), np.cos(p) * np.sin(yaw)], 1)


def ray_mix(n, seed, span=200.0):
    """n rays, a quarter of each family: camera rays (origins 1-30 m up, pitch -60 to +10 degrees), vertical rays (up and
    down, from above and below), underwater origins, and camera rays with a short t_max."""
    rng = np.random.default_rng(seed)
    r = np.zeros(n, rc.RAY)
    q = n // 4
    xz = rng.uniform(-span, span, (n, 2))
    y = np.concatenate([rng.uniform(1.0, 30.0, q), rng.uniform(-10.0, 30.0, q), rng.uniform(-15.0, -2.0, q),
                        rng.uniform(1.0, 30.0, n - 3 * q)])
    r["origin"] = np.stack([xz[:, 0], y, xz[:, 1]], 1)
    yaw = rng.uniform(0.0, 2.0 * np.pi, n)
    d = np.concatenate([_dirs(rng.uniform(-60.0, 10.0, q), yaw[:q]),
                        np.stack([np.zeros(q), rng.choice([-1.0, 1.0], q), np.zeros(q)], 1),
                        _dirs(rng.uniform(-10.0, 60.0, q), yaw[2 * q:3 * q]),
                        _dirs(rng.uniform(-60.0, 10.0, n - 3 * q), yaw[3 * q:])])
    r["direction"] = d * rng.uniform(0.5, 3.0, (n, 1))
    r["t_max"] = np.concatenate([np.full(3 * q, np.inf), rng.uniform(0.0, 20.0, n - 3 * q)])
    return r


def grazing(n, seed, span=200.0):
    """rays from inside the slab at pitches of -0.2 to -2 degrees: hundreds of samples before a crossing"""
    rng = np.random.default_rng(seed)
    r = np.zeros(n, rc.RAY)
    xz = rng.uniform(-span, span, (n, 2))
    r["origin"] = np.stack([xz[:, 0], np.full(n, 2.5), xz[:, 1]], 1)
    r["direction"] = _dirs(rng.uniform(-2.0, -0.2, n), rng.uniform(0.0, 2.0 * np.pi, n))
    r["t_max"] = np.inf
    return r


def test_record_layouts():
    from godotoceanwaves_b200.wave_generator import WaveGenerator
    assert rc.RAY.itemsize == 28 and rc.HIT.itemsize == 72
    assert list(rc.RAY.names) == ["origin", "direction", "t_max"]
    assert list(rc.HIT.names) == ["t", "position", "source_x", "source_z", "displacement", "gradient_foam", "gap", "residual",
                                  "status", "evaluations", "iterations", "unconverged"]
    assert WaveGenerator.RAY == rc.RAY and WaveGenerator.RAY_HIT == rc.HIT
    for dt, wg in [(rc.RAY, WaveGenerator.RAY), (rc.HIT, WaveGenerator.RAY_HIT)]:
        assert wg.itemsize == dt.itemsize and wg.names == dt.names
        for f in dt.names:
            assert wg.fields[f][1] == dt.fields[f][1], f
    assert (rc.MISS, rc.HIT_FROM_ABOVE, rc.HIT_FROM_BELOW, rc.TRUNCATED, rc.INVALID) == (0, 1, 2, 3, 4)


def test_flat_water_hits_at_the_analytic_parameter():
    d16 = np.zeros((2, 128, 128, 4), np.float16)
    scales = np.array([[1 / 64, 1 / 64, 1.0, 1.0], [1 / 16, 1 / 16, 0.5, 1.0]], np.float32)
    rng = np.random.default_rng(1)
    n = 400
    r = np.zeros(n, rc.RAY)
    oy = rng.integers(1, 64, n) * rng.choice([-0.25, 0.25], n)      # dyadic heights above and below
    r["origin"] = np.stack([rng.integers(-512, 512, n) * 0.5, oy, rng.integers(-512, 512, n) * 0.5], 1)
    dy = -np.sign(oy) * rng.integers(1, 8, n) * 0.125
    r["direction"] = np.stack([rng.integers(-8, 8, n) * 0.25, dy, rng.integers(-8, 8, n) * 0.25], 1)
    r["t_max"] = np.inf
    hit = rc.raycast(d16, d16, r, scales, 0.5, 1024, TOL, 8)
    assert np.array_equal(hit["status"], np.where(oy > 0, rc.HIT_FROM_ABOVE, rc.HIT_FROM_BELOW))
    assert np.all(np.abs(hit["gap"]) <= TOL)
    t_exact = -oy / dy
    # |gap| <= tolerance in binary32; the exact gap of the rounded t may exceed it by the rounding of o.y + t d.y (< 1e-5)
    assert np.all(np.abs(hit["t"] - t_exact) <= (float(TOL) + 1e-5) / np.abs(dy))
    assert np.all(hit["iterations"] == 0) and np.all(hit["residual"] == 0) and np.all(hit["unconverged"] == 0)


def test_trochoid_hits_match_a_float64_root():
    tex, scales, kv, A = trochoid()
    kn = np.linalg.norm(kv)
    khat = kv / kn
    rng = np.random.default_rng(2)
    n = 1500
    r = np.zeros(n, rc.RAY)
    r["origin"] = np.stack([rng.uniform(-100, 100, n), rng.uniform(2.5, 10.0, n), rng.uniform(-100, 100, n)], 1)   # above every crest
    # steeper than the steepest slope of the trochoid (30 degrees): one crossing per ray
    r["direction"] = _dirs(rng.uniform(-70.0, -35.0, n), rng.uniform(0.0, 2.0 * np.pi, n))
    r["t_max"] = np.inf
    hit = rc.raycast(tex, np.zeros_like(tex), r, scales, 0.25, 4096, TOL, 8)
    assert np.all(hit["status"] == rc.HIT_FROM_ABOVE)
    assert np.all(np.abs(hit["gap"]) <= TOL) and np.all(hit["residual"] <= TOL)

    # float64: the continuous trochoid's height along the ray, eta(Q) with s - A sin(|k| s) = k^.Q, and the root of
    # y(t) - eta(t) by bisection on the bracket [t - 0.05, t + 0.05] around the reported t (the gap is monotone there)
    o = r["origin"].astype(np.float64)
    d = r["direction"].astype(np.float64)

    def gap(t):
        p = o + t[:, None] * d
        q = khat[0] * p[:, 0] + khat[1] * p[:, 2]
        s = q.copy()
        for _ in range(60):
            s -= (s - A * np.sin(kn * s) - q) / (1.0 - A * kn * np.cos(kn * s))
        return p[:, 1] - A * np.cos(kn * s)

    lo = hit["t"].astype(np.float64) - 0.05
    hi = hit["t"].astype(np.float64) + 0.05
    assert np.all(gap(lo) > 0) and np.all(gap(hi) < 0)
    for _ in range(60):
        mid = 0.5 * (lo + hi)
        up = gap(mid) > 0
        lo, hi = np.where(up, mid, lo), np.where(up, hi, mid)
    t_root = 0.5 * (lo + hi)
    # the surface query's bound on the height error (tests/test_oracle_surface.py) plus the gap tolerance, over the rate at
    # which the gap falls along the ray: at least |d_y| less the steepest slope A|k| / sqrt(1 - (A|k|)^2) times |d_xz|
    h = 64.0 / 256
    e = h * h * A * kn * kn / 8.0 + A * 2.0 ** -11
    bound = e + A * kn * np.sqrt(2.0) * (e + float(TOL)) / (1.0 - A * kn) + 1e-5 + float(TOL)
    rate = np.abs(d[:, 1]) - A * kn / np.sqrt(1.0 - (A * kn) ** 2) * np.hypot(d[:, 0], d[:, 2])
    assert np.all(rate > 0)
    err = np.abs(hit["t"] - t_root) * rate
    assert err.max() <= bound, (err.max(), bound)


def test_demo_maps_ray_mix(demo_maps):
    d16, n16, scales = demo_maps
    rays = ray_mix(5000, 3)
    hit, tr = rc.raycast(d16, n16, rays, scales, 0.5, 1024, TOL, 8, trace=True)
    lo, hi, y_lo, y_hi, rho = rc.slab(d16, scales, TOL)
    assert rho == su.displacement_bound(d16, scales)
    st = hit["status"]
    hits = (st == rc.HIT_FROM_ABOVE) | (st == rc.HIT_FROM_BELOW)
    assert hits.mean() > 0.5 and np.any(st == rc.HIT_FROM_BELOW) and np.any(st == rc.MISS)
    assert not np.any(st == rc.INVALID)
    # hits resolved to |gap| <= tolerance, but for the few whose bracket closes on a jump of the inverted height (the inversion
    # ends on another preimage, or within its tolerance on either side, at adjacent binary32 parameters); every sample before a
    # hit on sample 0's side; the trace accounts for every evaluation
    assert np.mean(np.abs(hit["gap"][hits]) <= TOL) >= 0.99
    assert len(tr) == hit["evaluations"].sum()
    starts = np.concatenate([[0], np.cumsum(hit["evaluations"].astype(np.int64))[:-1]])
    for i in np.nonzero(hits)[0][:2000]:
        rows = tr[starts[i]:starts[i] + hit["evaluations"][i]]
        march = rows[rows["kind"] == 0]
        side0 = march["gap"][0] > 0
        assert np.all((march["gap"][:-1] > 0) == side0) and (march["gap"][-1] > 0) != side0
        assert np.all(np.diff(march["t"]) > 0)
        assert rows["iterations"].sum() == hit["iterations"][i]
        assert hit["status"][i] == (rc.HIT_FROM_ABOVE if side0 else rc.HIT_FROM_BELOW)
    # evaluation 0 of every ray whose origin is inside the slab is the surface query at the origin
    o = rays["origin"]
    inside = (o[:, 1] >= lo) & (o[:, 1] <= hi) & (hit["evaluations"] > 0)
    assert inside.sum() > 500
    first = tr[starts[inside]]
    assert np.all(first["t"] == 0)
    q = su.query_surface(d16, n16, o[inside][:, [0, 2]], scales, TOL, 8)
    assert first["source_x"].tobytes() == q["source_x"].tobytes() and first["source_z"].tobytes() == q["source_z"].tobytes()
    assert first["residual"].tobytes() == q["residual"].tobytes() and np.array_equal(first["iterations"], q["iterations"])
    # rays above the slab pointing up or level never evaluate
    up = (o[:, 1] > hi) & (rays["direction"][:, 1] >= 0)
    assert up.sum() > 50 and np.all(st[up] == rc.MISS) and np.all(hit["evaluations"][up] == 0)
    assert hit[up]["position"].tobytes() == o[up].tobytes() and np.all(hit["t"][up] == 0)
    # the record at the reported point is the map sample at its source
    ev = hit["evaluations"] > 0
    dd, gg = sp.sample_maps(d16, n16, np.stack([hit["source_x"][ev], hit["source_z"][ev]], 1), scales)
    assert dd.tobytes() == hit["displacement"][ev].tobytes() and gg.tobytes() == hit["gradient_foam"][ev].tobytes()
    assert np.array_equal(hit["gap"][ev], hit["position"][ev][:, 1] - dd[:, 1])


def test_heights_lie_inside_the_unpadded_slab(demo_maps):
    d16, n16, scales = demo_maps
    _, _, y_lo, y_hi, _ = rc.slab(d16, scales, TOL)
    pts = np.random.default_rng(4).uniform(-1000.0, 1000.0, (100000, 2)).astype(np.float32)
    d, _ = sp.sample_maps(d16, n16, pts, scales)
    assert y_lo < 0 < y_hi
    assert np.all(d[:, 1] >= y_lo) and np.all(d[:, 1] <= y_hi)


def test_direction_scaling_scales_t_exactly(demo_maps):
    d16, n16, scales = demo_maps
    rays = ray_mix(200, 5)
    hit = rc.raycast(d16, n16, rays, scales, 1.0, 256, TOL, 8)
    for k in (-3, 5):
        s = np.float32(2.0 ** k)
        r2 = rays.copy()
        r2["direction"] *= s
        r2["t_max"] /= s
        hit2 = rc.raycast(d16, n16, r2, scales, 1.0, 256, TOL, 8)
        assert hit2["t"].tobytes() == (hit["t"] / s).tobytes(), k
        for f in rc.HIT.names:
            if f != "t":
                assert hit2[f].tobytes() == hit[f].tobytes(), (k, f)


def test_truncation_continues_from_the_same_samples(demo_maps):
    d16, n16, scales = demo_maps
    rays = grazing(120, 6)
    hit, tr = rc.raycast(d16, n16, rays, scales, 1.0, 256, TOL, 8, trace=True)
    cap, cut = rc.raycast(d16, n16, rays, scales, 1.0, 16, TOL, 8, trace=True)
    marched = np.bincount(tr["ray"][tr["kind"] == 0], minlength=len(rays))
    long = marched > 16
    assert long.sum() > 40
    assert np.all(cap["status"][long] == rc.TRUNCATED) and np.all(cap["evaluations"][long] == 16)
    for i in np.nonzero(long)[0][:100]:
        a = tr[tr["ray"] == i][:16]
        b = cut[cut["ray"] == i]
        assert a.tobytes() == b.tobytes()
        assert cap["t"][i] == b["t"][-1] and cap["gap"][i] == b["gap"][-1]


def test_zero_iterations_is_a_height_field_march(demo_maps):
    d16, n16, scales = demo_maps
    rays = ray_mix(1000, 7)
    hit = rc.raycast(d16, n16, rays, scales, 1.0, 512, TOL, 0)
    ev = hit["evaluations"] > 0
    pos = hit["position"][ev]
    assert hit["source_x"][ev].tobytes() == pos[:, 0].tobytes() and hit["source_z"][ev].tobytes() == pos[:, 2].tobytes()
    d, _ = sp.sample_maps(d16, n16, pos[:, [0, 2]], scales)
    assert hit["gap"][ev].tobytes() == (pos[:, 1] - d[:, 1]).tobytes()
    assert np.all(hit["iterations"] == 0)


def test_invalid_rays(demo_maps):
    d16, n16, scales = demo_maps
    r = np.zeros(9, rc.RAY)
    r["origin"] = [[0, 5, 0]] * 9
    r["direction"] = [[0, -1, 0]] * 9
    r["t_max"] = np.inf
    r["origin"][0, 0] = np.nan
    r["origin"][1, 1] = np.inf
    r["direction"][2, 2] = -np.inf
    r["direction"][3] = 0
    r["direction"][4, 1] = np.nan
    r["t_max"][5] = -1.0
    r["t_max"][6] = np.nan
    r["t_max"][7] = -0.0                    # valid: t_max = 0 (-0 >= 0), one sample at most
    r["direction"][8] = [-0.0, 1e-30, 0.0]  # valid: tiny but not zero
    hit = rc.raycast(d16, n16, r, scales)
    assert np.all(hit["status"][:7] == rc.INVALID) and np.all(hit["evaluations"][:7] == 0)
    assert hit[:7].tobytes() == _invalid(7).tobytes()
    assert hit["status"][7] == rc.MISS and hit["status"][8] == rc.MISS


def _invalid(n):
    h = np.zeros(n, rc.HIT)
    h["status"] = rc.INVALID
    return h
