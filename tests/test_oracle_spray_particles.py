"""CPU checks of the spray-particle specification (oracle/spray_particles.py): the shader's hash, the emitter's restart
schedule, start() against ocean_extract_spray's specification, and process() on flat maps against the closed forms of
sea_spray_particle.gdshader:97-125."""
import numpy as np
import pytest

from oracle import pyoracle as po
from oracle import spray as sy
from oracle import spray_particles as sp

F = np.float32


@pytest.fixture(autouse=True)
def _det_math():
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    yield
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)


def _hash32_int(x: int, y: int):
    """sea_spray_particle.gdshader:32-38 restated on Python ints, every product reduced modulo 2^32"""
    m, w = 1103515245, 0xFFFFFFFF
    px, py = (m * ((x >> 1) ^ y)) & w, (m * ((y >> 1) ^ x)) & w
    h = (m * (px ^ (py >> 3))) & w
    n = h ^ (h >> 16)
    return [F(F((r & w) >> 1) / F(2147483648.0)) for r in (n, n * 16807, n * 48271)]


def _emitter(amount=4096, num_particles=None, E=None, seed=0, L=6.0, lifetime=3.0, randomness=0.25):
    e = sp.default_emitter()
    e["amount"], e["num_particles"] = amount, amount if num_particles is None else num_particles
    if E is not None:
        e["emission_transform"] = np.asarray(E, np.float32).reshape(12)
    e["random_seed"], e["emitter_lifetime"], e["lifetime"], e["lifetime_randomness"] = seed, L, lifetime, randomness
    return e


def _flat_maps(C=2, N=64, foam=1.0):
    disp = np.zeros((C, N, N, 4), np.float16)
    normal = np.zeros((C, N, N, 4), np.float16)
    normal[0, ..., 3] = foam
    return disp, normal, np.array([[1 / 50, 1 / 50, 1.0, 1.0], [1 / 17, 1 / 23, 0.75, 1.0]], np.float32)[:C]


def _rotated():
    c, s = np.cos(0.6), np.sin(0.6)
    R = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]]) @ np.array([[1, 0, 0], [0, np.cos(0.3), -np.sin(0.3)], [0, np.sin(0.3), np.cos(0.3)]])
    return np.concatenate([R * [12.0, 3.0, 20.0], [[4.5], [0.25], [-7.0]]], axis=1).astype(np.float32)


def test_hash32_matches_python_ints_with_wrap_around():
    rng = np.random.default_rng(3)
    x = np.concatenate([rng.integers(0, 2 ** 32, 3000, dtype=np.uint64), [0, 1, 2 ** 32 - 1, 2 ** 31, 2 ** 31 - 1]]).astype(np.uint32)
    y = np.concatenate([rng.integers(0, 2 ** 32, 3000, dtype=np.uint64), [2 ** 32 - 1, 0, 2 ** 32 - 1, 1, 2 ** 32 - 2]]).astype(np.uint32)
    got = sp.hash32(x, y)
    want = np.array([_hash32_int(int(a), int(b)) for a, b in zip(x, y)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert got.min() >= 0.0 and got.max() <= 1.0
    # the seed and time are added with wrap-around: uvec2(NUMBER, 1) + uint(TIME) + RANDOM_SEED
    number = np.array([2 ** 32 - 5, 7], np.uint32)
    with np.errstate(over="ignore"):
        p = number + np.uint32(3) + np.uint32(2 ** 32 - 1)
    assert p.tolist() == [2 ** 32 - 3, 9]


def test_restart_schedule_three_cycles_irregular_deltas():
    amount, L = 1000, 6.0
    rng = np.random.default_rng(11)
    deltas = rng.uniform(0.001, 0.09, 10000)
    deltas[::97] = 0.0                                              # empty frames restart nothing
    t = np.concatenate([[0.0], np.cumsum(deltas)])
    t = t[t < 3 * L]
    t = np.append(t, 3 * L)
    seen = [[] for _ in range(amount)]
    for t0, t1 in zip(t[:-1], t[1:]):
        k = sp.restart_cycles(amount, L, t0, t1)
        if t0 == t1:
            assert (k < 0).all()
        for i in np.nonzero(k >= 0)[0]:
            seen[i].append(int(k[i]))
    assert all(s == [0, 1, 2] for s in seen)                          # once per cycle, in order
    numbers = [k * amount + i for i in range(amount) for k in seen[i]]
    assert len(set(numbers)) == 3 * amount


def test_number_of_restarted_particles_and_their_start_fields():
    amount = 700
    e = _emitter(amount, num_particles=1024, E=_rotated(), seed=12345)
    disp, normal, scales = _flat_maps()
    grid = sy.spray_grid(1024, _rotated())
    st = np.zeros(amount, sp.PARTICLE)
    numbers = set()
    ts = [0.0, 0.7, 2.9, 3.0, 5.99, 6.0, 6.5, 11.0, 12.1, 17.95, 18.0]
    lo = F(3.0) - (F(3.0) * F(0.25)) * F(1.0)
    for t0, t1 in zip(ts[:-1], ts[1:]):
        k = sp.restart_cycles(amount, 6.0, t0, t1)
        st, _, _ = sp.frame(st, e, t0, t1, disp, normal, scales)
        r = np.nonzero(k >= 0)[0]
        assert np.array_equal(st["number"][r], (k[r] * amount + r).astype(np.uint32))
        numbers.update(st["number"][r].tolist())
        assert np.array_equal(st["userdata1"][r][:, [0, 2]].view(np.uint32), grid[r].view(np.uint32))      # START_POS.xz
        pl, start = st["userdata2"][r, 3], st["userdata1"][r, 3]
        assert ((pl >= lo) & (pl <= F(3.0))).all()
        assert ((start >= F(t1)) & (start <= F(t1) + (F(6.0) - pl))).all()
        assert (st["flags"][r] & sp.EMITTED).all()
    assert len(numbers) == 3 * amount


def test_restart_boundaries_and_long_deltas():
    amount, L = 4, 6.0                                              # r_k = 6 (k + i / 4): exact in binary64
    k = sp.restart_cycles(amount, L, 7.5, 8.0)                      # t0 == r_1 of particle 1 restarts it
    assert k.tolist() == [-1, 1, -1, -1]
    k = sp.restart_cycles(amount, L, 7.0, 7.5)                      # t1 == r_1 of particle 1 does not
    assert k.tolist() == [-1, -1, -1, -1]
    k = sp.restart_cycles(amount, L, 6.0, 6.0)
    assert k.tolist() == [-1, -1, -1, -1]
    k = sp.restart_cycles(amount, L, 1.0, 1.0 + 2.5 * L)            # a delta longer than L: once, with the largest k
    assert k.tolist() == [2, 2, 2, 1]
    big = 1000
    k = sp.restart_cycles(big, 0.37, 5.0, 5.0 + 7.3 * 0.37)
    f = np.arange(big) / big
    r = 0.37 * (k + f)
    assert (k >= 0).all() and (r >= 5.0).all() and (r < 5.0 + 7.3 * 0.37).all()
    assert (0.37 * ((k + 1) + f) >= 5.0 + 7.3 * 0.37).all()


def test_spawn_fields_equal_the_spray_candidates():
    """With PARTICLE_LIFETIME = LIFETIME every particle starts in its restart frame: the spawn test's ACTIVE set,
    SCALE_FACTOR and PARTICLE_SCALE are those of ocean_extract_spray's specification on the same maps."""
    rng = np.random.default_rng(5)
    C, N = 3, 64
    disp = rng.normal(0, 0.5, (C, N, N, 4)).astype(np.float16)
    normal = rng.normal(0, 0.05, (C, N, N, 4)).astype(np.float16)
    normal[..., 3] = rng.uniform(0.2, 0.42, (C, N, N))
    scales = np.array([[1 / 41, 1 / 93, 1, 1], [1 / 13, 1 / 13, 0.5, 1], [1 / 3.5, 1 / 7.25, 0.25, 1]], np.float32)
    E = np.array([[7.5, 0, 0, 3.25], [0, 1, 0, 0], [0, 0, 7.5, -11.0]], np.float32)
    e = _emitter(4096, E=E, L=3.0, lifetime=3.0, randomness=0.0)
    e["particle_scale"] = (0.6, 1.4, 0.6)
    st, inst, count = sp.frame(np.zeros(4096, sp.PARTICLE), e, 0.0, 3.0, disp, normal, scales)
    ref = sy.spray_candidates(normal, sy.spray_grid(4096, E), scales, (0.6, 1.4, 0.6))
    active = np.nonzero(st["flags"] & sp.ACTIVE)[0]
    assert 0 < len(ref) < 4096 and np.array_equal(active, ref["index"].astype(np.int64))
    assert (st["userdata3"][:, 3] == 1.0).all() and count == len(ref) == len(inst)
    assert np.array_equal(st["userdata3"][active, 2].view(np.uint32), ref["scale_factor"].view(np.uint32))
    assert np.array_equal(st["userdata2"][active, :3].view(np.uint32), ref["particle_scale"].view(np.uint32))


def _run(e, disp, normal, scales, seconds=8.0, hz=30.0):
    st = np.zeros(int(e["amount"]), sp.PARTICLE)
    t, frames = 0.0, []
    while t < seconds:
        t1 = t + 1.0 / hz
        st, inst, count = sp.frame(st, e, t, t1, disp, normal, scales)
        frames.append((t1, st, inst, count))
        t = t1
    return frames


def test_flat_water_follows_the_closed_forms():
    disp, normal, scales = _flat_maps()
    e = _emitter(2048, L=6.0)
    frames = _run(e, disp, normal, scales)
    total = finite = 0
    for t1, st, inst, count in frames:
        TIME = F(t1)
        live = (st["flags"] & sp.ACTIVE).astype(bool) & (st["userdata3"][:, 3] != 0)
        assert count == live.sum() == len(inst)
        p = st[live]
        start, pl = p["userdata1"][:, 3], p["userdata2"][:, 3]
        assert (TIME <= start + pl).all() and (TIME >= start).all()  # gone after PARTICLE_LIFETIME
        t = (TIME - start) / pl
        a = 2.5 * t.astype(np.float64) - 0.45
        h64 = -5.0 * a * a + 0.5
        h = p["transform"][:, 7]
        assert np.isfinite(h).all()
        # the rounding of 2.5t is amplified by 10a: within 8 ulp of the larger term (5 at most seen)
        assert (np.abs(h - h64) <= 8 * np.spacing(np.maximum(np.abs(5.0 * a * a), 0.5).astype(np.float32))).all()
        # scales: |column| = PARTICLE_SCALE * size^2 * shaping, PARTICLE_SCALE = (1 + 1e-3) particle_scale on foam 1
        size2 = (pl.astype(np.float64) / 3.0) ** 2
        ps = 1.001 * np.array([20.0, 8.5, 20.0])
        T = p["transform"].reshape(-1, 3, 4).astype(np.float64)
        norms = np.linalg.norm(T[:, :, :3], axis=1)
        ok = np.isfinite(norms).all(axis=1)
        tt = t.astype(np.float64)
        lg = np.log((F(1.0) + t).astype(np.float64))                # log(1.0 + t) of the shader: 1 + t is rounded first
        want = np.stack([ps[0] * size2 * lg, ps[1] * size2 * 3 * tt * np.exp(1 - 3 * tt), ps[2] * size2 * lg], axis=1)
        assert np.allclose(norms[ok], want[ok], rtol=2e-5, atol=1e-6)
        total += len(p)
        finite += ok.sum()
        # the instances are the states' TRANSFORM and CUSTOM
        assert np.array_equal(inst[:, :12].view(np.uint32), p["transform"].view(np.uint32))
        assert np.array_equal(inst[:, 12:].view(np.uint32), p["custom"].view(np.uint32))
    assert total > 0 and finite >= 0.99 * total
    # below t = 0.18 the parabola's base 2.5t - 0.45 is negative: pow(a, 2) as a * a keeps the height finite
    with np.errstate(divide="ignore", invalid="ignore"):                 # never-emitted particles have PARTICLE_LIFETIME 0
        early = [(F(t1) - st["userdata1"][:, 3]) / st["userdata2"][:, 3] for t1, st, _, _ in frames]
    assert any(((x >= 0) & (x < 0.18)).any() for x in early)


def test_basis_follows_the_emitter_axes():
    disp, normal, scales = _flat_maps()
    E = _rotated()
    e = _emitter(1024, E=E, seed=77)
    axes = E[:, :3].astype(np.float64) / np.linalg.norm(E[:, :3].astype(np.float64), axis=0)
    n = 0
    for _, st, inst, count in _run(e, disp, normal, scales, seconds=4.0):
        T = inst[:, :12].reshape(-1, 3, 4).astype(np.float64)
        cols = T[:, :, :3]
        norms = np.linalg.norm(cols, axis=1)
        ok = np.all(norms > 0, axis=1) & np.isfinite(norms).all(axis=1)
        d = cols[ok] / norms[ok][:, None, :]
        assert np.allclose(d, axes[None], atol=1e-5)
        n += ok.sum()
    assert n > 0


def test_never_emitted_particles_are_left_alone():
    disp, normal, scales = _flat_maps()
    e = _emitter(64)
    st, inst, count = sp.frame(np.zeros(64, sp.PARTICLE), e, 0.0, 0.0, disp, normal, scales)
    assert count == 0 and st.tobytes() == np.zeros(64, sp.PARTICLE).tobytes()
    assert sp.PARTICLE.itemsize == 120 and sp.EMITTER.itemsize == 88
