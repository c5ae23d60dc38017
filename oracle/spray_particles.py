"""CPU specification of the spray-particle op (ocean_spray_particles): one particle-process frame of the sea-spray emitter,
its restarts, start() and process(), with render-ready instances of the live particles.

TEST INFRASTRUCTURE ONLY -- the product path (godotoceanwaves_b200/csrc) never imports or calls this module.

Follows assets/shaders/spatial/sea_spray_particle.gdshader (hash32 :32-38, set_scale :39-43, start() :45-66,
exp_impulse :69-72, process() :74-126).  The reference does not contain Godot's particle engine: the emitter cycle below is
this library's statement of it, for a GPUParticles3D with explosiveness 0, randomness 0, local_coords = false, one_shot =
false and disable_velocity (main.tscn:133-140), not something derived from the reference.

EMITTER   amount, num_particles (the shader uniform: grid side t = uint(sqrt(float(num_particles)))), emission_transform
          (3 x 4 row-major, ocean_spray_grid's layout), particle_scale, lifetime, lifetime_randomness (uniforms),
          random_seed (RANDOM_SEED), emitter_lifetime (LIFETIME, binary64 as Godot's GPUParticles3D.lifetime).
PARTICLE  TRANSFORM as 3 x 4 row-major (columns basis x, basis y, basis z, origin), CUSTOM, USERDATA1..3, NUMBER and the
          flags ACTIVE (1) and EMITTED (2).  All zero = never emitted.  The basis is kept: set_scale re-normalises the
          previous frame's basis.

One call is the frame of emitter time [t0, t1), with TIME = (float)t1 and L = emitter_lifetime:

  restart   particle i restarts when some k >= 0 has t0 <= r_k < t1, r_k = L * ((double)k + (double)i / (double)amount)
            (binary64); the largest such k is taken.  NUMBER = k * amount + i (mod 2^32).  TRANSFORM = identity,
            CUSTOM = 0, ACTIVE and EMITTED set, then start() literally:
              rand = hash32(uvec2(NUMBER, 1) + uint(TIME) + RANDOM_SEED)             (uint32 arithmetic)
              coords = (vec2(uvec2(INDEX / t, INDEX % t)) / (float(t) - 1) - 0.5) * 10
              TRANSFORM = EMISSION_TRANSFORM * TRANSFORM, origin (coords.x, 0, coords.y)
              CUSTOM.z = rand.x;  PARTICLE_LIFETIME = lifetime - lifetime * lifetime_randomness * rand.y
              START_POS = POSITION;  START_TIME = TIME + rand.z * (LIFETIME - PARTICLE_LIFETIME);  HAS_STARTED = 0
              POSITION = (0, -1e10, 0);  set_scale(TRANSFORM, vec3(1e-3))
  process   on every ACTIVE particle (an inactive particle keeps its state until its next restart), literally:
              TIME > START_TIME + PARTICLE_LIFETIME  ->  ACTIVE = false
              else TIME >= START_TIME  ->  on the first such frame (HAS_STARTED == 0) the spawn test of oracle/spray.py at
              START_POS.xz, with PARTICLE_SCALE = vec3(foam_factor * (float(ACTIVE) + 1e-3)) * (1, nf, 1) * particle_scale
              and HAS_STARTED = 1; then, if ACTIVE:
                t = (TIME - START_TIME) / PARTICLE_LIFETIME;  CUSTOM.a = exp_impulse(t, 10)
                d = sum_i texture(displacements, START_POS.xz * map_scales[i].xy, i).xyz * map_scales[i].z
                d = d * (0.75, 1, 0.75);  d = d + (0, -5 * (2.5t - 0.45)^2 * SCALE_FACTOR + 0.5, 0)
                POSITION = START_POS + d
                size = PARTICLE_LIFETIME / lifetime;  m = vec3(size * size);  m.y *= exp_impulse(t, 3);  m.xz *= log(1 + t)
                set_scale(TRANSFORM, PARTICLE_SCALE * m)
  live      ACTIVE and HAS_STARTED != 0 after the frame.  A restarted particle that has not started yet sits at
            y = -1e10 with scale 1e-3 and is not an instance.
  instance  16 floats per live particle, in INDEX order: the 12 of TRANSFORM (basis.x.x, basis.y.x, basis.z.x, origin.x,
            ...; a Godot MultiMesh TRANSFORM_3D instance with custom data and no colours) and CUSTOM.xyzw.

Numeric policy (as oracle/spray.py): binary32, round to nearest, the shader's operation order, no contraction; IEEE division
and sqrt; normalize(v) = v / sqrt((v.x*v.x + v.y*v.y) + v.z*v.z); the mat4 product as sums in index order,
R[r][c] = ((E[r][0]*T[0][c] + E[r][1]*T[1][c]) + E[r][2]*T[2][c]) + E[r][3]*T[3][c]; exp and log are DETMATH's (the
oracle's MATH_EXP / MATH_LOG in MATH_DET mode, the device's expf_det / logf_det).  pow(a, 2.0) is taken as a * a: GLSL
leaves pow undefined for a < 0, and 2.5t - 0.45 < 0 for the first 18 % of every particle's life.  min(x, 1.0) of a NaN x
is 1.0 (IEEE minNum, the device's fminf; GLSL leaves it undefined): it decides the PARTICLE_SCALE and SCALE_FACTOR that a
NaN start position leaves in an inactive particle's state.  float(0x7FFFFFFF) is 2^31, and uint to float conversions
round to nearest.
"""
from __future__ import annotations

import numpy as np

from . import pyoracle as po
from .sampling import F, _mix, texture_bilinear

EMITTER = np.dtype([("amount", np.int32), ("num_particles", np.int32), ("emission_transform", np.float32, 12),
                    ("particle_scale", np.float32, 3), ("lifetime", np.float32), ("lifetime_randomness", np.float32),
                    ("random_seed", np.uint32), ("emitter_lifetime", np.float64)])                     # 88 B
PARTICLE = np.dtype([("transform", np.float32, 12), ("custom", np.float32, 4), ("userdata1", np.float32, 4),
                     ("userdata2", np.float32, 4), ("userdata3", np.float32, 4), ("number", np.uint32),
                     ("flags", np.uint32)])                                                          # 120 B
ACTIVE, EMITTED = 1, 2
U32 = np.uint32


def default_emitter() -> np.ndarray:
    """The reference scene's emitter (main.tscn:133-140, the shader's uniform defaults and its material's values)."""
    e = np.zeros((), EMITTER)
    e["amount"] = 32768
    e["num_particles"] = 32768
    e["emission_transform"] = (15 * np.eye(3, 4)).reshape(12)
    e["particle_scale"] = (20.0, 8.5, 20.0)
    e["lifetime"] = 3.0
    e["lifetime_randomness"] = 0.25
    e["random_seed"] = 0
    e["emitter_lifetime"] = 6.0
    return e


def hash32(px, py) -> np.ndarray:
    """sea_spray_particle.gdshader:32-38 on uint32 arrays: float32 [n][3]."""
    M = U32(1103515245)
    px, py = np.asarray(px, U32), np.asarray(py, U32)
    x = M * ((px >> U32(1)) ^ py)
    y = M * ((py >> U32(1)) ^ px)
    h = M * (x ^ (y >> U32(3)))
    n = h ^ (h >> U32(16))
    rz = (n, n * U32(16807), n * U32(48271))
    return np.stack([((r >> U32(1)) & U32(0x7FFFFFFF)).astype(np.float32) / F(2147483648.0) for r in rz], axis=-1)


def restart_cycles(amount: int, emitter_lifetime: float, t0: float, t1: float) -> np.ndarray:
    """The cycle k of each particle's restart in [t0, t1) (int64 [amount]), -1 for none: the largest k >= 0 with
    t0 <= r_k < t1, r_k = L * ((double)k + (double)i / (double)amount).  r_k is non-decreasing in k, so the largest k
    with r_k < t1 is found from an estimate by unit steps, and qualifies when r_k >= t0."""
    L, t0, t1 = np.float64(emitter_lifetime), np.float64(t0), np.float64(t1)
    f = np.arange(amount, dtype=np.float64) / np.float64(amount)

    def r(k):
        return L * (np.maximum(k, 0).astype(np.float64) + f)

    k = np.maximum(np.floor(t1 / L - f), -1.0).astype(np.int64)
    while True:
        up = r(k + 1) < t1
        if not up.any():
            break
        k = k + up
    while True:
        down = (k >= 0) & (r(k) >= t1)
        if not down.any():
            break
        k = k - down
    return np.where((k >= 0) & (r(k) >= t0), k, -1)


def _exp(x):
    return po.math_batch(po.MATH_EXP, x)[:, 0]


def _log(x):
    return po.math_batch(po.MATH_LOG, x)[:, 0]


def _exp_impulse(x, k):
    """:69-72"""
    h = F(k) * x
    return h * _exp(F(1.0) - h)


def _set_scale(T, s):
    """:39-43 on T [n][12] (3 x 4 row-major) and s [n][3]: basis column c = normalize(column c) * s[c]."""
    for c in range(3):
        x, y, z = T[:, c], T[:, 4 + c], T[:, 8 + c]
        n = np.sqrt((x * x + y * y) + z * z)
        T[:, c], T[:, 4 + c], T[:, 8 + c] = (x / n) * s[:, c], (y / n) * s[:, c], (z / n) * s[:, c]


def _start(p, idx, number, e, TIME):
    """start() :45-66 for the particles idx, after the restart's reset."""
    n = len(idx)
    u = U32(np.uint32(TIME))
    seed = U32(e["random_seed"])
    rand = hash32(number + u + seed, np.full(n, U32(1) + u + seed, U32))
    t = U32(np.sqrt(F(U32(e["num_particles"]))))
    i = idx.astype(U32)
    tm1 = F(t) - F(1.0)
    cx = ((i // t).astype(np.float32) / tm1 - F(0.5)) * F(10.0)
    cz = ((i % t).astype(np.float32) / tm1 - F(0.5)) * F(10.0)
    E = np.asarray(e["emission_transform"], np.float32).reshape(3, 4)
    one, zero = np.ones(n, np.float32), np.zeros(n, np.float32)
    Tin = (np.stack([one, zero, zero, zero]), np.stack([zero, one, zero, zero]), np.stack([zero, zero, one, zero]),
           np.stack([cx, zero, cz, one]))                            # columns of TRANSFORM; row k of column c = Tin[c][k]
    T = np.empty((n, 12), np.float32)
    for r in range(3):
        for c in range(4):
            col = Tin[c]
            T[:, 4 * r + c] = ((E[r, 0] * col[0] + E[r, 1] * col[1]) + E[r, 2] * col[2]) + E[r, 3] * col[3]
    lifetime, lr = F(e["lifetime"]), F(e["lifetime_randomness"])
    pl = lifetime - (lifetime * lr) * rand[:, 1]
    start_pos = T[:, [3, 7, 11]].copy()
    start_time = F(TIME) + rand[:, 2] * (F(e["emitter_lifetime"]) - pl)
    T[:, 3], T[:, 7], T[:, 11] = F(0.0), F(-1e10), F(0.0)
    _set_scale(T, np.full((n, 3), F(1e-3), np.float32))
    p["transform"][idx] = T
    p["custom"][idx, 2] = rand[:, 0]
    p["userdata2"][idx, 3] = pl
    p["userdata1"][idx, :3] = start_pos
    p["userdata1"][idx, 3] = start_time
    p["userdata3"][idx, 3] = F(0.0)


def _spawn_test(normal, sx, sz, scales, particle_scale):
    """process() :80-95: (active, SCALE_FACTOR, PARTICLE_SCALE [n][3]) at START_POS.xz, the arithmetic of oracle/spray.py."""
    n = len(sx)
    grad = np.zeros((n, 3), np.float32)
    for i in range(len(scales)):
        t = texture_bilinear(normal[i], sx * scales[i, 0], sz * scales[i, 1])
        grad = grad + t[:, [0, 1, 3]]
    gx, gy, foam = -grad[:, 0], -grad[:, 1], grad[:, 2]
    ny = F(1.0) / np.sqrt((gx * gx + F(1.0) * F(1.0)) + gy * gy)
    nf = _mix(F(0.25), F(1.0), np.fmin((ny - F(0.92)) / (F(0.99) - F(0.92)), F(1.0)))
    ff = _mix(F(0.25), F(1.0), np.fmin((foam - F(0.9)) / (F(1.0) - F(0.9)), F(1.0)))
    active = (nf >= F(0.0)) & (nf <= F(1.0)) & (foam > F(0.9))
    s = ff * (active.astype(np.float32) + F(1e-3))
    ps = np.asarray(particle_scale, np.float32)
    pscale = np.stack([(s * F(1.0)) * ps[0], (s * nf) * ps[1], (s * F(1.0)) * ps[2]], axis=1)
    return active, nf * ff, pscale


def _process(p, idx, e, TIME, displacement, normal, scales):
    """process() :74-126 for the ACTIVE particles idx."""
    T32 = F(TIME)
    st, pl = p["userdata1"][idx, 3], p["userdata2"][idx, 3]
    over = T32 > st + pl
    p["flags"][idx[over]] &= ~U32(ACTIVE)
    now = idx[~over & (T32 >= st)]
    first = now[p["userdata3"][now, 3] == F(0.0)]
    if len(first):
        active, sf, ps = _spawn_test(normal, p["userdata1"][first, 0], p["userdata1"][first, 2], scales, e["particle_scale"])
        p["flags"][first] = np.where(active, p["flags"][first] | U32(ACTIVE), p["flags"][first] & ~U32(ACTIVE))
        p["userdata3"][first, 2] = sf
        p["userdata2"][first, :3] = ps
        p["userdata3"][first, 3] = F(1.0)
    on = now[(p["flags"][now] & U32(ACTIVE)) != 0]
    if not len(on):
        return
    st, pl = p["userdata1"][on, 3], p["userdata2"][on, 3]
    t = (T32 - st) / pl
    p["custom"][on, 3] = _exp_impulse(t, 10.0)
    sx, sz = p["userdata1"][on, 0], p["userdata1"][on, 2]
    d = np.zeros((len(on), 3), np.float32)
    for i in range(len(scales)):
        tex = texture_bilinear(displacement[i], sx * scales[i, 0], sz * scales[i, 1])
        d = d + tex[:, :3] * scales[i, 2]
    d = d * np.array([0.75, 1.0, 0.75], np.float32)
    a = F(2.5) * t - F(0.45)
    d[:, 0] = d[:, 0] + F(0.0)
    d[:, 1] = d[:, 1] + ((F(-5.0) * (a * a)) * p["userdata3"][on, 2] + F(0.5))
    d[:, 2] = d[:, 2] + F(0.0)
    T = p["transform"][on]
    T[:, 3], T[:, 7], T[:, 11] = sx + d[:, 0], p["userdata1"][on, 1] + d[:, 1], sz + d[:, 2]
    size = pl / F(e["lifetime"])
    m = np.repeat((size * size)[:, None], 3, axis=1)
    m[:, 1] = m[:, 1] * _exp_impulse(t, 3.0)
    lg = _log(F(1.0) + t)
    m[:, 0] = m[:, 0] * lg
    m[:, 2] = m[:, 2] * lg
    _set_scale(T, p["userdata2"][on, :3] * m)
    p["transform"][on] = T


def frame(states, emitter, t0: float, t1: float, displacement, normal, map_scales, max_instances: int | None = None):
    """One call: states [amount] PARTICLE (not modified), the emitter (an EMITTER record), the frame [t0, t1), the maps
    ([C][N][N][4] float16) and map_scales [C][4].  Returns (new states, instances [min(count, max_instances)][16] float32,
    count)."""
    e = np.asarray(emitter, EMITTER).reshape(())
    amount = int(e["amount"])
    p = np.array(states, PARTICLE, copy=True).reshape(-1)
    assert len(p) == amount
    scales = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
    TIME = np.float32(t1)
    with np.errstate(all="ignore"):
        k = restart_cycles(amount, float(e["emitter_lifetime"]), t0, t1)
        idx = np.nonzero(k >= 0)[0]
        if len(idx):
            number = ((k[idx].astype(np.uint64) * np.uint64(amount) + idx.astype(np.uint64)) & np.uint64(0xFFFFFFFF)).astype(U32)
            p["transform"][idx] = np.eye(3, 4, dtype=np.float32).reshape(12)
            p["custom"][idx] = 0.0
            p["number"][idx] = number
            p["flags"][idx] |= U32(ACTIVE | EMITTED)
            _start(p, idx, number, e, TIME)
        act = np.nonzero((p["flags"] & U32(ACTIVE)) != 0)[0]
        if len(act):
            _process(p, act, e, TIME, displacement, normal, scales)
    live = ((p["flags"] & U32(ACTIVE)) != 0) & (p["userdata3"][:, 3] != F(0.0))
    count = int(live.sum())
    inst = np.concatenate([p["transform"][live], p["custom"][live]], axis=1).astype(np.float32)
    if max_instances is not None:
        inst = inst[:max_instances]
    return p, np.ascontiguousarray(inst), count
