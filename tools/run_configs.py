"""Times the BASELINE.json configs beyond the bench default, and the consumer ops, on the GPU.  Prints one JSON object per
config.

    python tools/run_configs.py [--updates] [--query] [--velocity] [--buoyancy] [--drag] [--bodies] [--raycast] [--spray-particles]
                                [--wake] [--wake-coupling] [--wake-foam] [--wake-obstacles]
                                [--wake-readers] [--sea-state] [--drifters] [--drive] [--hull]

Each flag runs its group of GROUPS; several flags run their groups in the table's order.  No flag runs --updates and then
--query.  An unknown argument exits before anything touches the GPU."""
import json
import os
import subprocess
import sys
import time
from functools import partial

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import godotoceanwaves_b200 as gow
from bench import synth_params
from godotoceanwaves_b200.native import check, load_library
from oracle import bodies as ob
from oracle import buoyancy as bu
from oracle import drag as dr
from oracle import drive as od
from oracle import hull as oh
from oracle import raycast as rc

DEV = torch.device("cuda", 0)


def warmed_generator(N, C, updates, configure=None):
    """A generator of C cascades of N x N after `updates` calls of update_all(0.02): (generator, parameters, map scales).
    configure(parameters), when given, edits the parameters before the first update."""
    g = gow.WaveGenerator()
    g.map_size = N
    g.init_gpu(max(2, C))
    p = [synth_params(gow.WaveCascadeParameters, c) for c in range(C)]
    if configure:
        configure(p)
    for _ in range(updates):
        g.update_all(0.02, p)
    return g, p, gow.WaveGenerator.map_scales(p)


def records(n, dtype):
    """A device buffer for n records of the numpy `dtype`; read it back with .cpu().numpy().view(dtype)."""
    return torch.empty(n * dtype.itemsize, dtype=torch.uint8, device=DEV)


def upload(a):
    """A numpy record array as a device buffer of its bytes."""
    return torch.from_numpy(a.view(np.uint8).copy()).to(DEV)


def seeded_points(n):
    """n device-resident points (x, z) in [-300, 300]^2 m, from seed 1."""
    return (torch.rand(n, 2, device=DEV, generator=torch.Generator(DEV).manual_seed(1)) * 600.0 - 300.0).contiguous()


def timed(g, call, reps, warmup, setup=None):
    """Milliseconds per call: setup(), `warmup` calls, a synchronise, then the generator's CUDA events around `reps` calls."""
    if setup:
        setup()
    for _ in range(warmup):
        call()
    g.synchronize()
    g.timer_start()
    for _ in range(reps):
        call()
    return g.timer_stop() / reps


def alternate(*windows, rounds=3):
    """Runs the windows (callables returning milliseconds per call) in turn for `rounds` rounds, so that clock ramp-up and
    neighbours hit each alike: one list of times per window."""
    times = [[] for _ in windows]
    for _ in range(rounds):
        for window, t in zip(windows, times):
            t.append(window())
    return times


def card(key="power_limit_and_max_sm_clock", fields="power.limit,clocks.max.sm"):
    """The card's name and its current `fields` (a --query-gpu list), as the "gpu" and `key` entries of a result line."""
    smi = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader", "-i", "0"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    return {"gpu": torch.cuda.get_device_name(0), key: smi}


def update_result(label, N, C, frames, ms, bytes_per_texel):
    texels = C * N * N * frames
    return {"config": label, "map_size": N, "cascades": C, "frames": frames, "ms_total": ms, "us_per_frame": 1e3 * ms / frames,
            "cascades_per_s": C * frames / (ms * 1e-3), "gtexels_per_s": texels / (ms * 1e-3) / 1e9,
            "algorithmic_GBps": bytes_per_texel * texels / (ms * 1e-3) / 1e9}


def run(N, C, frames, label, regen=False, fused=False):
    g, p, _ = warmed_generator(N, C, 3)
    if fused:
        g.update_frames(0.02, p, 70)    # item tables of the fused launches
    g.synchronize()
    g.timer_start()
    if fused:                           # ocean_update_frames: 256 / C frames per launch, chained on the device
        g.update_frames(0.02, p, frames)
    for f in range(0 if fused else frames):
        if regen:                       # cfg5: wind/fetch sweep, spectrum regenerated every step
            U = 5.0 + 25.0 * ((f * 7) % 26) / 25.0
            F = 10.0 ** (3.0 * ((f * 5) % 31) / 30.0)
            for q in p:
                q.wind_speed = U; q.fetch_length = F
        g.update_all(0.02, p)
    ms = g.timer_stop()
    g.free()
    print(json.dumps(update_result(label, N, C, frames, ms, 56.0 if regen else 40.0)), flush=True)


def run_sweep_batch(N, per_set, reps, label):
    """cfg5 as ONE batch: the 6 x 4 (U, F) grid points are 24 cascade sets of one generator; every step regenerates all 96
    spectra (one spectrum launch) and updates all maps (one persistent launch)."""
    grid = [(u, f) for u in (5.0, 10.0, 15.0, 20.0, 25.0, 30.0) for f in (1.0, 10.0, 100.0, 1000.0)]
    C = len(grid) * per_set

    def configure(p):
        for s, (u, f) in enumerate(grid):
            for c in range(per_set):
                p[s * per_set + c].wind_speed = u; p[s * per_set + c].fetch_length = f

    g, p, _ = warmed_generator(N, C, 3, configure)
    g.synchronize()
    g.timer_start()
    for r in range(reps):
        for q in p:
            q.should_generate_spectrum = True
        g.update_all(0.02, p)
    ms = g.timer_stop()
    g.free()
    print(json.dumps(update_result(label, N, C, reps, ms, 56.0)), flush=True)


def run_spectrum(N, C, reps, label):
    """k_spectrum_compute alone (spectrum_compute.glsl, a4): CUDA events around the launch (ocean_set_profiling), all C
    cascades dirty.  Algorithmic bytes: 16 B/texel written; the kernel is bound by the binary64 pipe (DETMATH), not by HBM."""
    g, p, _ = warmed_generator(N, C, 1)
    g.set_profiling(True)
    tot = 0.0
    for _ in range(reps):
        for q in p:
            q.should_generate_spectrum = True
        g.update_all(0.02, p)
        tot += g.last_kernel_times()[0]
    g.set_profiling(False)
    ms = tot / reps
    texels = C * N * N
    out = {"config": label, "map_size": N, "cascades": C, "kernel": "k_spectrum_compute", "us_per_launch": 1e3 * ms,
           "gtexels_per_s": texels / (ms * 1e-3) / 1e9, "algorithmic_GBps": 16.0 * texels / (ms * 1e-3) / 1e9,
           "frac_of_hbm_datasheet_3350": 16.0 * texels / (ms * 1e-3) / 1e9 / 3350.0, "bound": "fp64 pipe"}
    g.free()
    print(json.dumps(out), flush=True)


def run_spray(N, C, particles, reps, label):
    """Spray-candidate op (sea_spray_particle.gdshader:80-94) on device-resident candidates: count + scan + write kernels."""
    def configure(p):
        for q in p:
            q.whitecap = 0.9; q.foam_amount = 10.0

    g, _, scales = warmed_generator(N, C, 25, configure)
    pts = torch.from_numpy(gow.WaveGenerator.spray_grid(particles, np.array([[40, 0, 0, 0], [0, 1, 0, 0], [0, 0, 40, 0]], np.float32))).to(DEV)
    recs = records(particles, gow.WaveGenerator.SPRAY_RECORD)
    count = torch.zeros(1, dtype=torch.int32, device=DEV)
    ps = np.array([1, 1, 1], np.float32)
    lib = load_library()
    call = lambda: check(lib.ocean_extract_spray_device(g.context, particles, pts.data_ptr(), C, scales.ctypes.data, ps.ctypes.data, particles,
                                                        recs.data_ptr(), count.data_ptr()))
    per = timed(g, call, reps, 3)
    out = {"config": label, "map_size": N, "cascades": C, "candidates": particles, "active": int(count.item()), "us_per_call": 1e3 * per,
           "mcandidates_per_s": particles / (per * 1e-3) / 1e6}
    g.free()
    print(json.dumps(out), flush=True)


def run_spray_particles(N, C, amount, reps, label):
    """Spray-particle op (sea_spray_particle.gdshader start() and process()) on device-resident states: one 30 Hz
    particle-process frame per call (update + scan + write kernels), timed after 6 s of emitter time so that every
    particle has been emitted."""
    def configure(p):
        for q in p:
            q.whitecap = 0.9; q.foam_amount = 10.0

    g, _, scales = warmed_generator(N, C, 25, configure)
    e = gow.WaveGenerator.default_spray_emitter()
    e["amount"] = e["num_particles"] = amount
    states = torch.zeros(amount * gow.WaveGenerator.SPRAY_PARTICLE.itemsize, dtype=torch.uint8, device=DEV)
    inst = torch.empty(amount * 16, dtype=torch.float32, device=DEV)
    count = torch.zeros(1, dtype=torch.int32, device=DEV)
    lib = load_library()
    clock = [0.0]

    def call():
        t0 = clock[0]
        clock[0] = t0 + 1.0 / 30.0
        check(lib.ocean_spray_particles_device(g.context, e.ctypes.data, t0, clock[0], C, scales.ctypes.data, states.data_ptr(), amount, inst.data_ptr(),
                                               count.data_ptr()))

    per = alternate(lambda: timed(g, call, reps, 180 if clock[0] == 0.0 else 3))[0]
    out = {"config": label, **card(), "map_size": N, "cascades": C, "particles": amount, "live": int(count.item()),
           "us_per_call": [1e3 * v for v in per], "best_us": 1e3 * min(per), "mparticles_per_s": amount / (min(per) * 1e-3) / 1e6}
    g.free()
    print(json.dumps(out), flush=True)


def run_wake(N, sources, reps, label, substeps=8, dx=0.5):
    """Wake layer: ocean_wake_step_device with `sources` device-resident sources of radius 2 m spread over the window, moving
    at 3 m/s; `substeps` sub-steps of 1/60 s per call, the window fixed.  Per cell and sub-step the specification's step
    reads 169 values of s (13 x 13) and does 141 + 27 adds, 28 multiplies and 5 operations of the update."""
    g, _, _ = warmed_generator(128, 2, 1)
    g.wake_init(N, dx, 0.05, 32, 3.0)
    rng = np.random.default_rng(N + sources)
    s = np.zeros(sources, gow.WaveGenerator.WAKE_SOURCE)
    s["x"], s["z"] = rng.uniform(0, N * dx, sources), rng.uniform(0, N * dx, sources)
    s["vx"], s["vz"] = 3.0, 0.0
    s["radius"], s["head"], s["body"] = 2.0, 0.1, -1
    src = upload(s)
    lib = load_library()
    call = lambda: check(lib.ocean_wake_step_device(g.context, substeps / 60.0, substeps, 0, 0, sources, src.data_ptr(), 0, None))
    per = alternate(lambda: timed(g, call, reps, 3))[0]
    sub_us = [1e3 * v / substeps for v in per]
    best = min(sub_us)
    cells = N * N
    out = {"config": label, **card(), "size": N, "cell_size": dx, "sources": sources, "substeps_per_call": substeps,
           "us_per_substep": sub_us, "best_us_per_substep": best, "gcells_per_s": cells / (best * 1e-6) / 1e9,
           "smem_GBps_spec": 169 * 4 * cells / (best * 1e-6) / 1e9, "fp32_Gops_spec": 201 * cells / (best * 1e-6) / 1e9}
    g.free()
    print(json.dumps(out), flush=True)


def run_query(N, C, n_points, reps, label):
    """Map-query op (water.gdshader sampling contract) on device-resident points: kernel time only."""
    g, _, scales = warmed_generator(N, C, 2)
    pts = (torch.rand(n_points, 2, device=DEV) * 1000.0 - 500.0).contiguous()
    disp = torch.empty(n_points, 3, device=DEV)
    grad = torch.empty(n_points, 3, device=DEV)
    torch.cuda.synchronize()
    lib = load_library()
    call = lambda: check(lib.ocean_sample_maps_device(g.context, n_points, pts.data_ptr(), C, scales.ctypes.data, disp.data_ptr(), grad.data_ptr()))
    per = timed(g, call, reps, 3)
    gathered = n_points * C * 24 * 8           # 4 + 16 + 4 texel reads of 8 B per cascade and point
    out = {"config": label, "map_size": N, "cascades": C, "points": n_points, "us_per_call": 1e3 * per,
           "mpoints_per_s": n_points / (per * 1e-3) / 1e6, "gathered_GBps": gathered / (per * 1e-3) / 1e9,
           "io_GBps": n_points * 32 / (per * 1e-3) / 1e9}
    g.free()
    print(json.dumps(out), flush=True)


def run_surface(N, C, n_points, reps, label, tolerance=1e-3, max_iterations=8):
    """Surface-query op (ocean_query_surface_device) on device-resident points: kernel time from CUDA events, against
    ocean_sample_maps_device on the same points in the same run.  restarted = points that took more than max_iterations
    steps, i.e. ran the restart kernel (a first start that stalls early and then converges on a restart is not counted)."""
    g, _, scales = warmed_generator(N, C, 2)
    pts = seeded_points(n_points)
    recs = records(n_points, gow.WaveGenerator.SURFACE_SAMPLE)
    disp = torch.empty(n_points, 3, device=DEV)
    grad = torch.empty(n_points, 3, device=DEV)
    torch.cuda.synchronize()
    lib = load_library()
    query = lambda: check(lib.ocean_query_surface_device(g.context, n_points, pts.data_ptr(), C, scales.ctypes.data, tolerance, max_iterations,
                                                         recs.data_ptr()))
    sample = lambda: check(lib.ocean_sample_maps_device(g.context, n_points, pts.data_ptr(), C, scales.ctypes.data, disp.data_ptr(), grad.data_ptr()))
    t_query, t_sample = timed(g, query, reps, 3), timed(g, sample, reps, 3)
    t_query = min(t_query, timed(g, query, reps, 3))        # alternate: the first window also absorbs clock ramp-up
    rec = recs.cpu().numpy().view(gow.WaveGenerator.SURFACE_SAMPLE)
    out = {"config": label, "map_size": N, "cascades": C, "points": n_points, "tolerance": tolerance, "max_iterations": max_iterations,
           "us_per_call": 1e3 * t_query, "mpoints_per_s": n_points / (t_query * 1e-3) / 1e6, "sample_maps_us_per_call": 1e3 * t_sample,
           "ratio_to_sample_maps": t_query / t_sample, "frac_restarted": float(np.mean(rec["iterations"] > max_iterations)),
           "frac_converged": float(np.mean(rec["residual"] <= np.float32(tolerance))), "mean_iterations": float(np.mean(rec["iterations"]))}
    g.free()
    print(json.dumps(out), flush=True)


def _buoyancy_scene(n_bodies, per_body):
    """n_bodies bodies of per_body hull points each (points in [-2, 2]^3 m), random rotations, positions in [-300, 300] m
    around the surface: (bodies, hull) in the layouts of oracle/buoyancy.py."""
    rng = np.random.default_rng(1)
    hull = np.zeros(n_bodies * per_body, bu.POINT)
    hull["position"] = rng.uniform(-2.0, 2.0, (len(hull), 3))
    hull["volume"] = rng.uniform(0.01, 0.1, len(hull))
    hull["half_height"] = rng.uniform(0.05, 0.3, len(hull))
    q = rng.standard_normal((n_bodies, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                  2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                  2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], 1).reshape(n_bodies, 3, 3)
    t = np.stack([rng.uniform(-300, 300, n_bodies), rng.uniform(-1, 1, n_bodies), rng.uniform(-300, 300, n_bodies)], 1)
    bodies = np.zeros(n_bodies, bu.BODY)
    bodies["transform"] = np.concatenate([R, t[:, :, None]], 2).reshape(n_bodies, 12)
    bodies["first_point"] = np.arange(n_bodies) * per_body
    bodies["num_points"] = per_body
    return bodies, hull


def run_buoyancy(N, C, n_bodies, per_body, reps, label, tolerance=1e-3, max_iterations=8):
    """Buoyancy op (ocean_buoyancy_device) on device-resident hulls of `per_body` points per body: kernel time from CUDA
    events, against ocean_query_surface_device on the same world points in the same run, in alternating windows.  The card's
    name, power limit and max SM clock are read in the same run."""
    g, _, scales = warmed_generator(N, C, 2)
    bodies, hull = _buoyancy_scene(n_bodies, per_body)
    _, _, _, wp = bu.world_points(bodies, hull)
    n_points = len(wp)
    hull_d = upload(hull)
    pts_d = torch.from_numpy(np.ascontiguousarray(wp[:, [0, 2]])).to(DEV)
    res_d = records(n_bodies, bu.RESULT)
    recs_d = records(n_points, gow.WaveGenerator.SURFACE_SAMPLE)
    torch.cuda.synchronize()
    lib = load_library()
    buoy = lambda: check(lib.ocean_buoyancy_device(g.context, n_bodies, bodies.ctypes.data, len(hull), hull_d.data_ptr(), C, scales.ctypes.data,
                                                   1025.0, tolerance, max_iterations, res_d.data_ptr(), None))
    query = lambda: check(lib.ocean_query_surface_device(g.context, n_points, pts_d.data_ptr(), C, scales.ctypes.data, tolerance, max_iterations,
                                                         recs_d.data_ptr()))
    t_b, t_q = alternate(lambda: timed(g, buoy, reps, 3), lambda: timed(g, query, reps, 3))
    res = res_d.cpu().numpy().view(bu.RESULT)
    out = {"config": label, **card(), "map_size": N, "cascades": C,
           "bodies": n_bodies, "points_per_body": per_body, "world_points": n_points, "tolerance": tolerance, "max_iterations": max_iterations,
           "buoyancy_us_per_call": [1e3 * v for v in t_b], "query_surface_us_per_call": [1e3 * v for v in t_q],
           "overhead_over_query": min(t_b) / min(t_q) - 1.0, "mpoints_per_s": n_points / (min(t_b) * 1e-3) / 1e6,
           "frac_bodies_afloat": float(np.mean(res["submerged_volume"] > 0)),
           "frac_points_unconverged": float(res["unconverged"].sum()) / n_points}
    g.free()
    print(json.dumps(out), flush=True)


def run_body_forces(N, C, n_bodies, per_body, reps, label, tolerance=1e-3, max_iterations=8):
    """Body-forces op (ocean_body_forces_device: buoyancy plus drag) against ocean_buoyancy_device on the same bodies and
    device-resident hulls: CUDA events around each call, in alternating windows.  No velocity layer is stale inside the
    windows (the warm-up calls refresh them).  Reports both times, the overhead of the drag pass, and the fraction of world
    points that are submerged.  The card's name, power limit and max SM clock are read in the same run."""
    g, _, scales = warmed_generator(N, C, 2)
    bodies, hull = _buoyancy_scene(n_bodies, per_body)
    rng = np.random.default_rng(2)
    vel = np.zeros(n_bodies, dr.VELOCITY)
    vel["linear"] = rng.uniform(-2.0, 2.0, (n_bodies, 3))
    vel["angular"] = rng.uniform(-1.0, 1.0, (n_bodies, 3))
    cda = rng.uniform(0.01, 0.2, len(hull)).astype(np.float32)
    n_points = n_bodies * per_body
    hull_d = upload(hull)
    cda_d = torch.from_numpy(cda).to(DEV)
    hyd_d = records(n_bodies, bu.RESULT)
    drag_d = records(n_bodies, dr.RESULT)
    torch.cuda.synchronize()
    lib = load_library()
    forces = lambda: check(lib.ocean_body_forces_device(g.context, n_bodies, bodies.ctypes.data, vel.ctypes.data, len(hull), hull_d.data_ptr(),
                                                        cda_d.data_ptr(), C, scales.ctypes.data, 1025.0, tolerance, max_iterations,
                                                        hyd_d.data_ptr(), drag_d.data_ptr(), None))
    buoy = lambda: check(lib.ocean_buoyancy_device(g.context, n_bodies, bodies.ctypes.data, len(hull), hull_d.data_ptr(), C, scales.ctypes.data,
                                                   1025.0, tolerance, max_iterations, hyd_d.data_ptr(), None))
    t_f, t_b = alternate(lambda: timed(g, forces, reps, 3), lambda: timed(g, buoy, reps, 3))
    _, drag, smp = g.body_forces(bodies, vel, hull, cda, scales, 1025.0, tolerance, max_iterations, return_samples=True)
    body, j, _, wp = bu.world_points(bodies, hull)
    f = bu.submerged_fraction(smp["displacement"][:, 1], wp[:, 1], hull["half_height"][bodies["first_point"][body] + j])
    out = {"config": label, **card(), "map_size": N, "cascades": C,
           "bodies": n_bodies, "points_per_body": per_body, "world_points": n_points, "tolerance": tolerance, "max_iterations": max_iterations,
           "body_forces_us_per_call": [1e3 * v for v in t_f], "buoyancy_us_per_call": [1e3 * v for v in t_b],
           "overhead_over_buoyancy": min(t_f) / min(t_b) - 1.0, "frac_points_submerged": float(np.mean(f > 0)),
           "frac_bodies_with_drag": float(np.mean(drag["wetted_drag_area"] > 0))}
    g.free()
    print(json.dumps(out), flush=True)


def run_velocity(N, C, reps, label, sample_points=0):
    """ocean_update_velocity with every layer stale against ocean_update_all of the same cascades: CUDA events (the C ABI's
    device timer) around each call, in alternating windows of `reps` calls.  Every velocity call follows an update_all
    (which marks every layer stale) that is already queued on the stream, so the velocity kernels start right behind it.
    With sample_points, also one ocean_sample_velocity_device call against ocean_sample_maps_device on the same points.
    The card's name, power limit and SM clocks are read in the same run."""
    g, p, scales = warmed_generator(N, C, 3)
    assert g.update_velocity() == C
    g.synchronize()

    def window_update():
        tot = 0.0
        for _ in range(reps):
            g.timer_start()
            g.update_all(0.02, p)
            tot += g.timer_stop()
        return tot / reps

    def window_velocity():
        tot = 0.0
        for _ in range(reps):
            g.update_all(0.02, p)
            g.timer_start()
            n = g.update_velocity()
            tot += g.timer_stop()
            assert n == C
        return tot / reps

    t_u, t_v = alternate(window_update, window_velocity)
    texels = C * N * N
    out = {"config": label, **card("power_limit_sm_clock_max_sm_clock", "power.limit,clocks.sm,clocks.max.sm"), "map_size": N, "cascades": C,
           "velocity_us_per_call": [1e3 * v for v in t_v], "update_all_us_per_call": [1e3 * v for v in t_u],
           "velocity_over_update": min(t_v) / min(t_u), "velocity_algorithmic_GBps": 24.0 * texels / (min(t_v) * 1e-3) / 1e9}
    if sample_points:
        pts = seeded_points(sample_points)
        vel = torch.empty(sample_points, 3, device=DEV)
        disp = torch.empty(sample_points, 3, device=DEV)
        grad = torch.empty(sample_points, 3, device=DEV)
        torch.cuda.synchronize()
        lib = load_library()
        sv = lambda: check(lib.ocean_sample_velocity_device(g.context, sample_points, pts.data_ptr(), C, scales.ctypes.data, vel.data_ptr()))
        sm = lambda: check(lib.ocean_sample_maps_device(g.context, sample_points, pts.data_ptr(), C, scales.ctypes.data, disp.data_ptr(),
                                                        grad.data_ptr()))
        t_s, t_m = alternate(lambda: timed(g, sv, reps, 3), lambda: timed(g, sm, reps, 3))
        out.update({"sample_points": sample_points, "sample_velocity_us_per_call": [1e3 * v for v in t_s],
                    "sample_maps_us_per_call": [1e3 * v for v in t_m]})
    g.free()
    print(json.dumps(out), flush=True)


def _floating_scene(n_bodies, per_body):
    """_buoyancy_scene's hulls as floating bodies of 200 to 900 kg/m^3 of their hull volume, with random orientations and
    velocities: (bodies, states, hull, drag areas) in the layouts of oracle/bodies.py."""
    table, hull = _buoyancy_scene(n_bodies, per_body)
    rng = np.random.default_rng(3)
    bodies = np.zeros(n_bodies, ob.BODY)
    bodies["first_point"], bodies["num_points"] = table["first_point"], table["num_points"]
    bodies["mass"] = hull["volume"].reshape(n_bodies, per_body).sum(1) * rng.uniform(200.0, 900.0, n_bodies)
    bodies["inertia"] = bodies["mass"][:, None] * rng.uniform(0.5, 3.0, (n_bodies, 3))
    states = np.zeros(n_bodies, ob.STATE)
    states["position"] = table["transform"][:, [3, 7, 11]]
    q = rng.standard_normal((n_bodies, 4))
    states["orientation"] = q / np.linalg.norm(q, axis=1, keepdims=True)
    states["linear_velocity"] = rng.uniform(-2.0, 2.0, (n_bodies, 3))
    states["angular_velocity"] = rng.uniform(-1.0, 1.0, (n_bodies, 3))
    cda = rng.uniform(0.01, 0.2, len(hull)).astype(np.float32)
    return bodies, states, hull, cda


def run_bodies(N, C, n_bodies, per_body, substeps, reps, label, dt=1.0 / 60.0, tolerance=1e-3, max_iterations=8):
    """Floating-body integrator (ocean_simulate_bodies_device, S sub-steps per call, states in device memory) against
    S x ocean_body_forces_device on the same bodies and device-resident hulls (the integrator's own overhead), and against
    a host loop of S rounds of ocean_body_forces_device, read-back of the records and the numpy step of oracle/bodies.py
    (what the op saves a host).  Device times from CUDA events, the host loop from the wall clock after a synchronise; the
    states are restored before each window; alternating windows.  The card's name, power limit and max SM clock are read
    in the same run."""
    g, _, scales = warmed_generator(N, C, 2)
    bodies, states, hull, cda = _floating_scene(n_bodies, per_body)
    pose, vel = ob.pose(bodies, states)
    hull_d = upload(hull)
    cda_d = torch.from_numpy(cda).to(DEV)
    st0_d = upload(states)
    st_d = st0_d.clone()
    hyd_d = records(n_bodies, bu.RESULT)
    drag_d = records(n_bodies, dr.RESULT)
    torch.cuda.synchronize()
    lib = load_library()
    h = np.float32(dt) / np.float32(substeps)
    r2 = ob.radius2(bodies, hull)
    sim = lambda: check(lib.ocean_simulate_bodies_device(g.context, n_bodies, bodies.ctypes.data, st_d.data_ptr(), len(hull), hull_d.data_ptr(),
                                                         cda_d.data_ptr(), C, scales.ctypes.data, 1025.0, dt, substeps, tolerance,
                                                         max_iterations, hyd_d.data_ptr(), drag_d.data_ptr(), None))
    forces_once = lambda tbl, v: check(lib.ocean_body_forces_device(g.context, n_bodies, tbl.ctypes.data, v.ctypes.data, len(hull),
                                                                    hull_d.data_ptr(), cda_d.data_ptr(), C, scales.ctypes.data, 1025.0,
                                                                    tolerance, max_iterations, hyd_d.data_ptr(), drag_d.data_ptr(), None))

    def forces():
        for _ in range(substeps):
            forces_once(pose, vel)

    def host_loop():
        s = states
        g.synchronize()
        t0 = time.perf_counter()
        for _ in range(max(1, reps // 10)):
            for _ in range(substeps):
                tbl, v = ob.pose(bodies, s)
                forces_once(tbl, v)
                g.synchronize()                 # the records come from the generator's stream, not torch's
                hyd = hyd_d.cpu().numpy().view(bu.RESULT)
                drg = drag_d.cpu().numpy().view(dr.RESULT)
                s = ob.step(bodies, s, r2, hyd, drg, 1025.0, h)
        return (time.perf_counter() - t0) * 1e3 / max(1, reps // 10)

    restore = lambda: st_d.copy_(st0_d)
    t_s, t_f, t_h = alternate(lambda: timed(g, sim, reps, 3, restore), lambda: timed(g, forces, reps, 3, restore), host_loop)
    out = {"config": label, **card(), "map_size": N, "cascades": C,
           "bodies": n_bodies, "points_per_body": per_body, "substeps": substeps, "dt": dt, "max_iterations": max_iterations,
           "simulate_us_per_call": [1e3 * v for v in t_s], "S_x_body_forces_us": [1e3 * v for v in t_f],
           "host_loop_us_per_call": [1e3 * v for v in t_h], "overhead_over_S_x_body_forces": min(t_s) / min(t_f) - 1.0,
           "host_loop_over_simulate": min(t_h) / min(t_s)}
    g.free()
    print(json.dumps(out), flush=True)


def run_drive(N, C, n_bodies, per_body, substeps, reps, label, dt=1.0 / 60.0, tolerance=1e-3, max_iterations=8):
    """Driven bodies (ocean_simulate_driven_bodies_device) against ocean_simulate_bodies_device on the same fleet: every body
    with 2 thrusters, 2 foils and a tether to its neighbour (the last one anchored), loads on every body.  Device times from
    CUDA events, states restored before each window, alternating windows; the card's name, power limit and max SM clock are
    read in the same run."""
    g, _, scales = warmed_generator(N, C, 2)
    bodies, states, hull, cda = _floating_scene(n_bodies, per_body)
    rng = np.random.default_rng(5)
    B = n_bodies
    th = np.zeros(2 * B, od.THRUSTER)
    th["body"] = np.repeat(np.arange(B), 2)
    th["position"] = rng.uniform(-1.0, 1.0, (2 * B, 3))
    th["direction"] = (1.0, 0.0, 0.0)
    th["thrust"], th["half_height"] = 200.0, 0.3
    fo = np.zeros(2 * B, od.FOIL)
    fo["body"] = np.repeat(np.arange(B), 2)
    fo["position"] = rng.uniform(-1.0, 1.0, (2 * B, 3))
    fo["normal"] = (0.0, 0.0, 1.0)
    fo["area"], fo["half_height"] = 0.5, 0.3
    te = np.zeros(B, od.TETHER)
    te["body_a"] = np.arange(B)
    te["body_b"] = np.append(np.arange(1, B), -1)
    te["point_b"][-1] = states["position"][-1]
    ends = np.append(states["position"][1:], states["position"][-1:], 0)
    te["rest_length"] = np.linalg.norm(ends - states["position"], axis=1) * 0.99       # just taut at the start
    te["stiffness"], te["damping"] = 1e3, 50.0
    loads = np.zeros(B, od.LOAD)
    loads["force"] = (10.0, 0.0, 0.0)
    hull_d = upload(hull)
    cda_d = torch.from_numpy(cda).to(DEV)
    st0_d = upload(states)
    st_d = st0_d.clone()
    torch.cuda.synchronize()
    lib = load_library()
    plain = lambda: check(lib.ocean_simulate_bodies_device(g.context, B, bodies.ctypes.data, st_d.data_ptr(), len(hull), hull_d.data_ptr(),  # noqa: E731
                                                           cda_d.data_ptr(), C, scales.ctypes.data, 1025.0, dt, substeps, tolerance,
                                                           max_iterations, None, None, None))
    driven = lambda: check(lib.ocean_simulate_driven_bodies_device(  # noqa: E731
        g.context, B, bodies.ctypes.data, st_d.data_ptr(), len(hull), hull_d.data_ptr(), cda_d.data_ptr(), C, scales.ctypes.data, 1025.0, dt,
        substeps, tolerance, max_iterations, len(th), th.ctypes.data, len(fo), fo.ctypes.data, loads.ctypes.data, len(te), te.ctypes.data,
        None, None, None, None, None))
    restore = lambda: st_d.copy_(st0_d)  # noqa: E731
    t_p, t_d = alternate(lambda: timed(g, plain, reps, 3, restore), lambda: timed(g, driven, reps, 3, restore), rounds=5)
    out = {"config": label, **card(), "map_size": N, "cascades": C, "bodies": B, "points_per_body": per_body, "substeps": substeps,
           "thrusters": len(th), "foils": len(fo), "tethers": len(te), "simulate_us_per_call": [1e3 * v for v in t_p],
           "driven_us_per_call": [1e3 * v for v in t_d], "driven_over_simulate": min(t_d) / min(t_p) - 1.0}
    g.free()
    print(json.dumps(out), flush=True)


def _ellipsoid(nu, nv, radii):
    """A closed ellipsoid on a (u, v) grid with pinched poles, in Godot's winding: (vertices [(nv + 1) nu][3], triangles
    [2 nu nv][3])."""
    th = np.linspace(0, np.pi, nv + 1)
    ph = np.linspace(0, 2 * np.pi, nu, endpoint=False)
    grid = np.stack([np.outer(np.sin(th), np.cos(ph)), np.outer(np.cos(th), np.ones(nu)), np.outer(np.sin(th), np.sin(ph))], 2)
    idx = np.arange((nv + 1) * nu).reshape(nv + 1, nu)
    a, b, c, d = idx[:-1], np.roll(idx[:-1], -1, 1), idx[1:], np.roll(idx[1:], -1, 1)
    tris = np.concatenate([np.stack([a, c, b], -1).reshape(-1, 3), np.stack([b, c, d], -1).reshape(-1, 3)]).astype(np.int32)
    return (grid.reshape(-1, 3) * radii).astype(np.float32), tris


def run_hull(N, C, n_bodies, nu, nv, substeps, reps, label, dt=1.0 / 60.0):
    """Hull meshes (ocean_hull_forces_device, ocean_simulate_hull_bodies_device) on n_bodies sharing one ellipsoid of 2 nu nv
    triangles, against ocean_body_forces_device and ocean_simulate_bodies_device with hull points at the same vertices (the
    same surface queries): what the clip-and-reduce costs.  Device times from CUDA events, states restored before each window,
    alternating windows; the card's name, power limit and max SM clock are read in the same run."""
    g, _, scales = warmed_generator(N, C, 2)
    v, t = _ellipsoid(nu, nv, (3.0, 1.0, 1.5))
    meshes = np.zeros(1, oh.MESH)
    meshes[0] = (0, len(v), 0, len(t), 1.0, 0.05)
    vol = float(g.set_hull_meshes(meshes, v, t)[0])
    B = n_bodies
    rng = np.random.default_rng(9)
    states = np.zeros(B, ob.STATE)
    states["position"] = np.stack([rng.uniform(-300, 300, B), rng.uniform(-1, 1, B), rng.uniform(-300, 300, B)], 1)
    q = rng.standard_normal((B, 4))
    states["orientation"] = q / np.linalg.norm(q, axis=1, keepdims=True)
    states["linear_velocity"] = rng.uniform(-2.0, 2.0, (B, 3))
    hulls = np.zeros(B, oh.FLOATING)
    hulls["mass"], hulls["inertia"] = 0.5 * 1025.0 * vol, 0.5 * 1025.0 * vol
    table, vel = oh.pose(hulls, states)
    points = np.zeros(len(v), bu.POINT)
    points["position"], points["volume"], points["half_height"] = v, vol / len(v), 0.3
    bodies = np.zeros(B, ob.BODY)
    bodies["mass"], bodies["inertia"], bodies["num_points"] = hulls["mass"], hulls["inertia"], len(v)
    ptable, _ = ob.pose(bodies, states)
    hull_d = upload(points)
    cda_d = torch.from_numpy(np.full(len(v), 0.05, np.float32)).to(DEV)
    hyd_d, drag_d = records(B, bu.RESULT), records(B, dr.RESULT)
    st0_d = upload(states)
    st_d = st0_d.clone()
    torch.cuda.synchronize()
    lib = load_library()
    hull_forces = lambda: check(lib.ocean_hull_forces_device(g.context, B, table.ctypes.data, vel.ctypes.data, C, scales.ctypes.data,  # noqa: E731
                                                             1025.0, 1e-3, 8, hyd_d.data_ptr(), drag_d.data_ptr(), None))
    point_forces = lambda: check(lib.ocean_body_forces_device(g.context, B, ptable.ctypes.data, vel.ctypes.data, len(points),  # noqa: E731
                                                              hull_d.data_ptr(), cda_d.data_ptr(), C, scales.ctypes.data, 1025.0, 1e-3, 8,
                                                              hyd_d.data_ptr(), drag_d.data_ptr(), None))
    t_h, t_p = alternate(lambda: timed(g, hull_forces, reps, 3), lambda: timed(g, point_forces, reps, 3), rounds=5)
    out = {"config": label, **card(), "map_size": N, "cascades": C, "bodies": B, "triangles": len(t), "vertices": len(v),
           "hull_forces_us": [1e3 * x for x in t_h], "point_forces_us": [1e3 * x for x in t_p],
           "hull_over_points": min(t_h) / min(t_p) - 1.0}
    if substeps:
        restore = lambda: st_d.copy_(st0_d)  # noqa: E731
        hull_sim = lambda: check(lib.ocean_simulate_hull_bodies_device(g.context, B, hulls.ctypes.data, st_d.data_ptr(), C,  # noqa: E731
                                                                       scales.ctypes.data, 1025.0, dt, substeps, 1e-3, 8, None, None, None))
        point_sim = lambda: check(lib.ocean_simulate_bodies_device(g.context, B, bodies.ctypes.data, st_d.data_ptr(), len(points),  # noqa: E731
                                                                   hull_d.data_ptr(), cda_d.data_ptr(), C, scales.ctypes.data, 1025.0, dt,
                                                                   substeps, 1e-3, 8, None, None, None))
        s_h, s_p = alternate(lambda: timed(g, hull_sim, reps, 3, restore), lambda: timed(g, point_sim, reps, 3, restore), rounds=5)
        out.update(substeps=substeps, simulate_hull_us=[1e3 * x for x in s_h], simulate_points_us=[1e3 * x for x in s_p],
                   simulate_hull_over_points=min(s_h) / min(s_p) - 1.0)
    g.free()
    print(json.dumps(out), flush=True)


def run_simulate_coupling(N, C, n_bodies, per_body, substeps, reps, label, wake=512, dx=1.0, dt=1.0 / 60.0):
    """Wake coupling's cost in the body integrator: ocean_simulate_bodies_device on two generators with the same maps and a
    wake layer of wake x wake cells of dx centred on the world origin (it covers [-256, 256]^2 m of the scene's
    [-300, 300]^2 m), coupled (primed by one step with 64 sources) and uncoupled.  Device times from CUDA events, the states
    restored before each window, alternating windows; the card's name, power limit and max SM clock read in the same run."""
    bodies, states, hull, cda = _floating_scene(n_bodies, per_body)
    rng = np.random.default_rng(4)
    s = np.zeros(64, gow.WaveGenerator.WAKE_SOURCE)
    s["x"], s["z"] = rng.uniform(-200, 200, 64), rng.uniform(-200, 200, 64)
    s["vx"], s["radius"], s["head"], s["body"] = 3.0, 3.0, 0.2, -1
    lib = load_library()
    hull_d = upload(hull)
    cda_d = torch.from_numpy(cda).to(DEV)
    st0_d = upload(states)
    runs = []
    for coupled in (False, True):
        g, _, scales = warmed_generator(N, C, 2)
        g.wake_init(wake, dx, 0.05, 32, 3.0)
        g.wake_set_coupling(coupled)
        g.wake_step(0.1, 2, (-wake // 2, -wake // 2), s)
        st_d = st0_d.clone()
        torch.cuda.synchronize()
        sim = partial(lambda g, st_d, sc: check(lib.ocean_simulate_bodies_device(
            g.context, n_bodies, bodies.ctypes.data, st_d.data_ptr(), len(hull), hull_d.data_ptr(), cda_d.data_ptr(), C, sc.ctypes.data,
            1025.0, dt, substeps, 1e-3, 8, None, None, None)), g, st_d, scales)
        runs.append((g, sim, partial(lambda st_d: st_d.copy_(st0_d), st_d)))
    t_off, t_on = alternate(*[partial(lambda g, sim, restore: timed(g, sim, reps, 3, restore), *r) for r in runs])
    out = {"config": label, **card(), "map_size": N, "cascades": C, "bodies": n_bodies, "points_per_body": per_body,
           "substeps": substeps, "wake_size": wake, "wake_cell_size": dx,
           "uncoupled_us_per_call": [1e3 * v for v in t_off], "coupled_us_per_call": [1e3 * v for v in t_on],
           "coupled_over_uncoupled": min(t_on) / min(t_off) - 1.0}
    for g, _, _ in runs:
        g.free()
    print(json.dumps(out), flush=True)


def run_wake_step_coupling(N, sources, reps, label, substeps=8, dx=0.5):
    """Wake coupling's cost in the step call: run_wake's ocean_wake_step_device with the coupling off and on (one more
    kernel per call, the free surface e = h + phi at the end of the call); alternating windows on one generator."""
    g, _, _ = warmed_generator(128, 2, 1)
    g.wake_init(N, dx, 0.05, 32, 3.0)
    rng = np.random.default_rng(N + sources)
    s = np.zeros(sources, gow.WaveGenerator.WAKE_SOURCE)
    s["x"], s["z"] = rng.uniform(0, N * dx, sources), rng.uniform(0, N * dx, sources)
    s["vx"], s["vz"] = 3.0, 0.0
    s["radius"], s["head"], s["body"] = 2.0, 0.1, -1
    src = upload(s)
    lib = load_library()
    call = lambda: check(lib.ocean_wake_step_device(g.context, substeps / 60.0, substeps, 0, 0, sources, src.data_ptr(), 0, None))
    t_off, t_on = alternate(lambda: timed(g, call, reps, 3, lambda: g.wake_set_coupling(False)),
                            lambda: timed(g, call, reps, 3, lambda: g.wake_set_coupling(True)))
    out = {"config": label, **card(), "size": N, "cell_size": dx, "sources": sources, "substeps_per_call": substeps,
           "uncoupled_us_per_call": [1e3 * v for v in t_off], "coupled_us_per_call": [1e3 * v for v in t_on],
           "free_surface_us_per_call": 1e3 * (min(t_on) - min(t_off))}
    g.free()
    print(json.dumps(out), flush=True)


def run_wake_readers(reps, label, N=256, C=4, wake=512, dx=0.5):
    """Wake readers' cost (ocean_wake_set_readers): readers off against on, alternating windows on one generator, over C
    cascades of N x N and a coupled, foamed wake x wake layer stirred by 64 moving sources:
      the ray cast, 2^20 picking rays (run_raycast's scene a): one more kernel (the bounds of e) and one bilinear sample of e
      per evaluation;
      ocean_extract_spray_device on 2^20 candidates over the wake's window;
      ocean_spray_particles_device with 32768 and 2^20 particles, one 30 Hz frame per call after 6 s of emitter time."""
    g, _, scales = warmed_generator(N, C, 2)
    g.wake_init(wake, dx, 0.05, 32, 3.0)
    g.wake_set_coupling(True)
    g.wake_set_foam(0.05, 1.0, 0.2, 0.3)
    ext = wake * dx
    rng = np.random.default_rng(wake)
    s = np.zeros(64, gow.WaveGenerator.WAKE_SOURCE)
    s["x"], s["z"] = rng.uniform(-0.4 * ext, 0.4 * ext, 64), rng.uniform(-0.4 * ext, 0.4 * ext, 64)
    s["vx"], s["vz"] = rng.uniform(-6, 6, 64), rng.uniform(-6, 6, 64)
    s["radius"], s["head"], s["body"] = 2.0, 0.2, -1
    for _ in range(20):
        g.wake_step(0.1, 4, (-wake // 2, -wake // 2), s)
    lib = load_library()
    gpu = card()
    readers = lambda on: (lambda: g.wake_set_readers(raycast=on, spray=on))
    out = {"config": label, **gpu, "map_size": N, "cascades": C, "wake_size": wake, "cell_size": dx}
    rays = _picking_rays(1024)
    n = len(rays)
    rays_d = upload(rays)
    hits = records(n, rc.HIT)
    cast = lambda: check(lib.ocean_raycast_device(g.context, n, rays_d.data_ptr(), C, scales.ctypes.data, 0.5, 1024, 1e-3, 8,
                                                  hits.data_ptr()))
    t_off, t_on = alternate(lambda: timed(g, cast, reps, 2, readers(False)), lambda: timed(g, cast, reps, 2, readers(True)))
    out["raycast_2^20_ms"] = {"off": t_off, "on": t_on, "on_over_off": min(t_on) / min(t_off) - 1.0}
    m = 1 << 20
    E = np.array([[ext / 20, 0, 0, 0], [0, 1, 0, 0], [0, 0, ext / 20, 0]], np.float32)
    pts = torch.from_numpy(gow.WaveGenerator.spray_grid(m, E)).to(DEV)
    recs = records(m, gow.WaveGenerator.SPRAY_RECORD)
    count = torch.zeros(1, dtype=torch.int32, device=DEV)
    ps = np.array([1, 1, 1], np.float32)
    extract = lambda: check(lib.ocean_extract_spray_device(g.context, m, pts.data_ptr(), C, scales.ctypes.data, ps.ctypes.data, m,
                                                           recs.data_ptr(), count.data_ptr()))
    t_off, t_on = alternate(lambda: timed(g, extract, reps, 2, readers(False)), lambda: timed(g, extract, reps, 2, readers(True)))
    out["extract_spray_2^20_ms"] = {"off": t_off, "on": t_on, "on_over_off": min(t_on) / min(t_off) - 1.0, "active_on": int(count.item())}
    for amount in (32768, 1 << 20):
        e = gow.WaveGenerator.default_spray_emitter()
        e["amount"] = e["num_particles"] = amount
        e["emission_transform"] = E.reshape(12) if amount > 32768 else (15 * np.eye(3, 4)).reshape(12)
        states = torch.zeros(amount * gow.WaveGenerator.SPRAY_PARTICLE.itemsize, dtype=torch.uint8, device=DEV)
        inst = torch.empty(amount * 16, dtype=torch.float32, device=DEV)
        live = torch.zeros(1, dtype=torch.int32, device=DEV)
        clock = [0.0]

        def frame():
            t0 = clock[0]
            clock[0] = t0 + 1.0 / 30.0
            check(lib.ocean_spray_particles_device(g.context, e.ctypes.data, t0, clock[0], C, scales.ctypes.data, states.data_ptr(), amount,
                                                   inst.data_ptr(), live.data_ptr()))

        for _ in range(180):                           # 6 s of emitter time: every particle emitted
            frame()
        t_off, t_on = alternate(lambda: timed(g, frame, reps, 2, readers(False)), lambda: timed(g, frame, reps, 2, readers(True)))
        out[f"spray_particles_{amount}_ms"] = {"off": t_off, "on": t_on, "on_over_off": min(t_on) / min(t_off) - 1.0}
    g.free()
    print(json.dumps(out), flush=True)


def run_sea_state(N, C, reps, label):
    """The sea-state reduction (ocean_get_sea_state) with every cascade stale: each of `reps` rounds injects the spectra again
    (ocean_set_spectrum_amplitudes, outside the window), then the generator's CUDA events bracket one call -- its two kernels
    and the 10 C binary64 moments' copy to the host; the host wall time of the call, synchronise included, beside them."""
    g, p, scales = warmed_generator(N, C, 1)
    g.sea_state(scales)
    amps = [g.spectrum_to_host(c)[..., :2].copy().view(np.complex64)[..., 0] for c in range(C)]
    dev_ms, wall_us = [], []
    for _ in range(reps):
        for c in range(C):
            g.set_spectrum_amplitudes(c, amps[c])
        g.synchronize()
        t0 = time.perf_counter()
        g.timer_start()
        g.sea_state(scales)
        dev_ms.append(g.timer_stop())
        wall_us.append((time.perf_counter() - t0) * 1e6)
    spectrum_bytes = C * N * N * 16
    best = min(dev_ms)
    print(json.dumps({"config": label, **card(), "map_size": N, "cascades": C, "device_ms": sorted(dev_ms), "host_wall_us": sorted(wall_us),
                      "spectrum_MiB": spectrum_bytes / 2**20, "spectrum_GBps_at_best": spectrum_bytes / (best * 1e-3) / 1e9}), flush=True)
    g.free()


def run_drift(N, C, n, reps, label, wake=512, dx=0.5):
    """ocean_drift_device on n drifters with dt = 1/60 s, a current, wind and the wrap, wake read off against on (alternating
    windows on one generator; the sea state is fresh, so each call is the drift kernel alone).  The drifters lie in a 400 m box
    around the 512 x 512 wake window (16 moving sources), so the wake form samples the layer for part of them.  Per drifter the
    kernel reads and writes its 40 B record and writes a 48 B instance: 128 B of state traffic, beside the map gathers."""
    g, _, scales = warmed_generator(N, C, 2)
    g.wake_init(wake, dx, 0.05, 32, 3.0)
    ext = wake * dx
    rng = np.random.default_rng(n)
    s = np.zeros(16, gow.WaveGenerator.WAKE_SOURCE)
    s["x"], s["z"] = rng.uniform(-0.4 * ext, 0.4 * ext, 16), rng.uniform(-0.4 * ext, 0.4 * ext, 16)
    s["vx"], s["vz"] = rng.uniform(-6, 6, 16), rng.uniform(-6, 6, 16)
    s["radius"], s["head"], s["body"] = 2.0, 0.2, -1
    for _ in range(10):
        g.wake_step(0.1, 4, (-wake // 2, -wake // 2), s)
    d = np.zeros(n, gow.WaveGenerator.DRIFTER)
    d["x"], d["z"] = rng.uniform(-200, 200, n), rng.uniform(-200, 200, n)
    d["yaw"], d["yaw_rate"] = rng.uniform(-3, 3, n), rng.uniform(-1, 1, n)
    d["windage"], d["tilt"], d["scale"] = 0.02, 0.5, 1.0
    drifters = upload(d)
    inst = torch.empty(n * 12, dtype=torch.float32, device=DEV)
    lib = load_library()
    params = {on: gow.WaveGenerator.drift_params(current=(0.2, 0.1), wind=(6.0, 2.0), box=(-200.0, -200.0, 400.0, 400.0), read_wake=on)
              for on in (False, True)}
    call = lambda on: (lambda: check(lib.ocean_drift_device(g.context, 1.0 / 60.0, params[on].ctypes.data, n, drifters.data_ptr(), C,
                                                             scales.ctypes.data, inst.data_ptr())))
    call(False)()
    t_off, t_on = alternate(lambda: timed(g, call(False), reps, 3), lambda: timed(g, call(True), reps, 3))
    state_bytes = n * (2 * gow.WaveGenerator.DRIFTER.itemsize + 48)
    print(json.dumps({"config": label, **card(), "map_size": N, "cascades": C, "drifters": n, "wake_size": wake,
                      "ms_per_call": {"wake_off": t_off, "wake_on": t_on}, "us_per_call_best": {"wake_off": 1e3 * min(t_off), "wake_on": 1e3 * min(t_on)},
                      "state_GBps_at_best": {"wake_off": state_bytes / (min(t_off) * 1e-3) / 1e9, "wake_on": state_bytes / (min(t_on) * 1e-3) / 1e9}}),
          flush=True)
    g.free()


def run_wake_step_foam(N, sources, reps, label, substeps=8, dx=0.5):
    """Wake foam's cost in the step call: run_wake's ocean_wake_step_device with foam off and on (the foam form of the
    sub-step kernel: |v|^2 carried by the cull, w^2 |v|^2 summed beside phi, one more 4 B read and write per cell);
    alternating windows on one generator."""
    g, _, _ = warmed_generator(128, 2, 1)
    g.wake_init(N, dx, 0.05, 32, 3.0)
    rng = np.random.default_rng(N + sources)
    s = np.zeros(sources, gow.WaveGenerator.WAKE_SOURCE)
    s["x"], s["z"] = rng.uniform(0, N * dx, sources), rng.uniform(0, N * dx, sources)
    s["vx"], s["vz"] = 3.0, 0.0
    s["radius"], s["head"], s["body"] = 2.0, 0.1, -1
    src = upload(s)
    lib = load_library()
    call = lambda: check(lib.ocean_wake_step_device(g.context, substeps / 60.0, substeps, 0, 0, sources, src.data_ptr(), 0, None))
    t_off, t_on = alternate(lambda: timed(g, call, reps, 3, lambda: g.wake_set_foam(None)),
                            lambda: timed(g, call, reps, 3, lambda: g.wake_set_foam(0.05, 1.0, 0.05, 0.5)))
    out = {"config": label, **card(), "size": N, "cell_size": dx, "sources": sources, "substeps_per_call": substeps,
           "foam_off_us_per_call": [1e3 * v for v in t_off], "foam_on_us_per_call": [1e3 * v for v in t_on],
           "foam_us_per_call": 1e3 * (min(t_on) - min(t_off)), "foam_on_over_off": min(t_on) / min(t_off) - 1.0}
    g.free()
    print(json.dumps(out), flush=True)


def run_wake_step_obstacles(N, sources, reps, label, substeps=8, dx=0.5):
    """Wake obstacles' cost in the step call: run_wake's ocean_wake_step_device with no mask, with a coastline mask over the
    window (the rows z >= 0.6 N plus a wavy shore: about 40 % of the cells blocked) and with the same mask moved entirely
    outside the window (the obstacle form still runs, reading nothing but open cells); alternating windows on one generator."""
    g, _, _ = warmed_generator(128, 2, 1)
    g.wake_init(N, dx, 0.05, 32, 3.0)
    rng = np.random.default_rng(N + sources)
    s = np.zeros(sources, gow.WaveGenerator.WAKE_SOURCE)
    s["x"], s["z"] = rng.uniform(0, N * dx, sources), rng.uniform(0, 0.55 * N * dx, sources)
    s["vx"], s["vz"] = 3.0, 0.0
    s["radius"], s["head"], s["body"] = 2.0, 0.1, -1
    src = upload(s)
    q = np.arange(N)
    shore = (0.6 * N + 0.05 * N * np.sin(q * 4 * np.pi / N)).astype(int)
    mask = (np.arange(N)[:, None] >= shore[None, :]).astype(np.uint8)
    lib = load_library()
    call = lambda: check(lib.ocean_wake_step_device(g.context, substeps / 60.0, substeps, 0, 0, sources, src.data_ptr(), 0, None))
    t_off, t_on, t_out = alternate(lambda: timed(g, call, reps, 3, lambda: g.wake_set_obstacles(None)),
                                   lambda: timed(g, call, reps, 3, lambda: g.wake_set_obstacles(mask, (0, 0))),
                                   lambda: timed(g, call, reps, 3, lambda: g.wake_set_obstacles(mask, (10 * N, 0))))
    out = {"config": label, **card(), "size": N, "cell_size": dx, "sources": sources, "substeps_per_call": substeps,
           "blocked_share": float(mask.mean()),
           "mask_off_us_per_call": [1e3 * v for v in t_off], "coastline_us_per_call": [1e3 * v for v in t_on],
           "outside_us_per_call": [1e3 * v for v in t_out],
           "coastline_over_off": min(t_on) / min(t_off) - 1.0, "outside_over_off": min(t_out) / min(t_off) - 1.0}
    g.free()
    print(json.dumps(out), flush=True)


def _picking_rays(side, y=12.0, fov_deg=90.0, pitch_deg=-20.0):
    """side x side camera rays from (0, y, 0) through a square image plane of fov_deg pitched pitch_deg: (RAY array)."""
    f = np.tan(np.radians(fov_deg) / 2.0)
    u = (np.arange(side) + 0.5) / side * 2.0 - 1.0
    U, V = np.meshgrid(u * f, u * f)
    p = np.radians(pitch_deg)
    fwd = np.array([0.0, np.sin(p), np.cos(p)]); up = np.array([0.0, np.cos(p), -np.sin(p)]); right = np.array([1.0, 0.0, 0.0])
    d = fwd[None, :] + U.reshape(-1, 1) * right[None, :] + V.reshape(-1, 1) * up[None, :]
    r = np.zeros(side * side, rc.RAY)
    r["origin"] = [0.0, y, 0.0]
    r["direction"] = d / np.linalg.norm(d, axis=1, keepdims=True)
    r["t_max"] = np.inf
    return r


def _projectile_rays(n, seed=1):
    """n rays 30 to 90 degrees down from 5 to 50 m over [-300, 300]^2 m"""
    rng = np.random.default_rng(seed)
    p = np.radians(rng.uniform(-90.0, -30.0, n))
    yaw = rng.uniform(0.0, 2.0 * np.pi, n)
    r = np.zeros(n, rc.RAY)
    r["origin"] = np.stack([rng.uniform(-300, 300, n), rng.uniform(5.0, 50.0, n), rng.uniform(-300, 300, n)], 1)
    r["direction"] = np.stack([np.cos(p) * np.cos(yaw), np.sin(p), np.cos(p) * np.sin(yaw)], 1)
    r["t_max"] = np.inf
    return r


def run_raycast(N, C, reps, label, step=0.5, max_samples=1024, tolerance=1e-3, max_iterations=8):
    """Ray cast (ocean_raycast_device) on device-resident rays, two scenes: (a) 2^20 picking rays from a camera 12 m up
    through a 1024 x 1024 grid over a 90 degree field of view pitched 20 degrees down, (b) 2^16 projectile rays 30 to 90
    degrees down from 5 to 50 m.  CUDA events around each call, best of three windows alternating with
    ocean_query_surface_device on 2^20 points.  The card's name, power limit and max SM clock are read in the same run."""
    g, _, scales = warmed_generator(N, C, 2)
    lib = load_library()
    n_pts = 1 << 20
    pts = seeded_points(n_pts)
    recs = records(n_pts, gow.WaveGenerator.SURFACE_SAMPLE)
    query = lambda: check(lib.ocean_query_surface_device(g.context, n_pts, pts.data_ptr(), C, scales.ctypes.data, tolerance, max_iterations,
                                                         recs.data_ptr()))
    gpu = card()
    for scene, rays in (("picking: 2^20 rays, camera 12 m up, 90 deg fov pitched 20 deg down", _picking_rays(1024)),
                        ("projectiles: 2^16 rays 30-90 deg down from 5-50 m", _projectile_rays(1 << 16))):
        n = len(rays)
        rays_d = upload(rays)
        out_d = records(n, rc.HIT)
        cast = lambda: check(lib.ocean_raycast_device(g.context, n, rays_d.data_ptr(), C, scales.ctypes.data, step, max_samples, tolerance,
                                                      max_iterations, out_d.data_ptr()))
        t_r, t_q = alternate(lambda: timed(g, cast, reps, 2), lambda: timed(g, query, reps, 2))
        hit = out_d.cpu().numpy().view(rc.HIT)
        st = hit["status"]
        out = {"config": label, "scene": scene, **gpu, "map_size": N,
               "cascades": C, "rays": n, "step": step, "max_samples": max_samples, "tolerance": tolerance, "max_iterations": max_iterations,
               "raycast_us_per_call": [1e3 * v for v in t_r], "best_us": 1e3 * min(t_r), "mrays_per_s": n / (min(t_r) * 1e-3) / 1e6,
               "query_surface_2e20_us_per_call": [1e3 * v for v in t_q], "mean_evaluations": float(hit["evaluations"].mean()),
               "mean_newton_steps": float(hit["iterations"].mean()),
               "frac_hit": float(np.mean((st == rc.HIT_FROM_ABOVE) | (st == rc.HIT_FROM_BELOW))),
               "frac_truncated": float(np.mean(st == rc.TRUNCATED)), "frac_miss": float(np.mean(st == rc.MISS)),
               "frac_invalid": float(np.mean(st == rc.INVALID)),
               "frac_rays_with_unconverged": float(np.mean(hit["unconverged"] > 0)),
               "frac_evaluations_unconverged": float(hit["unconverged"].sum() / max(1, hit["evaluations"].sum()))}
        print(json.dumps(out), flush=True)
    g.free()


GROUPS = {          # flag: its configs, in the order they run
    "--updates": [
        partial(run, 256, 4, 2000, "cfg2 latency: one 256x256x4 set per launch (launch/latency-bound, L2-resident)"),
        partial(run, 256, 4, 2000, "cfg2 latency, fused frames (ocean_update_frames: 64 frames per launch)", fused=True),
        partial(run, 512, 4, 1000, "cfg3: 512x512x4, 1000-frame foam accumulate/decay loop, frame by frame"),
        partial(run, 512, 4, 1000, "cfg3: 512x512x4, 1000-frame foam accumulate/decay loop, fused frames (ocean_update_frames)", fused=True),
        partial(run, 1024, 8, 200, "cfg4 (1 GPU): 1024x1024x8"),
        partial(run, 256, 4, 300, "cfg5: 256x256x4 wind/fetch sweep, one grid point per step, spectrum regenerated every step", regen=True),
        partial(run_sweep_batch, 256, 4, 50, "cfg5 batched: the 6x4 (U,F) grid = 24 sets x 4 cascades per step, all spectra regenerated every step"),
        partial(run, 128, 1, 2000, "cfg1 shape on GPU: 128x128x1"),
        partial(run_spectrum, 256, 128, 10, "spectrum generation alone: 128 cascades of 256x256, one launch"),
        partial(run_spray, 256, 4, 1 << 20, 50, "spray candidates: 2^20 grid candidates x 4 cascades of 256x256"),
    ],
    "--query": [
        partial(run_query, 256, 4, 1 << 20, 50, "query op: 2^20 random points x 4 cascades of 256x256 (maps L2-resident)"),
        partial(run_query, 1024, 8, 1 << 20, 20, "query op: 2^20 random points x 8 cascades of 1024x1024 (maps 128 MiB)"),
        partial(run_surface, 256, 4, 1 << 20, 50, "surface query: 2^20 points in [-300, 300]^2 m x 4 cascades of 256x256"),
        partial(run_surface, 1024, 8, 1 << 20, 20, "surface query: 2^20 points in [-300, 300]^2 m x 8 cascades of 1024x1024"),
    ],
    "--velocity": [
        partial(run_velocity, 256, 4, 200, "velocity: 4 cascades of 256x256, every layer stale", sample_points=1 << 20),
        partial(run_velocity, 256, 128, 50, "velocity: the bench workload, 128 cascades of 256x256, every layer stale"),
        partial(run_velocity, 1024, 8, 20, "velocity: 8 cascades of 1024x1024, every layer stale"),
    ],
    "--buoyancy": [
        partial(run_buoyancy, 256, 4, 1 << 14, 64, 50, "buoyancy: 2^14 bodies x 64 points over 4 cascades of 256x256"),
        partial(run_buoyancy, 1024, 8, 1 << 14, 64, 20, "buoyancy: 2^14 bodies x 64 points over 8 cascades of 1024x1024"),
    ],
    "--drag": [
        partial(run_body_forces, 256, 4, 1 << 14, 64, 50, "body forces: 2^14 bodies x 64 points over 4 cascades of 256x256"),
        partial(run_body_forces, 1024, 8, 1 << 14, 64, 20, "body forces: 2^14 bodies x 64 points over 8 cascades of 1024x1024"),
    ],
    "--bodies": [
        partial(run_bodies, N, C, 1 << 14, 64, S, reps,
                f"floating bodies: 2^14 bodies x 64 points, {S} sub-step(s) of 1/60 s, {C} cascades of {N}x{N}")
        for S in (1, 4) for N, C, reps in ((256, 4, 50), (1024, 8, 20))
    ],
    "--raycast": [
        partial(run_raycast, 256, 4, 20, "ray cast over 4 cascades of 256x256"),
        partial(run_raycast, 1024, 8, 10, "ray cast over 8 cascades of 1024x1024"),
    ],
    "--spray-particles": [
        partial(run_spray_particles, 256, 4, 32768, 100, "spray particles: the reference emitter (32768 particles) over 4 cascades of 256x256"),
        partial(run_spray_particles, 256, 4, 1 << 20, 50, "spray particles: 2^20 particles over 4 cascades of 256x256"),
    ],
    "--wake": [
        partial(run_wake, N, k, 200 if N < 1024 else 50, f"wake layer: {N}x{N} cells, {k} source(s)")
        for N in (256, 512, 1024) for k in (1, 64, 1024)
    ],
    "--wake-coupling": [
        *[partial(run_simulate_coupling, N, C, 1 << 14, 64, S, reps,
                  f"wake coupling, simulate: 2^14 bodies x 64 points, {S} sub-step(s), {C} cascades of {N}x{N}, 512x512 wake")
          for S in (1, 4) for N, C, reps in ((256, 4, 50), (1024, 8, 20))],
        *[partial(run_wake_step_coupling, N, k, 200 if N < 1024 else 50, f"wake coupling, step: {N}x{N} cells, {k} source(s), 8 sub-steps")
          for N in (256, 512, 1024) for k in (1, 64, 1024)],
    ],
    "--wake-foam": [
        partial(run_wake_step_foam, N, k, 200 if N < 1024 else 50, f"wake foam, step: {N}x{N} cells, {k} source(s), 8 sub-steps")
        for N in (256, 512, 1024) for k in (1, 64, 1024)
    ],
    "--wake-readers": [
        partial(run_wake_readers, 20, "wake readers: ray cast, spray and spray particles, readers off vs on, 4 cascades of 256x256, "
                                      "coupled 512x512 wake with foam"),
    ],
    "--sea-state": [
        partial(run_sea_state, 1024, 8, 10, "sea state: the reduction over 8 cascades of 1024x1024, every cascade stale"),
    ],
    "--drifters": [
        partial(run_drift, N, 4, n, 200 if n < (1 << 20) else 50, f"drifters: {'2^16' if n < (1 << 20) else '2^20'} over 4 cascades of {N}x{N}, "
                "wake read off vs on")
        for N in (256, 1024) for n in (1 << 16, 1 << 20)
    ],
    "--drive": [
        partial(run_drive, N, C, 1 << 14, 64, S, reps,
                f"driven bodies: 2^14 bodies x 64 points, 2 thrusters, 2 foils and a tether each, {S} sub-step(s), {C} cascades of {N}x{N}, "
                "vs simulate_bodies")
        for S in (1, 4) for N, C, reps in ((256, 4, 50), (1024, 8, 20))
    ],
    "--hull": [
        partial(run_hull, 256, 4, 1 << 14, 16, 16, 4, 50, "hull meshes: 2^14 bodies sharing a 512-triangle ellipsoid (272 vertices), "
                "4 cascades of 256x256, vs points at the vertices; simulate at 4 sub-steps"),
        partial(run_hull, 1024, 8, 1 << 14, 16, 16, 4, 20, "hull meshes: 2^14 bodies sharing a 512-triangle ellipsoid (272 vertices), "
                "8 cascades of 1024x1024, vs points at the vertices; simulate at 4 sub-steps"),
        partial(run_hull, 256, 4, 1, 256, 128, 0, 50, "hull meshes: one body of 2^16 triangles (one warp), 4 cascades of 256x256, "
                "vs points at its vertices"),
    ],
    "--wake-obstacles": [
        partial(run_wake_step_obstacles, N, k, 200 if N < 1024 else 50, f"wake obstacles, step: {N}x{N} cells, {k} source(s), 8 sub-steps")
        for N in (256, 512, 1024) for k in (1, 64, 1024)
    ],
}
DEFAULT = ("--updates", "--query")


def main(args):
    unknown = [a for a in args if a not in GROUPS]
    if unknown:
        sys.exit(f"{os.path.basename(__file__)}: unknown argument(s) {' '.join(unknown)}; the flags are {' '.join(GROUPS)}")
    chosen = set(args or DEFAULT)
    for flag, configs in GROUPS.items():
        if flag in chosen:
            for config in configs:
                config()


if __name__ == "__main__":
    main(sys.argv[1:])
