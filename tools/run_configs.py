"""Times the BASELINE.json configs beyond the bench default (GPU).  Prints one JSON object per config."""
import json, math, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import godotoceanwaves_b200 as gow
from bench import synth_params

def run(N, C, frames, label, regen=False, fused=False):
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(max(2, C))
    p = [synth_params(gow.WaveCascadeParameters, c) for c in range(C)]
    for _ in range(3):
        g.update_all(0.02, p)
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
    texels = C * N * N * frames
    bytes_per_texel = 56.0 if regen else 40.0
    out = {"config": label, "map_size": N, "cascades": C, "frames": frames, "ms_total": ms, "us_per_frame": 1e3 * ms / frames,
           "cascades_per_s": C * frames / (ms * 1e-3), "gtexels_per_s": texels / (ms * 1e-3) / 1e9,
           "algorithmic_GBps": bytes_per_texel * texels / (ms * 1e-3) / 1e9}
    g.free()
    print(json.dumps(out), flush=True)

def run_sweep_batch(N, per_set, reps, label):
    """cfg5 as ONE batch: the 6 x 4 (U, F) grid points are 24 cascade sets of one generator; every step regenerates all 96
    spectra (one spectrum launch) and updates all maps (one persistent launch)."""
    grid = [(u, f) for u in (5.0, 10.0, 15.0, 20.0, 25.0, 30.0) for f in (1.0, 10.0, 100.0, 1000.0)]
    C = len(grid) * per_set
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(C)
    p = [synth_params(gow.WaveCascadeParameters, c) for c in range(C)]
    for s, (u, f) in enumerate(grid):
        for c in range(per_set):
            p[s * per_set + c].wind_speed = u; p[s * per_set + c].fetch_length = f
    for _ in range(3):
        g.update_all(0.02, p)
    g.synchronize()
    g.timer_start()
    for r in range(reps):
        for q in p:
            q.should_generate_spectrum = True
        g.update_all(0.02, p)
    ms = g.timer_stop()
    texels = C * N * N * reps
    out = {"config": label, "map_size": N, "cascades": C, "frames": reps, "ms_total": ms, "us_per_frame": 1e3 * ms / reps,
           "cascades_per_s": C * reps / (ms * 1e-3), "gtexels_per_s": texels / (ms * 1e-3) / 1e9,
           "algorithmic_GBps": 56.0 * texels / (ms * 1e-3) / 1e9}
    g.free()
    print(json.dumps(out), flush=True)


def run_spectrum(N, C, reps, label):
    """k_spectrum_compute alone (spectrum_compute.glsl, a4): CUDA events around the launch (ocean_set_profiling), all C
    cascades dirty.  Algorithmic bytes: 16 B/texel written; the kernel is bound by the binary64 pipe (DETMATH), not by HBM."""
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(C)
    p = [synth_params(gow.WaveCascadeParameters, c) for c in range(C)]
    g.update_all(0.02, p)
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
    import ctypes
    import numpy as np
    import torch
    from godotoceanwaves_b200.native import load_library, check
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(max(2, C))
    p = [synth_params(gow.WaveCascadeParameters, c) for c in range(C)]
    for q in p:
        q.whitecap = 0.9; q.foam_amount = 10.0
    for _ in range(25):
        g.update_all(0.02, p)
    scales = gow.WaveGenerator.map_scales(p)
    dev = torch.device("cuda", 0)
    pts = torch.from_numpy(gow.WaveGenerator.spray_grid(particles, np.array([[40, 0, 0, 0], [0, 1, 0, 0], [0, 0, 40, 0]], np.float32))).to(dev)
    recs = torch.empty(particles * 8, dtype=torch.float32, device=dev)
    count = torch.zeros(1, dtype=torch.int32, device=dev)
    ps = np.array([1, 1, 1], np.float32)
    lib = load_library()
    call = lambda: check(lib.ocean_extract_spray_device(g.context, particles, pts.data_ptr(), C, scales.ctypes.data, ps.ctypes.data, particles,
                                                        recs.data_ptr(), count.data_ptr()))
    for _ in range(3):
        call()
    g.synchronize()
    g.timer_start()
    for _ in range(reps):
        call()
    ms = g.timer_stop()
    out = {"config": label, "map_size": N, "cascades": C, "candidates": particles, "active": int(count.item()), "us_per_call": 1e3 * ms / reps,
           "mcandidates_per_s": particles / (ms / reps * 1e-3) / 1e6}
    g.free()
    print(json.dumps(out), flush=True)


if "--buoyancy" not in sys.argv:       # --buoyancy runs run_buoyancy (defined below) alone
    run(256, 4, 2000, "cfg2 latency: one 256x256x4 set per launch (launch/latency-bound, L2-resident)")
    run(256, 4, 2000, "cfg2 latency, fused frames (ocean_update_frames: 64 frames per launch)", fused=True)
    run(512, 4, 1000, "cfg3: 512x512x4, 1000-frame foam accumulate/decay loop, frame by frame")
    run(512, 4, 1000, "cfg3: 512x512x4, 1000-frame foam accumulate/decay loop, fused frames (ocean_update_frames)", fused=True)
    run(1024, 8, 200, "cfg4 (1 GPU): 1024x1024x8")
    run(256, 4, 300, "cfg5: 256x256x4 wind/fetch sweep, one grid point per step, spectrum regenerated every step", regen=True)
    run_sweep_batch(256, 4, 50, "cfg5 batched: the 6x4 (U,F) grid = 24 sets x 4 cascades per step, all spectra regenerated every step")
    run(128, 1, 2000, "cfg1 shape on GPU: 128x128x1")
    run_spectrum(256, 128, 10, "spectrum generation alone: 128 cascades of 256x256, one launch")
    run_spray(256, 4, 1 << 20, 50, "spray candidates: 2^20 grid candidates x 4 cascades of 256x256")


def run_query(N, C, n_points, reps, label):
    """Map-query op (water.gdshader sampling contract) on device-resident points: kernel time only."""
    import ctypes
    import numpy as np
    import torch
    from godotoceanwaves_b200.native import load_library, check
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(max(2, C))
    p = [synth_params(gow.WaveCascadeParameters, c) for c in range(C)]
    for _ in range(2):
        g.update_all(0.02, p)
    scales = gow.WaveGenerator.map_scales(p)
    dev = torch.device("cuda", 0)
    pts = (torch.rand(n_points, 2, device=dev) * 1000.0 - 500.0).contiguous()
    disp = torch.empty(n_points, 3, device=dev)
    grad = torch.empty(n_points, 3, device=dev)
    torch.cuda.synchronize()
    lib = load_library()
    call = lambda: check(lib.ocean_sample_maps_device(g.context, n_points, pts.data_ptr(), C, scales.ctypes.data, disp.data_ptr(), grad.data_ptr()))
    for _ in range(3):
        call()
    g.synchronize()
    g.timer_start()
    for _ in range(reps):
        call()
    ms = g.timer_stop()
    per = ms / reps
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
    import numpy as np
    import torch
    from godotoceanwaves_b200.native import load_library, check
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(max(2, C))
    p = [synth_params(gow.WaveCascadeParameters, c) for c in range(C)]
    for _ in range(2):
        g.update_all(0.02, p)
    scales = gow.WaveGenerator.map_scales(p)
    dev = torch.device("cuda", 0)
    pts = (torch.rand(n_points, 2, device=dev, generator=torch.Generator(dev).manual_seed(1)) * 600.0 - 300.0).contiguous()
    recs = torch.empty(n_points * 10, dtype=torch.int32, device=dev)        # ocean_surface_sample: 40 B
    disp = torch.empty(n_points, 3, device=dev)
    grad = torch.empty(n_points, 3, device=dev)
    torch.cuda.synchronize()
    lib = load_library()
    query = lambda: check(lib.ocean_query_surface_device(g.context, n_points, pts.data_ptr(), C, scales.ctypes.data, tolerance, max_iterations,
                                                         recs.data_ptr()))
    sample = lambda: check(lib.ocean_sample_maps_device(g.context, n_points, pts.data_ptr(), C, scales.ctypes.data, disp.data_ptr(), grad.data_ptr()))

    def timed(call):
        for _ in range(3):
            call()
        g.synchronize()
        g.timer_start()
        for _ in range(reps):
            call()
        return g.timer_stop() / reps

    t_query, t_sample = timed(query), timed(sample)
    t_query = min(t_query, timed(query))        # alternate: the first window also absorbs clock ramp-up
    rec = recs.cpu().numpy().view(gow.WaveGenerator.SURFACE_SAMPLE)
    out = {"config": label, "map_size": N, "cascades": C, "points": n_points, "tolerance": tolerance, "max_iterations": max_iterations,
           "us_per_call": 1e3 * t_query, "mpoints_per_s": n_points / (t_query * 1e-3) / 1e6, "sample_maps_us_per_call": 1e3 * t_sample,
           "ratio_to_sample_maps": t_query / t_sample, "frac_restarted": float(np.mean(rec["iterations"] > max_iterations)),
           "frac_converged": float(np.mean(rec["residual"] <= np.float32(tolerance))), "mean_iterations": float(np.mean(rec["iterations"]))}
    g.free()
    print(json.dumps(out), flush=True)


def run_buoyancy(N, C, n_bodies, per_body, reps, label, tolerance=1e-3, max_iterations=8):
    """Buoyancy op (ocean_buoyancy_device) on device-resident hulls of `per_body` points per body: kernel time from CUDA
    events, against ocean_query_surface_device on the same world points in the same run, in alternating windows.  The card's
    name, power limit and max SM clock are read in the same run."""
    import subprocess
    import numpy as np
    import torch
    from godotoceanwaves_b200.native import load_library, check
    from oracle import buoyancy as bu
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(max(2, C))
    p = [synth_params(gow.WaveCascadeParameters, c) for c in range(C)]
    for _ in range(2):
        g.update_all(0.02, p)
    scales = gow.WaveGenerator.map_scales(p)
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
    _, _, _, wp = bu.world_points(bodies, hull)
    n_points = len(wp)
    dev = torch.device("cuda", 0)
    hull_d = torch.from_numpy(hull.view(np.uint8).copy()).to(dev)
    pts_d = torch.from_numpy(np.ascontiguousarray(wp[:, [0, 2]])).to(dev)
    res_d = torch.empty(n_bodies * 12, dtype=torch.int32, device=dev)           # ocean_buoyancy_result: 48 B
    recs_d = torch.empty(n_points * 10, dtype=torch.int32, device=dev)          # ocean_surface_sample: 40 B
    torch.cuda.synchronize()
    lib = load_library()
    buoy = lambda: check(lib.ocean_buoyancy_device(g.context, n_bodies, bodies.ctypes.data, len(hull), hull_d.data_ptr(), C, scales.ctypes.data,
                                                   1025.0, tolerance, max_iterations, res_d.data_ptr(), None))
    query = lambda: check(lib.ocean_query_surface_device(g.context, n_points, pts_d.data_ptr(), C, scales.ctypes.data, tolerance, max_iterations,
                                                         recs_d.data_ptr()))

    def timed(call):
        for _ in range(3):
            call()
        g.synchronize()
        g.timer_start()
        for _ in range(reps):
            call()
        return g.timer_stop() / reps

    t_b, t_q = [], []
    for _ in range(3):                          # alternating windows: clock ramp-up and neighbours hit both alike
        t_b.append(timed(buoy))
        t_q.append(timed(query))
    res = res_d.cpu().numpy().view(bu.RESULT)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    out = {"config": label, "gpu": torch.cuda.get_device_name(0), "power_limit_and_max_sm_clock": smi, "map_size": N, "cascades": C,
           "bodies": n_bodies, "points_per_body": per_body, "world_points": n_points, "tolerance": tolerance, "max_iterations": max_iterations,
           "buoyancy_us_per_call": [1e3 * v for v in t_b], "query_surface_us_per_call": [1e3 * v for v in t_q],
           "overhead_over_query": min(t_b) / min(t_q) - 1.0, "mpoints_per_s": n_points / (min(t_b) * 1e-3) / 1e6,
           "frac_bodies_afloat": float(np.mean(res["submerged_volume"] > 0)),
           "frac_points_unconverged": float(res["unconverged"].sum()) / n_points}
    g.free()
    print(json.dumps(out), flush=True)


if "--buoyancy" in sys.argv:
    run_buoyancy(256, 4, 1 << 14, 64, 50, "buoyancy: 2^14 bodies x 64 points over 4 cascades of 256x256")
    run_buoyancy(1024, 8, 1 << 14, 64, 20, "buoyancy: 2^14 bodies x 64 points over 8 cascades of 1024x1024")
    sys.exit(0)

if "--query" in sys.argv or os.environ.get("OCEAN_RUN_QUERY", "1") != "0":
    run_query(256, 4, 1 << 20, 50, "query op: 2^20 random points x 4 cascades of 256x256 (maps L2-resident)")
    run_query(1024, 8, 1 << 20, 20, "query op: 2^20 random points x 8 cascades of 1024x1024 (maps 128 MiB)")
    run_surface(256, 4, 1 << 20, 50, "surface query: 2^20 points in [-300, 300]^2 m x 4 cascades of 256x256")
    run_surface(1024, 8, 1 << 20, 20, "surface query: 2^20 points in [-300, 300]^2 m x 8 cascades of 1024x1024")
