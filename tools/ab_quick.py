#!/usr/bin/env python
"""Same-box A/B of tuning builds of libocean.so without bench.py's start-up cost (run on the GPU machine).

  python tools/ab_quick.py [--env "VAR=1 VAR2=x"] lib_a.so lib_b.so ...

For every library (one child process each, OCEAN_LIB=<lib>): the bench workload (128 cascades of 256^2, synthetic
parameters of bench.synth_params), 5 warm-up steps, `--rounds` timed blocks of `--steps` steps (device timer of the
C ABI), then the CRC32 of both RGBA16F maps after exactly the same number of updates -- libraries whose CRC differs from
the first library's do NOT compute the same maps (differential parity against a build the oracle tests vouch for).
Prints  <lib> <env>  min ms/step, median ms/step, frac of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s), crc.
"""
import argparse
import json
import os
import subprocess
import sys
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def child(args):
    sys.path.insert(0, ROOT)
    import numpy as np
    import godotoceanwaves_b200 as gow
    from bench import synth_params, ALGO_BYTES_PER_TEXEL
    n, c = args.map_size, args.cascades
    g = gow.WaveGenerator()
    g.map_size = n
    g.init_gpu(c)
    p = [synth_params(gow.WaveCascadeParameters, i) for i in range(c)]
    for _ in range(5):
        g.update_all(0.02, p)
    g.synchronize()
    times = []
    for _ in range(args.rounds):
        g.timer_start()
        for _ in range(args.steps):
            g.update_all(0.02, p)
        times.append(g.timer_stop() / args.steps)
    crc = 0
    for first in range(0, c, 32):
        d, nm = g.maps_to_host(first, min(32, c - first))
        crc = zlib.crc32(nm.tobytes(), zlib.crc32(d.tobytes(), crc))
    g.free()
    times.sort()
    best, med = times[0], times[len(times) // 2]
    gbs = ALGO_BYTES_PER_TEXEL * n * n * c / (best * 1e-3) / 1e9
    print(json.dumps({"min_ms": best, "med_ms": med, "frac": gbs / 3350.0, "crc": crc}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="*")
    ap.add_argument("--env", action="append", default=None, help='environment settings to test with every library, e.g. "OCEAN_QUEUE_GROUP=6"')
    ap.add_argument("--steps", type=int, default=150)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--map-size", type=int, default=256)
    ap.add_argument("--cascades", type=int, default=128)
    ap.add_argument("--child", action="store_true")
    ap.add_argument("--timeout", type=int, default=60, help="seconds per library and setting (a hung build must not eat the batch)")
    args = ap.parse_args()
    if args.child:
        return child(args)
    ref_crc = None
    for lib in args.libs:
        for envs in (args.env or [""]):
            env = dict(os.environ, OCEAN_LIB=os.path.join(ROOT, lib) if not os.path.isabs(lib) else lib, OCEAN_ALLOW_MISSING="1")
            for kv in envs.split():
                k, v = kv.split("=", 1)
                env[k] = v
            cmd = [sys.executable, os.path.abspath(__file__), "--child", "--steps", str(args.steps), "--rounds", str(args.rounds),
                   "--map-size", str(args.map_size), "--cascades", str(args.cascades)]
            try:
                r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=args.timeout)
                d = json.loads(r.stdout.strip().splitlines()[-1])
            except Exception as e:   # a variant that crashes or hangs must not take the batch with it
                print(f"{lib} [{envs}] FAILED: {e}; stderr tail: {(r.stderr[-300:] if 'r' in dir() else '')}", flush=True)
                continue
            if ref_crc is None:
                ref_crc = d["crc"]
            same = "same-maps" if d["crc"] == ref_crc else "MAPS-DIFFER"
            print(f"{lib} [{envs}] min {d['min_ms']:.4f} med {d['med_ms']:.4f} ms/step frac {d['frac']:.4f} crc {d['crc']:08x} {same}", flush=True)


if __name__ == "__main__":
    main()
