#!/usr/bin/env python
"""Time the boundary between consecutive persistent updates on the bench workload (128 cascades of 256^2).

  python tools/step_boundary.py build [--rev REV] OUT.so     # needs nvcc (and git for --rev); no GPU
  python tools/step_boundary.py run LIB.so [LIB.so ...]      # on the GPU; one JSON line per library

`build` compiles a throwaway, instrumented copy of the library (the working tree's sources, or those of git revision REV):
thread 0 of every team of k_update_persistent reads %globaltimer when the team starts its first item and its last item, sums
the time it spends waiting for the row pass of B items (all of them, and those of the last queue group) and, when the team
leaves, writes the five values into a device array indexed by (launch, team).  A launch is identified by the order in which
teams leave (every launch has the same grid), which holds as long as launches do not run items concurrently.  The
instrumentation is patched into a temporary copy of the sources and is never part of the shipped library.

`run` performs 5 warm-up and 200 timed update_all steps and reports, per launch boundary (medians over the 199 boundaries):
  gap_us        previous launch's last team exit -> this launch's first item start
  drain_us      spread of the previous launch's team exits (first exit -> last exit)
  idle_team_us  team-microseconds idle after the queue emptied: sum over teams of (last exit - team exit)
  bwait_g15_us  thread-0 time of the B items of the last group spent waiting for their row pass (sum over teams)
  step_us       first item start -> first item start of the next launch
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_LAUNCHES, MAX_TEAMS, FIELDS = 256, 1024, 5

PRELUDE = r"""
__device__ unsigned long long g_sb_stamps[%d][%d][%d];
__device__ unsigned int g_sb_exits;
__device__ __forceinline__ unsigned long long sb_now() {
    unsigned long long t;
    asm volatile("mov.u64 %%0, %%%%globaltimer;" : "=l"(t));
    return t;
}
""" % (MAX_LAUNCHES, MAX_TEAMS, FIELDS)

EXPORT = r"""
extern "C" int ocean_sb_read(void* out, unsigned long long bytes, int reset) {
    if (cudaMemcpyFromSymbol(out, ocean::g_sb_stamps, bytes) != cudaSuccess) return 1;
    if (reset) {
        static unsigned long long zeros[%d][%d][%d];
        unsigned int z = 0;
        if (cudaMemcpyToSymbol(ocean::g_sb_stamps, zeros, sizeof zeros) != cudaSuccess) return 1;
        if (cudaMemcpyToSymbol(ocean::g_sb_exits, &z, sizeof z) != cudaSuccess) return 1;
    }
    return 0;
}
""" % (MAX_LAUNCHES, MAX_TEAMS, FIELDS)


def patch(src: str) -> str:
    def once(pattern, repl, s, flags=0):
        out, n = re.subn(pattern, repl, s, count=1, flags=flags)
        if n != 1:
            raise SystemExit(f"step_boundary: anchor not found: {pattern!r}")
        return out
    # device array + clock, just before the persistent kernel's definition
    src = once(r"(template <int N, bool TAPS>\n__global__ void __launch_bounds__\(Team<N>::THREADS, kTeamThreadsPerSm)",
               lambda m: PRELUDE + m.group(1), src)
    body_at = src.index("k_update_persistent(\n")
    head, body = src[:body_at], src[body_at:]
    body = once(r"(    const int tid = threadIdx.x;\n)",
                lambda m: m.group(1) + "    unsigned long long sb_first = 0, sb_last = 0, sb_bw = 0, sb_bw_last = 0;\n", body)
    body = once(r"(        const int code = s_code\[buf\];\n)        if \(code == -1\) break;\n",
                lambda m: m.group(1) +
                "        if (code == -1) {\n"
                "            if (tid == 0) {\n"
                "                const unsigned v = atomicAdd(&g_sb_exits, 1u);\n"
                "                unsigned long long* o = g_sb_stamps[(v / gridDim.x) % " + str(MAX_LAUNCHES) + "][blockIdx.x % " + str(MAX_TEAMS) + "];\n"
                "                o[0] = sb_first; o[1] = sb_last; o[2] = sb_now(); o[3] = sb_bw; o[4] = sb_bw_last;\n"
                "            }\n"
                "            break;\n"
                "        }\n"
                "        if (tid == 0) { sb_last = sb_now(); if (!sb_first) sb_first = sb_last; }\n", body)
    body = once(r"(            if \(tid == 0 && !panel_requested\) \{\n                uint32_t seen;\n                while \(true\) \{\n"
                r"(?:.*\n)*?                \}\n)(            \}\n)",
                lambda m: "            const unsigned long long sb_w0 = (tid == 0) ? sb_now() : 0;\n" + m.group(1) + m.group(2) +
                "            if (tid == 0) { const unsigned long long w = sb_now() - sb_w0; sb_bw += w;"
                " if (slot >= (int)(q.total / (Queue<N>::A_PER + Queue<N>::B_PER)) - 8) sb_bw_last += w; }\n", body)
    return head + body + EXPORT


def build(args):
    tmp = tempfile.mkdtemp(prefix="step_boundary_")
    try:
        if args.rev:
            arch = subprocess.run(["git", "-C", ROOT, "archive", args.rev, "godotoceanwaves_b200/csrc", "include"],
                                  check=True, stdout=subprocess.PIPE).stdout
            subprocess.run(["tar", "-x", "-C", tmp], input=arch, check=True)
        else:
            shutil.copytree(os.path.join(ROOT, "godotoceanwaves_b200", "csrc"), os.path.join(tmp, "godotoceanwaves_b200", "csrc"))
            shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, "include"))
        csrc = os.path.join(tmp, "godotoceanwaves_b200", "csrc")
        k = os.path.join(csrc, "ocean_kernels.cu")
        with open(k) as f:
            src = f.read()
        with open(k, "w") as f:
            f.write(patch(src))
        sys.path.insert(0, ROOT)
        from godotoceanwaves_b200 import build as nb
        cmd = [nb._nvcc(), *nb.NVCC_FLAGS, "-o", os.path.abspath(args.out)] + [os.path.join(csrc, s) for s in nb.SOURCES]
        subprocess.run(cmd, check=True)
        print("built", args.out)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def child(lib_path, steps, warmup):
    sys.path.insert(0, ROOT)
    import ctypes
    import numpy as np
    import godotoceanwaves_b200 as gow
    from bench import synth_params
    N, C = 256, 128
    g = gow.WaveGenerator()
    g.map_size = N
    g.init_gpu(C)
    p = [synth_params(gow.WaveCascadeParameters, i) for i in range(C)]
    lib = ctypes.CDLL(lib_path)
    lib.ocean_sb_read.argtypes = [ctypes.c_void_p, ctypes.c_ulonglong, ctypes.c_int]
    buf = np.zeros((MAX_LAUNCHES, MAX_TEAMS, FIELDS), dtype=np.uint64)
    for _ in range(warmup):
        g.update_all(0.02, p)
    g.synchronize()
    assert lib.ocean_sb_read(buf.ctypes.data, buf.nbytes, 1) == 0
    g.timer_start()
    for _ in range(steps):
        g.update_all(0.02, p)
    ms = g.timer_stop() / steps
    g.synchronize()
    assert lib.ocean_sb_read(buf.ctypes.data, buf.nbytes, 1) == 0
    g.free()
    teams = int((buf[0, :, 2] != 0).sum())
    L = buf[:steps, :teams].astype(np.int64)
    first, exit_, bw_last = L[:, :, 0], L[:, :, 2], L[:, :, 4]
    start = np.where(first > 0, first, np.iinfo(np.int64).max).min(axis=1)   # teams without an item have first == 0
    last_exit, first_exit = exit_.max(axis=1), exit_.min(axis=1)
    gap = (start[1:] - last_exit[:-1]) / 1e3
    drain = (last_exit - first_exit) / 1e3
    idle = (last_exit[:, None] - exit_).sum(axis=1) / 1e3
    step = (start[1:] - start[:-1]) / 1e3
    bw15 = bw_last.sum(axis=1) / 1e3
    med = lambda a: float(np.median(a))
    return {"lib": os.path.basename(lib_path), "teams": teams, "ms_per_step": ms, "step_us": med(step), "gap_us": med(gap),
            "gap_us_p90": float(np.percentile(gap, 90)), "drain_us": med(drain), "idle_team_us": med(idle),
            "idle_team_us_per_team": med(idle) / teams, "bwait_g15_us": med(bw15),
            "bwait_all_us": med(L[:, :, 3].sum(axis=1) / 1e3)}


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    b = sub.add_parser("build")
    b.add_argument("out")
    b.add_argument("--rev", default=None, help="git revision whose sources to instrument (default: the working tree)")
    r = sub.add_parser("run")
    r.add_argument("libs", nargs="+")
    r.add_argument("--steps", type=int, default=200)
    r.add_argument("--warmup", type=int, default=5)
    r.add_argument("--child", action="store_true")
    args = ap.parse_args()
    if args.cmd == "build":
        return build(args)
    if args.child:
        print(json.dumps(child(os.path.abspath(args.libs[0]), args.steps, args.warmup)))
        return
    for lib in args.libs:
        env = dict(os.environ, OCEAN_LIB=os.path.abspath(lib), OCEAN_ALLOW_MISSING="1")
        res = subprocess.run([sys.executable, os.path.abspath(__file__), "run", "--child", "--steps", str(args.steps),
                              "--warmup", str(args.warmup), lib], env=env, capture_output=True, text=True, timeout=300)
        out = res.stdout.strip().splitlines()
        print(out[-1] if res.returncode == 0 and out else json.dumps({"lib": lib, "error": res.stderr[-800:]}), flush=True)


if __name__ == "__main__":
    main()
