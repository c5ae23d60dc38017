#!/usr/bin/env python
"""Instruction mix of the persistent update kernel k_update_persistent<N, false>, from its SASS (CPU only).

  python tools/sass_mix.py [--map-size 256] [--cubin path/to/ocean_kernels.cubin] [--cascades 128]

Without --cubin, csrc/ocean_kernels.cu is compiled to a cubin in a temporary directory with build.py's nvcc flags.  Prints the
kernel's registers, stack frame and spills, its static opcode mix, and the mix split by where each instruction comes from, using
the line table (-lineinfo) and its inlining chains:

  A hot      item_a, minus the rolled loop of the self-mirrored row pair (q == 0, one item in 64 at 256^2)
  B once     item_b outside the layer-pair loop
  B loop     the layer-pair loop outside its two epilogues (runs twice per item)
  B pair 0   the displacement epilogue;  B pair 1  the normal / foam epilogue
  queue      the item loop of k_update_persistent outside the two item bodies (once per item)
  cold       the q == 0 rolled loop (A cold), the exact __fdiv_rn fix-up of item_b (B cold), the multi-frame waits, and what
             lies outside the item loop (the backward branch of the SASS that spans the most instructions)

From those it estimates the warp-instructions issued per update of the bench shape (128 cascades of 256^2: 64 A and 32 B items
per cascade, 4 warps per item): each hot instruction counts once per pass of its region, every loop inside a region (spin waits,
the two-iteration L2 discard loop) once, and instructions that only thread 0 runs as if every warp ran them.  It is an estimate
of issue work derived from the SASS, not a measurement.
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "godotoceanwaves_b200", "csrc")
KERNEL_SRC = os.path.join(CSRC, "ocean_kernels.cu")
CUDA_BIN = "/usr/local/cuda/bin"

FP32 = {"FADD", "FFMA", "FMUL"}
FP64 = {"DFMA", "DMUL", "DADD"}
INT_CTRL = {"LEA", "LOP3", "IADD3", "BRA", "MOV", "BSSY", "BSYNC", "ISETP", "SHF", "IMAD", "PLOP3", "CS2R", "SEL", "FSEL",
            "P2R", "R2P", "UMOV", "UIADD3", "ULEA", "ULOP3", "USHF", "UISETP", "USEL", "R2UR", "S2R", "S2UR", "ULDC", "LDC", "VIMNMX"}


def tool(name):
    p = os.path.join(CUDA_BIN, name)
    return p if os.path.exists(p) else name


def build_cubin(out_dir):
    sys.path.insert(0, ROOT)
    from godotoceanwaves_b200 import build
    flags = [f for f in build.NVCC_FLAGS if f not in ("-Xcompiler", "-fPIC", "-shared")]
    cubin = os.path.join(out_dir, "ocean_kernels.cubin")
    cmd = [build._nvcc(), *flags, "-Xptxas", "-v", "-cubin", "-o", cubin, KERNEL_SRC]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        raise SystemExit("nvcc failed:\n" + res.stdout)
    return cubin, res.stdout


def kernel_symbol(n, taps=False):
    return f"_ZN5ocean19k_update_persistentILi{n}ELb{1 if taps else 0}EE"


def ptxas_lines(ptxas_out, sym):
    """registers and spill line ptxas printed for the kernel (None when the cubin was not built here)"""
    if not ptxas_out:
        return None
    lines = ptxas_out.splitlines()
    for i, l in enumerate(lines):
        if "Compiling entry function" in l and sym in l:
            props = lines[i + 2].strip() if i + 2 < len(lines) else ""
            regs = lines[i + 3].strip() if i + 3 < len(lines) else ""
            return props, regs
    return None


def res_usage(cubin, sym):
    out = subprocess.run([tool("cuobjdump"), "-res-usage", cubin], capture_output=True, text=True).stdout.splitlines()
    for i, l in enumerate(out):
        if "Function " + sym in l and i + 1 < len(out):
            m = re.search(r"REG:(\d+) STACK:(\d+)", out[i + 1])
            if m:
                return int(m.group(1)), int(m.group(2))
    raise SystemExit(f"{sym} not found in {cubin}")


# ---- source regions (found by brace matching in ocean_kernels.cu, so the tool follows edits of the file) ----
def block_end(lines, start):
    """index of the line that closes the first '{' opened on or after line `start` (0-based)"""
    depth, opened = 0, False
    for i in range(start, len(lines)):
        for ch in lines[i]:
            if ch == "{":
                depth, opened = depth + 1, True
            elif ch == "}" and opened:           # a "} else {" line closes the previous block first
                depth -= 1
                if opened and depth == 0:
                    return i
    raise ValueError("unbalanced braces")


def find(lines, pattern, lo=0, hi=None):
    rx = re.compile(pattern)
    for i in range(lo, len(lines) if hi is None else hi):
        if rx.search(lines[i]):
            return i
    raise ValueError(f"pattern {pattern!r} not found in {KERNEL_SRC}")


def source_regions(src_path):
    lines = open(src_path).read().splitlines()
    r = {}
    a0 = find(lines, r"void item_a\(")
    r["item_a"] = (a0, block_end(lines, a0))
    c0 = find(lines, r"^\s*if \(q == 0\) \{", *r["item_a"])
    r["a_cold"] = (c0, block_end(lines, c0))
    b0 = find(lines, r"void item_b\(")
    r["item_b"] = (b0, block_end(lines, b0))
    l0 = find(lines, r"for \(int pair = 0; pair < 2; \+\+pair\)", *r["item_b"])
    r["b_loop"] = (l0, block_end(lines, l0))
    p0 = find(lines, r"^\s*if \(pair == 0\) \{", *r["b_loop"])
    p0e = block_end(lines, p0)
    r["b_pair0"] = (p0, p0e)
    r["b_pair1"] = (p0e, block_end(lines, p0e))           # "} else {" shares the closing line of pair 0
    # the exact fix-up: the innermost `if` block of pair 1 that calls __fdiv_rn
    fd = find(lines, r"__fdiv_rn\(", *r["b_pair1"])
    best = None
    for i in range(r["b_pair1"][0] + 1, fd):
        if re.match(r"^\s*if \(", lines[i]) and "{" in lines[i]:
            e = block_end(lines, i)
            if e >= fd:
                best = (i, e)
    r["b_cold"] = best
    k0 = find(lines, r"k_update_persistent\(")
    k1 = block_end(lines, k0)
    r["kernel"] = (k0, k1)
    r["call_a"] = find(lines, r"item_a<N>\(", k0, k1)
    r["call_b"] = find(lines, r"item_b<N, true, TAPS>\(", k0, k1)
    r["loop"] = (find(lines, r"while \(true\)", k0, k1), k1)
    r["multi_frame"] = []
    for i in range(k0, k1):
        if re.search(r"if \(q\.multi_frame", lines[i]) and "{" in lines[i]:
            r["multi_frame"].append((i, block_end(lines, i)))
    return r


def inside(line0, rng):
    return rng is not None and rng[0] <= line0 <= rng[1]


# ---- SASS with inlining chains ----
INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
LOC = re.compile(r'^\s*//## File "([^"]+)", line (\d+)')
LABEL = re.compile(r"^(\.L_x_\d+):")


def kernel_sass(cubin, sym):
    out = subprocess.run([tool("nvdisasm"), "-gi", "-c", cubin], capture_output=True, text=True)
    if out.returncode != 0:
        raise SystemExit("nvdisasm failed:\n" + out.stderr)
    insns, chain, in_kernel, last_was_insn, labels = [], [], False, True, {}
    for l in out.stdout.splitlines():
        if l.startswith(".text."):
            in_kernel = l.startswith(".text." + sym)
            continue
        if not in_kernel:
            continue
        m = LOC.match(l)
        if m:
            if last_was_insn:
                chain = []
            chain.append((m.group(1), int(m.group(2))))
            last_was_insn = False
            continue
        if LABEL.match(l):
            labels[LABEL.match(l).group(1)] = len(insns)
            continue
        m = INSN.match(l)
        if m:
            text = m.group(2)
            body = re.sub(r"^@!?U?P[T0-9]+\s+", "", text)
            op = body.split()[0]
            insns.append((op, text, list(chain)))
            last_was_insn = True
    # the item loop: the backward branch that spans the most instructions; what lies outside it runs once per team
    lo, hi = 0, -1
    for i, (op, text, _) in enumerate(insns):
        m = re.search(r"BRA\S* `\((\.L_x_\d+)\)", text)
        if m and m.group(1) in labels and labels[m.group(1)] <= i and i - labels[m.group(1)] > hi - lo:
            lo, hi = labels[m.group(1)], i
    return [(op, text, chain, lo <= i <= hi) for i, (op, text, chain) in enumerate(insns)]


def classify(chain, in_loop, r, kernel_file):
    """region of one instruction from its inlining chain (innermost frame first)"""
    if not in_loop:
        return "cold"
    frames = [ln - 1 for f, ln in chain if os.path.basename(f) == kernel_file]
    if not frames:
        return "cold"
    outer = frames[-1]
    if not inside(outer, r["kernel"]):
        return "cold"
    if any(inside(outer, mf) for mf in r["multi_frame"]):
        return "cold"
    if outer == r["call_a"]:
        return "A cold" if any(inside(x, r["a_cold"]) for x in frames) else "A hot"
    if outer == r["call_b"]:
        if any(inside(x, r["b_cold"]) for x in frames):
            return "B cold"
        body = [x for x in frames if inside(x, r["item_b"])]
        x = body[-1] if body else None
        if x is None:
            return "B once"
        if inside(x, r["b_pair0"]) and x != r["b_pair0"][1]:
            return "B pair 0"
        if inside(x, r["b_pair1"]):
            return "B pair 1"
        if inside(x, r["b_loop"]):
            return "B loop"
        return "B once"
    if inside(outer, r["loop"]):
        return "queue"
    return "cold"


# region -> passes per item of its kind; A items and B items per cascade at the bench shape
PASSES = {"A hot": ("A", 1), "B once": ("B", 1), "B loop": ("B", 2), "B pair 0": ("B", 1), "B pair 1": ("B", 1),
          "queue": ("AB", 1)}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--map-size", type=int, default=256, choices=(128, 256, 512, 1024))
    ap.add_argument("--cubin", help="disassemble this cubin instead of compiling csrc/ocean_kernels.cu")
    ap.add_argument("--cascades", type=int, default=128)
    ap.add_argument("--top", type=int, default=24, help="opcodes listed per table")
    args = ap.parse_args(argv)
    n = args.map_size
    sym = kernel_symbol(n)
    with tempfile.TemporaryDirectory() as tmp:
        ptxas_out = None
        cubin = args.cubin
        if cubin is None:
            cubin, ptxas_out = build_cubin(tmp)
        regs, stack = res_usage(cubin, sym)
        insns = kernel_sass(cubin, sym)
    info = ptxas_lines(ptxas_out, sym)
    r = source_regions(KERNEL_SRC)
    kfile = os.path.basename(KERNEL_SRC)

    threads = 128 if n <= 512 else 4 * (n // 16)
    warps = threads // 32
    rows_per_item = (threads // (2 * (n // 16))) // 2
    a_items = (n // 2) // rows_per_item
    b_items = n // (threads // (n // 16))

    print(f"k_update_persistent<{n}, false>: {regs} registers, {stack} bytes stack frame")
    if info:
        print("  ptxas: " + info[0])
    spills = 0
    if info:
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", info[0])
        spills = int(m.group(1)) + int(m.group(2)) if m else 0
    print(f"  spills: {'none' if spills == 0 and stack == 0 else f'{spills} bytes'}")

    total = collections.Counter(op.split(".")[0] for op, _, _, _ in insns)
    by_region = collections.defaultdict(collections.Counter)
    for op, _, chain, in_loop in insns:
        by_region[classify(chain, in_loop, r, kfile)][op.split(".")[0]] += 1

    def groups(c):
        fp32 = sum(v for k, v in c.items() if k in FP32)
        fp64 = sum(v for k, v in c.items() if k in FP64)
        mnmx = c.get("FMNMX", 0)
        intc = sum(v for k, v in c.items() if k in INT_CTRL)
        return fp32, intc, mnmx, fp64

    print(f"\nstatic SASS instructions: {len(insns)}")
    fp32, intc, mnmx, fp64 = groups(total)
    print(f"  FP32 (FADD/FFMA/FMUL) {fp32}   integer/address/control {intc}   FMNMX {mnmx}   fp64 (DFMA/DMUL/DADD) {fp64}")
    print("  " + "  ".join(f"{k} {v}" for k, v in total.most_common(args.top)))

    order = ["A hot", "A cold", "B once", "B loop", "B pair 0", "B pair 1", "B cold", "queue", "cold"]
    print("\nby region (static):")
    for reg in order:
        c = by_region.get(reg, collections.Counter())
        s = sum(c.values())
        fp32, intc, mnmx, fp64 = groups(c)
        print(f"  {reg:9s} {s:6d}   FP32 {fp32:5d}  int/ctrl {intc:5d}  FMNMX {mnmx:4d}  fp64 {fp64:3d}   "
              + " ".join(f"{k}:{v}" for k, v in c.most_common(8)))

    dyn = collections.Counter()
    for reg, (kind, passes) in PASSES.items():
        c = by_region.get(reg, collections.Counter())
        items = {"A": a_items, "B": b_items, "AB": a_items + b_items}[kind]
        for k, v in c.items():
            dyn[k] += v * passes * items * warps * args.cascades
    d = sum(dyn.values())
    print(f"\nestimated dynamic warp-instructions per step ({args.cascades} cascades of {n}^2, {a_items} A + {b_items} B items "
          f"per cascade, {warps} warps per item): {d / 1e6:.1f} M")
    fp32, intc, mnmx, fp64 = groups(dyn)
    print(f"  FP32 {fp32 / 1e6:.1f} M   integer/address/control {intc / 1e6:.1f} M   FMNMX {mnmx / 1e6:.2f} M   fp64 {fp64 / 1e6:.2f} M")
    print("  " + "  ".join(f"{k} {v / 1e6:.2f}M" for k, v in dyn.most_common(args.top)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
