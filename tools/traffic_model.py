#!/usr/bin/env python
"""Memory traffic of one update of the persistent kernel (k_update_persistent), per texel and per step, from the shape alone.

  python tools/traffic_model.py [--map-size 256] [--cascades 128] [--table-slots 4]

CPU only: the bytes follow from the buffer layouts (DESIGN section 3) and from what each work item reads and writes, not from a
measurement.  Two columns per stream: the bytes that pass through L2 and the bytes that come from or go to DRAM.  The row-pass
scratch is written and read back within one update; how much of it L2 holds depends on the queue shape and was not measured,
so its DRAM share is printed as a range.  Printed twice: with the previous foam read from normal_map.a (the whole 8 B texel
for 2 B of foam, and a bulk L2 prefetch of those rows per column-pass item) and with the foam plane (2 B read, 2 B written,
no prefetch).
"""
import argparse

# (stream, L2 bytes per texel, DRAM bytes per texel); a DRAM entry may be a (low, high) range
COMMON_HEAD = [
    ("spectrum, rows q <= N/2 only (16 B per texel, half the rows)", 8, 8),
    ("dispersion table (16 B per texel pair; no DRAM while the tables fit in L2)", 8, 0),
    ("row-pass scratch, written then read by TMA (32 B + 32 B)", 64, (0, 64)),
]
COMMON_TAIL = [
    ("displacement and normal maps, written (8 B + 8 B)", 16, 16),
]
LAYOUTS = {
    "foam in normal_map.a": COMMON_HEAD + [
        ("normal map, read only for foam (whole 8 B texel)", 8, 8),
    ] + COMMON_TAIL,
    "foam plane": COMMON_HEAD + [
        ("foam plane, read (2 B half)", 2, 2),
        ("foam plane, written (2 B half)", 2, 2),
    ] + COMMON_TAIL,
}


def _lo_hi(v):
    return v if isinstance(v, tuple) else (v, v)


def _fmt(v):
    lo, hi = _lo_hi(v)
    return f"{lo:g}" if lo == hi else f"{lo:g} to {hi:g}"


# bytes per texel of the bulk L2 prefetch of the previous foam issued for each column-pass item (W output rows of the cascade)
PREFETCH = {"foam in normal_map.a": 8, "foam plane": 0}


def columns_per_b_item(n):
    """TileB<N>::W of ocean_kernels.cu: a team of max(128, 4 N/16) threads, N/16 threads per column."""
    t = n // 16
    threads = max(128, 4 * t)
    return threads // t


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--map-size", type=int, default=256)
    ap.add_argument("--cascades", type=int, default=128)
    ap.add_argument("--table-slots", type=int, default=4, help="distinct (tile_length, depth) keys (bench.py: 4)")
    args = ap.parse_args()
    n, c = args.map_size, args.cascades
    texels = n * n * c
    mib = 1 << 20
    w = columns_per_b_item(n)
    print(f"{c} cascades of {n}^2 = {texels} texels per update; dispersion tables "
          f"{args.table_slots * (n // 2 + 1) * n * 16 / mib:.2f} MiB; column-pass items of {w} rows")
    for name, rows in LAYOUTS.items():
        print(f"\n## {name}\n")
        print("| stream | through L2, B/texel | from or to DRAM, B/texel | DRAM per update, MiB |")
        print("|---|---|---|---|")
        l2 = 0
        dram = (0, 0)
        for stream, b_l2, b_dram in rows:
            lo, hi = _lo_hi(b_dram)
            l2 += b_l2
            dram = (dram[0] + lo, dram[1] + hi)
            per_step = _fmt((lo * texels / mib, hi * texels / mib))
            print(f"| {stream} | {b_l2:g} | {_fmt(b_dram)} | {per_step} |")
        print(f"| **total** | **{l2:g}** | **{_fmt(dram)}** | **{_fmt((dram[0] * texels / mib, dram[1] * texels / mib))}** |")
        pf = PREFETCH[name] * w * n
        print(f"\nfoam prefetch per column-pass item: {pf / 1024:g} KiB; per update "
              f"{pf * (n // w) * c / mib:g} MiB installed in L2")


if __name__ == "__main__":
    main()
