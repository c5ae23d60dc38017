"""The Python record layouts against include/ocean.h, as the C++ compiler lays the structs out: every record dtype of
WaveGenerator and every ctypes struct of native.py, field by field (offset, size, element size and kind), from a probe
of offsetof / sizeof built with g++, the host compiler nvcc uses."""
import os
import re
import shutil
import subprocess

import numpy as np

from godotoceanwaves_b200 import native
from godotoceanwaves_b200.wave_generator import WaveGenerator

INCLUDE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")

PROBE = r"""#include <cstddef>
#include <cstdio>
#include <type_traits>
#include "ocean.h"
template <typename M> void field(const char* s, const char* f, size_t offset) {
    using E = std::remove_all_extents_t<M>;
    std::printf("%s %s %zu %zu %zu %c\n", s, f, offset, sizeof(M), sizeof(E),
                std::is_floating_point<E>::value ? 'f' : std::is_signed<E>::value ? 'i' : 'u');
}
int main() {
"""


def test_python_record_layouts_match_the_header(tmp_path):
    # WaveGenerator.RAY_HIT is struct ocean_ray_hit, and so on
    records = {"ocean_" + k.lower(): v for k, v in vars(WaveGenerator).items() if isinstance(v, np.dtype) and v.names}
    records.update(ocean_cascade_params=np.dtype(native.CascadeParamsC), ocean_scheduler=np.dtype(native.SchedulerC),
                   ocean_info=np.dtype(native.InfoC))
    declared = set(re.findall(r"typedef struct (ocean_\w+) \{", open(os.path.join(INCLUDE, "ocean.h")).read()))
    assert set(records) == declared, set(records) ^ declared
    src, want = [PROBE], []
    for s, dt in records.items():
        src.append(f'    std::printf("{s} (struct) %zu\\n", sizeof({s}));\n')
        want.append(f"{s} (struct) {dt.itemsize}")
        for f in dt.names:
            t, offset = dt.fields[f][:2]
            src.append(f'    field<decltype({s}::{f})>("{s}", "{f}", offsetof({s}, {f}));\n')
            want.append(f"{s} {f} {offset} {t.itemsize} {t.base.itemsize} {t.base.kind}")
    (tmp_path / "probe.cpp").write_text("".join(src) + "}\n")
    gxx = shutil.which("g++")
    assert gxx, "g++ (the host compiler of nvcc) is not on PATH"
    exe = str(tmp_path / "probe")
    res = subprocess.run([gxx, "-std=c++17", "-I", INCLUDE, str(tmp_path / "probe.cpp"), "-o", exe], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g == w
