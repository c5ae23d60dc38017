"""tools/sass_mix.py compiles the persistent update kernel, reads its SASS and reports the instruction mix (CPU only)."""
import os
import shutil
import subprocess
import sys

import pytest

from conftest import ROOT

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


@pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")
def test_sass_mix_runs_and_reports_no_spills():
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sass_mix.py")], capture_output=True, text=True, timeout=900,
                         cwd=ROOT)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    out = res.stdout
    assert "k_update_persistent<256, false>" in out and "0 bytes stack frame" in out
    assert "spills: none" in out
    assert "estimated dynamic warp-instructions per step" in out
