import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def _has_gpu() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


# ---- shared parameter sets (SURVEY appendix B: main.tscn:43-83, wave_cascade_parameters.gd:7-35)
DEMO_SETS = [
    dict(tile_length=(88.0, 88.0), displacement_scale=1.0, normal_scale=1.0, wind_speed=10.0, wind_direction=20.0,
         fetch_length=150.0, swell=0.8, spread=0.2, detail=1.0, whitecap=0.5, foam_amount=8.0),
    dict(tile_length=(57.0, 57.0), displacement_scale=0.75, normal_scale=1.0, wind_speed=5.0, wind_direction=15.0,
         fetch_length=150.0, swell=0.8, spread=0.4, detail=1.0, whitecap=0.5, foam_amount=0.0),
    dict(tile_length=(16.0, 16.0), displacement_scale=0.0, normal_scale=0.25, wind_speed=20.0, wind_direction=20.0,
         fetch_length=550.0, swell=0.8, spread=0.4, detail=1.0, whitecap=0.25, foam_amount=3.0),
    dict(tile_length=(50.0, 50.0), displacement_scale=1.0, normal_scale=1.0, wind_speed=20.0, wind_direction=0.0,
         fetch_length=550.0, swell=0.8, spread=0.2, detail=1.0, whitecap=0.5, foam_amount=5.0),
]


def demo_params(cls, c: int, **over):
    """Cascade c of the synthetic workload (SURVEY 8d): demo sets cycled, fixed seeds, time0 = 120 + pi*c."""
    import math
    kw = dict(DEMO_SETS[c % len(DEMO_SETS)])
    kw.update(spectrum_seed=(1234 + 17 * c, -5678 + 31 * c), time=120.0 + math.pi * c)
    kw.update(over)
    return cls(**kw)


# ---- parameter corners of wave_cascade_parameters.gd (clamps, @export_range sliders and beyond); shared by the CPU pin
# tests (oracle vs the reference shaders) and the GPU parity tests (CUDA vs oracle)
EDGE_CASES = {
    "anisotropic_tile": dict(tile_length=(93.0, 41.0)),
    "detail_damped_zeros": dict(detail=0.35, tile_length=(16.0, 16.0)),       # exp(-(1-detail)^2 k^2) underflows to exact 0
    "wind_negative_dir": dict(wind_direction=-135.0, wind_speed=3.0, fetch_length=2.0),
    "wind_360": dict(wind_direction=360.0, spread=1.0),
    "no_spread_swell2": dict(spread=0.0, swell=2.0),
    "shallow_long_waves": dict(tile_length=(4000.0, 4000.0)),                   # tanh(k*depth) < 1 on most texels
    "tiny_tile": dict(tile_length=(0.5, 0.5)),
    "whitecap_high_foam_max": dict(whitecap=1.6, foam_amount=10.0),
    "seed_wrap": dict(spectrum_seed=(-10000, 2147483600)),                      # uvec2(id + seed) wraps
    "late_time": dict(time=36000.0),
    "calm": dict(wind_speed=0.0001, fetch_length=0.0001),
}
