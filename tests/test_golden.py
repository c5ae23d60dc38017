"""Committed golden vectors (tests/golden/*.json, written by tools/make_golden.py FROM THE REFERENCE'S OWN SHADERS compiled
for the CPU, oracle/_ref): the C oracle and oracle/_ref reproduce them here, the CUDA path reproduces them on the H100."""
import glob
import json
import os
import zlib

import numpy as np
import pytest

from conftest import ROOT, demo_params

GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "*.json")))


def _crc(a) -> int:
    return zlib.crc32(np.ascontiguousarray(a).tobytes()) & 0xFFFFFFFF


def _sub(a, step) -> str:
    return np.ascontiguousarray(a[:, ::step, ::step]).tobytes().hex()


def _points(n, seed):
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-300.0, 300.0, (n, 2)).astype(np.float32)
    pts[:4] = np.array([[0, 0], [88.0, -88.0], [-1234.5, 987.25], [0.34375, 0.34375]], np.float32)
    return pts


def _scales(params):
    return np.array([[np.float32(1.0) / np.float32(p.tile_length[0]), np.float32(1.0) / np.float32(p.tile_length[1]),
                      p.displacement_scale, p.normal_scale] for p in params], np.float32)


def test_golden_files_present():
    assert len(GOLDEN) >= 3


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_reproduces_golden(path):
    from oracle import pyoracle as po
    from oracle import sampling as sp
    g = json.load(open(path))
    N, C = g["N"], g["C"]
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    gen = po.OracleWaveGenerator(N)
    gen.init_gpu(max(2, C))
    params = [demo_params(po.CascadeParams, c) for c in range(C)]
    for f in range(g["frames"]):
        gen.update_all(1.0 / 50.0, params)
        assert _crc(gen.displacement_map[:C]) == g["frames_crc"][f]["displacement"], f"displacement map, frame {f}"
        assert _crc(gen.normal_map[:C]) == g["frames_crc"][f]["normal"], f"normal/foam map, frame {f}"
    assert _crc(gen.spectrum[:C]) == g["spectrum_crc"]
    assert _sub(gen.spectrum[:C], g["subsample_step"]) == g["spectrum_sub"]
    assert _sub(gen.displacement_map[:C], g["subsample_step"]) == g["displacement_sub"]
    assert _sub(gen.normal_map[:C], g["subsample_step"]) == g["normal_sub"]
    q = g["query"]
    d, gr = sp.sample_maps(gen.displacement_map[:C].view(np.float16), gen.normal_map[:C].view(np.float16), _points(q["n"], q["points_seed"]),
                           _scales(params))
    assert _crc(d) == q["displacement_crc"] and _crc(gr) == q["gradient_foam_crc"]
    assert d[:4].tobytes().hex() == q["displacement_head"] and gr[:4].tobytes().hex() == q["gradient_foam_head"]


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_reference_shaders_reproduce_golden(path):
    """The provenance of the vectors: the compiled reference shaders (prebuilt oracle/_ref on the GPU box) give them."""
    from oracle import pyoracle as po
    from oracle import pyref as pr
    if not pr.available():
        pytest.skip("oracle/_ref is neither built nor buildable here")
    g = json.load(open(path))
    assert g["generator"].startswith("oracle/_ref")
    N, C = g["N"], g["C"]
    pr.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    gen = pr.RefWaveGenerator(N)
    gen.init_gpu(max(2, C))
    params = [demo_params(po.CascadeParams, c) for c in range(C)]
    for f in range(g["frames"]):
        gen.update_all(1.0 / 50.0, params)
        assert _crc(gen.displacement_map[:C]) == g["frames_crc"][f]["displacement"], f"displacement map, frame {f}"
        assert _crc(gen.normal_map[:C]) == g["frames_crc"][f]["normal"], f"normal/foam map, frame {f}"
    assert _crc(gen.spectrum[:C]) == g["spectrum_crc"]
    assert _sub(gen.spectrum[:C], g["subsample_step"]) == g["spectrum_sub"]


@pytest.mark.gpu
@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_cuda_reproduces_golden(path):
    import godotoceanwaves_b200 as gow
    g = json.load(open(path))
    N, C = g["N"], g["C"]
    gen = gow.WaveGenerator(); gen.map_size = N; gen.init_gpu(max(2, C))
    params = [demo_params(gow.WaveCascadeParameters, c) for c in range(C)]
    for f in range(g["frames"]):
        gen.update_all(1.0 / 50.0, params)
        d, n = gen.maps_to_host(0, C)
        assert _crc(d.view(np.uint16)) == g["frames_crc"][f]["displacement"], f"displacement map, frame {f}"
        assert _crc(n.view(np.uint16)) == g["frames_crc"][f]["normal"], f"normal/foam map, frame {f}"
    spec = np.stack([gen.spectrum_to_host(c) for c in range(C)])
    assert _crc(spec) == g["spectrum_crc"]
    assert _sub(spec, g["subsample_step"]) == g["spectrum_sub"]
    q = g["query"]
    dq, gq = gen.sample(_points(q["n"], q["points_seed"]), gow.WaveGenerator.map_scales(params))
    assert _crc(dq) == q["displacement_crc"] and _crc(gq) == q["gradient_foam_crc"]
    gen.free()
