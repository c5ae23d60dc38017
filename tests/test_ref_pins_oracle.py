"""Pins the oracle to the reference itself.

oracle/_ref/libocean_ref.so is the reference's OWN six compute shaders (assets/shaders/compute/*.glsl, text unmodified
apart from the lexical plumbing listed in oracle/ref/glsl2cpp.py) compiled for the CPU and driven like
assets/water/wave_generator.gd drives them (oracle/pyref.py).  These tests assert that oracle/ocean_oracle.c -- the C
restatement every GPU parity test compares the CUDA path against -- reproduces the shaders' outputs BIT FOR BIT: the
butterfly table, the spectrum texture, both halves of the FFT buffer and both RGBA16F maps, for the BASELINE configs that
a CPU finishes in seconds, the parameter corners, the update/_process interleaving and every numeric-policy mode.

The shaders' outputs are stored as CRC-32 of every resource after every checked update in tests/golden/ref_pins/ref_pins.json
(written by tools/make_golden.py from oracle/_ref), so the oracle is checked against them everywhere; where oracle/_ref is
available the shaders are run again and must still give the stored values.
"""
import json
import os
import zlib

import numpy as np
import pytest

from conftest import EDGE_CASES, ROOT, demo_params
from oracle import pyoracle as po
from oracle import pyref as pr

MODES = [("detmath_fma", po.MATH_DET, po.CONTRACT_FMA), ("detmath_strict", po.MATH_DET, po.CONTRACT_STRICT),
         ("libm_strict", po.MATH_LIBM, po.CONTRACT_STRICT), ("libm_fma", po.MATH_LIBM, po.CONTRACT_FMA)]
CONFIGS = [(128, 1, 1), (256, 4, 2)]
CONFIG_IDS = ["cfg1_128x1", "cfg2_256x4"]
RESOURCES = ("butterfly table", "spectrum texture", "fft_buffer (both halves)", "displacement map", "normal/foam map")
PINS_PATH = os.path.join(ROOT, "tests", "golden", "ref_pins", "ref_pins.json")


@pytest.fixture(autouse=True)
def _restore_modes():
    yield
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    if pr.available():
        pr.set_modes(po.MATH_DET, po.CONTRACT_FMA)


def _crc(a) -> int:
    return zlib.crc32(np.ascontiguousarray(a).tobytes()) & 0xFFFFFFFF


def state_crcs(g):
    return [_crc(g.butterfly), _crc(g.spectrum), _crc(g.fft_buffer), _crc(g.displacement_map), _crc(g.normal_map)]


def set_modes(gen_cls, math_mode, contract):
    po.set_modes(math_mode, contract)
    if gen_cls is pr.RefWaveGenerator:
        pr.set_modes(math_mode, contract)


# ---- the checked scenarios: each runs one generator class and returns the state CRCs after every checked update
def run_config(gen_cls, N, C, frames, math_mode, contract):
    """BASELINE.json configs[0] and configs[1]: every resource after each update."""
    set_modes(gen_cls, math_mode, contract)
    g, params = gen_cls(N), [demo_params(po.CascadeParams, c) for c in range(C)]
    states = []
    for _ in range(frames):
        g.update_all(1.0 / 50.0, params)
        states.append(state_crcs(g))
    states.append([float(p.time) for p in params])    # the host-side time bookkeeping
    return states


def run_corner(gen_cls, name):
    N, states = 128, []
    for contract in (po.CONTRACT_FMA, po.CONTRACT_STRICT):
        set_modes(gen_cls, po.MATH_DET, contract)
        g, params = gen_cls(N), [demo_params(po.CascadeParams, c, **EDGE_CASES[name]) for c in range(2)]
        for delta in (0.02, 0.0, 0.031):
            g.update_all(delta, params)
        states.append(state_crcs(g))
    return states


def run_foam_loop(gen_cls):
    """update()/_process() interleaving (wave_generator.gd:56-63,90-109) and the foam state carried through RGBA16F
    (fft_unpack.glsl:59-67) over 10 frames of the three demo cascades."""
    set_modes(gen_cls, po.MATH_DET, po.CONTRACT_FMA)
    N, C = 128, 3
    g, params = gen_cls(N), [demo_params(po.CascadeParams, c) for c in range(C)]
    rng = np.random.default_rng(11)
    for f in range(10):
        g.update(1.0 / 50.0 + float(rng.uniform(0, 0.004)), params)
        for _ in range(int(rng.integers(0, C + 1))):
            g.process()
        if f == 4:                                   # a parameter change mid-run regenerates one spectrum
            params[1].wind_speed = 12.5
            params[1].should_generate_spectrum = True
    g.update(0.02, params)
    while g.pass_num_cascades_remaining:
        g.process()
    assert g.normal_half()[0][..., 3].max() > 0
    return [state_crcs(g)]


def run_random(gen_cls, kw, contract, delta):
    """One draw over the whole @export_range space of wave_cascade_parameters.gd (and beyond): two updates at 128x128."""
    set_modes(gen_cls, po.MATH_DET, contract)
    g, params = gen_cls(128), [po.CascadeParams(**{k: tuple(v) if isinstance(v, list) else v for k, v in kw.items()})]
    states = []
    for _ in range(2):
        g.update_all(delta, params)
    states.append(state_crcs(g))
    return states


def _pins():
    with open(PINS_PATH) as f:
        return json.load(f)


def _assert_pinned(case, run):
    """The oracle reproduces the stored reference state CRCs; so do the reference shaders themselves where available."""
    want = _pins()[case]
    kinds = [po.OracleWaveGenerator] + ([pr.RefWaveGenerator] if pr.available() else [])
    for gen_cls in kinds:
        got = run(gen_cls)
        assert len(got) == len(want), (case, gen_cls.__name__)
        for k, (g, w) in enumerate(zip(got, want)):
            assert g == w, f"{case} ({gen_cls.__name__}), entry {k}: {_differing(g, w)} differ from the reference shaders"


def _differing(got, want) -> str:
    if len(got) != len(RESOURCES):
        return "cascade times"
    return ", ".join(RESOURCES[i] for i in range(len(RESOURCES)) if got[i] != want[i])


@pytest.mark.skipif(not pr.available(), reason="oracle/_ref (the reference shaders compiled for the CPU) is not available")
def test_reference_shaders_compiled():
    L = pr.lib()
    for s in pr.SHADERS:
        assert L.ref_has_shader(s.encode())
    import ctypes as C
    xyz = (C.c_int * 3)()
    assert L.ref_local_size(b"fft_compute", xyz) == 0 and tuple(xyz) == (1024, 1, 1)       # fft_compute.glsl:12
    assert L.ref_local_size(b"fft_unpack", xyz) == 0 and tuple(xyz) == (16, 16, 2)         # fft_unpack.glsl:11


@pytest.mark.parametrize("mode", MODES, ids=[m[0] for m in MODES])
@pytest.mark.parametrize("N,C,frames", CONFIGS, ids=CONFIG_IDS)
def test_oracle_reproduces_reference_shaders(N, C, frames, mode):
    """BASELINE.json configs[0] and configs[1]: every resource bit-identical after each update."""
    case = f"config/{N}x{C}x{frames}/{mode[0]}"
    _assert_pinned(case, lambda gen_cls: run_config(gen_cls, N, C, frames, mode[1], mode[2]))


@pytest.mark.parametrize("name", sorted(EDGE_CASES))
def test_oracle_reproduces_reference_shaders_on_parameter_corners(name):
    _assert_pinned(f"corner/{name}", lambda gen_cls: run_corner(gen_cls, name))


def test_foam_recurrence_and_scheduling_against_reference_shaders():
    _assert_pinned("foam_loop", run_foam_loop)


def test_half_conversion_of_the_oracle_equals_the_compilers():
    """RGBA16F stores: the oracle's hand-written RTNE float->half against _Float16 (what the reference build uses)."""
    L = po.lib()
    rng = np.random.default_rng(5)
    vals = np.concatenate([rng.standard_normal(20000).astype(np.float32) * np.float32(10.0) ** rng.integers(-9, 6, 20000).astype(np.float32),
                           np.array([0.0, -0.0, 65504.0, 65519.9, 65520.0, 1e-8, 5.96e-8, 2.98e-8, 2.9802325e-8, 6.1e-5, np.inf, -np.inf], np.float32)])
    got = np.array([L.oracle_float_to_half(float(v)) for v in vals], np.uint16)
    with np.errstate(over="ignore"):
        ref = vals.astype(np.float16).view(np.uint16)
    assert np.array_equal(got, ref)


def test_oracle_reproduces_reference_shaders_on_random_parameters():
    """Random draws over the whole @export_range space of wave_cascade_parameters.gd (and beyond), drawn once by
    hypothesis (tools/make_golden.py) and stored with the shaders' results: every resource bit-identical."""
    examples = _pins()["random"]
    assert len(examples) >= 12
    for i, ex in enumerate(examples):
        _assert_pinned_example(i, ex)


def _assert_pinned_example(i, ex):
    kinds = [po.OracleWaveGenerator] + ([pr.RefWaveGenerator] if pr.available() else [])
    for gen_cls in kinds:
        got = run_random(gen_cls, ex["kw"], ex["contract"], ex["delta"])
        assert got == ex["states"], f"random example {i} {ex['kw']} contract={ex['contract']} ({gen_cls.__name__}): {_differing(got[0], ex['states'][0])} differ"
