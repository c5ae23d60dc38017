"""GPU parity of the synthesis launch paths that the single-update tests of test_gpu_parity.py do not reach, against the
CPU oracle, bit for bit:

  * the production persistent kernel without taps (k_update_persistent<N, false>) at 512^2 and 1024^2, default queue;
  * fused frames (ocean_update_frames) at 1024^2;
  * the two-kernel pipeline (k_modulate_rowfft<N> + k_colfft_unpack<N, TAPS>) at every N, chunked by chunk_cascades(N),
    which every update takes while profiling is on;
  * switching between the two pipelines in the middle of a run (profiling on and off, pending cascades, fused frames);
  * the parameter corners and the generic-math kernels of test_gpu_parity.py (run there at 128^2) at 256^2 to 1024^2;
  * the cold exact-division fix-up of the column pass next to cascades that take the fast path.

The oracle of cascade c depends only on demo_params(c), so a few cascades of a large generator are checked against an
oracle that runs just those."""
import numpy as np
import pytest

from conftest import EDGE_CASES, demo_params
from oracle import pyoracle as po
from test_gpu_parity import _bits_equal, _pair, _same_values, check_edge_case, check_generic_math_path

pytestmark = pytest.mark.gpu


def _gow():
    import godotoceanwaves_b200 as gow
    return gow


def _chunk(N):
    """chunk_cascades(N) of ocean_kernels.cu: cascades per launch pair of the two-kernel pipeline (24 MiB of row-pass
    scratch at 32 B per texel): 48, 12, 3, 1 for N = 128, 256, 512, 1024."""
    return max(1, (24 << 20) // (N * N * 32))


def _generator(N, C):
    g = _gow().WaveGenerator()
    g.map_size = N
    g.init_gpu(C)
    return g


def _oracle(N, keep_f32=False):
    o = po.OracleWaveGenerator(N)
    o.keep_f32 = keep_f32
    return o


def _maps_equal(g, o, gpu_layers, oracle_layers):
    d16, n16 = g.maps_to_host(0, max(gpu_layers) + 1)
    for c, k in zip(gpu_layers, oracle_layers):
        assert _bits_equal(d16[c].view(np.uint16), o.displacement_map[k]), f"displacement of cascade {c}"
        assert _bits_equal(n16[c].view(np.uint16), o.normal_map[k]), f"normal/foam of cascade {c}"


@pytest.fixture(autouse=True)
def _modes():
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    yield
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)


@pytest.mark.parametrize("N,C", [(1024, 4), (512, 5)])
def test_persistent_kernel_default_queue(N, C):
    """k_update_persistent<N, false> with the default queue: at 1024^2 four groups of one cascade at lag 2, at 512^2
    groups of 2, 2 and 1 (a short last group).  A parameter edit before the third update runs the spectrum and table
    kernels again in the middle of the run."""
    gow = _gow()
    pg, pcpu = _pair(gow.WaveCascadeParameters, C)
    g = _generator(N, C)
    o = _oracle(N)
    launches = []
    for k, delta in enumerate((0.02, 0.02, 0.031)):
        if k == 2:
            pg[1].wind_speed = 7.5
            pcpu[1].wind_speed = 7.5
            pcpu[1].should_generate_spectrum = True
            assert pg[1].should_generate_spectrum
        before = g.info().kernel_launches
        g.update_all(delta, pg)
        o.update_all(delta, pcpu)
        launches.append(g.info().kernel_launches - before)
        _maps_equal(g, o, range(C), range(C))
    # one persistent launch per update (the two-kernel pipeline would take 2 per chunk), plus spectrum and tables
    assert launches[1] == 1 and launches[0] >= 2 and launches[2] >= 2, launches
    g.free()


def test_fused_frames_full_size():
    """ocean_update_frames at 1024^2 (256/C frames per launch) == five update_all calls == the oracle."""
    gow = _gow()
    N, C, frames = 1024, 2, 5
    pa, pcpu = _pair(gow.WaveCascadeParameters, C)
    pb, _ = _pair(gow.WaveCascadeParameters, C)
    a, b = _generator(N, C), _generator(N, C)
    o = _oracle(N)
    la, lb = a.info().kernel_launches, b.info().kernel_launches
    a.update_frames(0.02, pa, frames)
    for _ in range(frames):
        b.update_all(0.02, pb)
        o.update_all(0.02, pcpu)
    la, lb = a.info().kernel_launches - la, b.info().kernel_launches - lb
    assert la < lb, (la, lb)                                   # the frames after the first were fused
    assert [p.time for p in pa] == [p.time for p in pb] == [p.time for p in pcpu]
    da, na = a.maps_to_host(0, C)
    db, nb = b.maps_to_host(0, C)
    assert _bits_equal(da, db) and _bits_equal(na, nb)
    _maps_equal(a, o, range(C), range(C))
    a.free(); b.free()


@pytest.mark.parametrize("taps", [False, True], ids=["untapped", "taps"])
@pytest.mark.parametrize("N", [128, 256, 512, 1024])
def test_profiled_two_kernel_pipeline(N, taps):
    """Profiling on: chunk_cascades(N) + 1 cascades, so every update is two chunks of one launch pair each.
    Cascades of both chunks are compared with the oracle; with taps (k_colfft_unpack<N, true>) also their binary32 maps
    and row pass."""
    gow = _gow()
    ch = _chunk(N)
    C = ch + 1
    pick = sorted({0, ch - 1, ch})                             # first and last of chunk 1, the only cascade of chunk 2
    pg = [demo_params(gow.WaveCascadeParameters, c) for c in range(C)]
    pcpu = [demo_params(po.CascadeParams, c) for c in pick]
    g = _generator(N, C)
    g.set_profiling(True)
    if taps:
        g.enable_f32_taps(True)
    o = _oracle(N, keep_f32=taps)
    before = g.info().kernel_launches
    g.update_all(0.02, pg)
    o.update_all(0.02, pcpu)
    first = g.info().kernel_launches
    assert first - before == 2 * 2 + 2                         # two chunks, plus one spectrum and one table launch
    g.update_all(0.02, pg)
    o.update_all(0.02, pcpu)
    assert g.info().kernel_launches - first == 2 * 2
    _maps_equal(g, o, pick, range(len(pick)))
    if taps:
        for k, c in enumerate(pick):
            d32, n32 = g.f32_maps_to_host(c)
            assert _bits_equal(d32, o.displacement_f32[k]) and _bits_equal(n32, o.normal_f32[k]), f"binary32 maps of cascade {c}"
            rp = g.rowpass_to_host(c)
            assert _same_values(rp, np.ascontiguousarray(np.swapaxes(o.fft_buffer[k, 0], 1, 2))), f"row pass of cascade {c}"
    g.free()


def test_switching_pipelines_mid_run():
    """256^2 x 4 over 14 frames: profiled updates take the two-kernel pipeline, the others the persistent kernel, so the
    host re-uploads the completion counters at every switch.  Frames mix update() with cascades left pending, _process(),
    update_all() and update_frames() with profiling on (frame by frame) and off (fused), and end in the order of bench.py:
    profiling on for several frames, then off.  Foam is carried through all of it."""
    gow = _gow()
    N, C = 256, 4
    pg, pcpu = _pair(gow.WaveCascadeParameters, C)
    g = _generator(N, C)
    o = _oracle(N)
    rng = np.random.default_rng(21)
    frames = 0

    def profiled(n):
        _, row_ms, col_ms, chunk = g.last_kernel_times()
        assert row_ms > 0 and col_ms > 0 and chunk == min(n, _chunk(N)), (row_ms, col_ms, chunk, n)

    def update_all(prof):
        nonlocal frames
        g.set_profiling(prof)
        delta = 0.02 + float(rng.uniform(0, 0.004))
        g.update_all(delta, pg)
        o.update_all(delta, pcpu)
        frames += 1
        if prof:
            profiled(C)

    def update_process(prof, nproc):
        nonlocal frames
        g.set_profiling(prof)
        pending = o.pass_num_cascades_remaining
        delta = 0.02 + float(rng.uniform(0, 0.004))
        g.update(delta, pg)
        o.update(delta, pcpu)
        frames += 1
        if prof and pending:
            profiled(pending)                                  # update() flushed the pending cascades of the last pass
        for _ in range(nproc):
            g._process(0.0)
            o.process()
            if prof:
                profiled(1)
        assert g.pass_num_cascades_remaining == o.pass_num_cascades_remaining == C - nproc

    def update_frames(prof):
        nonlocal frames
        g.set_profiling(prof)
        g.update_frames(0.02, pg, 3)
        for _ in range(3):
            o.update_all(0.02, pcpu)
        frames += 3
        if prof:
            profiled(C)

    def checkpoint():
        assert [p.time for p in pg] == [p.time for p in pcpu]
        _maps_equal(g, o, range(C), range(C))

    update_all(False)
    update_process(False, 1)
    update_process(True, 2)                                    # flushes 3 pending cascades profiled, then 2 _process
    update_all(True)
    update_frames(False)                                       # fused
    checkpoint()
    update_process(True, 0)                                    # all four left pending ...
    update_frames(True)                                        # ... flushed by the first of three profiled frames
    update_process(False, 3)                                   # first unprofiled frame after the profiled ones
    checkpoint()
    update_all(False)
    update_process(False, 2)
    while o.pass_num_cascades_remaining:
        g._process(0.0)
        o.process()
    assert frames == 14 and g.pass_num_cascades_remaining == 0
    checkpoint()
    assert g.maps_to_host(0, 1)[1][0][..., 3].max() > 0       # foam was carried
    g.free()


@pytest.mark.parametrize("name", sorted(EDGE_CASES))
@pytest.mark.parametrize("N", [256, 512, 1024])
def test_edge_case_parameters_all_sizes(N, name):
    """test_edge_case_parameters (128x128) at the other map sizes: the column pass, its plan and its exact-division
    fix-up are a different kernel instance at each N."""
    check_edge_case(N, name)


@pytest.mark.parametrize("N", [256, 512, 1024])
def test_generic_math_path_all_sizes(N):
    """test_generic_math_path_for_extreme_tile_lengths (128x128) at the other map sizes."""
    check_generic_math_path(N)


@pytest.mark.parametrize("N", [128, 256, 512, 1024])
def test_division_fixup_beside_the_fast_path(N):
    """A calm cascade (every gradient numerator an exact zero: the cold div.rn.f32 fix-up of the column pass rewrites its
    gradients) in one launch with a demo cascade whose quotients keep the branch-free fast path; three updates as
    test_edge_case_parameters runs them."""
    gow = _gow()
    over = EDGE_CASES["calm"]
    pg = [demo_params(gow.WaveCascadeParameters, 0, **over), demo_params(gow.WaveCascadeParameters, 1)]
    pcpu = [demo_params(po.CascadeParams, 0, **over), demo_params(po.CascadeParams, 1)]
    g = _generator(N, 2)
    o = _oracle(N, keep_f32=True)
    for delta in (0.02, 0.0, 0.031):
        g.update_all(delta, pg)
        o.update_all(delta, pcpu)
    grad = np.abs(o.normal_f32[:, ..., :2])
    assert np.any(grad[0] < 2.0 ** -100)                       # the fix-up runs in cascade 0 ...
    assert np.all(grad[1] >= 2.0 ** -100)                      # ... and no gradient of cascade 1 needs it
    d16, n16 = g.maps_to_host(0, 2)
    for c in range(2):
        assert _same_values(d16[c].astype(np.float32), o.displacement_half()[c].astype(np.float32)), c
        assert _same_values(n16[c].astype(np.float32), o.normal_half()[c].astype(np.float32)), c
    g.free()
