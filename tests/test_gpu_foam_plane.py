"""The foam state lives in its own [C][N][N] binary16 plane: the column pass reads the previous foam from it and writes the new
foam to it and, as the same rounded half, into normal_map.a.  These tests pin that the plane and normal.a agree bit for bit
after every launch path (one persistent launch, persistent launches split at the dispatch-table size, the profiled two-kernel
pipeline, fused frames), and that ocean_get_foam_state / ocean_set_foam_state read and seed the state the next update
consumes, against the CPU oracle."""
import numpy as np
import pytest

from conftest import demo_params
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _modes():
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    yield
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)


def _gow():
    import godotoceanwaves_b200 as gow
    return gow


def _generator(N, C):
    g = _gow().WaveGenerator()
    g.map_size = N
    g.init_gpu(C)
    return g


def _oracle(N, C):
    o = po.OracleWaveGenerator(N)
    o.keep_f32 = False
    o.init_gpu(C)
    return o


def _params(n, **over):
    return ([demo_params(_gow().WaveCascadeParameters, c, whitecap=1.2, foam_amount=8.0, **over) for c in range(n)],
            [demo_params(po.CascadeParams, c, whitecap=1.2, foam_amount=8.0, **over) for c in range(n)])


def _plane_is_normal_alpha(g, count, what):
    _, n16 = g.maps_to_host(0, count)
    alpha = n16.view(np.uint16)[..., 3]
    for c in range(count):
        plane = g.get_foam_state(c).view(np.uint16)
        assert np.array_equal(plane, alpha[c]), f"{what}: foam plane != normal.a in cascade {c}"
    assert alpha.any(), f"{what}: no foam at all (the test would not see a stale plane)"


def _maps_equal_oracle(g, o, count, what):
    d16, n16 = g.maps_to_host(0, count)
    assert np.array_equal(d16.view(np.uint16), o.displacement_map[:count]), f"{what}: displacement differs from the oracle"
    assert np.array_equal(n16.view(np.uint16), o.normal_map[:count]), f"{what}: normal/foam differs from the oracle"


@pytest.mark.parametrize("path", ["persistent", "split_launches", "profiled", "fused_frames"])
def test_plane_equals_normal_alpha(path):
    """After several updates on each launch path the plane equals normal.a, and the maps equal the oracle's (so the plane
    carried the foam from update to update as normal.a did)."""
    N, C = (128, 300) if path == "split_launches" else (256, 12)   # 300 records: two persistent launches per update
    g, o = _generator(N, C), _oracle(N, C)
    pg, pc = _params(C)
    if path == "profiled":
        g.set_profiling(True)
    g.update_all(0.02, pg)
    o.update_all_batched(0.02, pc)
    if path == "fused_frames":
        g.update_frames(0.02, pg, 4)                # one launch: each frame's column pass reads the plane the previous one wrote
    else:
        for _ in range(4):
            g.update_all(0.02, pg)
    for _ in range(4):
        o.update_all_batched(0.02, pc)
    _maps_equal_oracle(g, o, C, path)
    _plane_is_normal_alpha(g, C, path)
    g.free()


def test_set_get_round_trip_and_seed():
    """set_foam_state writes the plane and normal.a; get_foam_state returns it unchanged; the next update starts from it
    exactly as the oracle does from the same normal.a, on both update paths."""
    N, C = 128, 3
    rng = np.random.default_rng(7)
    for profiled in (False, True):
        g, o = _generator(N, C), _oracle(N, C)
        g.set_profiling(profiled)
        pg, pc = _params(C)
        for _ in range(2):
            g.update_all(0.02, pg)
            o.update_all_batched(0.02, pc)
        seeds = {c: rng.uniform(0.0, 1.0, (N, N)).astype(np.float16) for c in (0, 2)}
        seeds[2][:8] = 0.0                              # exact zeros and ones as well
        seeds[2][8:16] = 1.0
        for c, f in seeds.items():
            g.set_foam_state(c, f)
            o.normal_map[c][..., 3] = f.view(np.uint16)
            assert np.array_equal(g.get_foam_state(c).view(np.uint16), f.view(np.uint16))
        _, n16 = g.maps_to_host(0, C)
        for c, f in seeds.items():
            assert np.array_equal(n16.view(np.uint16)[c][..., 3], f.view(np.uint16)), f"normal.a of cascade {c} is not the seed"
        g.update_all(0.02, pg)
        o.update_all_batched(0.02, pc)
        _maps_equal_oracle(g, o, C, f"update after set_foam_state (profiled={profiled})")
        _plane_is_normal_alpha(g, C, f"update after set_foam_state (profiled={profiled})")
        g.free()
