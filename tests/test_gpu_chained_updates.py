"""Consecutive single updates whose persistent launches overlap at the step boundary: a launch that directly follows another
update's persistent launch on the generator's stream is queued as its programmatic dependent (its teams start while the
previous launch drains, and wait for that grid before their first item), and the work counter is reset by the launch that
used it, not by a memset between the two.

On the bench workload (256^2 x 128 cascades of bench.synth_params) back-to-back update_all calls are interleaved with every
kind of call that ends such a chain -- an overlapped snapshot, a surface query, a velocity refresh, the profiled two-kernel
path and back, fused frames -- and every map of every cascade is compared bit for bit with the oracle, with one persistent
launch per update."""
import ctypes

import numpy as np
import pytest

from bench import synth_params
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu

N, C = 256, 128
DELTA = 1.0 / 50.0


def _gow():
    import godotoceanwaves_b200 as gow
    return gow


@pytest.fixture(autouse=True)
def _modes():
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    yield
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)


@pytest.fixture(autouse=True)
def _default_queue_shape(monkeypatch):
    monkeypatch.delenv("OCEAN_QUEUE_GROUP", raising=False)
    monkeypatch.delenv("OCEAN_QUEUE_LAG", raising=False)


def _maps_equal(d16, n16, o, what):
    bad_d = np.flatnonzero((d16.view(np.uint16) != o.displacement_map).reshape(C, -1).any(axis=1))
    bad_n = np.flatnonzero((n16.view(np.uint16) != o.normal_map).reshape(C, -1).any(axis=1))
    assert bad_d.size == 0 and bad_n.size == 0, \
        f"{what}: displacement differs in cascades {bad_d.tolist()}, normal/foam in cascades {bad_n.tolist()}"


def test_chained_updates_on_the_bench_workload():
    gow = _gow()
    lib = gow.load_library()
    pg = [synth_params(gow.WaveCascadeParameters, c) for c in range(C)]
    pc = [synth_params(po.CascadeParams, c) for c in range(C)]
    g = gow.WaveGenerator()
    g.map_size = N
    g.init_gpu(C)
    o = po.OracleWaveGenerator(N)
    o.keep_f32 = False
    o.init_gpu(C)
    pinned = []

    def launches():
        return g.info().kernel_launches

    def steps(k, what):
        """k back-to-back update_all calls: no other entry point in between, so launches 2..k are chained."""
        before = launches()
        for _ in range(k):
            g.update_all(DELTA, pg)
            o.update_all_batched(DELTA, pc)
        assert launches() - before == k, f"{what}: one persistent launch per update"

    def check(what):
        _maps_equal(*g.maps_to_host(), o, what)

    try:
        g.update_all(DELTA, pg)                         # spectra and dispersion tables, then the first (unchained) update
        o.update_all_batched(DELTA, pc)
        check("first update")
        steps(6, "back to back")
        check("six chained updates")

        # an overlapped snapshot between two updates: the maps it copies are those of the update before it
        n = C * N * N * 4
        ptrs = []
        for _ in range(2):
            p = ctypes.c_void_p()
            gow.native.check(lib.ocean_host_alloc(ctypes.byref(p), 2 * n))
            pinned.append(p.value)
            ptrs.append(p.value)
        gow.native.check(lib.ocean_snapshot_maps_to_host_async(g.context, 0, C, ptrs[0], ptrs[1]))
        snap = (o.displacement_map.copy(), o.normal_map.copy())
        steps(3, "after a snapshot")
        gow.native.check(lib.ocean_wait_snapshot(g.context))
        d = np.ctypeslib.as_array((ctypes.c_uint16 * n).from_address(ptrs[0])).reshape(C, N, N, 4)
        nm = np.ctypeslib.as_array((ctypes.c_uint16 * n).from_address(ptrs[1])).reshape(C, N, N, 4)
        assert np.array_equal(d, snap[0]) and np.array_equal(nm, snap[1]), "snapshot taken between chained updates"
        check("three updates after a snapshot")

        # a surface query and a velocity refresh between updates
        scales = g.map_scales(pg)
        pts = np.array([[0.0, 0.0], [13.5, -7.25], [250.0, 91.0]], dtype=np.float32)
        g.query_surface(pts, scales)
        steps(2, "after a surface query")
        assert g.update_velocity() == C
        steps(3, "after a velocity refresh")
        check("after a query and a velocity refresh")

        # the profiled two-kernel path and back
        g.set_profiling(True)
        g.update_all(DELTA, pg)
        o.update_all_batched(DELTA, pc)
        g.set_profiling(False)
        steps(3, "after the profiled path")
        check("after the profiled path")

        # fused frames after chained updates, and chained updates after fused frames
        before = launches()
        g.update_frames(DELTA, pg, 3)
        for _ in range(3):
            o.update_all_batched(DELTA, pc)
        assert launches() - before == 1 + 1                # frame 0 as update_all, frames 1 and 2 in one fused launch
        steps(4, "after fused frames")
        check("after fused frames")
        assert [p.time for p in pg] == [p.time for p in pc]
        assert g.maps_to_host(0, 1)[1][0][..., 3].max() > 0     # foam was carried
    finally:
        g.free()
        for p in pinned:
            gow.native.check(lib.ocean_host_free(p))
