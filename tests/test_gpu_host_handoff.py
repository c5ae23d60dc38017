"""The hand-off of the maps from the device to their consumer, byte for byte on the RGBA16F maps:

  * the overlapped snapshot (ocean_snapshot_maps_to_host_async / ocean_wait_snapshot): a device-to-device copy on the
    generator's stream, then a device-to-host copy on a second stream, ordered by two events.  It is the one path of the
    library that crosses streams, and bench.py's end-to-end figure runs through it;
  * ocean_copy_maps_to_host_async with ocean_synchronize, pinned (ocean_host_alloc) and pageable destinations;
  * the device pointers of ocean_get_maps, read through __cuda_array_interface__;
  * several generators sharing one device, each on its own stream with a persistent kernel sized for the whole device.

References: the CPU oracle at small shapes; at the bench shape, a second generator of that shape read after every step through
the synchronous copy (test_gpu_batch_shapes ties that path to the oracle there), kept as a CRC-32 per layer and step.  The
entry points the Python mirror does not wrap are called through load_library() and ctypes, as bench.py calls them.  Host
buffers start filled with a half NaN the maps never hold, so bytes no copy wrote stay recognisable."""
import ctypes
import zlib

import numpy as np
import pytest

from bench import synth_params
from oracle import pyoracle as po
from oracle import velocity as ov

pytestmark = pytest.mark.gpu

DELTA = 1.0 / 50.0
BENCH_N, BENCH_C = 256, 128          # bench.py's default workload: 32 sets of 4 cascades
BENCH_WARMUP = 5                     # bench.py's default --warmup
E2E_STEPS = 20                       # bench.py's e2e_steps at its default --steps: max(3, min(steps, 20))
BENCH_STEPS = 1 + BENCH_WARMUP + 2 + E2E_STEPS    # the creating update, the warm-up, two priming snapshots, the e2e loop
SENTINEL = 0x7E5A                    # a quiet half NaN: no map texel holds it
INVALID_ARGUMENT = 1                 # OCEAN_ERR_INVALID_ARGUMENT


def _gow():
    import godotoceanwaves_b200 as gow
    return gow


def _lib():
    return _gow().load_library()


def _check(status):
    _gow().native.check(status)


def _ptr(a):
    return None if a is None else a.ctypes.data


@pytest.fixture(autouse=True)
def _modes():
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    yield
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)


class _Handoff:
    """The generators and pinned host buffers of one test.  close() destroys the generators first -- which waits for their
    streams, the copy stream included, so no copy still writes -- and then frees the buffers."""

    def __init__(self):
        self.gens, self.bufs = [], []

    def generator(self, N, C):
        g = _gow().WaveGenerator()
        g.map_size = N
        g.init_gpu(C)
        self.gens.append(g)
        return g

    def pinned(self, *shape):
        """A uint16 array of `shape` in pinned memory from ocean_host_alloc, filled with SENTINEL."""
        n = int(np.prod(shape))
        p = ctypes.c_void_p()
        _check(_lib().ocean_host_alloc(ctypes.byref(p), 2 * n))
        self.bufs.append(p.value)
        a = np.ctypeslib.as_array((ctypes.c_uint16 * n).from_address(p.value)).reshape(shape)
        a.fill(SENTINEL)
        return a

    def pair(self, N, layers):
        return self.pinned(layers, N, N, 4), self.pinned(layers, N, N, 4)

    def close(self):
        for g in self.gens:
            g.free()
        while self.bufs:
            _check(_lib().ocean_host_free(self.bufs.pop()))


@pytest.fixture
def handoff():
    h = _Handoff()
    yield h
    h.close()


def _snapshot(g, first, count, disp, norm):
    _check(_lib().ocean_snapshot_maps_to_host_async(g.context, first, count, _ptr(disp), _ptr(norm)))


def _wait(g):
    _check(_lib().ocean_wait_snapshot(g.context))


def _copy_async(g, first, count, disp, norm):
    _check(_lib().ocean_copy_maps_to_host_async(g.context, first, count, _ptr(disp), _ptr(norm)))


def _crcs(maps):
    """CRC-32 of every layer of a [C][N][N][4] map."""
    return [zlib.crc32(np.ascontiguousarray(layer)) for layer in maps]


def _state(disp, norm):
    """(displacement CRCs, normal CRCs) of a state of the maps, from uint16 or float16 arrays."""
    return _crcs(disp.view(np.uint16)), _crcs(norm.view(np.uint16))


def _device_state(g):
    return _state(*g.maps_to_host())


def _oracle_state(o):
    return _state(o.displacement_map, o.normal_map)


def _oracle(N, C):
    o = po.OracleWaveGenerator(N)
    o.keep_f32 = False
    o.init_gpu(C)
    return o


def _untouched(buf, what):
    assert (buf == SENTINEL).all(), f"{what}: a copy wrote into a buffer it was not given"


def _expect(buf, state, which, first, count, what, history=None):
    """buf[0:count] holds layers [first, first + count) of map `which` (0 displacement, 1 normal) of `state`, and nothing
    was written after them.  With `history` (states by step) the message names the steps a wrong layer does match."""
    got = _crcs(buf[:count])
    bad = [first + k for k in range(count) if got[k] != state[which][first + k]]
    if bad:
        msg = f"{what}: {('displacement', 'normal')[which]} layers {bad[:8]}{'...' if len(bad) > 8 else ''} differ"
        if history is not None:
            c = bad[0]
            steps = [k for k, s in enumerate(history) if s[which][c] == got[c - first]]
            msg += f"; layer {c} holds the maps of step(s) {steps} (none: torn or never written)"
        raise AssertionError(msg)
    _untouched(buf[count:], f"{what}: beyond its {count} layers")


def _expect_pair(bufs, state, first, count, what, history=None):
    for which in (0, 1):
        _expect(bufs[which], state, which, first, count, what, history)


class _Launches:
    def __init__(self, g):
        self.g, self.last = g, g.info().kernel_launches

    def __call__(self):
        now = self.g.info().kernel_launches
        delta, self.last = now - self.last, now
        return delta


@pytest.fixture(scope="module")
def bench_reference():
    """history[k] = the state of bench's workload after k update_all(DELTA) from synth_params (history[0]: cleared maps), read
    after every step from a generator of that shape through the synchronous copy."""
    gow = _gow()
    params = [synth_params(gow.WaveCascadeParameters, c) for c in range(BENCH_C)]
    g = gow.WaveGenerator()
    g.map_size = BENCH_N
    g.init_gpu(BENCH_C)
    try:
        history = [_device_state(g)]
        for _ in range(BENCH_STEPS):
            g.update_all(DELTA, params)
            history.append(_device_state(g))
    finally:
        g.free()
    return history


def _bench_generator(handoff):
    gow = _gow()
    return handoff.generator(BENCH_N, BENCH_C), [synth_params(gow.WaveCascadeParameters, c) for c in range(BENCH_C)]


# ---------------------------------------------------------------------------------------------------------------------------
# 1. bench.py's end-to-end loop
# ---------------------------------------------------------------------------------------------------------------------------
def test_bench_e2e_loop(handoff, bench_reference):
    """bench.py's hand-off as it runs it: the creating update and the warm-up, two priming snapshots, then E2E_STEPS of
    update_all + snapshot into two pinned buffer pairs used alternately, with no host synchronisation until the final
    ocean_wait_snapshot.  The pairs hold exactly the maps of the last two steps, every cascade; the last step's also equal
    the oracle's for a subset of the cascades (they are independent, so the oracle runs only those)."""
    g, params = _bench_generator(handoff)
    g.update_all(DELTA, params)                                    # bench: shard.update_all creates the spectra
    for _ in range(BENCH_WARMUP):
        g.update_all(DELTA, params)
    g.synchronize()
    host = [handoff.pair(BENCH_N, BENCH_C) for _ in range(2)]
    for i in range(2):
        g.update_all(DELTA, params)
        _snapshot(g, 0, BENCH_C, *host[i])
    _wait(g)
    step = 1 + BENCH_WARMUP + 2
    for i in range(2):
        _expect_pair(host[i], bench_reference[step - 1 + i], 0, BENCH_C, f"priming snapshot {i}", bench_reference)
    g.synchronize()
    launches = _Launches(g)
    for i in range(E2E_STEPS):
        g.update_all(DELTA, params)
        _snapshot(g, 0, BENCH_C, *host[i & 1])
    _wait(g)
    assert step + E2E_STEPS == BENCH_STEPS
    for i in (E2E_STEPS - 2, E2E_STEPS - 1):
        _expect_pair(host[i & 1], bench_reference[step + 1 + i], 0, BENCH_C, f"e2e step {i}", bench_reference)
    assert launches() == E2E_STEPS                                  # one persistent launch per update; snapshots add none

    subset = [0, 1, 2, 3, 37, 64, 126, 127]
    pc = [synth_params(po.CascadeParams, c) for c in subset]
    o = _oracle(BENCH_N, len(subset))
    for _ in range(BENCH_STEPS):
        o.update_all_batched(DELTA, pc)
    last = host[(E2E_STEPS - 1) & 1]
    for k, c in enumerate(subset):
        assert np.array_equal(last[0][c], o.displacement_map[k]), f"displacement of cascade {c} differs from the oracle"
        assert np.array_equal(last[1][c], o.normal_map[k]), f"normal/foam of cascade {c} differs from the oracle"


# ---------------------------------------------------------------------------------------------------------------------------
# 2. every writer of the maps, every kind of range
# ---------------------------------------------------------------------------------------------------------------------------
# (writer, first, count, displacement destination?, normal destination?); the writer runs, then the snapshot is taken
SCHEDULE = [
    ("update_all", 0, 16, True, True),
    ("partial 3", 13, 3, True, True),      # update() + 3 x _process(): cascades 15, 14, 13 written
    ("frames 3", 0, 16, True, False),      # flushes cascades 0 .. 12, then three fused frames
    ("profiled", 5, 1, False, True),       # the two-kernel pipeline; a single layer
    (None, 0, 16, True, True),             # back to back: no writer since the last snapshot
    ("update_all", 1, 15, True, True),
    ("partial 1", 15, 1, True, True),      # the top layer, the only one written
    ("frames 2", 0, 16, True, True),
    ("profiled", 3, 8, True, False),
    ("update_all", 0, 1, False, True),
    (None, 0, 16, False, False),           # both destinations NULL: nothing to copy
    ("frames 4", 0, 16, True, True),
    ("partial 5", 11, 5, True, True),
    ("update_all", 0, 16, True, True),
    (None, 2, 7, True, True),
]


def test_every_snapshot_lands_intact(handoff):
    """256^2 x 16: a snapshot after each way of writing the maps on the generator's stream -- update_all, a partial pass
    (update + _process), fused frames, the profiled two-kernel update -- over ranges with first > 0, single layers and the
    whole stack, some with a NULL destination, two back to back; one pinned buffer pair per snapshot, no host
    synchronisation until the end.  Each buffer equals the oracle's maps at the moment of its call (one spare layer
    past the range stays unwritten), and a NULL destination leaves its buffer untouched."""
    N, C = 256, 16
    gow = _gow()
    g = handoff.generator(N, C)
    o = _oracle(N, C)
    pg = [synth_params(gow.WaveCascadeParameters, c) for c in range(C)]
    pc = [synth_params(po.CascadeParams, c) for c in range(C)]
    taken = []
    for writer, first, count, want_d, want_n in SCHEDULE:
        if writer == "update_all":
            g.update_all(DELTA, pg)
            o.update_all_batched(DELTA, pc)
        elif writer == "profiled":
            g.set_profiling(True)
            g.update_all(DELTA, pg)
            g.set_profiling(False)
            o.update_all_batched(DELTA, pc)
        elif writer is not None:
            kind, n = writer.split()
            if kind == "partial":
                g.update(DELTA, pg)
                o.update(DELTA, pc)
                for _ in range(int(n)):
                    g._process(0.0)
                    o.process()
            else:
                g.update_frames(DELTA, pg, int(n))
                for _ in range(int(n)):
                    o.update_all_batched(DELTA, pc)
        bufs = handoff.pair(N, count + 1)
        _snapshot(g, first, count, bufs[0] if want_d else None, bufs[1] if want_n else None)
        taken.append((bufs, _oracle_state(o), first, count, want_d, want_n, writer))
    _wait(g)
    for k, (bufs, state, first, count, want_d, want_n, writer) in enumerate(taken):
        what = f"snapshot {k} after {writer}, layers [{first}, {first + count})"
        for which, wanted in ((0, want_d), (1, want_n)):
            if wanted:
                _expect(bufs[which], state, which, first, count, what)
            else:
                _untouched(bufs[which], f"{what}: NULL {('displacement', 'normal')[which]} destination")
    assert [p.time for p in pg] == [p.time for p in pc]


# ---------------------------------------------------------------------------------------------------------------------------
# 3. what ocean_wait_snapshot waits for
# ---------------------------------------------------------------------------------------------------------------------------
def test_wait_returns_the_snapshotted_step(handoff, bench_reference):
    """A snapshot, six more updates enqueued at once, then ocean_wait_snapshot without ocean_synchronize: the buffer holds
    the snapshotted step, not a later one, while the generator's stream is still busy."""
    g, params = _bench_generator(handoff)
    bufs = handoff.pair(BENCH_N, BENCH_C)
    for _ in range(3):
        g.update_all(DELTA, params)
    _snapshot(g, 0, BENCH_C, *bufs)
    for _ in range(6):
        g.update_all(DELTA, params)
    _wait(g)
    _expect_pair(bufs, bench_reference[3], 0, BENCH_C, "snapshot of step 3", bench_reference)
    g.synchronize()
    assert _device_state(g) == bench_reference[9]


def test_destroy_delivers_a_snapshot_in_flight(handoff, bench_reference):
    """ocean_destroy right after a snapshot call: the snapshot still arrives whole."""
    g, params = _bench_generator(handoff)
    bufs = handoff.pair(BENCH_N, BENCH_C)
    for _ in range(2):
        g.update_all(DELTA, params)
    _snapshot(g, 0, BENCH_C, *bufs)
    g.free()
    _expect_pair(bufs, bench_reference[2], 0, BENCH_C, "snapshot delivered through ocean_destroy", bench_reference)


# ---------------------------------------------------------------------------------------------------------------------------
# 4. the asynchronous copy
# ---------------------------------------------------------------------------------------------------------------------------
def test_async_copy_equals_synchronous_copy(handoff):
    """ocean_copy_maps_to_host_async + ocean_synchronize == maps_to_host over several ranges, into pinned and pageable
    buffers, with NULL destinations.  Copies enqueued before an update hold the maps before it, those after it the new ones."""
    N, C = 256, 8
    gow = _gow()
    g = handoff.generator(N, C)
    pg = [synth_params(gow.WaveCascadeParameters, c) for c in range(C)]
    for _ in range(2):
        g.update_all(DELTA, pg)
    cases = [(0, C, True, True), (3, 4, True, True), (C - 1, 1, True, True), (0, 1, True, True), (2, 5, False, True),
             (1, 6, True, False), (4, 0, True, True)]

    def enqueue():
        out = []
        for pinned in (True, False):
            for first, count, want_d, want_n in cases:
                if pinned:
                    bufs = handoff.pair(N, count + 1)
                else:
                    bufs = tuple(np.full((count + 1, N, N, 4), SENTINEL, np.uint16) for _ in range(2))
                _copy_async(g, first, count, bufs[0] if want_d else None, bufs[1] if want_n else None)
                out.append((bufs, first, count, want_d, want_n, "pinned" if pinned else "pageable"))
        return out

    before = _device_state(g)
    copied_before = enqueue()
    g.update_all(DELTA, pg)
    copied_after = enqueue()
    _check(_lib().ocean_synchronize(g.context))
    after = _device_state(g)
    assert after != before
    for state, batch, when in ((before, copied_before, "before"), (after, copied_after, "after")):
        for bufs, first, count, want_d, want_n, kind in batch:
            what = f"{kind} copy of [{first}, {first + count}) enqueued {when} an update"
            for which, wanted in ((0, want_d), (1, want_n)):
                if wanted:
                    _expect(bufs[which], state, which, first, count, what)
                else:
                    _untouched(bufs[which], f"{what}: NULL destination")


# ---------------------------------------------------------------------------------------------------------------------------
# 5. bookkeeping and arguments
# ---------------------------------------------------------------------------------------------------------------------------
def test_snapshot_bookkeeping_and_arguments(handoff):
    """The first snapshot adds exactly its two [C][N][N] RGBA16F buffers to device_bytes and later ones add nothing;
    count == 0 is OK and allocates nothing; snapshots launch no kernel; waiting before any snapshot is OK.  A range outside
    the layers (including ones whose end overflows an int) or a NULL generator is OCEAN_ERR_INVALID_ARGUMENT for the
    snapshot, the asynchronous copy and the velocity copy alike, with nothing enqueued and nothing allocated."""
    N, C = 128, 4
    gow = _gow()
    lib = _lib()
    g = handoff.generator(N, C)
    pg = [synth_params(gow.WaveCascadeParameters, c) for c in range(C)]
    g.update_all(DELTA, pg)
    bufs = handoff.pair(N, C)
    launches = _Launches(g)
    bytes0 = g.info().device_bytes

    _wait(g)                                                               # no snapshot yet
    _snapshot(g, 0, 0, *bufs)
    _snapshot(g, C, 0, *bufs)
    _copy_async(g, 2, 0, *bufs)
    bad = [(-1, 1), (0, C + 1), (C, 1), (C + 1, 0), (1, -1), (2, C - 1), (1, 2**31 - 1), (2**31 - 1, 1), (-2**31, 2**31 - 1)]
    for first, count in bad:
        for fn in (lib.ocean_snapshot_maps_to_host_async, lib.ocean_copy_maps_to_host_async):
            assert fn(g.context, first, count, _ptr(bufs[0]), _ptr(bufs[1])) == INVALID_ARGUMENT, (fn.__name__, first, count)
    for fn in (lib.ocean_snapshot_maps_to_host_async, lib.ocean_copy_maps_to_host_async):
        assert fn(None, 0, 1, _ptr(bufs[0]), _ptr(bufs[1])) == INVALID_ARGUMENT, fn.__name__
    assert lib.ocean_wait_snapshot(None) == INVALID_ARGUMENT
    velocity = np.full((C, N, N, 4), SENTINEL, np.uint16)                 # the velocity copy shares the range check
    for first, count in bad:
        assert lib.ocean_copy_velocity_to_host(g.context, first, count, _ptr(velocity)) == INVALID_ARGUMENT, (first, count)
    _wait(g)
    g.synchronize()
    assert g.info().device_bytes == bytes0
    assert launches() == 0
    _untouched(bufs[0], "count 0 and rejected ranges")
    _untouched(bufs[1], "count 0 and rejected ranges")
    _untouched(velocity, "rejected velocity ranges")

    state = _device_state(g)
    _snapshot(g, 0, C, *bufs)
    assert g.info().device_bytes == bytes0 + 2 * C * N * N * 8
    _wait(g)
    _expect_pair(bufs, state, 0, C, "first snapshot")
    g.update_all(DELTA, pg)
    launches()
    more = handoff.pair(N, 2)
    _snapshot(g, 1, 2, *more)
    _snapshot(g, 0, C, *bufs)
    for first, count in bad:
        assert lib.ocean_snapshot_maps_to_host_async(g.context, first, count, _ptr(bufs[0]), _ptr(bufs[1])) == INVALID_ARGUMENT
    _wait(g)
    assert g.info().device_bytes == bytes0 + 2 * C * N * N * 8
    assert launches() == 0
    state = _device_state(g)
    _expect_pair(more, state, 1, 2, "snapshot of layers [1, 3)")
    _expect_pair(bufs, state, 0, C, "second snapshot")


# ---------------------------------------------------------------------------------------------------------------------------
# 6. the device pointers
# ---------------------------------------------------------------------------------------------------------------------------
class _DeviceMaps:
    """[C][N][N][4] float16 at a device address, for torch.as_tensor."""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": "<f2", "data": (ptr, False), "strides": None, "version": 3}


def test_device_pointers_hold_the_documented_layout(handoff):
    """ocean_get_maps: after ocean_synchronize the pointers, read in place through __cuda_array_interface__, hold what
    maps_to_host returns as [C][N][N][4] half, layer-major and tightly packed (layer_bytes == N^2 * 8, layer c at c *
    layer_bytes); the pointers stay the same through further updates and snapshots."""
    import torch
    N, C = 256, 6
    gow = _gow()
    g = handoff.generator(N, C)
    pg = [synth_params(gow.WaveCascadeParameters, c) for c in range(C)]
    dev = torch.device("cuda", g.device)

    def pointers():
        d, n, layer = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_size_t()
        _check(_lib().ocean_get_maps(g.context, ctypes.byref(d), ctypes.byref(n), ctypes.byref(layer)))
        return d.value, n.value, layer.value

    d_ptr, n_ptr, layer_bytes = pointers()
    assert layer_bytes == N * N * 8
    assert (d_ptr, n_ptr) == (g.descriptors["displacement_map"].rid, g.descriptors["normal_map"].rid)
    bufs = handoff.pair(N, C)
    for step in range(2):
        g.update_all(DELTA, pg)
        _snapshot(g, 0, C, *bufs)
        g.update_all(DELTA, pg)
        _check(_lib().ocean_synchronize(g.context))
        host = [m.view(np.uint16) for m in g.maps_to_host()]
        assert pointers() == (d_ptr, n_ptr, layer_bytes)
        for which, ptr in enumerate((d_ptr, n_ptr)):
            whole = torch.as_tensor(_DeviceMaps(ptr, (C, N, N, 4)), device=dev)
            assert whole.data_ptr() == ptr and whole.dtype == torch.float16
            assert np.array_equal(whole.cpu().numpy().view(np.uint16), host[which]), (step, which)
            for c in (0, C // 2, C - 1):
                layer = torch.as_tensor(_DeviceMaps(ptr + c * layer_bytes, (N, N, 4)), device=dev)
                assert np.array_equal(layer.cpu().numpy().view(np.uint16), host[which][c]), (step, which, c)
        _wait(g)


# ---------------------------------------------------------------------------------------------------------------------------
# 7. generators sharing a device
# ---------------------------------------------------------------------------------------------------------------------------
def test_generators_sharing_a_device(handoff, bench_reference):
    """The bench-shape generator A and a 1024^2 x 4 generator B alive together, their updates, fused frames, profiled updates,
    a velocity recompute and snapshots interleaved with no host synchronisation; a third generator (128^2 x 4) is created
    and run while both have work queued, and freed with its snapshot in flight while they are busy; B is freed while A is
    busy.  Every snapshot and final map equals the generator's own reference (A: bench_reference, B and the third: the
    oracle), and B's velocity maps equal oracle/velocity.py's.  Whether the kernels overlapped is not asserted."""
    gow = _gow()
    A, pa = _bench_generator(handoff)
    NB, CB = 1024, 4
    B = handoff.generator(NB, CB)
    pb = [synth_params(gow.WaveCascadeParameters, c) for c in range(CB)]
    ob, pob = _oracle(NB, CB), [synth_params(po.CascadeParams, c) for c in range(CB)]
    a_snaps, b_snaps = [], []
    a_step = 0

    def step_a(kind, frames=1):
        nonlocal a_step
        if kind == "frames":
            A.update_frames(DELTA, pa, frames)
        else:
            A.set_profiling(kind == "profiled")
            A.update_all(DELTA, pa)
            A.set_profiling(False)
        a_step += frames

    def step_b(kind, frames=1):
        if kind == "frames":
            B.update_frames(DELTA, pb, frames)
        else:
            B.set_profiling(kind == "profiled")
            B.update_all(DELTA, pb)
            B.set_profiling(False)
        for _ in range(frames):
            ob.update_all_batched(DELTA, pob)

    def snap_a(first, count):
        bufs = handoff.pair(BENCH_N, count + 1)
        _snapshot(A, first, count, *bufs)
        a_snaps.append((bufs, a_step, first, count))

    def snap_b(first, count):
        bufs = handoff.pair(NB, count + 1)
        _snapshot(B, first, count, *bufs)
        b_snaps.append((bufs, _oracle_state(ob), first, count))

    step_a("update_all")
    step_b("update_all")
    snap_a(0, BENCH_C)
    snap_b(0, CB)
    step_a("frames", 3)
    step_b("frames", 2)

    # a third generator, created and run while A and B have work queued
    NC, CC = 128, 4
    T = handoff.generator(NC, CC)
    pt = [synth_params(gow.WaveCascadeParameters, c) for c in range(4, 4 + CC)]
    ot, pot = _oracle(NC, CC), [synth_params(po.CascadeParams, c) for c in range(4, 4 + CC)]
    for _ in range(2):
        T.update_all(DELTA, pt)
        ot.update_all_batched(DELTA, pot)
    t_bufs = handoff.pair(NC, CC)
    _snapshot(T, 0, CC, *t_bufs)
    t_state = _oracle_state(ot)

    step_a("profiled")
    step_b("profiled")
    snap_a(5, 64)
    step_b("update_all")
    assert B.update_velocity() == CB
    snap_b(1, 2)
    T.free()                                                       # its snapshot in flight, A and B busy
    step_a("frames", 2)
    snap_a(0, BENCH_C)
    step_a("update_all")
    snap_b(0, CB)

    # B read back and freed while A is busy; A's last snapshot then taken
    step_a("frames", 3)
    assert B.update_velocity() == 0                                # nothing written since the recompute
    vel = B.velocity_to_host(0, CB).view(np.uint16)
    b_final = _device_state(B)
    _wait(B)
    B.free()
    snap_a(0, BENCH_C)
    _wait(A)
    A.synchronize()

    _expect_pair(t_bufs, t_state, 0, CC, "third generator's snapshot")
    for k, (bufs, step, first, count) in enumerate(a_snaps):
        _expect_pair(bufs, bench_reference[step], first, count, f"A snapshot {k} (step {step}, [{first}, {first + count}))",
                     bench_reference)
    assert _device_state(A) == bench_reference[a_step]
    for k, (bufs, state, first, count) in enumerate(b_snaps):
        _expect_pair(bufs, state, first, count, f"B snapshot {k} ([{first}, {first + count}))")
    assert b_final == _oracle_state(ob), "B's final maps differ from the oracle"
    for c in range(CB):
        half, _ = ov.velocity_maps(ob.spectrum[c], ob.butterfly, po.pc_spectrum_modulate(pob[c], c))
        assert np.array_equal(vel[c], half), f"B's velocity map of cascade {c} differs from oracle/velocity.py"
