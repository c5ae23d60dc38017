"""GPU parity of the update path at the batch shapes bench.py measures and at the limits of the dispatch tables, against the
CPU oracle, bit for bit on the RGBA16F maps of every cascade:

  * the bench workload, 256^2 x 128 cascades of bench.synth_params: one k_update_persistent<256, false> launch of 16 queue
    groups (8 cascades per group, lag 1) per update_all, through parameter edits, a partial pass, fused frames and the
    profiled two-kernel pipeline (11 chunks of 12);
  * the queue shapes OCEAN_QUEUE_GROUP / OCEAN_QUEUE_LAG select, at four sizes: every shape gives the same bytes;
  * more records than one launch takes (256 dispatch records travel by value per launch): split persistent launches, fused
    frames that fill the table exactly, leave it one short or fall back to one frame at a time, and the velocity recompute
    split at 256 jobs.

Only a multi-group queue runs column-pass items beside the row passes of the next group; in every queue a team whose row-pass
item is followed by a column-pass item with a complete row pass requests that item's first column panel early.  Every case
asserts that it took the path it is named for: launch counts (info().kernel_launches), the queue the generator builds
(ocean_debug_work_queue, which reads the same overrides) and the chunk size of the profiled pipeline (last_kernel_times)."""
import numpy as np
import pytest

from bench import synth_params
from oracle import pyoracle as po
from oracle import velocity as ov
from test_queue_protocol_cpu import _queue, batch_queue_shapes, default_queue

pytestmark = pytest.mark.gpu

TABLE = 256     # dispatch records per launch: kMaxPersistentCascades, kMaxLaunchCascades, kMaxVelocityLaunch


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
    """Without overrides from the environment unless a test sets them."""
    monkeypatch.delenv("OCEAN_QUEUE_GROUP", raising=False)
    monkeypatch.delenv("OCEAN_QUEUE_LAG", raising=False)


def _generator(N, C, taps=False):
    g = _gow().WaveGenerator()
    g.map_size = N
    g.init_gpu(C)
    if taps:
        g.enable_f32_taps(True)
    return g


def _oracle(N, C, cls=po.OracleWaveGenerator):
    o = cls(N)
    o.keep_f32 = False
    o.init_gpu(C)
    return o


def _params(n):
    gow = _gow()
    return [synth_params(gow.WaveCascadeParameters, c) for c in range(n)], [synth_params(po.CascadeParams, c) for c in range(n)]


class _Launches:
    """Kernel launches since the previous call."""

    def __init__(self, g):
        self.g = g
        self.last = g.info().kernel_launches

    def __call__(self):
        now = self.g.info().kernel_launches
        delta, self.last = now - self.last, now
        return delta


def _maps_equal(g, disp, norm, what):
    """The generator's maps of cascades [0, len(disp)) == the given uint16 maps, bit for bit, every cascade."""
    count = len(disp)
    d16, n16 = g.maps_to_host(0, count)
    bad_d = np.flatnonzero((d16.view(np.uint16) != disp).reshape(count, -1).any(axis=1))
    bad_n = np.flatnonzero((n16.view(np.uint16) != norm).reshape(count, -1).any(axis=1))
    assert bad_d.size == 0 and bad_n.size == 0, \
        f"{what}: displacement differs in cascades {bad_d.tolist()}, normal/foam in cascades {bad_n.tolist()}"


def _check(g, o, what):
    _maps_equal(g, o.displacement_map, o.normal_map, what)


def _untouched(g, first, what):
    """Layers [first, num_cascades) were never written."""
    d16, n16 = g.maps_to_host(first)
    assert not d16.view(np.uint16).any() and not n16.view(np.uint16).any(), f"{what}: layers from {first} on were written"


def _expected_queue(N, count, group, lag):
    """build_item_table restated: groups of `group` cascades, the column pass (B items) of a group `lag` groups behind its
    row pass (A items): A(g0) .. A(g_lag-1), then A(g) B(g - lag) for every later group, then the last B groups."""
    one = _queue(_gow().load_library(), N, 1, 1, 1, 0)
    a_per = sum(1 for b, _, _ in one if not b)
    b_per = len(one) - a_per
    G = -(-count // group)
    out = []
    for ph in range(G + lag):
        if ph < G:
            out += [(0, s, bx) for s in range(ph * group, min(count, (ph + 1) * group)) for bx in range(a_per)]
        if ph >= lag:
            out += [(1, s, bx) for s in range((ph - lag) * group, min(count, (ph - lag + 1) * group)) for bx in range(b_per)]
    return out


def _generator_queue(N, count):
    """The single-update queue a generator created now builds for `count` cascades (group and lag 0: the generator's own
    choice, OCEAN_QUEUE_GROUP / OCEAN_QUEUE_LAG included)."""
    return _queue(_gow().load_library(), N, count, 0, 0, 0)


# ---------------------------------------------------------------------------------------------------------------------------
# 1. the bench workload
# ---------------------------------------------------------------------------------------------------------------------------
def test_bench_workload():
    """256^2 x 128 cascades of bench.synth_params, one generator, every cascade compared with the oracle after every step:
    three update_all (parameter edits before the third), a partial pass flushed by update(), update_frames(0.02, 5) (two
    fused launches of 2 x 128 records), then the profiled two-kernel pipeline and back."""
    N, C = 256, 128
    assert default_queue(N) == (8, 1)
    assert _generator_queue(N, C) == _expected_queue(N, C, 8, 1)          # 16 groups
    pg, pc = _params(C)
    g, o = _generator(N, C), _oracle(N, C)
    launches = _Launches(g)

    def edit(c, **kw):
        for k, v in kw.items():
            setattr(pg[c], k, v)
            setattr(pc[c], k, v)
        pc[c].should_generate_spectrum = True
        assert pg[c].should_generate_spectrum

    def times_equal():
        assert [p.time for p in pg] == [p.time for p in pc]

    for k, delta in enumerate((0.02, 0.02, 0.031)):
        if k == 2:
            for c, wind in ((3, 7.5), (64, 13.0), (127, 31.0)):            # spectra regenerated for a scattered subset
                edit(c, wind_speed=wind)
            edit(40, tile_length=(70.0, 70.0))                              # a key no cascade has: a new dispersion-table slot
            edit(41, tile_length=(88.0, 88.0))                              # joins the slot of cascades 0, 4, 8, ...
        g.update_all(delta, pg)
        o.update_all_batched(delta, pc)
        # one persistent launch; the first call adds one spectrum and one table launch, the third the spectra of cascades
        # 3, 40, 41, 64 and 127 and the table of cascade 40
        assert launches() == (1 if k == 1 else 3), k
        _check(g, o, f"update_all {k}")
        times_equal()

    # a partial pass: update() arms 128 cascades, _process() runs 127 and 126, the next update() flushes the 126 still pending
    edit(40, tile_length=(88.0, 88.0))                                      # back to a shared key: its own slot is released
    g.update(0.021, pg)
    o.update(0.021, pc)
    assert launches() == 0
    for c in (127, 126):
        g._process(0.0)
        o.process()
        assert launches() == 1
        assert g.pass_num_cascades_remaining == o.pass_num_cascades_remaining == c
    _check(g, o, "two _process calls")
    g.update(0.019, pg)
    o.update(0.019, pc)
    assert launches() == 1 + 1                                              # the 126 cascades, and the new spectrum of cascade 40
    _check(g, o, "update() flushing 126 pending cascades")
    times_equal()

    # fused frames: the flush of the pass the last update() armed, frame 0 as update_all, then 2 launches of 2 frames x 128 records
    g.update_frames(0.02, pg, 5)
    for _ in range(5):
        o.update_all_batched(0.02, pc)
    assert launches() == 1 + 1 + 2
    assert g.pass_num_cascades_remaining == 0
    _check(g, o, "update_frames(0.02, 5)")
    times_equal()

    # profiling on: the two-kernel pipeline in 11 chunks of 12 cascades (a launch pair each); off again: the persistent kernel
    # after the host re-uploaded the completion counters
    g.set_profiling(True)
    for k in range(2):
        g.update_all(0.02, pg)
        o.update_all_batched(0.02, pc)
        assert launches() == 2 * 11
        _, row_ms, col_ms, chunk = g.last_kernel_times()
        assert chunk == 12 and row_ms > 0 and col_ms > 0, (row_ms, col_ms, chunk)
        _check(g, o, f"profiled update_all {k}")
    g.set_profiling(False)
    g.update_all(0.02, pg)
    o.update_all_batched(0.02, pc)
    assert launches() == 1
    _check(g, o, "update_all after profiling")
    times_equal()
    assert g.maps_to_host(0, 1)[1][0][..., 3].max() > 0                    # foam was carried
    g.free()


# ---------------------------------------------------------------------------------------------------------------------------
# 2. queue shapes
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def queue_oracle():
    """The oracle's maps of N^2 x C after update_all(0.02), update_all(0.031) and three more update_all(0.02), and the cascade
    times at the end; computed once per (N, C) and kept for one size at a time (the shapes of a size are consecutive)."""
    cache = {}

    def get(N, C):
        if (N, C) not in cache:
            cache.clear()
            _, pc = _params(C)
            o = _oracle(N, C)
            snaps = []
            for delta in (0.02, 0.031):
                o.update_all_batched(delta, pc)
                snaps.append((o.displacement_map.copy(), o.normal_map.copy()))
            for _ in range(3):
                o.update_all_batched(0.02, pc)
            snaps.append((o.displacement_map.copy(), o.normal_map.copy()))
            cache[(N, C)] = snaps, [p.time for p in pc]
        return cache[(N, C)]

    yield get
    cache.clear()


@pytest.mark.parametrize("N,C,shape,group,lag", batch_queue_shapes())
def test_queue_shapes(N, C, shape, group, lag, queue_oracle, monkeypatch):
    """One fresh generator per queue shape (item tables are cached per generator and built at its first update, so the
    overrides are set before it): two update_all and one 3-frame update_frames, each equal to the same oracle maps."""
    if group is not None:
        monkeypatch.setenv("OCEAN_QUEUE_GROUP", str(group))
    if lag is not None:
        monkeypatch.setenv("OCEAN_QUEUE_LAG", str(lag))
    dg, dl = default_queue(N)
    eg, el = group or dg, lag or dl
    items = _generator_queue(N, C)
    assert items == _expected_queue(N, C, eg, el), (eg, el)
    first_b = next(i for i, it in enumerate(items) if it[0])
    rows_first = all(it[0] for it in items[first_b:])                     # no row pass handed out after a column pass
    assert rows_first == (-(-C // eg) <= el + 1), (shape, eg, el)
    snaps, times = queue_oracle(N, C)
    pg, _ = _params(C)
    g = _generator(N, C)
    launches = _Launches(g)
    for k, delta in enumerate((0.02, 0.031)):
        g.update_all(delta, pg)
        assert launches() == (3 if k == 0 else 1)                          # first: spectrum and table launches too
        _maps_equal(g, *snaps[k], f"{shape}: update_all {k}")
    g.update_frames(0.02, pg, 3)
    assert launches() == 1 + 1                                            # frame 0, then frames 1 and 2 in one fused launch
    _maps_equal(g, *snaps[2], f"{shape}: update_frames(0.02, 3)")
    assert [p.time for p in pg] == times
    g.free()


# ---------------------------------------------------------------------------------------------------------------------------
# 3. dispatch-table boundaries (128^2: the oracle costs little)
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layers,count", [(256, 256), (257, 257), (300, 300), (300, 257)])
def test_update_all_across_dispatch_tables(layers, count):
    """update_all of `count` cascades is one persistent launch per 256 of them; the launches share one queue counter and one
    set of completion counters, and launch k takes the records from 256 k on.  Layers beyond `count` stay untouched."""
    N = 128
    pg, pc = _params(count)
    g, o = _generator(N, layers), _oracle(N, count)
    per_update = -(-count // TABLE)
    launches = _Launches(g)
    for k, delta in enumerate((0.02, 0.031)):
        g.update_all(delta, pg)
        o.update_all_batched(delta, pc)
        assert launches() == per_update + (2 if k == 0 else 0)
        _check(g, o, f"update_all {k} of {count} on {layers} layers")
    if count < layers:
        _untouched(g, count, f"{count} of {layers} layers")
    g.free()


def test_partial_pass_across_dispatch_tables():
    """An update() / _process() pass over 300 cascades: three _process calls, a flush of the 297 still pending by update() (two
    launches of 256 and 41 records), then update_all, which flushes 300 more and runs 300 (two launches each)."""
    N, C = 128, 300
    pg, pc = _params(C)
    g, o = _generator(N, C), _oracle(N, C)
    g.update_all(0.02, pg)
    o.update_all_batched(0.02, pc)
    launches = _Launches(g)
    g.update(0.021, pg)
    o.update(0.021, pc)
    for _ in range(3):
        g._process(0.0)
        o.process()
        assert launches() == 1
    assert g.pass_num_cascades_remaining == o.pass_num_cascades_remaining == 297
    _check(g, o, "three _process calls")
    g.update(0.019, pg)
    o.update(0.019, pc)
    assert launches() == 2
    _check(g, o, "update() flushing 297 pending cascades")
    g.update_all(0.02, pg)
    o.update_all_batched(0.02, pc)
    assert launches() == 2 + 2
    _check(g, o, "update_all after a pass")
    assert [p.time for p in pg] == [p.time for p in pc]
    g.free()


@pytest.mark.parametrize("count,frames,fused_launches", [
    (64, 10, 4),     # 4 frames per launch: 4 x 64 = 256 records, the table full; frame 0 + 4 + 4 + 1
    (85, 8, 4),      # 3 frames per launch: 255 records, one short; frame 0 + 3 + 3 + 1
    (86, 6, 4),      # 2 frames per launch (172 records); frame 0 + 2 + 2 + 1
    (128, 6, 4),     # 2 frames per launch: 2 x 128 = 256 records, full
    (129, 3, 3),     # fewer than 2 frames fit: one update_all per frame
    (300, 3, 6),     # one update_all per frame, each split in two launches
])
def test_fused_frames_at_table_limits(count, frames, fused_launches):
    """update_frames packs 256 // count frames per launch; below 2 it runs frame by frame.  Maps and parameters (time, foam
    rates) equal those of a second generator run frame by frame, and both equal the oracle."""
    N = 128
    pa, pc = _params(count)
    pb, _ = _params(count)
    a, b, o = _generator(N, count), _generator(N, count), _oracle(N, count)
    for g, p in ((a, pa), (b, pb)):
        g.update_all(0.02, p)
    o.update_all_batched(0.02, pc)
    la, lb = _Launches(a), _Launches(b)
    a.update_frames(0.02, pa, frames)
    for _ in range(frames):
        b.update_all(0.02, pb)
        o.update_all_batched(0.02, pc)
    assert la() == fused_launches
    assert lb() == frames * -(-count // TABLE)
    for field in ("time", "foam_grow_rate", "foam_decay_rate", "should_generate_spectrum"):
        assert [getattr(p, field) for p in pa] == [getattr(p, field) for p in pb], field
    assert [p.time for p in pa] == [p.time for p in pc]
    da, na = a.maps_to_host()
    _maps_equal(b, da.view(np.uint16), na.view(np.uint16), f"update_frames(0.02, {frames}) against frame by frame")
    _check(a, o, f"update_frames(0.02, {frames})")
    a.free()
    b.free()


# ---------------------------------------------------------------------------------------------------------------------------
# 4. velocity beyond one launch pair
# ---------------------------------------------------------------------------------------------------------------------------
def test_velocity_across_launch_pairs():
    """128^2 x 300 with taps: the recompute of 300 stale layers is two launch pairs of 256 and 44 jobs; after a partial pass
    (cascades 299 down to 250 updated) only those 50 are stale and recomputed.  Every layer, half map and binary32 tap, equals
    the oracle's after each."""
    N, C = 128, 300
    pg, pc = _params(C)
    g, o = _generator(N, C, taps=True), _oracle(N, C, ov.OracleWaveGenerator)

    def check(what):
        v = g.velocity_to_host(0, C).view(np.uint16)
        for c in range(C):
            half, f32 = o.velocity(c)
            assert np.array_equal(v[c], half), f"{what}: velocity map of cascade {c}"
            assert np.array_equal(g.velocity_f32_to_host(c).view(np.uint32), f32.view(np.uint32)), f"{what}: binary32 velocity of cascade {c}"

    g.update_all(0.02, pg)
    o.update_all(0.02, pc)
    launches = _Launches(g)
    assert g.update_velocity() == C
    assert launches() == 2 * 2
    check("300 stale layers")
    g.update(0.025, pg)
    o.update(0.025, pc)
    for _ in range(50):
        g._process(0.0)
        o.process()
    launches()
    assert g.update_velocity() == 50                                        # cascades 250 .. 299, across index 256
    assert launches() == 2
    check("50 stale layers from 250 on")
    assert g.update_velocity() == 0 and launches() == 0
    g.free()
