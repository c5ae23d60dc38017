"""GPU parity of the spray-particle op (ocean_spray_particles; sea_spray_particle.gdshader start() and process()) against its
numpy specification oracle/spray_particles.py, on the generator's own maps: byte-identical states and instances after every
call of several seconds of emitter time, flat water with foam on part of a tile, the device entry point, truncation, launch
counts, validation, a non-finite emitter, side effects and device memory."""
import ctypes as C

import numpy as np
import pytest

from conftest import demo_params
from oracle import pyoracle as po
from oracle import spray_particles as sp
from test_gpu_sampling import _same_or_both_nan
from test_gpu_spray import _generator
from test_gpu_surface import _crc

pytestmark = pytest.mark.gpu

INVALID = 1   # OCEAN_ERR_INVALID_ARGUMENT
FLOATS = ("transform", "custom", "userdata1", "userdata2", "userdata3")


@pytest.fixture(autouse=True)
def _det_math():
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)


def _same_states(a, b):
    """bit-identical states, except that a NaN only has to meet a NaN (see _same_or_both_nan)"""
    return len(a) == len(b) and all(_same_or_both_nan(a[f], b[f]) for f in FLOATS) and \
        np.array_equal(a["number"], b["number"]) and np.array_equal(a["flags"], b["flags"])


def _rotated_emitter(gow):
    e = gow.WaveGenerator.default_spray_emitter()
    c, s = np.cos(0.8), np.sin(0.8)
    R = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]]) @ np.array([[1, 0, 0], [0, np.cos(0.2), -np.sin(0.2)], [0, np.sin(0.2), np.cos(0.2)]])
    e["emission_transform"] = np.concatenate([R * [9.0, 2.5, 21.0], [[3.5], [0.25], [-12.0]]], axis=1).astype(np.float32).reshape(12)
    e["amount"], e["num_particles"] = 20000, 16384
    e["random_seed"] = 0x9E3779B9
    e["particle_scale"] = (0.6, 1.4, 0.6)
    return e


def _times(seed, seconds=8.0, hz=30.0, long_delta=7.0):
    """call boundaries: irregular 30 Hz deltas, one of them longer than the emitter lifetime"""
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.4, 1.6, int(seconds * hz)) / hz
    d[len(d) // 3] = long_delta
    return np.concatenate([[0.0], np.cumsum(d)])


@pytest.mark.parametrize("N,C", [(128, 3), (256, 4), (1024, 2)])
@pytest.mark.parametrize("kind", ["default", "rotated"])
def test_spray_particles_bit_exact(N, C, kind):
    gow, g, p = _generator(N, C, 25, whitecap=0.9, foam_amount=10.0)
    scales = gow.WaveGenerator.map_scales(p)
    e = gow.WaveGenerator.default_spray_emitter() if kind == "default" else _rotated_emitter(gow)
    amount = int(e["amount"])
    mine = ref = np.zeros(amount, sp.PARTICLE)
    maps = g.maps_to_host(0, C)
    t = _times(N + C)
    counts = []
    for j, (t0, t1) in enumerate(zip(t[:-1], t[1:])):
        if j % 8 == 7:                                              # the maps move on between calls
            g.update_all(1.0 / 50.0, p)
            maps = g.maps_to_host(0, C)
        mine, inst, count = g.spray_particles(e, mine, t0, t1, scales)
        with np.errstate(all="ignore"):
            ref, rinst, rcount = sp.frame(ref, e, t0, t1, maps[0], maps[1], scales)
        assert count == rcount == len(inst), (j, count, rcount)
        assert _same_states(mine, ref), j
        assert _same_or_both_nan(inst, rinst), j
        counts.append(count)
    assert max(counts) > 0 and all(c < amount for c in counts)
    assert (mine["flags"] & sp.EMITTED).all()
    g.free()


def _flat(N=256, C=2):
    """zero amplitudes: flat, still water; foam 1 on the left half of cascade 0's tile, 0 elsewhere"""
    import godotoceanwaves_b200 as gow
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(C)
    p = [demo_params(gow.WaveCascadeParameters, c) for c in range(C)]
    g.update_all(0.02, p)
    for c in range(C):
        g.set_spectrum_amplitudes(c, np.zeros((N, N), np.complex64))
    g.update_all(0.02, p)
    foam = np.zeros((N, N), np.float16)
    foam[:, : N // 2] = 1.0
    g.set_foam_state(0, foam)
    for c in range(1, C):
        g.set_foam_state(c, np.zeros((N, N), np.float16))
    scales = gow.WaveGenerator.map_scales(p)
    scales[0, :2] = 1.0 / 400.0                                     # the emitter box (+-75 m) spans 3/8 of cascade 0's tile
    return gow, g, scales


def test_flat_water_with_foam_on_part_of_the_tile():
    gow, g, scales = _flat()
    e = gow.WaveGenerator.default_spray_emitter()
    d16, n16 = g.maps_to_host(0, 2)
    assert not d16.any()
    st = ref = np.zeros(int(e["amount"]), sp.PARTICLE)
    t = _times(3, seconds=4.0, long_delta=1.0 / 30)
    seen = 0
    for t0, t1 in zip(t[:-1], t[1:]):
        st, inst, count = g.spray_particles(e, st, t0, t1, scales)
        with np.errstate(all="ignore"):
            ref, rinst, _ = sp.frame(ref, e, t0, t1, d16, n16, scales)
        assert _same_states(st, ref) and _same_or_both_nan(inst, rinst)
        live = ((st["flags"] & sp.ACTIVE) != 0) & (st["userdata3"][:, 3] != 0)
        x = st["userdata1"][live, 0]
        # foam 1 on texels [0, N/2) of the tile: the filtered foam passes 0.9 only within 0.1 texel of texel centres 0.5 ... 127.5
        u = x.astype(np.float64) * 256 / 400.0
        assert ((np.mod(u, 256) >= 0.39) & (np.mod(u, 256) <= 127.61)).all()
        tt = (np.float32(t1) - st["userdata1"][live, 3]) / st["userdata2"][live, 3]
        a = 2.5 * tt.astype(np.float64) - 0.45
        h64 = -5.0 * a * a + 0.5
        assert (np.abs(st["transform"][live, 7] - h64) <= 8 * np.spacing(np.maximum(5 * a * a, 0.5).astype(np.float32))).all()
        seen += count
    started = (st["userdata3"][:, 3] == 1.0)
    assert seen > 0 and started.sum() > ((st["flags"][started] & sp.ACTIVE) != 0).sum() > 0
    g.free()


def _foamy(N=256, C=4):
    gow, g, p = _generator(N, C, 25, whitecap=0.9, foam_amount=10.0)
    return gow, g, p, gow.WaveGenerator.map_scales(p)


def _warm(g, e, scales, until=5.0):
    st = None
    t = 0.0
    while t < until:
        st, _, _ = g.spray_particles(e, st, t, t + 1.0 / 30, scales)
        t += 1.0 / 30
    return st, t


def test_device_entry_point_equals_host_and_truncation():
    import torch
    from godotoceanwaves_b200.native import check, load_library
    gow, g, p, scales = _foamy()
    e = _rotated_emitter(gow)
    st, t = _warm(g, e, scales)
    new, inst, count = g.spray_particles(e, st, t, t + 0.04, scales)
    assert 0 < count < len(st)
    dev = torch.device("cuda", g.device)
    st_d = torch.from_numpy(st.view(np.uint8).copy()).to(dev)
    inst_d = torch.full((len(st) * 16,), -1.0, dtype=torch.float32, device=dev)
    count_d = torch.full((1,), -1, dtype=torch.int32, device=dev)
    ec = np.array(e, g.SPRAY_EMITTER)
    torch.cuda.synchronize()
    check(load_library().ocean_spray_particles_device(g.context, ec.ctypes.data, t, t + 0.04, 4, scales.ctypes.data, st_d.data_ptr(), len(st),
                                                      inst_d.data_ptr(), count_d.data_ptr()))
    g.synchronize()
    assert int(count_d.cpu()[0]) == count
    assert st_d.cpu().numpy().tobytes() == new.tobytes()
    assert inst_d.cpu().numpy()[:16 * count].tobytes() == inst.tobytes()
    assert (inst_d.cpu().numpy()[16 * count:] == -1.0).all()
    # max_instances drops instances, not the count
    for cap in (0, 7):
        few_st, few, c2 = g.spray_particles(e, st, t, t + 0.04, scales, max_instances=cap)
        assert c2 == count and few.tobytes() == inst[:cap].tobytes() and few_st.tobytes() == new.tobytes()
    g.free()


def _lib():
    from godotoceanwaves_b200.native import load_library
    return load_library()


def test_launch_counts_and_arguments():
    import torch
    gow, g, p, scales = _foamy(128, 2)
    e = gow.WaveGenerator.default_spray_emitter()
    e["amount"] = 5000
    st, t = _warm(g, e, scales, 1.0)
    before = g.info().kernel_launches
    g.spray_particles(e, st, t, t + 0.03, scales)
    assert g.info().kernel_launches - before == 3
    zero = e.copy()
    zero["amount"] = 0
    before = g.info().kernel_launches
    s0, i0, c0 = g.spray_particles(zero, None, t, t + 0.03, scales)
    assert g.info().kernel_launches == before and c0 == 0 and len(s0) == 0
    lib = _lib()
    dev = torch.device("cuda", g.device)
    st_d = torch.from_numpy(st.view(np.uint8).copy()).to(dev)
    inst = np.zeros((5000, 16), np.float32)
    inst_d = torch.zeros(5000 * 16, dtype=torch.float32, device=dev)
    count, count_d = C.c_int(-5), torch.zeros(1, dtype=torch.int32, device=dev)
    bad = []
    for field, value in (("amount", -1), ("num_particles", 0), ("lifetime", 0.0), ("lifetime", np.inf), ("lifetime", np.nan),
                         ("emitter_lifetime", 0.0), ("emitter_lifetime", np.inf), ("emitter_lifetime", -6.0),
                         ("lifetime_randomness", -0.01), ("lifetime_randomness", 1.01), ("lifetime_randomness", np.nan)):
        b = e.copy()
        b[field] = value
        bad.append((b, t, t + 0.03, 2, scales, 5000))
    bad += [(e, -1.0, 0.5, 2, scales, 5000), (e, 2.0, 1.0, 2, scales, 5000), (e, 0.0, np.inf, 2, scales, 5000),
            (e, np.nan, 1.0, 2, scales, 5000), (e, 0.0, 2.0 ** 33, 2, scales, 5000), (e, t, t + 0.03, 0, scales, 5000),
            (e, t, t + 0.03, 3, scales, 5000), (e, t, t + 0.03, 2, None, 5000), (e, t, t + 0.03, 2, scales, -1)]
    tiny = e.copy()
    tiny["emitter_lifetime"] = 1e-9
    bad.append((tiny, 0.0, 10.0, 2, scales, 5000))                  # t1 / emitter_lifetime >= 2^32
    for host in (True, False):
        for b, t0, t1, nc, sc, cap in bad:
            ec = np.array(b, g.SPRAY_EMITTER)
            s_host = st.copy()
            before = g.info().kernel_launches
            if host:
                rc = lib.ocean_spray_particles(g.context, ec.ctypes.data, t0, t1, nc, None if sc is None else sc.ctypes.data, s_host.ctypes.data,
                                               cap, inst.ctypes.data, C.byref(count))
            else:
                rc = lib.ocean_spray_particles_device(g.context, ec.ctypes.data, t0, t1, nc, None if sc is None else sc.ctypes.data,
                                                      st_d.data_ptr(), cap, inst_d.data_ptr(), count_d.data_ptr())
            assert rc == INVALID, (host, b, t0, t1, nc, cap)
            assert g.info().kernel_launches == before
            assert s_host.tobytes() == st.tobytes()
        # NULL where a count needs the buffer
        ec = np.array(e, g.SPRAY_EMITTER)
        fn = lib.ocean_spray_particles if host else lib.ocean_spray_particles_device
        st_host = st.copy()
        sp_ = st_host.ctypes.data if host else st_d.data_ptr()
        ip = inst.ctypes.data if host else inst_d.data_ptr()
        cp = C.byref(count) if host else count_d.data_ptr()
        before = g.info().kernel_launches
        assert fn(g.context, None, t, t + 0.03, 2, scales.ctypes.data, sp_, 5000, ip, cp) == INVALID
        assert fn(g.context, ec.ctypes.data, t, t + 0.03, 2, scales.ctypes.data, None, 5000, ip, cp) == INVALID
        assert fn(g.context, ec.ctypes.data, t, t + 0.03, 2, scales.ctypes.data, sp_, 5000, None, cp) == INVALID
        assert fn(g.context, ec.ctypes.data, t, t + 0.03, 2, scales.ctypes.data, sp_, 5000, ip, None) == INVALID
        assert g.info().kernel_launches == before
        # ... and NULL is fine where no count needs it
        assert fn(g.context, ec.ctypes.data, t, t + 0.03, 2, scales.ctypes.data, sp_, 0, None, cp) == 0
        z = np.array(zero, g.SPRAY_EMITTER)
        assert fn(g.context, z.ctypes.data, t, t + 0.03, 2, scales.ctypes.data, None, 0, None, cp) == 0
        assert g.info().kernel_launches == before + 3
    g.synchronize()
    assert int(count_d.cpu()[0]) == 0 and count.value == 0
    g.free()


def test_non_finite_emitter():
    gow, g, p, scales = _foamy(128, 2)
    d16, n16 = g.maps_to_host(0, 2)
    e = gow.WaveGenerator.default_spray_emitter()
    e["amount"] = 3000
    E = e["emission_transform"].copy()
    E[[0, 6, 11]] = [np.nan, np.inf, -np.inf]
    e["emission_transform"] = E
    st = ref = np.zeros(3000, sp.PARTICLE)
    for t0, t1 in zip(_times(9, 7.0)[:-1], _times(9, 7.0)[1:]):
        st, inst, count = g.spray_particles(e, st, t0, t1, scales)
        with np.errstate(all="ignore"):
            ref, _, rcount = sp.frame(ref, e, t0, t1, d16, n16, scales)
        assert _same_states(st, ref) and count == rcount == 0
    assert (st["flags"] & sp.EMITTED).all()
    g.free()


def test_spray_particles_leave_the_generator_alone():
    """Maps, foam, spectrum and velocity staleness are unchanged by the op, and the next update is bit-identical to that
    of a generator that never ran it."""
    import godotoceanwaves_b200 as gow
    N, Cn = 128, 3
    a = gow.WaveGenerator(); a.map_size = N; a.init_gpu(Cn)
    b = gow.WaveGenerator(); b.map_size = N; b.init_gpu(Cn)
    pa = [demo_params(gow.WaveCascadeParameters, c, whitecap=0.9, foam_amount=10.0) for c in range(Cn)]
    pb = [demo_params(gow.WaveCascadeParameters, c, whitecap=0.9, foam_amount=10.0) for c in range(Cn)]
    scales = gow.WaveGenerator.map_scales(pa)
    e = gow.WaveGenerator.default_spray_emitter()
    st, t = None, 0.0
    a.update_velocity()
    for k in range(4):
        a.update_all(1.0 / 50.0, pa)
        b.update_all(1.0 / 50.0, pb)
        a.update_velocity()
        for _ in range(3):
            st, _, _ = a.spray_particles(e, st, t, t + 0.5, scales)
            t += 0.5
        assert a.update_velocity() == 0
        da, na = a.maps_to_host(0, Cn)
        db, nb = b.maps_to_host(0, Cn)
        assert (_crc(da), _crc(na)) == (_crc(db), _crc(nb))
        for c in range(Cn):
            assert a.get_foam_state(c).tobytes() == b.get_foam_state(c).tobytes()
            assert a.spectrum_to_host(c).tobytes() == b.spectrum_to_host(c).tobytes()
    a.free()
    b.free()


def test_device_bytes_small_then_large_equals_large():
    gow, g1, p, scales = _foamy(128, 2)
    _, g2, _, _ = _foamy(128, 2)
    small, large = gow.WaveGenerator.default_spray_emitter(), gow.WaveGenerator.default_spray_emitter()
    small["amount"], large["amount"] = 300, 70000
    g1.spray_particles(small, None, 0.0, 1.0, scales, max_instances=10)
    g1.spray_particles(large, None, 0.0, 1.0, scales)
    g2.spray_particles(large, None, 0.0, 1.0, scales)
    assert g1.info().device_bytes == g2.info().device_bytes
    g1.free()
    g2.free()
