"""GPU parity of the body-forces op (ocean_body_forces: buoyancy plus quadratic drag against the water velocity, from one
surface query) against its numpy specification oracle/drag.py on the generator's own maps and velocity maps: bit-identical
32-byte drag records, 48-byte buoyancy records and 40-byte surface records; launches, staleness, isolation, arguments."""
import numpy as np
import pytest

from conftest import demo_params
from oracle import buoyancy as bu
from oracle import drag as dr
from test_gpu_buoyancy import _scene
from test_gpu_sampling import _gen, _same_or_both_nan
from test_gpu_surface import _crc, _records_match, _scales
from test_oracle_buoyancy import _bodies, _box, _transform

pytestmark = pytest.mark.gpu

RHO = 1025.0
INVALID = 1   # OCEAN_ERR_INVALID_ARGUMENT


def _motion(seed, bodies, hull):
    """Random body velocities (|linear| components up to 3 m/s, angular up to 1 rad/s) and drag areas (0.01 to 0.6 m^2)."""
    rng = np.random.default_rng(seed)
    vel = np.zeros(len(bodies), dr.VELOCITY)
    vel["linear"] = rng.uniform(-3, 3, (len(bodies), 3))
    vel["angular"] = rng.uniform(-1, 1, (len(bodies), 3))
    return vel, rng.uniform(0.01, 0.6, len(hull)).astype(np.float32)


@pytest.mark.parametrize("N,C", [(128, 3), (256, 4), (512, 2), (1024, 2)])
def test_body_forces_bit_exact(N, C):
    gow, g, params = _gen(N, C)
    d16, n16 = g.maps_to_host(0, C)
    sizes = np.random.default_rng(N + 1).integers(0, 100, 300)
    bodies, hull = _scene(150 + N, sizes)
    vel, cda = _motion(N, bodies, hull)
    restarted = False
    for factor in (1.0, 2.0):                                   # twice the displacement: many more restarts
        scales = _scales(gow, params, C)
        scales[:, 2] *= np.float32(factor)
        for maxit in (8, 0):
            hydro, drag, smp = g.body_forces(bodies, vel, hull, cda, scales, RHO, 1e-3, maxit, return_samples=True)
            v16 = g.velocity_to_host(0, C)
            ref_h, ref_d, ref_s = dr.body_forces(d16, n16, v16, bodies, vel, hull, cda, scales, RHO, 1e-3, maxit, return_samples=True)
            assert drag.tobytes() == ref_d.tobytes()
            assert hydro.tobytes() == ref_h.tobytes()
            assert smp.tobytes() == ref_s.tobytes()
            assert hydro.tobytes() == g.buoyancy(bodies, hull, scales, RHO, 1e-3, maxit).tobytes()
            restarted |= bool(np.any(smp["iterations"] > 8))
    assert restarted                                            # the restart kernel ran
    assert np.count_nonzero(drag["wetted_drag_area"]) > 100 and np.all(np.isfinite(drag["force"]))
    assert not drag[bodies["num_points"] == 0].tobytes().strip(b"\0")
    g.free()


def test_body_forces_mixed_scene():
    """3000 bodies: shared hulls, empty bodies, 1 to 70 000 points, a NaN in one rotation, an infinite translation and a NaN
    linear velocity.  NaN appears exactly where the specification has it; every other body is bit-identical."""
    gow, g, params = _gen(256, 4)
    d16, n16 = g.maps_to_host(0, 4)
    scales = _scales(gow, params, 4)
    rng = np.random.default_rng(161)
    sizes = rng.integers(1, 40, 3000)
    sizes[0], sizes[2], sizes[3], sizes[4], sizes[6] = 5, 1, 33, 70000, 37   # body 0 lends its hull to 1, 5, 9, ...
    sizes[10::97] = 0
    bodies, hull = _scene(162, sizes, share_every=4)
    bodies["transform"][7, 1] = np.nan
    bodies["transform"][8, 3] = np.inf
    bodies["transform"][6, 7] = -3.0                            # well under water
    vel, cda = _motion(163, bodies, hull)
    vel["linear"][6, 0] = np.nan
    hydro, drag, smp = g.body_forces(bodies, vel, hull, cda, scales, RHO, 1e-3, 8, return_samples=True)
    v16 = g.velocity_to_host(0, 4)
    with np.errstate(all="ignore"):
        ref_h, ref_d, ref_s = dr.body_forces(d16, n16, v16, bodies, vel, hull, cda, scales, RHO, 1e-3, 8, return_samples=True)
    bad = np.zeros(len(bodies), bool)
    bad[[6, 7, 8]] = True
    assert drag[~bad].tobytes() == ref_d[~bad].tobytes()
    assert hydro[~bad].tobytes() == ref_h[~bad].tobytes()
    for f in dr.RESULT.names:
        assert _same_or_both_nan(drag[bad][f], ref_d[bad][f]), f
    for f in ("force", "torque", "submerged_volume", "center_offset", "max_residual"):
        assert _same_or_both_nan(hydro[bad][f], ref_h[bad][f]), f
    assert np.isnan(drag["force"][6]).all() and np.isnan(drag["torque"][6]).all() and drag["wetted_drag_area"][6] > 0
    assert np.isfinite(drag[~bad]["force"]).all() and np.isfinite(drag[~bad]["torque"]).all()
    assert np.isfinite(drag["max_relative_speed"]).all()
    assert np.count_nonzero(drag["wetted_drag_area"]) > 1000
    empty = bodies["num_points"] == 0
    assert empty.sum() > 10 and not drag[empty].tobytes().strip(b"\0")
    assert _records_match(smp, ref_s)
    g.free()


def test_moving_with_the_water_feels_no_drag():
    """A one-point body whose velocity is ocean_sample_velocity at its record's source point (and no spin) gets a force and
    a torque of exactly 0."""
    gow, g, params = _gen(256, 4)
    scales = _scales(gow, params, 4)
    rng = np.random.default_rng(171)
    n = 2000
    hull = np.zeros(1, bu.POINT)
    hull["position"] = (0.3, -0.25, -0.2)
    hull["volume"], hull["half_height"] = 0.2, 0.5
    t = np.stack([rng.uniform(-150, 150, n), rng.uniform(-1.5, 0.5, n), rng.uniform(-150, 150, n)], 1)
    bodies = _bodies([_transform(t=ti) for ti in t], [(0, 1)] * n)
    vel = np.zeros(n, dr.VELOCITY)
    cda = np.full(1, 0.5, np.float32)
    _, _, smp = g.body_forces(bodies, vel, hull, cda, scales, RHO, 1e-3, 8, return_samples=True)
    vel["linear"] = g.sample_velocity(np.stack([smp["source_x"], smp["source_z"]], 1), scales)
    assert np.abs(vel["linear"]).max() > 0.1
    _, drag, smp2 = g.body_forces(bodies, vel, hull, cda, scales, RHO, 1e-3, 8, return_samples=True)
    assert smp2.tobytes() == smp.tobytes()
    wet = drag["wetted_drag_area"] > 0
    assert 0.2 < wet.mean() < 1.0
    assert not drag["force"].any() and not drag["torque"].any() and not drag["max_relative_speed"].any()
    g.free()


def test_zero_spectrum_translating_box_is_the_closed_form():
    """Maps made on the GPU from a zero spectrum are flat and still: a submerged voxel box moving at v = (3, 0, 4) feels
    exactly -1/2 rho (sum C_d A) |v| v, and the torque its lever arms give."""
    import godotoceanwaves_b200 as gow
    N, Cn = 256, 2
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(Cn)
    params = [demo_params(gow.WaveCascadeParameters, c) for c in range(Cn)]
    g.update_all(0.02, params)                                  # clears the dirty flags
    for c in range(Cn):
        g.set_spectrum_amplitudes(c, np.zeros((N, N), np.complex64))
    g.update_all(0.02, params)
    d16, _ = g.maps_to_host(0, Cn)
    assert not d16.astype(np.float32).any()
    hull = _box(4, 4, 4)
    c = np.array([1.0, -0.5, 2.0], np.float32)
    hull["position"] += c
    cda = np.full(len(hull), 0.25, np.float32)
    v = np.array([3.0, 0.0, 4.0])
    vel = np.zeros(2, dr.VELOCITY)
    vel["linear"] = v
    bodies = _bodies([_transform(t=(37.0, -5.0, -91.5)), _transform(t=(-12.0, 40.0, 3.0))], [(0, len(hull))] * 2)
    hydro, drag = g.body_forces(bodies, vel, hull, cda, gow.WaveGenerator.map_scales(params), RHO, 1e-3, 8)
    assert not g.velocity_to_host(0, Cn).astype(np.float32).any()
    half_rho = float(np.float32(0.5) * np.float32(RHO))
    assert drag["force"][0].tolist() == (-half_rho * 16.0 * 5.0 * v).tolist()
    assert drag["torque"][0].tolist() == (half_rho * 64.0 * np.cross(c.astype(np.float64), -0.25 * 5.0 * v)).tolist()
    assert drag["wetted_drag_area"][0] == 16.0 and drag["max_relative_speed"][0] == 5.0
    assert drag[1].tobytes() == bytes(32)                       # in the air
    assert hydro["submerged_volume"].tolist() == [8.0, 0.0]
    g.free()


def test_stale_velocity_is_refreshed_and_launch_counts():
    """After ocean_process one cascade's velocity layer is stale: the call refreshes it (nothing is stale afterwards) and
    matches the specification on the refreshed maps.  A call with no stale layer launches 6 kernels (4 at 0 steps)."""
    gow, g, params = _gen(256, 3)
    scales = _scales(gow, params, 3)
    bodies, hull = _scene(181, np.random.default_rng(180).integers(0, 60, 200))
    vel, cda = _motion(182, bodies, hull)
    g.body_forces(bodies, vel, hull, cda, scales)
    for step in range(2):
        g.update(0.03, params)
        g._process()
        before = g.info().kernel_launches
        hydro, drag = g.body_forces(bodies, vel, hull, cda, scales)
        assert g.info().kernel_launches - before > 6             # the refresh ran in the call ...
        assert g.update_velocity() == 0                          # ... and left nothing stale
        d16, n16 = g.maps_to_host(0, 3)
        ref_h, ref_d = dr.body_forces(d16, n16, g.velocity_to_host(0, 3), bodies, vel, hull, cda, scales)
        assert drag.tobytes() == ref_d.tobytes() and hydro.tobytes() == ref_h.tobytes()
    for maxit, launches in ((8, 6), (0, 4)):
        before = g.info().kernel_launches
        g.body_forces(bodies, vel, hull, cda, scales, RHO, 1e-3, maxit)
        assert g.info().kernel_launches - before == launches
    g.free()


def test_body_forces_device_equals_host():
    import torch
    from godotoceanwaves_b200.native import check, load_library
    gow, g, params = _gen(256, 4)
    scales = _scales(gow, params, 4)
    bodies, hull = _scene(191, np.random.default_rng(190).integers(0, 120, 800))
    vel, cda = _motion(192, bodies, hull)
    hydro, drag, smp = g.body_forces(bodies, vel, hull, cda, scales, RHO, 1e-3, 8, return_samples=True)
    dev = torch.device("cuda", g.device)
    hull_d = torch.from_numpy(hull.view(np.uint8).copy()).to(dev)
    cda_d = torch.from_numpy(cda).to(dev)
    hyd_d = torch.zeros(len(bodies) * 12, dtype=torch.int32, device=dev)
    drag_d = torch.zeros(len(bodies) * 8, dtype=torch.int32, device=dev)
    smp_d = torch.zeros(len(smp) * 10, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    lib = load_library()
    for samples in (smp_d, None):
        hyd_d.zero_()
        drag_d.zero_()
        check(lib.ocean_body_forces_device(g.context, len(bodies), bodies.ctypes.data, vel.ctypes.data, len(hull), hull_d.data_ptr(),
                                           cda_d.data_ptr(), 4, scales.ctypes.data, RHO, 1e-3, 8, hyd_d.data_ptr(), drag_d.data_ptr(),
                                           None if samples is None else samples.data_ptr()))
        g.synchronize()
        assert hyd_d.cpu().numpy().tobytes() == hydro.tobytes()
        assert drag_d.cpu().numpy().tobytes() == drag.tobytes()
    assert smp_d.cpu().numpy().tobytes() == smp.tobytes()
    g.free()


def test_body_forces_leave_the_generator_alone():
    """Maps, foam, spectrum and the next update's maps are byte-identical with and without body-forces calls."""
    import godotoceanwaves_b200 as gow
    N, Cn = 128, 3
    a = gow.WaveGenerator(); a.map_size = N; a.init_gpu(Cn)
    b = gow.WaveGenerator(); b.map_size = N; b.init_gpu(Cn)
    pa = [demo_params(gow.WaveCascadeParameters, c) for c in range(Cn)]
    pb = [demo_params(gow.WaveCascadeParameters, c) for c in range(Cn)]
    scales = gow.WaveGenerator.map_scales(pa)
    small, big = _scene(201, [3, 4]), _scene(202, np.full(700, 100))
    for k in range(3):
        a.update_all(1.0 / 50.0, pa)
        b.update_all(1.0 / 50.0, pb)
        for bodies, hull in (small, big) if k else (small,):     # staging sized by a small call first, then grown
            vel, cda = _motion(203 + k, bodies, hull)
            a.body_forces(bodies, vel, hull, cda, scales, return_samples=True)
        da, na = a.maps_to_host(0, Cn)
        db, nb = b.maps_to_host(0, Cn)
        assert (_crc(da), _crc(na)) == (_crc(db), _crc(nb))
        for c in range(Cn):
            assert a.get_foam_state(c).tobytes() == b.get_foam_state(c).tobytes()
            assert a.spectrum_to_host(c).tobytes() == b.spectrum_to_host(c).tobytes()
    a.free(); b.free()


def test_body_forces_arguments():
    """Every invalid argument returns OCEAN_ERR_INVALID_ARGUMENT and launches nothing (not even a velocity refresh), through
    both entry points."""
    from godotoceanwaves_b200.native import load_library
    gow, g, params = _gen(128, 2, frames=1)                     # the velocity layers are stale: a refresh would launch
    lib = load_library()
    scales = gow.WaveGenerator.map_scales(params)
    bodies, hull = _scene(211, [4, 0, 6])
    bodies["num_points"][1] = 0                                 # (_scene made it share body 0's hull)
    vel, cda = _motion(212, bodies, hull)
    hyd = np.zeros(len(bodies), bu.RESULT)
    drag = np.zeros(len(bodies), dr.RESULT)
    ok = dict(nb=len(bodies), b=bodies, v=vel.ctypes.data, np_=len(hull), p=hull.ctypes.data, a=cda.ctypes.data, nc=2, sc=scales.ctypes.data,
              rho=RHO, tol=1e-3, it=8, h=hyd.ctypes.data, d=drag.ctypes.data, s=None)

    def body_edit(**kw):
        b = bodies.copy()
        for k, v in kw.items():
            b[k][0] = v
        return b

    big = bodies[:2].copy()
    big["first_point"], big["num_points"] = 0, 2 ** 31 - 1        # 2^32 - 2 world points
    bad = [dict(nb=-1), dict(np_=-1), dict(rho=0.0), dict(rho=-1025.0), dict(rho=float("nan")), dict(rho=float("inf")),
           dict(tol=0.0), dict(tol=float("nan")), dict(it=-1), dict(it=65),
           dict(b=body_edit(num_points=-1)), dict(b=body_edit(first_point=-1)), dict(b=body_edit(first_point=7)),
           dict(b=body_edit(first_point=2 ** 31 - 2)), dict(nb=2, b=big, np_=2 ** 31 - 1),
           dict(b=None), dict(v=None), dict(p=None), dict(a=None), dict(h=None), dict(d=None), dict(nc=0), dict(nc=3), dict(sc=None)]
    for fn in (lib.ocean_body_forces, lib.ocean_body_forces_device):
        for kw in bad:
            a = dict(ok)
            a.update(kw)
            before = g.info().kernel_launches
            rc = fn(g.context, a["nb"], None if a["b"] is None else a["b"].ctypes.data, a["v"], a["np_"], a["p"], a["a"], a["nc"], a["sc"],
                    a["rho"], a["tol"], a["it"], a["h"], a["d"], a["s"])
            assert rc == INVALID, kw
            assert g.info().kernel_launches == before, kw
    # NULL is fine where no count needs the buffer
    empty = bodies[[1]]
    assert lib.ocean_body_forces(g.context, 1, empty.ctypes.data, vel.ctypes.data, 0, None, None, 2, scales.ctypes.data, RHO, 1e-3, 8,
                                 hyd.ctypes.data, drag.ctypes.data, None) == 0
    assert hyd[:1].tobytes() == bytes(48) and drag[:1].tobytes() == bytes(32)
    assert lib.ocean_body_forces(g.context, 0, None, None, 0, None, None, 0, None, RHO, 1e-3, 8, None, None, None) == 0
    h0, d0 = g.body_forces(bodies[:0], vel[:0], hull, cda, scales)
    assert len(h0) == 0 and len(d0) == 0
    h, d, s = g.body_forces(bodies, vel, hull, cda, scales, return_samples=True)
    assert len(h) == len(d) == 3 and len(s) == 10 and d[1].tobytes() == bytes(32)
    with pytest.raises(ValueError):
        g.body_forces(bodies, vel[:2], hull, cda, scales)
    g.free()
