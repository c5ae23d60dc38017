"""GPU parity of the buoyancy op (ocean_buoyancy: hull points on the displaced surface, summed per body) against its numpy
specification oracle/buoyancy.py on the generator's own maps: bit-identical 48-byte results and 40-byte surface records."""
import numpy as np
import pytest

from conftest import demo_params
from oracle import buoyancy as bu
from test_gpu_sampling import _gen, _same_or_both_nan
from test_gpu_surface import _crc, _records_match, _scales
from test_oracle_buoyancy import _bodies, _box, _random_rotations, _transform

pytestmark = pytest.mark.gpu

RHO = 1025.0


def _scene(seed, sizes, share_every=3):
    """Bodies of the given sizes, each with its own random hull (points in [-3, 3]^3 m, random volumes, every seventh half
    height 0), random rotations and positions in [-200, 200] m around the surface; every `share_every`-th body instead
    shares the hull of the first non-empty body."""
    rng = np.random.default_rng(seed)
    sizes = np.asarray(sizes, np.int64)
    hull = np.zeros(int(sizes.sum()), bu.POINT)
    hull["position"] = rng.uniform(-3, 3, (len(hull), 3))
    hull["volume"] = rng.uniform(0.01, 0.5, len(hull))
    hull["half_height"] = rng.uniform(0.05, 0.6, len(hull))
    hull["half_height"][::7] = 0.0
    R = _random_rotations(rng, len(sizes))
    t = np.stack([rng.uniform(-200, 200, len(sizes)), rng.uniform(-1, 1, len(sizes)), rng.uniform(-200, 200, len(sizes))], 1)
    starts = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    bodies = _bodies([_transform(R[i], t[i]) for i in range(len(sizes))], list(zip(starts, sizes)))
    donor = int(np.nonzero(sizes)[0][0])
    shared = np.arange(donor + 1, len(sizes), share_every)
    bodies["first_point"][shared] = bodies["first_point"][donor]
    bodies["num_points"][shared] = bodies["num_points"][donor]
    return bodies, hull


def _world_xz(bodies, hull):
    _, _, _, w = bu.world_points(bodies, hull)
    return np.stack([w[:, 0], w[:, 2]], 1)


@pytest.mark.parametrize("N,C", [(128, 3), (256, 4), (512, 2), (1024, 2)])
def test_buoyancy_bit_exact(N, C):
    gow, g, params = _gen(N, C)
    d16, n16 = g.maps_to_host(0, C)
    sizes = np.random.default_rng(N).integers(0, 100, 300)
    bodies, hull = _scene(50 + N, sizes)
    restarted = False
    for factor in (1.0, 2.0):                                   # twice the displacement: many more restarts
        scales = _scales(gow, params, C)
        scales[:, 2] *= np.float32(factor)
        for maxit in (8, 0):
            out, smp = g.buoyancy(bodies, hull, scales, RHO, 1e-3, maxit, return_samples=True)
            ref, rsmp = bu.buoyancy(d16, n16, bodies, hull, scales, RHO, 1e-3, maxit, return_samples=True)
            assert out.tobytes() == ref.tobytes()
            assert smp.tobytes() == rsmp.tobytes()
            restarted |= bool(np.any(smp["iterations"] > 8))
    assert restarted                                            # the restart kernel ran
    assert np.count_nonzero(out["submerged_volume"]) > 100
    assert not out[bodies["num_points"] == 0].tobytes().strip(b"\0")
    g.free()


def test_buoyancy_mixed_scene():
    """3000 bodies: shared hulls, empty bodies, 1 to 70 000 points, one body with a NaN in its rotation and one with an
    infinite translation.  Those two come out NaN exactly where the specification does; every other body is bit-identical."""
    gow, g, params = _gen(256, 4)
    d16, n16 = g.maps_to_host(0, 4)
    scales = _scales(gow, params, 4)
    rng = np.random.default_rng(61)
    sizes = rng.integers(1, 40, 3000)
    sizes[0], sizes[2], sizes[3], sizes[4] = 5, 1, 33, 70000          # body 0 lends its hull to bodies 1, 5, 9, ...
    sizes[10::97] = 0
    bodies, hull = _scene(62, sizes, share_every=4)
    bodies["transform"][7, 1] = np.nan
    bodies["transform"][8, 3] = np.inf
    assert bodies["num_points"][7] > 0 and bodies["num_points"][8] > 0
    out, smp = g.buoyancy(bodies, hull, scales, RHO, 1e-3, 8, return_samples=True)
    with np.errstate(all="ignore"):
        ref, rsmp = bu.buoyancy(d16, n16, bodies, hull, scales, RHO, 1e-3, 8, return_samples=True)
    bad = np.zeros(len(bodies), bool)
    bad[[7, 8]] = True
    assert out[~bad].tobytes() == ref[~bad].tobytes()
    for f in ("force", "torque", "submerged_volume", "center_offset", "max_residual"):
        assert _same_or_both_nan(out[bad][f], ref[bad][f]), f
    assert np.array_equal(out["unconverged"], ref["unconverged"])
    assert np.isnan(out["max_residual"][bad]).all() and np.isnan(out["torque"][7, 2])
    assert np.isfinite(out[~bad]["torque"]).all() and np.count_nonzero(out["submerged_volume"]) > 1000
    empty = bodies["num_points"] == 0
    assert empty.sum() > 10 and not out[empty].tobytes().strip(b"\0")     # all-zero records
    assert _records_match(smp, rsmp)
    g.free()


def test_buoyancy_samples_are_the_surface_query():
    gow, g, params = _gen(256, 4)
    scales = _scales(gow, params, 4)
    scales[:, 2] *= np.float32(2.0)
    bodies, hull = _scene(71, np.random.default_rng(70).integers(0, 80, 500))
    for maxit in (8, 0):
        _, smp = g.buoyancy(bodies, hull, scales, RHO, 1e-3, maxit, return_samples=True)
        assert smp.tobytes() == g.query_surface(_world_xz(bodies, hull), scales, 1e-3, maxit).tobytes()
    g.free()


def test_buoyancy_on_flat_gpu_maps_is_archimedes():
    """Maps made on the GPU from a zero spectrum are exactly flat: an upright voxel box at a dyadic draft d displaces A d."""
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
    hull = _box(4, 4, 4)                                        # A = 4 m^2, from y = -1 to 1
    drafts = [0.0, 0.125, 0.375, 0.5, 0.625, 1.0, 1.3125, 2.0]
    ty = [1.0 - d for d in drafts] + [1.5, -1.25]
    bodies = _bodies([_transform(t=(37.0, y, -91.5)) for y in ty], [(0, len(hull))] * len(ty))
    out = g.buoyancy(bodies, hull, gow.WaveGenerator.map_scales(params), RHO, 1e-3, 8)
    want = [4.0 * d for d in drafts] + [0.0, 8.0]
    assert out["submerged_volume"].tolist() == want
    assert out["force"][:, 1].tolist() == [np.float32(np.float32(RHO) * bu.G) * np.float32(v) for v in want]
    assert not out["torque"].any() and not out["center_offset"][:, [0, 2]].any()
    g.free()


def test_buoyancy_device_equals_host():
    import torch
    from godotoceanwaves_b200.native import check, load_library
    gow, g, params = _gen(256, 4)
    scales = _scales(gow, params, 4)
    bodies, hull = _scene(81, np.random.default_rng(80).integers(0, 120, 800))
    out, smp = g.buoyancy(bodies, hull, scales, RHO, 1e-3, 8, return_samples=True)
    dev = torch.device("cuda", g.device)
    hull_d = torch.from_numpy(hull.view(np.uint8).copy()).to(dev)
    res_d = torch.zeros(len(bodies) * 12, dtype=torch.int32, device=dev)
    smp_d = torch.zeros(len(smp) * 10, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    lib = load_library()
    for samples in (smp_d, None):
        res_d.zero_()
        check(lib.ocean_buoyancy_device(g.context, len(bodies), bodies.ctypes.data, len(hull), hull_d.data_ptr(), 4, scales.ctypes.data,
                                        RHO, 1e-3, 8, res_d.data_ptr(), None if samples is None else samples.data_ptr()))
        g.synchronize()
        assert res_d.cpu().numpy().tobytes() == out.tobytes()
    assert smp_d.cpu().numpy().tobytes() == smp.tobytes()
    g.free()


def test_buoyancy_launch_count():
    gow, g, params = _gen(128, 2, frames=1)
    scales = gow.WaveGenerator.map_scales(params)
    bodies, hull = _scene(91, [5, 0, 40])
    for maxit, launches in ((8, 5), (0, 3)):
        before = g.info().kernel_launches
        g.buoyancy(bodies, hull, scales, RHO, 1e-3, maxit)
        assert g.info().kernel_launches - before == launches
    g.free()


def test_buoyancy_leaves_the_generator_alone():
    """The op must not touch the maps, and the next update must still be bit-exact against the CPU oracle."""
    import godotoceanwaves_b200 as gow
    from oracle import pyoracle as po
    N, Cn = 128, 3
    po.set_modes(po.MATH_DET, po.CONTRACT_FMA)
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(Cn)
    ora = po.OracleWaveGenerator(N); ora.init_gpu(Cn)
    pg = [demo_params(gow.WaveCascadeParameters, c) for c in range(Cn)]
    pc = [demo_params(po.CascadeParams, c) for c in range(Cn)]
    for _ in range(2):
        g.update_all(1.0 / 50.0, pg)
        ora.update_all(1.0 / 50.0, pc)
    d, n = g.maps_to_host(0, Cn)
    before = (_crc(d), _crc(n))
    scales = gow.WaveGenerator.map_scales(pg)
    g.buoyancy(*_scene(101, [3, 4]), scales)                    # staging sized by a small call first ...
    g.buoyancy(*_scene(102, np.full(700, 100)), scales, return_samples=True)   # ... then grown
    g.query_surface(np.zeros((10, 2), np.float32), scales)
    d, n = g.maps_to_host(0, Cn)
    assert (_crc(d), _crc(n)) == before
    g.update_all(1.0 / 50.0, pg)
    ora.update_all(1.0 / 50.0, pc)
    d, n = g.maps_to_host(0, Cn)
    assert np.array_equal(d.view(np.uint16), ora.displacement_map[:Cn]) and np.array_equal(n.view(np.uint16), ora.normal_map[:Cn])
    g.free()


def test_buoyancy_arguments():
    """Every invalid argument returns OCEAN_ERR_INVALID_ARGUMENT and launches nothing, through both entry points."""
    from godotoceanwaves_b200.native import load_library
    gow, g, params = _gen(128, 2, frames=1)
    lib = load_library()
    scales = gow.WaveGenerator.map_scales(params)
    bodies, hull = _scene(111, [4, 0, 6])
    bodies["num_points"][1] = 0                                 # (_scene made it share body 0's hull)
    res = np.zeros(len(bodies), bu.RESULT)
    smp = np.zeros(16, bu.SURFACE_RECORD)
    ok = dict(nb=len(bodies), b=bodies, np_=len(hull), p=hull.ctypes.data, nc=2, sc=scales.ctypes.data, rho=RHO, tol=1e-3, it=8,
              r=res.ctypes.data, s=None)

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
           dict(b=None), dict(p=None), dict(r=None), dict(nc=0), dict(nc=3), dict(sc=None)]
    for fn in (lib.ocean_buoyancy, lib.ocean_buoyancy_device):
        for kw in bad:
            a = dict(ok)
            a.update(kw)
            before = g.info().kernel_launches
            rc = fn(g.context, a["nb"], None if a["b"] is None else a["b"].ctypes.data, a["np_"], a["p"], a["nc"], a["sc"], a["rho"],
                    a["tol"], a["it"], a["r"], a["s"])
            assert rc == 1, kw
            assert g.info().kernel_launches == before, kw
    # NULL is fine where no count needs the buffer
    empty = bodies[[1]]
    assert lib.ocean_buoyancy(g.context, 1, empty.ctypes.data, 0, None, 2, scales.ctypes.data, RHO, 1e-3, 8, res.ctypes.data, None) == 0
    assert res[:1].tobytes() == bytes(48)
    assert lib.ocean_buoyancy(g.context, 0, None, 0, None, 0, None, RHO, 1e-3, 8, None, None) == 0
    assert len(g.buoyancy(bodies[:0], hull, scales)) == 0
    out, s = g.buoyancy(bodies, hull, scales, return_samples=True)
    assert len(out) == 3 and len(s) == 10 and out[1].tobytes() == bytes(48)
    g.free()
