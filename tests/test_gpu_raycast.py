"""GPU parity of the ray cast (ocean_raycast) against its numpy specification oracle/raycast.py on the generator's own
maps: bit-identical 72-byte records, and the call's launches, validation and isolation."""
import zlib

import numpy as np
import pytest

from conftest import demo_params
from oracle import raycast as rc
from test_gpu_sampling import _gen, _same_or_both_nan
from test_gpu_surface import _scales
from test_oracle_raycast import grazing, ray_mix

pytestmark = pytest.mark.gpu

FLOAT_FIELDS = ("t", "position", "source_x", "source_z", "displacement", "gradient_foam", "gap", "residual")
COUNT_FIELDS = ("status", "evaluations", "iterations", "unconverged")


def _records_match(rec, ref):
    """bit-identical records, except that a NaN only has to meet a NaN (test_gpu_sampling._same_or_both_nan)"""
    return all(_same_or_both_nan(rec[f], ref[f]) for f in FLOAT_FIELDS) and all(np.array_equal(rec[f], ref[f]) for f in COUNT_FIELDS)


def _extreme_rays(seed):
    """rays with coordinates up to +-3e38, infinities and NaN in every field, and huge but finite directions"""
    rng = np.random.default_rng(seed)
    vals = np.array([3e38, -3e38, 1e30, -1e30, 2.0 ** 24, np.inf, -np.inf, np.nan], np.float32)
    r = ray_mix(8 * len(vals), seed)
    for j, v in enumerate(vals):
        for f in range(7):
            i = 8 * j + f + rng.integers(0, 2)
            if f < 3:
                r["origin"][i, f] = v
            elif f < 6:
                r["direction"][i, f - 3] = v
            else:
                r["t_max"][i] = v
    return r


@pytest.mark.parametrize("N,C", [(128, 3), (256, 4), (512, 2), (1024, 2)])
def test_raycast_bit_exact(N, C):
    gow, g, params = _gen(N, C)
    d16, n16 = g.maps_to_host(0, C)
    assert gow.WaveGenerator.RAY == rc.RAY and gow.WaveGenerator.RAY_HIT == rc.HIT
    rays = np.concatenate([ray_mix(400, 50 + N, 150.0), grazing(40, 60 + N), _extreme_rays(70 + N)])
    seen, restarted = set(), False
    for factor in (1.0, 2.0):                                   # twice the displacement: more restarts
        scales = _scales(gow, params, C)
        scales[:, 2] *= np.float32(factor)
        for iters in (8, 0):
            rec = g.raycast(rays, scales, 1.0, 128, 1e-3, iters)
            with np.errstate(all="ignore"):
                ref, trace = rc.raycast(d16, n16, rays, scales, 1.0, 128, 1e-3, iters, trace=True)
            assert _records_match(rec, ref), (factor, iters)
            seen |= set(np.unique(rec["status"]).tolist())
            restarted |= bool(np.any(trace["iterations"] > iters))     # more steps than one start can take: a restart ran
    assert seen == {rc.MISS, rc.HIT_FROM_ABOVE, rc.HIT_FROM_BELOW, rc.TRUNCATED, rc.INVALID} and restarted
    # the ordinary rays are unaffected by the extreme ones next to them
    plain = g.raycast(rays[:440], scales, 1.0, 128, 1e-3, 0)
    assert plain.tobytes() == rec[:440].tobytes()
    g.free()


def test_raycast_flat_water():
    """Zero-spectrum maps are exactly flat: every ray through y = 0 hits within tolerance / |d_y| of the analytic t."""
    gow, g, params = _gen(128, 2)                               # its updates cleared the dirty flags
    for c in range(2):
        g.set_spectrum_amplitudes(c, np.zeros((128, 128), np.complex64))
    g.update_all(1.0 / 50.0, params)
    d16, _ = g.maps_to_host(0, 2)
    assert not d16.astype(np.float32).any()
    rng = np.random.default_rng(3)
    n = 2000
    r = np.zeros(n, rc.RAY)
    oy = rng.integers(1, 64, n) * rng.choice([-0.25, 0.25], n)
    r["origin"] = np.stack([rng.integers(-512, 512, n) * 0.5, oy, rng.integers(-512, 512, n) * 0.5], 1)
    dy = -np.sign(oy) * rng.integers(1, 8, n) * 0.125
    r["direction"] = np.stack([rng.integers(-8, 8, n) * 0.25, dy, rng.integers(-8, 8, n) * 0.25], 1)
    r["t_max"] = np.inf
    scales = gow.WaveGenerator.map_scales(params)
    hit = g.raycast(r, scales)
    assert np.array_equal(hit["status"], np.where(oy > 0, rc.HIT_FROM_ABOVE, rc.HIT_FROM_BELOW))
    assert np.all(np.abs(hit["gap"]) <= np.float32(1e-3))
    assert np.all(np.abs(hit["t"] - (-oy / dy)) <= (1e-3 + 1e-5) / np.abs(dy))
    g.free()


def test_raycast_device_equals_host_and_launches():
    import torch
    from godotoceanwaves_b200.native import check, load_library
    gow, g, params = _gen(256, 4)
    scales = _scales(gow, params, 4)
    rays = ray_mix(4000, 9)
    host = g.raycast(rays, scales)
    dev = torch.device("cuda", g.device)
    rays_d = torch.from_numpy(rays.view(np.uint8).copy()).to(dev)
    out_d = torch.zeros(len(rays) * 18, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    before = g.info().kernel_launches
    check(load_library().ocean_raycast_device(g.context, len(rays), rays_d.data_ptr(), 4, scales.ctypes.data, 0.5, 1024, 1e-3, 8,
                                              out_d.data_ptr()))
    g.synchronize()
    assert g.info().kernel_launches - before == 2
    assert out_d.cpu().numpy().tobytes() == host.tobytes()
    g.free()


def test_raycast_arguments():
    from godotoceanwaves_b200.native import check, load_library
    gow, g, params = _gen(128, 2, frames=1)
    scales = gow.WaveGenerator.map_scales(params)
    rays = ray_mix(8, 1)
    assert len(g.raycast(np.zeros(0, rc.RAY), scales)) == 0
    bad = [dict(map_scales=np.zeros((3, 4), np.float32)), dict(map_scales=np.zeros((0, 4), np.float32)),
           dict(step=0.0), dict(step=-1.0), dict(step=float("nan")), dict(step=float("inf")),
           dict(max_samples=1), dict(max_samples=(1 << 20) + 1),
           dict(tolerance=0.0), dict(tolerance=float("nan")), dict(tolerance=float("inf")),
           dict(max_iterations=-1), dict(max_iterations=65)]
    before = g.info().kernel_launches
    for kw in bad:
        args = dict(map_scales=scales, step=0.5, max_samples=1024, tolerance=1e-3, max_iterations=8)
        args.update(kw)
        with pytest.raises(gow.OceanError):
            g.raycast(rays, **args)
    lib = load_library()
    out = np.zeros(8, rc.HIT)
    for n, p, o in [(-1, rays.ctypes.data, out.ctypes.data), (8, None, out.ctypes.data), (8, rays.ctypes.data, None)]:
        for fn in (lib.ocean_raycast, lib.ocean_raycast_device):
            with pytest.raises(gow.OceanError):
                check(fn(g.context, n, p, 2, scales.ctypes.data, 0.5, 1024, 1e-3, 8, o))
    for fn in (lib.ocean_raycast, lib.ocean_raycast_device):
        with pytest.raises(gow.OceanError):
            check(fn(g.context, 8, rays.ctypes.data, 2, None, 0.5, 1024, 1e-3, 8, out.ctypes.data))
    assert g.info().kernel_launches == before
    assert len(g.raycast(rays, scales, 0.5, 2, 1e-3, 64)) == 8 and len(g.raycast(rays, scales, 0.5, 1 << 20, 1e-3, 0)) == 8
    g.free()


def _crc(a) -> int:
    return zlib.crc32(np.ascontiguousarray(a).tobytes()) & 0xFFFFFFFF


def test_raycast_leaves_the_generator_alone():
    """The ray cast must not touch the maps, foam, spectrum or velocity staleness, and the next update must still be
    bit-exact against the CPU oracle."""
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

    def state():
        d, n = g.maps_to_host(0, Cn)
        return (_crc(d), _crc(n), tuple(_crc(g.get_foam_state(c)) for c in range(Cn)), tuple(_crc(g.spectrum_to_host(c)) for c in range(Cn)))

    before = state()
    scales = gow.WaveGenerator.map_scales(pg)
    g.raycast(ray_mix(3000, 11), scales)
    assert state() == before
    assert g.update_velocity() == Cn                    # still stale: the ray cast refreshed nothing
    g.update_all(1.0 / 50.0, pg)
    ora.update_all(1.0 / 50.0, pc)
    d, n = g.maps_to_host(0, Cn)
    assert np.array_equal(d.view(np.uint16), ora.displacement_map[:Cn]) and np.array_equal(n.view(np.uint16), ora.normal_map[:Cn])
    g.free()
