"""GPU parity of the surface query (ocean_query_surface; water.gdshader:28,37 inverted, then :27-39,42-84 sampled) against
its numpy specification oracle/surface.py on the generator's own maps: bit-identical 40-byte records."""
import zlib

import numpy as np
import pytest

from conftest import demo_params
from oracle import surface as su
from test_gpu_sampling import _aniso_gen, _extreme_points, _gen, _points, _same_or_both_nan

pytestmark = pytest.mark.gpu


def _scales(gow, params, C):
    scales = gow.WaveGenerator.map_scales(params)
    scales[:, 2] = [1.0, 0.75, 0.0, 0.5][:C]                   # displacement scales of main.tscn:43-83 (+ one more)
    scales[:, 3] = [1.0, 1.0, 0.25, 0.5][:C]
    return scales


def _records_match(rec, ref):
    """bit-identical records, except that a NaN only has to meet a NaN (see _same_or_both_nan)"""
    return all(_same_or_both_nan(rec[f], ref[f]) for f in ("source_x", "source_z", "displacement", "gradient_foam", "residual")) and \
        np.array_equal(rec["iterations"], ref["iterations"])


@pytest.mark.parametrize("N,C", [(128, 3), (256, 4), (512, 2), (1024, 2)])
def test_query_surface_bit_exact(N, C):
    gow, g, params = _gen(N, C)
    d16, n16 = g.maps_to_host(0, C)
    assert gow.WaveGenerator.SURFACE_SAMPLE.itemsize == 40 and gow.WaveGenerator.SURFACE_SAMPLE == su.RECORD
    pts = _points(20000, 23 + N, 300.0)
    for factor in (1.0, 2.0):                                   # twice the displacement: many more restarts
        scales = _scales(gow, params, C)
        scales[:, 2] *= np.float32(factor)
        rec = g.query_surface(pts, scales, 1e-3, 8)
        ref = su.query_surface(d16, n16, pts, scales, 1e-3, 8)
        assert rec.tobytes() == ref.tobytes()
        assert np.any(rec["iterations"] > 8)                    # the restart kernel ran
        assert np.mean(rec["residual"] <= np.float32(1e-3)) > 0.95
    # fewer cascades, other tolerance and step budget
    rec = g.query_surface(pts[:3000], scales[:1], 1e-2, 3)
    assert rec.tobytes() == su.query_surface(d16[:1], n16[:1], pts[:3000], scales[:1], 1e-2, 3).tobytes()
    g.free()


def test_query_surface_device_equals_host():
    import torch
    from godotoceanwaves_b200.native import check, load_library
    gow, g, params = _gen(256, 4)
    scales = _scales(gow, params, 4)
    scales[:, 2] *= np.float32(2.0)
    pts = _points(50000, 5, 300.0)
    host = g.query_surface(pts, scales, 1e-3, 8)
    dev = torch.device("cuda", g.device)
    pts_d = torch.from_numpy(pts).to(dev)
    out_d = torch.zeros(pts.shape[0] * 10, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    check(load_library().ocean_query_surface_device(g.context, pts.shape[0], pts_d.data_ptr(), 4, scales.ctypes.data, 1e-3, 8, out_d.data_ptr()))
    g.synchronize()
    assert out_d.cpu().numpy().tobytes() == host.tobytes()
    g.free()


def test_query_surface_anisotropic_signed_scales():
    """Non-square tiles make the Jacobian terms du*s.x and dv*s.y differ; negative displacement and normal scales."""
    gow, g, scales = _aniso_gen()
    d16, n16 = g.maps_to_host(0, 4)
    pts = _points(20000, 33, 300.0)
    rec = g.query_surface(pts, scales, 1e-3, 8)
    ref = su.query_surface(d16, n16, pts, scales, 1e-3, 8)
    assert rec.tobytes() == ref.tobytes()
    assert np.any(rec["iterations"] > 8)                        # the restart kernel ran
    assert np.mean(rec["residual"] <= np.float32(1e-3)) > 0.95
    g.free()


def test_query_surface_extreme_coordinates():
    """Huge, overflowing and non-finite world positions.  A non-finite query has a NaN residual: the GPU sends it to the
    restart list (r <= tol is false) and the specification does not (r > tol is false), yet both take no step."""
    gow, g, params = _gen(256, 4)
    d16, n16 = g.maps_to_host(0, 4)
    scales = _scales(gow, params, 4)
    pts, mask = _extreme_points(4000, 43)
    rec = g.query_surface(pts, scales, 1e-3, 8)
    with np.errstate(all="ignore"):
        ref = su.query_surface(d16, n16, pts, scales, 1e-3, 8)
    assert _records_match(rec, ref)
    bad = ~np.isfinite(pts).all(1)
    for r in (rec[bad], ref[bad]):
        assert np.all(r["iterations"] == 0) and np.isnan(r["residual"]).all()
        assert np.isnan(r["displacement"]).all() and np.isnan(r["gradient_foam"]).all()
    assert g.query_surface(pts[~mask], scales, 1e-3, 8).tobytes() == rec[~mask].tobytes()
    g.free()


def test_query_surface_restart_grid_stride():
    """More pending queries than k_surface_restart has threads (2048 blocks x 64): every thread runs its grid-stride loop
    more than once."""
    gow, g, params = _gen(256, 4)
    d16, n16 = g.maps_to_host(0, 4)
    scales = _scales(gow, params, 4)
    scales[:, 2] *= np.float32(2.0)
    pts = _points(200000, 47, 300.0)
    tol = np.float32(1e-6)
    qx, qz = pts[:, 0].copy(), pts[:, 1].copy()
    _, _, r0, _ = su._solve(d16, scales, qx, qz, qx, qz, tol, 1)
    assert np.count_nonzero(r0 > tol) > 2048 * 64                # pending after the first start
    rec = g.query_surface(pts, scales, 1e-6, 1)
    assert rec.tobytes() == su.query_surface(d16, n16, pts, scales, 1e-6, 1).tobytes()
    g.free()


def test_query_surface_zero_iterations_is_the_map_query():
    gow, g, params = _gen(256, 4)
    scales = _scales(gow, params, 4)
    pts = _points(20000, 6, 300.0)
    rec = g.query_surface(pts, scales, 1e-3, 0)
    d, gr = g.sample(pts, scales)
    assert rec["displacement"].tobytes() == d.tobytes() and rec["gradient_foam"].tobytes() == gr.tobytes()
    assert rec["source_x"].tobytes() == pts[:, 0].tobytes() and rec["source_z"].tobytes() == pts[:, 1].tobytes()
    assert np.all(rec["iterations"] == 0)
    g.free()


def test_query_surface_arguments_and_empty_batch():
    from godotoceanwaves_b200.native import check, load_library
    gow, g, params = _gen(128, 2, frames=1)
    scales = gow.WaveGenerator.map_scales(params)
    assert len(g.query_surface(np.zeros((0, 2), np.float32), scales)) == 0
    pts = np.zeros((4, 2), np.float32)
    bad = [dict(map_scales=np.zeros((3, 4), np.float32)),      # more cascades than layers
           dict(map_scales=np.zeros((0, 4), np.float32)),
           dict(tolerance=0.0), dict(tolerance=-1e-3), dict(tolerance=float("nan")), dict(tolerance=float("inf")),
           dict(max_iterations=-1), dict(max_iterations=65)]
    for kw in bad:
        args = dict(map_scales=scales, tolerance=1e-3, max_iterations=8)
        args.update(kw)
        with pytest.raises(gow.OceanError):
            g.query_surface(pts, **args)
    assert len(g.query_surface(pts, scales, 1e-3, 64)) == 4 and len(g.query_surface(pts, scales, 1e-3, 0)) == 4
    lib = load_library()
    out = np.zeros(4, gow.WaveGenerator.SURFACE_SAMPLE)
    for n, p, o in [(-1, pts.ctypes.data, out.ctypes.data), (4, None, out.ctypes.data), (4, pts.ctypes.data, None)]:
        for fn in (lib.ocean_query_surface, lib.ocean_query_surface_device):
            with pytest.raises(gow.OceanError):
                check(fn(g.context, n, p, 2, scales.ctypes.data, 1e-3, 8, o))
    with pytest.raises(gow.OceanError):
        check(lib.ocean_query_surface(g.context, 4, pts.ctypes.data, 2, None, 1e-3, 8, out.ctypes.data))
    g.free()


def _crc(a) -> int:
    return zlib.crc32(np.ascontiguousarray(a).tobytes()) & 0xFFFFFFFF


def test_query_surface_leaves_the_generator_alone():
    """The query shares the staging buffers of the other query ops: it must not touch the maps, and the next update must
    still be bit-exact against the CPU oracle."""
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
    g.sample(_points(1000, 7, 300.0), scales)                   # staging sized by a smaller batch first ...
    g.query_surface(_points(70000, 8, 300.0), scales)           # ... then grown by the query
    g.sample(_points(1000, 9, 300.0), scales)
    d, n = g.maps_to_host(0, Cn)
    assert (_crc(d), _crc(n)) == before
    g.update_all(1.0 / 50.0, pg)
    ora.update_all(1.0 / 50.0, pc)
    d, n = g.maps_to_host(0, Cn)
    assert np.array_equal(d.view(np.uint16), ora.displacement_map[:Cn]) and np.array_equal(n.view(np.uint16), ora.normal_map[:Cn])
    g.free()
