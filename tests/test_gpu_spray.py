"""GPU parity of the spray-candidate op (ocean_extract_spray; sea_spray_particle.gdshader:80-94) against its numpy
specification oracle/spray.py, on the generator's own maps.  Bar: bit-identical records, identical candidate set."""
import numpy as np
import pytest

from conftest import EDGE_CASES, demo_params
from oracle import spray as sy
from test_gpu_sampling import _extreme_points

pytestmark = pytest.mark.gpu


def _generator(N, C, frames, **over):
    import godotoceanwaves_b200 as gow
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(max(2, C))
    p = [demo_params(gow.WaveCascadeParameters, c, **over) for c in range(C)]
    for _ in range(frames):
        g.update_all(1.0 / 50.0, p)
    return gow, g, p


@pytest.mark.parametrize("N,C,particles", [(128, 3, 10000), (256, 4, 65536), (512, 2, 250000), (1024, 2, 250000)])
def test_spray_records_bit_exact(N, C, particles):
    # a foamy sea: enough updates of a rough sea state for the foam plane to pass 0.9 in places
    gow, g, p = _generator(N, C, 25, whitecap=0.9, foam_amount=10.0)
    _, n16 = g.maps_to_host(0, C)
    scales = gow.WaveGenerator.map_scales(p)
    E = np.array([[7.5, 0, 0, 3.25], [0, 1, 0, 0], [0, 0, 7.5, -11.0]], np.float32)          # a scaled, shifted emitter box
    pts = gow.WaveGenerator.spray_grid(particles, E)
    assert np.array_equal(pts.view(np.uint32), sy.spray_grid(particles, E).view(np.uint32))
    rec, count = g.extract_spray(pts, scales, (0.6, 1.4, 0.6))
    ref = sy.spray_candidates(n16, pts, scales, (0.6, 1.4, 0.6))
    assert count == len(rec) == len(ref) and 0 < count < particles, (count, len(ref))
    assert rec.tobytes() == ref.tobytes()
    # max_records cuts the output, not the count
    few, count2 = g.extract_spray(pts, scales, (0.6, 1.4, 0.6), max_records=7)
    assert count2 == count and few.tobytes() == ref[:7].tobytes()
    g.free()


def _foamy(N=256, C=4):
    """maps of a foamy sea, with non-square tiles in cascades 0 and 1 (the anisotropic_tile corner and its transpose)"""
    import godotoceanwaves_b200 as gow
    tiles = [EDGE_CASES["anisotropic_tile"]["tile_length"], (41.0, 93.0)]
    g = gow.WaveGenerator(); g.map_size = N; g.init_gpu(C)
    p = [demo_params(gow.WaveCascadeParameters, c, whitecap=0.9, foam_amount=10.0, **({"tile_length": tiles[c]} if c < 2 else {}))
         for c in range(C)]
    for _ in range(25):
        g.update_all(1.0 / 50.0, p)
    scales = gow.WaveGenerator.map_scales(p)
    scales[:, 3] = [1.0, 1.0, -0.25, 0.5][:C]                  # the spray test ignores the normal scale
    return gow, g, scales


def test_spray_anisotropic_tiles():
    gow, g, scales = _foamy()
    _, n16 = g.maps_to_host(0, 4)
    pts = gow.WaveGenerator.spray_grid(65536, np.array([[30.0, 0, 0, 3.25], [0, 1, 0, 0], [0, 0, 30.0, -11.0]], np.float32))
    rec, count = g.extract_spray(pts, scales, (0.6, 1.4, 0.6))
    ref = sy.spray_candidates(n16, pts, scales, (0.6, 1.4, 0.6))
    assert count == len(rec) == len(ref) and 0 < count < len(pts), (count, len(ref))
    assert rec.tobytes() == ref.tobytes()
    g.free()


def test_spray_extreme_coordinates():
    """Huge, overflowing and non-finite start positions: the same candidates and records as the specification; a
    non-finite start is never a candidate, and no start changes another's record."""
    gow, g, scales = _foamy()
    _, n16 = g.maps_to_host(0, 4)
    pts, mask = _extreme_points(20000, 45)
    rec, count = g.extract_spray(pts, scales, (0.6, 1.4, 0.6))
    with np.errstate(all="ignore"):
        ref = sy.spray_candidates(n16, pts, scales, (0.6, 1.4, 0.6))
    assert count == len(rec) == len(ref) > 0 and rec.tobytes() == ref.tobytes()
    assert not np.any(~np.isfinite(pts[rec["index"]]))
    ordinary = np.nonzero(~mask)[0]
    sub, _ = g.extract_spray(pts[ordinary], scales, (0.6, 1.4, 0.6))
    mine = rec[~mask[rec["index"]]]
    assert np.array_equal(ordinary[sub["index"]], mine["index"])
    for f in ("start_x", "start_z", "scale_factor", "particle_scale", "foam"):
        assert np.array_equal(sub[f].view(np.uint32), mine[f].view(np.uint32)), f
    g.free()


def test_extract_spray_device_equals_host():
    import torch
    from godotoceanwaves_b200.native import check, load_library
    gow, g, scales = _foamy()
    pts = gow.WaveGenerator.spray_grid(65536, np.array([[7.5, 0, 0, 3.25], [0, 1, 0, 0], [0, 0, 7.5, -11.0]], np.float32))
    ps = np.array([0.6, 1.4, 0.6], np.float32)
    rec, count = g.extract_spray(pts, scales, ps)
    assert count > 0
    dev = torch.device("cuda", g.device)
    pts_d = torch.from_numpy(pts).to(dev)
    rec_d = torch.zeros(len(pts) * 8, dtype=torch.int32, device=dev)            # 32-byte records
    count_d = torch.full((1,), -1, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    check(load_library().ocean_extract_spray_device(g.context, len(pts), pts_d.data_ptr(), 4, scales.ctypes.data, ps.ctypes.data,
                                                    len(pts), rec_d.data_ptr(), count_d.data_ptr()))
    g.synchronize()
    assert int(count_d.cpu()[0]) == count
    assert rec_d.cpu().numpy().tobytes()[:32 * count] == rec.tobytes()
    g.free()


def test_spray_calm_sea_has_no_candidates_and_empty_input():
    gow, g, p = _generator(128, 2, 2, foam_amount=0.0)
    scales = gow.WaveGenerator.map_scales(p)
    rec, count = g.extract_spray(gow.WaveGenerator.spray_grid(4096), scales)
    assert count == 0 and len(rec) == 0
    rec, count = g.extract_spray(np.zeros((0, 2), np.float32), scales)
    assert count == 0
    g.free()
