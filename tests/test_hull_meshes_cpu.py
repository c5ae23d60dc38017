"""Hull mesh registration without a device: ocean_hull_set_meshes checks its arguments before the generator handle, so every
malformed mesh set is rejected with its own message, and a valid one gets as far as the missing generator.  Also
WaveGenerator.weld_faces on Godot's triangle soup."""
import numpy as np
import pytest

from godotoceanwaves_b200 import native
from godotoceanwaves_b200.wave_generator import WaveGenerator
from oracle import hull as oh

INVALID = 1


def _set(meshes, vertices, triangles, volumes=None):
    lib = native.load_library()
    m = np.ascontiguousarray(meshes, oh.MESH)
    v = np.ascontiguousarray(vertices, np.float32).reshape(-1, 3)
    t = np.ascontiguousarray(triangles, np.int32).reshape(-1, 3)
    ptr = lambda x: None if x is None or x.size == 0 else x.ctypes.data  # noqa: E731
    rc = lib.ocean_hull_set_meshes(None, len(m), ptr(m), len(v), ptr(v), len(t), ptr(t), ptr(volumes))
    return rc, lib.ocean_last_error().decode()


def _tetra():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    t = np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]], np.int32)     # clockwise seen from outside
    m = np.zeros(1, oh.MESH)
    m["num_vertices"], m["num_triangles"], m["normal_drag"], m["tangential_drag"] = 4, 4, 1.0, 0.1
    return m, v, t


def test_a_valid_set_reaches_the_generator_check():
    m, v, t = _tetra()
    assert oh.volumes(m, v, t)[0] == pytest.approx(1.0 / 6.0, rel=1e-6)
    rc, msg = _set(m, v, t)
    assert rc == INVALID and "generator handle is NULL" in msg


def _variants():
    m, v, t = _tetra()
    out = []

    def case(name, mm=m, vv=v, tt=t, note=""):
        out.append(pytest.param(mm, vv, tt, note, id=name))

    for field, value, note in [("first_vertex", -1, "vertices"), ("num_vertices", 5, "vertices"), ("num_vertices", -1, "vertices"),
                               ("first_triangle", 1, "triangles"), ("num_triangles", 5, "triangles"), ("num_triangles", -2, "triangles"),
                               ("normal_drag", -0.5, "drag"), ("tangential_drag", np.inf, "drag"), ("normal_drag", np.nan, "drag")]:
        mm = m.copy()
        mm[field] = value
        case(f"{field}={value}", mm=mm, note=note)
    mm = m.copy()
    mm["num_vertices"] = 3                                      # index 3 is now outside the mesh's range
    case("index_outside_mesh", mm=mm, note="index")
    tt = t.copy()
    tt[2, 1] = -1
    case("negative_index", tt=tt, note="index")
    for bad in (np.nan, np.inf, -np.inf):
        vv = v.copy()
        vv[2, 1] = bad
        case(f"vertex_{bad}", vv=vv, note="not finite")
    return out


@pytest.mark.parametrize("meshes,vertices,triangles,note", _variants())
def test_malformed_sets_are_rejected(meshes, vertices, triangles, note):
    rc, msg = _set(meshes, vertices, triangles)
    assert rc == INVALID and note in msg and "generator" not in msg


def test_counts_and_null_arrays_are_rejected():
    lib = native.load_library()
    m, v, t = _tetra()
    for args, note in [((-1, m.ctypes.data, 4, v.ctypes.data, 4, t.ctypes.data), "negative"),
                       ((1, m.ctypes.data, -4, v.ctypes.data, 4, t.ctypes.data), "negative"),
                       ((1, None, 4, v.ctypes.data, 4, t.ctypes.data), "NULL"),
                       ((1, m.ctypes.data, 4, None, 4, t.ctypes.data), "NULL"),
                       ((1, m.ctypes.data, 4, v.ctypes.data, 4, None), "NULL"),
                       ((1, m.ctypes.data, 2 ** 30, v.ctypes.data, 4, t.ctypes.data), "2^31"),
                       ((1, m.ctypes.data, 4, v.ctypes.data, 2 ** 30, t.ctypes.data), "2^31")]:
        assert lib.ocean_hull_set_meshes(None, *args, None) == INVALID
        assert note in lib.ocean_last_error().decode()


def test_weld_faces_keeps_winding_and_order():
    m, v, t = _tetra()
    soup = v[t].reshape(-1, 3)                                  # Mesh.get_faces(): three corners per triangle
    wv, wt = WaveGenerator.weld_faces(soup)
    assert wv.dtype == np.float32 and wt.dtype == np.int32
    assert np.array_equal(wv[wt], v[t])                        # the same triangles, corner for corner
    assert len(wv) == 4 and wt[0].tolist() == [0, 1, 2]        # numbered in order of first appearance
    mesh = m.copy()
    assert oh.volumes(mesh, wv, wt)[0] == pytest.approx(oh.volumes(m, v, t)[0], rel=1e-7)
    with pytest.raises(ValueError):
        WaveGenerator.weld_faces(soup[:-1])
