"""WaveGenerator -- mirror of assets/water/wave_generator.gd on top of libocean.so.

Same public surface as the reference node: ``map_size``, ``init_gpu(num_cascades)``,
``update(delta, parameters)``, ``_process(delta)`` (one pending cascade per call, highest index
first), ``descriptors['displacement_map' | 'normal_map']`` and the two static JONSWAP helpers.
All numerics happen in the CUDA library; this class only marshals parameters."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .native import CascadeParamsC, InfoC, OceanError, check, load_library

G = 9.81        # wave_generator.gd:5
DEPTH = 20.0    # wave_generator.gd:6


class _Descriptor:
    """Stand-in for RenderingContext.Descriptor (render_context.gd:23-28): ``rid`` is the device
    pointer of the layered RGBA16F map instead of a Vulkan RID."""

    def __init__(self, rid: int, layer_bytes: int):
        self.rid = rid
        self.layer_bytes = layer_bytes


def _same_record(a, b) -> bool:
    """ctypes hands out a fresh wrapper object per array access: compare the addresses of the underlying C records."""
    return C.addressof(a) == C.addressof(b)


class WaveGenerator:
    def __init__(self, device: int = 0):
        self.map_size = 0                       # wave_generator.gd:8
        self.device = device
        self.context = None                     # :9 (the native handle once init_gpu ran)
        self.descriptors = {}                   # :11
        self.pass_parameters = []               # :14
        self._num_cascades = 0
        self._carr = None
        self._seen = None
        self._wake_size = 0
        self._hull_vertex_counts = np.zeros(0, np.int64)      # num_vertices of each registered hull mesh

    # ---- wave_generator.gd:17-54
    def init_gpu(self, num_cascades: int) -> None:
        lib = load_library()
        if self.context:
            self.free()
        h = C.c_void_p()
        check(lib.ocean_create(int(self.device), int(self.map_size), int(num_cascades), C.byref(h)))
        self.context = h
        self._num_cascades = int(num_cascades)
        self._hull_vertex_counts = np.zeros(0, np.int64)
        disp, norm, layer = C.c_void_p(), C.c_void_p(), C.c_size_t()
        check(lib.ocean_get_maps(h, C.byref(disp), C.byref(norm), C.byref(layer)))
        self.descriptors = {"displacement_map": _Descriptor(disp.value, layer.value),
                            "normal_map": _Descriptor(norm.value, layer.value)}

    # ---- parameter marshalling
    def _marshal(self, parameters):
        n = len(parameters)
        if self._carr is None or len(self._carr) != n:
            self._carr = (CascadeParamsC * n)()
            self._seen = [None] * n
        seen = self._seen
        for i, p in enumerate(parameters):
            key = (id(p), p._version)
            # untouched objects are already current in the C array -- provided the library-mutated fields (time, dirty
            # flag) were last exchanged with THIS record and not with another generator's
            if seen[i] != key or (p._synced is not None and not _same_record(p._synced, self._carr[i])):
                p.to_c(self._carr[i])
                seen[i] = key
        return self._carr

    def _readback(self, parameters):
        for i, p in enumerate(parameters):
            p.from_c(self._carr[i])

    # ---- wave_generator.gd:56-63
    def _process(self, delta: float = 0.0) -> None:
        if not self.context or not self.pass_parameters:
            return
        arr = self._marshal(self.pass_parameters)
        check(load_library().ocean_process(self.context, arr, len(self.pass_parameters)))
        self._readback(self.pass_parameters)

    # ---- wave_generator.gd:90-109
    def _auto_init(self, parameters) -> None:
        """wave_generator.gd:92-93 creates the resources on the first update; a NEW generator has empty spectrum textures,
        so every cascade must regenerate (what water.gd:84-87 does when it sets the generator up)."""
        if not self.context:
            self.init_gpu(max(2, len(parameters)))
            for p in parameters:
                p.should_generate_spectrum = True

    def update(self, delta: float, parameters) -> None:
        assert len(parameters) != 0
        self._auto_init(parameters)
        arr = self._marshal(parameters)
        check(load_library().ocean_update(self.context, float(delta), arr, len(parameters)))
        self._readback(parameters)
        self.pass_parameters = parameters

    def update_all(self, delta: float, parameters) -> None:
        """update() + every pending cascade in one batched launch (the throughput path)."""
        assert len(parameters) != 0
        self._auto_init(parameters)
        arr = self._marshal(parameters)
        check(load_library().ocean_update_all(self.context, float(delta), arr, len(parameters)))
        self._readback(parameters)
        self.pass_parameters = parameters

    def update_frames(self, delta: float, parameters, frames: int) -> None:
        """`frames` consecutive update_all(delta) calls fused into a few launches (ocean_update_frames): bit-identical
        results, without the per-frame launch and host latency."""
        assert len(parameters) != 0
        self._auto_init(parameters)
        arr = self._marshal(parameters)
        check(load_library().ocean_update_frames(self.context, float(delta), arr, len(parameters), int(frames)))
        self._readback(parameters)
        self.pass_parameters = parameters

    @property
    def pass_num_cascades_remaining(self) -> int:      # wave_generator.gd:15
        return self.info().pending_cascades if self.context else 0

    # ---- wave_generator.gd:111-113
    def free(self) -> None:
        if self.context:
            check(load_library().ocean_destroy(self.context))
            self.context = None
            self.descriptors = {}

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    # ---- wave_generator.gd:116-121
    @staticmethod
    def JONSWAP_alpha(wind_speed: float = 20.0, fetch_length: float = 550e3) -> float:
        return load_library().ocean_jonswap_alpha(float(wind_speed), float(fetch_length))

    @staticmethod
    def JONSWAP_peak_angular_frequency(wind_speed: float = 20.0, fetch_length: float = 550e3) -> float:
        return load_library().ocean_jonswap_peak_angular_frequency(float(wind_speed), float(fetch_length))

    # ---- host hand-off and taps
    def _require(self):
        if not self.context:
            raise OceanError("init_gpu() has not been called")

    def synchronize(self) -> None:
        self._require()
        check(load_library().ocean_synchronize(self.context))

    def info(self) -> InfoC:
        self._require()
        out = InfoC()
        check(load_library().ocean_get_info(self.context, C.byref(out)))
        return out

    def maps_to_host(self, first: int = 0, count: int | None = None):
        """(displacement, normal) as float16 arrays [count, N, N, 4] (what texture_update would upload)."""
        self._require()
        count = self._num_cascades - first if count is None else count
        N = self.map_size
        d = np.empty((count, N, N, 4), np.float16)
        n = np.empty((count, N, N, 4), np.float16)
        check(load_library().ocean_copy_maps_to_host(self.context, first, count, d.ctypes.data, n.ctypes.data))
        return d, n

    def spectrum_to_host(self, cascade: int) -> np.ndarray:
        self._require()
        N = self.map_size
        out = np.empty((N, N, 4), np.float32)
        check(load_library().ocean_copy_spectrum_to_host(self.context, cascade, out.ctypes.data))
        return out

    def set_spectrum_amplitudes(self, cascade: int, amplitudes) -> None:
        """Replaces spectrum_compute's output of one cascade by amplitudes [N][N] complex64 (or [N][N][2] float32): A(id) per
        texel; the library completes the texture with conj A(mod(-id, N)) (spectrum_compute.glsl:121-124)."""
        self._require()
        a = np.ascontiguousarray(np.asarray(amplitudes).astype(np.complex64)).view(np.float32).reshape(self.map_size, self.map_size, 2)
        check(load_library().ocean_set_spectrum_amplitudes(self.context, cascade, a.ctypes.data))

    def enable_f32_taps(self, enable: bool = True) -> None:
        self._require()
        check(load_library().ocean_enable_f32_taps(self.context, 1 if enable else 0))

    def f32_maps_to_host(self, cascade: int):
        self._require()
        N = self.map_size
        d = np.empty((N, N, 4), np.float32)
        n = np.empty((N, N, 4), np.float32)
        check(load_library().ocean_copy_f32_maps_to_host(self.context, cascade, d.ctypes.data, n.ctypes.data))
        return d, n

    def rowpass_to_host(self, cascade: int) -> np.ndarray:
        self._require()
        N = self.map_size
        out = np.empty((4, N, N, 2), np.float32)
        check(load_library().ocean_copy_rowpass_to_host(self.context, cascade, out.ctypes.data))
        return out

    # -- map queries: the water shader's sampling contract as an op (water.gdshader:27-39,42-84) ----------------
    @staticmethod
    def map_scales(parameters) -> np.ndarray:
        """map_scales[i] = (1/tile_length.x, 1/tile_length.y, displacement_scale, normal_scale), water.gd:102-110
        (the divisions are float32, as Vector2.ONE / tile_length is in Godot)."""
        out = np.empty((len(parameters), 4), np.float32)
        for i, p in enumerate(parameters):
            out[i, 0] = np.float32(1.0) / np.float32(p.tile_length[0])
            out[i, 1] = np.float32(1.0) / np.float32(p.tile_length[1])
            out[i, 2] = p.displacement_scale
            out[i, 3] = p.normal_scale
        return out

    def sample(self, points_xz, map_scales) -> tuple:
        """(displacement [n][3], gradient_foam [n][3]) float32 at world positions points_xz [n][2], summed over the
        len(map_scales) first cascades: what vertex() and fragment() of water.gdshader read at UV = VERTEX.xz."""
        self._require()
        pts = np.ascontiguousarray(points_xz, np.float32).reshape(-1, 2)
        sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
        n = pts.shape[0]
        disp = np.empty((n, 3), np.float32)
        grad = np.empty((n, 3), np.float32)
        check(load_library().ocean_sample_maps(self.context, n, pts.ctypes.data, sc.shape[0], sc.ctypes.data,
                                               disp.ctypes.data, grad.ctypes.data))
        return disp, grad

    # -- velocity maps: the time derivative of the displacement map (include/ocean.h, ocean_update_velocity) -----------
    def update_velocity(self) -> int:
        """Recomputes the velocity layers whose maps changed since their last computation (asynchronous); returns their number."""
        self._require()
        n = C.c_int(0)
        check(load_library().ocean_update_velocity(self.context, C.byref(n)))
        return n.value

    def velocity_to_host(self, first: int = 0, count: int | None = None) -> np.ndarray:
        """The velocity maps (vx, vy, vz, 0) as float16 [count, N, N, 4], brought up to date first."""
        self._require()
        count = self._num_cascades - first if count is None else count
        N = self.map_size
        v = np.empty((count, N, N, 4), np.float16)
        check(load_library().ocean_copy_velocity_to_host(self.context, first, count, v.ctypes.data))
        return v

    def velocity_f32_to_host(self, cascade: int) -> np.ndarray:
        """One velocity layer before the half conversion, float32 [N, N, 4] (needs enable_f32_taps)."""
        self._require()
        N = self.map_size
        out = np.empty((N, N, 4), np.float32)
        check(load_library().ocean_copy_f32_velocity_to_host(self.context, cascade, out.ctypes.data))
        return out

    def sample_velocity(self, points_xz, map_scales) -> np.ndarray:
        """Water velocity [n][3] float32 at the UNDISPLACED points points_xz [n][2], summed over the len(map_scales) first
        cascades like the displacement of sample().  For the velocity at a world position pass query_surface()'s source point."""
        self._require()
        pts = np.ascontiguousarray(points_xz, np.float32).reshape(-1, 2)
        sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
        out = np.empty((pts.shape[0], 3), np.float32)
        check(load_library().ocean_sample_velocity(self.context, pts.shape[0], pts.ctypes.data, sc.shape[0], sc.ctypes.data,
                                                   out.ctypes.data))
        return out

    # -- surface query: the surface at a world position (inverts the horizontal displacement, then samples) ----------
    SURFACE_SAMPLE = np.dtype([("source_x", np.float32), ("source_z", np.float32), ("displacement", np.float32, 3),
                               ("gradient_foam", np.float32, 3), ("residual", np.float32), ("iterations", np.uint32)])  # struct ocean_surface_sample

    def query_surface(self, points_xz, map_scales, tolerance: float = 1e-3, max_iterations: int = 8) -> np.ndarray:
        """SURFACE_SAMPLE rows for world positions points_xz [n][2]: the undisplaced point P whose rendered surface point
        lies over the query (P + D_xz(P) = Q within `tolerance` where residual <= tolerance), and the maps sampled at P:
        displacement[1] is the water height at Q, normalize(-g.x, 1, -g.y) of gradient_foam the normal (include/ocean.h)."""
        self._require()
        pts = np.ascontiguousarray(points_xz, np.float32).reshape(-1, 2)
        sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
        out = np.zeros(pts.shape[0], self.SURFACE_SAMPLE)
        check(load_library().ocean_query_surface(self.context, pts.shape[0], pts.ctypes.data, sc.shape[0], sc.ctypes.data,
                                                 float(tolerance), int(max_iterations), out.ctypes.data))
        return out

    # -- ray cast: the first crossing of each ray with the displaced surface ------------------------------------------
    RAY = np.dtype([("origin", np.float32, 3), ("direction", np.float32, 3), ("t_max", np.float32)])   # struct ocean_ray
    RAY_HIT = np.dtype([("t", np.float32), ("position", np.float32, 3), ("source_x", np.float32), ("source_z", np.float32),
                        ("displacement", np.float32, 3), ("gradient_foam", np.float32, 3), ("gap", np.float32), ("residual", np.float32),
                        ("status", np.uint32), ("evaluations", np.uint32), ("iterations", np.uint32),
                        ("unconverged", np.uint32)])                                         # struct ocean_ray_hit
    RAY_MISS, RAY_HIT_FROM_ABOVE, RAY_HIT_FROM_BELOW, RAY_TRUNCATED, RAY_INVALID = range(5)  # OCEAN_RAY_*

    def raycast(self, rays, map_scales, step: float = 0.5, max_samples: int = 1024, tolerance: float = 1e-3,
                max_iterations: int = 8) -> np.ndarray:
        """RAY_HIT rows, one per RAY row of `rays`: the first crossing of origin + t * direction, t in [0, t_max], with the
        displaced surface (include/ocean.h, ocean_raycast).  `step` is the horizontal sample spacing in metres; status is
        one of the RAY_* constants, and a hit has |gap| <= tolerance when its refinement converged."""
        self._require()
        r = np.ascontiguousarray(rays, self.RAY).reshape(-1)
        sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
        out = np.zeros(len(r), self.RAY_HIT)
        check(load_library().ocean_raycast(self.context, len(r), r.ctypes.data, sc.shape[0], sc.ctypes.data, float(step), int(max_samples),
                                           float(tolerance), int(max_iterations), out.ctypes.data))
        return out

    # -- buoyancy: per-body hydrostatic force and torque from hull points on the displaced surface -------------------
    BUOYANCY_POINT = np.dtype([("position", np.float32, 3), ("volume", np.float32), ("half_height", np.float32)])   # struct ocean_buoyancy_point
    BUOYANCY_BODY = np.dtype([("transform", np.float32, 12), ("first_point", np.int32), ("num_points", np.int32)])  # struct ocean_buoyancy_body
    BUOYANCY_RESULT = np.dtype([("force", np.float32, 3), ("torque", np.float32, 3), ("submerged_volume", np.float32),
                                ("center_offset", np.float32, 3), ("max_residual", np.float32),
                                ("unconverged", np.uint32)])                                  # struct ocean_buoyancy_result

    def buoyancy(self, bodies, points, map_scales, density: float = 1025.0, tolerance: float = 1e-3, max_iterations: int = 8,
                 return_samples: bool = False):
        """BUOYANCY_RESULT rows, one per BUOYANCY_BODY row of `bodies` (a 3 x 4 row-major body-to-world transform and a range
        of the BUOYANCY_POINT rows of `points`; ranges may overlap): the hydrostatic force, the torque about the body origin,
        the submerged volume and the centre-of-buoyancy offset this tick (include/ocean.h, ocean_buoyancy).  With
        return_samples, also the SURFACE_SAMPLE of every world point, body by body."""
        self._require()
        b = np.ascontiguousarray(bodies, self.BUOYANCY_BODY).reshape(-1)
        p = np.ascontiguousarray(points, self.BUOYANCY_POINT).reshape(-1)
        sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
        out = np.zeros(len(b), self.BUOYANCY_RESULT)
        world = int(np.maximum(b["num_points"], 0).astype(np.int64).sum())
        samples = np.zeros(world, self.SURFACE_SAMPLE) if return_samples else None
        check(load_library().ocean_buoyancy(self.context, len(b), b.ctypes.data, len(p), p.ctypes.data, sc.shape[0], sc.ctypes.data,
                                            float(density), float(tolerance), int(max_iterations), out.ctypes.data,
                                            None if samples is None else samples.ctypes.data))
        return (out, samples) if return_samples else out

    # -- body forces: buoyancy plus quadratic drag against the water velocity, from one surface query ---------------
    BODY_VELOCITY = np.dtype([("linear", np.float32, 3), ("angular", np.float32, 3)])   # struct ocean_body_velocity
    DRAG_RESULT = np.dtype([("force", np.float32, 3), ("torque", np.float32, 3), ("wetted_drag_area", np.float32),
                            ("max_relative_speed", np.float32)])                      # struct ocean_drag_result

    def body_forces(self, bodies, velocities, points, drag_areas, map_scales, density: float = 1025.0, tolerance: float = 1e-3,
                    max_iterations: int = 8, return_samples: bool = False):
        """(BUOYANCY_RESULT rows, DRAG_RESULT rows), one each per BUOYANCY_BODY row of `bodies`: the records buoyancy() returns,
        and the quadratic drag against the water velocity (include/ocean.h, ocean_body_forces).  `velocities` holds one
        BODY_VELOCITY row per body (world frame; `linear` is the velocity of the body ORIGIN), `drag_areas` one C_d A (m^2)
        per BUOYANCY_POINT row of `points`.  With return_samples, also the SURFACE_SAMPLE of every world point."""
        self._require()
        b = np.ascontiguousarray(bodies, self.BUOYANCY_BODY).reshape(-1)
        v = np.ascontiguousarray(velocities, self.BODY_VELOCITY).reshape(-1)
        p = np.ascontiguousarray(points, self.BUOYANCY_POINT).reshape(-1)
        a = np.ascontiguousarray(drag_areas, np.float32).reshape(-1)
        sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
        if len(v) != len(b) or len(a) != len(p):
            raise ValueError(f"{len(v)} velocities for {len(b)} bodies, or {len(a)} drag areas for {len(p)} points")
        hydro = np.zeros(len(b), self.BUOYANCY_RESULT)
        drag = np.zeros(len(b), self.DRAG_RESULT)
        world = int(np.maximum(b["num_points"], 0).astype(np.int64).sum())
        samples = np.zeros(world, self.SURFACE_SAMPLE) if return_samples else None
        check(load_library().ocean_body_forces(self.context, len(b), b.ctypes.data, v.ctypes.data, len(p), p.ctypes.data, a.ctypes.data,
                                               sc.shape[0], sc.ctypes.data, float(density), float(tolerance), int(max_iterations),
                                               hydro.ctypes.data, drag.ctypes.data, None if samples is None else samples.ctypes.data))
        return (hydro, drag, samples) if return_samples else (hydro, drag)

    # -- floating bodies: sub-stepped buoyancy and drag, the body state advanced on the device ----------------------
    FLOATING_BODY = np.dtype([("mass", np.float32), ("inertia", np.float32, 3), ("first_point", np.int32),
                              ("num_points", np.int32)])                                     # struct ocean_floating_body
    BODY_STATE = np.dtype([("position", np.float32, 3), ("orientation", np.float32, 4), ("linear_velocity", np.float32, 3),
                           ("angular_velocity", np.float32, 3)])                            # struct ocean_body_state

    def simulate_bodies(self, bodies, states, points, drag_areas, map_scales, dt: float, substeps: int = 1, density: float = 1025.0,
                        tolerance: float = 1e-3, max_iterations: int = 8, return_records: bool = False,
                        return_transforms: bool = False):
        """The BODY_STATE rows of `states` advanced by `substeps` sub-steps of dt / substeps (include/ocean.h,
        ocean_simulate_bodies): buoyancy, drag and gravity on each FLOATING_BODY row of `bodies` (mass, principal inertia,
        a range of the BUOYANCY_POINT rows of `points` and of `drag_areas`).  The state's origin is the centre of mass and its
        orientation a unit quaternion (x, y, z, w).  Returns the new states (a new array); with return_records also the
        (BUOYANCY_RESULT, DRAG_RESULT) rows of the last sub-step, with return_transforms also the [n][12] float32 3 x 4
        row-major [R | position] of each new state."""
        self._require()
        b = np.ascontiguousarray(bodies, self.FLOATING_BODY).reshape(-1)
        s = np.array(states, self.BODY_STATE, copy=True).reshape(-1)
        p = np.ascontiguousarray(points, self.BUOYANCY_POINT).reshape(-1)
        a = np.ascontiguousarray(drag_areas, np.float32).reshape(-1)
        sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
        if len(s) != len(b) or len(a) != len(p):
            raise ValueError(f"{len(s)} states for {len(b)} bodies, or {len(a)} drag areas for {len(p)} points")
        hydro = np.zeros(len(b), self.BUOYANCY_RESULT) if return_records else None
        drag = np.zeros(len(b), self.DRAG_RESULT) if return_records else None
        transforms = np.zeros((len(b), 12), np.float32) if return_transforms else None
        ptr = lambda x: None if x is None else x.ctypes.data  # noqa: E731
        check(load_library().ocean_simulate_bodies(self.context, len(b), b.ctypes.data, s.ctypes.data, len(p), p.ctypes.data, a.ctypes.data,
                                                   sc.shape[0], sc.ctypes.data, float(density), float(dt), int(substeps), float(tolerance),
                                                   int(max_iterations), ptr(hydro), ptr(drag), ptr(transforms)))
        out = (s,)
        if return_records:
            out += (hydro, drag)
        if return_transforms:
            out += (transforms,)
        return out if len(out) > 1 else s

    # -- driven and moored bodies: thrusters, hull foils, applied loads and tethers in the integrator ------------------
    THRUSTER = np.dtype([("body", np.int32), ("position", np.float32, 3), ("direction", np.float32, 3), ("thrust", np.float32),
                         ("half_height", np.float32)])                                    # struct ocean_thruster
    FOIL = np.dtype([("body", np.int32), ("position", np.float32, 3), ("normal", np.float32, 3), ("area", np.float32),
                     ("half_height", np.float32)])                                        # struct ocean_foil
    BODY_LOAD = np.dtype([("force", np.float32, 3), ("torque", np.float32, 3)])           # struct ocean_body_load
    TETHER = np.dtype([("body_a", np.int32), ("body_b", np.int32), ("point_a", np.float32, 3), ("point_b", np.float32, 3),
                       ("rest_length", np.float32), ("stiffness", np.float32), ("damping", np.float32)])      # struct ocean_tether
    DRIVE_RESULT = np.dtype([("force", np.float32, 3), ("torque", np.float32, 3), ("wetted_foil_area", np.float32),
                             ("max_normal_speed", np.float32)])                           # struct ocean_drive_result

    def drive_bodies(self, bodies, states, points, drag_areas, map_scales, dt: float, substeps: int = 1, density: float = 1025.0,
                     tolerance: float = 1e-3, max_iterations: int = 8, thrusters=None, foils=None, loads=None, tethers=None,
                     return_records: bool = False, return_tensions: bool = False, return_transforms: bool = False):
        """simulate_bodies with the THRUSTER, FOIL and TETHER rows and one BODY_LOAD row per body (loads may be None) acting on
        the bodies (include/ocean.h, ocean_simulate_driven_bodies).  Returns the new states; with return_records also the
        (BUOYANCY_RESULT, DRAG_RESULT, DRIVE_RESULT) rows of the last sub-step, with return_tensions the last sub-step's tension
        of each tether (float32), with return_transforms the [n][12] float32 transforms of the new states."""
        self._require()
        b = np.ascontiguousarray(bodies, self.FLOATING_BODY).reshape(-1)
        s = np.array(states, self.BODY_STATE, copy=True).reshape(-1)
        p = np.ascontiguousarray(points, self.BUOYANCY_POINT).reshape(-1)
        a = np.ascontiguousarray(drag_areas, np.float32).reshape(-1)
        sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
        th = np.ascontiguousarray(np.zeros(0, self.THRUSTER) if thrusters is None else thrusters, self.THRUSTER).reshape(-1)
        fo = np.ascontiguousarray(np.zeros(0, self.FOIL) if foils is None else foils, self.FOIL).reshape(-1)
        te = np.ascontiguousarray(np.zeros(0, self.TETHER) if tethers is None else tethers, self.TETHER).reshape(-1)
        ld = None if loads is None else np.ascontiguousarray(loads, self.BODY_LOAD).reshape(-1)
        if len(s) != len(b) or len(a) != len(p) or (ld is not None and len(ld) != len(b)):
            raise ValueError(f"{len(s)} states for {len(b)} bodies, {len(a)} drag areas for {len(p)} points, or loads of another length")
        hydro = np.zeros(len(b), self.BUOYANCY_RESULT) if return_records else None
        drag = np.zeros(len(b), self.DRAG_RESULT) if return_records else None
        drive = np.zeros(len(b), self.DRIVE_RESULT) if return_records else None
        tensions = np.zeros(len(te), np.float32) if return_tensions else None
        transforms = np.zeros((len(b), 12), np.float32) if return_transforms else None
        ptr = lambda x: None if x is None or x.size == 0 else x.ctypes.data  # noqa: E731
        check(load_library().ocean_simulate_driven_bodies(
            self.context, len(b), ptr(b), ptr(s), len(p), ptr(p), ptr(a), sc.shape[0], sc.ctypes.data, float(density), float(dt),
            int(substeps), float(tolerance), int(max_iterations), len(th), ptr(th), len(fo), ptr(fo), ptr(ld), len(te), ptr(te),
            ptr(hydro), ptr(drag), ptr(drive), ptr(tensions), ptr(transforms)))
        out = (s,)
        if return_records:
            out += (hydro, drag, drive)
        if return_tensions:
            out += (tensions,)
        if return_transforms:
            out += (transforms,)
        return out if len(out) > 1 else s

    # -- hull meshes: pressure and drag integrated over the wetted triangles of a triangle-mesh hull -------------------
    HULL_MESH = np.dtype([("first_vertex", np.int32), ("num_vertices", np.int32), ("first_triangle", np.int32), ("num_triangles", np.int32),
                          ("normal_drag", np.float32), ("tangential_drag", np.float32)])     # struct ocean_hull_mesh
    HULL_BODY = np.dtype([("transform", np.float32, 12), ("mesh", np.int32), ("reserved", np.int32)])      # struct ocean_hull_body
    FLOATING_HULL = np.dtype([("mass", np.float32), ("inertia", np.float32, 3), ("mesh", np.int32)])      # struct ocean_floating_hull

    @staticmethod
    def weld_faces(faces):
        """(vertices [V][3] float32, triangles [T][3] int32) from triangle soup [T * 3][3] (Godot's Mesh.get_faces()): corners with
        identical coordinates become one vertex, numbered in order of first appearance, and each triangle keeps its winding.
        A welded hull queries each vertex once where the soup queries it once per triangle that touches it."""
        f = np.ascontiguousarray(faces, np.float32).reshape(-1, 3)
        if len(f) % 3:
            raise ValueError(f"{len(f)} corners are not whole triangles")
        _, first, inverse = np.unique(f.view(np.dtype((np.void, 12))).reshape(-1), return_index=True, return_inverse=True)
        order = np.argsort(first, kind="stable")           # unique rows in order of first appearance
        rank = np.empty_like(order)
        rank[order] = np.arange(len(order))
        return f[first[order]].copy(), rank[inverse.reshape(-1)].astype(np.int32).reshape(-1, 3)

    def set_hull_meshes(self, meshes, vertices, triangles) -> np.ndarray:
        """Registers the HULL_MESH rows of `meshes` (ranges of `vertices` [V][3] float32 and of `triangles` [T][3] int32, indices
        local to each mesh's vertex range, Godot's clockwise winding) on the device (include/ocean.h, ocean_hull_set_meshes);
        an empty `meshes` releases the set.  Returns each mesh's enclosed signed volume (float32, negative when wound inward)."""
        self._require()
        m = np.ascontiguousarray(meshes, self.HULL_MESH).reshape(-1)
        v = np.ascontiguousarray(vertices, np.float32).reshape(-1, 3)
        t = np.ascontiguousarray(triangles, np.int32).reshape(-1, 3)
        volumes = np.zeros(len(m), np.float32)
        ptr = lambda x: None if x.size == 0 else x.ctypes.data  # noqa: E731
        check(load_library().ocean_hull_set_meshes(self.context, len(m), ptr(m), len(v), ptr(v), len(t), ptr(t), ptr(volumes)))
        self._hull_vertex_counts = m["num_vertices"].astype(np.int64)
        return volumes

    def hull_forces(self, bodies, velocities, map_scales, density: float = 1025.0, tolerance: float = 1e-3, max_iterations: int = 8,
                    return_samples: bool = False):
        """(BUOYANCY_RESULT rows, DRAG_RESULT rows), one each per HULL_BODY row of `bodies` (a 3 x 4 row-major transform and the
        index of a registered mesh) with its BODY_VELOCITY row: hydrostatic pressure and drag integrated over the mesh's wetted
        triangles (include/ocean.h, ocean_hull_forces).  With return_samples, also the SURFACE_SAMPLE of every world vertex."""
        self._require()
        b = np.ascontiguousarray(bodies, self.HULL_BODY).reshape(-1)
        v = np.ascontiguousarray(velocities, self.BODY_VELOCITY).reshape(-1)
        sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
        if len(v) != len(b):
            raise ValueError(f"{len(v)} velocities for {len(b)} bodies")
        hydro = np.zeros(len(b), self.BUOYANCY_RESULT)
        drag = np.zeros(len(b), self.DRAG_RESULT)
        samples = None
        if return_samples:                                      # an unknown mesh index is rejected by the call itself
            counts = self._hull_vertex_counts
            known = b["mesh"][(b["mesh"] >= 0) & (b["mesh"] < len(counts))]
            samples = np.zeros(int(counts[known].sum()), self.SURFACE_SAMPLE)
        ptr = lambda x: None if x is None or x.size == 0 else x.ctypes.data  # noqa: E731
        check(load_library().ocean_hull_forces(self.context, len(b), ptr(b), ptr(v), sc.shape[0], sc.ctypes.data, float(density),
                                               float(tolerance), int(max_iterations), ptr(hydro), ptr(drag), ptr(samples)))
        return (hydro, drag, samples) if return_samples else (hydro, drag)

    def simulate_hull_bodies(self, bodies, states, map_scales, dt: float, substeps: int = 1, density: float = 1025.0,
                             tolerance: float = 1e-3, max_iterations: int = 8, return_records: bool = False,
                             return_transforms: bool = False):
        """simulate_bodies on hull meshes (include/ocean.h, ocean_simulate_hull_bodies): each FLOATING_HULL row of `bodies` (mass,
        principal inertia, a registered mesh) advanced from its BODY_STATE row.  Returns the new states; with return_records also
        the (BUOYANCY_RESULT, DRAG_RESULT) rows of the last sub-step, with return_transforms the [n][12] float32 transforms."""
        self._require()
        b = np.ascontiguousarray(bodies, self.FLOATING_HULL).reshape(-1)
        s = np.array(states, self.BODY_STATE, copy=True).reshape(-1)
        sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
        if len(s) != len(b):
            raise ValueError(f"{len(s)} states for {len(b)} bodies")
        hydro = np.zeros(len(b), self.BUOYANCY_RESULT) if return_records else None
        drag = np.zeros(len(b), self.DRAG_RESULT) if return_records else None
        transforms = np.zeros((len(b), 12), np.float32) if return_transforms else None
        ptr = lambda x: None if x is None or x.size == 0 else x.ctypes.data  # noqa: E731
        check(load_library().ocean_simulate_hull_bodies(self.context, len(b), ptr(b), ptr(s), sc.shape[0], sc.ctypes.data, float(density),
                                                        float(dt), int(substeps), float(tolerance), int(max_iterations), ptr(hydro),
                                                        ptr(drag), ptr(transforms)))
        out = (s,)
        if return_records:
            out += (hydro, drag)
        if return_transforms:
            out += (transforms,)
        return out if len(out) > 1 else s

    # -- spray candidates: the spawn test of sea_spray_particle.gdshader:80-94 as a stream compaction --------------
    SPRAY_RECORD = np.dtype([("index", np.uint32), ("start_x", np.float32), ("start_z", np.float32), ("scale_factor", np.float32),
                             ("particle_scale", np.float32, 3), ("foam", np.float32)])     # struct ocean_spray_record

    @staticmethod
    def spray_grid(num_particles: int, emission_transform=None) -> np.ndarray:
        """START_POS.xz of the emitter's particle grid (sea_spray_particle.gdshader:47,52-54), float32 [num_particles][2]."""
        out = np.empty((num_particles, 2), np.float32)
        et = None if emission_transform is None else np.ascontiguousarray(emission_transform, np.float32).reshape(12)
        check(load_library().ocean_spray_grid(num_particles, None if et is None else et.ctypes.data, out.ctypes.data))
        return out

    def extract_spray(self, points_xz, map_scales, particle_scale=(1.0, 1.0, 1.0), max_records: int | None = None):
        """The ACTIVE spray candidates among points_xz [n][2] as SPRAY_RECORD rows in candidate order, and their total
        number (which exceeds len(records) when max_records cut the output)."""
        self._require()
        pts = np.ascontiguousarray(points_xz, np.float32).reshape(-1, 2)
        sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
        ps = np.ascontiguousarray(particle_scale, np.float32).reshape(3)
        n = pts.shape[0]
        cap = n if max_records is None else int(max_records)
        recs = np.zeros(cap, self.SPRAY_RECORD)
        count = C.c_int(0)
        check(load_library().ocean_extract_spray(self.context, n, pts.ctypes.data, sc.shape[0], sc.ctypes.data, ps.ctypes.data, cap,
                                                 recs.ctypes.data, C.byref(count)))
        return recs[:min(count.value, cap)], count.value

    # -- spray particles: one particle-process frame of the spray emitter, with the live particles as instances ------
    SPRAY_EMITTER = np.dtype([("amount", np.int32), ("num_particles", np.int32), ("emission_transform", np.float32, 12),
                              ("particle_scale", np.float32, 3), ("lifetime", np.float32), ("lifetime_randomness", np.float32),
                              ("random_seed", np.uint32), ("emitter_lifetime", np.float64)])        # struct ocean_spray_emitter
    SPRAY_PARTICLE = np.dtype([("transform", np.float32, 12), ("custom", np.float32, 4), ("userdata1", np.float32, 4),
                               ("userdata2", np.float32, 4), ("userdata3", np.float32, 4), ("number", np.uint32),
                               ("flags", np.uint32)])                                              # struct ocean_spray_particle

    @staticmethod
    def default_spray_emitter() -> np.ndarray:
        """The reference scene's emitter (ocean_default_spray_emitter) as a 0-d SPRAY_EMITTER array."""
        e = np.zeros((), WaveGenerator.SPRAY_EMITTER)
        check(load_library().ocean_default_spray_emitter(e.ctypes.data))
        return e

    def spray_particles(self, emitter, states, t0: float, t1: float, map_scales, max_instances: int | None = None):
        """One particle-process frame [t0, t1) of the emitter (include/ocean.h, ocean_spray_particles): the restarts, start()
        and process() of sea_spray_particle.gdshader on the SPRAY_PARTICLE rows of `states` (None = amount never-emitted
        particles).  Returns (new states, instances [n][16] float32 of the live particles in INDEX order, number of live
        particles), where n = min(count, max_instances)."""
        self._require()
        e = np.array(emitter, self.SPRAY_EMITTER).reshape(())
        amount = max(int(e["amount"]), 0)
        s = np.zeros(amount, self.SPRAY_PARTICLE) if states is None else np.array(states, self.SPRAY_PARTICLE, copy=True).reshape(-1)
        if len(s) != amount:
            raise ValueError(f"{len(s)} states for an emitter of {amount} particles")
        sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
        cap = amount if max_instances is None else int(max_instances)
        inst = np.zeros((max(cap, 0), 16), np.float32)
        count = C.c_int(0)
        check(load_library().ocean_spray_particles(self.context, e.ctypes.data, float(t0), float(t1), sc.shape[0], sc.ctypes.data,
                                                   s.ctypes.data, cap, inst.ctypes.data, C.byref(count)))
        return s, inst[:min(count.value, cap)], count.value

    # -- wake layer: a local height field driven by moving sources and floating bodies --------------------------------
    WAKE_PARAMS = np.dtype([("size", np.int32), ("sponge_cells", np.int32), ("cell_size", np.float32), ("damping", np.float32),
                            ("sponge_damping", np.float32)])                                     # struct ocean_wake_params
    WAKE_SOURCE = np.dtype([("x", np.float32), ("z", np.float32), ("vx", np.float32), ("vz", np.float32), ("radius", np.float32),
                            ("head", np.float32), ("body", np.int32)])                           # struct ocean_wake_source

    @staticmethod
    def wake_kernel_taps() -> np.ndarray:
        """The 28 float32 taps G[a][b] of the wake step's stencil, (0,0), (1,0), (1,1), ... (6,6) (no device needed)."""
        out = np.zeros(28, np.float32)
        check(load_library().ocean_wake_kernel_taps(out.ctypes.data))
        return out

    def wake_init(self, size: int, cell_size: float = 0.5, damping: float = 0.0, sponge_cells: int = 48,
                  sponge_damping: float = 1.0) -> None:
        """(Re)create the wake layer, zeroed at origin (0, 0): size x size cells of cell_size metres (include/ocean.h,
        ocean_wake_init).  size = 0 releases it."""
        self._require()
        p = np.array((int(size), int(sponge_cells), float(cell_size), float(damping), float(sponge_damping)), self.WAKE_PARAMS)
        check(load_library().ocean_wake_init(self.context, p.ctypes.data))
        self._wake_size = int(size)

    def wake_step(self, dt: float, substeps: int = 1, origin=(0, 0), sources=None, states=None) -> None:
        """Advance the wake layer by `substeps` sub-steps of dt / substeps with the window at `origin` (whole cells), forced
        by the WAKE_SOURCE rows of `sources`; `states` are the BODY_STATE rows body-attached sources follow."""
        self._require()
        src = np.zeros(0, self.WAKE_SOURCE) if sources is None else np.ascontiguousarray(sources, self.WAKE_SOURCE).reshape(-1)
        st = np.zeros(0, self.BODY_STATE) if states is None else np.ascontiguousarray(states, self.BODY_STATE).reshape(-1)
        check(load_library().ocean_wake_step(self.context, float(dt), int(substeps), int(origin[0]), int(origin[1]), len(src),
                                             src.ctypes.data if len(src) else None, len(st), st.ctypes.data if len(st) else None))

    def wake_map(self):
        """(map [N][N][4] float16 (h, dh/dx, dh/dz, 0), world rect (x0, z0, width, depth)) of the wake layer."""
        import torch
        self._require()
        n = self._wake_size
        dev = torch.empty(n * n * 4, dtype=torch.float16, device=torch.device("cuda", self.device))
        rect = np.zeros(4, np.float32)
        torch.cuda.synchronize(dev.device)
        check(load_library().ocean_wake_render_map(self.context, dev.data_ptr(), rect.ctypes.data))
        self.synchronize()
        return dev.cpu().numpy().reshape(n, n, 4), rect

    def sample_wake(self, points_xz) -> np.ndarray:
        """[n][3] float32 (h, dh/dx, dh/dz) of the wake layer at world points (x, z), bilinear; 0 outside the window."""
        self._require()
        pts = np.ascontiguousarray(points_xz, np.float32).reshape(-1, 2)
        out = np.zeros((len(pts), 3), np.float32)
        check(load_library().ocean_sample_wake(self.context, len(pts), pts.ctypes.data, out.ctypes.data))
        return out

    def wake_state(self):
        """(h, h_prev, origin): host copies of the wake layer's fields ([N][N] float32) and its origin in cells."""
        self._require()
        n = self._wake_size
        h, hp, o = np.zeros((n, n), np.float32), np.zeros((n, n), np.float32), np.zeros(2, np.int64)
        check(load_library().ocean_wake_get_state(self.context, h.ctypes.data, hp.ctypes.data, o.ctypes.data))
        return h, hp, (int(o[0]), int(o[1]))

    def set_wake_state(self, h, h_prev, origin=(0, 0)) -> None:
        self._require()
        n = self._wake_size
        h = np.ascontiguousarray(h, np.float32)
        hp = np.ascontiguousarray(h_prev, np.float32)
        if h.shape != (n, n) or hp.shape != (n, n):
            raise ValueError(f"wake fields must be [{n}][{n}]")
        check(load_library().ocean_wake_set_state(self.context, h.ctypes.data, hp.ctypes.data, int(origin[0]), int(origin[1])))

    def wake_set_coupling(self, enable: bool) -> None:
        """Couple the wake layer into the surface query, buoyancy, body forces and the body integrator (include/ocean.h,
        ocean_wake_set_coupling): they read the wake free surface h + phi of the last step call.  Off releases the snapshots."""
        self._require()
        check(load_library().ocean_wake_set_coupling(self.context, int(enable)))

    def wake_coupling(self):
        """(e, e_old, origins, T): the coupling's snapshots ([N][N] float32), their origins ((e.x, e.z), (e_old.x, e_old.z))
        in cells and the interval between them; zeros and T = 0 until the first coupled step call."""
        self._require()
        n = self._wake_size
        e, eo, o, t = np.zeros((n, n), np.float32), np.zeros((n, n), np.float32), np.zeros(4, np.int64), np.zeros(1, np.float32)
        check(load_library().ocean_wake_get_coupling(self.context, e.ctypes.data, eo.ctypes.data, o.ctypes.data, t.ctypes.data))
        return e, eo, ((int(o[0]), int(o[1])), (int(o[2]), int(o[3]))), np.float32(t[0])

    WAKE_FOAM_PARAMS = np.dtype([("whitecap", np.float32), ("grow_rate", np.float32), ("stir_rate", np.float32),
                                 ("decay_rate", np.float32)])                                   # struct ocean_wake_foam_params

    def wake_set_foam(self, whitecap: float | None = 0.3, grow_rate: float = 1.0, stir_rate: float = 0.0,
                      decay_rate: float = 0.5) -> None:
        """Advance a foam field with the wake layer (include/ocean.h, ocean_wake_set_foam): white water where beta = c / dx
        exceeds `whitecap` and where sources stir the water, decaying at `decay_rate`; it becomes the render map's fourth
        channel.  whitecap=None turns foam off and releases the field; enabling zeroes it, changing parameters keeps it."""
        self._require()
        if whitecap is None:
            check(load_library().ocean_wake_set_foam(self.context, None))
            return
        p = np.array((float(whitecap), float(grow_rate), float(stir_rate), float(decay_rate)), self.WAKE_FOAM_PARAMS)
        check(load_library().ocean_wake_set_foam(self.context, p.ctypes.data))

    def wake_foam(self) -> np.ndarray:
        """A host copy of the wake layer's foam field F ([N][N] float32, window order)."""
        self._require()
        n = self._wake_size
        out = np.zeros((n, n), np.float32)
        check(load_library().ocean_wake_get_foam_state(self.context, out.ctypes.data))
        return out

    def set_wake_foam(self, foam) -> None:
        self._require()
        n = self._wake_size
        f = np.ascontiguousarray(foam, np.float32)
        if f.shape != (n, n):
            raise ValueError(f"the wake foam field must be [{n}][{n}]")
        check(load_library().ocean_wake_set_foam_state(self.context, f.ctypes.data))

    def wake_set_obstacles(self, mask, origin=(0, 0)) -> None:
        """Block wake waves with a world-fixed mask (include/ocean.h, ocean_wake_set_obstacles): mask [depth][width], nonzero
        where the cell is land, a quay or a breakwater; row r is world cell row origin[1] + r along z, column q world cell
        column origin[0] + q along x (cells of the layer's cell size).  mask=None removes it."""
        self._require()
        if mask is None:
            check(load_library().ocean_wake_set_obstacles(self.context, None, 0, 0, 0, 0))
            return
        m = np.ascontiguousarray(np.asarray(mask) != 0, np.uint8)
        if m.ndim != 2:
            raise ValueError("the obstacle mask must be [depth][width]")
        check(load_library().ocean_wake_set_obstacles(self.context, m.ctypes.data, m.shape[1], m.shape[0], int(origin[0]),
                                                      int(origin[1])))

    def wake_set_readers(self, raycast: bool = False, spray: bool = False) -> None:
        """Let the ray cast and spray read the wake layer (include/ocean.h, ocean_wake_set_readers): raycast=True makes the
        ray cast hit the coupled surface while the coupling is live; spray=True adds the layer's slopes and foam to the spawn
        test and its height to the spray particles.  Both False (the default) reads nothing."""
        self._require()
        readers = (1 if raycast else 0) | (2 if spray else 0)
        check(load_library().ocean_wake_set_readers(self.context, readers))

    # -- sea state and drifters: the spectra's moments, and debris that rides the waves and drifts with the Stokes drift --
    SEA_STATE = np.dtype([("m_minus1", np.float64), ("m0", np.float64), ("m1", np.float64), ("m2", np.float64),
                          ("direction", np.float64, 2), ("slope", np.float64, 2), ("stokes", np.float64, 2),
                          ("significant_wave_height", np.float64), ("mean_period", np.float64), ("zero_crossing_period", np.float64),
                          ("energy_period", np.float64), ("mean_direction", np.float64), ("directional_spread", np.float64),
                          ("mean_square_slope", np.float64), ("stokes_speed", np.float64)])      # struct ocean_sea_state
    DRIFTER = np.dtype([("x", np.float64), ("z", np.float64), ("yaw", np.float32), ("yaw_rate", np.float32), ("windage", np.float32),
                        ("tilt", np.float32), ("offset", np.float32), ("scale", np.float32)])   # struct ocean_drifter
    DRIFT_PARAMS = np.dtype([("current", np.float32, 2), ("wind", np.float32, 2), ("stokes_scale", np.float32), ("flags", np.uint32),
                             ("box", np.float64, 4)])                                            # struct ocean_drift_params
    DRIFT_WRAP, DRIFT_READ_WAKE = 1, 2                                                           # OCEAN_DRIFT_*

    def sea_state(self, map_scales):
        """The sea state of the len(map_scales) first cascades (include/ocean.h, ocean_get_sea_state): (total, per_cascade),
        a 0-d SEA_STATE of the surface as rendered (moments scaled by displacement_scale^2 and summed) and the unscaled
        SEA_STATE of each cascade."""
        self._require()
        sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
        per = np.zeros(sc.shape[0], self.SEA_STATE)
        total = np.zeros((), self.SEA_STATE)
        check(load_library().ocean_get_sea_state(self.context, sc.shape[0], sc.ctypes.data, per.ctypes.data, total.ctypes.data))
        return total, per

    @staticmethod
    def drift_params(current=(0.0, 0.0), wind=(0.0, 0.0), stokes_scale: float = 1.0, box=None, read_wake: bool = False) -> np.ndarray:
        """A 0-d DRIFT_PARAMS: box = (x0, z0, width, depth) turns the wrap on; read_wake makes the render read the wake layer."""
        p = np.zeros((), WaveGenerator.DRIFT_PARAMS)
        p["current"] = current
        p["wind"] = wind
        p["stokes_scale"] = stokes_scale
        p["flags"] = (WaveGenerator.DRIFT_WRAP if box is not None else 0) | (WaveGenerator.DRIFT_READ_WAKE if read_wake else 0)
        if box is not None:
            p["box"] = box
        return p

    def drift(self, drifters, dt: float, map_scales, params=None, render: bool = True):
        """Advance the DRIFTER rows of `drifters` by dt (include/ocean.h, ocean_drift; dt = 0 only renders) under params
        (a DRIFT_PARAMS, default drift_params()).  Returns (new drifters, instances [n][12] float32 or None without render)."""
        self._require()
        d = np.array(drifters, self.DRIFTER, copy=True).reshape(-1)
        p = self.drift_params() if params is None else np.array(params, self.DRIFT_PARAMS).reshape(())
        sc = np.ascontiguousarray(map_scales, np.float32).reshape(-1, 4)
        inst = np.zeros((len(d), 12), np.float32) if render else None
        check(load_library().ocean_drift(self.context, float(dt), p.ctypes.data, len(d), d.ctypes.data, sc.shape[0], sc.ctypes.data,
                                         None if inst is None else inst.ctypes.data))
        return d, inst

    def twiddles_to_host(self) -> np.ndarray:
        self._require()
        out = np.empty((self.map_size - 1, 2), np.float32)
        check(load_library().ocean_copy_twiddles_to_host(self.context, out.ctypes.data))
        return out

    def get_foam_state(self, cascade: int) -> np.ndarray:
        self._require()
        out = np.empty((self.map_size, self.map_size), np.float16)
        check(load_library().ocean_get_foam_state(self.context, cascade, out.ctypes.data))
        return out

    def set_foam_state(self, cascade: int, foam: np.ndarray) -> None:
        self._require()
        foam = np.ascontiguousarray(foam, np.float16)
        assert foam.shape == (self.map_size, self.map_size)
        check(load_library().ocean_set_foam_state(self.context, cascade, foam.ctypes.data))

    def timer_start(self) -> None:
        check(load_library().ocean_timer_start(self.context))

    def timer_stop(self) -> float:
        ms = C.c_float()
        check(load_library().ocean_timer_stop(self.context, C.byref(ms)))
        return ms.value

    def set_profiling(self, enable: bool = True) -> None:
        check(load_library().ocean_set_profiling(self.context, 1 if enable else 0))

    def last_kernel_times(self):
        """(spectrum_ms, rowpass_ms, colpass_ms, chunk_cascades) of the most recent launch sequence; the two
        kernel times are those of the first L2-sized chunk of `chunk_cascades` cascades."""
        a, b, c, n = C.c_float(), C.c_float(), C.c_float(), C.c_int()
        check(load_library().ocean_get_last_kernel_times(self.context, C.byref(a), C.byref(b), C.byref(c), C.byref(n)))
        return a.value, b.value, c.value, n.value
