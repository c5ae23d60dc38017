"""ctypes binding of libocean.so (include/ocean.h).  Fails loudly when the library is missing."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.environ.get("OCEAN_LIB") or os.path.join(_HERE, "libocean.so")   # OCEAN_LIB: A/B builds while tuning
_lib = None


class OceanError(RuntimeError):
    """Raised for every non-zero status returned by the C ABI (message = ocean_last_error())."""


class CascadeParamsC(C.Structure):
    """struct ocean_cascade_params (include/ocean.h) <- wave_cascade_parameters.gd:2-42"""
    _fields_ = [("tile_length", C.c_float * 2),
                ("displacement_scale", C.c_double), ("normal_scale", C.c_double),
                ("wind_speed", C.c_double), ("wind_direction", C.c_double), ("fetch_length", C.c_double),
                ("swell", C.c_double), ("spread", C.c_double), ("detail", C.c_double),
                ("whitecap", C.c_double), ("foam_amount", C.c_double),
                ("spectrum_seed", C.c_int32 * 2), ("should_generate_spectrum", C.c_int32),
                ("time", C.c_double), ("foam_grow_rate", C.c_double), ("foam_decay_rate", C.c_double)]


class SchedulerC(C.Structure):
    """struct ocean_scheduler (include/ocean.h) <- water.gd:51,62-63"""
    _fields_ = [("updates_per_second", C.c_double), ("time", C.c_double), ("next_update_time", C.c_double)]


class InfoC(C.Structure):
    _fields_ = [("device", C.c_int32), ("map_size", C.c_int32), ("num_cascades", C.c_int32),
                ("pending_cascades", C.c_int32), ("kernel_launches", C.c_uint64),
                ("cascade_updates", C.c_uint64), ("device_bytes", C.c_uint64)]


class RayC(C.Structure):
    """struct ocean_ray (include/ocean.h), 28 B: origin, direction (need not be unit), t_max (+inf allowed)"""
    _fields_ = [("origin", C.c_float * 3), ("direction", C.c_float * 3), ("t_max", C.c_float)]


class RayHitC(C.Structure):
    """struct ocean_ray_hit (include/ocean.h), 72 B"""
    _fields_ = [("t", C.c_float), ("position", C.c_float * 3), ("source_x", C.c_float), ("source_z", C.c_float),
                ("displacement", C.c_float * 3), ("gradient_foam", C.c_float * 3), ("gap", C.c_float), ("residual", C.c_float),
                ("status", C.c_uint32), ("evaluations", C.c_uint32), ("iterations", C.c_uint32), ("unconverged", C.c_uint32)]


class BuoyancyPointC(C.Structure):
    """struct ocean_buoyancy_point (include/ocean.h), 20 B: body-local position, volume (m^3), half height (m)"""
    _fields_ = [("position", C.c_float * 3), ("volume", C.c_float), ("half_height", C.c_float)]


class BuoyancyBodyC(C.Structure):
    """struct ocean_buoyancy_body (include/ocean.h), 56 B: 3 x 4 row-major body-to-world [R | t], hull-point range"""
    _fields_ = [("transform", C.c_float * 12), ("first_point", C.c_int32), ("num_points", C.c_int32)]


class BuoyancyResultC(C.Structure):
    """struct ocean_buoyancy_result (include/ocean.h), 48 B"""
    _fields_ = [("force", C.c_float * 3), ("torque", C.c_float * 3), ("submerged_volume", C.c_float),
                ("center_offset", C.c_float * 3), ("max_residual", C.c_float), ("unconverged", C.c_uint32)]


class BodyVelocityC(C.Structure):
    """struct ocean_body_velocity (include/ocean.h), 24 B: world-frame velocity of the body origin (m/s), angular velocity (rad/s)"""
    _fields_ = [("linear", C.c_float * 3), ("angular", C.c_float * 3)]


class DragResultC(C.Structure):
    """struct ocean_drag_result (include/ocean.h), 32 B"""
    _fields_ = [("force", C.c_float * 3), ("torque", C.c_float * 3), ("wetted_drag_area", C.c_float), ("max_relative_speed", C.c_float)]


class FloatingBodyC(C.Structure):
    """struct ocean_floating_body (include/ocean.h), 24 B: mass (kg), principal inertia (kg m^2), range into the hull points"""
    _fields_ = [("mass", C.c_float), ("inertia", C.c_float * 3), ("first_point", C.c_int32), ("num_points", C.c_int32)]


class BodyStateC(C.Structure):
    """struct ocean_body_state (include/ocean.h), 52 B: centre of mass, unit quaternion (x, y, z, w), world-frame velocities"""
    _fields_ = [("position", C.c_float * 3), ("orientation", C.c_float * 4), ("linear_velocity", C.c_float * 3),
                ("angular_velocity", C.c_float * 3)]


class SprayEmitterC(C.Structure):
    """struct ocean_spray_emitter (include/ocean.h), 88 B"""
    _fields_ = [("amount", C.c_int32), ("num_particles", C.c_int32), ("emission_transform", C.c_float * 12),
                ("particle_scale", C.c_float * 3), ("lifetime", C.c_float), ("lifetime_randomness", C.c_float),
                ("random_seed", C.c_uint32), ("emitter_lifetime", C.c_double)]


class SprayParticleC(C.Structure):
    """struct ocean_spray_particle (include/ocean.h), 120 B: TRANSFORM (3 x 4 row-major), CUSTOM, USERDATA1..3, NUMBER, flags"""
    _fields_ = [("transform", C.c_float * 12), ("custom", C.c_float * 4), ("userdata1", C.c_float * 4), ("userdata2", C.c_float * 4),
                ("userdata3", C.c_float * 4), ("number", C.c_uint32), ("flags", C.c_uint32)]


class WakeParamsC(C.Structure):
    """struct ocean_wake_params (include/ocean.h), 20 B"""
    _fields_ = [("size", C.c_int32), ("sponge_cells", C.c_int32), ("cell_size", C.c_float), ("damping", C.c_float),
                ("sponge_damping", C.c_float)]


class WakeSourceC(C.Structure):
    """struct ocean_wake_source (include/ocean.h), 28 B"""
    _fields_ = [("x", C.c_float), ("z", C.c_float), ("vx", C.c_float), ("vz", C.c_float), ("radius", C.c_float),
                ("head", C.c_float), ("body", C.c_int32)]


assert C.sizeof(WakeParamsC) == 20 and WakeParamsC.sponge_damping.offset == 16
assert C.sizeof(WakeSourceC) == 28 and WakeSourceC.body.offset == 24
assert C.sizeof(SprayEmitterC) == 88 and SprayEmitterC.emitter_lifetime.offset == 80
assert C.sizeof(SprayParticleC) == 120 and SprayParticleC.flags.offset == 116

# every symbol include/ocean.h declares: name -> (restype, argtypes)
_H = C.c_void_p
_P = C.POINTER
SIGNATURES = {
    "ocean_default_cascade_params": (C.c_int, [_P(CascadeParamsC)]),
    "ocean_create": (C.c_int, [C.c_int, C.c_int, C.c_int, _P(_H)]),
    "ocean_destroy": (C.c_int, [_H]),
    "ocean_update": (C.c_int, [_H, C.c_double, _P(CascadeParamsC), C.c_int]),
    "ocean_process": (C.c_int, [_H, _P(CascadeParamsC), C.c_int]),
    "ocean_update_all": (C.c_int, [_H, C.c_double, _P(CascadeParamsC), C.c_int]),
    "ocean_update_frames": (C.c_int, [_H, C.c_double, _P(CascadeParamsC), C.c_int, C.c_int]),
    "ocean_scheduler_init": (C.c_int, [_P(SchedulerC), C.c_double]),
    "ocean_scheduler_set_rate": (C.c_int, [_P(SchedulerC), C.c_double]),
    "ocean_scheduler_tick": (C.c_int, [_P(SchedulerC), C.c_double, _P(C.c_double)]),
    "ocean_water_frame": (C.c_int, [_H, _P(SchedulerC), C.c_double, _P(CascadeParamsC), C.c_int, _P(C.c_int)]),
    "ocean_map_scales": (C.c_int, [_P(CascadeParamsC), C.c_int, C.c_void_p]),
    "ocean_water_default_time": (C.c_double, [C.c_int]),
    "ocean_get_maps": (C.c_int, [_H, _P(C.c_void_p), _P(C.c_void_p), _P(C.c_size_t)]),
    "ocean_copy_maps_to_host": (C.c_int, [_H, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ocean_copy_maps_to_host_async": (C.c_int, [_H, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ocean_snapshot_maps_to_host_async": (C.c_int, [_H, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ocean_wait_snapshot": (C.c_int, [_H]),
    "ocean_synchronize": (C.c_int, [_H]),
    "ocean_host_alloc": (C.c_int, [_P(C.c_void_p), C.c_size_t]),
    "ocean_host_free": (C.c_int, [C.c_void_p]),
    "ocean_copy_spectrum_to_host": (C.c_int, [_H, C.c_int, C.c_void_p]),
    "ocean_set_spectrum_amplitudes": (C.c_int, [_H, C.c_int, C.c_void_p]),
    "ocean_enable_f32_taps": (C.c_int, [_H, C.c_int]),
    "ocean_copy_f32_maps_to_host": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_void_p]),
    "ocean_copy_rowpass_to_host": (C.c_int, [_H, C.c_int, C.c_void_p]),
    "ocean_copy_twiddles_to_host": (C.c_int, [_H, C.c_void_p]),
    "ocean_detmath_expf": (C.c_float, [C.c_float]),
    "ocean_debug_frame_protocol": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ocean_debug_work_queue": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]),
    "ocean_sample_maps": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ocean_sample_maps_device": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ocean_query_surface": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_float, C.c_int, C.c_void_p]),
    "ocean_query_surface_device": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_float, C.c_int, C.c_void_p]),
    "ocean_raycast": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_float, C.c_int, C.c_float, C.c_int, C.c_void_p]),
    "ocean_raycast_device": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_float, C.c_int, C.c_float, C.c_int, C.c_void_p]),
    "ocean_buoyancy": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_float, C.c_float, C.c_int,
                                 C.c_void_p, C.c_void_p]),
    "ocean_buoyancy_device": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_float, C.c_float, C.c_int,
                                        C.c_void_p, C.c_void_p]),
    "ocean_body_forces": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_float,
                                    C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ocean_body_forces_device": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                           C.c_float, C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ocean_simulate_bodies": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                        C.c_float, C.c_float, C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ocean_simulate_bodies_device": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                               C.c_float, C.c_float, C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ocean_update_velocity": (C.c_int, [_H, _P(C.c_int)]),
    "ocean_get_velocity_map": (C.c_int, [_H, _P(C.c_void_p), _P(C.c_size_t)]),
    "ocean_copy_velocity_to_host": (C.c_int, [_H, C.c_int, C.c_int, C.c_void_p]),
    "ocean_copy_f32_velocity_to_host": (C.c_int, [_H, C.c_int, C.c_void_p]),
    "ocean_sample_velocity": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "ocean_sample_velocity_device": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "ocean_spray_grid":(C.c_int, [C.c_int, C.c_void_p, C.c_void_p]),
    "ocean_extract_spray": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, _P(C.c_int)]),
    "ocean_extract_spray_device": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "ocean_default_spray_emitter": (C.c_int, [_P(SprayEmitterC)]),
    "ocean_spray_particles": (C.c_int, [_H, _P(SprayEmitterC), C.c_double, C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                        C.c_void_p, _P(C.c_int)]),
    "ocean_spray_particles_device": (C.c_int, [_H, _P(SprayEmitterC), C.c_double, C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                               C.c_void_p, C.c_void_p]),
    "ocean_wake_kernel_taps": (C.c_int, [C.c_void_p]),
    "ocean_wake_init": (C.c_int, [_H, _P(WakeParamsC)]),
    "ocean_wake_step": (C.c_int, [_H, C.c_double, C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_int, C.c_void_p]),
    "ocean_wake_step_device": (C.c_int, [_H, C.c_double, C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_int, C.c_void_p]),
    "ocean_wake_render_map": (C.c_int, [_H, C.c_void_p, C.c_void_p]),
    "ocean_sample_wake": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_void_p]),
    "ocean_sample_wake_device": (C.c_int, [_H, C.c_int, C.c_void_p, C.c_void_p]),
    "ocean_wake_get_state": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ocean_wake_set_state": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64]),
    "ocean_get_foam_state": (C.c_int, [_H, C.c_int, C.c_void_p]),
    "ocean_set_foam_state": (C.c_int, [_H, C.c_int, C.c_void_p]),
    "ocean_jonswap_alpha": (C.c_double, [C.c_double, C.c_double]),
    "ocean_jonswap_peak_angular_frequency": (C.c_double, [C.c_double, C.c_double]),
    "ocean_timer_start": (C.c_int, [_H]),
    "ocean_timer_stop": (C.c_int, [_H, _P(C.c_float)]),
    "ocean_set_profiling": (C.c_int, [_H, C.c_int]),
    "ocean_get_last_kernel_times": (C.c_int, [_H, _P(C.c_float), _P(C.c_float), _P(C.c_float), _P(C.c_int)]),
    "ocean_selftest_math": (C.c_int, [_H, _P(C.c_uint64), _P(C.c_uint64)]),
    "ocean_debug_device_math": (C.c_int, [_H, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ocean_get_info": (C.c_int, [_H, _P(InfoC)]),
    "ocean_last_error": (C.c_char_p, []),
    "ocean_version": (C.c_char_p, []),
}


def native_library_path() -> str:
    return _LIB_PATH


def load_library() -> C.CDLL:
    """Loads libocean.so from the package directory.  No fallback: a missing library is an error."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise OceanError(
                f"{_LIB_PATH} is missing: build it with `python -m godotoceanwaves_b200.build` "
                "(or __graft_entry__.build()). There is no CPU fallback.")
        lib = C.CDLL(_LIB_PATH)
        tolerant = bool(os.environ.get("OCEAN_LIB")) and os.environ.get("OCEAN_ALLOW_MISSING") == "1"   # A/B timing of OLDER builds only
        for name, (restype, argtypes) in SIGNATURES.items():
            if tolerant and not hasattr(lib, name):
                continue
            fn = getattr(lib, name)          # AttributeError if the export is missing
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
    return _lib


def check(status: int) -> None:
    if status != 0:
        msg = load_library().ocean_last_error()
        raise OceanError(f"libocean status {status}: {msg.decode() if msg else '?'}")
