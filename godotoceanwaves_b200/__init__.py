"""godotoceanwaves_b200 -- H100-native drop-in for the wave-generation hot path of
2Retr0/GodotOceanWaves (spectrum -> time propagation -> packed inverse FFTs -> maps).

The product is the CUDA library ``libocean.so`` (C ABI in ``include/ocean.h``); this package is
the Python host-side mirror of the reference's GDScript interface for that path:

  WaveCascadeParameters  <- assets/water/wave_cascade_parameters.gd
  WaveGenerator          <- assets/water/wave_generator.gd
  Water                  <- assets/water/water.gd (scheduler, start times, map_scales, texture hand-off)
  RenderingContext.create_push_constant <- assets/render_context.gd:122-135

There is no CPU fallback: importing works anywhere, but creating a generator without the
compiled extension or without an sm_90 GPU (H100) raises ``OceanError``.
"""
from .native import OceanError, load_library, native_library_path  # noqa: F401
from .render_context import RenderingContext  # noqa: F401
from .wave_cascade_parameters import WaveCascadeParameters  # noqa: F401
from .wave_generator import DEPTH, G, WaveGenerator  # noqa: F401
from .water import Water  # noqa: F401

__all__ = ["WaveCascadeParameters", "WaveGenerator", "Water", "RenderingContext", "OceanError", "load_library",
           "native_library_path", "G", "DEPTH"]
