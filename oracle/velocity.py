"""oracle/velocity.py -- TEST INFRASTRUCTURE (not part of the product).

The velocity maps (include/ocean.h, ocean_update_velocity): ctypes front-end of their binary32 specification
(oracle/velocity_oracle.c, linked against the main oracle library so that both share the numeric modes pyoracle.set_modes
selects), a wave-generator restatement that remembers the push constants of the update that built each cascade's maps, and
an independent float64 model of the derivative on top of oracle/numpy_model.py.
"""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from . import numpy_model as nm
from . import pyoracle as po

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "velocity_oracle.c")
_LIB_PATH = os.path.join(_HERE, "libocean_velocity_oracle.so")
# oracle/Makefile's flags; the library resolves libocean_oracle.so next to itself
_CFLAGS = ["-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-mfma", "-Wall", "-Wextra"]


def build(force: bool = False) -> str:
    base = po.build()
    deps = [_SRC, base, os.path.abspath(__file__)]
    stale = (not os.path.exists(_LIB_PATH)) or any(os.path.getmtime(d) > os.path.getmtime(_LIB_PATH) for d in deps)
    if force or stale:
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else (shutil.which("gcc") or "gcc")
        tmp = f"{_LIB_PATH}.tmp{os.getpid()}"
        subprocess.run([cc, *_CFLAGS, "-o", tmp, _SRC, "-L", _HERE, "-l:libocean_oracle.so", "-Wl,-rpath,$ORIGIN", "-lm"],
                       check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        os.replace(tmp, _LIB_PATH)
    return _LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        po.lib()                      # the main oracle first: the velocity library binds to this very copy (modes, FFT)
        build()
        L = C.CDLL(_LIB_PATH)
        fp = C.POINTER(C.c_float)
        hp = C.POINTER(C.c_uint16)
        pcp = C.POINTER(po.PcSpectrumModulate)
        L.oracle_velocity_modulate.argtypes = [fp, fp, C.c_int, pcp]
        L.oracle_velocity_unpack.argtypes = [fp, hp, fp, C.c_int]
        L.oracle_velocity_update.argtypes = [fp, fp, fp, hp, fp, C.c_int, pcp]
        _lib = L
    return _lib


def velocity_maps(spectrum: np.ndarray, butterfly: np.ndarray, pcm) -> tuple:
    """oracle_velocity_update of one cascade: spectrum [N][N][4] float32 (the texture as stored), the butterfly of
    pyoracle's generator and the PcSpectrumModulate of the update that built the maps.  Returns (half bits [N][N][4]
    uint16, binary32 [N][N][4])."""
    N = spectrum.shape[0]
    vel = np.zeros((N, N, 4), np.uint16)
    f32 = np.zeros((N, N, 4), np.float32)
    buf = np.zeros((2, 4, N, N, 2), np.float32)
    lib().oracle_velocity_update(po._fp(np.ascontiguousarray(spectrum, np.float32)), po._fp(buf), po._fp(butterfly), po._hp(vel),
                                 po._fp(f32), N, C.byref(pcm))
    return vel, f32


class OracleWaveGenerator(po.OracleWaveGenerator):
    """pyoracle's restatement of wave_generator.gd plus what the velocity maps need: the push constants of the update that
    built each cascade's current maps (velocity_source) and the velocity map they define."""

    def __init__(self, map_size: int):
        super().__init__(map_size)
        self.velocity_source = {}     # cascade -> PcSpectrumModulate

    def _update(self, cascade_index: int, parameters) -> None:
        # the same push constants oracle_cascade_update receives (_update changes only the dirty flag before packing them)
        self.velocity_source[cascade_index] = po.pc_spectrum_modulate(parameters[cascade_index], cascade_index)
        super()._update(cascade_index, parameters)

    def update_all_batched(self, delta: float, parameters) -> None:
        raise NotImplementedError("use update_all: the batched CPU baseline does not record the velocity sources")

    def velocity(self, cascade: int) -> tuple:
        """(half bits [N][N][4] uint16, binary32 [N][N][4]) of one cascade, from its spectrum texture as stored now; a
        cascade whose maps were never written has a zero map."""
        pcm = self.velocity_source.get(cascade)
        if pcm is None:
            N = self.map_size
            return np.zeros((N, N, 4), np.uint16), np.zeros((N, N, 4), np.float32)
        return velocity_maps(self.spectrum[cascade], self.butterfly, pcm)


def float64_velocity(h0, h0m, N, tile_length, depth, time, phase_fp32=True):
    """The velocity fields (vx, vy, vz) [3, y, x] in float64: dh/dt = i w (h0 e^{i w t} - h0m e^{-i w t}), packed like
    numpy_model.modulate()'s first two layers and transformed by numpy_model.ifft_maps.  With phase_fp32, w and the phase
    w*time are the binary32 values of modulate(phase_fp32=True)."""
    ys, xs = np.meshgrid(np.arange(N), np.arange(N), indexing="ij")
    if phase_fp32:
        f32 = np.float32
        kvx = ((xs.astype(f32) - f32(N * 0.5)) * f32(2.0) * f32(nm.PI32) / f32(tile_length[0]))
        kvy = ((ys.astype(f32) - f32(N * 0.5)) * f32(2.0) * f32(nm.PI32) / f32(tile_length[1]))
        k = np.sqrt(kvx * kvx + kvy * kvy) + f32(1e-6)
        th = np.tanh((k * f32(depth)).astype(np.float64)).astype(f32)
        w32 = np.sqrt(f32(nm.G32) * k * th)
        phase = (w32 * f32(time)).astype(np.float64)
        w = w32.astype(np.float64)
        kux = (kvx / k).astype(np.float64)
        kuy = (kvy / k).astype(np.float64)
    else:
        kvx = (xs - N * 0.5) * 2.0 * nm.PI32 / tile_length[0]
        kvy = (ys - N * 0.5) * 2.0 * nm.PI32 / tile_length[1]
        k = np.sqrt(kvx * kvx + kvy * kvy) + 1e-6
        w = np.sqrt(nm.G32 * k * np.tanh(k * depth))
        phase = w * time
        kux, kuy = kvx / k, kvy / k
    m = np.exp(1j * phase)
    ht = 1j * w * (h0 * m - h0m * np.conj(m))
    hti = 1j * ht
    vx, vy, vz = hti * kuy, ht, hti * kux
    fields = nm.ifft_maps(np.stack([vx + 1j * vy, vz]))
    return np.stack([fields[0].real, fields[0].imag, fields[1].real])
