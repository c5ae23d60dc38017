"""Specification of the wake layer's obstacles (include/ocean.h, "Wake layer", ocean_wake_set_obstacles; csrc/ocean_wake.cu's
k_wake_step_obstacles, k_wake_step_foam_obstacles and k_wake_free_surface_obstacles match it bit for bit): a world-fixed
binary mask of blocked cells that wake waves reflect from and cannot cross.

It composes oracle/wake.py, oracle/wake_foam.py and oracle/wake_coupling.py and changes none of them.  The mask is bytes
[depth][width]: row r is world cell row mz + r along z, column q world cell column mx + q along x, nonzero = blocked; every
cell outside the rectangle is open.  Window cell (i, j) of a window at origin (ox, oz) is world cell (ox + i, oz + j), and
B(i, j) says whether it is blocked, read in the window of the step call (on a scrolled first sub-step, the new window).
Per sub-step, in binary32 as the layer's specification:
    s = +0 where B, else h + phi          (the convolution reads blocked cells as it reads cells outside the window)
    h_new = +0 where B, else (a1 h - a2 h_prev) - a3 c
    F' = +0 where B, else wake_foam.update's F'                  (foam on)
    e = +0 where B, else h + phi_end                             (coupling on, the free surface of the call)
h_prev is the previous h, unmasked (on a scrolled sub-step the scrolled h).  Without a mask every operation is the layer's.
"""
from __future__ import annotations

import numpy as np

from oracle import wake
from oracle import wake_coupling
from oracle import wake_foam

f32 = np.float32
ZERO = f32(0.0)


def blocked(mask, mask_origin, window_origin, n) -> np.ndarray:
    """B [N][N] bool of the window at window_origin: the mask cells of window cells (i, j), in exact integer arithmetic."""
    out = np.zeros((n, n), bool)
    if mask is None:
        return out
    m = np.asarray(mask)
    depth, width = m.shape
    qx = int(window_origin[0]) - int(mask_origin[0])        # mask column of window column 0 (Python ints: exact)
    qz = int(window_origin[1]) - int(mask_origin[1])
    i0, i1 = max(0, -qx), min(n, width - qx)                # window columns whose mask column lies in [0, width)
    j0, j1 = max(0, -qz), min(n, depth - qz)
    if i0 < i1 and j0 < j1:
        out[j0:j1, i0:i1] = m[qz + j0:qz + j1, qx + i0:qx + i1] != 0
    return out


class Layer(wake_foam.Layer):
    """The wake layer with an obstacle mask, and with foam when `foam` (wake_foam.FOAM_PARAMS) is given.  Without a mask it
    steps as wake.Layer (no foam) or wake_foam.Layer (foam) do; with one, as the module docstring says."""

    def __init__(self, params, foam=None):
        super().__init__(params, foam)
        self.foam_on = foam is not None
        self.mask = None
        self.mask_origin = (0, 0)

    def set_obstacles(self, mask, origin=(0, 0)):
        """A copy of `mask` ([depth][width], nonzero = blocked) at world cell `origin`; None removes it."""
        self.mask = None if mask is None else (np.asarray(mask) != 0).copy()
        self.mask_origin = (int(origin[0]), int(origin[1]))
        return self

    def blocked(self, origin=None) -> np.ndarray:
        return blocked(self.mask, self.mask_origin, self.origin if origin is None else origin, self.n)

    def step(self, dt, substeps, origin, sources=None, states=None):
        if self.mask is None:
            return wake_foam.Layer.step(self, dt, substeps, origin, sources, states) if self.foam_on \
                else wake.Layer.step(self, dt, substeps, origin, sources, states)
        h = wake.substep(dt, substeps)
        assert wake.stable(self.cell_size, h)
        di, dj = int(origin[0]) - self.origin[0], int(origin[1]) - self.origin[1]
        self.h, self.h_prev = wake.scroll(self.h, di, dj), wake.scroll(self.h_prev, di, dj)
        if self.foam_on:
            self.foam = wake.scroll(self.foam, di, dj)
        self.origin = (int(origin[0]), int(origin[1]))
        B = self.blocked()
        a1, a2, a3 = wake.coefficients(self.params, h)
        rg = wake.ring(self.n, int(self.params["sponge_cells"]))
        a1, a2, a3 = a1[rg], a2[rg], a3[rg]
        g = wake.taps()
        d, gh, sh = wake_foam.constants(self.foam_params, h)
        src = np.zeros(0, wake.SOURCE) if sources is None else np.asarray(sources, wake.SOURCE).reshape(-1)
        for k in range(int(substeps)):
            tau = f32(k) * h
            phi = wake.rasterise(self.n, self.cell_size, self.origin, src, states, tau) if len(src) else np.zeros_like(self.h)
            with np.errstate(all="ignore"):
                s = np.where(B, ZERO, self.h + phi)
            c = wake.convolve(s, g)
            with np.errstate(all="ignore"):
                new = np.where(B, ZERO, (a1 * self.h - a2 * self.h_prev) - a3 * c)
            if self.foam_on:
                sigma = wake_foam.stir(self.n, self.cell_size, self.origin, src, states, tau) if len(src) else np.zeros_like(self.h)
                F = wake_foam.update(self.foam, c, sigma, self.cell_size, self.foam_params["whitecap"], d, gh, sh)
                self.foam = np.where(B, ZERO, F)
            self.h_prev, self.h = self.h, new
        return self

    def render_map(self) -> np.ndarray:
        return wake_foam.render_map(self.h, self.foam, self.cell_size) if self.foam_on else wake.render_map(self.h, self.cell_size)


def free_surface(layer: Layer, sources, states, dt, substeps) -> np.ndarray:
    """wake_coupling.free_surface, +0 on the blocked cells of the layer's window."""
    e = wake_coupling.free_surface(layer, sources, states, dt, substeps)
    return np.where(layer.blocked(), ZERO, e) if layer.mask is not None else e


def step(layer: Layer, coupling: wake_coupling.Coupling | None, dt, substeps, origin, sources=None, states=None) -> Layer:
    """wake_coupling.step of a layer with obstacles: the snapshots take the masked free surface (on a priming call, both)."""
    priming = coupling is not None and not coupling.primed
    wake_coupling.step(layer, coupling, dt, substeps, origin, sources, states)
    if coupling is not None and layer.mask is not None:
        coupling.e = free_surface(layer, sources, states, dt, substeps)
        if priming:
            coupling.e_old = coupling.e.copy()
    return layer
