"""CPU restatement of the map-sampling contract of the reference's water shader (SURVEY 8f row f2).

TEST INFRASTRUCTURE ONLY -- the product path (godotoceanwaves_b200/csrc) never imports or calls this module.

Follows assets/shaders/spatial/water.gdshader:
  * vertex():   displacement(UV) = sum_i texture(displacements, vec3(UV*scales_i.xy, i)).xyz * scales_i.z      (:31-36)
  * fragment(): gradient/foam(UV) = sum_i mix(texture_bicubic(normals, c_i), texture(normals, c_i),
                                               min(1, ppm_i*0.1)).xyw * vec3(scales_i.ww, 1),
                ppm_i = map_size * min(scales_i.x, scales_i.y)                                               (:72-84)
  * cubic_weights / texture_bicubic                                                                           (:42-70)
with map_scales[i] = (1/tile_length.x, 1/tile_length.y, displacement_scale, normal_scale) (assets/water/water.gd:102-110).

Numeric policy (parity unpinned: the reference leaves `texture()` to the sampler hardware, whose weight precision Vulkan
does not fix): every operation is binary32, round to nearest, in the order written in the shader; `texture()` is an
exact-weight bilinear filter with REPEAT addressing,
    x = u*N - 0.5, x0 = floor(x), f = x - x0, texel indices x0 mod N and (x0+1) mod N,
    mix(mix(t00, t10, fx), mix(t01, t11, fx), fy),   mix(a, b, t) = a*(1 - t) + b*t,
on the half texels widened to binary32.  numpy float32 arithmetic rounds every operation once and never contracts, so
this file *is* the specification the CUDA kernel (compiled with -fmad=false) reproduces bit for bit.
"""
from __future__ import annotations

import numpy as np

F = np.float32


def _mix(a, b, t):
    """GLSL mix: a*(1-t) + b*t, every operation rounded to binary32."""
    return a * (F(1.0) - t) + b * t


def wrap_texel(x0: np.ndarray, N: int) -> np.ndarray:
    """REPEAT texel index x0 mod N of floor(x) = x0, defined for every binary32: x0 is clamped to [-2^62, 2^62] before
    the conversion to int64, which is exact (a binary32 of magnitude >= 2^62 is a multiple of 2^39, hence of N, and so is
    2^62); fmax sends NaN to -2^62, i.e. to texel 0."""
    lim = F(2.0 ** 62)
    return np.mod(np.fmin(np.fmax(x0, -lim), lim).astype(np.int64), N)


def texture_bilinear(tex: np.ndarray, u: np.ndarray, v: np.ndarray) -> np.ndarray:
    """tex: [N][N][4] float16 (row y, column x); u, v: float32 [n] normalised coordinates.  Returns float32 [n][4]."""
    N = tex.shape[0]
    n = F(N)
    x = u * n - F(0.5)
    y = v * n - F(0.5)
    x0 = np.floor(x)
    y0 = np.floor(y)
    fx = (x - x0)[:, None]
    fy = (y - y0)[:, None]
    ix0 = wrap_texel(x0, N)
    iy0 = wrap_texel(y0, N)
    ix1 = np.mod(ix0 + 1, N)
    iy1 = np.mod(iy0 + 1, N)
    t = tex.astype(np.float32)
    t00, t10 = t[iy0, ix0], t[iy0, ix1]
    t01, t11 = t[iy1, ix0], t[iy1, ix1]
    return _mix(_mix(t00, t10, fx), _mix(t01, t11, fx), fy)


def cubic_weights(a: np.ndarray):
    """water.gdshader:42-51."""
    a2 = a * a
    a3 = a2 * a
    w0 = -a3 + a2 * F(3.0) - a * F(3.0) + F(1.0)
    w1 = a3 * F(3.0) - a2 * F(6.0) + F(4.0)
    w2 = -a3 * F(3.0) + a2 * F(3.0) + a * F(3.0) + F(1.0)
    w3 = a3
    six = F(6.0)
    return w0 / six, w1 / six, w2 / six, w3 / six


def texture_bicubic(tex: np.ndarray, u: np.ndarray, v: np.ndarray) -> np.ndarray:
    """water.gdshader:55-70 (four bilinear taps, GPU Gems 2 ch. 20)."""
    N = tex.shape[0]
    dims = F(N)
    dims_inv = F(1.0) / dims
    ux = u * dims + F(0.5)
    vy = v * dims + F(0.5)
    flx, fly = np.floor(ux), np.floor(vy)
    fu, fv = ux - flx, vy - fly                                       # fract()
    wx0, wx1, wx2, wx3 = cubic_weights(fu)
    wy0, wy1, wy2, wy3 = cubic_weights(fv)
    gx, gy, gz, gw = wx0 + wx1, wx2 + wx3, wy0 + wy1, wy2 + wy3       # vec4(wx.xz + wx.yw, wy.xz + wy.yw)
    hx = (wx1 / gx + F(-1.5) + flx) * dims_inv
    hy = (wx3 / gy + F(0.5) + flx) * dims_inv
    hz = (wy1 / gz + F(-1.5) + fly) * dims_inv
    hw = (wy3 / gw + F(0.5) + fly) * dims_inv
    wx = (gx / (gx + gy))[:, None]
    wy = (gz / (gz + gw))[:, None]
    return _mix(_mix(texture_bilinear(tex, hy, hw), texture_bilinear(tex, hx, hw), wx),
                _mix(texture_bilinear(tex, hy, hz), texture_bilinear(tex, hx, hz), wx), wy)


def sample_maps(displacement: np.ndarray, normal: np.ndarray, points_xz: np.ndarray, map_scales: np.ndarray):
    """displacement, normal: [C][N][N][4] float16; points_xz: [n][2] world coordinates (UV = VERTEX.xz, :27);
    map_scales: [C][4] float32.  Returns (displacement [n][3], gradient_foam [n][3]) float32."""
    pts = np.ascontiguousarray(points_xz, np.float32)
    sc = np.ascontiguousarray(map_scales, np.float32)
    C, N = displacement.shape[0], displacement.shape[1]
    n = pts.shape[0]
    disp = np.zeros((n, 3), np.float32)
    grad = np.zeros((n, 3), np.float32)
    for i in range(C):
        u = pts[:, 0] * sc[i, 0]
        v = pts[:, 1] * sc[i, 1]
        disp = disp + texture_bilinear(displacement[i], u, v)[:, :3] * sc[i, 2]                     # :34-35
        ppm = F(N) * min(sc[i, 0], sc[i, 1])                                                         # :80
        t = min(F(1.0), ppm * F(0.1))
        m = _mix(texture_bicubic(normal[i], u, v), texture_bilinear(normal[i], u, v), t)            # :83
        grad = grad + m[:, [0, 1, 3]] * np.array([sc[i, 3], sc[i, 3], F(1.0)], np.float32)
    return disp, grad
