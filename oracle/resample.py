"""Vectorised numpy fp64 restatement of the whole-volume 3-D inference steps around the network
(XModel.inference / inference_patch, reference model/modelVNet.py:678-698, model/modelUnet.py:684-763).

SimpleITK is not available to the tests, so the two resamples are specified here rather than recorded:
``ResampleImageFilter`` with an identity transform maps output index i to the continuous input index u = i * r
(r = S_in / S_out, or new spacing / old spacing), samples only where -0.5 <= u < S_in - 0.5 on every axis (ITK's
inside-buffer rule; 0 elsewhere), and casts the fp64 sample to the input's pixel type.  ``normalize`` restates
dataprocess/utils.py:182-204 (numpy's 'linear' percentiles) and is pinned bit for bit to fixtures recorded from the
reference function itself (tests/golden/infer3d.npz).  Arrays are (D, H, W); sizes at the API are ITK (x, y, z).
"""
from __future__ import annotations

import numpy as np

_RANGE = {np.dtype(np.uint8): (0.0, 255.0), np.dtype(np.int16): (-32768.0, 32767.0),
          np.dtype(np.int32): (-2147483648.0, 2147483647.0)}


def spacing_size(size_xyz, spacing, new_spacing):
    """resize_image_itk's output size (dataprocess/utils.py:132-135): (S / (new / old)).astype(int)"""
    factor = np.array(new_spacing, float) / np.array(spacing, float)
    return tuple(int(v) for v in (np.array(size_xyz) / factor).astype(np.int64))


def size_ratio(in_zyx, out_zyx):
    """per-axis input-index step of the size form: S_in / S_out (fp64)"""
    return tuple(float(a) / float(b) for a, b in zip(in_zyx, out_zyx))


def _axis_linear(n_out, r, S):
    u = np.arange(n_out, dtype=np.float64) * r
    inside = (u >= -0.5) & (u < S - 0.5)
    i0 = np.maximum(np.floor(u), 0.0)
    d = np.maximum(u - i0, 0.0)
    i0 = np.minimum(i0, S - 1).astype(np.int64)
    i1 = np.minimum(i0 + 1, S - 1)
    return inside, i0, i1, d


def cast_pixel(v, dtype):
    """fp64 sample -> the input's pixel type (integers: clamped to the type's range, truncated toward zero) -> fp32"""
    dtype = np.dtype(dtype)
    if dtype == np.float32:
        return v.astype(np.float32)
    lo, hi = _RANGE[dtype]
    return np.trunc(np.clip(v, lo, hi)).astype(dtype).astype(np.float32)


def resample_linear_f64(vol, out_zyx, ratio_zyx):
    """the fp64 trilinear sample before the cast (0 outside the buffer)"""
    D, H, W = vol.shape
    (iz, z0, z1, dz), (iy, y0, y1, dy), (ix, x0, x1, dx) = (
        _axis_linear(n, r, S) for n, r, S in zip(out_zyx, ratio_zyx, (D, H, W)))
    v = vol.astype(np.float64)

    def g(zi, yi, xi):
        return v[zi[:, None, None], yi[None, :, None], xi[None, None, :]]

    def lerp(a, b, d):
        return a + (b - a) * d

    dx3, dy3, dz3 = dx[None, None, :], dy[None, :, None], dz[:, None, None]
    c00 = lerp(g(z0, y0, x0), g(z0, y0, x1), dx3)
    c01 = lerp(g(z0, y1, x0), g(z0, y1, x1), dx3)
    c10 = lerp(g(z1, y0, x0), g(z1, y0, x1), dx3)
    c11 = lerp(g(z1, y1, x0), g(z1, y1, x1), dx3)
    out = lerp(lerp(c00, c01, dy3), lerp(c10, c11, dy3), dz3)
    inside = iz[:, None, None] & iy[None, :, None] & ix[None, None, :]
    return np.where(inside, out, 0.0)


def resample_linear(vol, out_zyx, ratio_zyx):
    """ResampleImageFilter (linear, identity transform) -> fp32 array holding the input pixel type's values"""
    return cast_pixel(resample_linear_f64(vol, out_zyx, ratio_zyx), vol.dtype)


def truncate(x, lower, upper):
    """ConvertitkTrunctedValue's clamp (dataprocess/utils.py:158-160), fp32, upper first"""
    x = x.astype(np.float32).copy()
    x[x > np.float32(upper)] = np.float32(upper)
    x[x < np.float32(lower)] = np.float32(lower)
    return x


def meanstd_stats(x):
    """NormalizeImageFilter's statistics: mean and the N - 1 deviation from (sum x^2 - (sum x)^2 / N) / (N - 1)"""
    v = x.astype(np.float64).ravel()
    n = float(v.size)
    s1, s2 = float(np.sum(v)), float(np.sum(v * v))
    return s1 / n, float(np.sqrt((s2 - s1 * s1 / n) / (n - 1.0)))


def meanstd(x):
    mean, sd = meanstd_stats(x)
    return ((x.astype(np.float64) - mean) / sd).astype(np.float32)


def percentile_linear(sorted_vals, q):
    """np.percentile(a, q) (method 'linear') from the sorted values: vi = (n - 1) * (q / 100), numpy's _lerp"""
    n = sorted_vals.size
    vi = float(n - 1) * (q / 100.0)
    if vi >= n - 1:
        return float(sorted_vals[-1])
    prev = np.floor(vi)
    g = vi - prev
    a, b = float(sorted_vals[int(prev)]), float(sorted_vals[int(prev) + 1])
    diff = b - a
    return b - diff * (1.0 - g) if g >= 0.5 else a + diff * g


def normalize_stats(x):
    """normalize()'s (t, b, mean, std, unchanged): 5th / 95th percentiles, mean and population std of the nonzero
    clipped voxels, and whether the reference returns the clipped volume unchanged (either std is 0)"""
    s = np.sort(x.astype(np.float64).ravel())
    t, b = percentile_linear(s, 5), percentile_linear(s, 95)
    c = np.clip(x.astype(np.float64), t, b)
    nz = c[np.nonzero(c)]
    unchanged = t == b or nz.size == 0 or bool(nz.min() == nz.max())
    mean = float(np.mean(nz)) if nz.size else float("nan")
    std = float(np.std(nz)) if nz.size else float("nan")
    return t, b, mean, std, unchanged


def normalize(x):
    """dataprocess/utils.py:182-204 on an image holding integer or fp32 values, computed in fp64 (numpy's arithmetic
    for integer images) -> fp64"""
    t, b, mean, std, unchanged = normalize_stats(x)
    c = np.clip(x.astype(np.float64), t, b)
    return c if unchanged else (c - mean) / std


def _axis_nearest(n_out, r, S):
    u = np.arange(n_out, dtype=np.float64) * r
    inside = (u >= -0.5) & (u < S - 0.5)
    k = np.minimum(np.floor(u + 0.5), S - 1)
    return inside, np.where(inside, k, 0).astype(np.int64)


def resample_nearest(src, ratio_zyx, valid_zyx, out_zyx):
    """NN resample (index = floor(u + 0.5), RoundHalfIntegerUp) of src onto a (valid) grid, placed in the corner of a
    zero (out) array: inference_patch's crop / pad (modelUnet.py:752-757).  Keeps src's dtype."""
    out = np.zeros(out_zyx, dtype=src.dtype)
    vz, vy, vx = (min(v, o) for v, o in zip(valid_zyx, out_zyx))
    (iz, kz), (iy, ky), (ix, kx) = (_axis_nearest(n, r, S) for n, r, S in zip((vz, vy, vx), ratio_zyx, src.shape))
    val = src[kz[:, None, None], ky[None, :, None], kx[None, None, :]]
    inside = iz[:, None, None] & iy[None, :, None] & ix[None, None, :]
    out[:vz, :vy, :vx] = np.where(inside, val, 0)
    return out


def integer_boundary_points(vol, out_zyx, ratio_zyx, tol=1e-9):
    """count of samples whose fp64 value lies within tol of an integer (where the cast's truncation can flip under a
    different rounding of the same formula)"""
    v = resample_linear_f64(vol, out_zyx, ratio_zyx)
    return np.abs(v - np.round(v)) <= tol


def window_origins(size, patch):
    """inference_patch's window origins along one axis (modelUnet.py:719-736): loop index x over range(0, S, p // 2),
    origin x * p, clamped to S - p where the window would end past the volume"""
    out = []
    for x in range(0, size, patch // 2):
        o = x * patch if (x + 1) * patch <= size else size - patch
        if o not in out:
            out.append(o)
    return sorted(out)
