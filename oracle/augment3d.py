"""Numpy fp64 restatement of the reference's 3-D augmentation warp (``ImageDataGenerator3D.random_transform`` and
``standardize``, dataprocess/Augmentation/images_masks_3dtransform.py), written from scipy's observed behaviour.

The warp is ``scipy.ndimage.affine_transform(v, M, off, order=0, mode=fill_mode, cval=cval)`` per channel.  For the
output index (i0, i1, i2) and each input axis h of length n:

    cc = off[h];  cc += M[h, 0] * i0;  cc += M[h, 1] * i1;  cc += M[h, 2] * i2      every product and sum rounded

(summing the products first changes the index on ties).  cc then goes through the mode's coordinate map, which only
acts when cc lies outside [0, n - 1] (S = the period, trunc = truncation toward zero, all arithmetic fp64):

    nearest    cc < 0 -> 0;  cc > n - 1 -> n - 1
    constant   outside -> cval for the whole voxel (so -0.4999 is outside, n - 0.5 is inside)
    reflect    S = 2n.  cc < 0: if cc < -S: cc += S * trunc(-cc / S); then cc < -n ? cc + S : (cc > -1e-15 ? 1e-15 : -cc) - 1
               cc > n - 1: cc -= S * trunc(cc / S); if cc >= n: cc = S - cc - 1
    mirror     S = 2n - 2.  cc < 0: cc += S * trunc(-cc / S); then cc <= 1 - n ? cc + S : -cc
               cc > n - 1: cc -= S * trunc(cc / S); if cc >= n: cc = S - cc
    wrap       S = n - 1 (the old period).  cc < 0: cc += S * (trunc(-cc / S) + 1);  cc > n - 1: cc -= S * trunc(cc / S)

(n == 1: reflect, mirror and wrap give 0).  The index is k = floor(cc + 0.5); a k outside [0, n - 1] (the mapped cc
can still round up to n, or down to -1) is folded back as scipy folds spline taps that leave the array: 'reflect'
repeats the edge voxel (-1 -> 0, n -> n - 1), 'mirror' reflects about it (n -> n - 2); 'nearest', 'constant' and
'wrap' never produce such an index.  Pinned bit for bit against ``scipy.ndimage.affine_transform`` by
tests/test_augment3d_cpu.py.

After the warp (steps 3-5 of the reference): the channel shift clip(x_c + u_c, min, max) in fp32, min / max over every
channel of the warped sample; the flips; ``x *= rescale`` (fp32 multiply by fp32(rescale) for a Python number, fp64
multiply rounded once to fp32 for a numpy float64).
"""
from __future__ import annotations

import numpy as np

MODES = ("nearest", "constant", "reflect", "wrap", "mirror")


def _fold_index(k: np.ndarray, n: int, mode: str) -> np.ndarray:
    """an index one step outside [0, n - 1] folded back: 'reflect' repeats the edge voxel, 'mirror' reflects about
    it"""
    if n <= 1:
        return np.zeros_like(k)
    e = 1 if mode == "reflect" else 0
    return np.where(k < 0, -e - k, 2 * n - 2 + e - k)


def map_axis(cc: np.ndarray, n: int, mode: str):
    """fp64 source coordinates along one axis of length n -> (int64 index, inside mask).  inside is False only for
    'constant' outside [0, n - 1]."""
    cc = np.array(cc, dtype=np.float64, copy=True)
    inside = np.ones(cc.shape, dtype=bool)
    lo, hi = cc < 0, cc > n - 1
    if mode == "nearest":
        cc[lo] = 0.0
        cc[hi] = float(n - 1)
    elif mode == "constant":
        inside = ~(lo | hi)
        cc[~inside] = 0.0
    elif n <= 1:
        cc[lo | hi] = 0.0
    elif mode == "reflect":
        s2 = float(2 * n)
        t = cc[lo]
        far = t < -s2
        t[far] = s2 * np.trunc(-t[far] / s2) + t[far]
        t = np.where(t < -n, t + s2, np.where(t > -1e-15, 1e-15, -t) - 1.0)
        cc[lo] = t
        t = cc[hi]
        t = t - s2 * np.trunc(t / s2)
        cc[hi] = np.where(t >= n, s2 - t - 1.0, t)
    elif mode == "mirror":
        s2 = float(2 * n - 2)
        t = cc[lo]
        t = s2 * np.trunc(-t / s2) + t
        cc[lo] = np.where(t <= 1 - n, t + s2, -t)
        t = cc[hi]
        t = t - s2 * np.trunc(t / s2)
        cc[hi] = np.where(t >= n, s2 - t, t)
    elif mode == "wrap":
        sz = float(n - 1)
        t = cc[lo]
        cc[lo] = t + sz * (np.trunc(-t / sz) + 1.0)
        t = cc[hi]
        cc[hi] = t - sz * np.trunc(t / sz)
    else:
        raise ValueError(f"unknown mode {mode!r}")
    k = np.floor(cc + 0.5).astype(np.int64)
    bad = (k < 0) | (k >= n)
    if bad.any():
        k[bad] = _fold_index(k[bad], n, mode)
    return k, inside


def source_coords(matrix: np.ndarray, offset: np.ndarray, shape):
    """scipy's per-axis source coordinate, fp64, in its order of operations: three (D, H, W) arrays"""
    m = np.asarray(matrix, dtype=np.float64)
    off = np.asarray(offset, dtype=np.float64)
    i0, i1, i2 = np.meshgrid(*(np.arange(s, dtype=np.float64) for s in shape), indexing="ij")
    out = []
    for h in range(3):
        cc = np.full(tuple(shape), off[h])
        cc = cc + m[h, 0] * i0
        cc = cc + m[h, 1] * i1
        cc = cc + m[h, 2] * i2
        out.append(cc)
    return out


def warp_indices(matrix, offset, shape, mode):
    """-> (k0, k1, k2, inside) int64 / bool (D, H, W) arrays of the order-0 gather"""
    coords = source_coords(matrix, offset, shape)
    ks, inside = [], np.ones(tuple(shape), dtype=bool)
    for h in range(3):
        k, ok = map_axis(coords[h], int(shape[h]), mode)
        ks.append(k)
        inside &= ok
    return ks[0], ks[1], ks[2], inside


def affine_order0(v: np.ndarray, matrix, offset, mode="nearest", cval=0.0) -> np.ndarray:
    """``scipy.ndimage.affine_transform(v, matrix, offset, order=0, mode=mode, cval=cval)`` for a 3-D fp32 / fp64 /
    uint8 array (output of v's dtype)"""
    v = np.asarray(v)
    k0, k1, k2, inside = warp_indices(matrix, offset, v.shape, mode)
    out = v[k0, k1, k2]
    if not inside.all():
        out = out.copy()
        out[~inside] = fill_value(cval, v.dtype)
    return out


def fill_value(cval, dtype):
    """scipy's cval written to an output of ``dtype``: floats take it as is; unsigned integers round half up from 0
    and saturate (scipy's output cast); signed integers round half away from zero"""
    dtype = np.dtype(dtype)
    if dtype.kind == "f":
        return dtype.type(cval)
    c = float(cval)
    info = np.iinfo(dtype)
    if dtype.kind == "u":
        t = c + 0.5 if c > 0 else 0.0
    else:
        t = c + 0.5 if c > 0 else c - 0.5
    t = min(max(t, float(info.min)), float(info.max))
    return dtype.type(int(t))


def channel_shift(x: np.ndarray, shifts) -> np.ndarray:
    """clip(x_c + u_c, min(x), max(x)) in fp32 over the last axis of a (D, H, W, C) fp32 sample; u_c Python floats"""
    lo, hi = np.min(x), np.max(x)
    return np.stack([np.clip(x[..., c] + np.float32(u), lo, hi) for c, u in enumerate(shifts)], axis=-1)


def rescale_sample(x: np.ndarray, rescale) -> np.ndarray:
    """``standardize``'s ``x *= rescale`` on an fp32 sample"""
    if not rescale:
        return x
    if np.result_type(np.float32, rescale) == np.float64:
        return (x.astype(np.float64) * np.float64(rescale)).astype(np.float32)
    return (x * np.float32(rescale)).astype(np.float32)


def transform_sample(x, y, matrix4, mode="nearest", cval=0.0, shifts=None, flips=(False, False, False),
                     rescale=None):
    """the whole chain on one sample: x fp32 (D, H, W, C), y (D, H, W, Cy) of any dtype, matrix4 the centred 4x4
    matrix; flips are (axis 0, axis 1, axis 2).  Returns (x fp32, y of y's dtype); rescale is applied only when given
    (``standardize``, the flow path)."""
    m4 = np.asarray(matrix4, dtype=np.float64)
    mat, off = m4[:3, :3], m4[:3, 3]
    x = np.asarray(x)
    y = np.asarray(y)
    xo = np.stack([affine_order0(x[..., c], mat, off, mode, cval) for c in range(x.shape[-1])], axis=-1)
    yo = np.stack([affine_order0(y[..., c], mat, off, mode, cval) for c in range(y.shape[-1])], axis=-1)
    if shifts is not None:
        xo = channel_shift(xo, shifts)
    for axis, f in enumerate(flips):
        if f:
            xo = np.flip(xo, axis)
            yo = np.flip(yo, axis)
    xo = rescale_sample(np.ascontiguousarray(xo), rescale)
    return np.ascontiguousarray(xo), np.ascontiguousarray(yo)


def warp_batch(x, y, entries, mode="nearest", cval=0.0, shift=False, rescale=None, label_out=None):
    """the device launch restated: x fp32 (N, D, H, W, C), y uint8 / fp32 (N, D, H, W), ``entries`` one
    (3x3 block (9 values, row-major), offset[3], fp32 channel shifts, flip bits) per sample; ``rescale`` as numpy would
    take it (a Python float multiplies in fp32, a numpy float64 in fp64).  label_out None keeps y's dtype, "int64"
    widens (fp32 truncated toward zero), "binary" is int64 (y != 0)."""
    x = np.asarray(x, dtype=np.float32)
    y = np.asarray(y)
    xo, yo = np.empty_like(x), np.empty(y.shape, dtype=y.dtype)
    for s, (m, off, shifts, flip) in enumerate(entries):
        m4 = np.eye(4)
        m4[:3, :3] = np.asarray(m, dtype=np.float64).reshape(3, 3)
        m4[:3, 3] = off
        flips = tuple(bool(int(flip) >> a & 1) for a in range(3))
        xs, ys = transform_sample(x[s], y[s][..., None], m4, mode, cval, list(shifts) if shift else None, flips,
                                  rescale)
        xo[s], yo[s] = xs, ys[..., 0]
    if label_out == "binary":
        return xo, (yo != 0).astype(np.int64)
    if label_out == "int64":
        return xo, (np.trunc(yo).astype(np.int64) if yo.dtype.kind == "f" else yo.astype(np.int64))
    return xo, yo
