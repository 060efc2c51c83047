"""Numpy restatement of OpenCV's uint8 bilinear resize, ``cv2.resize(img, (W, H))`` with the default INTER_LINEAR, as
the reference's 2-D paths call it: the datasets (model/dataset.py:63,140,154) and the 2-D ``inference`` methods
(model/modelVNet.py:231-242,450-461, model/modelUnet.py:231-242,450-461, model/modelResNet.py:212-221,428-437).

Per axis (source size s, destination size d, destination index i):

    scale = 1.0 / (d / s)                                   fp64 (not s / d: the two can differ by an ulp)
    f     = (float)((i + 0.5) * scale - 0.5)                fp64 multiply and subtract, each rounded, then fp32
    k     = floor(f);  f = f - k                            fp32
    x axis: k < 0 -> k = 0, f = 0;  k >= s - 1 -> k = s - 1, f = 0;  taps k, min(k + 1, s - 1)
    y axis: f is not clamped; taps clamp(k, 0, s - 1), clamp(k + 1, 0, s - 1)
    c0 = rint((1 - f) * 2048), c1 = rint(f * 2048)          fp32, round half to even

Horizontal pass r = src[k] * c0 + src[k + 1] * c1 (int32); vertical pass, OpenCV's fixed-point SIMD form,
out = (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2, saturated to [0, 255].  Exact 2x downscales
(which OpenCV routes to INTER_AREA) give the same bytes under this rule.

Pinned by tests/golden/resize2d.npz (outputs of cv2 itself) and, where cv2 imports, a seeded sweep against it.
"""
from __future__ import annotations

import numpy as np


def axis_coeffs(s: int, d: int, x_axis: bool):
    """(tap0 int64 [d], tap1 int64 [d], c0 int32 [d], c1 int32 [d]) of one axis"""
    scale = 1.0 / (float(d) / float(s))
    i = np.arange(d, dtype=np.float64)
    f = ((i + 0.5) * scale - 0.5).astype(np.float32)
    k = np.floor(f)
    f = (f - k).astype(np.float32)
    k = k.astype(np.int64)
    if x_axis:
        lo, hi = k < 0, k >= s - 1
        f = np.where(lo | hi, np.float32(0.0), f).astype(np.float32)
        k = np.where(lo, 0, np.where(hi, s - 1, k))
        k0, k1 = k, np.minimum(k + 1, s - 1)
    else:
        k0, k1 = np.clip(k, 0, s - 1), np.clip(k + 1, 0, s - 1)
    c0 = np.rint((np.float32(1.0) - f) * np.float32(2048.0)).astype(np.int32)
    c1 = np.rint(f * np.float32(2048.0)).astype(np.int32)
    return k0, k1, c0, c1


def resize_u8(img: np.ndarray, dsize) -> np.ndarray:
    """``cv2.resize(img, dsize)``: uint8 (H, W) -> uint8 (dsize[1], dsize[0])"""
    img = np.asarray(img)
    assert img.dtype == np.uint8 and img.ndim == 2
    oW, oH = int(dsize[0]), int(dsize[1])
    H, W = img.shape
    x0, x1, a0, a1 = axis_coeffs(W, oW, True)
    y0, y1, b0, b1 = axis_coeffs(H, oH, False)
    src = img.astype(np.int32)
    r = src[:, x0] * a0 + src[:, x1] * a1                       # (H, oW) int32
    r0, r1 = r[y0] >> 4, r[y1] >> 4
    v = (((b0[:, None] * r0) >> 16) + ((b1[:, None] * r1) >> 16) + 2) >> 2
    return np.clip(v, 0, 255).astype(np.uint8)


def resize_u8_batch(images, dsize) -> np.ndarray:
    """a sequence of uint8 (H_n, W_n) images -> uint8 (N, dsize[1], dsize[0])"""
    return np.stack([resize_u8(im, dsize) for im in images])


def to_unit_float(v: np.ndarray) -> np.ndarray:
    """the reference's ``/ 255.`` followed by ``.float()``: fp32 (float)((double)v / 255.0)"""
    return (np.asarray(v).astype(np.float64) / 255.0).astype(np.float32)
