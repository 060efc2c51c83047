"""Write tests/golden/augment2d.npz: each pixel stage of Segmenation_Aug (dataprocess/AugData.py) on its own, computed
by cv2 (OpenCV 4.13, the version csrc/augment2d.cu matches): cv2.flip, cv2.filter2D with every motion-kernel shape
class at k = 3, 5, 7, cv2.medianBlur(3), cv2.blur((3, 3)), cv2.warpAffine (INTER_LINEAR images, INTER_NEAREST masks,
BORDER_REFLECT_101) at the ShiftScaleRotate limits and with shifts deep into the reflected border, and cv2.LUT with
tables at the brightness / contrast limits (the alpha = 1 and beta = 0 skips included).  Gray and BGR inputs, odd
sizes, 1-pixel-wide images, 512 x 512 and 700 x 1000 sources.

    python tests/golden/make_golden_augment2d.py

Keys: ``meta`` (a JSON list, one dict per case: stage, parameters, shape, and ``src``: the key of its source, shared by
the cases that filter or warp the same image, or ``None`` for the large sources, which are
``oracle.augment2d.pattern_image(*shape)``), the sources, and ``out_<i>`` per case, except that a large case records
the SHA-256 of its output bytes (``sha256``) instead.
"""
from __future__ import annotations

import json
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from oracle import augment2d as oa  # noqa: E402


def image(h, w, c, seed):
    """a patterned uint8 image with noise (edges and ramps, so every stage changes it)"""
    y, x = np.mgrid[0:h, 0:w]
    base = ((x * 7 + y * 3) ^ ((x * y) >> 4)) & 255
    chans = [(base + 53 * k) & 255 for k in range(c)]
    img = np.stack(chans, axis=-1) if c == 3 else chans[0]
    img = img + np.random.default_rng(seed).integers(0, 40, img.shape)
    return np.ascontiguousarray(np.clip(img, 0, 255).astype(np.uint8))


LINES = {            # (xs, ys, xe, ye) as fractions of k - 1: the motion kernel's shape classes
    "horizontal": (0, .5, 1, .5),
    "vertical": (.5, 0, .5, 1),
    "diagonal": (0, 0, 1, 1),
    "antidiagonal": (1, 0, 0, 1),
    "steep": (0, 0, .5, 1),
    "shallow": (0, 1, 1, .5),
    "short": (0, 0, .5, 0),
}


def main():
    cases, arrays = [], {}

    def source(src):
        """store a source once -> its key"""
        key = f"src_{sum(1 for k in arrays if k.startswith('src_'))}"
        arrays[key] = src
        return key

    def add(stage, src, out, key=None, **params):
        i = len(cases)
        if key is None and max(src.shape[:2]) >= 512:
            cases.append(dict(stage=stage, shape=list(src.shape), src=None, sha256=oa.digest(out), **params))
            return
        cases.append(dict(stage=stage, shape=list(src.shape), src=key or source(src), **params))
        arrays[f"out_{i}"] = out

    sizes = [(37, 53), (9, 1), (1, 13), (1, 1), (16, 7), (5, 2)]
    seed = 0
    # flips
    for c in (1, 3):
        for h, w in sizes[:3]:
            for hf, vf in ((1, 0), (0, 1), (1, 1)):
                seed += 1
                src = image(h, w, c, seed)
                add("flip", src, oa.flip(src, hf, vf), hflip=hf, vflip=vf)
    # motion blur: every shape class at k = 3, 5, 7, gray and BGR, the odd sizes (one source per size)
    motion_src = []
    for c in (1, 3):
        for h, w in sizes[:4] if c == 1 else sizes[:2]:
            seed += 1
            src = image(h, w, c, seed)
            motion_src.append((src, source(src)))
    for k in (3, 5, 7):
        for name, (a, b, cc, d) in LINES.items():
            xs, ys, xe, ye = (int(round(v * (k - 1))) for v in (a, b, cc, d))
            kernel = oa.motion_kernel(k, xs, ys, xe, ye)
            for src, key in motion_src:
                add("motion", src, oa.blur(src, "motion", kernel), key, k=k, line=[xs, ys, xe, ye],
                    kernel=kernel.tolist())
    # median and box blur
    for kind in ("median", "box"):
        for c in (1, 3):
            for h, w in sizes:
                seed += 1
                src = image(h, w, c, seed)
                add(kind, src, oa.blur(src, kind))
    # warps: ShiftScaleRotate's limits, and shifts far into the reflected border
    warps = [(45, 0.8, 0.0625, 0.0625), (-45, 1.2, -0.0625, -0.0625), (45, 1.2, -0.0625, 0.0625),
             (-45, 0.8, 0.0625, -0.0625), (0, 1.0, 0.0, 0.0), (13.7, 0.93, 0.031, -0.017), (-30, 0.8, 0.9, -1.7),
             (90, 1.0, 2.5, 3.25)]
    for c in (1, 3):
        for h, w in sizes + [(64, 48)]:
            seed += 1
            src = image(h, w, c, seed)
            mask = (image(h, w, 1, seed + 1000) > 128).astype(np.uint8) * 255
            key, mkey = source(src), source(mask)
            for ssr in warps:
                m = oa.ssr_matrix(h, w, *ssr)
                add("warp", src, oa.warp(src, m), key, ssr=list(ssr))
                add("warp_mask", mask, oa.warp(mask, m, nearest=True), mkey, ssr=list(ssr))
    # large sources: 512 x 512 and 700 x 1000 (both orientations)
    for h, w, c in ((512, 512, 1), (512, 512, 3), (700, 1000, 1), (1000, 700, 1)):
        src = oa.pattern_image(h, w, c)
        ssr = warps[0]
        add("warp", src, oa.warp(src, oa.ssr_matrix(h, w, *ssr)), ssr=list(ssr))
        kernel = oa.motion_kernel(7, 0, 0, 6, 3)
        add("motion", src, oa.blur(src, "motion", kernel), k=7, line=[0, 0, 6, 3], kernel=kernel.tolist())
    # tables: the alpha / beta limits and the skips
    for alpha, beta in ((0.7, 0.0), (1.3, 0.0), (1.0, 0.3), (1.0, -0.3), (0.7, -0.3), (1.3, 0.3), (1.0, 0.0),
                        (1.1234, -0.0567)):
        for c in (1, 3):
            seed += 1
            src = image(23, 31, c, seed)
            add("lut", src, cv2.LUT(src, oa.bc_table(alpha, beta)), alpha=alpha, beta=beta)
    arrays["meta"] = np.array(json.dumps(cases))
    np.savez_compressed(os.path.join(HERE, "augment2d.npz"), **arrays)
    print(len(cases), "cases")


if __name__ == "__main__":
    main()
