"""Restatement of the reference's 2-D augmentation (``Segmenation_Aug``, dataprocess/AugData.py) as albumentations 1.1.0
runs it, with every pixel stage applied by cv2 itself.

``Segmenation_Aug`` composes HorizontalFlip(0.5), VerticalFlip(0.5), OneOf([MotionBlur(0.2), MedianBlur(3, 0.1),
Blur(3, 0.1)], 0.2), ShiftScaleRotate(0.0625, 0.2, 45, 0.2) and RandomBrightnessContrast(0.3, 0.3, 0.2).  In
albumentations 1.1.0 every draw comes from Python's global ``random``, in call order:

    Compose          random() (against p = 1)
    each transform   random() < p, drawn before force_apply is looked at; then its get_params() when it applies
    OneOf            random() < 0.2; then np.random.RandomState(randint(0, 2**32 - 1)).choice(3, p=[.5, .25, .25]),
                     and the member is called with force_apply=True (it still draws its own random())
    MotionBlur       k = choice(arange(3, 8, 2)); xs, xe = randint(0, k - 1) x 2; ys, ye = sample(range(k), 2) when
                     xs == xe, else randint(0, k - 1) x 2; cv2.line(uint8 k x k, (xs, ys), (xe, ye), 1, 1), fp32,
                     divided by its sum (fp32, as numpy < 1.20 computed it)
    Median / Blur    choice(arange(3, 4, 2)) (one draw for a one-element choice)
    ShiftScaleRotate uniform(-45, 45), uniform(0.8, 1.2), uniform(-.0625, .0625) for dx, then for dy
    BrightnessContr. alpha = 1 + uniform(-.3, .3), beta = 0 + uniform(-.3, .3)

The mask (``cv2.imread(path, 0)`` in the reference) takes the flips and the warp (INTER_NEAREST) only.  Not verified
against albumentations itself, which is not a dependency of the project; DESIGN.md section 2 lists what rests on this reading.
"""
from __future__ import annotations

import hashlib
import random

import cv2
import numpy as np

ONEOF_P = (0.5, 0.25, 0.25)          # (0.2, 0.1, 0.1) normalised, as OneOf does
BLURS = ("motion", "median", "box")


def motion_kernel(k, xs, ys, xe, ye):
    kernel = np.zeros((k, k), dtype=np.uint8)
    cv2.line(kernel, (xs, ys), (xe, ye), 1, thickness=1)
    return kernel.astype(np.float32) / np.float32(kernel.sum())


def draw():
    """one call of the Compose -> its parameters, drawn from ``random`` in albumentations 1.1.0's order"""
    d = {"hflip": False, "vflip": False, "blur": None, "kernel": None, "ssr": None, "bc": None}
    random.random()                                   # Compose, p = 1
    d["hflip"] = random.random() < 0.5
    d["vflip"] = random.random() < 0.5
    if random.random() < 0.2:                         # OneOf
        which = int(np.random.RandomState(random.randint(0, 2 ** 32 - 1)).choice(3, p=list(ONEOF_P)))
        random.random()                               # the member's own p test (force_apply=True)
        d["blur"] = BLURS[which]
        if which == 0:
            k = int(random.choice(np.arange(3, 8, 2)))
            xs, xe = random.randint(0, k - 1), random.randint(0, k - 1)
            if xs == xe:
                ys, ye = random.sample(range(k), 2)
            else:
                ys, ye = random.randint(0, k - 1), random.randint(0, k - 1)
            d["kernel"] = motion_kernel(k, xs, ys, xe, ye)
        else:
            random.choice(np.arange(3, 4, 2))
    if random.random() < 0.2:                         # ShiftScaleRotate
        angle = random.uniform(-45, 45)
        scale = random.uniform(-0.2 + 1.0, 0.2 + 1.0)
        dx = random.uniform(-0.0625, 0.0625)
        dy = random.uniform(-0.0625, 0.0625)
        d["ssr"] = (angle, scale, dx, dy)
    if random.random() < 0.2:                         # RandomBrightnessContrast
        alpha = 1.0 + random.uniform(-0.3, 0.3)
        beta = 0.0 + random.uniform(-0.3, 0.3)
        d["bc"] = (alpha, beta)
    return d


def ssr_matrix(h, w, angle, scale, dx, dy):
    m = cv2.getRotationMatrix2D((w / 2, h / 2), angle, scale)
    m[0, 2] += dx * w
    m[1, 2] += dy * h
    return m


def bc_table(alpha, beta):
    lut = np.arange(0, 256).astype("float32")
    if alpha != 1:
        lut *= alpha
    if beta != 0:
        lut += beta * 255
    return np.clip(lut, 0, 255).astype(np.uint8)


# ---------------------------------------------------------------------------------------------- one stage each
def flip(img, h, v):
    if h:
        img = np.ascontiguousarray(img[:, ::-1])
    if v:
        img = np.ascontiguousarray(img[::-1])
    return img


def blur(img, kind, kernel=None):
    if kind == "motion":
        return cv2.filter2D(img, -1, kernel)
    if kind == "median":
        return cv2.medianBlur(img, 3)
    return cv2.blur(img, (3, 3))


def warp(img, m, nearest=False):
    h, w = img.shape[:2]
    return cv2.warpAffine(img, m, (w, h), flags=cv2.INTER_NEAREST if nearest else cv2.INTER_LINEAR,
                          borderMode=cv2.BORDER_REFLECT_101)


def apply(d, image, mask=None):
    """the drawn stages on one uint8 image ((h, w) or (h, w, 3)) and its optional (h, w) mask -> (image, mask)"""
    image = flip(image, d["hflip"], d["vflip"])
    mask = None if mask is None else flip(mask, d["hflip"], d["vflip"])
    if d["blur"] is not None:
        image = blur(image, d["blur"], d["kernel"])
    if d["ssr"] is not None:
        m = ssr_matrix(image.shape[0], image.shape[1], *d["ssr"])
        image = warp(image, m)
        mask = None if mask is None else warp(mask, m, nearest=True)
    if d["bc"] is not None:
        image = cv2.LUT(image, bc_table(*d["bc"]))
    return image, mask


def compose(image, mask=None):
    """``transform_compose(image=..., mask=...)``: draw, then apply"""
    return apply(draw(), image, mask)


def as_bgr_gray(image, d):
    """a gray image augmented as the reference's BGR file path does (gray-valued BGR, read back with
    ``cv2.imread(path, 0)``, which returns channel 0 for gray-valued pixels)"""
    out, _ = apply(d, np.repeat(image[..., None], 3, axis=2))
    return np.ascontiguousarray(out[..., 0])


def pattern_image(h, w, c):
    """the deterministic large fixture source: ramps and a checkerboard of 37 x 29 cells, c channels offset by 53"""
    y, x = np.mgrid[0:h, 0:w]
    base = (x // 2 + y // 3 + 96 * ((x // 37 + y // 29) % 2)) & 255
    chans = [((base + 53 * k) & 255).astype(np.uint8) for k in range(c)]
    return np.ascontiguousarray(np.stack(chans, axis=-1) if c == 3 else chans[0])


def digest(a):
    """SHA-256 of an output's bytes, how the fixture records its large outputs"""
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
