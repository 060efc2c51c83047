"""The reference's 2-D data augmentation on the GPU: ``Segmenation_Aug`` (dataprocess/AugData.py), albumentations'
HorizontalFlip, VerticalFlip, OneOf(MotionBlur, MedianBlur, Blur), ShiftScaleRotate and RandomBrightnessContrast as
albumentations 1.1.0 composes them.

Every random draw stays on the host, from Python's global ``random`` in albumentations 1.1.0's order (and one
``np.random.RandomState`` for OneOf's pick), so a seed gives the reference's parameters and leaves ``random`` in the
reference's state.  The motion kernel (``cv2.line``), the warp matrix (``cv2.getRotationMatrix2D``, inverted with
``cv2.invertAffineTransform``) and the brightness-contrast table (numpy) are made on the host with the reference's own
calls.  The pixel work -- flips, ``cv2.filter2D`` / ``medianBlur`` / ``blur``, ``cv2.warpAffine`` and ``cv2.LUT`` --
runs in csrc/augment2d.cu, byte for byte OpenCV 4.13's, for a whole batch of images of any sizes.

    aug = Segmenation_Aug()
    out = aug.transform_compose(image=img_bgr, mask=mask)      # numpy, as albumentations' Compose
    aug.DataAugmentation("train.csv", 100, aug_path)           # the reference's BMP files, one launch per row
    x, y = aug.transform_batch(images_u8, masks_u8)            # per training step, device tensors

Documented differences: a mask whose (h, w) differs from its image raises ``ValueError`` (albumentations 1.1.0 does
not check); inputs must be uint8 (``TypeError``) with 1 or 3 channels (``ValueError``) and sides up to 8192.  The
motion kernel is divided by its sum in fp32, as albumentations 1.1.0 did with the numpy of its time (numpy 2 would
promote it to fp64).  The per-step forms of a gray image (``transform_batch``, ``InputStager(augment=...)``) give what
the reference's BGR files give when the datasets read them back with ``cv2.imread(path, 0)``, which for MotionBlur
can differ from cv2 run on the gray image itself in the last (w % 4) columns (OpenCV's scalar tail).
"""
from __future__ import annotations

import random

import numpy as np
import torch

from . import runtime
from ._abi import (AUG2D_BLUR, AUG2D_BLURS, AUG2D_HFLIP, AUG2D_LUT, AUG2D_MAX_SIDE, AUG2D_VFLIP, AUG2D_WARP,
                   aug2d_param_entry)

_ONEOF_P = [0.5, 0.25, 0.25]        # OneOf's (0.2, 0.1, 0.1), normalised
_BLURS = ("motion", "median", "box")


# ---------------------------------------------------------------------------------------------- host-only functions
def draw_params():
    """One call of the reference's Compose -> its parameters, drawn from ``random`` in albumentations 1.1.0's order:
    {"hflip", "vflip": bool, "blur": None / "motion" / "median" / "box", "kernel": fp32 k x k motion kernel or None,
    "ssr": None / (angle, scale, dx, dy), "bc": None / (alpha, beta)}"""
    d = {"hflip": False, "vflip": False, "blur": None, "kernel": None, "ssr": None, "bc": None}
    random.random()                                   # Compose(p=1) draws before it runs
    d["hflip"] = random.random() < 0.5
    d["vflip"] = random.random() < 0.5
    if random.random() < 0.2:                         # OneOf(p=0.2)
        which = int(np.random.RandomState(random.randint(0, 2 ** 32 - 1)).choice(3, p=_ONEOF_P))
        random.random()                               # the chosen member's p test, ignored under force_apply
        d["blur"] = _BLURS[which]
        if which == 0:
            d["kernel"] = _motion_kernel()
        else:
            random.choice(np.arange(3, 4, 2))         # MedianBlur / Blur ksize: a one-element choice still draws
    if random.random() < 0.2:                         # ShiftScaleRotate
        d["ssr"] = (random.uniform(-45, 45), random.uniform(-0.2 + 1.0, 0.2 + 1.0),
                    random.uniform(-0.0625, 0.0625), random.uniform(-0.0625, 0.0625))
    if random.random() < 0.2:                         # RandomBrightnessContrast
        alpha = 1.0 + random.uniform(-0.3, 0.3)
        d["bc"] = (alpha, 0.0 + random.uniform(-0.3, 0.3))
    return d


def _motion_kernel():
    import cv2
    k = int(random.choice(np.arange(3, 8, 2)))
    xs, xe = random.randint(0, k - 1), random.randint(0, k - 1)
    if xs == xe:
        ys, ye = random.sample(range(k), 2)
    else:
        ys, ye = random.randint(0, k - 1), random.randint(0, k - 1)
    kernel = np.zeros((k, k), dtype=np.uint8)
    cv2.line(kernel, (xs, ys), (xe, ye), 1, thickness=1)
    return kernel.astype(np.float32) / np.float32(kernel.sum())


def inverse_matrix(h, w, ssr):
    """ShiftScaleRotate's 2x3 matrix for an (h, w) image, inverted as warpAffine inverts it"""
    import cv2
    angle, scale, dx, dy = ssr
    m = cv2.getRotationMatrix2D((w / 2, h / 2), angle, scale)
    m[0, 2] += dx * w
    m[1, 2] += dy * h
    return cv2.invertAffineTransform(m).reshape(-1)


def brightness_table(alpha, beta):
    lut = np.arange(0, 256).astype("float32")
    if alpha != 1:
        lut *= alpha
    if beta != 0:
        lut += beta * 255
    return np.clip(lut, 0, 255).astype(np.uint8)


def kernel_taps(kernel):
    """the nonzero taps of a motion kernel in row-major order -> [(dy, dx, weight)] from the centre"""
    r = kernel.shape[0] // 2
    return [(i - r, j - r, float(kernel[i, j])) for i, j in zip(*np.nonzero(kernel))]


def param_entry(d, h, w, c, src, dst, mask_src=-1, mask_dst=0, filter_cn=None):
    """one draw for an (h, w, c) image -> (``b200seg_aug2d_param`` bytes, its stage bits)"""
    flags = (AUG2D_HFLIP if d["hflip"] else 0) | (AUG2D_VFLIP if d["vflip"] else 0)
    blur, taps, minv, lut = 0, (), None, None
    if d["blur"] is not None:
        flags |= AUG2D_BLUR
        blur = AUG2D_BLURS[d["blur"]]
        if d["blur"] == "motion":
            taps = kernel_taps(d["kernel"])
    if d["ssr"] is not None:
        flags |= AUG2D_WARP
        minv = inverse_matrix(h, w, d["ssr"])
    if d["bc"] is not None:
        flags |= AUG2D_LUT
        lut = brightness_table(*d["bc"]).tobytes()
    return aug2d_param_entry(src, dst, mask_src, mask_dst, h, w, c, flags, blur, taps, minv, lut,
                             filter_cn), flags


def check_pair(image, mask=None):
    """(h, w, c) of a uint8 image with 1 or 3 channels, and its mask's agreement; raises on anything else"""
    if image.dtype not in (np.uint8, torch.uint8):
        raise TypeError(f"Segmenation_Aug: images must be uint8, got {image.dtype}")
    shape = tuple(image.shape)
    if len(shape) == 2:
        c = 1
    elif len(shape) == 3 and shape[2] in (1, 3):
        c = shape[2]
    else:
        raise ValueError(f"Segmenation_Aug: images must be (h, w) or (h, w, c) with c in {{1, 3}}, got {shape}")
    h, w = shape[:2]
    if not (1 <= h <= AUG2D_MAX_SIDE and 1 <= w <= AUG2D_MAX_SIDE):
        raise ValueError(f"Segmenation_Aug: image sides must be in [1, {AUG2D_MAX_SIDE}], got {shape}")
    if mask is not None:
        if mask.dtype not in (np.uint8, torch.uint8):
            raise TypeError(f"Segmenation_Aug: masks must be uint8, got {mask.dtype}")
        if tuple(mask.shape) != (h, w):
            raise ValueError(f"Segmenation_Aug: the mask's shape {tuple(mask.shape)} differs from its image's {(h, w)}")
    return h, w, c


def _current_device():
    return torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")


def launch(be, src, entries, out, msrc=None, mout=None):
    """one ragged batch on the device: ``entries`` [(entry bytes, stage bits, h * w)]; src / out (and msrc / mout)
    flat uint8 device buffers at the entries' offsets"""
    table = torch.frombuffer(bytearray(b"".join(e for e, _, _ in entries)), dtype=torch.uint8)
    if src.is_cuda:
        table = table.pin_memory()
    params = table.to(src.device, non_blocking=True)
    stages = 0
    for _, f, _ in entries:
        stages |= f
    ws = be.augment2d_workspace(out.numel(), src.device) if stages & AUG2D_BLUR else None
    be.augment2d(src, params, len(entries), max(hw for _, _, hw in entries), stages, out, msrc=msrc, mout=mout, ws=ws)


# ---------------------------------------------------------------------------------------------- the augmenter
class Segmenation_Aug(object):
    """``Segmenation_Aug`` of the reference: ``transform_compose`` and ``DataAugmentation``, with the pixel work on
    the current CUDA device; ``transform_batch`` is the per-training-step form."""

    def __init__(self):
        self.aug_path = None
        self.transform_compose = self._compose

    # ------------------------------------------------------------------ reference API
    def _compose(self, image=None, mask=None, **kwargs):
        """albumentations' ``Compose(image=..., mask=...)``: numpy uint8 (h, w) or (h, w, 3) image and optional
        (h, w) mask -> {"image", "mask"} (other keys pass through)"""
        image = np.asarray(image)
        h, w, c = check_pair(image, None if mask is None else np.asarray(mask))
        out = self._run_copies(image, None if mask is None else np.asarray(mask), [draw_params()], filter_cn=c)
        res = dict(kwargs)
        res["image"] = out[0][0].reshape(image.shape)
        if mask is not None:
            res["mask"] = out[1][0]
        return res

    def DataAugmentation(self, filepath, number=100, aug_path=None):
        """the reference's offline augmentation: for each CSV row (image path, mask path), ``number`` transformed
        pairs written to aug_path/Image/{row}_{i}.bmp and aug_path/Mask/{row}_{i}.bmp; one launch per row"""
        import cv2
        import pandas as pd
        data = pd.read_csv(filepath).iloc[:, :].values
        self.aug_path = aug_path
        for index in range(data.shape[0]):
            src_image = cv2.imread(data[index][0])
            src_mask = cv2.imread(data[index][1], 0)
            check_pair(src_image, src_mask)
            draws = [draw_params() for _ in range(number)]
            images, masks = self._run_copies(src_image, src_mask, draws, filter_cn=src_image.shape[2])
            for i in range(number):
                cv2.imwrite(self.aug_path + '/Image/' + str(index) + '_' + str(i) + '.bmp', images[i])
                cv2.imwrite(self.aug_path + '/Mask/' + str(index) + '_' + str(i) + '.bmp', masks[i])

    # ------------------------------------------------------------------ per training step
    def transform_batch(self, images_u8, masks_u8=None):
        """images uint8 (N, H, W) or (N, H, W, 3) device tensors (and optional uint8 (N, H, W) masks) -> new tensors of
        the same shapes, each image with fresh draws, in one small table copy and one launch on the current stream.
        A gray batch is augmented as the reference's BGR files are read back by the 2-D datasets."""
        if images_u8.dtype != torch.uint8:
            raise TypeError(f"transform_batch: images must be uint8, got {images_u8.dtype}")
        if images_u8.dim() not in (3, 4) or (images_u8.dim() == 4 and images_u8.shape[3] != 3):
            raise ValueError(f"transform_batch: images must be (N, H, W) or (N, H, W, 3), got {tuple(images_u8.shape)}")
        n = images_u8.shape[0]
        h, w, c = check_pair(images_u8[0], None if masks_u8 is None else masks_u8[0])
        if masks_u8 is not None and tuple(masks_u8.shape) != (n, h, w):
            raise ValueError(f"transform_batch: masks must be (N, H, W) = {(n, h, w)}, got {tuple(masks_u8.shape)}")
        per = h * w * c
        entries = []
        for i in range(n):
            e, f = param_entry(draw_params(), h, w, c, i * per, i * per, -1 if masks_u8 is None else i * h * w,
                               i * h * w, filter_cn=3)
            entries.append((e, f, h * w))
        src = images_u8.contiguous()
        out = torch.empty_like(src)
        msrc = mout = None
        if masks_u8 is not None:
            msrc = masks_u8.contiguous()
            mout = torch.empty_like(msrc)
        launch(runtime.get_backend(src), src.view(-1), entries, out.view(-1),
               None if msrc is None else msrc.view(-1), None if mout is None else mout.view(-1))
        return out, mout

    # ------------------------------------------------------------------ plumbing
    @staticmethod
    def _run_copies(image, mask, draws, filter_cn):
        """one numpy image (and mask), len(draws) augmented copies -> (numpy (K, h, w[, c]), (K, h, w) or None): the
        source goes up once and every entry reads it"""
        h, w = image.shape[:2]
        c = 1 if image.ndim == 2 else image.shape[2]
        dev = _current_device()
        src = torch.from_numpy(np.ascontiguousarray(image).reshape(-1)).to(dev)
        msrc = None if mask is None else torch.from_numpy(np.ascontiguousarray(mask).reshape(-1)).to(dev)
        per = h * w * c
        entries = []
        for i, d in enumerate(draws):
            e, f = param_entry(d, h, w, c, 0, i * per, -1 if mask is None else 0, i * h * w, filter_cn=filter_cn)
            entries.append((e, f, h * w))
        out = torch.empty(len(draws) * per, dtype=torch.uint8, device=dev)
        mout = None if mask is None else torch.empty(len(draws) * h * w, dtype=torch.uint8, device=dev)
        launch(runtime.get_backend(src), src, entries, out, msrc, mout)
        images = out.cpu().numpy().reshape((len(draws),) + image.shape)
        masks = None if mout is None else mout.cpu().numpy().reshape(len(draws), h, w)
        return images, masks
