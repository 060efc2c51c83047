"""Forward-only inference path (SURVEY.md 8f-3): ``predict`` of the reference wrappers
(model/modelVNet.py:655-676, model/modelUnet.py:641-662) and the sliding-window ``inference_patch``
(model/modelUnet.py:707-763) on the drop-in networks.

The reference runs the net, copies the fp32 probabilities to the host and thresholds / arg-maxes them with numpy.
Here the head kernel writes the uint8 mask directly (``b200seg_head_mask``: neither logits nor probs are
materialised) and only the mask crosses PCIe (1 byte per voxel instead of 4*C).
"""
from __future__ import annotations

from typing import Sequence

import numpy as np
import torch

from . import runtime
from .engine import Engine


def _require_segmenter(model) -> None:
    if getattr(model, "_arch", None) == "resnet":
        raise TypeError(f"{type(model).__name__} is a classifier: it has no segmentation mask to predict; call the "
                        "model itself for its (N, numclass) logits, as the reference's ResNet predict does")


@torch.no_grad()
def predict_mask(model, x: torch.Tensor, out_threshold: float = 0.5) -> torch.Tensor:
    """x (N, Cin, [D,] H, W) on the model's device -> uint8 mask (N, [D,] H, W): ``(sigmoid > out_threshold) * 255``
    for a one-class head, ``argmax`` over the classes otherwise (model/modelVNet.py:668-675).  Eval-mode forward.
    Segmentation nets only: a classifier (ResNet2d / ResNet3d) raises ``TypeError``."""
    _require_segmenter(model)
    be = runtime.get_backend(x)
    eng = Engine(be, runtime.act_dtype(), model._dims)
    eng.mask_threshold = float(out_threshold)
    P = dict(zip(model._pnames, [p.detach() for _, p in model.named_parameters()]))
    xx = x.detach()
    if xx.dtype != torch.float32:
        xx = xx.float()
    mask, _ = getattr(eng, model._arch + "_forward")(P, xx, None, False)
    return mask


def predict(model, full_img, out_threshold: float = 0.5) -> np.ndarray:
    """``XModel.predict(full_img, out_threshold)`` (model/modelVNet.py:655-676): numpy image (Cin, [D,] H, W) ->
    numpy uint8 mask ([D,] H, W)."""
    _require_segmenter(model)
    dev = next(model.parameters()).device
    img = torch.as_tensor(np.ascontiguousarray(full_img)).float().unsqueeze(0).to(dev)
    was_training = model.training
    model.eval()
    try:
        mask = predict_mask(model, img, out_threshold)
    finally:
        model.train(was_training)
    return mask[0].cpu().numpy().astype(np.uint8)


def _starts(size: int, patch: int, step: int):
    """window origins along one axis: stride ``step``, the last window clamped to the volume end"""
    if size <= patch:
        return [0]
    s = list(range(0, size - patch + 1, step))
    if s[-1] != size - patch:
        s.append(size - patch)
    return s


@torch.no_grad()
def sliding_window_mask(model, image, patch_size: Sequence[int], step: Sequence[int] = None, batch: int = 4,
                        out_threshold: float = 0.5) -> np.ndarray:
    """``inference_patch`` (model/modelUnet.py:707-763) without the SimpleITK resampling around it: tile the volume
    (Cin, D, H, W) [or image (Cin, H, W)] with ``patch_size`` windows every ``step`` voxels (default: half a patch, as
    the reference), predict ``batch`` windows per forward on the device, accumulate the masks on the device and
    binarise the union (``out_mask[out_mask != 0] = 1``).  Only the final uint8 volume is copied to the host."""
    _require_segmenter(model)
    dev = next(model.parameters()).device
    vol = torch.as_tensor(np.ascontiguousarray(image)).float().to(dev)
    dims = model._dims
    if vol.dim() != dims + 1:
        raise ValueError(f"expected (Cin, {'D, ' if dims == 3 else ''}H, W), got {tuple(vol.shape)}")
    patch = tuple(int(p) for p in patch_size)
    step = tuple(int(s) for s in step) if step is not None else tuple(max(1, p // 2) for p in patch)
    sp = tuple(vol.shape[1:])
    if any(s < p for s, p in zip(sp, patch)):
        raise ValueError(f"volume {sp} is smaller than the patch {patch}")
    origins = [()]
    for size, p, s in zip(sp, patch, step):
        origins = [o + (a,) for o in origins for a in _starts(size, p, s)]
    acc = torch.zeros(sp, dtype=torch.int32, device=dev)
    was_training = model.training
    model.eval()
    try:
        for i in range(0, len(origins), batch):
            chunk = origins[i:i + batch]
            xb = torch.stack([vol[(slice(None),) + tuple(slice(a, a + p) for a, p in zip(o, patch))] for o in chunk])
            mb = predict_mask(model, xb, out_threshold)
            for o, m in zip(chunk, mb):
                acc[tuple(slice(a, a + p) for a, p in zip(o, patch))] += m.to(torch.int32)
    finally:
        model.train(was_training)
    return (acc != 0).to(torch.uint8).cpu().numpy()


__all__ = ["predict_mask", "predict", "sliding_window_mask"]
