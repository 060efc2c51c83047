"""voxelmorph's ``SpatialTransformer`` as the reference's ``networks/VNet3dregistration.py`` uses it (lines 6-45,
171-206), on the GPU: ``warp3d(moving_image, moving_label, ddf)`` returns what
``SpatialTransformer(vol_size)(moving_image, ddf)`` and ``SpatialTransformer(vol_size, mode="nearest")(moving_label,
ddf)`` return -- ``F.grid_sample(src, new_locs, align_corners=True)`` at the locations the reference builds from the
displacement field -- in one launch of ``csrc/warp3d.cu``, and its backward gives d loss / d ddf in one more.

Sampling positions are torch's own fp32 numbers (the reference's normalisation, then grid_sample's
unnormalisation, without FMA contraction), so the nearest-sampled label is bit-identical to torch's and the trilinear
image uses the same cells and weights.  As in torch, the nearest path passes no gradient to ``ddf``.

A displacement of +-inf or NaN puts its sample outside the volume, as does any coordinate at or beyond -2 or s + 1:
there the moved image and label are 0 and d loss / d ddf is exactly 0 (plus the addend), which is what torch's
grid_sample and its autograd give on the GPU for the same coordinates.

Differences from the reference, by design:
  * inputs must be fp32 CUDA tensors (``TypeError`` otherwise);
  * the moving image and label are data: neither may require a gradient (``ValueError``); the reference would
    propagate one into the image through grid_sample.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import runtime


def _check(moving_image: Optional[torch.Tensor], moving_label: Optional[torch.Tensor], ddf: torch.Tensor):
    if ddf.dim() != 5 or ddf.shape[1] != 3:
        raise ValueError(f"ddf must be (N, 3, D, H, W), got shape {tuple(ddf.shape)}")
    n, _, d, h, w = ddf.shape
    if min(d, h, w) < 2:
        raise ValueError(f"every spatial extent must be at least 2, got {(d, h, w)}")
    if moving_image is None and moving_label is None:
        raise ValueError("nothing to warp: moving_image and moving_label are both None")
    for name, t in (("ddf", ddf), ("moving_image", moving_image), ("moving_label", moving_label)):
        if t is None:
            continue
        if t.dtype != torch.float32:
            raise TypeError(f"{name} must be float32, got {t.dtype}")
        if t.device != ddf.device:
            raise ValueError(f"{name} is on {t.device}, ddf on {ddf.device}")
        if t is not ddf:
            if t.dim() != 5 or t.shape[0] != n or tuple(t.shape[2:]) != (d, h, w):
                raise ValueError(f"{name} must be (N, C, D, H, W) = ({n}, C, {d}, {h}, {w}), got {tuple(t.shape)}")
            if t.shape[1] < 1:
                raise ValueError(f"{name} has no channels")
            if t.requires_grad:
                raise ValueError(f"{name} requires a gradient; the warp computes d loss / d ddf only")


class _Warp3d(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ddf, moving_image, moving_label):
        be = runtime.get_backend(ddf)
        field = ddf.detach().permute(0, 2, 3, 4, 1).contiguous()      # (N, D, H, W, 3): a no-op for the head's output
        image = moving_image.detach().contiguous() if moving_image is not None else None
        label = moving_label.detach().contiguous() if moving_label is not None else None
        moved_image = torch.empty_like(image) if image is not None else None
        moved_label = torch.empty_like(label) if label is not None else None
        be.warp3d(field, image, label, moved_image, moved_label)
        ctx.save_for_backward(field, image)
        if moved_label is not None:
            ctx.mark_non_differentiable(moved_label)
        return moved_image, moved_label

    @staticmethod
    def backward(ctx, g_image, g_label):
        field, image = ctx.saved_tensors
        if image is None or g_image is None or not ctx.needs_input_grad[0]:
            return None, None, None
        be = runtime.get_backend(field)
        gddf = torch.empty_like(field)
        be.warp3d_bwd(field, image, g_image.contiguous(), None, gddf)
        return gddf.permute(0, 4, 1, 2, 3), None, None


def warp3d(moving_image: Optional[torch.Tensor], moving_label: Optional[torch.Tensor],
           ddf: torch.Tensor) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
    """(moved_image, moved_label): ``moving_image`` (N, Ci, D, H, W) sampled trilinearly and ``moving_label``
    (N, Cl, D, H, W) by nearest neighbour at grid + ``ddf`` (N, 3, D, H, W; channel i displaces axis i of D, H, W),
    zero outside the volume.  Either input may be None (its output is None).  Differentiable in ``ddf`` through the
    image only."""
    _check(moving_image, moving_label, ddf)
    return _Warp3d.apply(ddf, moving_image, moving_label)
