"""Functional CPU restatement of the reference's UNet3dthin (networks/Unet3dthin.py:6-86), test infrastructure only.

Same conventions as ``oracle.nets``: a ``state_dict``-style mapping, explicit dropout scales ``masks`` ((N, C) tensors
in module-call order, ``None`` = eval mode), autograd for the backward pass.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from .nets import _Masks, _draw, _gdr, unet_mask_channels

Tensor = torch.Tensor


def unetthin_state_spec(in_channels: int, out_channels: int, f: int = 16) -> List[Tuple[str, Tuple[int, ...]]]:
    """Names/shapes of UNet3dthin's 56 tensors in registration order (Unet3dthin.py:17-31): five encoder-side blocks,
    four decoder blocks, the 1x1x1 head; no transposed convolutions."""
    spec = []

    def block(mod, name, ci, co):                                    # Unet3dthin.py:64-86 (bias=False convs)
        spec.append((f"{mod}.{name}conv1.weight", (co, ci, 3, 3, 3)))
        spec.append((f"{mod}.{name}norm1.weight", (co,)))
        spec.append((f"{mod}.{name}norm1.bias", (co,)))
        spec.append((f"{mod}.{name}conv2.weight", (co, co, 3, 3, 3)))
        spec.append((f"{mod}.{name}norm2.weight", (co,)))
        spec.append((f"{mod}.{name}norm2.bias", (co,)))

    block("encoder1", "enc1", in_channels, f)
    block("encoder2", "enc2", f, 2 * f)
    block("encoder3", "enc3", 2 * f, 4 * f)
    block("encoder4", "enc4", 4 * f, 8 * f)
    block("bottleneck", "bottleneck", 8 * f, 16 * f)
    block("decoder4", "dec4", 16 * f, 8 * f)
    block("decoder3", "dec3", 8 * f, 4 * f)
    block("decoder2", "dec2", 4 * f, 2 * f)
    block("decoder1", "dec1", 2 * f, f)
    spec.append(("conv.weight", (out_channels, f, 1, 1, 1)))          # Unet3dthin.py:31
    spec.append(("conv.bias", (out_channels,)))
    return spec


def draw_dropout_masks_unetthin(n: int, f: int = 16, device="cpu", dtype=torch.float32) -> List[Tensor]:
    """the 18 Dropout3d draws of UNet3dthin.forward in call order: the same channel list as UNet3d's"""
    return [_draw(n, c, 3, device, dtype) for c in unet_mask_channels(f)]


def up2(x: Tensor) -> Tensor:
    """nn.Upsample(scale_factor=(2, 2, 2), mode='trilinear') of Unet3dthin.py:26 (align_corners defaults to False)"""
    return F.interpolate(x, scale_factor=(2, 2, 2), mode="trilinear")


def unetthin_forward(sd: Dict[str, Tensor], x: Tensor,
                     masks: Optional[Sequence[Tensor]] = None) -> Tuple[Tensor, Tensor]:
    """UNet3dthin.forward (Unet3dthin.py:33-62).  Returns (logits, probs)."""
    mk = _Masks(masks)

    def block(mod: str, name: str, h: Tensor) -> Tensor:
        for j in (1, 2):
            h = F.conv3d(h, sd[f"{mod}.{name}conv{j}.weight"], None, padding=1)
            h = _gdr(h, sd[f"{mod}.{name}norm{j}.weight"], sd[f"{mod}.{name}norm{j}.bias"], mk)
        return h

    enc1 = block("encoder1", "enc1", x)
    enc2 = block("encoder2", "enc2", F.max_pool3d(enc1, 2, 2))
    enc3 = block("encoder3", "enc3", F.max_pool3d(enc2, 2, 2))
    enc4 = block("encoder4", "enc4", F.max_pool3d(enc3, 2, 2))
    h = block("bottleneck", "bottleneck", F.max_pool3d(enc4, 2, 2))
    for k, enc in ((4, enc4), (3, enc3), (2, enc2), (1, enc1)):       # Unet3dthin.py:40-54
        h = up2(block(f"decoder{k}", f"dec{k}", h)) + enc
    logits = F.conv3d(h, sd["conv.weight"], sd["conv.bias"])
    probs = torch.sigmoid(logits) if logits.shape[1] == 1 else torch.softmax(logits, dim=1)
    return logits, probs
