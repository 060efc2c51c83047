"""Functional CPU restatement of the reference networks (test infrastructure only).

Every function takes a ``state_dict``-style mapping (reference key names, App. A of
SURVEY.md) and plain tensors; autograd gives the backward pass.  Citations are to
the reference checkout (``$PYTORCHDEEPLEARING_REFERENCE``) files.

Dropout: ``nn.Dropout3d/2d(p=0.2)`` in train mode multiplies by a per-(sample, channel)
Bernoulli(0.8)/0.8 scale drawn as ``x.new_empty((N,C,1,1,1)).bernoulli_(0.8).div_(0.8)``
in module-call order (SURVEY.md section 0.5).  Here the scales are an explicit argument
``masks`` = list of ``(N, C)`` tensors in call order; ``None`` means eval mode.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor
P_DROP = 0.2          # networks/VNet3d.py:113-125 (prob=0.2), Unet3d.py:65 (prob=0.2)
GROUPS = 8            # nn.GroupNorm(8, C): VNet3d.py:9,30,50,66 ; Unet3d.py:73,82
EPS = 1e-5            # torch default GroupNorm eps


# --------------------------------------------------------------------------------------
# state_dict layouts (SURVEY.md App. A), in registration order
# --------------------------------------------------------------------------------------
def vnet3d_state_spec(image_channel: int, numclass: int, f: int = 16, dims: int = 3) -> List[Tuple[str, Tuple[int, ...]]]:
    """Names/shapes of VNet3d's 128 tensors (networks/VNet3d.py:25-127); ``dims=2``: VNet2d (networks/VNet2d.py:25-127,
    the same tree with 2-D kernels)."""
    spec: List[Tuple[str, Tuple[int, ...]]] = []

    def conv(name, co, ci, k):
        spec.append((name + ".weight", (co, ci) + (k,) * dims))
        spec.append((name + ".bias", (co,)))

    def gn(name, c):
        spec.append((name + ".weight", (c,)))
        spec.append((name + ".bias", (c,)))

    conv("in_tr.conv1", f, image_channel, 3)          # VNet3d.py:28
    conv("in_tr.conv2", f, image_channel, 1)          # VNet3d.py:29
    gn("in_tr.bn1", f)                                # VNet3d.py:30
    for name, ci, co, n in (("down_tr32", f, 2 * f, 2), ("down_tr64", 2 * f, 4 * f, 3),
                            ("down_tr128", 4 * f, 8 * f, 3), ("down_tr256", 8 * f, 16 * f, 3)):
        conv(name + ".down_conv", co, ci, 2)          # VNet3d.py:49
        gn(name + ".bn1", co)                         # VNet3d.py:50
        for i in range(n):                            # VNet3d.py:53 -> :18-22
            conv(f"{name}.ops.{i}.conv1", co, co, 3)  # VNet3d.py:8
            gn(f"{name}.ops.{i}.bn1", co)             # VNet3d.py:9
    for name, ci, co, n in (("up_tr256", 16 * f, 8 * f, 3), ("up_tr128", 8 * f, 4 * f, 3),
                            ("up_tr64", 4 * f, 2 * f, 2), ("up_tr32", 2 * f, f, 1)):
        spec.append((name + ".up_conv.weight", (ci, co) + (2,) * dims))   # ConvTranspose3d, VNet3d.py:65
        spec.append((name + ".up_conv.bias", (co,)))
        gn(name + ".bn", co)                          # VNet3d.py:66
        for i in range(n):                            # VNet3d.py:69
            conv(f"{name}.ops.{i}.conv1", co, co, 3)
            gn(f"{name}.ops.{i}.bn1", co)
        conv(name + ".conv", co, ci, 1)               # VNet3d.py:70 (registered after ops)
    conv("out_tr.conv", numclass, f, 1)               # VNet3d.py:88
    return spec


def unet_state_spec(in_channels: int, out_channels: int, dims: int, f: int = 16):
    """Names/shapes of UNet3d / UNet2d's 64 tensors (networks/Unet3d.py:17-34,65-86)."""
    k3 = (3,) * dims
    k2 = (2,) * dims
    k1 = (1,) * dims
    spec = []

    def block(mod, name, ci, co):
        spec.append((f"{mod}.{name}conv1.weight", (co, ci) + k3))   # bias=False, Unet3d.py:67-72
        spec.append((f"{mod}.{name}norm1.weight", (co,)))
        spec.append((f"{mod}.{name}norm1.bias", (co,)))
        spec.append((f"{mod}.{name}conv2.weight", (co, co) + k3))
        spec.append((f"{mod}.{name}norm2.weight", (co,)))
        spec.append((f"{mod}.{name}norm2.bias", (co,)))

    block("encoder1", "enc1", in_channels, f)
    block("encoder2", "enc2", f, 2 * f)
    block("encoder3", "enc3", 2 * f, 4 * f)
    block("encoder4", "enc4", 4 * f, 8 * f)
    block("bottleneck", "bottleneck", 8 * f, 16 * f)
    for k, c in ((4, 8 * f), (3, 4 * f), (2, 2 * f), (1, f)):
        spec.append((f"upconv{k}.weight", (2 * c, c) + k2))          # ConvTranspose, Unet3d.py:26-32
        spec.append((f"upconv{k}.bias", (c,)))
        block(f"decoder{k}", f"dec{k}", 2 * c, c)
    spec.append(("conv.weight", (out_channels, f) + k1))             # Unet3d.py:34
    spec.append(("conv.bias", (out_channels,)))
    return spec


def init_state_dict(spec, seed: int = 0, dtype=torch.float32, randomize_affine: bool = False) -> Dict[str, Tensor]:
    """``initialize_weights`` semantics (networks/__init__.py:11-26): Kaiming-normal
    (fan_in, relu gain) conv / conv-transpose weights, zero biases, GroupNorm gamma=1 beta=0.
    ``randomize_affine`` perturbs biases / gamma / beta so that tests exercise them."""
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, Tensor] = {}
    for name, shape in spec:
        if len(shape) > 1:
            fan_in = shape[1]
            for s in shape[2:]:
                fan_in *= s
            std = (2.0 / fan_in) ** 0.5
            sd[name] = torch.randn(shape, generator=g, dtype=torch.float64).mul_(std).to(dtype)
        else:
            is_gamma = name.endswith(".weight")
            base = torch.ones(shape, dtype=torch.float64) if is_gamma else torch.zeros(shape, dtype=torch.float64)
            if randomize_affine:
                base = base + 0.2 * torch.randn(shape, generator=g, dtype=torch.float64)
            sd[name] = base.to(dtype)
    return sd


# --------------------------------------------------------------------------------------
# dropout mask draws (same call order and same RNG calls as the reference modules)
# --------------------------------------------------------------------------------------
def _draw(n: int, c: int, dims: int, device, dtype) -> Tensor:
    shape = (n, c) + (1,) * dims
    return torch.empty(shape, device=device, dtype=dtype).bernoulli_(1 - P_DROP).div_(1 - P_DROP).view(n, c)


def vnet3d_mask_channels(f: int = 16) -> List[int]:
    """Channel count of each of the 34 dropout calls of VNet3d.forward, in call order."""
    ch = [f, f]                                          # VNet3d.py:36,38
    for co, n in ((2 * f, 2), (4 * f, 3), (8 * f, 3), (16 * f, 3)):
        ch += [co] * (1 + n)                             # VNet3d.py:56-57
    for co, n in ((8 * f, 3), (4 * f, 3), (2 * f, 2), (f, 1)):
        ch += [co] * (2 + n)                             # VNet3d.py:73,75,76
    return ch


def unet_mask_channels(f: int = 16) -> List[int]:
    ch = []
    for c in (f, 2 * f, 4 * f, 8 * f, 16 * f, 8 * f, 4 * f, 2 * f, f):
        ch += [c, c]
    return ch


def draw_dropout_masks_vnet3d(n: int, f: int = 16, device="cpu", dtype=torch.float32, dims: int = 3) -> List[Tensor]:
    return [_draw(n, c, dims, device, dtype) for c in vnet3d_mask_channels(f)]


def draw_dropout_masks_unet(n: int, dims: int, f: int = 16, device="cpu", dtype=torch.float32) -> List[Tensor]:
    return [_draw(n, c, dims, device, dtype) for c in unet_mask_channels(f)]


# --------------------------------------------------------------------------------------
# building blocks
# --------------------------------------------------------------------------------------
class _Masks:
    def __init__(self, masks: Optional[Sequence[Tensor]]):
        self.masks = list(masks) if masks is not None else None
        self.i = 0

    def apply(self, x: Tensor) -> Tensor:
        if self.masks is None:
            return x
        m = self.masks[self.i]
        self.i += 1
        return x * m.to(x.dtype).view(m.shape + (1,) * (x.dim() - 2))


def _gdr(x: Tensor, gamma: Tensor, beta: Tensor, mk: _Masks) -> Tensor:
    """relu(dropout(GroupNorm8(x)))  -- VNet3d.py:14 / Unet3d.py:73-75."""
    return F.relu(mk.apply(F.group_norm(x, GROUPS, gamma, beta, EPS)))


def vnet3d_forward(sd: Dict[str, Tensor], x: Tensor, masks: Optional[Sequence[Tensor]] = None,
                   f: int = 16) -> Tuple[Tensor, Tensor]:
    """VNet3d.forward (networks/VNet3d.py:129-158); a 4-D input runs VNet2d.forward (networks/VNet2d.py:129-158,
    the same graph with 2-D ops).  Returns (logits, probs)."""
    mk = _Masks(masks)
    conv3d = F.conv3d if x.dim() == 5 else F.conv2d
    convT3d = F.conv_transpose3d if x.dim() == 5 else F.conv_transpose2d
    p = "in_tr."
    # InputTransition3d.forward, VNet3d.py:34-43 (one bn1 shared by both branches)
    a = _gdr(conv3d(x, sd[p + "conv1.weight"], sd[p + "conv1.bias"], padding=1),
             sd[p + "bn1.weight"], sd[p + "bn1.bias"], mk)
    b = _gdr(conv3d(x, sd[p + "conv2.weight"], sd[p + "conv2.bias"]),
             sd[p + "bn1.weight"], sd[p + "bn1.bias"], mk)
    out16 = a + b

    def lu_stack(prefix: str, h: Tensor, n: int) -> Tensor:
        for i in range(n):                                             # VNet3d.py:13-15
            q = f"{prefix}.ops.{i}."
            h = _gdr(conv3d(h, sd[q + "conv1.weight"], sd[q + "conv1.bias"], padding=1),
                     sd[q + "bn1.weight"], sd[q + "bn1.bias"], mk)
        return h

    def down(prefix: str, h: Tensor, n: int) -> Tensor:                # VNet3d.py:55-59
        d = _gdr(conv3d(h, sd[prefix + ".down_conv.weight"], sd[prefix + ".down_conv.bias"], stride=2),
                 sd[prefix + ".bn1.weight"], sd[prefix + ".bn1.bias"], mk)
        return lu_stack(prefix, d, n) + d

    def up(prefix: str, h: Tensor, skip: Tensor, n: int) -> Tensor:    # VNet3d.py:72-80
        u = _gdr(convT3d(h, sd[prefix + ".up_conv.weight"], sd[prefix + ".up_conv.bias"], stride=2),
                 sd[prefix + ".bn.weight"], sd[prefix + ".bn.bias"], mk)
        xcat = torch.cat((u, skip), 1)
        xcat = _gdr(conv3d(xcat, sd[prefix + ".conv.weight"], sd[prefix + ".conv.bias"]),
                    sd[prefix + ".bn.weight"], sd[prefix + ".bn.bias"], mk)
        return lu_stack(prefix, xcat, n) + xcat

    out32 = down("down_tr32", out16, 2)
    out64 = down("down_tr64", out32, 3)
    out128 = down("down_tr128", out64, 3)
    out256 = down("down_tr256", out128, 3)
    out = up("up_tr256", out256, out128, 3)
    out = up("up_tr128", out, out64, 3)
    out = up("up_tr64", out, out32, 2)
    out = up("up_tr32", out, out16, 1)
    logits = conv3d(out, sd["out_tr.conv.weight"], sd["out_tr.conv.bias"])   # VNet3d.py:94
    if logits.shape[1] == 1:                                                     # VNet3d.py:95-98
        probs = torch.sigmoid(logits)
    else:
        probs = torch.softmax(logits, dim=1)
    return logits, probs


def unet_forward(sd: Dict[str, Tensor], x: Tensor, dims: int,
                 masks: Optional[Sequence[Tensor]] = None) -> Tuple[Tensor, Tensor]:
    """UNet3d.forward / UNet2d.forward (networks/Unet3d.py:36-62, Unet2d.py:36-62)."""
    mk = _Masks(masks)
    conv = F.conv3d if dims == 3 else F.conv2d
    convT = F.conv_transpose3d if dims == 3 else F.conv_transpose2d
    pool = F.max_pool3d if dims == 3 else F.max_pool2d

    def block(mod: str, name: str, h: Tensor) -> Tensor:              # Unet3d.py:65-86
        for j in (1, 2):
            h = conv(h, sd[f"{mod}.{name}conv{j}.weight"], None, padding=1)
            h = _gdr(h, sd[f"{mod}.{name}norm{j}.weight"], sd[f"{mod}.{name}norm{j}.bias"], mk)
        return h

    enc1 = block("encoder1", "enc1", x)
    enc2 = block("encoder2", "enc2", pool(enc1, 2, 2))
    enc3 = block("encoder3", "enc3", pool(enc2, 2, 2))
    enc4 = block("encoder4", "enc4", pool(enc3, 2, 2))
    h = block("bottleneck", "bottleneck", pool(enc4, 2, 2))
    for k, enc in ((4, enc4), (3, enc3), (2, enc2), (1, enc1)):
        h = convT(h, sd[f"upconv{k}.weight"], sd[f"upconv{k}.bias"], stride=2)   # Unet3d.py:44
        h = torch.cat((h, enc), dim=1)                                            # Unet3d.py:45
        h = block(f"decoder{k}", f"dec{k}", h)
    logits = conv(h, sd["conv.weight"], sd["conv.bias"])
    if logits.shape[1] == 1:
        probs = torch.sigmoid(logits)
    else:
        probs = torch.softmax(logits, dim=1)
    return logits, probs
