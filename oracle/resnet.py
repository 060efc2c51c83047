"""Functional CPU restatement of the reference classifiers ``networks/ResNet3d.py`` / ``networks/ResNet2d.py`` (test
infrastructure only; same conventions as ``oracle/nets.py``: a ``state_dict``-style mapping in, autograd for the
backward, dropout scales as an explicit list of ``(N, C)`` tensors in call order, ``None`` = eval mode).

Two facts about the reference fix the semantics:
  * ``DownTransition*.__init__`` reads an undefined module global ``prob`` (ResNet3d.py:51), so the nets only build
    with ``prob`` injected; the restatement uses p = 0.2, as every other Dropout of the reference nets.
  * ``do1`` is an in-place Dropout applied to ``down`` (ResNet3d.py:54-55), so the residual ``torch.add(out, down)``
    adds the dropped tensor.  With p > 0 the reference's own backward raises (the in-place dropout overwrites what the
    in-place ReLU's backward needs); the function restated here is its train-mode forward, and its gradient is the
    exact autograd gradient of that function.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from .nets import _Masks, _draw, _gdr

Tensor = torch.Tensor

_BLOCKS = (("down_tr32", 16, 32, 2), ("down_tr64", 32, 64, 3), ("down_tr128", 64, 128, 3), ("down_tr256", 128, 256, 3))


def resnet_state_spec(image_channel: int, numclass: int, dims: int = 3) -> List[Tuple[str, Tuple[int, ...]]]:
    """Names/shapes of the 70 tensors of ResNet3d (ResNet3d.py:84-96) / ResNet2d (``dims=2``), registration order."""
    spec: List[Tuple[str, Tuple[int, ...]]] = []

    def conv(name, co, ci, k):
        spec.append((name + ".weight", (co, ci) + (k,) * dims))
        spec.append((name + ".bias", (co,)))

    def gn(name, c):
        spec.append((name + ".weight", (c,)))
        spec.append((name + ".bias", (c,)))

    conv("in_tr.conv1", 16, image_channel, 3)          # ResNet3d.py:27
    conv("in_tr.conv2", 16, image_channel, 1)          # ResNet3d.py:28
    gn("in_tr.bn1", 16)                                # ResNet3d.py:29
    for name, ci, co, n in _BLOCKS:
        conv(name + ".down_conv", co, ci, 2)           # ResNet3d.py:47
        gn(name + ".bn1", co)                          # ResNet3d.py:48
        for i in range(n):                             # ResNet3d.py:50 -> :5-21
            conv(f"{name}.ops.{i}.conv1", co, co, 3)
            gn(f"{name}.ops.{i}.bn1", co)
    spec += [("fc_layers.0.weight", (128, 256)), ("fc_layers.0.bias", (128,)),        # ResNet3d.py:93-96
             ("fc_layers.2.weight", (numclass, 128)), ("fc_layers.2.bias", (numclass,))]
    return spec


def resnet_mask_channels() -> List[int]:
    """Channel count of each of the four dropout calls of ResNet*.forward (one ``do1`` per DownTransition)."""
    return [co for _, _, co, _ in _BLOCKS]


def draw_dropout_masks_resnet(n: int, dims: int = 3, device="cpu", dtype=torch.float32) -> List[Tensor]:
    return [_draw(n, c, dims, device, dtype) for c in resnet_mask_channels()]


def resnet_forward(sd: Dict[str, Tensor], x: Tensor, dims: int, masks: Optional[Sequence[Tensor]] = None) -> Tensor:
    """ResNet3d.forward / ResNet2d.forward (ResNet3d.py:98-118).  Returns the (N, numclass) logits."""
    mk = _Masks(masks)
    nomask = _Masks(None)
    conv = F.conv3d if dims == 3 else F.conv2d
    p = "in_tr."
    # InputTransition3d.forward, ResNet3d.py:32-41 (one bn1 for both branches, no dropout)
    a = _gdr(conv(x, sd[p + "conv1.weight"], sd[p + "conv1.bias"], padding=1), sd[p + "bn1.weight"],
             sd[p + "bn1.bias"], nomask)
    b = _gdr(conv(x, sd[p + "conv2.weight"], sd[p + "conv2.bias"]), sd[p + "bn1.weight"], sd[p + "bn1.bias"], nomask)
    h = a + b
    for name, _, _, n in _BLOCKS:                                      # DownTransition3d.forward, ResNet3d.py:53-58
        d = F.relu(F.group_norm(conv(h, sd[name + ".down_conv.weight"], sd[name + ".down_conv.bias"], stride=2),
                                8, sd[name + ".bn1.weight"], sd[name + ".bn1.bias"], 1e-5))
        d = mk.apply(d)                                                # in-place do1: ``down`` itself is dropped
        o = d
        for i in range(n):
            q = f"{name}.ops.{i}."
            o = _gdr(conv(o, sd[q + "conv1.weight"], sd[q + "conv1.bias"], padding=1), sd[q + "bn1.weight"],
                     sd[q + "bn1.bias"], nomask)
        h = o + d
    pooled = h.reshape(h.shape[0], h.shape[1], -1).mean(dim=2)         # GlobalAveragePooling, ResNet3d.py:66-69
    hidden = F.relu(F.linear(pooled, sd["fc_layers.0.weight"], sd["fc_layers.0.bias"]))
    return F.linear(hidden, sd["fc_layers.2.weight"], sd["fc_layers.2.bias"])
