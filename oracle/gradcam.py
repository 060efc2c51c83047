"""fp64 restatement of the reference's Grad-CAM map (model/visualization.py:146-193, steps after the hooks) and a
ResNet2d forward that keeps the stage outputs (test infrastructure only).

Given the hooked activations A and gradients g of each target stage ((N, C, h, w), forward order):
  w = mean_{h,w} g;  cam = max(sum_c w_c A_c, 0);  s = (cam - min) / (1e-7 + max(cam - min)) per image;
  resize s to (H, W) with OpenCV's INTER_LINEAR coefficients (computed exactly as OpenCV does, in float32);
  m = mean over the stages;  result = (m - min) / (1e-7 + max(m - min)) per image.
Every operation after the coefficients is fp64."""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from .nets import _Masks, _gdr
from .resnet import _BLOCKS

STAGES = ("in_tr",) + tuple(b[0] for b in _BLOCKS)


def cv_linear_coeffs(dst: int, src: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """OpenCV's INTER_LINEAR taps along one axis: (first source index, second source index, float32 weights (dst, 2))"""
    scale = 1.0 / (dst / src)
    i0 = np.zeros(dst, np.int64)
    a = np.zeros((dst, 2), np.float32)
    for d in range(dst):
        fx = np.float32((d + 0.5) * scale - 0.5)
        s = int(np.floor(fx))
        fx = np.float32(fx - np.float32(s))
        if s < 0:
            fx, s = np.float32(0), 0
        if s >= src - 1:
            fx, s = np.float32(0), src - 1
        i0[d] = s
        a[d] = (np.float32(1) - fx, fx)
    return i0, np.minimum(i0 + 1, src - 1), a


def resize_linear(img: np.ndarray, H: int, W: int) -> np.ndarray:
    """cv2.resize(img, (W, H)) of one (h, w) image in fp64 arithmetic (a same-size resize is a copy)"""
    h, w = img.shape
    if (h, w) == (H, W):
        return img.astype(np.float64)
    x0, x1, ax = cv_linear_coeffs(W, w)
    y0, y1, ay = cv_linear_coeffs(H, h)
    src = img.astype(np.float64)
    ax, ay = ax.astype(np.float64), ay.astype(np.float64)
    rows = src[:, x0] * ax[:, 0] + src[:, x1] * ax[:, 1]
    return rows[y0] * ay[:, :1] + rows[y1] * ay[:, 1:]


def _scale(img: np.ndarray) -> np.ndarray:
    img = img - img.min()
    return img / (1e-7 + img.max())


def grad_cam_map(acts: Sequence[np.ndarray], grads: Sequence[np.ndarray], H: int, W: int) -> np.ndarray:
    """(N, H, W) fp64 map from the stages' A and g ((N, C, h, w) each, forward order)"""
    per = []
    for a, g in zip(acts, grads):
        a, g = np.asarray(a, np.float64), np.asarray(g, np.float64)
        w = g.mean(axis=(2, 3))
        cam = np.maximum(np.einsum("nc,nchw->nhw", w, a), 0.0)
        per.append(np.stack([resize_linear(_scale(c), H, W) for c in cam]))
    m = np.mean(np.stack(per, axis=1), axis=1)
    return np.stack([_scale(i) for i in m])


def resnet2d_stages(sd: Dict[str, torch.Tensor], x: torch.Tensor) -> Tuple[torch.Tensor, List[torch.Tensor]]:
    """ResNet2d.forward in eval mode (as ``oracle.resnet.resnet_forward``) -> (logits, [output of each of STAGES])"""
    nomask = _Masks(None)
    p = "in_tr."
    a = _gdr(F.conv2d(x, sd[p + "conv1.weight"], sd[p + "conv1.bias"], padding=1), sd[p + "bn1.weight"],
             sd[p + "bn1.bias"], nomask)
    b = _gdr(F.conv2d(x, sd[p + "conv2.weight"], sd[p + "conv2.bias"]), sd[p + "bn1.weight"], sd[p + "bn1.bias"], nomask)
    h = a + b
    outs = [h]
    for name, _, _, n in _BLOCKS:
        d = F.relu(F.group_norm(F.conv2d(h, sd[name + ".down_conv.weight"], sd[name + ".down_conv.bias"], stride=2),
                                8, sd[name + ".bn1.weight"], sd[name + ".bn1.bias"], 1e-5))
        o = d
        for i in range(n):
            q = f"{name}.ops.{i}."
            o = _gdr(F.conv2d(o, sd[q + "conv1.weight"], sd[q + "conv1.bias"], padding=1), sd[q + "bn1.weight"],
                     sd[q + "bn1.bias"], nomask)
        h = o + d
        outs.append(h)
    pooled = h.mean(dim=(2, 3))
    hidden = F.relu(F.linear(pooled, sd["fc_layers.0.weight"], sd["fc_layers.0.bias"]))
    return F.linear(hidden, sd["fc_layers.2.weight"], sd["fc_layers.2.bias"]), outs


def stage_grads(sd: Dict[str, torch.Tensor], x: torch.Tensor, target, layers: Sequence[str]):
    """(A, g) of each stage in ``layers`` (forward order) for d(sum_i logit[i, t_i]); ``target`` None: each row's
    arg-max.  Runs in x's dtype and device.  -> ([A], [g], classes)"""
    with torch.enable_grad():
        logits, outs = resnet2d_stages(sd, x.detach().requires_grad_(True))
        t = logits.argmax(1) if target is None else torch.full((x.shape[0],), int(target), dtype=torch.int64,
                                                               device=x.device)
        idx = [STAGES.index(s) for s in layers]
        gs = torch.autograd.grad(logits.gather(1, t[:, None]).sum(), [outs[i] for i in idx])
    return [outs[i].detach() for i in idx], list(gs), t
