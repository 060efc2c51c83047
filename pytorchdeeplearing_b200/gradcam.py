"""Grad-CAM of the drop-in ResNet2d (reference model/visualization.py:65-238, ``GradCAM``, called by
``MutilResNet2dModel.Grad_CAM_Visual``, model/modelResNet.py:419-426) on the GPU.

One eval-mode forward keeps the stage outputs; the backward of d(sum_i logit[i, t_i]) computes data gradients only
and stops after the earliest target stage (``Engine.resnet_backward(..., stages=...)``); the CAM -- channel weights,
weighted sum, clamp, min-max scale, OpenCV-rule bilinear resize, mean over the stages, final scale -- runs in
``csrc/gradcam.cu``.  Nothing leaves the device and no parameter's ``.grad`` changes.

Documented differences from the reference:
  * ``GradCAM.__call__`` unpacks ``output, prob, label = model(x)`` (visualization.py:201), which raises on the
    reference's own ResNet2d (one output); here the logits are the output and ``label`` is each row's arg-max.
  * the reference leaves the CAM loss's gradients in the parameters' ``.grad``; here ``.grad`` is untouched.
  * the resize follows OpenCV's portable INTER_LINEAR rule; OpenCV builds with IPP round some float32 outputs
    differently (a few float32 ulps).
"""
from __future__ import annotations

import operator
from typing import Sequence

import torch

from . import runtime
from .engine import Engine, RESNET_STAGES
from .networks.ResNet2d import ResNet2d

__all__ = ["grad_cam", "GradCAM"]


def _supported(what: str) -> NotImplementedError:
    return NotImplementedError(f"Grad-CAM: {what}; supported: the drop-in ResNet2d with target layers "
                               f"{', '.join(RESNET_STAGES)}")


def _check_model(model) -> None:
    if not isinstance(model, ResNet2d):
        raise _supported(f"model {type(model).__name__} is not supported")


def _category(model, target_category) -> int:
    """-1 (each row's arg-max) or a class index in [0, numclass)"""
    if target_category is None:
        return -1
    t = operator.index(target_category)
    if not 0 <= t < model.numclass:
        raise ValueError(f"target_category {t} is outside [0, {model.numclass})")
    return t


def _grad_cam(model, x: torch.Tensor, target: int, stages: Sequence[str]):
    """-> ((N, H, W) fp32 map, (N,) int64 classes) on x's device; ``stages`` in forward order (repeats allowed)"""
    if x.dim() != 4:
        raise RuntimeError(f"expected a 4-D input (N,C,H,W), got {tuple(x.shape)}")
    for s in x.shape[2:]:
        if s % 16 != 0:
            raise RuntimeError(f"spatial sizes must be multiples of 16 (four stride-2 stages), got {tuple(x.shape[2:])}")
    names = model._pnames
    params = [p.detach() for _, p in model.named_parameters()]
    xx = x.detach()
    if xx.dtype != torch.float32:
        xx = xx.float()
    be = runtime.get_backend(xx)
    eng = Engine(be, runtime.act_dtype(), 2)
    logits = eng.resnet_forward(dict(zip(names, params)), xx, None, need_grad=True)
    n = logits.shape[0]
    dlogits = torch.empty_like(logits)
    category = torch.empty(n, dtype=torch.int64, device=logits.device)
    be.gradcam_target(logits, target, dlogits, category)
    found = eng.resnet_backward(dlogits, stages=sorted(set(stages), key=RESNET_STAGES.index))
    out = torch.empty((n,) + tuple(xx.shape[2:]), dtype=torch.float32, device=xx.device)
    be.gradcam([found[s] for s in stages], out)
    return out, category


def grad_cam(model, x: torch.Tensor, target_category=None, layers=("down_tr256",)) -> torch.Tensor:
    """Grad-CAM maps of a drop-in ``ResNet2d`` for the images ``x`` (N, C, H, W): an (N, H, W) fp32 tensor on x's
    device, each map min-max scaled to [0, 1).

    ``target_category``: the class whose logit is explained, for every image; ``None`` takes each image's arg-max,
    chosen on the device.  ``layers``: stage names from ``in_tr``, ``down_tr32``, ``down_tr64``, ``down_tr128``,
    ``down_tr256``; several average their maps, as the reference's ``aggregate_multi_layers``.  The network runs
    in eval mode (no dropout) whatever ``model.training`` is."""
    _check_model(model)
    layers = [layers] if isinstance(layers, str) else list(layers)
    if not layers:
        raise ValueError("Grad-CAM needs at least one target layer")
    for name in layers:
        if name not in RESNET_STAGES:
            raise _supported(f"target layer {name!r} is not supported")
    stages = sorted(layers, key=RESNET_STAGES.index)     # the reference's hooks record in forward order
    return _grad_cam(model, x, _category(model, target_category), stages)[0]


class GradCAM:
    """``model/visualization.py`` GradCAM with the reference's constructor and call: ``GradCAM(model, target_layers,
    reshape_transform=None, use_cuda=False)(input_tensor, target_category=None)`` -> numpy float32 (N, H, W).

    ``target_layers`` are modules of the drop-in ResNet2d (``model.in_tr``, ``model.down_tr32`` ...
    ``model.down_tr256``), matched by identity within ``model.named_modules()``."""

    def __init__(self, model, target_layers, reshape_transform=None, use_cuda=False):
        _check_model(model)
        if reshape_transform is not None:
            raise _supported("reshape_transform is not supported")
        self.model = model.eval()
        self.target_layers = target_layers
        self.reshape_transform = reshape_transform
        self.cuda = use_cuda
        if self.cuda:
            self.model = model.cuda()
        names = {id(m): name for name, m in model.named_modules()}
        stages = []
        for layer in target_layers:
            name = names.get(id(layer))
            if name not in RESNET_STAGES:
                raise _supported(f"target layer {name or type(layer).__name__!r} is not supported")
            stages.append(name)
        if not stages:
            raise ValueError("Grad-CAM needs at least one target layer")
        self._stages = sorted(stages, key=RESNET_STAGES.index)

    def __call__(self, input_tensor, target_category=None):
        target = _category(self.model, target_category)
        dev = next(self.model.parameters()).device
        cam, category = _grad_cam(self.model, input_tensor.to(dev), target, self._stages)
        if target_category is None:
            cats = category.tolist()
            print(f"category id: {cats[0] if len(cats) == 1 else cats}")
        return cam.cpu().numpy()

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc_value, exc_tb):
        if isinstance(exc_value, IndexError):
            print(f"An exception occurred in CAM with block: {exc_type}. Message: {exc_value}")
            return True
