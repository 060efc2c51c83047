"""Drop-in soft-clDice losses of the reference ``model/lossescldice.py``: ``soft_skeletonize``, ``norm_intersection``,
``Binary_Soft_cldice_loss`` and ``Mutil_Soft_cldice_loss`` with the same names and signatures, computed by the kernels
of ``csrc/cldice.cu``.

The reference module raises as shipped (``x.size().tolist()``; ``if shape == 4`` compares a list with an int; its
classes define ``__int__`` instead of ``__init__``; the multi-class loop drops the channel axis).  This module runs
the evident intent, pinned in DESIGN.md section 2: ``thresh_width`` rounds of
``m = -maxpool(-x); c = relu(maxpool(m) - m); x = relu(x - c)`` with 3x3 (4-D input) or 3x3x3 (5-D input) windows,
stride 1, padding 1; the binary loss of lossescldice.py:52-59 with ``smooth = 1e-5``, ``eps = 1e-7``; and the
multi-class loss over ``input[:, c:c+1]`` and the one-hot ``target[:, c:c+1]``, weighted by ``alpha[c]``, summed and
divided by C.  Inputs are used as given: no sigmoid or softmax is applied.

One launch per round fuses both pools, the contour and the ReLU over a shared-memory tile; the skeleton is
bit-identical to torch's fp32 sequence.  The loss's last round also forms the per-(n, c) sums, a one-block finalize
forms the loss, and the backward runs the ten rounds in reverse as fixed-order gathers.  The gradient is taken with
respect to ``pred`` / ``input`` only; a target that requires grad raises ``ValueError``.

Differences from the reference's intent, by design:
  * inputs must be fp32 CUDA tensors (``TypeError`` otherwise), 4-D or 5-D (``ValueError`` otherwise);
  * ``thresh_width`` must be an integer in [0, 64];
  * skeletons and gradients come back NCDHW-contiguous whatever the input's memory format.
Under ``runtime.enable_data_parallel`` the losses all-reduce their per-class sums {sum iflat * tflat, sum iflat,
sum tflat}, so every rank gets the global-batch loss and its slice of the global-batch gradient.

The drop-in networks' ``probs`` output carries no gradient: to train a drop-in net with clDice, form the
probabilities from its logits (``torch.sigmoid`` / ``torch.softmax``) and pass those.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import runtime
from .losses import _check_labels_default

MAX_ROUNDS = 64
LOSS_ROUNDS = 10                            # Binary_Soft_cldice_loss calls soft_skeletonize(pred) with its default


def _shape5(x):
    return (x.shape[0], x.shape[1], 1) + tuple(x.shape[2:]) if x.dim() == 4 else tuple(x.shape)


def _check_one(x, what="input"):
    if x.dim() not in (4, 5):
        raise ValueError(f"expected (N, C, H, W) or (N, C, D, H, W) {what}, got shape {tuple(x.shape)}")
    if x.dtype != torch.float32:
        raise TypeError(f"clDice {what} must be float32, got {x.dtype}")
    if x.numel() == 0:
        raise ValueError("empty input")


def _check(a, b):
    _check_one(a)
    if a.shape != b.shape:
        raise ValueError(f"inputs differ in shape: {tuple(a.shape)} vs {tuple(b.shape)}")
    if b.dtype != torch.float32:
        raise TypeError(f"clDice inputs must be float32, got {a.dtype} / {b.dtype}")
    if a.device != b.device:
        raise ValueError(f"inputs are on different devices: {a.device} / {b.device}")


def _check_rounds(thresh_width):
    if isinstance(thresh_width, bool) or int(thresh_width) != thresh_width or not 0 <= thresh_width <= MAX_ROUNDS:
        raise ValueError(f"thresh_width must be an integer in [0, {MAX_ROUNDS}], got {thresh_width!r}")
    return int(thresh_width)


class _SkeletonFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, rounds):
        be = runtime.get_backend(x)
        xd = x.detach()
        need = ctx.needs_input_grad[0]
        nf = rounds if need else min(rounds, 2)
        fields = torch.empty((nf,) + tuple(x.shape), dtype=torch.float32, device=x.device)
        be.cldice_skeleton(xd, rounds, fields)
        ctx.rounds = rounds
        ctx.save_for_backward(xd, fields if need else None)
        return fields[(rounds - 1) % nf]

    @staticmethod
    def backward(ctx, g):
        x, fields = ctx.saved_tensors
        be = runtime.get_backend(x)
        g = g.detach().to(torch.float32).contiguous()
        grad = torch.empty(x.shape, dtype=torch.float32, device=x.device)
        scratch = torch.empty_like(grad) if ctx.rounds > 1 else None
        be.cldice_bwd(x, ctx.rounds, fields, grad, scratch, grad_skeleton=g)
        return grad, None


def soft_skeletonize(x, thresh_width=10):
    """reference model/lossescldice.py:5-21 (repaired): ``thresh_width`` rounds of soft erosion-minus-opening of an
    (N, C, H, W) or (N, C, D, H, W) fp32 tensor; 0 rounds return ``x`` itself, as the reference's empty loop does"""
    rounds = _check_rounds(thresh_width)
    _check_one(x)
    if rounds == 0:
        return x
    return _SkeletonFunction.apply(x, rounds)


class _NormFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cl, vessel):
        be = runtime.get_backend(cl)
        a, b = cl.detach(), vessel.detach()
        n, c = a.shape[:2]
        sums = torch.empty((n * c, 2), dtype=torch.float64, device=a.device)
        out = torch.empty((n, c), dtype=torch.float32, device=a.device)
        be.cldice_norm(a, b, sums, out)
        ctx.save_for_backward(a, b, sums)
        return out

    @staticmethod
    def backward(ctx, g):
        a, b, sums = ctx.saved_tensors
        be = runtime.get_backend(a)
        g = g.detach().to(torch.float32).contiguous()
        ga = torch.empty(a.shape, dtype=torch.float32, device=a.device) if ctx.needs_input_grad[0] else None
        gb = torch.empty(a.shape, dtype=torch.float32, device=a.device) if ctx.needs_input_grad[1] else None
        if ga is not None or gb is not None:
            be.cldice_norm_bwd(a, b, sums, g, ga, gb)
        return ga, gb


def norm_intersection(center_line, vessel):
    """reference model/lossescldice.py:24-34: (sum cl * vessel + 1) / (sum cl + 1) per (n, c) -> (N, C) fp32"""
    _check(center_line, vessel)
    return _NormFunction.apply(center_line, vessel)


class _ClDiceFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target, labels, alpha, smooth, eps):
        be = runtime.get_backend(pred)
        p = pred.detach()
        t = labels if labels is not None else target.detach()
        dev = p.device
        n, c = p.shape[:2]
        per_class = labels is not None
        need = ctx.needs_input_grad[0]
        fp = torch.empty((LOSS_ROUNDS if need else 2,) + tuple(p.shape), dtype=torch.float32, device=dev)
        ft = torch.empty((2,) + tuple(p.shape), dtype=torch.float32, device=dev)
        ws = be.cldice_workspace(p)
        be.cldice_skeleton(p, LOSS_ROUNDS, fp, other=t, pass_=0, ws=ws)
        be.cldice_skeleton(t, LOSS_ROUNDS, ft, other=p, pass_=1, ws=ws)
        ng = c if per_class else 1
        stats = torch.empty(8 * n * c + 3 * ng + 1, dtype=torch.float64, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        shape = _shape5(p)
        be.cldice_finalize(shape, per_class, per_class, alpha, smooth, eps, ws, stats, loss)
        enabled, group = runtime.dp_state()
        if enabled:
            import torch.distributed as dist
            dist.all_reduce(stats[8 * n * c:8 * n * c + 3 * ng], op=dist.ReduceOp.SUM, group=group)
            be.cldice_finalize(shape, per_class, per_class, alpha, smooth, eps, ws, stats, loss, reduce=False)
        if per_class and _check_labels_default() and not runtime.is_capturing(dev):
            bad = int(stats[-1].item())             # the reference's F.one_hot raises too
            if bad:
                raise RuntimeError(f"{bad} label value(s) outside [0, {c}): class labels must be in [0, numclass)")
        ctx.save_for_backward(p, t, fp if need else None, ft[(LOSS_ROUNDS - 1) % 2], stats)
        return loss

    @staticmethod
    def backward(ctx, gout):
        p, t, fp, skt, stats = ctx.saved_tensors
        be = runtime.get_backend(p)
        g = gout.detach().to(torch.float32).reshape(1).contiguous()
        grad = torch.empty(p.shape, dtype=torch.float32, device=p.device)
        scratch = torch.empty_like(grad)
        be.cldice_bwd(p, LOSS_ROUNDS, fp, grad, scratch, target=t, target_skeleton=skt, stats=stats, gout=g)
        return grad, None, None, None, None, None


def _no_target_grad(target):
    if target.requires_grad:
        raise ValueError("clDice takes its gradient with respect to the prediction only: the target must not "
                         "require grad")


class Binary_Soft_cldice_loss(nn.Module):
    """reference model/lossescldice.py:37-59 (its ``__int__`` run as the initialiser): pred and target fp32 of one
    shape (N, C, H, W) or (N, C, D, H, W); the loss sums iflat and tflat over every (n, c)"""

    def __init__(self):
        super().__init__()
        self.smooth = 1e-5
        self.eps = 1e-7

    def forward(self, pred, target):
        _check(pred, target)
        _no_target_grad(target)
        return _ClDiceFunction.apply(pred, target, None, None, self.smooth, self.eps)


class Mutil_Soft_cldice_loss(nn.Module):
    """reference model/lossescldice.py:62-84 (its ``__int__`` run as the initialiser, channel axis kept): input fp32
    (N, C, H, W) or (N, C, D, H, W); target integer class indices (N, *spatial) or (N, 1, *spatial), one-hot encoded;
    the binary loss of each class, weighted by alpha[c], summed and divided by C"""

    def __init__(self, alpha):
        super().__init__()
        self.alpha = alpha
        self.bscldice = Binary_Soft_cldice_loss()

    def _alpha_on(self, device):
        """alpha as a device fp32 vector; a host sequence is uploaded once per (values, device), so a captured step
        copies nothing from the host"""
        if torch.is_tensor(self.alpha):
            return self.alpha.detach().to(device=device, dtype=torch.float32).reshape(-1)
        key = (str(device), tuple(float(a) for a in self.alpha))
        if getattr(self, "_alpha_key", None) != key:
            self._alpha_dev = torch.tensor(key[1], dtype=torch.float32, device=device)
            self._alpha_key = key
        return self._alpha_dev

    def forward(self, input, target):
        _check_one(input)
        _no_target_grad(target)
        n, c = input.shape[:2]
        spatial = tuple(input.shape[2:])
        if tuple(target.shape) not in ((n,) + spatial, (n, 1) + spatial):
            raise ValueError(f"target shape {tuple(target.shape)} does not match input {tuple(input.shape)}: expected "
                             f"(N, *spatial) or (N, 1, *spatial)")
        if target.device != input.device:
            raise ValueError(f"input and target are on different devices: {input.device} / {target.device}")
        labels = target.detach().long().reshape((n,) + spatial).contiguous()
        alpha = self._alpha_on(input.device)
        if alpha.numel() < c:
            raise ValueError(f"alpha has {alpha.numel()} weights for {c} classes")
        return _ClDiceFunction.apply(input, None, labels, alpha.contiguous(), self.bscldice.smooth,
                                     self.bscldice.eps)


__all__ = ["soft_skeletonize", "norm_intersection", "Binary_Soft_cldice_loss", "Mutil_Soft_cldice_loss"]
