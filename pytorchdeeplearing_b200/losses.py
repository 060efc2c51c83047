"""Drop-in hot-path losses of the reference ``model/losses.py`` (same class names, constructor
arguments and ``forward(y_pred_logits, y_true) -> 0-dim fp32 tensor``).

Each loss is ONE fused reduction pass over logits + labels (``b200seg_loss_partials``), a
scalar finalize (``b200seg_loss_finalize``) and ONE elementwise backward pass writing
d loss / d logits (``b200seg_loss_bwd``) -- closed forms of SURVEY.md App. C -- instead of
the ~10-15 elementwise/reduce launches of the reference.  Under data parallelism the
partial sums are all-reduced so the value and gradient equal the reference evaluated on the
GLOBAL batch (Dice sums run over batch and space, model/losses.py:50-51,315-317).
"""
from __future__ import annotations

import os

import torch
import torch.nn as nn

from . import runtime

DICE, CE, FOCAL = 1, 2, 4
JACCARD, ELDICE, TVERSKY, SS = 8, 16, 32, 64     # include/b200seg.h B200SEG_LOSS_*: each one alone
LOVASZ = 128                                     # not a finalize term: the sort-based Lovasz-Softmax path
LOVASZ_HINGE = 256                               # not a finalize term: the sort-based binary Lovasz hinge path


def _check_labels_default() -> bool:
    return os.environ.get("B200SEG_CHECK_LABELS", "1") != "0"


def prepare_logits(logits: torch.Tensor):
    """channels-last fp32 view (N, ..., C) of NCDHW / NCHW logits (free when they come from the drop-in networks).
    Classifier logits (N, C) become an (N, 1, 1, 1, C) volume of one voxel per sample, which is what the reference's
    ``.view(bs, C, -1)`` makes of them (model/losses.py:143,253); ``perm`` is then None."""
    z = logits.detach()
    if z.dim() == 2:
        perm = None
        z = z.reshape(z.shape[0], 1, 1, 1, z.shape[1])
    else:
        perm = (0, 2, 3, 4, 1) if z.dim() == 5 else (0, 2, 3, 1)
        z = z.permute(*perm)
    if z.dtype != torch.float32:
        z = z.float()                               # losses.py:47 ``.float()``
    if not z.is_contiguous():
        z = z.contiguous()
    return z, perm


def prepare_labels(labels: torch.Tensor, c: int):
    """int64 class indices as the reference's datasets deliver them (model/dataset.py:114); the binary losses take
    ``y_true.float()`` (model/losses.py:47,144), so a floating-point target is kept as fp32 soft targets there."""
    t = labels.detach()
    if c == 1 and t.is_floating_point():
        if t.dtype != torch.float32:
            t = t.float()
    elif t.dtype != torch.int64:
        t = t.long()
    if not t.is_contiguous():
        t = t.contiguous()
    return t


def logits_grad(dz: torch.Tensor, perm):
    """d loss / d logits in the caller's layout: the inverse of ``prepare_logits``"""
    if perm is None:
        return dz.view(dz.shape[0], dz.shape[-1])
    inv = (0, 4, 1, 2, 3) if dz.dim() == 5 else (0, 3, 1, 2)
    return dz.permute(*inv)


class _FusedLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels, terms, alpha, gamma, alpha_f, owner):
        be = runtime.get_backend(logits)
        c = logits.shape[1]
        z, perm = prepare_logits(logits)
        t = prepare_labels(labels, c)
        if t.numel() * c != z.numel():
            raise RuntimeError(f"label shape {tuple(labels.shape)} does not match logits {tuple(logits.shape)}")
        dev = z.device
        n = z.shape[0]
        buf = torch.zeros(be.part_size(c) + n * c * 3, dtype=torch.float64, device=dev)
        part, metric = buf[:be.part_size(c)], buf[be.part_size(c):].view(n, c, 3)
        if terms == SS:
            be.loss_partials_ss(z, t, part, metric)
        else:
            be.loss_partials(z, t, float(gamma), float(alpha_f), part, metric)
        enabled, group = runtime.dp_state()
        if enabled:
            import torch.distributed as dist
            dist.all_reduce(part, op=dist.ReduceOp.SUM, group=group)     # SURVEY.md section 8e (C2)
        if c > 1 and _check_labels_default() and not runtime.is_capturing(dev):
            bad = int(part[-1].item())               # the reference raises too (F.one_hot / F.cross_entropy)
            if bad:
                raise RuntimeError(f"{bad} label value(s) outside [0, {c}): class labels must be in [0, numclass)")
        loss = torch.empty((), dtype=torch.float32, device=dev)
        lcoef = torch.empty(2 * c + 3 if c > 1 else 5, dtype=torch.float32, device=dev)
        if alpha is None:
            alpha = torch.ones(c, dtype=torch.float32, device=dev)
        else:
            alpha = torch.as_tensor(alpha, dtype=torch.float32, device=dev)
        be.loss_finalize(part, c, terms, alpha, float(gamma), float(alpha_f), loss, lcoef)
        if owner is not None:
            owner._metric_sums = metric               # per-sample sums of the step's accuracy (SURVEY 8f-2)
        ctx.save_for_backward(z, t, lcoef)
        ctx.perm = perm
        ctx.terms = terms
        return loss

    @staticmethod
    def backward(ctx, gout):
        z, t, lcoef = ctx.saved_tensors
        be = runtime.get_backend(z)
        dz = torch.empty_like(z)
        g = gout.detach().to(torch.float32).reshape(1).contiguous()
        if ctx.terms == SS:
            be.loss_bwd_ss(z, t, lcoef, g, dz)
        else:
            be.loss_bwd(z, t, lcoef, g, dz)
        return logits_grad(dz, ctx.perm), None, None, None, None, None, None


def ignore_label(ignore):
    """the label value LovaszLoss(ignore=...) drops, as an int, or None (no integer label can equal it)"""
    if ignore is None:
        return None
    v = float(ignore)
    return int(v) if v.is_integer() else None


def lovasz_check(c: int) -> None:
    """what the reference raises for LovaszLoss on this class count / run mode"""
    if c == 1:
        # model/lovasz.py:127-129 with classes="present" (the only form LovaszLoss uses)
        raise ValueError("Sigmoid output possible only with 1 class")
    if runtime.dp_state()[0]:
        raise RuntimeError("LovaszLoss does not run under data parallelism: its value on the global batch needs one "
                           "sort over every rank's voxels")


def lovasz_scale_size(n: int, c: int, per_image: bool) -> int:
    return n * c if per_image else c


class _LovaszLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels, per_image, ignore, owner):
        c = logits.shape[1]
        lovasz_check(c)
        be = runtime.get_backend(logits)
        z, perm = prepare_logits(logits)
        t = prepare_labels(labels, c)
        if t.numel() * c != z.numel():
            raise RuntimeError(f"label shape {tuple(labels.shape)} does not match logits {tuple(logits.shape)}")
        dev, n = z.device, z.shape[0]
        # the per-step accuracy sums come from the fused partial-sum pass of the other losses (its loss sums unused)
        buf = torch.zeros(be.part_size(c) + n * c * 3, dtype=torch.float64, device=dev)
        metric = buf[be.part_size(c):].view(n, c, 3)
        be.loss_partials(z, t, 2.0, 0.25, buf[:be.part_size(c)], metric)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        coef = torch.empty_like(z)
        scale = torch.empty(lovasz_scale_size(n, c, per_image), dtype=torch.float32, device=dev)
        be.lovasz_fwd(z, t, per_image, ignore_label(ignore), loss, coef, scale)
        if owner is not None:
            owner._metric_sums = metric
        ctx.save_for_backward(z, t, coef, scale)
        ctx.perm = perm
        ctx.per_image = per_image
        return loss

    @staticmethod
    def backward(ctx, gout):
        z, t, coef, scale = ctx.saved_tensors
        be = runtime.get_backend(z)
        dz = torch.empty_like(z)
        g = gout.detach().to(torch.float32).reshape(1).contiguous()
        be.lovasz_bwd(z, t, ctx.per_image, coef, scale, g, dz)
        return logits_grad(dz, ctx.perm), None, None, None, None


def lovasz_hinge_check(c: int, labels: torch.Tensor) -> None:
    """what BinaryLovaszLoss refuses: more than one logit channel, floating-point labels, data parallelism"""
    if c != 1:
        raise ValueError(f"BinaryLovaszLoss takes logits of one channel, got {c}")
    if labels.is_floating_point():
        raise TypeError(f"BinaryLovaszLoss takes integer labels 0 / 1 (or ignore_index), got {labels.dtype}")
    if runtime.dp_state()[0]:
        raise RuntimeError("BinaryLovaszLoss does not run under data parallelism: its value on the global batch needs "
                           "one sort over every rank's voxels")


def lovasz_hinge_bad_labels(bad: torch.Tensor) -> None:
    """raise if the hinge's label count found values other than 0, 1 and ignore_index (synchronises)"""
    n = int(bad.item())
    if n:
        raise ValueError(f"{n} label value(s) other than 0 and 1: BinaryLovaszLoss takes binary labels "
                         "(or ignore_index)")


class _LovaszHingeLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels, per_image, ignore, owner):
        if logits.dim() not in (2, 4, 5):
            raise ValueError(f"BinaryLovaszLoss takes (N, 1), (N, 1, H, W) or (N, 1, D, H, W) logits, got "
                             f"{tuple(logits.shape)}")
        lovasz_hinge_check(logits.shape[1], labels)
        be = runtime.get_backend(logits)
        z, perm = prepare_logits(logits)
        t = prepare_labels(labels, 1)
        if t.numel() != z.numel():
            raise RuntimeError(f"label shape {tuple(labels.shape)} does not match logits {tuple(logits.shape)}")
        dev, n = z.device, z.shape[0]
        buf = torch.zeros(be.part_size(1) + n * 3, dtype=torch.float64, device=dev)
        metric = buf[be.part_size(1):].view(n, 1, 3)
        be.loss_partials(z, t, 2.0, 0.25, buf[:be.part_size(1)], metric)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        coef = torch.empty_like(z)
        bad = torch.empty(1, dtype=torch.int64, device=dev)
        be.lovasz_hinge_fwd(z, t, per_image, ignore_label(ignore), loss, coef, bad)
        if _check_labels_default() and not runtime.is_capturing(dev):
            lovasz_hinge_bad_labels(bad)
        if owner is not None:
            owner._metric_sums = metric
        ctx.save_for_backward(coef)
        ctx.perm = perm
        return loss

    @staticmethod
    def backward(ctx, gout):
        coef, = ctx.saved_tensors
        be = runtime.get_backend(coef)
        dz = torch.empty_like(coef)
        g = gout.detach().to(torch.float32).reshape(1).contiguous()
        be.lovasz_hinge_bwd(coef, g, dz)
        return logits_grad(dz, ctx.perm), None, None, None, None


class _LossBase(nn.Module):
    """Common part of the loss modules: after every ``forward`` the per-sample sums of the reference's per-step
    accuracy (model/metric.py:146-181) are available from the SAME pass over logits + labels."""

    _metric_sums = None

    def last_metric(self) -> torch.Tensor:
        """fp32 [2] = (dice, iou) of the last forward: ``dice_coeff(probs, y)`` for one class,
        ``multiclass_dice_coeff(probs, y)`` otherwise -- without reading ``probs``.  On classifier logits (N, C) it
        is the same Dice / IoU formula over one voxel per sample, not a classification accuracy."""
        if self._metric_sums is None:
            raise RuntimeError("no forward has run yet")
        be = runtime.get_backend(self._metric_sums)
        out = torch.empty(2, dtype=torch.float32, device=self._metric_sums.device)
        be.metric_finalize(self._metric_sums, out)
        return out

    def last_dice(self) -> torch.Tensor:
        return self.last_metric()[0]


def loss_spec(lossfn):
    """(terms, alpha, gamma, alpha_f) of one of the loss modules below (used by graphed.GraphedStep)."""
    name = type(lossfn).__name__
    table = {"BinaryDiceLoss": DICE, "BinaryCrossEntropyLoss": CE, "BinaryFocalLoss": FOCAL,
             "BinaryCrossEntropyDiceLoss": DICE | CE, "BinaryDiceFocalLoss": DICE | FOCAL,
             "MutilCrossEntropyLoss": CE, "MutilFocalLoss": FOCAL, "MutilDiceLoss": DICE,
             "MutilCrossEntropyDiceLoss": DICE | CE,
             "BinaryJaccardLoss": JACCARD, "BinaryELDiceLoss": ELDICE, "BinaryTverskyLoss": TVERSKY,
             "BinarySSLoss": SS, "MutilELDiceLoss": ELDICE, "LovaszLoss": LOVASZ,
             "BinaryLovaszLoss": LOVASZ_HINGE}
    if name not in table:
        raise TypeError(f"{name} is not a pytorchdeeplearing_b200 loss")
    alpha = getattr(lossfn, "alpha", None) if name.startswith("Mutil") and (table[name] & (DICE | ELDICE)) else None
    gamma = float(getattr(lossfn, "gamma", 2.0))
    alpha_f = float(getattr(lossfn, "alpha", 0.25)) if name in ("BinaryFocalLoss", "BinaryDiceFocalLoss") else 0.25
    if name == "BinaryTverskyLoss":
        alpha_f, gamma = float(lossfn.alpha), float(lossfn.beta)
    elif name == "BinarySSLoss":
        alpha_f = float(lossfn.r)
    return table[name], alpha, gamma, alpha_f


def _call(logits, labels, terms, alpha=None, gamma=2.0, alpha_f=0.25, owner=None):
    return _FusedLoss.apply(logits, labels, terms, alpha, gamma, alpha_f, owner)


# ------------------------------------------------------------------------------ binary (sigmoid head)
class BinaryDiceLoss(_LossBase):
    """reference model/losses.py:33-53"""

    def __init__(self):
        super().__init__()
        self.smooth = 1e-5
        self.eps = 1e-7

    def forward(self, y_pred_logits, y_true):
        return _call(y_pred_logits, y_true, DICE, owner=self)


class BinaryCrossEntropyLoss(_LossBase):
    """reference model/losses.py:129-147"""

    def forward(self, y_pred_logits, y_true):
        return _call(y_pred_logits, y_true, CE, owner=self)


class BinaryFocalLoss(_LossBase):
    """reference model/losses.py:150-181 (alpha applied to both classes)"""

    def __init__(self, alpha=0.25, gamma=2):
        super().__init__()
        self.alpha = alpha
        self.gamma = gamma

    def forward(self, y_pred_logits, y_true):
        return _call(y_pred_logits, y_true, FOCAL, gamma=self.gamma, alpha_f=self.alpha, owner=self)


class BinaryCrossEntropyDiceLoss(_LossBase):
    """reference model/losses.py:184-197"""

    def forward(self, y_pred_logits, y_true):
        return _call(y_pred_logits, y_true, DICE | CE, owner=self)


class BinaryDiceFocalLoss(_LossBase):
    """BinaryDiceLoss + BinaryFocalLoss() in one pass (BASELINE.json config 5 "Dice+focal";
    the reference has no class for it -- SURVEY.md a14)."""

    def __init__(self, alpha=0.25, gamma=2):
        super().__init__()
        self.alpha = alpha
        self.gamma = gamma

    def forward(self, y_pred_logits, y_true):
        return _call(y_pred_logits, y_true, DICE | FOCAL, gamma=self.gamma, alpha_f=self.alpha, owner=self)


# ------------------------------------------------------------------------------ multi-class (softmax head)
class MutilCrossEntropyLoss(_LossBase):
    """reference model/losses.py:247-260 (``alpha`` stored but unused, as in the reference)"""

    def __init__(self, alpha):
        super().__init__()
        self.alpha = alpha

    def forward(self, y_pred_logits, y_true):
        return _call(y_pred_logits, y_true, CE, owner=self)


class MutilFocalLoss(_LossBase):
    """reference model/losses.py:263-285 (``alpha`` / ``torch`` stored but unused)"""

    def __init__(self, alpha, gamma=2, torch=True):
        super().__init__()
        self.gamma = gamma
        self.alpha = alpha
        self.torch = torch

    def forward(self, y_pred_logits, y_true):
        return _call(y_pred_logits, y_true, FOCAL, gamma=self.gamma, owner=self)


class MutilDiceLoss(_LossBase):
    """reference model/losses.py:288-325 (negative generalised Dice over present classes)"""

    def __init__(self, alpha):
        super().__init__()
        self.alpha = alpha

    def forward(self, y_pred_logits, y_true):
        return _call(y_pred_logits, y_true, DICE, alpha=self.alpha, owner=self)


class MutilCrossEntropyDiceLoss(_LossBase):
    """reference model/losses.py:328-342"""

    def __init__(self, alpha):
        super().__init__()
        self.alpha = alpha

    def forward(self, y_pred_logits, y_true):
        return _call(y_pred_logits, y_true, DICE | CE, alpha=self.alpha, owner=self)


# ------------------------------------------------------------------------------ further reference losses
class BinaryJaccardLoss(_LossBase):
    """reference model/losses.py:9-30"""

    def __init__(self):
        super().__init__()
        self.smooth = 1e-5
        self.eps = 1e-7

    def forward(self, y_pred_logits, y_true):
        return _call(y_pred_logits, y_true, JACCARD, owner=self)


class BinaryELDiceLoss(_LossBase):
    """reference model/losses.py:56-74: clamp((-log(dsc + smooth))^0.3, 0, 2)"""

    def __init__(self):
        super().__init__()
        self.smooth = 1e-5
        self.eps = 1e-7

    def forward(self, y_pred_logits, y_true):
        return _call(y_pred_logits, y_true, ELDICE, owner=self)


class BinarySSLoss(_LossBase):
    """reference model/losses.py:77-99 (sensitivity-specificity, weight r)"""

    def __init__(self):
        super().__init__()
        self.smooth = 1e-5
        self.r = 0.1

    def forward(self, y_pred_logits, y_true):
        return _call(y_pred_logits, y_true, SS, alpha_f=self.r, owner=self)


class BinaryTverskyLoss(_LossBase):
    """reference model/losses.py:102-126: clamp(1 - tversky, 0, 2)"""

    def __init__(self):
        super().__init__()
        self.smooth = 1e-5
        self.alpha = 0.3
        self.beta = 0.7

    def forward(self, y_pred_logits, y_true):
        return _call(y_pred_logits, y_true, TVERSKY, gamma=self.beta, alpha_f=self.alpha, owner=self)


class MutilELDiceLoss(_LossBase):
    """reference model/losses.py:345-382: the sum over ALL classes of (-log(d_c present_c alpha_c + smooth))^0.3,
    divided by the number of present classes, clamped to [0, 2]"""

    def __init__(self, alpha):
        super().__init__()
        self.alpha = alpha

    def forward(self, y_pred_logits, y_true):
        return _call(y_pred_logits, y_true, ELDICE, alpha=self.alpha, owner=self)


class LovaszLoss(_LossBase):
    """reference model/losses.py:462-473 -> model/lovasz.py:90-138 (Lovasz-Softmax over the classes present in the
    labels).  As in the reference the logits themselves are taken as the probabilities.  Labels outside [0, C) are
    background for every class; C == 1 raises.  Not available under data parallelism (it needs a global sort)."""

    def __init__(self, per_image=False, ignore=None):
        super().__init__()
        self.ignore = ignore
        self.per_image = per_image

    def forward(self, logits, target):
        return _LovaszLoss.apply(logits, target, bool(self.per_image), self.ignore, self)


class BinaryLovaszLoss(_LossBase):
    """reference model/losses.py:235-242 -> model/lovasz.py:35-84 (binary Lovasz hinge on one logit channel).  The
    reference's constructor never runs nn.Module.__init__ (an unbound super), so its objects cannot be called; this one
    can.  Labels must be integer 0 / 1 or ``ignore_index``; a sample with every voxel ignored adds 0 (with per_image,
    it still counts in the mean).  Not available under data parallelism (it needs a global sort)."""

    def __init__(self, per_image: bool = False, ignore_index=None):
        super().__init__()
        self.ignore_index = ignore_index
        self.per_image = per_image

    def forward(self, logits, target):
        return _LovaszHingeLoss.apply(logits, target, bool(self.per_image), self.ignore_index, self)


def lovasz_hinge(logits, labels, per_image=True, ignore_index=None):
    """model/lovasz.py:35-50 ``_lovasz_hinge`` (its defaults) on the logit layouts of BinaryLovaszLoss"""
    return _LovaszHingeLoss.apply(logits, labels, bool(per_image), ignore_index, None)


__all__ = ["BinaryDiceLoss", "BinaryCrossEntropyLoss", "BinaryFocalLoss", "BinaryCrossEntropyDiceLoss",
           "BinaryDiceFocalLoss", "MutilCrossEntropyLoss", "MutilFocalLoss", "MutilDiceLoss",
           "MutilCrossEntropyDiceLoss", "BinaryJaccardLoss", "BinaryELDiceLoss", "BinarySSLoss", "BinaryTverskyLoss",
           "MutilELDiceLoss", "LovaszLoss", "BinaryLovaszLoss", "lovasz_hinge"]
