"""CPU restatement of the further losses of ``model/losses.py`` (test infrastructure only): Jaccard, exponential-log
Dice, Tversky, sensitivity-specificity and Lovasz-Softmax (``model/lovasz.py``).

Same conventions as ``oracle/losses.py``: ``z`` = logits ``(N, C, *spatial)``, ``t`` = labels ``(N, *spatial)``,
fp32 by default, ``dtype=torch.float64`` for noise-floor runs.  Pinned to ``tests/golden/losses_ext.npz``, which the
real reference produced (``tests/golden/make_golden_losses_ext.py``).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .losses import EPS, SMOOTH, _flat_binary

Tensor = torch.Tensor


def binary_jaccard(z: Tensor, t: Tensor, dtype=torch.float32) -> Tensor:
    """BinaryJaccardLoss.forward, model/losses.py:19-30."""
    zf, tf = _flat_binary(z, t, dtype)
    p = torch.sigmoid(zf)
    inter = (p * tf).sum()
    return 1.0 - (inter + SMOOTH) / (p.sum() + tf.sum() - inter + SMOOTH).clamp_min(EPS)


def binary_eldice(z: Tensor, t: Tensor, dtype=torch.float32) -> Tensor:
    """BinaryELDiceLoss.forward, model/losses.py:66-74."""
    zf, tf = _flat_binary(z, t, dtype)
    p = torch.sigmoid(zf)
    dsc = (2.0 * (p * tf).sum() + SMOOTH) / (p.sum() + tf.sum() + SMOOTH).clamp_min(EPS)
    return torch.clamp(torch.pow(-torch.log(dsc + SMOOTH), 0.3), 0, 2)


def binary_tversky(z: Tensor, t: Tensor, alpha: float = 0.3, beta: float = 0.7, dtype=torch.float32) -> Tensor:
    """BinaryTverskyLoss.forward, model/losses.py:113-126."""
    zf, tf = _flat_binary(z, t, dtype)
    p = torch.sigmoid(zf)
    tp, fp, fn = (p * tf).sum(), (p * (1 - tf)).sum(), ((1 - p) * tf).sum()
    return torch.clamp(1 - (tp + SMOOTH) / (tp + alpha * fp + beta * fn + SMOOTH), 0, 2)


def binary_ss(z: Tensor, t: Tensor, r: float = 0.1, dtype=torch.float32) -> Tensor:
    """BinarySSLoss.forward, model/losses.py:87-99."""
    zf, tf = _flat_binary(z, t, dtype)
    p = torch.sigmoid(zf)
    se = (p - tf) ** 2
    return r * (se * tf).sum() / (SMOOTH + tf.sum()) + (1 - r) * (se * (1 - tf)).sum() / (SMOOTH + (1 - tf).sum())


def multi_eldice(z: Tensor, t: Tensor, alpha: Tensor, dtype=torch.float32) -> Tensor:
    """MutilELDiceLoss.forward, model/losses.py:358-382: absent classes still add (-log smooth)^0.3."""
    n, c = z.shape[0], z.shape[1]
    p = torch.softmax(z.to(dtype).reshape(n, c, -1), dim=1)
    oh = F.one_hot(t.long().reshape(n, -1), c).permute(0, 2, 1).to(dtype)
    d = ((2.0 * (oh * p).sum((0, 2)) + SMOOTH) / ((oh + p).sum((0, 2)) + SMOOTH)).clamp_min(EPS)
    present = oh.sum((0, 2)) > 0
    dice = d * present.to(dtype) * alpha.to(dtype)
    return torch.clamp(torch.pow(-torch.log(dice + SMOOTH), 0.3).sum() / torch.count_nonzero(present), 0, 2)


def _mean(values):
    """model/lovasz.py:166-182 (ignore_nan=False, empty=0)"""
    values = list(values)
    if not values:
        return 0
    acc = values[0]
    for v in values[1:]:
        acc = acc + v
    return acc if len(values) == 1 else acc / len(values)


def _lovasz_flat(probas: Tensor, labels: Tensor, dtype) -> Tensor:
    """model/lovasz.py:110-138 with classes="present".  The errors are formed in fp32 as in the reference and sorted
    stably (ties in ascending flat index); the Lovasz gradient and the dot product run in ``dtype``."""
    losses = []
    for c in range(probas.shape[1]):
        fg32 = (labels == c).to(torch.float32)
        if fg32.sum() == 0:
            continue
        e32 = (fg32 - probas[:, c].float()).abs()
        perm = torch.sort(e32.detach(), dim=0, descending=True, stable=True).indices
        fg = fg32.to(dtype)[perm]
        gts = fg.sum()
        jac = 1.0 - (gts - fg.cumsum(0)) / (gts + (1 - fg).cumsum(0))
        if len(fg) > 1:
            jac[1:] = jac[1:] - jac[:-1].clone()
        losses.append(torch.dot(e32.to(dtype)[perm], jac))
    return _mean(losses)


def _flatten(probas: Tensor, labels: Tensor, ignore):
    c = probas.shape[1]
    p = torch.movedim(probas, 1, -1).reshape(-1, c)
    lab = labels.reshape(-1)
    if ignore is None:
        return p, lab
    keep = lab != ignore
    return p[keep], lab[keep]


def lovasz_softmax(z: Tensor, t: Tensor, per_image: bool = False, ignore=None, dtype=torch.float32) -> Tensor:
    """LovaszLoss.forward, model/losses.py:472-473 -> model/lovasz.py:90-107: the logits are the probabilities."""
    if z.shape[1] == 1:
        raise ValueError("Sigmoid output possible only with 1 class")
    if per_image:
        out = _mean(_lovasz_flat(*_flatten(z[i:i + 1], t[i:i + 1], ignore), dtype) for i in range(z.shape[0]))
    else:
        out = _lovasz_flat(*_flatten(z, t, ignore), dtype)
    return out if torch.is_tensor(out) else torch.zeros((), dtype=dtype)
