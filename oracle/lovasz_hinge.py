"""CPU restatement of the binary Lovasz hinge of ``model/lovasz.py:35-84`` (``BinaryLovaszLoss``, ``model/losses.py:
235-242``; test infrastructure only).

``z`` = logits of one channel, ``(N, 1, *spatial)`` or ``(N, 1)``; ``t`` = integer labels 0 / 1 (or ``ignore``) with
as many elements.  The errors are formed in fp32 as in the reference and sorted stably (ties in ascending flat index);
the Lovasz gradient, the dot product and the mean over samples run in ``dtype``.  Pinned to
``tests/golden/lovasz_hinge.npz``, which the real reference produced (``tests/golden/make_golden_lovasz_hinge.py``).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .losses_ext import _mean

Tensor = torch.Tensor


def _hinge_flat(z: Tensor, lab: Tensor, dtype) -> Tensor:
    """model/lovasz.py:53-70"""
    if lab.numel() == 0:
        return z.sum().to(dtype) * 0.0                 # only ignored voxels: 0, no gradient
    e32 = 1.0 - z.float() * (2.0 * lab.float() - 1.0)
    perm = torch.sort(e32.detach(), dim=0, descending=True, stable=True).indices
    fg = lab.to(dtype)[perm]
    gts = fg.sum()
    jac = 1.0 - (gts - fg.cumsum(0)) / (gts + (1 - fg).cumsum(0))
    if len(fg) > 1:
        jac[1:] = jac[1:] - jac[:-1].clone()
    return torch.dot(F.relu(e32.to(dtype)[perm]), jac)


def _flatten(z: Tensor, t: Tensor, ignore):
    """model/lovasz.py:73-84"""
    z, t = z.reshape(-1), t.reshape(-1)
    if ignore is None:
        return z, t
    keep = t != ignore
    return z[keep], t[keep]


def lovasz_hinge(z: Tensor, t: Tensor, per_image: bool = False, ignore=None, dtype=torch.float32) -> Tensor:
    """BinaryLovaszLoss.forward -> model/lovasz.py:35-50; per_image: the mean over the samples of dim 0."""
    if per_image:
        n = z.shape[0]
        tn = t.reshape(n, -1)
        return _mean(_hinge_flat(*_flatten(z[i], tn[i], ignore), dtype) for i in range(n))
    return _hinge_flat(*_flatten(z, t, ignore), dtype)
