"""Drop-in SSIM losses of the reference ``model/lossesSSIM.py``: ``SSIM``, ``SSIM3D``, ``ssim`` and ``ssim3D`` with the
same names, signatures and attributes, computed by the separable-window kernels of ``csrc/ssim.cu``.

The reference filters five fields with a dense k^2 / k^3 depthwise window (``F.conv2d`` / ``F.conv3d``,
lossesSSIM.py:49-93) and lets autograd run five more dense convolutions backward.  Here one forward pass filters the
five fields separably along H, W (and D), forms the SSIM map and writes its fp64 partial sums (plus the backward
coefficients when an input needs a gradient); a small finalize sums the partials in a fixed order, and one backward
pass applies the adjoint filter to the coefficients.

Differences from the reference, by design:
  * inputs must be fp32 CUDA tensors (the reference also takes fp64; anything but fp32 raises ``TypeError``);
  * ``window_size`` must lie in [1, 31] (``ValueError`` otherwise);
  * the modules keep no cached ``window`` tensor (nothing reads it); ``window_size``, ``size_average`` and ``channel``
    are kept, and ``channel`` follows the last input as in the reference.
Under ``runtime.enable_data_parallel`` the mean forms all-reduce (sum of S, element count), so every rank gets the
global-batch value and gradient scale; the per-sample forms need no exchange.
"""
from __future__ import annotations

from math import exp

import torch
import torch.nn as nn

from . import runtime

MAX_WINDOW = 31


def gaussian_taps(window_size: int, sigma: float = 1.5) -> torch.Tensor:
    """the 1-D window of lossesSSIM.py:28-30, bit for bit: fp32 values of Python ``exp``, divided by their fp32 sum"""
    g = torch.tensor([exp(-(x - window_size // 2) ** 2 / float(2 * sigma ** 2)) for x in range(window_size)],
                     dtype=torch.float32)
    return g / g.sum()


def map_shape(shape, window_size: int):
    """spatial extents of the SSIM map: L + 2 (k // 2) - k + 1 per axis (one longer than L for an even window)"""
    p = window_size // 2
    return tuple(s + 2 * p - window_size + 1 for s in shape[2:])


def _check(img1: torch.Tensor, img2: torch.Tensor, window_size, dims: int) -> int:
    if isinstance(window_size, bool) or int(window_size) != window_size or not 1 <= window_size <= MAX_WINDOW:
        raise ValueError(f"window_size must be an integer in [1, {MAX_WINDOW}], got {window_size!r}")
    if img1.dim() != dims + 2:
        name = "(N, C, H, W)" if dims == 2 else "(N, C, D, H, W)"
        raise ValueError(f"expected {name} input, got shape {tuple(img1.shape)}")
    if img1.shape != img2.shape:
        raise ValueError(f"img1 and img2 differ in shape: {tuple(img1.shape)} vs {tuple(img2.shape)}")
    if img1.dtype != torch.float32 or img2.dtype != torch.float32:
        raise TypeError(f"SSIM inputs must be float32, got {img1.dtype} / {img2.dtype}")
    if img1.device != img2.device:
        raise ValueError(f"img1 and img2 are on different devices: {img1.device} / {img2.device}")
    if img1.numel() == 0:
        raise ValueError("empty input")
    return int(window_size)


class _SSIMFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img1, img2, window_size, size_average, dims):
        be = runtime.get_backend(img1)
        x, y = img1.detach(), img2.detach()
        dev, n = x.device, x.shape[0]
        taps = gaussian_taps(window_size)
        ms = map_shape(x.shape, window_size)
        need = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        nmap = x.shape[0] * x.shape[1]
        for v in ms:
            nmap *= v
        coef = torch.empty((4, nmap), dtype=torch.float64, device=dev) if need else None
        ws = be.ssim_fwd(x, y, window_size, taps, coef)
        if size_average:
            acc = torch.empty(2, dtype=torch.float64, device=dev)
            value = torch.empty((), dtype=torch.float32, device=dev)
        elif dims == 2:
            acc = torch.empty(n, dtype=torch.float64, device=dev)
            value = torch.empty(n, dtype=torch.float32, device=dev)
        else:                                    # S.mean(1).mean(1).mean(1) of (N, C, D', H', W') -> (N, W')
            acc = torch.empty((n, ms[-1]), dtype=torch.float64, device=dev)
            value = torch.empty((n, ms[-1]), dtype=torch.float32, device=dev)
        be.ssim_finalize(x, window_size, size_average, ws, acc, value)
        enabled, group = runtime.dp_state()
        if enabled and size_average:
            import torch.distributed as dist
            dist.all_reduce(acc, op=dist.ReduceOp.SUM, group=group)     # (sum S, count) over the global batch
            be.ssim_finalize(x, window_size, size_average, ws, acc, value, reduce=False)
        ctx.save_for_backward(x, y, coef, acc)
        ctx.window_size, ctx.size_average = window_size, size_average
        ctx.taps = taps
        return value

    @staticmethod
    def backward(ctx, gout):
        x, y, coef, acc = ctx.saved_tensors
        be = runtime.get_backend(x)
        g = gout.detach().to(torch.float32).contiguous()
        g1 = torch.empty(x.shape, dtype=torch.float32, device=x.device) if ctx.needs_input_grad[0] else None
        g2 = torch.empty(x.shape, dtype=torch.float32, device=x.device) if ctx.needs_input_grad[1] else None
        be.ssim_bwd(x, y, ctx.window_size, ctx.taps, coef, ctx.size_average, g, acc, g1, g2)
        return g1, g2, None, None, None


def _ssim(img1, img2, window_size, size_average, dims):
    k = _check(img1, img2, window_size, dims)
    return _SSIMFunction.apply(img1, img2, k, bool(size_average), dims)


def ssim(img1, img2, window_size=11, size_average=True):
    """reference model/lossesSSIM.py:148-155: 2-D SSIM of (N, C, H, W) images"""
    return _ssim(img1, img2, window_size, size_average, 2)


def ssim3D(img1, img2, window_size=11, size_average=True):
    """reference model/lossesSSIM.py:158-167: 3-D SSIM of (N, C, D, H, W) volumes; with size_average=False the result
    has shape (N, W') as in the reference (its three means run over C, D and H)"""
    return _ssim(img1, img2, window_size, size_average, 3)


class SSIM(nn.Module):
    """reference model/lossesSSIM.py:96-118"""

    def __init__(self, window_size=11, size_average=True):
        super().__init__()
        self.window_size = window_size
        self.size_average = size_average
        self.channel = 1

    def forward(self, img1, img2):
        out = ssim(img1, img2, self.window_size, self.size_average)
        self.channel = img1.shape[1]
        return out


class SSIM3D(nn.Module):
    """reference model/lossesSSIM.py:121-145"""

    def __init__(self, window_size=11, size_average=True):
        super().__init__()
        self.window_size = window_size
        self.size_average = size_average
        self.channel = 1

    def forward(self, img1, img2):
        out = ssim3D(img1, img2, self.window_size, self.size_average)
        self.channel = img1.shape[1]
        return out


__all__ = ["SSIM", "SSIM3D", "ssim", "ssim3D", "gaussian_taps"]
