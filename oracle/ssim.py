"""Restatement of the reference's SSIM operator sequence (model/lossesSSIM.py:28-93) from its formulas: a Gaussian window
(sigma 1.5) built in fp32, five depthwise convolutions with zero padding k // 2, the SSIM map and its reduction.

``dtype=torch.float32`` is what the reference computes; ``torch.float64`` (the fp32 window and inputs, widened) is the
arbiter the GPU kernels are held to.  Runs on either device; gradients come from autograd."""
from math import exp

import torch
import torch.nn.functional as F

C1 = 0.01 ** 2
C2 = 0.03 ** 2


def gaussian(window_size: int, sigma: float = 1.5) -> torch.Tensor:
    g = torch.tensor([exp(-(x - window_size // 2) ** 2 / float(2 * sigma ** 2)) for x in range(window_size)],
                     dtype=torch.float32)
    return g / g.sum()


def window(window_size: int, dims: int) -> torch.Tensor:
    """fp32 (k, k) = g_i g_j, or (k, k, k) = g_i (g_j g_k), each product rounded to fp32 once"""
    g = gaussian(window_size)
    w2 = g[:, None] * g[None, :]
    if dims == 2:
        return w2
    return (g[:, None] * w2.reshape(1, -1)).reshape(window_size, window_size, window_size)


def ssim_map(img1, img2, window_size=11, dims=3, dtype=torch.float32):
    x, y = img1.to(dtype), img2.to(dtype)
    c = x.shape[1]
    w = window(window_size, dims).to(device=x.device, dtype=dtype)
    w = w.expand(c, 1, *w.shape).contiguous()
    conv = F.conv2d if dims == 2 else F.conv3d
    p = window_size // 2

    def filt(t):
        return conv(t, w, padding=p, groups=c)

    mu1, mu2 = filt(x), filt(y)
    s11 = filt(x * x) - mu1 * mu1
    s22 = filt(y * y) - mu2 * mu2
    s12 = filt(x * y) - mu1 * mu2
    return ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s11 + s22 + C2))


def ssim(img1, img2, window_size=11, size_average=True, dims=None, dtype=torch.float32):
    """SSIM (dims 2) / SSIM3D (dims 3; default from the input rank); size_average=False gives
    S.mean(1).mean(1).mean(1): (N,) for 2-D, (N, W') for 3-D"""
    dims = dims or img1.dim() - 2
    s = ssim_map(img1, img2, window_size, dims, dtype)
    if size_average:
        return s.mean()
    return s.mean(1).mean(1).mean(1)
