"""Restatement of the reference's soft-clDice (model/lossescldice.py) with its four defects repaired as DESIGN.md
section 2 pins them: ``thresh_width`` rounds of ``m = -maxpool(-x); c = relu(maxpool(m) - m); x = relu(x - c)``
(3x3 windows for 4-D input, 3x3x3 for 5-D, stride 1, padding 1), norm_intersection with smooth 1, the binary loss of
lossescldice.py:52-59 and the multi-class loss over ``[:, c:c+1]`` slices of the input and the one-hot target.

``soft_skeletonize`` is the torch operator sequence in the input's dtype: in fp32 it is what the reference computes.
``skeleton_fixed`` is the arbiter the GPU gradient is held to: every round's routing (the min-pool's and max-pool's
argument indices) and its ReLU masks (``relu'(0) = 0``) are taken from the fp32 forward of ``ref``, and the round is
then evaluated in x's dtype (fp64) with those choices: m = x[argmin], M = m[argmax], x' = (x - (M - m) b) a, with
a = [x - c > 0] and b = [M - m > 0].  Gradients come from autograd.  Runs on either device."""
import torch
import torch.nn.functional as F


def _pool(x):
    return F.max_pool2d if x.dim() == 4 else F.max_pool3d


def _win(x):
    return (3, 3) if x.dim() == 4 else (3, 3, 3)


def soft_skeletonize(x, thresh_width=10):
    pool = _pool(x)
    for _ in range(thresh_width):
        m = pool(x * -1, _win(x), 1, 1) * -1
        contour = F.relu(pool(m, _win(x), 1, 1) - m)
        x = F.relu(x - contour)
    return x


def routing(x, thresh_width=10):
    """per round of the fp32 forward of x: (argmin indices, argmax indices, a, b) -- flat spatial indices per (n, c)
    as max_pool returns them, and the two ReLU masks as booleans"""
    pool = _pool(x)
    out = []
    x = x.detach().float()
    for _ in range(thresh_width):
        nm, imin = pool(x * -1, _win(x), 1, 1, return_indices=True)
        m = nm * -1
        M, imax = pool(m, _win(x), 1, 1, return_indices=True)
        d = M - m
        e = x - F.relu(d)
        out.append((imin, imax, e > 0, d > 0))
        x = F.relu(e)
    return out


def _gather(t, idx):
    return t.flatten(2).gather(2, idx.flatten(2)).view_as(t)


def skeleton_fixed(x, thresh_width=10, ref=None):
    """the skeleton of x evaluated in x's dtype with the routing and ReLU masks of the fp32 forward of ``ref``
    (default: x itself rounded to fp32)"""
    plan = routing(x if ref is None else ref, thresh_width)
    for imin, imax, a, b in plan:
        m = _gather(x, imin)
        d = _gather(m, imax) - m
        x = (x - d * b.to(x.dtype)) * a.to(x.dtype)
    return x


def norm_intersection(center_line, vessel, smooth=1.0):
    clf = center_line.reshape(*center_line.shape[:2], -1)
    vf = vessel.reshape(*vessel.shape[:2], -1)
    return ((clf * vf).sum(-1) + smooth) / (clf.sum(-1) + smooth)


def binary_loss(pred, target, skeleton=soft_skeletonize, smooth=1e-5, eps=1e-7):
    iflat = norm_intersection(skeleton(pred), target)
    tflat = norm_intersection(skeleton(target), pred)
    intersection = iflat * tflat
    cldsc = (2. * intersection.sum() + smooth) / (iflat.sum() + tflat.sum() + smooth).clamp_min(eps)
    return (1. - cldsc).mean()


def one_hot(labels, c, like):
    """(N, *spatial) or (N, 1, *spatial) integer labels -> one-hot (N, C, *spatial) in like's dtype"""
    y = F.one_hot(labels.long().reshape(labels.shape[0], -1), c).permute(0, 2, 1)
    return y.reshape(like.shape).to(like.dtype)


def mutil_loss(inp, labels, alpha, skeleton=soft_skeletonize, smooth=1e-5, eps=1e-7):
    c = inp.shape[1]
    y = one_hot(labels, c, inp)
    dice = 0
    for k in range(c):
        dice = dice + binary_loss(inp[:, k:k + 1], y[:, k:k + 1], skeleton, smooth, eps) * alpha[k]
    return dice / c


def fixed_skeleton(x, thresh_width=10):
    """the ``skeleton`` argument of binary_loss / mutil_loss for the fp64 arbiter: x (an fp64 copy of fp32 values, so
    rounding it back is exact) routed by its own fp32 forward"""
    return skeleton_fixed(x, thresh_width, ref=x.detach().float())
