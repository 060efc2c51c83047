#!/usr/bin/env python
"""Generate tests/golden/cldice.npz by RUNNING THE REFERENCE's OWN model/lossescldice.py bodies in the build container.

Usage (build container only; $PYTORCHDEEPLEARING_REFERENCE does not exist on the GPU box):
    python tests/golden/make_golden_cldice.py

The module raises as shipped; its defects are bridged outside the source, which is not changed:
  * ``soft_skeletonize`` calls ``x.size().tolist()`` and compares the result with 4 / 5 (lossescldice.py:10-16).  The
    inputs are given as ``RankSized`` tensors, a subclass whose ``size()`` returns a tuple whose ``tolist()``
    is the rank, so the reference's own 2-D / 3-D loop runs.
  * ``Binary_Soft_cldice_loss`` defines ``__int__`` instead of ``__init__`` (lossescldice.py:42): each instance's own
    ``__int__()`` is called once after construction, which sets ``smooth = 1e-5`` and ``eps = 1e-7``.
  * ``Mutil_Soft_cldice_loss.forward`` indexes ``input[:, c, ...]`` and drops the channel axis (lossescldice.py:83).
    Its six-line loop is restated in ``mutil`` below with ``[:, c:c+1]``; the binary loss it calls is the reference's.
Predictions lie on the grid k / 256 (see ``quantize``), and so do both skeletons (each round only selects and subtracts
grid values); those three arrays are stored as their exact uint16 codes k (``grid_code``; the value is k / 256 in
fp32).  Per case: pred, target (uint8: 0 / 1 for the binary cases, class labels for the multi-class cases, plus
alpha), the reference's skeletons of pred and of the (one-hot) target, the loss (fp32), and the full gradient with
respect to pred (fp32).
"""
import importlib
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PYTORCHDEEPLEARING_REFERENCE", "reference")
sys.path.insert(0, REF)


class _RankSize(tuple):
    """the size tuple, with ``tolist()`` answering the rank"""

    def tolist(self):
        return len(self)


class RankSized(torch.Tensor):
    """a tensor whose ``size()`` answers ``tolist()`` with its rank (the bridge for lossescldice.py:10)"""

    def size(self, *args):
        s = super().size(*args)
        return s if args else _RankSize(s)


def import_cldice():
    pkg = types.ModuleType("model")
    pkg.__path__ = [os.path.join(REF, "model")]
    sys.modules["model"] = pkg
    return importlib.import_module("model.lossescldice")


def binary_loss(L):
    loss = L.Binary_Soft_cldice_loss()
    loss.__int__()                  # the reference's intended initialiser
    return loss


def mutil(L, inp, target, alpha):
    """Mutil_Soft_cldice_loss.forward (lossescldice.py:75-84) with the channel axis kept: [:, c:c+1]"""
    bscldice = binary_loss(L)
    Batchsize, Channel = inp.shape[0], inp.shape[1]
    y_true = target.long().contiguous().view(Batchsize, -1)
    y_true = F.one_hot(y_true, Channel).permute(0, 2, 1).reshape(inp.shape).float().as_subclass(RankSized)
    dice = 0
    for channel in range(0, Channel):
        dice += bscldice(inp[:, channel:channel + 1, ...], y_true[:, channel:channel + 1, ...]) * alpha[channel]
    return dice / Channel, y_true


def smooth_noise(shape, g, passes=2):
    x = torch.rand(shape, generator=g)
    pool = F.avg_pool2d if len(shape) == 4 else F.avg_pool3d
    for _ in range(passes):
        x = pool(x, 3, 1, 1)
    return (x - x.mean()) / x.std()


def quantize(x):
    """values on the grid k / 256: exact in fp32, every round's differences stay on the grid, ties are frequent, and
    the stored arrays compress to a small fixture"""
    return torch.round(x * 256.0) / 256.0


def grid_code(x):
    """an fp32 array on the grid k / 256 in [0, 1] -> its exact uint16 codes k (x = k / 256 bit for bit)"""
    k = torch.round(x * 256.0)
    assert torch.equal(k / 256.0, x) and k.min() >= 0 and k.max() <= 256
    return k.numpy().astype(np.uint16)


# name -> (shape, kind): "random" preds in (0, 1); "plateau" preds clamped to exact 0 / 1 plateaus
CASES = {
    "bin2d": ((2, 1, 64, 64), "random"),
    "bin3d_plateau": ((2, 1, 32, 32, 32), "plateau"),
    "mutil3d_c3": ((2, 3, 16, 16, 16), "random"),
    "mutil2d_c3": ((2, 3, 48, 48), "plateau"),
}
ALPHA = [0.5, 1.0, 2.0]


def main():
    L = import_cldice()
    g = torch.Generator().manual_seed(2026)
    res = {}
    for name, (shape, kind) in CASES.items():
        n, c = shape[:2]
        z = smooth_noise(shape, g)
        pred = quantize(torch.sigmoid(3.0 * z)) if kind == "random" else quantize((0.5 + z).clamp(0, 1))
        if name.startswith("bin"):
            target = (smooth_noise(shape, g) > 0.3).float()
            p = pred.clone().requires_grad_(True)
            loss = binary_loss(L)(p.as_subclass(RankSized), target.as_subclass(RankSized))
            tsk = L.soft_skeletonize(target.as_subclass(RankSized))
        else:
            if kind == "random":
                pred = quantize(torch.softmax(3.0 * z, 1))
            target = smooth_noise((n, c) + shape[2:], g).argmax(1)
            p = pred.clone().requires_grad_(True)
            loss, onehot = mutil(L, p.as_subclass(RankSized), target, ALPHA)
            tsk = L.soft_skeletonize(onehot)
            res[name + "_alpha"] = np.array(ALPHA, dtype=np.float32)
        psk = L.soft_skeletonize(pred.as_subclass(RankSized))
        loss.backward()
        res[name + "_pred"] = grid_code(pred)
        res[name + "_target"] = target.numpy().astype(np.uint8)      # 0 / 1 targets and class labels < 256
        res[name + "_sk_pred"] = grid_code(psk.as_subclass(torch.Tensor).detach())
        res[name + "_sk_target"] = grid_code(tsk.as_subclass(torch.Tensor).detach())
        res[name + "_loss"] = np.array(loss.item(), dtype=np.float32)
        res[name + "_grad"] = p.grad.numpy()
        print(f"{name}: loss {loss.item():.6f}, skeleton mass {psk.sum().item():.2f}, "
              f"zeros in pred {(pred == 0).sum().item()}, ones {(pred == 1).sum().item()}")
    np.savez_compressed(os.path.join(HERE, "cldice.npz"), **res)


if __name__ == "__main__":
    main()
