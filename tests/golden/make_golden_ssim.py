#!/usr/bin/env python
"""Generate tests/golden/ssim.npz by RUNNING THE UNMODIFIED REFERENCE model/lossesSSIM.py in the build container.

Usage (build container only; $PYTORCHDEEPLEARING_REFERENCE does not exist on the GPU box):
    python tests/golden/make_golden_ssim.py

``model/lossesSSIM.py`` is imported from $PYTORCHDEEPLEARING_REFERENCE through the same stub ``model`` package as
make_golden_losses_ext.py.  For every case the file holds both inputs, the value and the gradients of BOTH inputs
(non-scalar values are backpropagated with a stored random cotangent ``<case>_cot``), and ``taps<k>``, the
reference's 1-D window for every window size used.  Inputs are images in [0, 1) with a correlated second image, and
one 0-255-scaled pair whose large means make sigma^2 = E[x^2] - mu^2 cancel heavily.
"""
import importlib
import os
import sys
import types

import numpy as np
import torch

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PYTORCHDEEPLEARING_REFERENCE", "reference")
sys.path.insert(0, REF)

# name -> (constructor or function name, kwargs, input shape, scale)
CASES = {
    "ssim2d_c1": ("SSIM", {}, (2, 1, 20, 24), 1.0),
    "ssim2d_c3_per_sample": ("SSIM", {"size_average": False}, (2, 3, 20, 24), 1.0),
    "ssim2d_fn_k10": ("ssim", {"window_size": 10}, (2, 2, 17, 21), 1.0),
    "ssim3d_c1": ("SSIM3D", {}, (2, 1, 12, 14, 16), 1.0),
    "ssim3d_c2_per_sample": ("SSIM3D", {"size_average": False}, (2, 2, 12, 14, 16), 1.0),
    "ssim3d_fn_k5": ("ssim3D", {"window_size": 5}, (1, 1, 12, 14, 16), 1.0),
    "ssim3d_fn_k10": ("ssim3D", {"window_size": 10}, (2, 1, 12, 14, 16), 1.0),
    "ssim3d_d3": ("SSIM3D", {}, (1, 1, 3, 14, 16), 1.0),
    "ssim3d_scaled255": ("SSIM3D", {}, (1, 1, 12, 14, 16), 255.0),
}


def import_ssim():
    pkg = types.ModuleType("model")
    pkg.__path__ = [os.path.join(REF, "model")]
    sys.modules["model"] = pkg
    return importlib.import_module("model.lossesSSIM")


def make_pair(shape, scale, g):
    x = torch.rand(shape, generator=g)
    y = (0.7 * x + 0.3 * torch.rand(shape, generator=g)).clamp(0, 1)
    return scale * x, scale * y


def main():
    L = import_ssim()
    g = torch.Generator().manual_seed(2025)
    res = {}
    ks = set()
    for name, (fn, kw, shape, scale) in CASES.items():
        x, y = make_pair(shape, scale, g)
        a, b = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
        if fn in ("SSIM", "SSIM3D"):
            v = getattr(L, fn)(**kw)(a, b)
        else:
            v = getattr(L, fn)(a, b, **kw)
        if v.dim() == 0:
            v.backward()
        else:
            cot = torch.randn(v.shape, generator=g)
            res[name + "_cot"] = cot.numpy()
            v.backward(cot)
        res[name + "_x"], res[name + "_y"] = x.numpy(), y.numpy()
        res[name + "_value"] = v.detach().numpy()
        res[name + "_gx"] = a.grad.numpy()
        res[name + "_gy"] = b.grad.numpy()
        ks.add(kw.get("window_size", 11))
        print(f"{name}: value shape {tuple(v.shape)}, mean {v.detach().mean().item():.6f}")
    for k in sorted(ks):
        res[f"taps{k}"] = L.gaussian(k, 1.5).numpy()
    np.savez_compressed(os.path.join(HERE, "ssim.npz"), **res)


if __name__ == "__main__":
    main()
