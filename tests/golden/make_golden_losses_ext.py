#!/usr/bin/env python
"""Generate tests/golden/losses_ext.npz by RUNNING THE UNMODIFIED REFERENCE losses in the build container.

Usage (build container only; $PYTORCHDEEPLEARING_REFERENCE does not exist on the GPU box):
    python tests/golden/make_golden_losses_ext.py

``model/losses.py`` is imported from $PYTORCHDEEPLEARING_REFERENCE through the same stub ``model`` package as
make_golden.py.  For every case the file holds the loss value and d loss / d logits of the reference class:
Jaccard / ELDice / Tversky / SS (binary, hard and soft targets), MutilELDice (with and without an absent class) and
LovaszLoss (C = 2 and 5, per_image, ignore, labels outside [0, C), and logits quantised to 1/8 for heavy ties).
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


def import_losses():
    pkg = types.ModuleType("model")
    pkg.__path__ = [os.path.join(REF, "model")]
    sys.modules["model"] = pkg
    return importlib.import_module("model.losses")


def main():
    L = import_losses()
    g = torch.Generator().manual_seed(2024)
    zb = 2.0 * torch.randn((2, 1, 6, 10, 12), generator=g)
    tb = (torch.rand((2, 6, 10, 12), generator=g) > 0.6).long()
    ts = torch.rand((2, 6, 10, 12), generator=g)
    zm = 2.0 * torch.randn((2, 4, 6, 10, 12), generator=g)
    tm = torch.randint(0, 4, (2, 6, 10, 12), generator=g)
    tm_absent = tm.clone()
    tm_absent[tm_absent == 2] = 0
    alpha = torch.tensor([0.5, 1.0, 2.0, 1.5])
    z2 = torch.randn((2, 2, 8, 10, 12), generator=g)
    t2 = torch.randint(0, 2, (2, 8, 10, 12), generator=g)
    t2x = t2.clone()
    t2x[torch.rand(t2.shape, generator=g) < 0.05] = 255       # ignored with ignore=255, else background everywhere
    z5 = torch.randn((2, 5, 6, 8, 10), generator=g)
    t5 = torch.randint(0, 5, (2, 6, 8, 10), generator=g)
    t5[1][t5[1] == 3] = 1                                      # class 3 absent from sample 1 (per_image)
    zq = torch.round(4.0 * torch.randn((2, 3, 8, 8, 8), generator=g)) / 8.0
    tq = torch.randint(0, 3, (2, 8, 8, 8), generator=g)
    cases = {
        "BinaryJaccardLoss": (L.BinaryJaccardLoss(), "zb", "tb"),
        "BinaryJaccardLoss_soft": (L.BinaryJaccardLoss(), "zb", "ts"),
        "BinaryELDiceLoss": (L.BinaryELDiceLoss(), "zb", "tb"),
        "BinaryELDiceLoss_soft": (L.BinaryELDiceLoss(), "zb", "ts"),
        "BinaryTverskyLoss": (L.BinaryTverskyLoss(), "zb", "tb"),
        "BinaryTverskyLoss_soft": (L.BinaryTverskyLoss(), "zb", "ts"),
        "BinarySSLoss": (L.BinarySSLoss(), "zb", "tb"),
        "BinarySSLoss_soft": (L.BinarySSLoss(), "zb", "ts"),
        "MutilELDiceLoss": (L.MutilELDiceLoss(alpha), "zm", "tm"),
        "MutilELDiceLoss_absent": (L.MutilELDiceLoss(alpha), "zm", "tm_absent"),
        "LovaszLoss_c2": (L.LovaszLoss(), "z2", "t2"),
        "LovaszLoss_c2_ignore255": (L.LovaszLoss(ignore=255), "z2", "t2x"),
        "LovaszLoss_c2_outside": (L.LovaszLoss(), "z2", "t2x"),
        "LovaszLoss_c5": (L.LovaszLoss(), "z5", "t5"),
        "LovaszLoss_c5_per_image": (L.LovaszLoss(per_image=True), "z5", "t5"),
        "LovaszLoss_c5_ignore": (L.LovaszLoss(ignore=2), "z5", "t5"),
        "LovaszLoss_c5_per_image_ignore": (L.LovaszLoss(per_image=True, ignore=0), "z5", "t5"),
        "LovaszLoss_ties": (L.LovaszLoss(), "zq", "tq"),
    }
    inputs = {"zb": zb, "tb": tb, "ts": ts, "zm": zm, "tm": tm, "tm_absent": tm_absent, "z2": z2, "t2": t2,
              "t2x": t2x, "z5": z5, "t5": t5, "zq": zq, "tq": tq}
    res = {k: v.numpy() for k, v in inputs.items()}
    res["alpha"] = alpha.numpy()
    for name, (fn, zk, tk) in cases.items():
        z = inputs[zk].clone().requires_grad_(True)
        v = fn(z, inputs[tk])
        v.backward()
        res[name + "_value"] = np.array(v.item())
        res[name + "_grad"] = z.grad.detach().numpy().astype(np.float32).copy()
        print(f"{name}: {v.item():.8f}")
    np.savez_compressed(os.path.join(HERE, "losses_ext.npz"), **res)


if __name__ == "__main__":
    main()
