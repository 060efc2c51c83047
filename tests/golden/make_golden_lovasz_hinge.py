#!/usr/bin/env python
"""Generate tests/golden/lovasz_hinge.npz by RUNNING THE UNMODIFIED REFERENCE binary Lovasz hinge in the build container.

Usage (build container only; $PYTORCHDEEPLEARING_REFERENCE does not exist on the GPU box):
    python tests/golden/make_golden_lovasz_hinge.py

``model/losses.py`` is imported from $PYTORCHDEEPLEARING_REFERENCE through the same stub ``model`` package as
make_golden_losses_ext.py.  ``BinaryLovaszLoss()`` constructs there, but its ``super(BinaryLovaszLoss).__init__()`` is
an unbound super, so nn.Module.__init__ never runs and calling the object raises AttributeError; the script asserts
that, then runs the class's ``forward`` body on the constructed object and ``model.lovasz._lovasz_hinge`` itself with
the same arguments, asserts the two agree bit for bit, and stores the value and d loss / d logits of every case.
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
    return importlib.import_module("model.losses"), importlib.import_module("model.lovasz")


def main():
    L, LZ = import_losses()
    g = torch.Generator().manual_seed(2025)
    z3 = 2.0 * torch.randn((2, 1, 6, 10, 12), generator=g)
    t3 = (torch.rand((2, 6, 10, 12), generator=g) > 0.6).long()
    t3x = t3.clone()
    t3x[torch.rand(t3.shape, generator=g) < 0.05] = 255
    t3one = t3.clone()
    t3one[1] = 255                                               # sample 1 entirely ignored
    t3zero = torch.zeros_like(t3)                                # no foreground
    zsat = (2.0 * t3 - 1.0).unsqueeze(1) * (1.0 + torch.rand((2, 1, 6, 10, 12), generator=g))   # every margin met
    zq = torch.round(4.0 * torch.randn((2, 1, 6, 10, 12), generator=g)) / 8.0                 # heavy ties
    z2 = 2.0 * torch.randn((3, 1, 16, 20), generator=g)
    t2 = (torch.rand((3, 16, 20), generator=g) > 0.5).long()
    zc = 2.0 * torch.randn((4, 1), generator=g)
    tc = torch.tensor([1, 0, 1, 1])
    inputs = {"z3": z3, "t3": t3, "t3x": t3x, "t3one": t3one, "t3zero": t3zero, "zsat": zsat, "zq": zq, "z2": z2,
              "t2": t2, "zc": zc, "tc": tc}
    cases = {
        "b3": ("z3", "t3", {}),
        "b3_per_image": ("z3", "t3", {"per_image": True}),
        "ignore255": ("z3", "t3x", {"ignore_index": 255}),
        "one_ignored": ("z3", "t3one", {"ignore_index": 255}),
        "one_ignored_per_image": ("z3", "t3one", {"per_image": True, "ignore_index": 255}),
        "no_fg": ("z3", "t3zero", {}),
        "satisfied": ("zsat", "t3", {}),
        "ties": ("zq", "t3", {}),
        "b2": ("z2", "t2", {}),
        "cls": ("zc", "tc", {}),
    }
    obj = L.BinaryLovaszLoss()
    try:
        obj(z3, t3)
    except AttributeError:
        pass
    else:
        raise AssertionError("the reference BinaryLovaszLoss object was expected not to be callable")
    res = {k: v.numpy() for k, v in inputs.items()}
    for name, (zk, tk, kw) in cases.items():
        obj = L.BinaryLovaszLoss(**kw)
        out = []
        for fn in (lambda z, t: L.BinaryLovaszLoss.forward(obj, z, t),
                   lambda z, t: LZ._lovasz_hinge(z, t, per_image=kw.get("per_image", False),
                                                 ignore_index=kw.get("ignore_index"))):
            z = inputs[zk].clone().requires_grad_(True)
            v = fn(z, inputs[tk])
            v.backward()
            out.append((v.item(), z.grad.detach().numpy().astype(np.float32).copy()))
        assert out[0][0] == out[1][0] and np.array_equal(out[0][1], out[1][1]), name
        res[name + "_value"] = np.array(out[0][0])
        res[name + "_grad"] = out[0][1]
        print(f"{name}: {out[0][0]:.8f}")
    np.savez_compressed(os.path.join(HERE, "lovasz_hinge.npz"), **res)


if __name__ == "__main__":
    main()
