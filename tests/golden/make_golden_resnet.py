#!/usr/bin/env python
"""Generate tests/golden/resnet.npz by RUNNING THE UNMODIFIED REFERENCE classifiers (networks/ResNet2d.py,
networks/ResNet3d.py) and losses (model/losses.py).

Usage (needs the reference checkout at $PYTORCHDEEPLEARING_REFERENCE):
    python tests/golden/make_golden_resnet.py

The reference's ``DownTransition*.__init__`` reads an undefined module global ``prob`` (ResNet3d.py:51): it is set to
0.2 in the imported module's namespace before construction; the reference's source is not changed.  Weights come from
``oracle.init_state_dict`` over ``oracle.resnet.resnet_state_spec`` and are loaded with ``strict=True``.

Per case (net, loss): eval-mode logits, the loss and a (norm, sum) table of every parameter gradient.  Per net:
train-mode logits after ``torch.manual_seed(TRAIN_SEED)`` (the reference's train-mode backward raises, see
oracle/resnet.py, so only its forward is recorded).
"""
import importlib
import os
import sys
import types

import numpy as np
import torch

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ.get("PYTORCHDEEPLEARING_REFERENCE", "reference")
sys.path.insert(0, REF)

import oracle  # noqa: E402
from oracle import resnet as ores  # noqa: E402

TRAIN_SEED = 11
# (tag, dims, spatial, batch, numclass, loss, weight seed)
CASES = [
    ("r2d_k10_ce", 2, (64, 64), 4, 10, "MutilCrossEntropyLoss", 0),
    ("r2d_k10_focal", 2, (64, 64), 4, 10, "MutilFocalLoss", 0),
    ("r2d_k1_bce", 2, (64, 64), 4, 1, "BinaryCrossEntropyLoss", 1),
    ("r2d_k1_focal", 2, (64, 64), 4, 1, "BinaryFocalLoss", 1),
    ("r3d_k4_ce", 3, (32, 32, 32), 2, 4, "MutilCrossEntropyLoss", 2),
    ("r3d_k4_focal", 3, (32, 32, 32), 2, 4, "MutilFocalLoss", 2),
    ("r3d_k1_bce", 3, (32, 32, 32), 2, 1, "BinaryCrossEntropyLoss", 3),
    ("r3d_k1_focal", 3, (32, 32, 32), 2, 1, "BinaryFocalLoss", 3),
]


def case_inputs(dims, spatial, n, k, seed):
    """x ~ N(0, 1) (oracle.make_inputs); labels: (N,) int64 class indices, or (N, 1) fp32 0/1 for one class"""
    x, _ = oracle.make_inputs(n, 1, spatial, 2, seed=100 + seed)
    g = torch.Generator().manual_seed(200 + seed)
    if k == 1:
        y = (torch.rand((n, 1), generator=g) > 0.5).float()
    else:
        y = torch.randint(0, k, (n,), generator=g)
    return x, y


def import_reference():
    nets = {}
    for dims in (2, 3):
        mod = importlib.import_module(f"networks.ResNet{dims}d")
        mod.prob = 0.2
        nets[dims] = getattr(mod, f"ResNet{dims}d")
    pkg = types.ModuleType("model")
    pkg.__path__ = [os.path.join(REF, "model")]
    sys.modules["model"] = pkg
    return nets, importlib.import_module("model.losses")


def make_loss(losses, name):
    return getattr(losses, name)(torch.ones(1)) if name.startswith("Mutil") else getattr(losses, name)()


def main():
    nets, losses = import_reference()
    out = {"train_seed": np.array(TRAIN_SEED)}
    for tag, dims, spatial, n, k, lossname, seed in CASES:
        spec = ores.resnet_state_spec(1, k, dims)
        sd = oracle.init_state_dict(spec, seed=seed, randomize_affine=True)
        model = nets[dims](1, k)
        assert [s for s, _ in spec] == list(model.state_dict().keys())
        model.load_state_dict(sd, strict=True)
        x, y = case_inputs(dims, spatial, n, k, seed)
        model.eval()
        logits = model(x)
        loss = make_loss(losses, lossname)(logits, y)
        loss.backward()
        g = dict(model.named_parameters())
        out[tag + "_logits"] = logits.detach().numpy()
        out[tag + "_loss"] = np.array(loss.item())
        out[tag + "_grads"] = np.array([[g[s].grad.double().norm().item(), g[s].grad.double().sum().item()]
                                        for s, _ in spec])
        if lossname.endswith("CrossEntropyLoss"):
            model.train()
            torch.manual_seed(TRAIN_SEED)
            with torch.no_grad():
                out[tag + "_train_logits"] = model(x).numpy()
    path = os.path.join(HERE, "resnet.npz")
    np.savez_compressed(path, **out)
    print(path, len(out))


if __name__ == "__main__":
    main()
