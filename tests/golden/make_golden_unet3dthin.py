#!/usr/bin/env python
"""Generate tests/golden/unet3dthin.npz by RUNNING THE UNMODIFIED REFERENCE UNet3dthin (networks/Unet3dthin.py).

Usage (needs the reference checkout, which the GPU machines do not have):
    PYTORCHDEEPLEARING_REFERENCE=/path/to/reference python tests/golden/make_golden_unet3dthin.py

Weights come from ``oracle.init_state_dict`` (seeded, randomised affine) and are loaded with
``load_state_dict(strict=True)``, which also proves that ``oracle.unetthin.unetthin_state_spec`` is the reference's
layout.  Per case the file records, under the case tag:
  ``<tag>.logits``        eval-mode logits at every other voxel per axis ([:, :, ::2, ::2, ::2]; keeps the file small)
  ``<tag>.logits_fp``     sum, mean, std, max |.| of the full eval logits
  ``<tag>.argmax_sum``    sum of the full arg-max (sigmoid > 0.5 for one class)
  ``<tag>.loss``          the reference loss on the eval logits
  ``<tag>.grads``         (norm, sum) of every parameter gradient of that loss, in state_dict order
  ``<tag>.train_logits``  train-mode logits (same subsample) after ``torch.manual_seed(<tag>.train_seed)``
and ``init``: (sum, sum of squares) of every tensor of ``UNet3dthin(1, 2)`` built after ``torch.manual_seed(init_seed)``
and passed through the reference's ``initialize_weights``.
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
from oracle import nets as onets  # noqa: E402
from oracle import unetthin as othin  # noqa: E402

# tag: (in_channels, classes, init_features, input shape, weight seed, input seed, loss, train-mode seed)
CASES = {
    "c2_32": (1, 2, 16, (2, 1, 32, 32, 32), 0, 1234, "MutilDiceLoss", 7),
    "c5_32x48x48": (1, 5, 16, (1, 1, 32, 48, 48), 1, 1234, "MutilCrossEntropyDiceLoss", 11),
    "c1_32": (1, 1, 16, (1, 1, 32, 32, 32), 2, 1234, "BinaryDiceLoss", 13),
    "c3_f8_32": (2, 3, 8, (1, 2, 32, 32, 32), 3, 1234, "MutilCrossEntropyDiceLoss", 17),
}


def sub(t: torch.Tensor) -> np.ndarray:
    return t.detach()[:, :, ::2, ::2, ::2].contiguous().numpy().astype(np.float32)


def fingerprint(t: torch.Tensor) -> np.ndarray:
    t = t.detach().double()
    return np.array([t.sum().item(), t.mean().item(), t.std().item(), t.abs().max().item()])


def main():
    torch.set_num_threads(8)
    from networks.Unet3dthin import UNet3dthin
    pkg = types.ModuleType("model")
    pkg.__path__ = [os.path.join(REF, "model")]
    sys.modules["model"] = pkg
    L = importlib.import_module("model.losses")
    out = {}
    for tag, (cin, ncls, f, shape, wseed, xseed, lossname, tseed) in CASES.items():
        spec = othin.unetthin_state_spec(cin, ncls, f)
        sd = onets.init_state_dict(spec, seed=wseed, randomize_affine=True)
        model = UNet3dthin(cin, ncls, init_features=f)
        model.load_state_dict(sd, strict=True)
        names = [n for n, _ in spec]
        assert list(model.state_dict().keys()) == names, "state_dict order differs from the oracle spec"
        x, y = oracle.make_inputs(shape[0], cin, shape[2:], ncls, seed=xseed)
        lossfn = getattr(L, lossname)() if lossname.startswith("Binary") else getattr(L, lossname)(torch.ones(ncls))
        model.eval()
        model.zero_grad()
        logits, probs = model(x)
        loss = lossfn(logits, y)
        loss.backward()
        g = dict(model.named_parameters())
        out[tag + ".logits"] = sub(logits)
        out[tag + ".logits_fp"] = fingerprint(logits)
        am = (probs > 0.5).sum() if ncls == 1 else probs.argmax(1).sum()
        out[tag + ".argmax_sum"] = np.array(int(am.item()))
        out[tag + ".loss"] = np.array(loss.item())
        out[tag + ".grads"] = np.array([[g[n].grad.double().norm().item(), g[n].grad.double().sum().item()]
                                        for n in names])
        model.train()
        torch.manual_seed(tseed)
        with torch.no_grad():
            lt, _ = model(x)
        out[tag + ".train_logits"] = sub(lt)
        out[tag + ".train_seed"] = np.array(tseed)
        print(f"{tag}: loss={loss.item():.7f} logits_sum={out[tag + '.logits_fp'][0]:.4f} "
              f"argmax_sum={int(out[tag + '.argmax_sum'])}")
    from networks import initialize_weights
    torch.manual_seed(5)
    model = UNet3dthin(1, 2)
    model.apply(initialize_weights)
    out["init"] = np.array([[v.double().sum().item(), (v.double() ** 2).sum().item()]
                            for v in model.state_dict().values()])
    out["init_seed"] = np.array(5)
    np.savez_compressed(os.path.join(HERE, "unet3dthin.npz"), **out)


if __name__ == "__main__":
    main()
