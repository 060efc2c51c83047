#!/usr/bin/env python
"""Generate tests/golden/*.npz by RUNNING THE UNMODIFIED REFERENCE in the build container.

Usage (build container only; $PYTORCHDEEPLEARING_REFERENCE does not exist on the GPU box):
    python tests/golden/make_golden.py

The reference modules are imported from $PYTORCHDEEPLEARING_REFERENCE (read-only) with
  * the non-invasive ``VNet3d`` constructor shim for the ``networks/VNet3d.py:127`` typo
    (``self.feature`` vs ``self.features``), and
  * a stub ``model`` package so that ``model/losses.py`` can be imported without the absent
    I/O-only modules (SimpleITK, skimage, torchsummary, matplotlib) -- SURVEY.md App. E.
Weights come from ``oracle.init_state_dict`` (seeded, randomised affine so that biases and
GroupNorm affine parameters matter) and are loaded with ``load_state_dict(strict=True)``,
which also proves the state_dict layout in ``oracle/nets.py`` equals the reference's.
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


def import_reference():
    from networks.VNet3d import VNet3d
    from networks.Unet3d import UNet3d
    from networks.Unet2d import UNet2d

    class VNet3dFixed(VNet3d):
        feature = property(lambda self: self.features)

    pkg = types.ModuleType("model")
    pkg.__path__ = [os.path.join(REF, "model")]
    sys.modules["model"] = pkg
    losses = importlib.import_module("model.losses")
    return VNet3dFixed, UNet3d, UNet2d, losses


def fingerprint(t: torch.Tensor):
    t = t.detach().double()
    return np.array([t.sum().item(), t.mean().item(), t.std().item(), t.abs().max().item()])


def grads_table(module, names):
    g = dict(module.named_parameters())
    return np.array([[g[n].grad.double().norm().item(), g[n].grad.double().sum().item()] for n in names])


def run_case(tag, ref_model, spec, sd, x, y, ref_loss, masks_seed=None):
    out = {}
    names = [n for n, _ in spec]
    ref_model.load_state_dict(sd, strict=True)
    assert list(ref_model.state_dict().keys()) == names, "state_dict order differs from oracle spec"
    ref_model.eval()
    ref_model.zero_grad()
    logits, probs = ref_model(x)
    loss = ref_loss(logits, y)
    loss.backward()
    out["logits_fp"] = fingerprint(logits)
    out["probs_fp"] = fingerprint(probs)
    out["loss"] = np.array(loss.item())
    out["grads"] = grads_table(ref_model, names)
    out["argmax_sum"] = np.array(int(((probs > 0.5).sum() if probs.shape[1] == 1 else probs.argmax(1).sum()).item()))
    out["logits"] = logits.detach().numpy().astype(np.float32)
    if masks_seed is not None:
        ref_model.train()
        torch.manual_seed(masks_seed)
        lt, _ = ref_model(x)
        out["train_logits"] = lt.detach().numpy().astype(np.float32)
        out["train_seed"] = np.array(masks_seed)
        ref_model.eval()
    w = torch.cat([v.double().flatten() for v in sd.values()])
    out["weights_fp"] = np.array([w.sum().item(), w.abs().sum().item(), (w * w).sum().item()])
    out["x_fp"] = fingerprint(x)
    out["y_sum"] = np.array(int(y.sum().item()))
    np.savez_compressed(os.path.join(HERE, tag + ".npz"), **out)
    print(f"{tag}: loss={loss.item():.7f} logits_sum={out['logits_fp'][0]:.4f} argmax_sum={out['argmax_sum']}")
    return out


def main():
    torch.set_num_threads(8)
    VNet3dFixed, UNet3d, UNet2d, L = import_reference()

    # ---- networks ---------------------------------------------------------------------
    spec = onets.vnet3d_state_spec(1, 2)
    sd = onets.init_state_dict(spec, seed=0, randomize_affine=True)
    x, y = oracle.make_inputs(2, 1, (16, 16, 16), 2)
    run_case("vnet3d_c2_16", VNet3dFixed(1, 2), spec, sd, x, y, L.MutilDiceLoss(torch.ones(2)), masks_seed=7)

    x, y = oracle.make_inputs(1, 1, (32, 32, 32), 2)
    run_case("vnet3d_c2_32", VNet3dFixed(1, 2), spec, sd, x, y, L.MutilCrossEntropyDiceLoss(torch.ones(2)))

    spec1 = onets.vnet3d_state_spec(1, 1)
    sd1 = onets.init_state_dict(spec1, seed=3, randomize_affine=True)
    x, y = oracle.make_inputs(1, 1, (16, 16, 16), 1)
    run_case("vnet3d_c1_16", VNet3dFixed(1, 1), spec1, sd1, x, y.unsqueeze(1)[:, 0], L.BinaryDiceLoss())

    spec = onets.unet_state_spec(1, 4, 3)
    sd = onets.init_state_dict(spec, seed=1, randomize_affine=True)
    x, y = oracle.make_inputs(1, 1, (16, 16, 16), 4)
    run_case("unet3d_c4_16", UNet3d(1, 4), spec, sd, x, y, L.MutilCrossEntropyDiceLoss(torch.ones(4)), masks_seed=11)

    spec = onets.unet_state_spec(1, 1, 2)
    sd = onets.init_state_dict(spec, seed=2, randomize_affine=True)
    x, y = oracle.make_inputs(2, 1, (32, 32), 1)

    class DiceFocal(torch.nn.Module):
        def forward(self, z, t):
            return L.BinaryDiceLoss()(z, t) + L.BinaryFocalLoss()(z, t)

    run_case("unet2d_c1_32", UNet2d(1, 1), spec, sd, x, y, DiceFocal(), masks_seed=13)
    x, y = oracle.make_inputs(2, 1, (128, 128), 1)
    o = run_case("unet2d_c1_128", UNet2d(1, 1), spec, sd, x, y, L.BinaryDiceLoss())
    # keep the repo small: the 128x128 case stores fingerprints only
    d = dict(np.load(os.path.join(HERE, "unet2d_c1_128.npz")))
    d.pop("logits")
    np.savez_compressed(os.path.join(HERE, "unet2d_c1_128.npz"), **d)

    # ---- losses on fixed logits (values + d loss / d logits fingerprints) ---------------
    g = torch.Generator().manual_seed(99)
    res = {}
    zb = (2.0 * torch.randn((2, 1, 6, 10, 12), generator=g)).requires_grad_(True)
    tb = (torch.rand((2, 6, 10, 12), generator=g) > 0.6).long()
    zm = (2.0 * torch.randn((2, 4, 6, 10, 12), generator=g)).requires_grad_(True)
    tm = torch.randint(0, 4, (2, 6, 10, 12), generator=g)
    tm_absent = tm.clone()
    tm_absent[tm_absent == 2] = 0
    alpha = torch.tensor([0.5, 1.0, 2.0, 1.5])
    cases = {
        "BinaryDiceLoss": (L.BinaryDiceLoss(), zb, tb),
        "BinaryCrossEntropyLoss": (L.BinaryCrossEntropyLoss(), zb, tb),
        "BinaryFocalLoss": (L.BinaryFocalLoss(), zb, tb),
        "BinaryCrossEntropyDiceLoss": (L.BinaryCrossEntropyDiceLoss(), zb, tb),
        "MutilDiceLoss": (L.MutilDiceLoss(alpha), zm, tm),
        "MutilDiceLoss_absent": (L.MutilDiceLoss(alpha), zm, tm_absent),
        "MutilCrossEntropyLoss": (L.MutilCrossEntropyLoss(alpha), zm, tm),
        "MutilCrossEntropyLoss_absent": (L.MutilCrossEntropyLoss(alpha), zm, tm_absent),
        "MutilFocalLoss": (L.MutilFocalLoss(alpha, gamma=2), zm, tm),
        "MutilFocalLoss_g3": (L.MutilFocalLoss(alpha, gamma=3), zm, tm),
        "MutilCrossEntropyDiceLoss": (L.MutilCrossEntropyDiceLoss(alpha), zm, tm),
    }
    for name, (fn, z, t) in cases.items():
        z.grad = None
        v = fn(z, t)
        v.backward()
        res[name + "_value"] = np.array(v.item())
        res[name + "_grad"] = z.grad.detach().numpy().astype(np.float32).copy()
        print(f"loss {name}: {v.item():.8f}")
    res["zb"] = zb.detach().numpy()
    res["tb"] = tb.numpy()
    res["zm"] = zm.detach().numpy()
    res["tm"] = tm.numpy()
    res["tm_absent"] = tm_absent.numpy()
    res["alpha"] = alpha.numpy()
    np.savez_compressed(os.path.join(HERE, "losses.npz"), **res)


if __name__ == "__main__":
    main()
