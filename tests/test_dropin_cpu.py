"""The drop-in's reference-facing contract on the emulated backend, against tests/golden/dropin.json."""
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import runtime
from emu_backend import EmuBackend

_GDIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN = json.load(open(os.path.join(_GDIR, "dropin.json")))
sys.path.insert(0, _GDIR)
from make_golden_dropin import layout_digest, init_digest  # noqa: E402


@pytest.fixture()
def emu():
    runtime._set_backend_for_testing(EmuBackend())
    prev = runtime.get_precision()
    runtime.set_precision("fp32")
    yield
    b200.uninstall()
    runtime._set_backend_for_testing(None)
    runtime.set_precision(prev)


@pytest.fixture()
def ref_tree(monkeypatch):
    """stand-ins binding the names the reference modules bind"""
    mods = {}
    for modname, names in GOLDEN["bindings"].items():
        m = types.ModuleType(modname)
        for n in names:
            setattr(m, n, type(n, (), {"__module__": modname}))
        monkeypatch.setitem(sys.modules, modname, m)
        mods[modname] = m
    yield mods
    b200.uninstall()


def test_install_rebinds_and_uninstall_restores(ref_tree):
    mv, mu, ml, mm = (ref_tree[k] for k in ("model.modelVNet", "model.modelUnet", "model.losses", "model.metric"))
    orig = {"VNet3d": mv.VNet3d, "UNet2d": mu.UNet2d, "dice": mv.dice_coeff, "loss": ml.BinaryDiceLoss}
    n = b200.install()
    assert n == sum(len(v) for v in GOLDEN["bindings"].values())
    assert n >= 20
    assert mv.VNet3d is b200.VNet3d and mv.VNet2d is b200.VNet2d
    assert mu.UNet2d is b200.UNet2d and mu.UNet3d is b200.UNet3d
    assert mv.MutilDiceLoss is b200.MutilDiceLoss and mu.BinaryFocalLoss is b200.BinaryFocalLoss
    assert ml.MutilCrossEntropyDiceLoss is b200.MutilCrossEntropyDiceLoss
    assert mv.dice_coeff is b200.dice_coeff and mm.multiclass_dice_coeff is b200.multiclass_dice_coeff
    assert ref_tree["networks.VNet3d"].VNet3d is b200.VNet3d
    assert b200.install() == 0                                   # idempotent
    b200.uninstall()
    assert mv.VNet3d is orig["VNet3d"] and mu.UNet2d is orig["UNet2d"]
    assert mv.dice_coeff is orig["dice"] and ml.BinaryDiceLoss is orig["loss"]


def test_state_dict_layout_and_init_match_reference_golden(emu):
    """state_dict layouts equal the reference networks' and initialize_weights leaves what the reference's does"""
    nets = {"VNet3d(1,2)": b200.VNet3d(1, 2), "VNet2d(1,1)": b200.VNet2d(1, 1), "UNet3d(1,4)": b200.UNet3d(1, 4),
            "UNet2d(1,1)": b200.UNet2d(1, 1)}
    for key, m in nets.items():
        assert layout_digest(m) == GOLDEN["layouts"][key], key
    sd = nets["VNet3d(1,2)"].state_dict()
    assert len(sd) == 128 and sum(v.numel() for v in sd.values()) == 9492658      # SURVEY.md App. A
    assert list(sd)[:4] == ["in_tr.conv1.weight", "in_tr.conv1.bias", "in_tr.conv2.weight", "in_tr.conv2.bias"]
    assert len(nets["UNet2d(1,1)"].state_dict()) == 64 and len(nets["VNet2d(1,1)"].state_dict()) == 128
    for key in ("VNet3d(1,2)", "UNet2d(1,1)"):
        m = nets[key]
        m.apply(b200.initialize_weights)
        assert init_digest(m) == GOLDEN["init"][key], key
    for name in GOLDEN["bindings"]["model.losses"]:
        assert isinstance(getattr(b200, name)(*([torch.ones(2)] if name.startswith("Mutil") else [])),
                          torch.nn.Module)


def test_one_training_step_on_the_dropin(emu, tmp_path):
    """one training step (forward, loss, Dice, AdamW), a checkpoint round trip and predict on UNet2d"""
    rng = np.random.RandomState(0)
    imgs = torch.as_tensor(rng.rand(2, 1, 32, 32).astype(np.float32))
    masks = torch.as_tensor((rng.rand(2, 1, 32, 32) > 0.7).astype(np.float32))
    torch.manual_seed(0)
    model = b200.UNet2d(1, 1)
    model.apply(b200.initialize_weights)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    lossfn = b200.BinaryDiceLoss()
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3)
    model.train()
    logits, probs = model(imgs)
    loss = lossfn(logits, masks)
    dice = b200.dice_coeff(probs.detach(), masks)
    opt.zero_grad()
    loss.backward()
    opt.step()
    assert torch.isfinite(loss) and 0.0 <= float(dice) <= 1.0
    ckpt = tmp_path / "BinaryUNet2d.pth"
    torch.save(model.state_dict(), str(ckpt))
    sd = torch.load(str(ckpt))
    assert list(sd.keys()) == list(before.keys()) and len(sd) == 64
    assert all(torch.isfinite(v).all() for v in sd.values())
    changed = sum(int(not torch.equal(sd[k], before[k])) for k in sd)
    assert changed > 32                                          # one AdamW step moved them
    model.load_state_dict(sd)
    pred = b200.predict(model, np.zeros((1, 32, 32), np.float32))
    assert pred.shape == (32, 32) and pred.dtype == np.uint8
