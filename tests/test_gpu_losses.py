"""Every hot-path loss class of the drop-in (SURVEY.md rows a11-a18) on the GPU, through the C ABI, against
(1) the fixtures the REAL reference produced (tests/golden/losses.npz: value + d loss / d logits, including the
absent-class and gamma=3 cases; reference model/losses.py:33-53,129-197,247-342) and (2) the CPU oracle on other
shapes / class counts.  Closes the CUDA-vs-reference gap for BinaryDice / BinaryCE / BinaryFocal / MutilCE."""
import os

import numpy as np
import pytest
import torch

import oracle
import pytorchdeeplearing_b200 as b200
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

GOLD_CASES = [
    ("BinaryDiceLoss", "BinaryDiceLoss", "b", None),
    ("BinaryCrossEntropyLoss", "BinaryCrossEntropyLoss", "b", None),
    ("BinaryFocalLoss", "BinaryFocalLoss", "b", None),
    ("BinaryCrossEntropyDiceLoss", "BinaryCrossEntropyDiceLoss", "b", None),
    ("MutilDiceLoss", "MutilDiceLoss", "m", None),
    ("MutilDiceLoss_absent", "MutilDiceLoss", "ma", None),
    ("MutilCrossEntropyLoss", "MutilCrossEntropyLoss", "m", None),
    ("MutilCrossEntropyLoss_absent", "MutilCrossEntropyLoss", "ma", None),
    ("MutilFocalLoss", "MutilFocalLoss", "m", 2),
    ("MutilFocalLoss_g3", "MutilFocalLoss", "m", 3),
    ("MutilCrossEntropyDiceLoss", "MutilCrossEntropyDiceLoss", "m", None),
]


def _make(name, alpha, gamma):
    cls = getattr(b200, name)
    if name.startswith("Binary"):
        return cls()
    if name == "MutilFocalLoss":
        return cls(alpha, gamma=gamma if gamma is not None else 2)
    return cls(alpha)


@pytest.mark.parametrize("key,name,which,gamma", GOLD_CASES)
@pytest.mark.parametrize("channels_last", [False, True])
def test_loss_class_matches_reference_fixture(key, name, which, gamma, channels_last):
    gold = dict(np.load(os.path.join(GOLDEN, "losses.npz")))
    if which == "b":
        z, t = torch.from_numpy(gold["zb"]), torch.from_numpy(gold["tb"])
    else:
        z = torch.from_numpy(gold["zm"])
        t = torch.from_numpy(gold["tm"] if which == "m" else gold["tm_absent"])
    z = z.cuda()
    if channels_last:       # what the drop-in networks hand over: NDHWC memory behind an NCDHW shape
        z = z.permute(0, 2, 3, 4, 1).contiguous().permute(0, 4, 1, 2, 3)
    z.requires_grad_(True)
    alpha = torch.from_numpy(gold["alpha"]).cuda()
    v = _make(name, alpha, gamma)(z, t.cuda())
    assert v.dim() == 0 and v.dtype == torch.float32
    v.backward()
    assert abs(v.item() - float(gold[key + "_value"])) < 3e-6
    ref = torch.from_numpy(gold[key + "_grad"])
    got = z.grad.cpu()
    assert got.shape == ref.shape
    assert (got - ref).abs().max() < 1e-8 + 1e-4 * ref.abs().max()


ORACLE_CASES = [
    ("BinaryDiceLoss", 1, (2, 16, 24, 40)),
    ("BinaryCrossEntropyLoss", 1, (1, 8, 8, 8)),
    ("BinaryFocalLoss", 1, (3, 1, 32, 48)),
    ("BinaryDiceFocalLoss", 1, (2, 1, 64, 64)),
    ("BinaryCrossEntropyDiceLoss", 1, (2, 8, 16, 16)),
    ("MutilDiceLoss", 2, (2, 16, 16, 16)),
    ("MutilCrossEntropyLoss", 3, (2, 8, 24, 16)),
    ("MutilFocalLoss", 5, (1, 8, 16, 40)),
    ("MutilCrossEntropyDiceLoss", 8, (1, 8, 8, 24)),
    ("MutilCrossEntropyDiceLoss", 11, (2, 4, 8, 24)),     # > 8 classes: generic kernels
    ("MutilFocalLoss", 9, (1, 4, 8, 8)),
]


@pytest.mark.parametrize("name,c,shape", ORACLE_CASES)
@pytest.mark.parametrize("gamma", [2, 3])
def test_loss_class_matches_oracle(name, c, shape, gamma):
    if "Focal" not in name and gamma == 3:
        pytest.skip("gamma only enters the focal terms")
    n, sp = shape[0], shape[1:]
    g = torch.Generator().manual_seed(7 + c)
    z = 2.0 * torch.randn((n, c) + sp, generator=g)
    if c == 1:
        t = (torch.rand((n,) + sp, generator=g) > 0.6).long()
    else:
        t = torch.randint(0, c, (n,) + sp, generator=g)
        t[t == c - 1] = 0                                     # one class absent (present-mask path)
    alpha = torch.linspace(0.5, 1.5, c)
    zo = z.clone().requires_grad_(True)
    if name == "BinaryFocalLoss":
        vo = oracle.losses.binary_focal(zo, t, gamma=gamma)
    elif name == "BinaryDiceFocalLoss":
        vo = oracle.losses.binary_dice(zo, t) + oracle.losses.binary_focal(zo, t, gamma=gamma)
    else:
        vo = oracle.loss_forward(name, zo, t, alpha, gamma)
    vo.backward()
    zc = z.cuda().requires_grad_(True)
    if name in ("BinaryFocalLoss", "BinaryDiceFocalLoss"):
        fn = getattr(b200, name)(gamma=gamma)
    else:
        fn = _make(name, alpha.cuda(), gamma)
    v = fn(zc, t.cuda())
    v.backward()
    assert abs(v.item() - vo.item()) < 5e-6 * max(1.0, abs(vo.item()))
    ref = zo.grad
    assert (zc.grad.cpu() - ref).abs().max() < 1e-9 + 2e-4 * ref.abs().max()


def test_out_of_range_labels_raise():
    """The reference raises in F.one_hot / F.cross_entropy for a label outside [0, C) (model/losses.py:254,311);
    the fused kernels flag it and the loss call raises instead of reading out of bounds."""
    z = torch.randn(1, 3, 8, 8, 8, device="cuda")
    t = torch.randint(0, 3, (1, 8, 8, 8), device="cuda")
    t[0, 1, 2, 3] = 3
    with pytest.raises(RuntimeError, match="label"):
        b200.MutilDiceLoss(torch.ones(3).cuda())(z, t)
    t[0, 1, 2, 3] = -1
    with pytest.raises(RuntimeError, match="label"):
        b200.MutilCrossEntropyLoss(torch.ones(3).cuda())(z, t)
    z12 = torch.randn(1, 12, 4, 8, 8, device="cuda")
    t12 = torch.randint(0, 12, (1, 4, 8, 8), device="cuda")
    t12[0, 0, 0, 0] = 255
    with pytest.raises(RuntimeError, match="label"):
        b200.MutilCrossEntropyDiceLoss(torch.ones(12).cuda())(z12, t12)


def test_binary_soft_targets_kept():
    """Binary losses take ``y_true.float()`` in the reference (model/losses.py:47,144): a float target is used as
    is, not truncated to an integer."""
    g = torch.Generator().manual_seed(3)
    z = torch.randn((2, 1, 8, 16, 16), generator=g)
    t = torch.rand((2, 8, 16, 16), generator=g)
    zo = z.clone().requires_grad_(True)
    vo = oracle.losses.binary_bce_dice(zo, t)
    vo.backward()
    zc = z.cuda().requires_grad_(True)
    v = b200.BinaryCrossEntropyDiceLoss()(zc, t.cuda())
    v.backward()
    assert abs(v.item() - vo.item()) < 5e-6
    assert (zc.grad.cpu() - zo.grad).abs().max() < 2e-4 * zo.grad.abs().max()
