"""The further reference losses (Jaccard, ELDice, Tversky, SS, MutilELDice, Lovasz-Softmax) without a GPU: the CPU
oracle against the fixtures the real reference produced (tests/golden/losses_ext.npz), the C == 1 refusal of
LovaszLoss, install()/uninstall() of the six names, and GraphedStep / loss_spec on the emulated backend."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import losses_ext as ox
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import losses as bl, runtime
from conftest import GOLDEN
from emu_backend import EmuBackend

NEW = ("BinaryJaccardLoss", "BinaryELDiceLoss", "BinarySSLoss", "BinaryTverskyLoss", "MutilELDiceLoss", "LovaszLoss")

SUM_CASES = [
    ("BinaryJaccardLoss", "zb", "tb", ox.binary_jaccard),
    ("BinaryJaccardLoss_soft", "zb", "ts", ox.binary_jaccard),
    ("BinaryELDiceLoss", "zb", "tb", ox.binary_eldice),
    ("BinaryELDiceLoss_soft", "zb", "ts", ox.binary_eldice),
    ("BinaryTverskyLoss", "zb", "tb", ox.binary_tversky),
    ("BinaryTverskyLoss_soft", "zb", "ts", ox.binary_tversky),
    ("BinarySSLoss", "zb", "tb", ox.binary_ss),
    ("BinarySSLoss_soft", "zb", "ts", ox.binary_ss),
    ("MutilELDiceLoss", "zm", "tm", None),
    ("MutilELDiceLoss_absent", "zm", "tm_absent", None),
]
LOVASZ_CASES = [
    ("LovaszLoss_c2", "z2", "t2", {}),
    ("LovaszLoss_c2_ignore255", "z2", "t2x", {"ignore": 255}),
    ("LovaszLoss_c2_outside", "z2", "t2x", {}),
    ("LovaszLoss_c5", "z5", "t5", {}),
    ("LovaszLoss_c5_per_image", "z5", "t5", {"per_image": True}),
    ("LovaszLoss_c5_ignore", "z5", "t5", {"ignore": 2}),
    ("LovaszLoss_c5_per_image_ignore", "z5", "t5", {"per_image": True, "ignore": 0}),
    ("LovaszLoss_ties", "zq", "tq", {}),
]


def _gold():
    return dict(np.load(os.path.join(GOLDEN, "losses_ext.npz")))


@pytest.mark.parametrize("key,zk,tk,fn", SUM_CASES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_sum_based_oracle_matches_reference_fixture(key, zk, tk, fn, dtype):
    gold = _gold()
    z = torch.from_numpy(gold[zk]).requires_grad_(True)
    t = torch.from_numpy(gold[tk])
    if fn is None:
        v = ox.multi_eldice(z, t, torch.from_numpy(gold["alpha"]), dtype=dtype)
    else:
        v = fn(z, t, dtype=dtype)
    v.backward()
    assert abs(v.item() - float(gold[key + "_value"])) < 2e-6
    ref = torch.from_numpy(gold[key + "_grad"])
    assert (z.grad.float() - ref).abs().max() < 1e-4 * ref.abs().max() + 1e-9


@pytest.mark.parametrize("key,zk,tk,kw", LOVASZ_CASES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_lovasz_oracle_matches_reference_fixture(key, zk, tk, kw, dtype):
    """fp32: the reference's own arithmetic; fp64: the restatement the GPU kernels are held to (stable tie order, fp64
    Lovasz gradient).  The value agrees to round-off; the fp32 gradient carries the cancellation of
    jaccard[1:] - jaccard[:-1] (model/lovasz.py:31), hence the looser gradient bound.  On the tie-heavy input the
    reference's unstable torch.sort orders ties differently, which moves the gradient but not the value."""
    gold = _gold()
    z = torch.from_numpy(gold[zk]).requires_grad_(True)
    v = ox.lovasz_softmax(z, torch.from_numpy(gold[tk]), dtype=dtype, **kw)
    v.backward()
    want = float(gold[key + "_value"])
    assert abs(v.item() - want) < 1e-6 * max(1.0, abs(want))
    if key == "LovaszLoss_ties":
        return
    ref = torch.from_numpy(gold[key + "_grad"])
    assert (z.grad.float() - ref).abs().max() < 1e-2 * ref.abs().max()


def test_lovasz_with_one_class_raises():
    with pytest.raises(ValueError, match="Sigmoid output possible only with 1 class"):
        b200.LovaszLoss()(torch.rand(1, 1, 4, 4, 4), torch.zeros(1, 4, 4, 4, dtype=torch.long))


def test_new_classes_keep_the_reference_attributes():
    assert (b200.BinaryJaccardLoss().smooth, b200.BinaryJaccardLoss().eps) == (1e-5, 1e-7)
    assert (b200.BinaryELDiceLoss().smooth, b200.BinaryELDiceLoss().eps) == (1e-5, 1e-7)
    assert (b200.BinarySSLoss().smooth, b200.BinarySSLoss().r) == (1e-5, 0.1)
    tv = b200.BinaryTverskyLoss()
    assert (tv.smooth, tv.alpha, tv.beta) == (1e-5, 0.3, 0.7)
    assert b200.MutilELDiceLoss([1.0, 2.0]).alpha == [1.0, 2.0]
    lv = b200.LovaszLoss(per_image=True, ignore=255)
    assert (lv.per_image, lv.ignore) == (True, 255)
    assert bl.loss_spec(tv) == (bl.TVERSKY, None, 0.7, 0.3)
    assert bl.loss_spec(b200.BinarySSLoss())[0] == bl.SS and bl.loss_spec(b200.BinarySSLoss())[3] == 0.1
    assert bl.loss_spec(b200.MutilELDiceLoss([1.0, 2.0]))[:2] == (bl.ELDICE, [1.0, 2.0])
    assert bl.loss_spec(lv)[0] == bl.LOVASZ


def test_install_rebinds_the_six_names_and_uninstall_restores(monkeypatch):
    m = types.ModuleType("model.losses")
    orig = {n: type(n, (), {}) for n in NEW}
    for n, o in orig.items():
        setattr(m, n, o)
    monkeypatch.setitem(sys.modules, "model.losses", m)
    try:
        assert b200.install() == len(NEW)
        for n in NEW:
            assert getattr(m, n) is getattr(b200, n)
    finally:
        b200.uninstall()
    for n in NEW:
        assert getattr(m, n) is orig[n]


# ------------------------------------------------------------------------------------------------ emulated backend
class _ExtEmu(EmuBackend):
    """EmuBackend plus the new entry points, in fp64 torch: the sum-based finalize differentiates the closed form with
    respect to the partial sums (d loss / d p = a t + b with a = dL/dI, b = dL/dP); Lovasz keeps the whole gradient
    in ``coef``."""

    def loss_partials_ss(self, logits, labels, part, metric=None):
        super().loss_partials(logits, labels, 2.0, 0.25, part, metric)
        z, t = logits.reshape(-1).double(), labels.reshape(-1).double()
        se = (torch.sigmoid(z) - t) ** 2
        part[3] = (se * t).sum()           # in place of the cross-entropy / focal sums
        part[4] = (se * (1 - t)).sum()

    def loss_finalize(self, part, c, terms, alpha, gamma, alpha_f, loss, lcoef):
        if not terms & (bl.JACCARD | bl.ELDICE | bl.TVERSKY | bl.SS):
            return super().loss_finalize(part, c, terms, alpha, gamma, alpha_f, loss, lcoef)
        pt = part.double()
        lcoef.zero_()
        with torch.enable_grad():
            return self._finalize_ext(pt, c, terms, alpha, gamma, alpha_f, loss, lcoef)

    @staticmethod
    def _finalize_ext(pt, c, terms, alpha, gamma, alpha_f, loss, lcoef):
        s, eps = 1e-5, 1e-7
        if c == 1:
            I, P = pt[0].clone().requires_grad_(True), pt[1].clone().requires_grad_(True)
            T, V = pt[2], pt[5]
            if terms == bl.JACCARD:
                val = 1 - (I + s) / (P + T - I + s).clamp_min(eps)
            elif terms == bl.ELDICE:
                val = torch.clamp(torch.pow(-torch.log((2 * I + s) / (P + T + s).clamp_min(eps) + s), 0.3), 0, 2)
            elif terms == bl.TVERSKY:
                val = torch.clamp(1 - (I + s) / (I + alpha_f * (P - I) + gamma * (T - I) + s), 0, 2)
            else:
                r = alpha_f
                loss.copy_((r * pt[3] / (s + T) + (1 - r) * pt[4] / (s + V - T)).float())
                lcoef[0], lcoef[1] = float(r / (s + T)), float((1 - r) / (s + V - T))
                return
            gI, gP = torch.autograd.grad(val, (I, P))
            lcoef[0], lcoef[1] = float(gI), float(gP)
        else:
            I, Ps = pt[0:c].clone().requires_grad_(True), pt[c:2 * c].clone().requires_grad_(True)
            Cn = pt[2 * c:3 * c]
            present = (Cn > 0).double()
            d = ((2 * I + s) / (Cn + Ps + s)).clamp_min(eps) * present * alpha.double()
            val = torch.clamp(torch.pow(-torch.log(d + s), 0.3).sum() / present.sum(), 0, 2)
            gI, gP = torch.autograd.grad(val, (I, Ps))
            lcoef[0:c], lcoef[c:2 * c] = gI.float(), gP.float()
        loss.copy_(val.detach().float())

    def loss_bwd_ss(self, logits, labels, lcoef, gscale, dlogits):
        z, t = logits.reshape(-1).double(), labels.reshape(-1).double()
        p = torch.sigmoid(z)
        wf, wb = float(lcoef[0]), float(lcoef[1])
        g = 2 * (p - t) * (wf * t + wb * (1 - t)) * p * (1 - p) * gscale.double()
        dlogits.copy_(g.float().reshape(dlogits.shape))

    def lovasz_fwd(self, logits, labels, per_image, ignore, loss, coef, seg_scale):
        dims = logits.dim()
        z = logits.detach().double().movedim(-1, 1).requires_grad_(True)
        with torch.enable_grad():
            v = ox.lovasz_softmax(z, labels, per_image=per_image, ignore=ignore, dtype=torch.float64)
            g, = torch.autograd.grad(v, z) if v.requires_grad else (torch.zeros_like(z),)
        coef.copy_(g.movedim(1, dims - 1).float())
        loss.copy_(v.detach().float())

    def lovasz_bwd(self, logits, labels, per_image, coef, seg_scale, gscale, dlogits):
        dlogits.copy_(coef * gscale)


@pytest.fixture()
def emu():
    runtime._set_backend_for_testing(_ExtEmu())
    prev = runtime.get_precision()
    runtime.set_precision("fp32")
    yield
    runtime._set_backend_for_testing(None)
    runtime.set_precision(prev)


@pytest.mark.parametrize("lossname,ncls", [("BinaryTverskyLoss", 1), ("BinarySSLoss", 1), ("BinaryJaccardLoss", 1),
                                           ("MutilELDiceLoss", 2), ("LovaszLoss", 2)])
def test_graphed_step_takes_the_new_losses_on_the_emulated_backend(emu, lossname, ncls):
    """the step program (GraphedStep, eager form) and the autograd path give the same loss and gradients"""
    import oracle
    from oracle import nets as onets
    from pytorchdeeplearing_b200.graphed import GraphedStep
    spec = onets.unet_state_spec(1, ncls, 2)
    sd = onets.init_state_dict(spec, seed=4, randomize_affine=True)
    model = b200.UNet2d(1, ncls)
    model.load_state_dict(sd, strict=True)
    model.eval()
    x, y = oracle.make_inputs(2, 1, (16, 16), ncls, seed=9)
    lossfn = getattr(b200, lossname)(torch.ones(ncls)) if lossname.startswith("Mutil") else getattr(b200, lossname)()
    logits, _ = model(x)
    loss = lossfn(logits, y)
    loss.backward()
    ref = {n: p.grad.clone() for n, p in model.named_parameters()}
    for p in model.parameters():
        p.grad = None
    step = GraphedStep(model, lossfn, x, y, warmup=1, use_graph=False)
    loss2 = step(x, y)
    assert abs(loss2.item() - loss.item()) < 1e-6
    for n, p in model.named_parameters():
        assert (p.grad - ref[n]).abs().max() <= 1e-5 * ref[n].abs().max() + 1e-9, n
