"""The binary Lovasz hinge (BinaryLovaszLoss, lovasz_hinge) without a GPU: the CPU oracle against the fixtures the real
reference produced (tests/golden/lovasz_hinge.npz), the constructor the reference meant, the refusals (logit channels,
float labels, label values, data parallelism), install()/uninstall(), loss_spec, and the module, the functional form
and GraphedStep on the emulated backend."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import lovasz_hinge as oh
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import losses as bl, runtime
from conftest import GOLDEN
from emu_backend import EmuBackend

CASES = [
    ("b3", "z3", "t3", {}),
    ("b3_per_image", "z3", "t3", {"per_image": True}),
    ("ignore255", "z3", "t3x", {"ignore_index": 255}),
    ("one_ignored", "z3", "t3one", {"ignore_index": 255}),
    ("one_ignored_per_image", "z3", "t3one", {"per_image": True, "ignore_index": 255}),
    ("no_fg", "z3", "t3zero", {}),
    ("satisfied", "zsat", "t3", {}),
    ("ties", "zq", "t3", {}),
    ("b2", "z2", "t2", {}),
    ("cls", "zc", "tc", {}),
]


def _gold():
    return dict(np.load(os.path.join(GOLDEN, "lovasz_hinge.npz")))


def _oracle_kw(kw):
    return {"per_image": kw.get("per_image", False), "ignore": kw.get("ignore_index")}


@pytest.mark.parametrize("key,zk,tk,kw", CASES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_oracle_matches_reference_fixture(key, zk, tk, kw, dtype):
    """fp32: the reference's own arithmetic; fp64: the restatement the GPU kernels are held to.  The value agrees to
    round-off; the fp32 gradient carries the cancellation of jaccard[1:] - jaccard[:-1] (model/lovasz.py:31).  On the
    tie-heavy input the reference's unstable torch.sort orders ties differently, which moves the gradient only."""
    gold = _gold()
    z = torch.from_numpy(gold[zk]).requires_grad_(True)
    v = oh.lovasz_hinge(z, torch.from_numpy(gold[tk]), dtype=dtype, **_oracle_kw(kw))
    v.backward()
    want = float(gold[key + "_value"])
    assert abs(v.item() - want) < 1e-6 * max(1.0, abs(want))
    if key == "ties":
        return
    ref = torch.from_numpy(gold[key + "_grad"])
    assert (z.grad.float() - ref).abs().max() <= 1e-2 * ref.abs().max()


def test_fixture_cases_cover_the_documented_edges():
    gold = _gold()
    assert float(gold["satisfied_value"]) == 0.0 and not gold["satisfied_grad"].any()
    z = gold["z3"][:, 0]
    e = np.where(gold["t3zero"] == 1, 1 - z, 1 + z)
    assert float(gold["no_fg_value"]) == pytest.approx(max(float(e.max()), 0.0), rel=1e-6)     # relu(max e)
    assert not gold["one_ignored_grad"][1].any()
    assert float(gold["one_ignored_per_image_value"]) == pytest.approx(float(gold["one_ignored_value"]) / 2, rel=1e-6)
    zq = gold["zq"].reshape(-1)
    assert len(np.unique(zq)) < zq.size // 4                                   # the tie case has ties


def test_constructor_and_attributes():
    lv = b200.BinaryLovaszLoss()
    assert isinstance(lv, torch.nn.Module) and (lv.per_image, lv.ignore_index) == (False, None)
    lv = b200.BinaryLovaszLoss(per_image=True, ignore_index=255)
    assert (lv.per_image, lv.ignore_index) == (True, 255)
    assert hasattr(lv, "_backward_hooks") and list(lv.parameters()) == []
    assert b200.lovasz_hinge is bl.lovasz_hinge


def test_loss_spec():
    lv = b200.BinaryLovaszLoss(per_image=True, ignore_index=255)
    assert bl.loss_spec(lv) == (bl.LOVASZ_HINGE, None, 2.0, 0.25)
    assert bl.LOVASZ_HINGE not in (bl.DICE, bl.CE, bl.FOCAL, bl.JACCARD, bl.ELDICE, bl.TVERSKY, bl.SS, bl.LOVASZ)


def test_refusals_before_any_backend_call():
    z = torch.rand(2, 1, 4, 6, 6)
    t = torch.randint(0, 2, (2, 4, 6, 6))
    with pytest.raises(ValueError, match="one channel"):
        b200.BinaryLovaszLoss()(torch.rand(2, 2, 4, 6, 6), t)
    with pytest.raises(ValueError, match="logits"):
        b200.BinaryLovaszLoss()(torch.rand(2, 1, 6), t)
    with pytest.raises(TypeError, match="integer labels"):
        b200.BinaryLovaszLoss()(z, t.float())
    with pytest.raises(TypeError, match="integer labels"):
        b200.lovasz_hinge(z, t.double())
    # the multi-class loss still refuses one class
    with pytest.raises(ValueError, match="Sigmoid output possible only with 1 class"):
        b200.LovaszLoss()(z, t)


def test_refuses_data_parallel():
    import torch.distributed as dist
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(29800 + os.getpid() % 150))
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        b200.enable_data_parallel()
        z = torch.rand(1, 1, 4, 8, 8, requires_grad=True)
        t = torch.randint(0, 2, (1, 4, 8, 8))
        with pytest.raises(RuntimeError, match="data parallelism"):
            b200.BinaryLovaszLoss()(z, t)
        with pytest.raises(RuntimeError, match="data parallelism"):
            b200.lovasz_hinge(z, t)
    finally:
        b200.disable_data_parallel()
        dist.destroy_process_group()


def test_install_rebinds_the_name_and_uninstall_restores(monkeypatch):
    m = types.ModuleType("model.losses")
    orig = type("BinaryLovaszLoss", (), {})
    m.BinaryLovaszLoss = orig
    monkeypatch.setitem(sys.modules, "model.losses", m)
    try:
        assert b200.install() == 1
        assert m.BinaryLovaszLoss is b200.BinaryLovaszLoss
    finally:
        b200.uninstall()
    assert m.BinaryLovaszLoss is orig


# ------------------------------------------------------------------------------------------------ emulated backend
class _HingeEmu(EmuBackend):
    """EmuBackend plus the hinge entry points, in fp64 torch over the oracle; coef holds d loss / d logits"""

    def lovasz_hinge_fwd(self, logits, labels, per_image, ignore, loss, coef, bad=None):
        z = logits.detach().double().requires_grad_(True)
        with torch.enable_grad():
            v = oh.lovasz_hinge(z, labels, per_image=per_image, ignore=ignore, dtype=torch.float64)
            g, = torch.autograd.grad(v, z) if v.requires_grad else (torch.zeros_like(z),)
        coef.copy_(g.float())
        loss.copy_(v.detach().float())
        if bad is not None:
            valid = torch.ones_like(labels, dtype=torch.bool) if ignore is None else labels != ignore
            bad.fill_(int(((labels != 0) & (labels != 1) & valid).sum()))

    def lovasz_hinge_bwd(self, coef, gscale, dlogits):
        dlogits.copy_(coef * gscale)


@pytest.fixture()
def emu():
    runtime._set_backend_for_testing(_HingeEmu())
    prev = runtime.get_precision()
    runtime.set_precision("fp32")
    yield
    runtime._set_backend_for_testing(None)
    runtime.set_precision(prev)


@pytest.mark.parametrize("layout", ["ncdhw", "channels_last", "nchw", "classifier"])
@pytest.mark.parametrize("kw", [{}, {"per_image": True, "ignore_index": 255}])
def test_module_and_functional_on_the_emulated_backend(emu, layout, kw):
    """the layouts reach the backend as one-channel channels-last volumes, and the gradient comes back in the caller's
    layout; the module's defaults are the reference class's, the functional's are _lovasz_hinge's (per_image=True)"""
    g = torch.Generator().manual_seed(7)
    shape = {"ncdhw": (2, 1, 4, 6, 8), "channels_last": (2, 1, 4, 6, 8), "nchw": (3, 1, 6, 8), "classifier": (5, 1)}
    z0 = torch.randn(shape[layout], generator=g)
    t = (torch.rand((shape[layout][0],) + shape[layout][2:], generator=g) > 0.6).long()
    if kw:
        t[torch.rand(t.shape, generator=g) < 0.1] = 255
    z = z0.clone()
    if layout == "channels_last":
        z = z.permute(0, 2, 3, 4, 1).contiguous().permute(0, 4, 1, 2, 3)
    z.requires_grad_(True)
    lv = b200.BinaryLovaszLoss(**kw)
    v = lv(z, t)
    v.backward()
    zo = z0.clone().requires_grad_(True)
    vo = oh.lovasz_hinge(zo, t, dtype=torch.float64, **_oracle_kw(kw))
    vo.backward()
    assert abs(v.item() - vo.item()) < 1e-6 * max(1.0, abs(vo.item()))
    assert z.grad.shape == z0.shape and (z.grad - zo.grad).abs().max() <= 1e-6 * zo.grad.abs().max()
    lv.last_metric()                                            # the accuracy sums came from the same pass
    z.grad = None
    vf = b200.lovasz_hinge(z, t, ignore_index=kw.get("ignore_index"))
    vfo = oh.lovasz_hinge(z0, t, per_image=True, ignore=kw.get("ignore_index"), dtype=torch.float64)
    assert abs(vf.item() - vfo.item()) < 1e-6 * max(1.0, abs(vfo.item()))


def test_label_values_are_checked(emu, monkeypatch):
    z = torch.randn(2, 1, 4, 6, 6, requires_grad=True)
    t = torch.randint(0, 2, (2, 4, 6, 6))
    t[0, 0, 0, 0] = 2
    with pytest.raises(ValueError, match="1 label value"):
        b200.BinaryLovaszLoss()(z, t)
    t[0, 0, 0, 0] = 255
    with pytest.raises(ValueError, match="1 label value"):
        b200.BinaryLovaszLoss()(z, t)
    b200.BinaryLovaszLoss(ignore_index=255)(z, t)               # the ignored value is not a bad label
    b200.BinaryLovaszLoss(ignore_index=255.0)(z, t)             # an integral float matches the label
    with pytest.raises(ValueError, match="1 label value"):
        b200.BinaryLovaszLoss(ignore_index=254.5)(z, t)          # a non-integer float matches no label
    monkeypatch.setenv("B200SEG_CHECK_LABELS", "0")
    b200.BinaryLovaszLoss()(z, t)


def test_graphed_step_on_the_emulated_backend(emu):
    """the step program (GraphedStep, eager form) and the autograd path give the same loss and gradients; the step
    refuses what the module refuses, at construction"""
    import oracle
    from oracle import nets as onets
    from pytorchdeeplearing_b200.graphed import GraphedStep
    spec = onets.unet_state_spec(1, 1, 2)
    sd = onets.init_state_dict(spec, seed=4, randomize_affine=True)
    model = b200.UNet2d(1, 1)
    model.load_state_dict(sd, strict=True)
    model.eval()
    x, y = oracle.make_inputs(2, 1, (16, 16), 1, seed=9)
    for kw in ({}, {"per_image": True, "ignore_index": 255}):
        yk = y.clone()
        if kw:
            yk[0, :3] = 255
        lossfn = b200.BinaryLovaszLoss(**kw)
        logits, _ = model(x)
        loss = lossfn(logits, yk)
        loss.backward()
        ref = {n: p.grad.clone() for n, p in model.named_parameters()}
        for p in model.parameters():
            p.grad = None
        step = GraphedStep(model, lossfn, x, yk, warmup=1, use_graph=False)
        loss2 = step(x, yk)
        step.check_labels()
        assert abs(loss2.item() - loss.item()) < 1e-6
        for n, p in model.named_parameters():
            assert (p.grad - ref[n]).abs().max() <= 1e-5 * ref[n].abs().max() + 1e-9, n
        for p in model.parameters():
            p.grad = None
    with pytest.raises(TypeError, match="integer labels"):
        GraphedStep(model, b200.BinaryLovaszLoss(), x, y.float(), warmup=1, use_graph=False)
    bad = y.clone()
    bad[0, 0, 0] = 3
    with pytest.raises(ValueError, match="1 label value"):
        GraphedStep(model, b200.BinaryLovaszLoss(), x, bad, warmup=1, use_graph=False)
    model2 = b200.UNet2d(1, 2)
    with pytest.raises(ValueError, match="one channel"):
        GraphedStep(model2, b200.BinaryLovaszLoss(), x, y, warmup=1, use_graph=False)
