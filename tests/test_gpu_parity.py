"""Network-level parity on the GPU (through the public nn.Module API and the C ABI):
parity mode (fp32) must match the CPU oracle to 1e-3 relative with identical argmax masks
(BASELINE.json north_star); perf mode (bf16) is checked against its documented error budget.
Golden fixtures come from the real reference (tests/golden/make_golden.py)."""
import os

import numpy as np
import pytest
import torch

import oracle
from oracle import nets as onets
import pytorchdeeplearing_b200 as b200
from conftest import GOLDEN

pytestmark = pytest.mark.gpu
torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))


@pytest.fixture(autouse=True)
def _restore_precision():
    prev = b200.get_precision()
    yield
    b200.set_precision(prev)


def _build(kind, cin, ncls, seed):
    if kind == "vnet3d":
        spec = onets.vnet3d_state_spec(cin, ncls)
        model = b200.VNet3d(cin, ncls)
        ofwd = lambda sd, x, masks=None: onets.vnet3d_forward(sd, x, masks)
        draw = lambda n: onets.draw_dropout_masks_vnet3d(n)
    else:
        dims = 3 if kind == "unet3d" else 2
        spec = onets.unet_state_spec(cin, ncls, dims)
        model = (b200.UNet3d if dims == 3 else b200.UNet2d)(cin, ncls)
        ofwd = lambda sd, x, masks=None: onets.unet_forward(sd, x, dims, masks)
        draw = lambda n: onets.draw_dropout_masks_unet(n, dims)
    sd = onets.init_state_dict(spec, seed=seed, randomize_affine=True)
    model.load_state_dict(sd, strict=True)
    return spec, sd, model.cuda(), ofwd, draw


CASES = [
    ("vnet3d", 1, 2, (32, 32, 32), 2, "MutilDiceLoss", b200.MutilDiceLoss),
    ("vnet3d", 1, 1, (16, 32, 48), 1, "BinaryCrossEntropyDiceLoss", b200.BinaryCrossEntropyDiceLoss),
    ("vnet3d", 2, 3, (16, 16, 16), 1, "MutilCrossEntropyDiceLoss", b200.MutilCrossEntropyDiceLoss),
    ("unet3d", 1, 4, (32, 32, 32), 1, "MutilCrossEntropyDiceLoss", b200.MutilCrossEntropyDiceLoss),
    ("unet2d", 1, 1, (128, 128), 2, "BinaryDiceFocalLoss", b200.BinaryDiceFocalLoss),
    ("unet2d", 3, 2, (32, 64), 2, "MutilFocalLoss", b200.MutilFocalLoss),
]


@pytest.mark.parametrize("kind,cin,ncls,spatial,n,lossname,losscls", CASES)
@pytest.mark.parametrize("train", [False, True])
def test_fp32_parity_forward_backward(kind, cin, ncls, spatial, n, lossname, losscls, train):
    b200.set_precision("fp32")
    spec, sd, model, ofwd, draw = _build(kind, cin, ncls, seed=5)
    x, y = oracle.make_inputs(n, cin, spatial, ncls, seed=77)
    alpha = torch.linspace(0.5, 1.5, ncls)
    masks = None
    if train:
        torch.manual_seed(3)
        masks = draw(n)
        model.train()
        model.dropout_masks = masks
    else:
        model.eval()
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    lo, po = ofwd(sdg, x, masks)
    loss_o = oracle.loss_forward(lossname, lo, y, alpha)
    loss_o.backward()
    lossfn = losscls(alpha.cuda()) if lossname.startswith("Mutil") else losscls()
    logits, probs = model(x.cuda())
    loss = lossfn(logits, y.cuda())
    loss.backward()
    torch.cuda.synchronize()
    lg = logits.detach().cpu()
    assert lg.shape == lo.shape
    r = ((lg - lo).norm() / lo.norm()).item()
    assert r < 1e-3, r                                   # north_star tolerance
    assert r < 2e-5, r                                   # what fp32 FFMA actually delivers
    if ncls > 1:
        assert torch.equal(lg.argmax(1), lo.argmax(1))   # identical argmax masks
    else:
        assert torch.equal(lg > 0, lo > 0)
    assert (probs.detach().cpu() - po).abs().max() < 1e-4
    assert abs(loss.item() - loss_o.item()) < 1e-4 * max(1, abs(loss_o.item()))
    # Gradients: a ReLU / max-pool decision that flips between two fp32 evaluations (pre-activation within
    # ~1e-7 of zero) moves one element of an activation-gradient tensor by O(1) of its size, i.e. a relative
    # norm change of ~1/sqrt(#elements) ~ 1e-3 that then propagates to earlier layers; this is a property of
    # the function, not of an implementation (DESIGN.md section 7; tests/diag_layers.py shows the single
    # flipped element behind a 1e-3 deviation).  One flip near the output perturbs every earlier parameter.
    errs = {}
    for name, p in model.named_parameters():
        go = sdg[name].grad
        errs[name] = ((p.grad.cpu() - go).norm() / (go.norm() + 1e-12)).item()
    worst = max(errs, key=errs.get)
    assert float(np.median(list(errs.values()))) < 5e-3, float(np.median(list(errs.values())))
    assert errs[worst] < 2e-2, (worst, errs[worst])
    cos = min(torch.nn.functional.cosine_similarity(p.grad.cpu().flatten(), sdg[n].grad.flatten(), dim=0).item()
              for n, p in model.named_parameters())
    assert cos > 0.9998, cos


def test_golden_fixtures_from_reference_fp32():
    b200.set_precision("fp32")
    for tag, ctor, shape, ncls, seed in (("vnet3d_c2_16", lambda: b200.VNet3d(1, 2), (2, 1, 16, 16, 16), 2, 0),
                                         ("vnet3d_c2_32", lambda: b200.VNet3d(1, 2), (1, 1, 32, 32, 32), 2, 0),
                                         ("unet3d_c4_16", lambda: b200.UNet3d(1, 4), (1, 1, 16, 16, 16), 4, 1),
                                         ("unet2d_c1_32", lambda: b200.UNet2d(1, 1), (2, 1, 32, 32), 1, 2)):
        gold = dict(np.load(os.path.join(GOLDEN, tag + ".npz")))
        model = ctor().eval()
        spec = [(k, tuple(v.shape)) for k, v in model.state_dict().items()]
        model.load_state_dict(onets.init_state_dict(spec, seed=seed, randomize_affine=True))
        model.cuda()
        x, _ = oracle.make_inputs(shape[0], shape[1], shape[2:], ncls)
        with torch.no_grad():
            logits, probs = model(x.cuda())
        ref = torch.from_numpy(gold["logits"])
        lg = logits.cpu()
        assert ((lg - ref).norm() / ref.norm()).item() < 2e-5
        if ncls > 1:
            assert torch.equal(lg.argmax(1), ref.argmax(1))
            assert int(probs.argmax(1).sum()) == int(gold["argmax_sum"])


def test_vnet3d_96_full_size_parity_fp32():
    """BASELINE.json config 2 at full size: VNet3d(1,2), (2,1,96,96,96): logits within 1e-3 relative
    of the CPU oracle and identical argmax masks; loss and gradient norms agree."""
    b200.set_precision("fp32")
    spec, sd, model, ofwd, _ = _build("vnet3d", 1, 2, seed=0)
    model.eval()
    x, y = oracle.make_inputs(2, 1, (96, 96, 96), 2)
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    lo, _ = ofwd(sdg, x)
    loss_o = oracle.loss_forward("MutilDiceLoss", lo, y, torch.ones(2))
    loss_o.backward()
    logits, probs = model(x.cuda())
    loss = b200.MutilDiceLoss(torch.ones(2).cuda())(logits, y.cuda())
    loss.backward()
    lg = logits.detach().cpu()
    r = ((lg - lo).norm() / lo.norm()).item()
    assert r < 1e-3, r
    flips = int((lg.argmax(1) != lo.argmax(1)).sum())
    assert flips == 0, flips
    assert abs(loss.item() - loss_o.item()) < 1e-5
    errs = [((p.grad.cpu() - sdg[n].grad).norm() / (sdg[n].grad.norm() + 1e-12)).item()
            for n, p in model.named_parameters()]
    assert float(np.median(errs)) < 5e-3, float(np.median(errs))
    assert max(errs) < 2e-2, max(errs)


@pytest.mark.parametrize("kind,cin,ncls,spatial,n,lossname,losscls", CASES[:1] + CASES[3:5])
def test_bf16_perf_mode_error_budget(kind, cin, ncls, spatial, n, lossname, losscls):
    """bf16 storage cannot meet 1e-3 (SURVEY.md section 0.8: ~1e-2 normwise, <1 % argmax flips on
    random-init nets); this pins the measured budget so regressions are caught."""
    b200.set_precision("bf16")
    spec, sd, model, ofwd, _ = _build(kind, cin, ncls, seed=5)
    model.eval()
    x, y = oracle.make_inputs(n, cin, spatial, ncls, seed=77)
    alpha = torch.ones(ncls)
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    lo, _ = ofwd(sdg, x)
    loss_o = oracle.loss_forward(lossname, lo, y, alpha)
    loss_o.backward()
    lossfn = losscls(alpha.cuda()) if lossname.startswith("Mutil") else losscls()
    logits, probs = model(x.cuda())
    loss = lossfn(logits, y.cuda())
    loss.backward()
    lg = logits.detach().cpu()
    r = ((lg - lo).norm() / lo.norm()).item()
    assert r < 4e-2, r
    if ncls > 1:
        flips = (lg.argmax(1) != lo.argmax(1)).float().mean().item()
    else:
        flips = ((lg > 0) != (lo > 0)).float().mean().item()
    assert flips < 2e-2, flips
    assert abs(loss.item() - loss_o.item()) < 2e-2
    errs = [((p.grad.cpu() - sdg[nm].grad).norm() / (sdg[nm].grad.norm() + 1e-12)).item()
            for nm, p in model.named_parameters()]
    # measured: gradient noise grows from ~0.3 % at the head to ~20-30 % (relative norm) at the deepest
    # layers of a random-init net -- bf16 rounding of activation gradients amplified by the GroupNorm
    # backward projection (same figures from the CPU emulation of the bf16 data flow)
    assert float(np.median(errs)) < 0.35, float(np.median(errs))


def test_dropout_train_mode_runs_and_is_seeded():
    b200.set_precision("bf16")
    _, _, model, _, _ = _build("vnet3d", 1, 2, seed=0)
    model.train()
    x, _ = oracle.make_inputs(1, 1, (16, 16, 16), 2)
    torch.manual_seed(11)
    a, _ = model(x.cuda())
    torch.manual_seed(11)
    b, _ = model(x.cuda())
    torch.manual_seed(12)
    c, _ = model(x.cuda())
    assert torch.equal(a, b) and not torch.equal(a, c)      # same seed -> same masks -> bit-identical forward
