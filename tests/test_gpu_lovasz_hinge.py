"""The binary Lovasz hinge (BinaryLovaszLoss, lovasz_hinge) on the GPU, through the C ABI: the stable segmented radix
sort of the Lovasz-Softmax loss with hinge keys, exact prefix counts and an fp64 Lovasz gradient.  Against the fixtures
the real reference produced (tests/golden/lovasz_hinge.npz) and the fp64 oracle (oracle/lovasz_hinge.py) on both
logit layouts; large volumes; run-to-run bit identity; the label count; the all-ignored sample; GraphedStep replay; the
data-parallel refusal."""
import os

import numpy as np
import pytest
import torch

import oracle
from oracle import lovasz_hinge as oh
from oracle import nets as onets
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import runtime
from pytorchdeeplearing_b200.graphed import GraphedStep
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

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


def _dev_logits(z, channels_last):
    z = z.cuda()
    if channels_last and z.dim() > 2:       # what the drop-in networks hand over: channels-last memory, NC... shape
        perm = (0, 2, 3, 4, 1) if z.dim() == 5 else (0, 2, 3, 1)
        inv = (0, 4, 1, 2, 3) if z.dim() == 5 else (0, 3, 1, 2)
        z = z.permute(*perm).contiguous().permute(*inv)
    return z.requires_grad_(True)


def _run(fn, z, t):
    v = fn(z, t)
    assert v.dim() == 0 and v.dtype == torch.float32
    v.backward()
    return v.item(), z.grad.cpu()


def _oracle(z, t, per_image=False, ignore_index=None):
    """fp64 oracle with the stable tie order, evaluated by torch on the GPU (test infrastructure)"""
    zo = z.detach().cuda().requires_grad_(True)
    v = oh.lovasz_hinge(zo, t.cuda(), per_image=per_image, ignore=ignore_index, dtype=torch.float64)
    v.backward()
    return v.item(), zo.grad.cpu()


@pytest.mark.parametrize("key,zk,tk,kw", CASES)
@pytest.mark.parametrize("channels_last", [False, True])
def test_matches_reference_fixture_and_fp64_oracle(key, zk, tk, kw, channels_last):
    gold = _gold()
    z0, t = torch.from_numpy(gold[zk]), torch.from_numpy(gold[tk])
    z = _dev_logits(z0, channels_last)
    lv = b200.BinaryLovaszLoss(**kw)
    v, g = _run(lv, z, t.cuda())
    lv.last_metric()                                            # the accuracy sums came from the same pass
    want = float(gold[key + "_value"])
    assert abs(v - want) < 1e-6 * max(1.0, abs(want))
    if key != "ties":                       # the reference's unstable sort orders ties differently (value unaffected)
        ref = torch.from_numpy(gold[key + "_grad"])
        assert (g - ref).abs().max() <= 1e-2 * ref.abs().max()
    vo, go = _oracle(z0, t, **kw)
    assert abs(v - vo) < 1e-6 * max(1.0, abs(vo))
    assert (g.double() - go).abs().max() <= 1e-5 * go.abs().max()
    if key == "satisfied":
        assert v == 0.0 and torch.count_nonzero(g) == 0


@pytest.mark.parametrize("shape,kw", [((2, 1, 96, 96, 96), {}), ((2, 1, 96, 96, 96), {"per_image": True}),
                                      ((2, 1, 96, 96, 96), {"per_image": True, "ignore_index": 255}),
                                      ((1, 1, 128, 112, 112), {}), ((1, 1, 128, 112, 112), {"ignore_index": 255})])
def test_large_against_fp64_oracle(shape, kw):
    g = torch.Generator().manual_seed(sum(shape) + len(kw))
    z0 = 2.0 * torch.randn(shape, generator=g)
    t = (torch.rand((shape[0],) + shape[2:], generator=g) > 0.7).long()
    if "ignore_index" in kw:
        t[torch.rand(t.shape, generator=g) < 0.05] = 255
    z = _dev_logits(z0, True)
    v, gr = _run(b200.BinaryLovaszLoss(**kw), z, t.cuda())
    vo, go = _oracle(z0, t, **kw)
    assert abs(v - vo) < 1e-6 * abs(vo)
    assert (gr.double() - go).abs().max() < 1e-5 * go.abs().max()


def test_functional_defaults_and_label_shapes():
    """lovasz_hinge takes _lovasz_hinge's defaults (per_image=True); labels of any shape with N*vox elements"""
    g = torch.Generator().manual_seed(3)
    z0 = torch.randn((3, 1, 8, 10, 12), generator=g)
    t = (torch.rand((3, 8, 10, 12), generator=g) > 0.5).long()
    vo, go = _oracle(z0, t, per_image=True)
    for tt in (t, t.unsqueeze(1), t.to(torch.uint8), t.bool()):
        z = _dev_logits(z0, True)
        v, gr = _run(b200.lovasz_hinge, z, tt.cuda())
        assert abs(v - vo) < 1e-6 * abs(vo) and (gr.double() - go).abs().max() < 1e-5 * go.abs().max()


def test_two_runs_are_bit_identical():
    g = torch.Generator().manual_seed(5)
    z0 = torch.round(8 * torch.randn((2, 1, 32, 48, 40), generator=g)) / 16      # ties across several tiles
    t = (torch.rand((2, 32, 48, 40), generator=g) > 0.6).long()
    for kw in ({}, {"per_image": True}):
        outs = []
        for _ in range(2):
            z = _dev_logits(z0, True)
            outs.append(_run(b200.BinaryLovaszLoss(**kw), z, t.cuda()))
        assert outs[0][0] == outs[1][0] and torch.equal(outs[0][1], outs[1][1])


def test_label_count_and_all_ignored_sample():
    """the key pass counts labels other than 0, 1 and ignore_index (ValueError); a sample whose every voxel is ignored
    adds 0 and gets a zero gradient even where a logit is infinite (the reference gives NaN there)"""
    z = torch.randn(2, 1, 4, 8, 8, device="cuda", requires_grad=True)
    t = torch.randint(0, 2, (2, 4, 8, 8), device="cuda")
    t[1, 0, 0, :3] = 7
    with pytest.raises(ValueError, match="3 label value"):
        b200.BinaryLovaszLoss()(z, t)
    t[1] = 255
    with torch.no_grad():
        z[1, 0, 0, 0, 0] = float("inf")
    v, g = _run(b200.BinaryLovaszLoss(per_image=True, ignore_index=255), z, t)
    vo, go = _oracle(z.detach()[:1].cpu(), t[:1].cpu())
    assert abs(v - vo / 2) < 1e-6 * max(1.0, abs(vo)) and torch.count_nonzero(g[1]) == 0
    v, g = _run(b200.BinaryLovaszLoss(ignore_index=0), torch.randn(2, 1, 4, 8, 8, device="cuda", requires_grad=True),
                torch.zeros_like(t))
    assert v == 0.0 and torch.count_nonzero(g) == 0


def test_graphed_step_replay_equals_eager():
    """VNet3d(1, 1) step captured with BinaryLovaszLoss: replayed loss and gradients equal the autograd path"""
    prev = b200.get_precision()
    b200.set_precision("bf16")
    try:
        spec = onets.vnet3d_state_spec(1, 1)
        model = b200.VNet3d(1, 1)
        model.load_state_dict(onets.init_state_dict(spec, seed=3, randomize_affine=True), strict=True)
        model = model.cuda().eval()
        x, y = oracle.make_inputs(2, 1, (32, 32, 32), 1, seed=5)
        xc, yc = x.cuda(), y.cuda()
        for kw in ({}, {"per_image": True}):
            lossfn = b200.BinaryLovaszLoss(**kw)
            logits, probs = model(xc)
            loss_e = lossfn(logits, yc)
            loss_e.backward()
            ref = {n: p.grad.clone() for n, p in model.named_parameters()}
            dice_e = lossfn.last_dice().item()
            for p in model.parameters():
                p.grad = None
            step = GraphedStep(model, lossfn, xc, yc, warmup=1)
            assert step.graph is not None
            loss_g = step(xc, yc)
            torch.cuda.synchronize()
            step.check_labels()
            assert abs(loss_g.item() - loss_e.item()) < 1e-6
            assert abs(step.dice.item() - dice_e) < 1e-6
            for n, p in model.named_parameters():
                assert (p.grad - ref[n]).norm() <= 2e-5 * ref[n].norm() + 1e-12, n
            for p in model.parameters():
                p.grad = None
    finally:
        b200.set_precision(prev)


def test_refuses_data_parallel():
    import torch.distributed as dist
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(29500 + os.getpid() % 300))
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        b200.enable_data_parallel()
        z = torch.rand(1, 1, 4, 8, 8, device="cuda", requires_grad=True)
        t = torch.randint(0, 2, (1, 4, 8, 8), device="cuda")
        with pytest.raises(RuntimeError, match="data parallelism"):
            b200.BinaryLovaszLoss()(z, t)
    finally:
        b200.disable_data_parallel()
        dist.destroy_process_group()


def test_abi_rejects_empty_batch():
    be = runtime.get_backend(torch.zeros(1, device="cuda"))
    assert int(be.lib.b200seg_lovasz_hinge_workspace(0, 10, 0)) == 0
    assert int(be.lib.b200seg_lovasz_hinge_workspace(2, 10, 1)) > 0
