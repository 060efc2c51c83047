"""The further reference losses on the GPU, through the C ABI: BinaryJaccard / BinaryELDice / BinaryTversky / BinarySS /
MutilELDice (new finalize forms over the fused partial sums) and LovaszLoss (stable segmented radix sort + Lovasz
gradient scan), against the fixtures the real reference produced (tests/golden/losses_ext.npz) and the fp64 oracle
(oracle/losses_ext.py); the radix sort alone against torch.sort(stable=True); run-to-run bit identity; GraphedStep
replay; the data-parallel refusal of LovaszLoss."""
import os

import numpy as np
import pytest
import torch

import oracle
from oracle import losses_ext as ox
from oracle import nets as onets
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import runtime
from pytorchdeeplearing_b200.graphed import GraphedStep
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

SUM_CASES = [
    ("BinaryJaccardLoss", "BinaryJaccardLoss", "zb", "tb"),
    ("BinaryJaccardLoss_soft", "BinaryJaccardLoss", "zb", "ts"),
    ("BinaryELDiceLoss", "BinaryELDiceLoss", "zb", "tb"),
    ("BinaryELDiceLoss_soft", "BinaryELDiceLoss", "zb", "ts"),
    ("BinaryTverskyLoss", "BinaryTverskyLoss", "zb", "tb"),
    ("BinaryTverskyLoss_soft", "BinaryTverskyLoss", "zb", "ts"),
    ("BinarySSLoss", "BinarySSLoss", "zb", "tb"),
    ("BinarySSLoss_soft", "BinarySSLoss", "zb", "ts"),
    ("MutilELDiceLoss", "MutilELDiceLoss", "zm", "tm"),
    ("MutilELDiceLoss_absent", "MutilELDiceLoss", "zm", "tm_absent"),
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


def _dev_logits(z, channels_last):
    z = z.cuda()
    if channels_last:       # what the drop-in networks hand over: NDHWC memory behind an NCDHW shape
        z = z.permute(0, 2, 3, 4, 1).contiguous().permute(0, 4, 1, 2, 3)
    return z.requires_grad_(True)


def _run(fn, z, t):
    v = fn(z, t)
    assert v.dim() == 0 and v.dtype == torch.float32
    v.backward()
    return v.item(), z.grad.cpu()


def _oracle_lovasz(z, t, **kw):
    """fp64 oracle with the stable tie order, evaluated by torch on the GPU (test infrastructure)"""
    zo = z.detach().cuda().requires_grad_(True)
    v = ox.lovasz_softmax(zo, t.cuda(), dtype=torch.float64, **kw)
    v.backward()
    return v.item(), zo.grad.cpu()


@pytest.mark.parametrize("key,name,zk,tk", SUM_CASES)
@pytest.mark.parametrize("channels_last", [False, True])
def test_sum_based_class_matches_reference_fixture(key, name, zk, tk, channels_last):
    gold = _gold()
    z = _dev_logits(torch.from_numpy(gold[zk]), channels_last)
    fn = getattr(b200, name)(torch.from_numpy(gold["alpha"]).cuda()) if name.startswith("Mutil") else getattr(b200, name)()
    v, g = _run(fn, z, torch.from_numpy(gold[tk]).cuda())
    assert abs(v - float(gold[key + "_value"])) < 3e-6
    ref = torch.from_numpy(gold[key + "_grad"])
    assert (g - ref).abs().max() < 1e-8 + 1e-4 * ref.abs().max()
    fn.last_metric()                                            # the accuracy sums came from the same pass


@pytest.mark.parametrize("key,zk,tk,kw", LOVASZ_CASES)
@pytest.mark.parametrize("channels_last", [False, True])
def test_lovasz_matches_reference_fixture_and_fp64_oracle(key, zk, tk, kw, channels_last):
    gold = _gold()
    z0, t = torch.from_numpy(gold[zk]), torch.from_numpy(gold[tk])
    z = _dev_logits(z0, channels_last)
    v, g = _run(b200.LovaszLoss(**kw), z, t.cuda())
    want = float(gold[key + "_value"])
    assert abs(v - want) < 1e-6 * max(1.0, abs(want))
    if key != "LovaszLoss_ties":            # the reference's unstable sort orders ties differently (value unaffected)
        ref = torch.from_numpy(gold[key + "_grad"])
        assert (g - ref).abs().max() < 1e-2 * ref.abs().max()
    vo, go = _oracle_lovasz(z0, t, **kw)
    assert abs(v - vo) < 1e-6 * max(1.0, abs(vo))
    assert (g.double() - go).abs().max() < 1e-5 * go.abs().max()


@pytest.mark.parametrize("shape,c,kw", [((2, 96, 96, 96), 2, {}), ((1, 128, 112, 112), 5, {}),
                                        ((2, 48, 48, 48), 3, {"per_image": True, "ignore": 1})])
def test_lovasz_large_against_fp64_oracle(shape, c, kw):
    g = torch.Generator().manual_seed(11 + c)
    z0 = torch.randn((shape[0], c) + shape[1:], generator=g)
    t = torch.randint(0, c, shape, generator=g)
    z = _dev_logits(z0, True)
    v, gr = _run(b200.LovaszLoss(**kw), z, t.cuda())
    vo, go = _oracle_lovasz(z0, t, **kw)
    assert abs(v - vo) < 1e-6 * abs(vo)
    assert (gr.double() - go).abs().max() < 1e-5 * go.abs().max()


def test_lovasz_empty_classes_and_all_ignored():
    z = torch.rand(2, 3, 4, 8, 8, device="cuda", requires_grad=True)
    t = torch.zeros(2, 4, 8, 8, dtype=torch.long, device="cuda")
    t[1] = 2                                                     # class 1 absent everywhere, class 2 in sample 1
    for kw in ({}, {"per_image": True}):
        v, g = _run(b200.LovaszLoss(**kw), z, t)
        vo, go = _oracle_lovasz(z.detach().cpu(), t.cpu(), **kw)
        assert abs(v - vo) < 1e-6 * max(1.0, abs(vo)) and (g.double() - go).abs().max() < 1e-5 * go.abs().max()
        z.grad = None
    v, g = _run(b200.LovaszLoss(ignore=0), z, torch.zeros_like(t))   # every voxel ignored: 0, no gradient
    assert v == 0.0 and torch.count_nonzero(g) == 0


def _torch_sorted(keys, vals):
    k64 = keys.long() & 0xFFFFFFFF
    s = torch.sort(k64, dim=1, stable=True)
    return s.values, torch.gather(vals, 1, s.indices)


@pytest.mark.parametrize("nseg,ln,kind", [(1, 1, "rand"), (3, 4096, "rand"), (2, 4097, "ties"), (5, 10000, "ties"),
                                          (1, 300001, "rand"), (4, 65537, "bytes"), (2, 0, "rand")])
def test_radix_sort_is_torch_stable_sort(nseg, ln, kind):
    be = runtime.get_backend(torch.zeros(1, device="cuda"))
    g = torch.Generator().manual_seed(ln + nseg)
    if kind == "rand":
        k = torch.randint(-2 ** 31, 2 ** 31 - 1, (nseg, ln), generator=g, dtype=torch.int64)
    elif kind == "ties":
        k = torch.randint(0, 4, (nseg, ln), generator=g) * 0x01010101 - 2 ** 31
    else:                                                        # one non-constant byte per pass
        k = torch.randint(0, 2, (nseg, ln), generator=g) << (8 * torch.randint(0, 4, (nseg, ln), generator=g))
    keys = k.to(torch.int32).cuda()
    vals = torch.arange(nseg * ln, dtype=torch.int32).reshape(nseg, ln).cuda()
    ko, vo = be.radix_sort_pairs(keys, vals)
    wk, wv = _torch_sorted(keys.cpu(), vals.cpu())
    assert torch.equal(ko.cpu().long() & 0xFFFFFFFF, wk)
    assert torch.equal(vo.cpu(), wv)


@pytest.mark.parametrize("name", ["BinaryTverskyLoss", "BinarySSLoss", "MutilELDiceLoss", "LovaszLoss"])
def test_two_runs_are_bit_identical(name):
    g = torch.Generator().manual_seed(5)
    c = 1 if name.startswith("Binary") else 3
    z0 = torch.randn((2, c, 32, 48, 40), generator=g)
    t = (torch.rand((2, 32, 48, 40), generator=g) > 0.6).long() if c == 1 else torch.randint(0, c, (2, 32, 48, 40))
    fn = getattr(b200, name)(torch.ones(c).cuda()) if name.startswith("Mutil") else getattr(b200, name)()
    outs = []
    for _ in range(2):
        z = _dev_logits(z0, True)
        outs.append(_run(fn, z, t.cuda()))
    assert outs[0][0] == outs[1][0] and torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("lossname", ["BinaryTverskyLoss", "LovaszLoss"])
def test_graphed_step_replay_equals_eager(lossname):
    """VNet3d step captured with the new loss: replayed loss and gradients equal the autograd path"""
    prev = b200.get_precision()
    b200.set_precision("bf16")
    try:
        ncls = 1 if lossname == "BinaryTverskyLoss" else 2
        spec = onets.vnet3d_state_spec(1, ncls)
        model = b200.VNet3d(1, ncls)
        model.load_state_dict(onets.init_state_dict(spec, seed=3, randomize_affine=True), strict=True)
        model = model.cuda().eval()
        x, y = oracle.make_inputs(2, 1, (32, 32, 32), ncls, seed=5)
        xc, yc = x.cuda(), y.cuda()
        lossfn = getattr(b200, lossname)()
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
        assert abs(loss_g.item() - loss_e.item()) < 1e-6
        assert abs(step.dice.item() - dice_e) < 1e-6
        for n, p in model.named_parameters():
            assert (p.grad - ref[n]).norm() <= 2e-5 * ref[n].norm() + 1e-12, n
    finally:
        b200.set_precision(prev)


def test_lovasz_refuses_data_parallel():
    import torch.distributed as dist
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(29500 + os.getpid() % 300))
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        b200.enable_data_parallel()
        z = torch.rand(1, 2, 4, 8, 8, device="cuda", requires_grad=True)
        t = torch.randint(0, 2, (1, 4, 8, 8), device="cuda")
        with pytest.raises(RuntimeError, match="data parallelism"):
            b200.LovaszLoss()(z, t)
    finally:
        b200.disable_data_parallel()
        dist.destroy_process_group()
