"""ResNet2d / ResNet3d classifiers on CPU: the oracle (oracle/resnet.py) pinned to outputs of the reference itself
(tests/golden/resnet.npz), and the drop-in's layer program, losses on (N, C) logits, GraphedStep, install and data
parallelism on the emulated backend, with the classifier head emulated below."""
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

import oracle
from oracle import resnet as ores
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import runtime
from emu_backend import EmuBackend

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = dict(np.load(os.path.join(HERE, "golden", "resnet.npz")))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_resnet import CASES, TRAIN_SEED, case_inputs  # noqa: E402

torch.set_num_threads(max(1, min(8, os.cpu_count() or 1)))

LOSSES = ("MutilCrossEntropyLoss", "MutilFocalLoss", "BinaryCrossEntropyLoss", "BinaryFocalLoss")


class ClsEmuBackend(EmuBackend):
    """EmuBackend plus the two classifier-head entry points (b200seg_cls_head_fwd / _bwd) in torch ops"""

    def cls_head_fwd(self, x, w1, b1, w2, b2, pooled, hidden, logits):
        p = x.float().reshape(x.shape[0], -1, x.shape[-1]).mean(1)
        h = F.relu(F.linear(p, w1, b1))
        pooled.copy_(p)
        hidden.copy_(h)
        logits.copy_(F.linear(h, w2, b2))

    def cls_head_bwd(self, dlogits, pooled, hidden, w1, w2, work, dx, dw1, db1, dw2, db2):
        n, c = pooled.shape
        vox = dx.numel() // (n * c)
        dh = (dlogits @ w2) * (hidden > 0)
        dp = (dh @ w1) / vox
        dw1.copy_(dh.t() @ pooled)
        db1.copy_(dh.sum(0))
        dw2.copy_(dlogits.t() @ hidden)
        db2.copy_(dlogits.sum(0))
        dx.copy_(dp.view(n, 1, 1, 1, c).expand(dx.shape).to(dx.dtype))


@pytest.fixture(autouse=True)
def _emu():
    runtime._set_backend_for_testing(ClsEmuBackend())
    prev = runtime.get_precision()
    runtime.set_precision("fp32")
    yield
    b200.uninstall()
    runtime._set_backend_for_testing(None)
    runtime.set_precision(prev)


def _net(dims, k):
    return (b200.ResNet3d if dims == 3 else b200.ResNet2d)(1, k)


def _lossfn(name, k):
    cls = getattr(b200, name)
    return cls(torch.ones(k)) if name.startswith("Mutil") else cls()


def _rel(a, b):
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


# ------------------------------------------------------------------------------ oracle vs the reference's outputs
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_matches_reference_fixtures(case):
    tag, dims, spatial, n, k, lossname, seed = case
    spec = ores.resnet_state_spec(1, k, dims)
    assert len(spec) == 70 and len(GOLD[tag + "_grads"]) == 70
    sd = {s: v.requires_grad_(True) for s, v in oracle.init_state_dict(spec, seed=seed, randomize_affine=True).items()}
    x, y = case_inputs(dims, spatial, n, k, seed)
    logits = ores.resnet_forward(sd, x, dims)
    ref = torch.from_numpy(GOLD[tag + "_logits"])
    assert _rel(logits.detach(), ref) < 1e-5
    loss = oracle.loss_forward(lossname, logits, y, torch.ones(k))
    assert abs(loss.item() - float(GOLD[tag + "_loss"])) < 1e-5 * max(1.0, abs(float(GOLD[tag + "_loss"])))
    loss.backward()
    table = GOLD[tag + "_grads"]
    for (name, _), (gnorm, gsum) in zip(spec, table):
        g = sd[name].grad.double()
        assert abs(g.norm().item() - gnorm) <= 1e-4 * gnorm + 1e-9, name
        assert abs(g.sum().item() - gsum) <= 1e-4 * gnorm + 1e-9, name
    if tag + "_train_logits" in GOLD:
        torch.manual_seed(TRAIN_SEED)
        masks = ores.draw_dropout_masks_resnet(n, dims)
        with torch.no_grad():
            lt = ores.resnet_forward(sd, x, dims, masks)
        assert _rel(lt, torch.from_numpy(GOLD[tag + "_train_logits"])) < 1e-5


# ------------------------------------------------------------------------------ module contract
@pytest.mark.parametrize("dims", [2, 3])
def test_state_dict_layout_roundtrip_and_initialize_weights(dims):
    m = _net(dims, 3)
    spec = ores.resnet_state_spec(1, 3, dims)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == spec
    assert sum(p.numel() for p in m.parameters()) == (2554115 if dims == 2 else 7410211)
    sd = oracle.init_state_dict(spec, seed=3, randomize_affine=True)
    m.load_state_dict(sd, strict=True)
    assert all(torch.equal(m.state_dict()[k], v) for k, v in sd.items())
    m.apply(b200.initialize_weights)
    s = m.state_dict()
    for name, shape in spec:
        v = s[name]
        if name.startswith("fc_layers") and name.endswith(".weight"):        # kaiming_uniform_, a = 0
            bound = (6.0 / shape[1]) ** 0.5
            assert v.abs().max() <= bound and v.abs().max() > 0.9 * bound, name
        elif len(shape) > 1:                                                # kaiming_normal_, relu gain
            fan_in = int(np.prod(shape[1:]))
            assert abs(v.std().item() / (2.0 / fan_in) ** 0.5 - 1) < 0.35, name
        elif name.endswith(".bias"):
            assert torch.all(v == 0), name
        else:
            assert torch.all(v == 1), name
    assert m._mask_channels() == ores.resnet_mask_channels() == [32, 64, 128, 256]


# ------------------------------------------------------------------------------ engine vs oracle
ENGINE_CASES = [(dims, lossname) for dims in (2, 3) for lossname in LOSSES]


@pytest.mark.parametrize("dims,lossname", ENGINE_CASES)
@pytest.mark.parametrize("train", [False, True])
def test_forward_backward_vs_oracle(dims, lossname, train):
    k = 1 if lossname.startswith("Binary") else (5 if dims == 2 else 3)
    spatial, n = ((32, 32), 3) if dims == 2 else ((16, 16, 16), 2)
    spec = ores.resnet_state_spec(1, k, dims)
    sd = oracle.init_state_dict(spec, seed=7, randomize_affine=True)
    model = _net(dims, k)
    model.load_state_dict(sd, strict=True)
    x, y = case_inputs(dims, spatial, n, k, 5)
    masks = None
    if train:
        torch.manual_seed(3)
        masks = ores.draw_dropout_masks_resnet(n, dims)
        model.train()
        model.dropout_masks = masks
    else:
        model.eval()
    sdg = {s: v.clone().requires_grad_(True) for s, v in sd.items()}
    lo = ores.resnet_forward(sdg, x, dims, masks)
    loss_o = oracle.loss_forward(lossname, lo, y, torch.ones(k))
    loss_o.backward()
    logits = model(x)
    assert isinstance(logits, torch.Tensor) and logits.shape == (n, k) and logits.dtype == torch.float32
    loss = _lossfn(lossname, k)(logits, y)
    loss.backward()
    assert _rel(logits.detach(), lo.detach()) < 5e-6
    assert abs(loss.item() - loss_o.item()) < 1e-5 * max(1, abs(loss_o.item()))
    for name, p in model.named_parameters():
        assert p.grad is not None, name
        assert _rel(p.grad, sdg[name].grad) < 2e-4, name


def test_train_mode_draw_reproduces_reference_stream():
    """no injected masks: the module draws its four masks from the default generator as the reference's do1 calls do"""
    tag, dims, spatial, n, k, _, seed = CASES[0]
    model = _net(dims, k)
    model.load_state_dict(oracle.init_state_dict(ores.resnet_state_spec(1, k, dims), seed=seed, randomize_affine=True))
    model.train()
    x, _ = case_inputs(dims, spatial, n, k, seed)
    torch.manual_seed(TRAIN_SEED)
    with torch.no_grad():
        logits = model(x)
    assert _rel(logits, torch.from_numpy(GOLD[tag + "_train_logits"])) < 5e-6


@pytest.mark.parametrize("lossname", LOSSES)
def test_losses_take_classifier_logits(lossname):
    """(N, C) logits with (N,) or (N, 1) labels give the oracle's value and gradient (the reference's view(bs, C, -1))"""
    k = 1 if lossname.startswith("Binary") else 6
    g = torch.Generator().manual_seed(1)
    z = torch.randn(9, k, generator=g) * 2
    y = (torch.rand(9, generator=g) > 0.5).float() if k == 1 else torch.randint(0, k - 1, (9,), generator=g)
    for lab in (y, y.view(9, 1)):
        zo = z.clone().requires_grad_(True)
        lo = oracle.loss_forward(lossname, zo, lab, torch.ones(k))
        lo.backward()
        zd = z.clone().requires_grad_(True)
        ld = _lossfn(lossname, k)(zd, lab)
        ld.backward()
        assert zd.grad.shape == z.shape
        assert abs(ld.item() - lo.item()) < 1e-6 * max(1, abs(lo.item()))
        assert _rel(zd.grad, zo.grad) < 1e-5


# ------------------------------------------------------------------------------ GraphedStep
@pytest.mark.parametrize("dims", [2, 3])
def test_graphed_step_phases_equal_autograd(dims):
    from pytorchdeeplearing_b200.graphed import GraphedStep
    k = 4
    spatial, n = ((32, 32), 2) if dims == 2 else ((16, 16, 16), 2)
    model = _net(dims, k)
    model.load_state_dict(oracle.init_state_dict(ores.resnet_state_spec(1, k, dims), seed=2, randomize_affine=True))
    model.train()
    torch.manual_seed(8)
    model.dropout_masks = ores.draw_dropout_masks_resnet(n, dims)
    x, y = case_inputs(dims, spatial, n, k, 6)
    lossfn = b200.MutilCrossEntropyLoss(torch.ones(k))
    loss = lossfn(model(x), y)
    loss.backward()
    ref = {s: p.grad.clone() for s, p in model.named_parameters()}
    for p in model.parameters():
        p.grad = None
    step = GraphedStep(model, lossfn, x, y, warmup=1, use_graph=False)
    assert abs(step.loss.item() - loss.item()) < 1e-6 * max(1, abs(loss.item()))
    for s, p in model.named_parameters():
        assert _rel(p.grad, ref[s]) < 1e-5, s


# ------------------------------------------------------------------------------ install, refusals
def test_install_rebinds_resnet_and_uninstall_restores(monkeypatch):
    mods = {}
    for modname, names in (("networks.ResNet2d", ["ResNet2d"]), ("networks.ResNet3d", ["ResNet3d"]),
                           ("model.modelResNet", ["ResNet2d", "ResNet3d", "MutilCrossEntropyLoss", "BinaryFocalLoss"])):
        m = types.ModuleType(modname)
        for name in names:
            setattr(m, name, type(name, (), {"__module__": modname}))
        monkeypatch.setitem(sys.modules, modname, m)
        mods[modname] = m
    orig = {(mn, name): getattr(m, name) for mn, m in mods.items() for name in vars(m) if not name.startswith("__")}
    assert b200.install() == len(orig)
    assert mods["networks.ResNet2d"].ResNet2d is b200.ResNet2d
    assert mods["networks.ResNet3d"].ResNet3d is b200.ResNet3d
    mr = mods["model.modelResNet"]
    assert mr.ResNet2d is b200.ResNet2d and mr.ResNet3d is b200.ResNet3d
    assert mr.MutilCrossEntropyLoss is b200.MutilCrossEntropyLoss and mr.BinaryFocalLoss is b200.BinaryFocalLoss
    b200.uninstall()
    assert all(getattr(mods[mn], name) is obj for (mn, name), obj in orig.items())


def test_clear_errors():
    m3 = b200.ResNet3d(1, 2).eval()
    with pytest.raises(RuntimeError, match="5-D input"):
        m3(torch.zeros(2, 1, 32, 32))
    with pytest.raises(RuntimeError, match="multiples of 16"):
        m3(torch.zeros(1, 1, 16, 24, 16))
    with pytest.raises(RuntimeError, match="multiples of 16"):
        b200.ResNet2d(1, 2)(torch.zeros(1, 1, 40, 32))
    for fn, arg in ((b200.predict, np.zeros((1, 16, 16, 16), np.float32)),
                    (b200.predict_mask, torch.zeros(1, 1, 16, 16, 16)),
                    (b200.sliding_window_mask, np.zeros((1, 16, 16, 16), np.float32))):
        with pytest.raises(TypeError, match="classifier"):
            if fn is b200.sliding_window_mask:
                fn(m3, arg, (16, 16, 16))
            else:
                fn(m3, arg)


# ------------------------------------------------------------------------------ data parallel (gloo, 2 ranks)
def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from test_resnet_cpu import ClsEmuBackend as Emu
    runtime._set_backend_for_testing(Emu())
    runtime.set_precision("fp32")
    k = 4
    model = b200.ResNet2d(1, k)
    model.load_state_dict(oracle.init_state_dict(ores.resnet_state_spec(1, k, 2), seed=4, randomize_affine=True))
    lossfn = b200.MutilCrossEntropyLoss(torch.ones(k))
    x, y = case_inputs(2, (32, 32), 2 * world, k, 9)
    errs = []
    for train in (False, True):
        model.train(train)
        torch.manual_seed(21)
        loss_g = lossfn(model(x), y)
        loss_g.backward()
        ref = {s: p.grad.clone() for s, p in model.named_parameters()}
        for p in model.parameters():
            p.grad = None
        b200.enable_data_parallel()
        sl = slice(2 * rank, 2 * rank + 2)
        torch.manual_seed(21)
        loss = lossfn(model(x[sl]), y[sl])
        loss.backward()
        b200.disable_data_parallel()
        errs.append(abs(loss.item() - loss_g.item()))
        errs.append(max(_rel(p.grad, ref[s]) for s, p in model.named_parameters()))
        for p in model.parameters():
            p.grad = None
    q.put((rank, errs))
    dist.destroy_process_group()


def test_two_rank_sharding_matches_global_batch():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000) + 13
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, (dl_eval, ge_eval, dl_train, ge_train) in res:
        assert dl_eval < 1e-6 and dl_train < 1e-6, (rank, dl_eval, dl_train)
        assert ge_eval < 1e-4 and ge_train < 1e-4, (rank, ge_eval, ge_train)
