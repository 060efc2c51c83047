"""UNet3dthin (reference networks/Unet3dthin.py) on the CPU: the oracle against the reference's recorded outputs, the
drop-in's state_dict and initialisation, the layer program on the emulated backend against the fixtures (eval and
train mode), ``install()`` and a two-rank data-parallel run."""
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import oracle
from oracle import nets as onets
from oracle import unetthin as othin
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import runtime
from emu_backend import EmuBackend

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = dict(np.load(os.path.join(HERE, "golden", "unet3dthin.npz")))

torch.set_num_threads(max(1, min(8, os.cpu_count() or 1)))

# tag: (in_channels, classes, init_features, input shape, weight seed, loss); as in make_golden_unet3dthin.py
CASES = {
    "c2_32": (1, 2, 16, (2, 1, 32, 32, 32), 0, "MutilDiceLoss"),
    "c5_32x48x48": (1, 5, 16, (1, 1, 32, 48, 48), 1, "MutilCrossEntropyDiceLoss"),
    "c1_32": (1, 1, 16, (1, 1, 32, 32, 32), 2, "BinaryDiceLoss"),
    "c3_f8_32": (2, 3, 8, (1, 2, 32, 32, 32), 3, "MutilCrossEntropyDiceLoss"),
}


class ThinEmuBackend(EmuBackend):
    """the emulated backend; its two upsample ops are torch's trilinear interpolation and its autograd"""


@pytest.fixture()
def emu():
    runtime._set_backend_for_testing(ThinEmuBackend())
    prev = runtime.get_precision()
    runtime.set_precision("fp32")
    yield
    runtime._set_backend_for_testing(None)
    runtime.set_precision(prev)


def _case(tag):
    cin, ncls, f, shape, wseed, lossname = CASES[tag]
    spec = othin.unetthin_state_spec(cin, ncls, f)
    sd = onets.init_state_dict(spec, seed=wseed, randomize_affine=True)
    x, y = oracle.make_inputs(shape[0], cin, shape[2:], ncls, seed=1234)
    return spec, sd, x, y, ncls, f, lossname


def _sub(t):
    return t.detach()[:, :, ::2, ::2, ::2]


def _grads_table(grads, names):
    return np.array([[grads[n].double().norm().item(), grads[n].double().sum().item()] for n in names])


# gradient agreement with the fixture (relative to each gradient's norm).  MutilDiceLoss on c2_32 is ill-conditioned in
# fp32: the oracle's own fp32 gradients differ from its fp64 ones by 6.5e-3 there, so that case gets a looser bound.
GRAD_TOL = {"c2_32": 2e-2, "c5_32x48x48": 2e-4, "c1_32": 2e-4, "c3_f8_32": 2e-4}


def _check_grads(table, tag, spec):
    ref, tol = GOLD[tag + ".grads"], GRAD_TOL[tag]
    root_numel = np.sqrt([float(np.prod(shape)) for _, shape in spec])
    assert np.all(np.abs(table[:, 0] - ref[:, 0]) <= tol * ref[:, 0] + 1e-9), tag
    # |sum(d)| <= sqrt(numel) * |d|: the sums follow from the norm bound
    assert np.all(np.abs(table[:, 1] - ref[:, 1]) <= tol * ref[:, 0] * root_numel + 1e-9), tag


@pytest.mark.parametrize("tag", list(CASES))
def test_oracle_matches_reference_fixture(tag):
    spec, sd, x, y, ncls, f, lossname = _case(tag)
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    lo, po = othin.unetthin_forward(sdg, x)
    ref = torch.from_numpy(GOLD[tag + ".logits"])
    assert (_sub(lo) - ref).norm() / ref.norm() < 5e-6
    am = (po > 0.5).sum() if ncls == 1 else po.argmax(1).sum()
    assert int(am) == int(GOLD[tag + ".argmax_sum"])
    alpha = None if lossname.startswith("Binary") else torch.ones(ncls)
    loss = oracle.loss_forward(lossname, lo, y, alpha)
    assert abs(loss.item() - float(GOLD[tag + ".loss"])) < 1e-5 * max(1.0, abs(loss.item()))
    loss.backward()
    _check_grads(_grads_table({k: v.grad for k, v in sdg.items()}, [n for n, _ in spec]), tag, spec)
    # train mode: the reference's per-module draws, in call order
    torch.manual_seed(int(GOLD[tag + ".train_seed"]))
    masks = othin.draw_dropout_masks_unetthin(x.shape[0], f)
    lt, _ = othin.unetthin_forward(sd, x, masks)
    ref = torch.from_numpy(GOLD[tag + ".train_logits"])
    assert (_sub(lt) - ref).norm() / ref.norm() < 5e-6


def test_state_dict_layout_and_initialize_weights():
    m = b200.UNet3dthin(1, 2)
    spec = othin.unetthin_state_spec(1, 2)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == spec
    assert len(spec) == 56 and sum(p.numel() for p in m.parameters()) == 5298002
    assert all(isinstance(getattr(m, f"decoder{k}")[0], torch.nn.Conv3d) for k in (1, 2, 3, 4))
    assert isinstance(m.encoder1[1], torch.nn.GroupNorm) and isinstance(m.conv, torch.nn.Conv3d)
    # constructor and initialize_weights consume the generator as the reference's do: same values
    torch.manual_seed(int(GOLD["init_seed"]))
    m = b200.UNet3dthin(1, 2)
    m.apply(b200.initialize_weights)
    got = np.array([[v.double().sum().item(), (v.double() ** 2).sum().item()] for v in m.state_dict().values()])
    np.testing.assert_allclose(got, GOLD["init"], rtol=1e-9, atol=1e-9)
    m2 = b200.UNet3dthin(1, 2, init_features=8)
    m2.load_state_dict(onets.init_state_dict(othin.unetthin_state_spec(1, 2, 8)), strict=True)


@pytest.mark.parametrize("tag", list(CASES))
def test_dropin_on_emulated_backend_matches_fixture(emu, tag):
    spec, sd, x, y, ncls, f, lossname = _case(tag)
    cin = x.shape[1]
    model = b200.UNet3dthin(cin, ncls, init_features=f)
    model.load_state_dict(sd, strict=True)
    model.eval()
    lossfn = getattr(b200, lossname)() if lossname.startswith("Binary") else getattr(b200, lossname)(torch.ones(ncls))
    logits, probs = model(x)
    assert logits.shape == (x.shape[0], ncls) + tuple(x.shape[2:])
    ref = torch.from_numpy(GOLD[tag + ".logits"])
    assert (_sub(logits) - ref).norm() / ref.norm() < 5e-6
    loss = lossfn(logits, y)
    assert abs(loss.item() - float(GOLD[tag + ".loss"])) < 1e-5 * max(1.0, abs(loss.item()))
    loss.backward()
    _check_grads(_grads_table({n: p.grad for n, p in model.named_parameters()}, [n for n, _ in spec]), tag, spec)
    # train mode: the drop-in draws its masks from the default generator exactly as the reference modules do
    model.train()
    torch.manual_seed(int(GOLD[tag + ".train_seed"]))
    with torch.no_grad():
        lt, _ = model(x)
    ref = torch.from_numpy(GOLD[tag + ".train_logits"])
    assert (_sub(lt) - ref).norm() / ref.norm() < 5e-6


def test_dropin_train_mode_gradients_match_oracle(emu):
    spec, sd, x, y, ncls, f, lossname = _case("c2_32")
    model = b200.UNet3dthin(1, 2)
    model.load_state_dict(sd, strict=True)
    torch.manual_seed(3)
    masks = othin.draw_dropout_masks_unetthin(2)
    model.train()
    model.dropout_masks = masks
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    lo, _ = othin.unetthin_forward(sdg, x, masks)
    alpha = torch.tensor([0.7, 1.3])
    oracle.loss_forward("MutilCrossEntropyDiceLoss", lo, y, alpha).backward()
    logits, _ = model(x)
    b200.MutilCrossEntropyDiceLoss(alpha)(logits, y).backward()
    assert (logits - lo).norm() / lo.norm() < 5e-6
    for n, p in model.named_parameters():
        go = sdg[n].grad
        assert (p.grad - go).norm() / (go.norm() + 1e-12) < 2e-4, n


def test_emulated_upsample_ops_are_adjoint():
    be = ThinEmuBackend()
    g = torch.Generator().manual_seed(0)
    a = torch.randn((2, 3, 5, 4, 8), generator=g, dtype=torch.float64).float()
    gs = torch.randn((2, 6, 10, 8, 8), generator=g, dtype=torch.float64).float()
    s = torch.empty_like(gs)
    be.upsample_add(a, torch.zeros_like(gs), s)
    ga = torch.empty_like(a)
    be.upsample_bwd(gs, ga)
    lhs = (s.double() * gs.double()).sum()
    rhs = (a.double() * ga.double()).sum()
    assert abs(lhs - rhs) < 1e-4 * abs(lhs)


def test_plain_schedule_and_input_size_check(monkeypatch):
    from pytorchdeeplearing_b200 import engine
    monkeypatch.delenv("B200SEG_OVERLAP", raising=False)
    assert engine.overlap_mask("unetthin", 3) == 0
    assert b200.UNet3dthin._arch == "unetthin"
    assert hasattr(engine.Engine, "unetthin_forward") and hasattr(engine.Engine, "unetthin_backward")
    with pytest.raises(RuntimeError, match="multiples of 16"):
        b200.UNet3dthin(1, 2)(torch.zeros(1, 1, 16, 16, 24))


def test_install_rebinds_a_planted_unet3dthin_module(monkeypatch):
    """``install()`` rebinds ``UNet3dthin`` in ``networks.Unet3dthin`` (a stand-in here: the real reference module is
    never imported into this process) and ``uninstall()`` restores it"""
    stand_in = type("UNet3dthin", (), {"__module__": "networks.Unet3dthin"})
    mod = types.ModuleType("networks.Unet3dthin")
    mod.UNet3dthin = stand_in
    monkeypatch.setitem(sys.modules, "networks.Unet3dthin", mod)
    try:
        n = b200.install()
        assert n >= 1 and mod.UNet3dthin is b200.UNet3dthin
        assert b200.install() == 0
    finally:
        b200.uninstall()
    assert mod.UNet3dthin is stand_in


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import oracle
    from oracle import nets as onets
    import pytorchdeeplearing_b200 as b200
    from pytorchdeeplearing_b200 import runtime
    from pytorchdeeplearing_b200.graphed import GraphedStep
    from test_unet3dthin_cpu import ThinEmuBackend
    runtime._set_backend_for_testing(ThinEmuBackend())
    runtime.set_precision("fp32")
    model, lossfn = b200.UNet3dthin(1, 2), b200.MutilCrossEntropyDiceLoss(torch.ones(2))
    spec = [(k, tuple(v.shape)) for k, v in model.state_dict().items()]
    model.load_state_dict(onets.init_state_dict(spec, seed=4, randomize_affine=True))
    x, y = oracle.make_inputs(2 * world, 1, (16, 16, 16), 2, seed=9)
    sl = slice(2 * rank, 2 * rank + 2)
    # eval: autograd path; the single-process result on the GLOBAL batch first (no collectives)
    model.eval()
    loss_g = lossfn(model(x)[0], y)
    loss_g.backward()
    ref = {n: p.grad.clone() for n, p in model.named_parameters()}
    for p in model.parameters():
        p.grad = None
    b200.enable_data_parallel()
    loss = lossfn(model(x[sl])[0], y[sl])
    loss.backward()
    b200.disable_data_parallel()
    err = max(((p.grad - ref[n]).norm() / (ref[n].norm() + 1e-12)).item() for n, p in model.named_parameters())
    # train: every rank takes its rows of the global-batch dropout draw; GraphedStep drives the engine directly
    model.train()
    for p in model.parameters():
        p.grad = None
    torch.manual_seed(21)
    loss_t = lossfn(model(x)[0], y)
    loss_t.backward()
    ref_t = {n: p.grad.clone() for n, p in model.named_parameters()}
    b200.enable_data_parallel()
    torch.manual_seed(21)
    step = GraphedStep(model, lossfn, x[sl], y[sl], warmup=1, use_graph=False)
    b200.disable_data_parallel()
    err_t = max(((p.grad - ref_t[n]).norm() / (ref_t[n].norm() + 1e-12)).item() for n, p in model.named_parameters())
    q.put((rank, max(abs(loss.item() - loss_g.item()), abs(step.loss.item() - loss_t.item())), max(err, err_t)))
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
    for rank, dloss, gerr in res:
        assert dloss < 1e-6, (rank, dloss)
        assert gerr < 1e-4, (rank, gerr)
