"""Grad-CAM of ResNet2d on the GPU (csrc/gradcam.cu + the data-gradient-only ResNet backward) against the reference's
maps (tests/golden/gradcam.npz) and the fp64 oracle (oracle/gradcam.py)."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import gradcam as og
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import runtime
from pytorchdeeplearing_b200.engine import Engine, RESNET_STAGES

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = dict(np.load(os.path.join(HERE, "golden", "gradcam.npz")))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_gradcam import CASES, case_weights  # noqa: E402

IDS = [c[0] for c in CASES]
# end to end against the reference's map, fp32 storage (the engine's fp32 convolutions vs the reference's CPU ones);
# measured maximum 3.3e-6 over the six cases on an H100 80GB HBM3
FP32_BOUND = 1e-5
# end to end in bf16 against the fp64 oracle on the same weights: bf16 activations and data gradients, and the
# per-image min-max scale magnifies them where a map's range is small; measured maximum 0.19 (r64_n3), 0.012-0.059
# on the other cases, on an H100 80GB HBM3
BF16_BOUND = 0.3


@pytest.fixture
def precision():
    prev = runtime.get_precision()
    yield runtime.set_precision
    runtime.set_precision(prev)


def _stages(tag):
    n = len([k for k in GOLD if k.startswith(tag + "/A")])
    return [GOLD[f"{tag}/A{i}"] for i in range(n)], [GOLD[f"{tag}/g{i}"] for i in range(n)]


def _cl(a, dtype=torch.float32):
    """(N, C, h, w) numpy -> (N, 1, h, w, C) channels-last CUDA"""
    return torch.from_numpy(a).cuda().permute(0, 2, 3, 1).unsqueeze(1).contiguous().to(dtype)


def _model(k, seed):
    m = b200.ResNet2d(1, k)
    m.load_state_dict(case_weights(k, seed))
    return m.cuda()


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_kernels_on_reference_stages(case):
    """fed the reference's hooked fp32 A and g: as close to fp64 as the reference itself, plus 2^-22"""
    tag, hw, n, k, stages, target, seed = case
    acts, grads = _stages(tag)
    want = og.grad_cam_map(acts, grads, *hw)
    be = runtime.get_backend(torch.empty(0, device="cuda"))
    out = torch.empty((n,) + hw, dtype=torch.float32, device="cuda")
    be.gradcam([(_cl(a), _cl(g)) for a, g in zip(acts, grads)], out)
    ours = float(np.abs(out.cpu().numpy() - want).max())
    ref = float(np.abs(GOLD[tag + "/map"] - want).max())
    print(f"{tag}: max |ours - fp64| = {ours:.3e}, max |reference - fp64| = {ref:.3e}")
    assert ours <= ref + 2.0 ** -22
    out2 = torch.empty_like(out)
    be.gradcam([(_cl(a), _cl(g)) for a, g in zip(acts, grads)], out2)
    assert torch.equal(out, out2)
    # bf16 operands take the same kernels
    outb = torch.empty_like(out)
    be.gradcam([(_cl(a, torch.bfloat16), _cl(g, torch.bfloat16)) for a, g in zip(acts, grads)], outb)
    assert float((outb - out).abs().max()) < 0.05


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_end_to_end_fp32_matches_reference(case, precision):
    precision("fp32")
    tag, hw, n, k, stages, target, seed = case
    m = _model(k, seed)
    for p in m.parameters():
        p.grad = torch.full_like(p, 0.25)
    x = torch.from_numpy(GOLD[tag + "/x"]).cuda()
    out = b200.grad_cam(m, x, target, stages)
    err = float((out.cpu() - torch.from_numpy(GOLD[tag + "/map"])).abs().max())
    print(f"{tag}: fp32 end to end, max |ours - reference| = {err:.3e}")
    assert err <= FP32_BOUND
    assert all(torch.equal(p.grad, torch.full_like(p, 0.25)) for p in m.parameters())
    assert torch.equal(out, b200.grad_cam(m, x, target, stages))
    if target is None:
        logits = m.eval()(x)
        assert int(logits[0].argmax()) == int(GOLD[tag + "/category"])


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_end_to_end_bf16_matches_fp64_oracle(case, precision):
    precision("bf16")
    tag, hw, n, k, stages, target, seed = case
    m = _model(k, seed)
    x = torch.from_numpy(GOLD[tag + "/x"])
    out = b200.grad_cam(m, x.cuda(), target, stages)
    sd = {s: v.detach().double().cpu() for s, v in m.state_dict().items()}
    A, g, _ = og.stage_grads(sd, x.double(), target, stages)
    want = og.grad_cam_map([a.numpy() for a in A], [v.numpy() for v in g], *hw)
    err = float(np.abs(out.cpu().numpy() - want).max())
    print(f"{tag}: bf16 end to end, max |ours - fp64 oracle| = {err:.3e}")
    assert err <= BF16_BOUND
    assert torch.equal(out, b200.grad_cam(m, x.cuda(), target, stages))


@pytest.mark.parametrize("mode", ["fp32", "bf16"])
def test_stage_gradients_bit_identical_to_full_backward(mode, precision):
    precision(mode)
    m = _model(10, 0)
    P = dict(zip(m._pnames, [p.detach() for p in m.parameters()]))
    x = torch.randn(4, 1, 64, 64, generator=torch.Generator().manual_seed(5)).cuda()
    be = runtime.get_backend(x)
    dl = torch.zeros(4, 10, device="cuda")
    dl[:, 3] = 1
    T = runtime.act_dtype()
    for stage in RESNET_STAGES:
        eng = Engine(be, T, 2)
        eng.resnet_forward(P, x, None, need_grad=True)
        got = eng.resnet_backward(dl, stages=[stage])[stage][1]
        full = Engine(be, T, 2)
        full.resnet_forward(P, x, None, need_grad=True)
        seen = {}
        orig = full.bwd_layer
        # d loss / d (stage output): what the stage's last residual op receives, or for in_tr what down_tr32's down
        # convolution hands back
        last = {"down_tr32": 1}.get(stage, 2)

        def spy(L, g_act, need_dx, *a, **kw):
            if L.wname == f"{stage}.ops.{last}.conv1.weight":
                seen["g"] = g_act.clone()
            r = orig(L, g_act, need_dx, *a, **kw)
            if stage == "in_tr" and L.wname == "down_tr32.down_conv.weight":
                seen["g"] = r.clone()
            return r
        full.bwd_layer = spy
        full.resnet_backward(dl)
        torch.cuda.synchronize()
        want = seen["g"]
        assert torch.equal(got, want), (mode, stage)


def test_batched_validation_set_and_reruns(precision):
    """128 images at the reference's ResNet2d size in one call; each row equals its own single-image call"""
    precision("bf16")
    m = _model(10, 0)
    x = torch.randn(128, 1, 64, 64, generator=torch.Generator().manual_seed(1)).cuda()
    a = b200.grad_cam(m, x, None, ["down_tr128", "down_tr256"])
    assert a.shape == (128, 64, 64) and bool(torch.isfinite(a).all())
    assert float(a.amin()) >= 0 and float(a.amax()) <= 1
    assert torch.equal(a, b200.grad_cam(m, x, None, ["down_tr128", "down_tr256"]))
    precision("fp32")
    b = b200.grad_cam(m, x, None, ["down_tr256"])
    for i in (0, 77):
        assert float((b[i] - b200.grad_cam(m, x[i:i + 1], None, ["down_tr256"])[0]).abs().max()) < 1e-4


def test_gradcam_class_on_gpu(capsys):
    tag, hw, n, k, stages, target, seed = CASES[5]
    m = _model(k, seed)
    cam = b200.GradCAM(m, [getattr(m, s) for s in stages])
    out = cam(torch.from_numpy(GOLD[tag + "/x"]), None)
    assert "category id:" in capsys.readouterr().out
    assert isinstance(out, np.ndarray) and out.shape == (n,) + hw and out.dtype == np.float32
