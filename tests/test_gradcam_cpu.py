"""Grad-CAM of ResNet2d on CPU: the fp64 oracle (oracle/gradcam.py) against maps of the reference's own GradCAM
(tests/golden/gradcam.npz), the drop-in's host logic (eval forward, data-gradient-only backward, stage selection,
GradCAM class, install) on the emulated backend, and the refusals."""
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle
from oracle import gradcam as og
from oracle import resnet as ores
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import runtime
from pytorchdeeplearing_b200.engine import Engine, RESNET_STAGES
from test_resnet_cpu import ClsEmuBackend

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = dict(np.load(os.path.join(HERE, "golden", "gradcam.npz")))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_gradcam import CASES, case_input, case_weights  # noqa: E402

# the reference's map vs the fp64 oracle fed the same hooked A and g: fp32 rounding of the reference and OpenCV's
# IPP resize only (measured maximum 5.2e-7 over the six cases)
ORACLE_BOUND = 2e-6


class CamEmuBackend(ClsEmuBackend):
    """the classifier-head emulation plus the Grad-CAM entry points (b200seg_gradcam_*) in fp64 torch ops"""

    def gradcam_target(self, logits, target, dlogits, category):
        t = logits.argmax(1) if target < 0 else torch.full((logits.shape[0],), target, dtype=torch.int64)
        category.copy_(t)
        dlogits.copy_(F.one_hot(t, logits.shape[1]).to(dlogits.dtype))

    def gradcam(self, stages, out):
        """per stage w = mean g, relu(sum_c w A), min-max scale, bilinear (half-pixel centres, clamped borders) to
        out's size; mean over the stages, min-max scale"""
        H, W = out.shape[1:]

        def scale(m):
            m = m - m.amin(dim=(1, 2), keepdim=True)
            return m / (1e-7 + m.amax(dim=(1, 2), keepdim=True))

        acc = 0
        for a, g in stages:
            a, g = a[:, 0].double(), g[:, 0].double()                     # (N, h, w, C)
            cam = scale((a * g.mean(dim=(1, 2), keepdim=True)).sum(-1).clamp_min(0))
            if cam.shape[1:] != (H, W):
                cam = F.interpolate(cam[:, None], size=(H, W), mode="bilinear", align_corners=False)[:, 0]
            acc = acc + cam
        out.copy_(scale(acc / len(stages)).float())


def case_stages(tag):
    n = len([k for k in GOLD if k.startswith(tag + "/A")])
    return [GOLD[f"{tag}/A{i}"] for i in range(n)], [GOLD[f"{tag}/g{i}"] for i in range(n)]


@pytest.fixture(autouse=True)
def _emu():
    runtime._set_backend_for_testing(CamEmuBackend())
    prev = runtime.get_precision()
    runtime.set_precision("fp32")
    yield
    b200.uninstall()
    runtime._set_backend_for_testing(None)
    runtime.set_precision(prev)


# ------------------------------------------------------------------------------ oracle vs the reference's maps
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_matches_reference_maps(case):
    tag, hw, n, k, stages, target, seed = case
    sd = case_weights(k, seed)
    np.testing.assert_allclose([float(v.double().sum()) for v in sd.values()], GOLD[tag + "/wsum"], rtol=0, atol=0)
    assert torch.equal(case_input(hw, n, seed), torch.from_numpy(GOLD[tag + "/x"]))
    acts, grads = case_stages(tag)
    ref = GOLD[tag + "/map"]
    got = og.grad_cam_map(acts, grads, *hw)
    err = float(np.abs(got - ref).max())
    print(f"{tag}: max |oracle - reference| = {err:.3e}")
    assert err <= ORACLE_BOUND
    # the fp64 forward / backward of the oracle reproduces the hooked tensors and the class
    A, g, t = og.stage_grads({s: v.double() for s, v in sd.items()}, torch.from_numpy(GOLD[tag + "/x"]).double(),
                             target, stages)
    assert int(t[0]) == int(GOLD[tag + "/category"])
    for a64, g64, a32, g32 in zip(A, g, acts, grads):
        np.testing.assert_allclose(a64.numpy(), a32, rtol=1e-4, atol=1e-4 * np.abs(a32).max())
        np.testing.assert_allclose(g64.numpy(), g32, rtol=1e-4, atol=1e-4 * np.abs(g32).max())


def test_cv_coefficients_follow_opencv_rule():
    i0, i1, a = og.cv_linear_coeffs(64, 4)
    assert i0[0] == 0 and a[0, 1] == 0 and i0[-1] == 3 and i1[-1] == 3 and a[-1, 1] == 0
    assert np.all(a.sum(1) == 1) and np.all(i1 - i0 <= 1)
    img = np.arange(12, dtype=np.float32).reshape(3, 4)
    assert np.array_equal(og.resize_linear(img, 3, 4), img)


# ------------------------------------------------------------------------------ drop-in host logic (emulated)
def _model(k, seed):
    m = b200.ResNet2d(1, k)
    m.load_state_dict(case_weights(k, seed))
    return m


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_grad_cam_matches_reference(case):
    tag, hw, n, k, stages, target, seed = case
    m = _model(k, seed)
    for p in m.parameters():
        p.grad = torch.full_like(p, 0.5)
    got = b200.grad_cam(m, torch.from_numpy(GOLD[tag + "/x"]), target, stages)
    assert got.dtype == torch.float32 and got.shape == (n,) + hw
    err = float((got - torch.from_numpy(GOLD[tag + "/map"])).abs().max())
    print(f"{tag}: max |emulated drop-in - reference| = {err:.3e}")
    assert err < 1e-3
    assert all(torch.equal(p.grad, torch.full_like(p, 0.5)) for p in m.parameters())


def test_stage_gradients_equal_full_backward():
    """the data-gradient-only backward hands back exactly the g the full backward carries at each stage"""
    tag, hw, n, k, _, _, seed = CASES[0]
    m = _model(k, seed)
    P = dict(zip(m._pnames, [p.detach() for p in m.parameters()]))
    x = torch.from_numpy(GOLD[tag + "/x"])
    be = runtime.get_backend(x)
    dl = torch.zeros(n, k)
    dl[:, 3] = 1
    for stage in RESNET_STAGES:
        eng = Engine(be, torch.float32, 2)
        eng.resnet_forward(P, x, None, need_grad=True)
        found = eng.resnet_backward(dl, stages=[stage])
        assert list(found) == [stage]
        calls = []
        eng2 = Engine(be, torch.float32, 2)
        eng2.resnet_forward(P, x, None, need_grad=True)
        orig = eng2.bwd_layer

        def spy(L, g_act, need_dx, *a, **kw):
            calls.append((L.wname, g_act.clone()))
            return orig(L, g_act, need_dx, *a, **kw)
        eng2.bwd_layer = spy
        flat = eng2.resnet_backward(dl)
        assert isinstance(flat, torch.Tensor)
        # the gradient w.r.t. a stage's output is the one the next layer's backward receives as an addend-free input
        first = {"in_tr": "in_tr.conv1.weight", "down_tr32": "down_tr32.ops.1.conv1.weight",
                 "down_tr64": "down_tr64.ops.2.conv1.weight", "down_tr128": "down_tr128.ops.2.conv1.weight",
                 "down_tr256": "down_tr256.ops.2.conv1.weight"}[stage]
        want = next(g for w, g in calls if w == first)
        assert torch.equal(found[stage][1], want)
        expect_out = {"in_tr": eng.saved["down_tr32"][0].x, "down_tr256": eng.saved["head"][0]}.get(stage)
        if expect_out is None:
            nxt = RESNET_STAGES[RESNET_STAGES.index(stage) + 1]
            expect_out = eng.saved[nxt][0].x
        assert found[stage][0] is expect_out


def test_data_only_backward_skips_weight_gradients():
    tag, hw, n, k, _, _, seed = CASES[0]
    m = _model(k, seed)
    P = dict(zip(m._pnames, [p.detach() for p in m.parameters()]))
    x = torch.from_numpy(GOLD[tag + "/x"])
    be = runtime.get_backend(x)
    count = {"wgrad": 0, "conv": 0}

    class Counting(type(be)):
        def wgrad(self, *a, **k):
            count["wgrad"] += 1
            return super().wgrad(*a, **k)

        def conv(self, *a, **k):
            count["conv"] += 1
            return super().conv(*a, **k)
    eng = Engine(Counting(), torch.float32, 2)
    eng.resnet_forward(P, x, None, need_grad=True)
    fwd = count["conv"]
    eng.resnet_backward(torch.ones(n, k), stages=["down_tr128"])
    assert count["wgrad"] == 0
    assert count["conv"] - fwd == 4              # the data gradients of down_tr256 (3 ops + down conv), then stop
    assert not eng._data_only


def test_target_none_takes_each_rows_argmax_and_repeats_average():
    tag, hw, n, k, stages, _, seed = CASES[3]
    m = _model(k, seed)
    x = torch.from_numpy(GOLD[tag + "/x"])
    logits = m.eval()(x)
    per_row = torch.stack([b200.grad_cam(m, x[i:i + 1], int(logits[i].argmax()), stages)[0] for i in range(n)])
    assert (b200.grad_cam(m, x, None, stages) - per_row).abs().max() < 1e-4
    one = b200.grad_cam(m, x, 2, ["down_tr128"])
    assert torch.allclose(b200.grad_cam(m, x, 2, ["down_tr128", "down_tr128"]), one, atol=1e-6)
    # layer order does not matter: the reference's hooks record in forward order
    assert torch.equal(b200.grad_cam(m, x, 2, ["down_tr256", "in_tr"]), b200.grad_cam(m, x, 2, ["in_tr", "down_tr256"]))


def test_gradcam_class_contract(capsys):
    tag, hw, n, k, stages, target, seed = CASES[5]
    m = _model(k, seed)
    m.train()
    x = torch.from_numpy(GOLD[tag + "/x"])
    with b200.GradCAM(model=m, target_layers=[getattr(m, s) for s in stages], use_cuda=False) as cam:
        assert not m.training
        out = cam(input_tensor=x, target_category=None)
    assert f"category id: {int(GOLD[tag + '/category'])}" in capsys.readouterr().out
    assert isinstance(out, np.ndarray) and out.dtype == np.float32 and out.shape == (n,) + hw
    assert np.abs(out - GOLD[tag + "/map"]).max() < 1e-3
    with b200.GradCAM(m, [m.down_tr256]) as cam:
        raise IndexError("swallowed as in the reference")
    assert "swallowed as in the reference" in capsys.readouterr().out
    cam(x, 3)
    assert capsys.readouterr().out == ""             # no print with an explicit category


def test_errors():
    m = _model(10, 0)
    x = torch.zeros(1, 1, 32, 32)
    with pytest.raises(ValueError, match="outside"):
        b200.grad_cam(m, x, 10)
    with pytest.raises(ValueError, match="outside"):
        b200.GradCAM(m, [m.down_tr256])(x, -1)
    for bad in ("bn1", "down_tr64.ops.0", "fc_layers"):
        with pytest.raises(NotImplementedError, match="down_tr256"):
            b200.grad_cam(m, x, 0, [bad])
    for mod in (m.down_tr64.bn1, m.down_tr64.ops[0], m.in_tr.conv1, torch.nn.Conv2d(1, 1, 1)):
        with pytest.raises(NotImplementedError, match="in_tr, down_tr32"):
            b200.GradCAM(m, [mod])
    with pytest.raises(NotImplementedError, match="reshape_transform"):
        b200.GradCAM(m, [m.down_tr256], reshape_transform=lambda t: t)
    with pytest.raises(NotImplementedError, match="ResNet3d"):
        b200.grad_cam(b200.ResNet3d(1, 2), torch.zeros(1, 1, 16, 16, 16))
    with pytest.raises(NotImplementedError, match="VNet2d"):
        b200.GradCAM(b200.VNet2d(1, 2), [])
    with pytest.raises(RuntimeError, match="multiples of 16"):
        b200.grad_cam(m, torch.zeros(1, 1, 40, 32))


# ------------------------------------------------------------------------------ install
def test_install_rebinds_gradcam(monkeypatch):
    mods = {}
    for modname in ("model.visualization", "model.modelResNet"):
        mod = types.ModuleType(modname)
        mod.GradCAM = type("GradCAM", (), {})
        monkeypatch.setitem(sys.modules, modname, mod)
        mods[modname] = mod
    orig = {k: v.GradCAM for k, v in mods.items()}
    assert b200.install() == 2
    assert all(v.GradCAM is b200.GradCAM for v in mods.values())
    b200.uninstall()
    assert all(v.GradCAM is orig[k] for k, v in mods.items())


def test_installed_grad_cam_visual(monkeypatch):
    """the unmodified reference MutilResNet2dModel.Grad_CAM_Visual, with install(), returns the (H, W) map"""
    import ref_harness
    if not ref_harness.available():
        pytest.skip("no reference checkout named by PYTORCHDEEPLEARING_REFERENCE")
    for name in list(sys.modules):
        if name == "model" or name.startswith(("model.", "networks", "dataprocess")):
            monkeypatch.delitem(sys.modules, name)
    monkeypatch.setattr(sys, "path", list(sys.path))
    before = set(sys.modules)
    try:
        _grad_cam_visual()
    finally:
        b200.uninstall()
        for name in set(sys.modules) - before:      # later tests must not see the reference's modules
            del sys.modules[name]


def _grad_cam_visual():
    import ref_harness
    ref_harness.import_reference()
    import importlib
    importlib.import_module("networks.ResNet2d").prob = 0.2
    mr = importlib.import_module("model.modelResNet")
    b200.install()
    assert mr.GradCAM is b200.GradCAM
    tag, hw, n, k, stages, target, seed = CASES[0]
    wrapper = object.__new__(mr.MutilResNet2dModel)
    wrapper.model, wrapper.device, wrapper.use_cuda = _model(k, seed), torch.device("cpu"), False
    img = GOLD[tag + "/x"][0]
    cam = wrapper.Grad_CAM_Visual(img, 3, [wrapper.model.down_tr256])
    assert cam.shape == hw and cam.dtype == np.float32
    assert np.abs(cam - GOLD[tag + "/map"][0]).max() < 1e-3
