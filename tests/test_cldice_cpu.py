"""Soft-clDice (reference model/lossescldice.py, repaired) without a GPU: the oracle against the fixtures the
reference's own bodies produced (tests/golden/cldice.npz) -- skeletons bit for bit, loss and gradient to fp32
rounding --, the fixed-routing fp64 arbiter against fp64 autograd, the argument checks, install()/uninstall() of
model.lossescldice, and the documentation of the defect bridges in the fixture script."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import cldice as ocl
import pytorchdeeplearing_b200 as b200
from conftest import GOLDEN

CASES = ("bin2d", "bin3d_plateau", "mutil3d_c3", "mutil2d_c3")
NAMES = ("soft_skeletonize", "norm_intersection", "Binary_Soft_cldice_loss", "Mutil_Soft_cldice_loss")


def gold():
    return dict(np.load(os.path.join(GOLDEN, "cldice.npz")))


def grid_value(codes):
    """the fixture's uint16 grid codes k -> the fp32 values k / 256 they stand for (exact)"""
    return torch.from_numpy(codes.astype(np.float32)) / 256.0


def case_inputs(g, case):
    pred = grid_value(g[case + "_pred"])
    alpha = torch.from_numpy(g[case + "_alpha"]) if case + "_alpha" in g else None
    target = torch.from_numpy(g[case + "_target"])                 # uint8 in the fixture
    target = target.float() if alpha is None else target.long()
    return pred, target, alpha


def oracle_loss(pred, target, alpha, skeleton=ocl.soft_skeletonize):
    if alpha is None:
        return ocl.binary_loss(pred, target.to(pred.dtype), skeleton)
    return ocl.mutil_loss(pred, target, alpha.to(pred.dtype), skeleton)


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_the_reference_fixture(case):
    g = gold()
    pred, target, alpha = case_inputs(g, case)
    tgt = target if alpha is None else ocl.one_hot(target, pred.shape[1], pred)
    sk_p, sk_t = ocl.soft_skeletonize(pred), ocl.soft_skeletonize(tgt)
    assert torch.equal(sk_p.view(torch.int32), grid_value(g[case + "_sk_pred"]).view(torch.int32))
    assert torch.equal(sk_t.view(torch.int32), grid_value(g[case + "_sk_target"]).view(torch.int32))
    assert not torch.equal(sk_p, pred)                      # the rounds ran
    p = pred.clone().requires_grad_(True)
    loss = oracle_loss(p, target, alpha)
    loss.backward()
    want = float(g[case + "_loss"])
    assert abs(loss.item() - want) <= 4 * np.finfo(np.float32).eps * max(1.0, abs(want))
    ref = torch.from_numpy(g[case + "_grad"])
    assert (p.grad - ref).abs().max() <= 1e-5 * ref.abs().max()


def test_fixtures_hold_exact_plateaus():
    g = gold()
    for case in ("bin3d_plateau", "mutil2d_c3"):
        p = g[case + "_pred"]
        assert (p == 0).sum() > 1000 and (p == 256).sum() > 1000


@pytest.mark.parametrize("case", CASES)
def test_fixed_routing_arbiter_is_the_fp64_function(case):
    """with the fp32 forward's routing, the fp64 skeleton, loss and gradient agree with the reference's fp32 values to
    fp32 rounding"""
    g = gold()
    pred, target, alpha = case_inputs(g, case)
    sk64 = ocl.fixed_skeleton(pred.double())
    assert (sk64 - ocl.soft_skeletonize(pred).double()).abs().max() <= 1e-6
    p = pred.double().requires_grad_(True)
    loss = oracle_loss(p, target, alpha, ocl.fixed_skeleton)
    loss.backward()
    assert abs(loss.item() - float(g[case + "_loss"])) < 1e-5
    ref = torch.from_numpy(g[case + "_grad"]).double()
    assert (p.grad - ref).abs().max() <= 1e-4 * ref.abs().max()


def test_argument_checks():
    x = torch.rand(1, 1, 6, 6, 6)
    with pytest.raises(RuntimeError, match="CUDA"):
        b200.soft_skeletonize(x)                              # no CPU fallback
    with pytest.raises(RuntimeError, match="CUDA"):
        b200.Binary_Soft_cldice_loss()(x, x)
    with pytest.raises(TypeError, match="float32"):
        b200.soft_skeletonize(x.double())
    with pytest.raises(TypeError, match="float32"):
        b200.Binary_Soft_cldice_loss()(x, x.half())
    with pytest.raises(ValueError, match="shape"):
        b200.Binary_Soft_cldice_loss()(x, x[:, :, :5])
    with pytest.raises(ValueError, match=r"\(N, C, H, W\)"):
        b200.soft_skeletonize(x[0, 0])
    with pytest.raises(ValueError, match="empty"):
        b200.soft_skeletonize(x[:0])
    with pytest.raises(ValueError, match="shape"):
        b200.norm_intersection(x, x[:, :, 1:])
    for t in (-1, 65, 2.5, True):
        with pytest.raises(ValueError, match="thresh_width"):
            b200.soft_skeletonize(x, t)
    assert b200.soft_skeletonize(x, 0) is x                  # the reference's empty loop returns x itself
    with pytest.raises(ValueError, match="target"):
        b200.Binary_Soft_cldice_loss()(x, x.clone().requires_grad_(True))
    m = b200.Mutil_Soft_cldice_loss([1.0, 1.0])
    z = torch.rand(1, 2, 6, 6, 6)
    with pytest.raises(ValueError, match="target"):
        m(z, torch.zeros(1, 6, 6, 6, requires_grad=True))
    with pytest.raises(ValueError, match="target shape"):
        m(z, torch.zeros(1, 2, 6, 6, 6, dtype=torch.long))
    with pytest.raises(ValueError, match="alpha"):
        b200.Mutil_Soft_cldice_loss([1.0])(z, torch.zeros(1, 6, 6, 6, dtype=torch.long))


def test_constructors_run_the_intended_initialisers():
    b = b200.Binary_Soft_cldice_loss()
    assert (b.smooth, b.eps) == (1e-5, 1e-7) and isinstance(b, torch.nn.Module)
    m = b200.Mutil_Soft_cldice_loss([0.5, 2.0])
    assert m.alpha == [0.5, 2.0] and isinstance(m.bscldice, b200.Binary_Soft_cldice_loss)


def test_install_rebinds_model_lossescldice_and_uninstall_restores(monkeypatch):
    m = types.ModuleType("model.lossescldice")
    orig = {n: type(n, (), {}) for n in NAMES}
    for n, o in orig.items():
        setattr(m, n, o)
    monkeypatch.setitem(sys.modules, "model.lossescldice", m)
    try:
        assert b200.install() == len(NAMES)
        for n in NAMES:
            assert getattr(m, n) is getattr(b200, n)
    finally:
        b200.uninstall()
    for n in NAMES:
        assert getattr(m, n) is orig[n]


def test_fixture_script_documents_its_defect_bridges():
    path = os.path.join(GOLDEN, "make_golden_cldice.py")
    doc = open(path).read().split('"""')[1]
    for needle in ("tolist()", "__int__", "[:, c:c+1]", "lossescldice.py:10", "lossescldice.py:42",
                   "lossescldice.py:83", "not changed"):
        assert needle in doc, needle
    src = open(path).read()
    assert "loss.__int__()" in src and "channel:channel + 1" in src
