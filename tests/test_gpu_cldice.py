"""Soft-clDice on the H100 (csrc/cldice.cu): skeletons bit-identical to torch's fp32 operator sequence run on the host
(thresh_width 0..10, 2-D and 3-D, tile remainders, extents of 1 and 2, N*C up to 8, NCDHW and channels-last); the
reference fixtures; gradients against the fp64 arbiter routed by the fp32 forward (oracle.cldice.fixed_skeleton), at
least as close as torch's fp32 autograd of the restatement, on random and plateau inputs; bit-identical reruns;
CUDA graph capture; no backward without requires_grad; a target that requires grad raises."""
import os

import numpy as np
import pytest
import torch

from oracle import cldice as ocl
import pytorchdeeplearing_b200 as b200
from conftest import GOLDEN
from test_cldice_cpu import CASES, case_inputs, grid_value, oracle_loss

pytestmark = pytest.mark.gpu


def gold():
    return dict(np.load(os.path.join(GOLDEN, "cldice.npz")))


def layout(t, channels_last):
    if not channels_last:
        return t.contiguous()
    return t.contiguous(memory_format=torch.channels_last_3d if t.dim() == 5 else torch.channels_last)


def field(shape, kind, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(shape, generator=g)
    if kind == "plateau":
        x = (2 * x - 0.5).clamp(0, 1)                  # exact 0 / 1 plateaus
    elif kind == "binary":
        x = (x > 0.6).float()
    return x


SHAPES = [
    (2, 1, 64, 64),
    (1, 3, 37, 45),
    (2, 1, 1, 70),
    (1, 2, 2, 33),
    (2, 1, 32, 32, 32),
    (1, 2, 9, 17, 41),
    (2, 4, 5, 6, 7),                                   # N*C = 8
    (1, 1, 1, 20, 30),
    (1, 1, 2, 2, 40),
    (1, 1, 33, 1, 5),
]


@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("shape", SHAPES)
def test_skeleton_bit_identical_to_torch_fp32(shape, channels_last):
    for kind, seed in (("random", 1), ("plateau", 2), ("binary", 3)):
        x = field(shape, kind, seed + sum(shape))
        xd = layout(x.cuda(), channels_last)
        want = x
        for t in range(11):
            got = b200.soft_skeletonize(xd, t)
            if t:
                want = ocl.soft_skeletonize(want, 1)
            assert got.shape == x.shape
            assert torch.equal(got.cpu().view(torch.int32), want.view(torch.int32)), (kind, t)


@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("case", CASES)
def test_fixture_cases(case, channels_last):
    g = gold()
    pred, target, alpha = case_inputs(g, case)
    p = layout(pred.cuda(), channels_last).requires_grad_(True)
    if alpha is None:
        loss = b200.Binary_Soft_cldice_loss()(p, layout(target.cuda(), channels_last))
    else:
        loss = b200.Mutil_Soft_cldice_loss(alpha.tolist())(p, target.cuda())
    loss.backward()
    want = float(g[case + "_loss"])
    assert loss.dtype == torch.float32 and loss.shape == ()
    assert abs(loss.item() - want) <= 4 * np.finfo(np.float32).eps * max(1.0, abs(want))
    sk = b200.soft_skeletonize(p.detach())
    assert torch.equal(sk.cpu().view(torch.int32), grid_value(g[case + "_sk_pred"]).view(torch.int32))
    # the gradient is held to the fp64 arbiter, at least as close as the reference's own fp32 autograd
    p64 = pred.double().requires_grad_(True)
    oracle_loss(p64, target, alpha, ocl.fixed_skeleton).backward()
    ref32 = torch.from_numpy(g[case + "_grad"]).double()
    e = (p.grad.cpu().double() - p64.grad).norm().item()
    e32 = (ref32 - p64.grad).norm().item()
    assert e <= max(e32, 1e-6 * p64.grad.norm().item()), (e, e32)


def _loss_grad(fn, pred, *args):
    p = pred.clone().requires_grad_(True)
    loss = fn(p, *args)
    loss.backward()
    return loss.detach(), p.grad


GRAD_CASES = [
    ((2, 1, 40, 40, 40), "random", None),
    ((2, 1, 40, 40, 40), "plateau", None),
    ((1, 2, 19, 23, 35), "plateau", None),
    ((8, 1, 100, 70), "random", None),
    ((2, 3, 24, 24, 24), "random", [0.5, 1.0, 2.0]),
    ((2, 3, 60, 50), "plateau", [1.0, 1.0, 1.0]),
]


@pytest.mark.parametrize("shape,kind,alpha", GRAD_CASES)
def test_gradient_against_the_fp64_arbiter(shape, kind, alpha):
    """one routing and ReLU mask set from the fp32 forward: the fp64 arbiter is the function the kernels
    differentiate; the drop-in must be at least as close to it as torch's fp32 autograd"""
    pred = field(shape, kind, 11 + len(shape))
    if alpha is None:
        target = field(shape, "binary", 12)
        args32, args64 = (target,), (target.double(),)
        gpu = _loss_grad(b200.Binary_Soft_cldice_loss(), pred.cuda(), target.cuda())
    else:
        target = torch.randint(0, shape[1], (shape[0],) + shape[2:], generator=torch.Generator().manual_seed(13))
        gpu = _loss_grad(b200.Mutil_Soft_cldice_loss(alpha), pred.cuda(), target.cuda())
        args32 = args64 = None
    if alpha is None:
        l32, g32 = _loss_grad(lambda p, t: ocl.binary_loss(p, t), pred, *args32)
        l64, g64 = _loss_grad(lambda p, t: ocl.binary_loss(p, t, ocl.fixed_skeleton), pred.double(), *args64)
    else:
        a = torch.tensor(alpha)
        l32, g32 = _loss_grad(lambda p: ocl.mutil_loss(p, target, a), pred)
        l64, g64 = _loss_grad(lambda p: ocl.mutil_loss(p, target, a.double(), ocl.fixed_skeleton), pred.double())
    assert abs(gpu[0].item() - l64.item()) <= max(abs(l32.item() - l64.item()), 1e-6)
    e = (gpu[1].cpu().double() - g64).norm().item()
    e32 = (g32.double() - g64).norm().item()
    assert e <= max(e32, 1e-7 * g64.norm().item()), (e, e32)


def test_skeleton_gradient_against_the_fp64_arbiter():
    x = field((2, 1, 30, 31, 33), "plateau", 21)
    cot = torch.randn(x.shape, generator=torch.Generator().manual_seed(22))
    xd = x.cuda().requires_grad_(True)
    b200.soft_skeletonize(xd, 7).backward(cot.cuda())
    x64 = x.double().requires_grad_(True)
    ocl.skeleton_fixed(x64, 7, ref=x).backward(cot.double())
    x32 = x.clone().requires_grad_(True)
    ocl.soft_skeletonize(x32, 7).backward(cot)
    e = (xd.grad.cpu().double() - x64.grad).norm().item()
    e32 = (x32.grad.double() - x64.grad).norm().item()
    assert e <= max(e32, 1e-7 * x64.grad.norm().item()), (e, e32)


def test_norm_intersection_and_its_gradient():
    a = field((2, 3, 9, 10, 11), "random", 31)
    v = field((2, 3, 9, 10, 11), "random", 32)
    ad, vd = a.cuda().requires_grad_(True), v.cuda().requires_grad_(True)
    cot = torch.randn(2, 3, generator=torch.Generator().manual_seed(33))
    r = b200.norm_intersection(ad, vd)
    r.backward(cot.cuda())
    a64, v64 = a.double().requires_grad_(True), v.double().requires_grad_(True)
    r64 = ocl.norm_intersection(a64, v64)
    r64.backward(cot.double())
    assert r.shape == (2, 3) and (r.detach().cpu().double() - r64).abs().max() < 1e-6
    assert (ad.grad.cpu().double() - a64.grad).abs().max() <= 1e-6 * a64.grad.abs().max()
    assert (vd.grad.cpu().double() - v64.grad).abs().max() <= 1e-6 * v64.grad.abs().max()


def test_reruns_are_bit_identical():
    pred = field((2, 1, 36, 40, 44), "plateau", 41).cuda()
    target = field((2, 1, 36, 40, 44), "binary", 42).cuda()
    a = _loss_grad(b200.Binary_Soft_cldice_loss(), pred, target)
    b = _loss_grad(b200.Binary_Soft_cldice_loss(), pred, target)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_cuda_graph_capture_replays_the_eager_result():
    pred = field((2, 3, 20, 24, 28), "random", 51).cuda()
    labels = torch.randint(0, 3, (2, 20, 24, 28), generator=torch.Generator().manual_seed(52)).cuda()
    lossfn = b200.Mutil_Soft_cldice_loss([1.0, 0.5, 2.0])
    eager = _loss_grad(lossfn, pred, labels)
    p = pred.clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            p.grad = None
            lossfn(p, labels).backward()
    torch.cuda.current_stream().wait_stream(s)
    p.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        v = lossfn(p, labels)
        v.backward()
    p.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(v.detach(), eager[0]) and torch.equal(p.grad, eager[1])


def test_no_backward_without_requires_grad_and_target_grad_raises():
    pred = field((1, 1, 12, 13, 14), "random", 61).cuda()
    target = field((1, 1, 12, 13, 14), "binary", 62).cuda()
    loss = b200.Binary_Soft_cldice_loss()(pred, target)
    assert not loss.requires_grad
    with torch.no_grad():
        assert not b200.soft_skeletonize(pred.clone().requires_grad_(True)).requires_grad
    with pytest.raises(ValueError, match="target"):
        b200.Binary_Soft_cldice_loss()(pred, target.clone().requires_grad_(True))
    with pytest.raises(RuntimeError, match="label"):
        b200.Mutil_Soft_cldice_loss([1.0, 1.0])(pred.expand(1, 2, 12, 13, 14).contiguous(),
                                                torch.full((1, 12, 13, 14), 2, device="cuda"))
