"""SSIM / SSIM3D on the H100 (csrc/ssim.cu): every reference fixture with NCDHW-contiguous and channels-last-strided
inputs; random volumes (tile remainders, 2-D, extents smaller than the window, odd and even windows, 0-1 and 0-255
values) against the fp64 oracle, where the kernels must be at least as close as the reference's own fp32 operator
sequence (within 2x of its error); bit-identical reruns; no gradient for an input without requires_grad; and a CUDA
graph capture of forward plus backward."""
import os

import numpy as np
import pytest
import torch

from oracle import ssim as oss
import pytorchdeeplearing_b200 as b200
from conftest import GOLDEN
from test_ssim_cpu import CASES, call, value_and_grads

pytestmark = pytest.mark.gpu


def _gold():
    return dict(np.load(os.path.join(GOLDEN, "ssim.npz")))


def _layout(t, channels_last):
    if not channels_last:
        return t.contiguous()
    return t.contiguous(memory_format=torch.channels_last_3d if t.dim() == 5 else torch.channels_last)


@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("case", list(CASES))
def test_fixture_cases(case, channels_last):
    gold = _gold()
    name, kw = CASES[case]
    x = _layout(torch.from_numpy(gold[case + "_x"]).cuda(), channels_last).requires_grad_(True)
    y = _layout(torch.from_numpy(gold[case + "_y"]).cuda(), channels_last).requires_grad_(True)
    if channels_last and x.shape[1] > 1:
        assert not x.is_contiguous()
    cot = torch.from_numpy(gold[case + "_cot"]).cuda() if case + "_cot" in gold else None
    v, gx, gy = value_and_grads(call(b200, name, kw, x, y), x, y, cot)
    want = torch.from_numpy(gold[case + "_value"])
    assert v.dtype == torch.float32 and v.shape == want.shape
    assert (v.cpu().double() - want.double()).abs().max() < 1e-5
    for g, key in ((gx, "_gx"), (gy, "_gy")):
        ref = torch.from_numpy(gold[case + key]).double()
        assert g.shape == ref.shape
        assert (g.cpu().double() - ref).abs().max() <= 1e-4 * ref.abs().max()


def _pair(shape, scale, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(shape, generator=g, device="cuda")
    y = (0.7 * x + 0.3 * torch.rand(shape, generator=g, device="cuda")).clamp(0, 1)
    return (scale * x).contiguous(), (scale * y).contiguous()


def _run(fn, x, y, cot):
    a, b = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    v = fn(a, b)
    (v * cot).sum().backward()
    return v.detach().double(), a.grad.double(), b.grad.double()


RANDOM = [
    ((2, 1, 96, 96, 96), 11, True),
    ((1, 2, 37, 41, 53), 11, True),
    ((1, 2, 37, 41, 53), 11, False),
    ((2, 3, 45, 70), 11, True),                 # 2-D (the kernels' D = 1)
    ((2, 1, 45, 70), 10, False),
    ((1, 1, 9, 5, 7), 11, True),                # H and W smaller than the window
    ((2, 1, 4, 30, 6), 15, False),
    ((1, 1, 20, 23, 40), 1, True),
    ((1, 1, 20, 23, 40), 3, False),
    ((2, 1, 20, 23, 40), 10, True),
    ((1, 2, 16, 18, 35), 15, True),
    ((1, 1, 33, 34, 35), 31, True),             # the largest window: the smallest tiles
]


@pytest.mark.parametrize("scale", [1.0, 255.0])
@pytest.mark.parametrize("shape,k,size_average", RANDOM)
def test_random_inputs_at_least_as_close_to_fp64_as_the_reference(shape, k, size_average, scale):
    dims = len(shape) - 2
    x, y = _pair(shape, scale, seed=hash((shape, k)) % 1000)
    ms = shape[2:]
    ms = tuple(s + 2 * (k // 2) - k + 1 for s in ms)
    vshape = () if size_average else ((shape[0],) if dims == 2 else (shape[0], ms[-1]))
    cot = torch.randn(vshape, device="cuda") if vshape else torch.ones((), device="cuda")
    fn = b200.ssim if dims == 2 else b200.ssim3D
    got = _run(lambda a, b: fn(a, b, k, size_average), x, y, cot)
    ref64 = _run(lambda a, b: oss.ssim(a, b, k, size_average, dims, torch.float64), x, y, cot.double())
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False        # the reference's fp32 arithmetic without TF32: the stricter bar
    try:
        ref32 = _run(lambda a, b: oss.ssim(a, b, k, size_average, dims, torch.float32), x, y, cot)
    finally:
        torch.backends.cudnn.allow_tf32 = prev

    def verr(v):
        return (v - ref64[0]).abs().max().item()

    def gerr(g, r):
        return ((g - r).norm() / r.norm()).item()

    assert got[0].shape == ref64[0].shape
    assert verr(got[0]) <= max(2 * verr(ref32[0]), 1e-6), (verr(got[0]), verr(ref32[0]))
    for i in (1, 2):
        e, e32 = gerr(got[i], ref64[i]), gerr(ref32[i], ref64[i])
        assert e <= max(2 * e32, 1e-5), (i, e, e32)


def test_reruns_are_bit_identical():
    x, y = _pair((2, 2, 40, 44, 50), 1.0, seed=3)
    for size_average in (True, False):
        cot = torch.ones(()) if size_average else torch.randn(2, 50)
        a = _run(lambda p, q: b200.ssim3D(p, q, 11, size_average), x, y, cot.cuda())
        b = _run(lambda p, q: b200.ssim3D(p, q, 11, size_average), x, y, cot.cuda())
        for u, v in zip(a, b):
            assert torch.equal(u, v)


def test_no_gradient_for_an_input_without_requires_grad():
    x, y = _pair((1, 1, 20, 22, 24), 1.0, seed=4)
    a, b = x.clone(), y.clone().requires_grad_(True)
    b200.ssim3D(a, b).backward()
    assert a.grad is None and b.grad is not None
    full = _run(lambda p, q: b200.ssim3D(p, q), x, y, torch.ones((), device="cuda"))
    assert torch.equal(b.grad.double(), full[2])
    with torch.no_grad():
        v = b200.SSIM()(x[:, :, 0], y[:, :, 0])
    assert not v.requires_grad


def test_cuda_graph_capture_replays_the_eager_result():
    """forward plus backward captured into one CUDA graph: nothing in either synchronises with the host"""
    x, y = _pair((2, 1, 32, 36, 40), 1.0, seed=5)
    eager = _run(lambda p, q: b200.ssim3D(p, q), x, y, torch.ones((), device="cuda"))
    a, b = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            a.grad = b.grad = None
            b200.ssim3D(a, b).backward()
    torch.cuda.current_stream().wait_stream(s)
    a.grad = b.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        v = b200.ssim3D(a, b)
        v.backward()
    a.grad.zero_()
    b.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(v.detach().double(), eager[0])
    assert torch.equal(a.grad.double(), eager[1]) and torch.equal(b.grad.double(), eager[2])
