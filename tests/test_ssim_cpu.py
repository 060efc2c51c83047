"""SSIM / SSIM3D (reference model/lossesSSIM.py) without a GPU: the oracle against the fixtures the real reference
produced (tests/golden/ssim.npz), the host's 1-D taps bit for bit, the modules' attributes and return shapes, the
refusals, install()/uninstall() of model.lossesSSIM, and the host logic on an emulated backend: the backward
coefficients and the adjoint filter against fp64 autograd, and a two-rank gloo run against the global batch."""
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ssim as oss
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import runtime
from pytorchdeeplearing_b200.ssim import gaussian_taps, map_shape
from conftest import GOLDEN

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

# fixture case -> (callable name, kwargs)
CASES = {
    "ssim2d_c1": ("SSIM", {}),
    "ssim2d_c3_per_sample": ("SSIM", {"size_average": False}),
    "ssim2d_fn_k10": ("ssim", {"window_size": 10}),
    "ssim3d_c1": ("SSIM3D", {}),
    "ssim3d_c2_per_sample": ("SSIM3D", {"size_average": False}),
    "ssim3d_fn_k5": ("ssim3D", {"window_size": 5}),
    "ssim3d_fn_k10": ("ssim3D", {"window_size": 10}),
    "ssim3d_d3": ("SSIM3D", {}),
    "ssim3d_scaled255": ("SSIM3D", {}),
}


def _gold():
    return dict(np.load(os.path.join(GOLDEN, "ssim.npz")))


def call(mod, name, kw, x, y):
    """the fixture case's callable from ``mod`` (the drop-in package or the reference module)"""
    if name in ("SSIM", "SSIM3D"):
        return getattr(mod, name)(**kw)(x, y)
    return getattr(mod, name)(x, y, **kw)


def value_and_grads(v, x, y, cot):
    (v * cot).sum().backward() if cot is not None else v.backward()
    return v.detach(), x.grad, y.grad


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_oracle_matches_reference_fixture(case, dtype):
    gold = _gold()
    name, kw = CASES[case]
    x = torch.from_numpy(gold[case + "_x"]).requires_grad_(True)
    y = torch.from_numpy(gold[case + "_y"]).requires_grad_(True)
    v = oss.ssim(x, y, kw.get("window_size", 11), kw.get("size_average", True), dims=x.dim() - 2, dtype=dtype)
    cot = torch.from_numpy(gold[case + "_cot"]).to(dtype) if case + "_cot" in gold else None
    v, gx, gy = value_and_grads(v, x, y, cot)
    want = torch.from_numpy(gold[case + "_value"])
    assert v.shape == want.shape
    assert (v.double() - want.double()).abs().max() < 1e-5
    for g, key in ((gx, "_gx"), (gy, "_gy")):
        ref = torch.from_numpy(gold[case + key]).double()
        assert (g.double() - ref).abs().max() <= 1e-4 * ref.abs().max()


def test_host_taps_equal_the_reference_bit_for_bit():
    gold = _gold()
    keys = [k for k in gold if k.startswith("taps")]
    assert sorted(keys) == ["taps10", "taps11", "taps5"]
    for key in keys:
        k = int(key[4:])
        want = gold[key]
        assert want.dtype == np.float32
        assert np.array_equal(gaussian_taps(k).numpy().view(np.uint32), want.view(np.uint32))
        assert np.array_equal(oss.gaussian(k).numpy().view(np.uint32), want.view(np.uint32))


def test_map_shape_follows_the_padding_rule():
    assert map_shape((2, 1, 20, 24, 28), 11) == (20, 24, 28)
    assert map_shape((2, 1, 20, 24, 28), 10) == (21, 25, 29)
    assert map_shape((1, 1, 3, 5), 1) == (3, 5)


def test_constructor_defaults_and_attributes():
    for cls in (b200.SSIM, b200.SSIM3D):
        m = cls()
        assert (m.window_size, m.size_average, m.channel) == (11, True, 1)
        m = cls(window_size=7, size_average=False)
        assert (m.window_size, m.size_average) == (7, False)
        assert not hasattr(m, "window")
        assert isinstance(m, torch.nn.Module)


def test_refusals():
    x = torch.rand(1, 1, 8, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        b200.ssim3D(x, x)                               # no CPU fallback
    with pytest.raises(TypeError, match="float32"):
        b200.ssim3D(x.double(), x.double())
    with pytest.raises(TypeError, match="float32"):
        b200.ssim(x[:, :, 0].half(), x[:, :, 0].half())
    with pytest.raises(ValueError, match="shape"):
        b200.ssim3D(x, x[:, :, :7])
    with pytest.raises(ValueError, match=r"\(N, C, H, W\)"):
        b200.ssim(x, x)
    with pytest.raises(ValueError, match=r"\(N, C, D, H, W\)"):
        b200.SSIM3D()(x[:, :, 0], x[:, :, 0])
    for k in (0, 32, -1, 2.5):
        with pytest.raises(ValueError, match="window_size"):
            b200.ssim3D(x, x, window_size=k)


def test_install_rebinds_model_lossesSSIM_and_uninstall_restores(monkeypatch):
    names = ("SSIM", "SSIM3D", "ssim", "ssim3D")
    m = types.ModuleType("model.lossesSSIM")
    orig = {n: type(n, (), {}) for n in names}
    for n, o in orig.items():
        setattr(m, n, o)
    monkeypatch.setitem(sys.modules, "model.lossesSSIM", m)
    try:
        assert b200.install() == len(names)
        for n in names:
            assert getattr(m, n) is getattr(b200, n)
    finally:
        b200.uninstall()
    for n in names:
        assert getattr(m, n) is orig[n]


# ------------------------------------------------------------------------------------------------ emulated backend
class SsimEmu:
    """The three SSIM entry points in fp64 torch, with the closed-form coefficients of csrc/ssim.cu and the adjoint
    filter as a transposed convolution: checks the host logic and the backward formulas without a GPU."""

    @staticmethod
    def _conv(t, k, dims, transpose=False):
        c = t.shape[1]
        w = oss.window(k, dims).double()
        w = w.expand(c, 1, *w.shape).contiguous()
        if transpose:
            f = F.conv_transpose2d if dims == 2 else F.conv_transpose3d
        else:
            f = F.conv2d if dims == 2 else F.conv3d
        return f(t, w, padding=k // 2, groups=c)

    def ssim_fwd(self, img1, img2, window_size, taps, coef):
        dims, k = img1.dim() - 2, window_size
        x, y = img1.double(), img2.double()
        mu1, mu2 = self._conv(x, k, dims), self._conv(y, k, dims)
        m11, m22, m12 = self._conv(x * x, k, dims), self._conv(y * y, k, dims), self._conv(x * y, k, dims)
        A, B = 2 * mu1 * mu2 + oss.C1, 2 * (m12 - mu1 * mu2) + oss.C2
        Q, R = mu1 ** 2 + mu2 ** 2 + oss.C1, (m11 - mu1 ** 2) + (m22 - mu2 ** 2) + oss.C2
        S = A * B / (Q * R)
        if coef is not None:
            d1 = 2 * mu2 * B / (Q * R) - 2 * mu1 * S / Q + 2 * mu1 * S / R - 2 * mu2 * A / (Q * R)
            d2 = 2 * mu1 * B / (Q * R) - 2 * mu2 * S / Q + 2 * mu2 * S / R - 2 * mu1 * A / (Q * R)
            coef.copy_(torch.stack([d1, d2, -S / R, 2 * A / (Q * R)]).reshape(4, -1))
        return S

    def ssim_finalize(self, img1, window_size, size_average, ws, acc, value, reduce=True):
        if reduce:
            if size_average:
                acc.copy_(torch.tensor([ws.sum().item(), float(ws.numel())], dtype=torch.float64))
            else:
                acc.copy_(ws.sum((1, 2, 3)))            # (N,) for 2-D, (N, W') for 3-D
        cnt = acc[1] if size_average else ws.numel() / acc.numel()
        value.copy_((acc[0] / cnt if size_average else acc / cnt).float())

    def ssim_bwd(self, img1, img2, window_size, taps, coef, size_average, gout, acc, grad1, grad2):
        dims, k = img1.dim() - 2, window_size
        n, c = img1.shape[:2]
        cf = coef.reshape(4, n, c, *map_shape(img1.shape, k))
        g = gout.double()
        if size_average:
            s = g / acc[1]
        elif dims == 2:
            s = g.reshape(n, 1, 1, 1) / (cf[0].numel() / n)
        else:
            s = g.reshape(n, 1, 1, 1, -1) / (cf[0].numel() / g.numel())
        f = [self._conv(s * cf[i], k, dims, transpose=True) for i in range(4)]
        x, y = img1.double(), img2.double()
        if grad1 is not None:
            grad1.copy_(f[0] + 2 * x * f[2] + y * f[3])
        if grad2 is not None:
            grad2.copy_(f[1] + 2 * y * f[2] + x * f[3])


@pytest.fixture()
def emu():
    runtime._set_backend_for_testing(SsimEmu())
    yield
    runtime._set_backend_for_testing(None)


@pytest.mark.parametrize("case", list(CASES))
def test_emulated_backend_matches_fp64_autograd(emu, case):
    """value, both gradients and the return shape of the drop-in (host logic + closed-form backward) against fp64
    autograd of the oracle"""
    gold = _gold()
    name, kw = CASES[case]
    x0, y0 = torch.from_numpy(gold[case + "_x"]), torch.from_numpy(gold[case + "_y"])
    cot = torch.from_numpy(gold[case + "_cot"]) if case + "_cot" in gold else None
    x, y = x0.clone().requires_grad_(True), y0.clone().requires_grad_(True)
    v, gx, gy = value_and_grads(call(b200, name, kw, x, y), x, y, cot)
    xr, yr = x0.double().requires_grad_(True), y0.double().requires_grad_(True)
    vr = oss.ssim(xr, yr, kw.get("window_size", 11), kw.get("size_average", True), dtype=torch.float64)
    vr, gxr, gyr = value_and_grads(vr, xr, yr, None if cot is None else cot.double())
    assert v.dtype == torch.float32 and v.shape == vr.shape == gold[case + "_value"].shape
    assert (v.double() - vr).abs().max() < 1e-6
    for g, r in ((gx, gxr), (gy, gyr)):
        assert g.dtype == torch.float32 and g.shape == r.shape
        assert (g.double() - r).norm() <= 1e-6 * r.norm()


def test_emulated_backend_shapes_channel_and_partial_gradients(emu):
    x = torch.rand(2, 3, 9, 10)
    m = b200.SSIM(size_average=False)
    assert m(x, x).shape == (2,) and m.channel == 3
    m3 = b200.SSIM3D(size_average=False, window_size=4)
    v = m3(torch.rand(2, 2, 5, 6, 7), torch.rand(2, 2, 5, 6, 7))
    assert v.shape == (2, 8) and m3.channel == 2                 # (N, W') with W' = W + 1 for an even window
    assert b200.ssim3D(torch.rand(1, 1, 4, 5, 6), torch.rand(1, 1, 4, 5, 6)).shape == ()
    a, b = torch.rand(1, 1, 6, 7, 8), torch.rand(1, 1, 6, 7, 8, requires_grad=True)
    b200.ssim3D(a, b).backward()
    assert a.grad is None and b.grad is not None


# ------------------------------------------------------------------------------------------------ data parallel
def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import pytorchdeeplearing_b200 as b200
    from pytorchdeeplearing_b200 import runtime
    from test_ssim_cpu import SsimEmu
    runtime._set_backend_for_testing(SsimEmu())
    g = torch.Generator().manual_seed(5)
    x = torch.rand((2 * world, 2, 6, 7, 9), generator=g)
    y = (0.6 * x + 0.4 * torch.rand(x.shape, generator=g))
    errs = []
    for size_average in (True, False):
        xg, yg = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
        vg = b200.ssim3D(xg, yg, 5, size_average)
        vg.sum().backward()
        sl = slice(2 * rank, 2 * rank + 2)
        b200.enable_data_parallel()
        xs, ys = x[sl].clone().requires_grad_(True), y[sl].clone().requires_grad_(True)
        v = b200.ssim3D(xs, ys, 5, size_average)
        v.sum().backward()
        b200.disable_data_parallel()
        want = vg.detach() if size_average else vg.detach()[sl]
        errs.append((v.detach() - want).abs().max().item())
        for gl, gg in ((xs.grad, xg.grad[sl]), (ys.grad, yg.grad[sl])):
            errs.append(((gl - gg).norm() / gg.norm()).item())
    q.put((rank, max(errs)))
    dist.destroy_process_group()


def test_two_rank_gloo_matches_global_batch():
    """rank r holds samples [2r, 2r+2): the mean is the global-batch mean on every rank and each rank's gradient is
    its slice of the global-batch gradient; the per-sample form needs no exchange"""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, err in res:
        assert err < 1e-6, (rank, err)
