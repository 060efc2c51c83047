"""UNet3dthin on the GPU: the trilinear upsample-and-add kernel and its adjoint bit for bit, the adjoint identity,
rejected arguments, the convolution families the net takes, fp32 parity with the oracle at both benchmark sizes, and
the bf16 / train / captured / inference modes."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle
from oracle import nets as onets
from oracle import unetthin as othin
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import _abi
from test_gpu_conv_exact import (C, GUARD, IN_FILL, K3, Q, Guarded, W, _check_stats_guard, _k, _run_conv,
                                 assert_bitwise, assert_guards, check_stats, exact_bound, stats_chain,
                                 tiles_per_sample, wgrad_bound)

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = dict(np.load(os.path.join(HERE, "golden", "unet3dthin.npz")))


@pytest.fixture(scope="module")
def be():
    return _abi.CudaBackend()


@pytest.fixture(autouse=True)
def _restore_precision():
    prev = b200.get_precision()
    yield
    b200.set_precision(prev)


# ------------------------------------------------------------------------------------------------ fp64 restatement
def _taps(n, device):
    """per fine index of an axis with n coarse cells: (i0, i1, w0, w1) of torch's align_corners=False scale-2 rule"""
    j = torch.arange(2 * n, device=device)
    k = j // 2
    odd = (j % 2) == 1
    i0 = torch.where(odd, k, (k - 1).clamp(min=0))
    i1 = torch.where(odd, (k + 1).clamp(max=n - 1), k)
    w0 = torch.where(odd, torch.full_like(j, 3), torch.full_like(j, 1)).double() / 4
    w1 = 1 - w0
    w0 = torch.where((~odd) & (k == 0), torch.ones_like(w0), w0)           # fine 0: coarse 0 with 1
    w1 = torch.where((~odd) & (k == 0), torch.zeros_like(w1), w1)
    w0 = torch.where(odd & (k == n - 1), torch.ones_like(w0), w0)          # last fine: last coarse with 1
    w1 = torch.where(odd & (k == n - 1), torch.zeros_like(w1), w1)
    return i0, i1, w0, w1


def up2_ref(a):
    """(N, D, H, W, C) fp64 -> (N, 2D, 2H, 2W, C), one axis at a time (exact for grid operands)"""
    out = a.double()
    for ax in (1, 2, 3):
        i0, i1, w0, w1 = _taps(out.shape[ax], out.device)
        shp = [1] * 5
        shp[ax] = -1
        out = out.index_select(ax, i0) * w0.view(shp) + out.index_select(ax, i1) * w1.view(shp)
    return out


def up2t_ref(g):
    """the adjoint of up2_ref: (N, 2D, 2H, 2W, C) -> (N, D, H, W, C) in fp64"""
    out = g.double()
    for ax in (1, 2, 3):
        n = out.shape[ax] // 2
        i0, i1, w0, w1 = _taps(n, out.device)
        shp = [1] * 5
        shp[ax] = -1
        size = list(out.shape)
        size[ax] = n
        acc = torch.zeros(size, dtype=torch.float64, device=out.device)
        acc.index_add_(ax, i0, out * w0.view(shp))
        acc.index_add_(ax, i1, out * w1.view(shp))
        out = acc
    return out


def grid(shape, dtype, gen, lo=-8, hi=8, k=3):
    """small integers x 2^-k: representable in bf16, and every fp32 sum of the kernels is exact"""
    return (torch.randint(lo, hi + 1, shape, generator=gen).double() * 2.0 ** -k).to(dtype)


def test_restatement_matches_torch_interpolate():
    g = torch.Generator().manual_seed(0)
    for shp in ((1, 1, 1, 1, 8), (2, 3, 5, 7, 16), (1, 4, 2, 6, 8)):
        a = torch.randn(shp, generator=g, dtype=torch.float64)
        want = F.interpolate(a.permute(0, 4, 1, 2, 3), scale_factor=2, mode="trilinear").permute(0, 2, 3, 4, 1)
        assert torch.allclose(up2_ref(a), want, rtol=0, atol=1e-12)
        gs = torch.randn(want.shape, generator=g, dtype=torch.float64)
        ai = a.permute(0, 4, 1, 2, 3).clone().requires_grad_(True)
        (ga,) = torch.autograd.grad(F.interpolate(ai, scale_factor=2, mode="trilinear"), ai, gs.permute(0, 4, 1, 2, 3))
        assert torch.allclose(up2t_ref(gs), ga.permute(0, 2, 3, 4, 1), rtol=0, atol=1e-12)


# --------------------------------------------------------------------------------------------- kernels bit for bit
SHAPES = [  # (N, coarse D, H, W, C)
    (1, 1, 1, 1, 8), (1, 1, 2, 3, 16), (2, 3, 5, 7, 32), (1, 4, 4, 4, 64), (3, 2, 3, 2, 128), (1, 3, 1, 5, 256),
    (2, 6, 6, 6, 128), (2, 12, 12, 12, 64), (2, 24, 24, 24, 32), (2, 48, 48, 48, 16),       # 2 x 96^3
    (1, 8, 7, 7, 128), (1, 16, 14, 14, 64), (1, 32, 28, 28, 32), (1, 64, 56, 56, 16),       # 1 x 128 x 112 x 112
]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_upsample_kernels_bitwise(be, shape, dtype):
    n, d, h, w, c = shape
    fine = (n, 2 * d, 2 * h, 2 * w, c)
    gen = torch.Generator().manual_seed(sum(shape))
    a, e, gs = grid(shape, dtype, gen), grid(fine, dtype, gen), grid(fine, dtype, gen)
    A, E, S = Guarded(shape, dtype, device="cuda"), Guarded(fine, dtype, device="cuda"), Guarded(fine, dtype, device="cuda")
    A.view.copy_(a)
    E.view.copy_(e)
    GS, GA = Guarded(fine, dtype, device="cuda"), Guarded(shape, dtype, device="cuda")
    GS.view.copy_(gs)
    A.outside0, E.outside0, GS.outside0 = (t.buf.cpu()[~t.inside].clone() for t in (A, E, GS))
    be.upsample_add(A.view, E.view, S.view)
    be.upsample_bwd(GS.view, GA.view)
    torch.cuda.synchronize()
    want_s = (up2_ref(a.cuda()) + e.cuda().double()).to(dtype)
    want_ga = up2t_ref(gs.cuda()).to(dtype)
    assert_bitwise(S.view, want_s, "upsample2_add")
    assert_bitwise(GA.view, want_ga, "upsample2_bwd")
    for t, what in ((A, "a"), (E, "e"), (S, "S"), (GS, "gS"), (GA, "ga")):
        assert_guards(t, what)
    # reruns are bit-identical
    s2, ga2 = torch.empty_like(S.view), torch.empty_like(GA.view)
    be.upsample_add(A.view, E.view, s2)
    be.upsample_bwd(GS.view, ga2)
    assert torch.equal(s2.view(torch.int16 if dtype == torch.bfloat16 else torch.int32),
                       S.view.contiguous().view(torch.int16 if dtype == torch.bfloat16 else torch.int32))
    assert torch.equal(ga2.view(torch.int16 if dtype == torch.bfloat16 else torch.int32),
                       GA.view.contiguous().view(torch.int16 if dtype == torch.bfloat16 else torch.int32))


@pytest.mark.parametrize("shape", [(2, 3, 5, 7, 32), (2, 48, 48, 48, 16), (1, 8, 7, 7, 128)],
                         ids=lambda s: "x".join(map(str, s)))
def test_adjoint_identity_and_torch_autograd(be, shape):
    n, d, h, w, c = shape
    g = torch.Generator(device="cuda").manual_seed(1)
    a = torch.randn(shape, generator=g, device="cuda")
    gs = torch.randn((n, 2 * d, 2 * h, 2 * w, c), generator=g, device="cuda")
    s, ga = torch.empty_like(gs), torch.empty_like(a)
    be.upsample_add(a, torch.zeros_like(gs), s)
    be.upsample_bwd(gs, ga)
    lhs = (s.double() * gs.double()).sum().item()
    rhs = (a.double() * ga.double()).sum().item()
    assert abs(lhs - rhs) <= 1e-5 * (s.double().abs() * gs.double().abs()).sum().item()
    ai = a.permute(0, 4, 1, 2, 3).double().requires_grad_(True)
    (want,) = torch.autograd.grad(F.interpolate(ai, scale_factor=2, mode="trilinear"), ai,
                                  gs.permute(0, 4, 1, 2, 3).double())
    assert ((ga.double() - want.permute(0, 2, 3, 4, 1)).norm() / want.norm()).item() < 1e-6


def test_out_of_contract_arguments_are_rejected(be):
    def t(shape, dtype=torch.bfloat16):
        return torch.zeros(shape, dtype=dtype, device="cuda")
    a, s = t((1, 2, 2, 2, 16)), t((1, 4, 4, 4, 16))
    bad = [
        ("shape", lambda: be.upsample_add(a, s, t((1, 4, 4, 6, 16)))),
        ("skip shape", lambda: be.upsample_add(a, t((1, 4, 4, 4, 8)), s)),
        ("dtype", lambda: be.upsample_add(a, t((1, 4, 4, 4, 16), torch.float32), s)),
        ("C % 8", lambda: be.upsample_add(t((1, 2, 2, 2, 12)), t((1, 4, 4, 4, 12)), t((1, 4, 4, 4, 12)))),
        ("pitch", lambda: be.upsample_add(t((1, 2, 2, 2, 20))[..., :16], s, s)),
        ("alignment", lambda: be.upsample_add(t((1, 2, 2, 2, 24))[..., 4:20], s, s)),
        ("bwd shape", lambda: be.upsample_bwd(s, t((1, 2, 2, 3, 16)))),
        ("bwd dtype", lambda: be.upsample_bwd(s, t((1, 2, 2, 2, 16), torch.float32))),
        ("bwd C % 8", lambda: be.upsample_bwd(t((1, 4, 4, 4, 4)), t((1, 2, 2, 2, 4)))),
    ]
    for what, call in bad:
        with pytest.raises(RuntimeError, match="libb200seg error -1"):
            call()
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ conv families
def _convs(n, sp, f=16, cin=1):
    """(name, x shape, y shape) of every forward convolution of UNet3dthin and its data-gradient twin"""
    sps = [tuple(sp)]
    for _ in range(4):
        sps.append(tuple(s // 2 for s in sps[-1]))
    ch = [f, 2 * f, 4 * f, 8 * f, 16 * f]
    out = []
    ins = [cin, f, 2 * f, 4 * f, 8 * f]
    for i in range(5):
        out.append((f"enc{i}.conv1", sps[i], ins[i], ch[i]))
        out.append((f"enc{i}.conv2", sps[i], ch[i], ch[i]))
    dins = {4: 16 * f, 3: 8 * f, 2: 4 * f, 1: 2 * f}
    for k in (4, 3, 2, 1):
        out.append((f"dec{k}.conv1", sps[k], dins[k], ch[k - 1]))
        out.append((f"dec{k}.conv2", sps[k], ch[k - 1], ch[k - 1]))
    return out


@pytest.mark.parametrize("n,sp", [(2, (96, 96, 96)), (1, (128, 112, 112))], ids=["2x96", "1x128x112x112"])
def test_every_convolution_takes_a_tensor_core_family_in_bf16(be, n, sp):
    from pytorchdeeplearing_b200.engine import K3
    paths = {}
    for name, s, ci, co in _convs(n, sp):
        vox = s[0] * s[1] * s[2]
        w = torch.randn((co, ci, 3, 3, 3), device="cuda")
        # (the network input reaches the first convolution as fp32)
        x = torch.empty((n,) + s + (ci,), dtype=torch.float32 if ci == 1 else torch.bfloat16, device="cuda")
        y = torch.empty((n,) + s + (co,), dtype=torch.bfloat16, device="cuda")
        wf = be.pack_weight(w, K3, "fwd", torch.bfloat16, 3, vox=vox)
        paths[name] = be.conv_path(K3, 3, x, wf, y)
        if not name.startswith("enc0.conv1"):           # the first layer has no data gradient
            wd = be.pack_weight(w, K3, "dgrad", torch.bfloat16, 3, vox=vox)
            paths[name + ".dgrad"] = be.conv_path(K3, 3, y, wd, x)
    generic = {k: v for k, v in paths.items() if v == "GENERIC"}
    assert not generic, generic
    print(paths)


# ------------------------------------------------- every convolution of the net in bf16, bit for bit
# Each forward, data-gradient and weight-gradient convolution of UNet3dthin at both benchmark sizes runs on the kernel
# family the engine gives it (the operand is packed with the layer's own voxel count, as Engine._prepack does), on
# guarded, pitched buffers, with the exact-sum operands of test_gpu_conv_exact.py, and is compared bit for bit with an
# fp64 reference (computed on the GPU: every partial sum of the grid operands is exact in fp64).
SIZES = {"2x96": (2, (96, 96, 96)), "1x128x112x112": (1, (128, 112, 112))}
LAYERS = [(size, name) for size, (n, sp) in SIZES.items() for name, *_ in _convs(n, sp)]


def _layer(size, name):
    n, sp = SIZES[size]
    _, s, ci, co = next(c for c in _convs(n, sp) if c[0] == name)
    return n, s, ci, co


def _engine_path(be, n, s, ci, co, which):
    """the family b200seg_conv takes for this layer as the engine calls it"""
    vox = s[0] * s[1] * s[2]
    w = torch.zeros((co, ci, 3, 3, 3), device="cuda")
    # (the network input reaches the first convolution as fp32)
    x = torch.empty((n,) + s + (ci,), dtype=torch.float32 if ci == 1 else torch.bfloat16, device="cuda")
    y = torch.empty((n,) + s + (co,), dtype=torch.bfloat16, device="cuda")
    wp = be.pack_weight(w, K3, which, torch.bfloat16, 3, vox=vox)
    return be.conv_path(K3, 3, x, wp, y) if which == "fwd" else be.conv_path(K3, 3, y, wp, x)


def _ref_conv(cs, x, w):
    """fp64 reference of the layer's forward conv or its data gradient (the transposed conv), on x's device"""
    xin = x.permute(0, 4, 1, 2, 3)
    if cs["which"] == "fwd":
        out = F.conv3d(xin, w, None, padding=1)
    else:
        out = F.conv_transpose3d(xin, w, None, padding=1)
    return out.permute(0, 2, 3, 4, 1).contiguous()


def _grid_dev(shape, k, e, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(-k, k + 1, shape, generator=g, device="cuda").double() * 2.0 ** -e


@pytest.mark.parametrize("which", ["fwd", "dgrad"])
@pytest.mark.parametrize("size,name", LAYERS, ids=[f"{s}-{nm}" for s, nm in LAYERS])
def test_every_convolution_bitwise_bf16(be, size, name, which):
    n, s, ci, co = _layer(size, name)
    if which == "dgrad" and ci == 1:
        pytest.skip("the first layer has no data gradient")
    path = _engine_path(be, n, s, ci, co, which)
    assert path != "GENERIC", (size, name, which)
    ys, c_out = (s, co) if which == "fwd" else (s, ci)
    # statistics only where their fp32 chain bound stays 100x below one tile's share of a channel sum
    stats = which == "fwd" and stats_chain(path, n, ys, c_out) * tiles_per_sample(ys) * 2.0 ** -24 * 100 <= 1
    cs = C(path, K3, which, 3, n, s, ci, co, halo=path in ("HALO3", "HALO_WS"), bias=False, addend=False,
           stats=stats, x_f32=ci == 1, x_dense=ci == 1)
    c_in = ci if which == "fwd" else co
    x = _grid_dev((n,) + s + (c_in,), 4, 2, seed=len(name) + ci)
    w = _grid_dev((co, ci, 3, 3, 3), 8, 5, seed=co + 7)
    assert exact_bound(cs, x, w, None, None) < 2 ** 20 * Q
    v = _ref_conv(cs, x, w)
    want = v.float().bfloat16()
    gy, gx, _, gs = _run_conv(be, cs, w, x, None, None, stats)
    assert_bitwise(gy.view, want, f"{size} {name} {which} ({path})")
    assert_guards(gy, f"{name} {which}")
    assert_guards(gx, f"{name} {which} input")
    if stats:
        _check_stats_guard(gs, name)
        check_stats(gs[GUARD:-GUARD].view(n, c_out, 2), v, stats_chain(path, n, ys, c_out), name)


@pytest.mark.parametrize("size,name", LAYERS, ids=[f"{s}-{nm}" for s, nm in LAYERS])
def test_every_weight_gradient_bitwise(be, size, name):
    n, s, ci, co = _layer(size, name)
    ws = W(None, K3, 3, n, s, ci, co, a_dtype="f32" if ci == 1 else "bf16", a_dense=ci == 1)
    assert 2 * wgrad_bound(ws) < 2 ** 24 * 0.5
    g = torch.Generator(device="cuda").manual_seed(ci + co)
    a = torch.randint(-1, 2, (n,) + s + (ci,), generator=g, device="cuda").double()
    b = torch.randint(-1, 2, (n,) + s + (co,), generator=g, device="cuda").double() * 0.5
    w0 = torch.zeros((co, ci, 3, 3, 3), dtype=torch.float64, device="cuda", requires_grad=True)
    with torch.enable_grad():
        F.conv3d(a.permute(0, 4, 1, 2, 3), w0, None, padding=1).backward(b.permute(0, 4, 1, 2, 3))
    want = w0.grad.reshape(co, ci, 27).permute(2, 1, 0).contiguous().float()
    adt = torch.float32 if ci == 1 else torch.bfloat16
    ga = Guarded(a.shape, adt, fill=IN_FILL, device="cuda", dense=ci == 1)
    ga.view.copy_(a.to(adt))
    gb = Guarded(b.shape, torch.bfloat16, fill=IN_FILL, device="cuda")
    gb.view.copy_(b.bfloat16())
    buf = torch.full((2 * GUARD + want.numel(),), float("nan"), device="cuda")
    buf[GUARD:-GUARD] = 0
    dwp = buf[GUARD:-GUARD].view(want.shape)
    path = be.wgrad_path(K3, 3, ga.view, gb.view)
    be.wgrad(K3, 3, ga.view, gb.view, dwp)
    torch.cuda.synchronize()
    assert_bitwise(dwp.view(27, ci, co, 1, 1), want.view(27, ci, co, 1, 1), f"{size} {name} wgrad ({path})")
    assert bool(torch.cat([buf[:GUARD], buf[-GUARD:]]).isnan().all()), f"{name}: dwp guard band written"
    assert_guards(ga, name + " a")
    assert_guards(gb, name + " b")


# --------------------------------------------------------------------------------------------- network parity
def _model(cin, ncls, seed, f=16):
    spec = othin.unetthin_state_spec(cin, ncls, f)
    sd = onets.init_state_dict(spec, seed=seed, randomize_affine=True)
    model = b200.UNet3dthin(cin, ncls, init_features=f)
    model.load_state_dict(sd, strict=True)
    return sd, model.cuda()


def _oracle(sd, x, y, lossname, alpha, masks=None):
    """the oracle in fp64 on the GPU (cuDNN fp64 has no reduced-precision modes)"""
    sdg = {k: v.cuda().double().requires_grad_(True) for k, v in sd.items()}
    ms = None if masks is None else [m.cuda().double() for m in masks]
    lo, po = othin.unetthin_forward(sdg, x.cuda().double(), ms)
    loss = oracle.loss_forward(lossname, lo, y.cuda(), None if alpha is None else alpha.cuda().double(),
                               dtype=torch.float64)
    loss.backward()
    return lo.detach(), po.detach(), loss.item(), {k: v.grad.detach() for k, v in sdg.items()}


@pytest.mark.parametrize("n,sp,ncls", [(2, (96, 96, 96), 2), (1, (128, 112, 112), 5)], ids=["2x96_c2", "1x128x112x112_c5"])
def test_fp32_parity_at_benchmark_sizes(n, sp, ncls):
    b200.set_precision("fp32")
    sd, model = _model(1, ncls, seed=5)
    model.eval()
    x, y = oracle.make_inputs(n, 1, sp, ncls, seed=77)
    alpha = torch.linspace(0.5, 1.5, ncls)
    lossname = "MutilCrossEntropyDiceLoss"
    lo, po, loss_o, go = _oracle(sd, x, y, lossname, alpha)
    logits, probs = model(x.cuda())
    loss = b200.MutilCrossEntropyDiceLoss(alpha.cuda())(logits, y.cuda())
    loss.backward()
    torch.cuda.synchronize()
    r = ((logits.double() - lo).norm() / lo.norm()).item()
    assert r < 1e-3, r
    assert torch.equal(logits.argmax(1), lo.argmax(1))
    assert abs(loss.item() - loss_o) < 1e-4 * max(1, abs(loss_o))
    errs = {nm: ((p.grad.double() - go[nm]).norm() / (go[nm].norm() + 1e-12)).item()
            for nm, p in model.named_parameters()}
    worst = max(errs, key=errs.get)
    assert float(np.median(list(errs.values()))) < 5e-3, float(np.median(list(errs.values())))
    assert errs[worst] < 2e-2, (worst, errs[worst])
    cos = min(F.cosine_similarity(p.grad.double().flatten(), go[nm].flatten(), dim=0).item()
              for nm, p in model.named_parameters())
    assert cos > 0.9998, cos
    # predict / sliding-window masks agree with the arg-max of these logits
    mask = b200.predict(model, x[0].numpy())
    assert np.array_equal(mask, logits[0].argmax(0).cpu().numpy().astype(np.uint8))
    with torch.no_grad():
        big = b200.predict_mask(model, x[:1].cuda())
    assert torch.equal(big[0].cpu(), logits[0].argmax(0).cpu().to(torch.uint8))
    # sliding windows of half the volume (rounded down to a multiple of 16) every quarter: 27 overlapping windows;
    # the union must equal the union of each window's own arg-max mask
    from pytorchdeeplearing_b200.inference import _starts
    patch = tuple(s_ // 2 // 16 * 16 for s_ in sp)
    step = tuple(p // 2 for p in patch)
    sw = b200.sliding_window_mask(model, x[0].numpy(), patch, step=step, batch=1)
    assert sw.shape == tuple(sp)
    want = torch.zeros(sp, dtype=torch.int32)
    origins = [(a, b, c) for a in _starts(sp[0], patch[0], step[0]) for b in _starts(sp[1], patch[1], step[1])
               for c in _starts(sp[2], patch[2], step[2])]
    assert len(origins) >= 27
    with torch.no_grad():
        for o in origins:
            win = tuple(slice(a, a + p) for a, p in zip(o, patch))
            lw, _ = model(x[:1, :, win[0], win[1], win[2]].cuda())
            want[win] += (lw[0].argmax(0) != 0).cpu().int()
    assert np.array_equal(sw, (want != 0).numpy().astype(np.uint8))


def test_bf16_error_budget():
    b200.set_precision("bf16")
    sd, model = _model(1, 2, seed=5)
    model.eval()
    x, y = oracle.make_inputs(2, 1, (96, 96, 96), 2, seed=77)
    lo, po, loss_o, go = _oracle(sd, x, y, "MutilDiceLoss", torch.ones(2))
    logits, _ = model(x.cuda())
    loss = b200.MutilDiceLoss(torch.ones(2).cuda())(logits, y.cuda())
    loss.backward()
    r = ((logits.double() - lo).norm() / lo.norm()).item()
    agree = (logits.argmax(1) == lo.argmax(1)).double().mean().item()
    assert r < 5e-2 and agree > 0.99, (r, agree)
    assert abs(loss.item() - loss_o) < 2e-2
    cos = [F.cosine_similarity(p.grad.double().flatten(), go[nm].flatten(), dim=0).item()
           for nm, p in model.named_parameters()]
    assert float(np.median(cos)) > 0.99 and min(cos) > 0.9, (float(np.median(cos)), min(cos))


@pytest.mark.parametrize("tag", ["c2_32", "c5_32x48x48", "c1_32", "c3_f8_32"])
def test_golden_fixtures_on_the_gpu(tag):
    """the reference's own eval and train-mode logits (train: the drop-in's one-launch Philox masks = torch's
    per-module bernoulli_ draws on the CUDA generator is checked separately; here the CPU draws are handed in)"""
    b200.set_precision("fp32")
    cin, ncls, f, shape, wseed = {"c2_32": (1, 2, 16, (2, 1, 32, 32, 32), 0),
                                  "c5_32x48x48": (1, 5, 16, (1, 1, 32, 48, 48), 1),
                                  "c1_32": (1, 1, 16, (1, 1, 32, 32, 32), 2),
                                  "c3_f8_32": (2, 3, 8, (1, 2, 32, 32, 32), 3)}[tag]
    sd, model = _model(cin, ncls, wseed, f)
    x, _ = oracle.make_inputs(shape[0], cin, shape[2:], ncls, seed=1234)
    model.eval()
    with torch.no_grad():
        logits, _ = model(x.cuda())
    ref = torch.from_numpy(GOLD[tag + ".logits"])
    sub = logits[:, :, ::2, ::2, ::2].cpu()
    assert ((sub - ref).norm() / ref.norm()).item() < 2e-5
    torch.manual_seed(int(GOLD[tag + ".train_seed"]))
    model.train()
    model.dropout_masks = othin.draw_dropout_masks_unetthin(shape[0], f)
    with torch.no_grad():
        lt, _ = model(x.cuda())
    model.dropout_masks = None
    ref = torch.from_numpy(GOLD[tag + ".train_logits"])
    assert ((lt[:, :, ::2, ::2, ::2].cpu() - ref).norm() / ref.norm()).item() < 2e-5


def test_dropout_masks_equal_torch_per_module_draws():
    b200.set_precision("fp32")
    sd, model = _model(1, 2, seed=1)
    x, _ = oracle.make_inputs(2, 1, (32, 32, 32), 2, seed=3)
    xc = x.cuda()
    model.train()
    torch.manual_seed(42)
    with torch.no_grad():
        got, _ = model(xc)                                   # one-launch Philox masks
    torch.manual_seed(42)
    model.dropout_masks = othin.draw_dropout_masks_unetthin(2, device="cuda")
    with torch.no_grad():
        want, _ = model(xc)
    model.dropout_masks = None
    assert torch.equal(got, want)


@pytest.mark.parametrize("train", [False, True])
def test_graphed_step_with_fused_adamw_equals_eager_steps(train):
    """three steps (the warm-up step of the constructor, then two replays) against three eager steps from the same
    weights; every step on both sides starts from the same generator seed, so train mode draws the same masks"""
    b200.set_precision("bf16")
    from pytorchdeeplearing_b200.graphed import GraphedStep
    x, y = oracle.make_inputs(1, 1, (64, 64, 64), 2, seed=4)
    x, y = x.cuda(), y.cuda()
    sd, m_graph = _model(1, 2, seed=6)
    _, m_eager = _model(1, 2, seed=6)
    m_graph.train(train)
    m_eager.train(train)
    lossfn = b200.MutilDiceLoss(torch.ones(2).cuda())
    opt_g = b200.FusedAdamW(m_graph.parameters(), lr=1e-3)
    opt_e = b200.FusedAdamW(m_eager.parameters(), lr=1e-3)
    torch.manual_seed(100)
    step = GraphedStep(m_graph, lossfn, x, y, warmup=1, optimizer=opt_g)     # the warm-up is step 1
    assert step.graph is not None
    losses_g = []
    for i in (1, 2):
        torch.manual_seed(100 + i)
        losses_g.append(float(step()))
    losses_e = []
    for i in range(3):
        torch.manual_seed(100 + i)
        opt_e.zero_grad()
        logits, _ = m_eager(x)
        loss = lossfn(logits, y)
        loss.backward()
        opt_e.step()
        losses_e.append(loss.item())
    torch.cuda.synchronize()
    assert np.allclose(losses_g, losses_e[1:], rtol=1e-4, atol=1e-5), (losses_g, losses_e)
    for (nm, pg), pe in zip(m_graph.named_parameters(), m_eager.parameters()):
        d = (pg.detach() - pe.detach()).abs().flatten()
        assert d.mean().item() < 3e-5, (nm, d.mean().item())


def test_reruns_are_bit_identical():
    """the forward (logits) is bit-identical; the weight gradients are sums whose split-K partials are accumulated
    atomically by the existing weight-gradient kernels, so they are held to fp32 rounding instead"""
    b200.set_precision("bf16")
    sd, model = _model(1, 2, seed=8)
    model.eval()
    x, y = oracle.make_inputs(1, 1, (64, 64, 64), 2, seed=5)
    lossfn = b200.MutilDiceLoss(torch.ones(2).cuda())
    outs = []
    for _ in range(2):
        for p in model.parameters():
            p.grad = None
        logits, _ = model(x.cuda())
        lossfn(logits, y.cuda()).backward()
        outs.append((logits.detach().clone(), [p.grad.clone() for p in model.parameters()]))
    assert torch.equal(outs[0][0], outs[1][0])
    for a, b in zip(outs[0][1], outs[1][1]):
        assert ((a - b).norm() / (b.norm() + 1e-30)).item() < 1e-5
