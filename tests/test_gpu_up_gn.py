"""The fused first layer of up_tr32 (csrc/up_gn.cu) against the per-layer calls it replaces, on the same tensors:

  conv UP (pointwise mma.sync, statistics in the epilogue) -> apply_gn into the concat's left half        forward
  gn_bwd_reduce_gn -> gn_bwd_apply_gn -> wgrad (DOWN kind) + the DOWN-kind data-gradient conv            backward

The fused kernels recompute y from the coarse input with the pointwise kernel's own fragments and mma chain, so given
the same statistics the forward activation is bit-identical, and given the same backward sums so is every dy they
form on chip.  What may differ is summation order: the fp64 atomics of the statistics and sums across CTAs, the fp32
lane partials of the backward sums, the fp32 accumulation order of the data gradient (the unfused kernel runs on
wgmma) and the fp32 atomics of the weight and GroupNorm-parameter gradients.  Each comparison states its bound.
Outputs live inside larger allocations whose guard bands (and the other half of the pitched concat buffer) hold a
NaN pattern that must survive."""
import pytest
import torch

from emu_backend import UP, DOWN

pytestmark = pytest.mark.gpu

DEV = "cuda"
GUARD = 256
NAN16 = 0x7FC1


def _be():
    from pytorchdeeplearing_b200 import runtime
    return runtime.cuda_backend()


def _guarded(shape, ld, off=0):
    """(N,D,H,W,C) bf16 view with channel pitch ``ld`` starting ``off`` channels into a NaN-filled allocation"""
    n, d, h, w, c = shape
    buf = torch.empty(2 * GUARD + n * d * h * w * ld, dtype=torch.bfloat16, device=DEV)
    buf.view(torch.int16).fill_(NAN16)
    return buf, buf.as_strided(shape, (d * h * w * ld, h * w * ld, w * ld, ld, 1), GUARD + off)


def _view_mask(buf, v):
    m = torch.zeros(buf.numel(), dtype=torch.bool, device=DEV)
    n, d, h, w, c = v.shape
    st = v.stride()
    lin = (torch.arange(n, device=DEV).view(-1, 1, 1, 1, 1) * st[0] + torch.arange(d, device=DEV).view(1, -1, 1, 1, 1) * st[1]
           + torch.arange(h, device=DEV).view(1, 1, -1, 1, 1) * st[2] + torch.arange(w, device=DEV).view(1, 1, 1, -1, 1) * st[3]
           + torch.arange(c, device=DEV).view(1, 1, 1, 1, -1))
    m[(v.data_ptr() - buf.data_ptr()) // buf.element_size() + lin.reshape(-1)] = True
    return m


def _untouched(buf, v):
    return bool((buf.view(torch.int16)[~_view_mask(buf, v)] == NAN16).all())


def _case(n, sp, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    r = lambda *s, sc=1.0: (torch.randn(*s, generator=g) * sc).to(DEV)
    x = r(n, *sp, 32).to(torch.bfloat16)
    w = r(32, 16, 2, 2, 2, sc=0.1)                       # ConvTranspose3d(32, 16, 2, 2): (Cin, Cout, 2, 2, 2)
    bias = r(16, sc=0.1)
    gamma, beta = r(16, sc=0.2) + 1.0, r(16, sc=0.1)
    scale = ((torch.rand(n, 16, generator=g) > 0.2).float() * 1.25).to(DEV)
    fine = tuple(2 * s for s in sp)
    gcat = r(n, *fine, 32).to(torch.bfloat16)            # the concat's gradient; the layer reads its left half
    return x, w, bias, gamma, beta, scale, gcat


def _operands(be, x, w):
    sp = tuple(x.shape[1:4])
    fvox, cvox = 8 * sp[0] * sp[1] * sp[2], sp[0] * sp[1] * sp[2]
    return (be.pack_weight(w, UP, "fwd", torch.bfloat16, 3, vox=fvox),
            be.pack_weight(w, UP, "dgrad", torch.bfloat16, 3, vox=cvox))


SHAPES = [(2, (48, 48, 48)), (2, (9, 16, 32))]


@pytest.mark.parametrize("n,sp", SHAPES)
def test_up_gn_matches_per_layer_calls(n, sp):
    be = _be()
    x, w, bias, gamma, beta, scale, gcat = _case(n, sp, seed=sum(sp) + n)
    wf, wd = _operands(be, x, w)
    assert be.up_gn_ok(x, wf, 16, 3)
    fine = tuple(2 * s for s in sp)
    fvox = fine[0] * fine[1] * fine[2]
    y = torch.empty((n,) + fine + (16,), dtype=torch.bfloat16, device=DEV)
    assert be.conv_path(UP, 3, x, wf, y) == "PW_MMA"
    st_old = torch.zeros((n, 16, 2), dtype=torch.float64, device=DEV)
    be.conv(UP, 3, x, wf, bias, y, st_old, None)
    gn = (st_old, gamma, beta, scale, fvox, 8, 1e-5)

    # statistics: the same per-CTA partials as the pointwise epilogue; only the order of the fp64 atomics differs
    st_new = torch.zeros_like(st_old)
    be.up_gn_stats(x, wf, bias, st_new)
    torch.testing.assert_close(st_new, st_old, rtol=1e-12, atol=1e-9)

    # forward activation into the left half of a pitched concat buffer: bit-identical, right half and guards untouched
    shape = (n,) + fine + (16,)
    _, out_old = _guarded(shape, 32)
    buf_n, out_new = _guarded(shape, 32)
    be.apply_gn(y, gn, None, None, None, out_old)
    be.up_gn_apply(x, wf, bias, gn, out_new)
    torch.cuda.synchronize()
    assert torch.equal(out_new.contiguous().view(torch.int16), out_old.contiguous().view(torch.int16))
    assert _untouched(buf_n, out_new)

    # backward sums over the concat gradient's left half
    grad = gcat[..., :16]
    old_sums = torch.zeros((n, 16, 3), dtype=torch.float64, device=DEV)
    be.gn_bwd_reduce_gn(grad, y, gn, old_sums)
    new_sums = torch.zeros_like(old_sums)
    be.up_gn_bwd_sums(x, wf, bias, gn, grad, new_sums)
    # bound: fp32 partials of at most a few hundred terms each, then fp64 -> 1e-5 of the sum of |terms|
    gf, yf = grad.double(), y.double()
    mag = torch.stack([gf.abs().sum((1, 2, 3)), (gf * yf).abs().sum((1, 2, 3)), yf.abs().sum((1, 2, 3))], -1)
    assert ((new_sums - old_sums).abs() <= 1e-5 * mag + 1e-6).all(), (new_sums - old_sums).abs().max()

    # gradients, from the SAME sums (so every dy is the same bf16 value)
    z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=DEV)
    o_dw, o_dg, o_db, o_dbias = z(8, 16, 32), z(16), z(16), z(16)
    dy = torch.empty_like(y)
    be.gn_bwd_apply_gn(grad, y, gn, old_sums, dy, o_dg, o_db, o_dbias)
    be.wgrad(DOWN, 3, dy, x, o_dw)
    o_dx = torch.empty_like(x)
    be.conv(DOWN, 3, dy, wd, None, o_dx, None, None)
    n_dw, n_dg, n_db, n_dbias = z(8, 16, 32), z(16), z(16), z(16)
    buf_x, n_dx = _guarded(tuple(x.shape), 32)
    be.up_gn_bwd(x, wf, bias, gn, grad, old_sums, n_dw, n_dx, n_dg, n_db, n_dbias)
    torch.cuda.synchronize()
    assert _untouched(buf_x, n_dx)
    # dx: fp32 sums of the same 128 bf16 products per value in another order, then one bf16 rounding -> at most one
    # bf16 ulp (2^-7 relative) apart, plus 1e-4 of the largest value for cancellation
    dn, do = n_dx.float(), o_dx.float()
    assert ((dn - do).abs() <= 2.0 ** -7 * do.abs() + 1e-4 * do.abs().max()).all(), (dn - do).abs().max()
    # dW: fp32 sums of the same bf16 products in another grouping -> 1e-5 of sum |dy| * max |x| per channel
    bound = 1e-5 * dy.double().abs().sum((0, 1, 2, 3)) * x.abs().max().item() + 1e-6
    assert ((n_dw - o_dw).double().abs() <= bound.view(1, 16, 1)).all(), (n_dw - o_dw).abs().max()
    # d gamma, d beta, d bias: the same fp64 expressions of the same sums, then fp32 atomics in another order
    for new, old in ((n_dg, o_dg), (n_db, o_db), (n_dbias, o_dbias)):
        torch.testing.assert_close(new, old, rtol=1e-5, atol=1e-5 * old.abs().max().item() + 1e-7)

    # the data gradient has no atomics: a second run gives the same bits
    dx2 = torch.empty_like(x)
    be.up_gn_bwd(x, wf, bias, gn, grad, old_sums, z(8, 16, 32), dx2, z(16), z(16), z(16))
    torch.cuda.synchronize()
    assert torch.equal(dx2.view(torch.int16), n_dx.contiguous().view(torch.int16))


def test_up_gn_graph_replay_equals_eager():
    be = _be()
    n, sp = 2, (9, 16, 32)
    x, w, bias, gamma, beta, scale, gcat = _case(n, sp, seed=11)
    wf, _ = _operands(be, x, w)
    fine = tuple(2 * s for s in sp)
    fvox = fine[0] * fine[1] * fine[2]
    st = torch.zeros((n, 16, 2), dtype=torch.float64, device=DEV)
    sums = torch.zeros((n, 16, 3), dtype=torch.float64, device=DEV)
    out = torch.empty((n,) + fine + (32,), dtype=torch.bfloat16, device=DEV)
    dx = torch.empty_like(x)
    grads = [torch.zeros(s, dtype=torch.float32, device=DEV) for s in ((8, 16, 32), 16, 16, 16)]
    gn = (st, gamma, beta, scale, fvox, 8, 1e-5)

    def step():
        for t in [st, sums] + grads:
            t.zero_()
        be.up_gn_stats(x, wf, bias, st)
        be.up_gn_apply(x, wf, bias, gn, out[..., :16])
        be.up_gn_bwd_sums(x, wf, bias, gn, gcat[..., :16], sums)
        be.up_gn_bwd(x, wf, bias, gn, gcat[..., :16], sums, grads[0], dx, *grads[1:])

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    eager = [t.clone() for t in [out[..., :16], dx, st, sums] + grads]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    graph.replay()
    torch.cuda.synchronize()
    replay = [out[..., :16], dx, st, sums] + grads
    # the activation and dx depend on the statistics / sums only through fp32 coefficients of fp64 sums whose atomics
    # may land in another order: equal bits, or within bf16 rounding
    for a, b in zip(replay[:2], eager[:2]):
        assert torch.equal(a.contiguous().view(torch.int16), b.view(torch.int16)) or \
            torch.allclose(a.float(), b.float(), rtol=1e-2, atol=1e-2)
    for a, b in zip(replay[2:], eager[2:]):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-5 * b.abs().max().item() + 1e-9)


class _WithoutUpGn:
    """the CUDA backend minus the fused up_tr32 layer: the engine takes the per-layer calls"""

    def __init__(self, inner):
        self.inner = inner

    def __getattr__(self, name):
        if name.startswith("up_gn"):
            raise AttributeError(name)
        return getattr(self.inner, name)


class _Counting:
    def __init__(self, inner):
        self.inner = inner
        self.fused_calls = 0

    def __getattr__(self, name):
        fn = getattr(self.inner, name)
        if name in ("up_gn_stats", "up_gn_apply", "up_gn_bwd_sums", "up_gn_bwd"):
            def wrapped(*a, **k):
                self.fused_calls += 1
                return fn(*a, **k)
            return wrapped
        return fn


def test_graphed_vnet_step_fused_vs_per_layer():
    import pytorchdeeplearing_b200 as b200
    from pytorchdeeplearing_b200 import runtime
    from pytorchdeeplearing_b200.graphed import GraphedStep
    import oracle

    b200.set_precision("bf16")
    x, y = oracle.make_inputs(2, 1, (64, 64, 64), 2, seed=3)
    x, y = x.to(DEV), y.to(DEV)

    def run(backend):
        runtime._set_backend_for_testing(backend)
        try:
            torch.manual_seed(0)
            m = b200.VNet3d(1, 2)
            m.apply(b200.initialize_weights)
            m = m.to(DEV).train()
            lossfn = b200.MutilDiceLoss(torch.ones(2, device=DEV))
            torch.manual_seed(100)
            step = GraphedStep(m, lossfn, x, y, warmup=1)
            loss = float(step())
            torch.cuda.synchronize()
            norms = torch.stack([p.grad.double().norm() for p in m.parameters()])
            return loss, float(step.dice), norms, m
        finally:
            runtime._set_backend_for_testing(None)

    be = runtime.cuda_backend()
    fused = _Counting(be)
    l_new, d_new, n_new, m = run(fused)
    assert fused.fused_calls > 0
    l_old, d_old, n_old, _ = run(_WithoutUpGn(be))
    assert abs(l_new - l_old) <= 1e-3 * max(1.0, abs(l_old)), (l_new, l_old)
    assert abs(d_new - d_old) <= 1e-3, (d_new, d_old)
    names = [k for k, _ in m.named_parameters()]
    rel = ((n_new - n_old).abs() / n_old.clamp_min(1e-12)).tolist()
    bad = [(k, r) for k, r in zip(names, rel) if r > 5e-2]
    assert not bad, bad
