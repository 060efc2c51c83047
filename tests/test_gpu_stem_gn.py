"""The fused input block (csrc/stem_gn.cu) against the per-branch calls it replaces, on the same tensors:

  stem conv (K3 and K1, statistics in the epilogue) -> apply_gn(y_a, y_b)                       forward
  gn_bwd_reduce_gn -> gn_bwd_apply_gn -> wgrad, per branch                                    backward

The fused kernels recompute y_a, y_b from the image with the stem's own instruction sequence, so given the same
statistics the forward activation is bit-identical, and given the same backward sums so is every dy they form on
chip.  What may differ is summation order: the fp64 atomics of the statistics and sums across CTAs, the fp32 lane
partials of the backward sums (grouped by tile instead of by grid stride), and the fp32 atomics of the weight and
GroupNorm-parameter gradients (the backward kernel runs one CTA per SM, the stem weight gradient two).  Each
comparison states its bound.  Outputs live inside larger allocations whose guard bands (and the other half of the
pitched skip buffer) hold a NaN pattern that must survive."""
import pytest
import torch

from emu_backend import K3, K1

pytestmark = pytest.mark.gpu

DEV = "cuda"
GUARD = 256
NAN16 = 0x7FC1


def _be():
    from pytorchdeeplearing_b200 import runtime
    return runtime.cuda_backend()


def _guarded(shape, ld, dtype=torch.bfloat16, off=0):
    """(N,D,H,W,C) view with channel pitch ``ld`` starting ``off`` channels into a NaN-filled allocation with guards"""
    n, d, h, w, c = shape
    vox = n * d * h * w
    buf = torch.empty(2 * GUARD + vox * ld, dtype=dtype, device=DEV)
    buf.view(torch.int16).fill_(NAN16)
    return buf, buf.as_strided(shape, (d * h * w * ld, h * w * ld, w * ld, ld, 1), GUARD + off)


def _untouched(buf, view_mask):
    """every element of ``buf`` outside the view still holds the sentinel"""
    bits = buf.view(torch.int16)
    return bool((bits[~view_mask] == NAN16).all())


def _view_mask(buf, v):
    m = torch.zeros(buf.numel(), dtype=torch.bool, device=DEV)
    base = v.data_ptr() - buf.data_ptr()
    n, d, h, w, c = v.shape
    st = v.stride()
    lin = (torch.arange(n, device=DEV).view(-1, 1, 1, 1, 1) * st[0] + torch.arange(d, device=DEV).view(1, -1, 1, 1, 1) * st[1]
           + torch.arange(h, device=DEV).view(1, 1, -1, 1, 1) * st[2] + torch.arange(w, device=DEV).view(1, 1, 1, -1, 1) * st[3]
           + torch.arange(c, device=DEV).view(1, 1, 1, 1, -1))
    m[base // buf.element_size() + lin.reshape(-1)] = True
    return m


def _case(n, sp, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    r = lambda *s, sc=1.0: (torch.randn(*s, generator=g) * sc).to(DEV)
    x = r(n, *sp, 1, sc=2.0)
    w3, w1 = r(16, 1, 3, 3, 3, sc=0.3), r(16, 1, 1, 1, 1, sc=0.5)
    b3, b1 = r(16, sc=0.1), r(16, sc=0.1)
    gamma, beta = r(16, sc=0.2) + 1.0, r(16, sc=0.1)
    keep = lambda: ((torch.rand(n, 16, generator=g) > 0.2).float() * 1.25).to(DEV)
    grad = r(n, *sp, 16).to(torch.bfloat16)
    return x, w3, w1, b3, b1, gamma, beta, keep(), keep(), grad


def _old_forward(be, x, p3, p1, b3, b1, gamma, beta, s3, s1):
    n, sp = x.shape[0], tuple(x.shape[1:4])
    vox = sp[0] * sp[1] * sp[2]
    ya = torch.empty((n,) + sp + (16,), dtype=torch.bfloat16, device=DEV)
    yb = torch.empty_like(ya)
    st3 = torch.zeros((n, 16, 2), dtype=torch.float64, device=DEV)
    st1 = torch.zeros_like(st3)
    be.conv(K3, 3, x, p3, b3, ya, st3, None)
    be.conv(K1, 3, x, p1, b1, yb, st1, None)
    gn3 = (st3, gamma, beta, s3, vox, 8, 1e-5)
    gn1 = (st1, gamma, beta, s1, vox, 8, 1e-5)
    return ya, yb, gn3, gn1


SHAPES = [(2, (96, 96, 96)), (3, (7, 24, 48)), (1, (3, 8, 16)), (2, (5, 16, 112))]


@pytest.mark.parametrize("n,sp", SHAPES)
def test_stem_gn_matches_per_branch_calls(n, sp):
    be = _be()
    x, w3, w1, b3, b1, gamma, beta, s3, s1, grad = _case(n, sp, seed=sum(sp) + n)
    assert be.stem_gn_ok(x, 16, 3)
    vox = sp[0] * sp[1] * sp[2]
    p3 = be.pack_weight(w3, K3, "fwd", torch.bfloat16, 3, vox=vox)
    p1 = be.pack_weight(w1, K1, "fwd", torch.bfloat16, 3, vox=vox)
    ya, yb, gn3, gn1 = _old_forward(be, x, p3, p1, b3, b1, gamma, beta, s3, s1)

    # statistics: the same per-CTA partials as the stem epilogue; only the order of the fp64 atomics differs
    st3 = torch.zeros((n, 16, 2), dtype=torch.float64, device=DEV)
    st1 = torch.zeros_like(st3)
    be.stem_gn_stats(x, p3, b3, p1, b1, st3, st1)
    for new, old in ((st3, gn3[0]), (st1, gn1[0])):
        torch.testing.assert_close(new, old, rtol=1e-12, atol=1e-9)

    # forward activation into the right half of a pitched skip buffer: bit-identical, left half and guards untouched
    shape = (n,) + sp + (16,)
    buf_o, out_old = _guarded(shape, 32, off=16)
    buf_n, out_new = _guarded(shape, 32, off=16)
    be.apply_gn(ya, gn3, yb, gn1, None, out_old)
    be.stem_gn_apply(x, p3, b3, p1, b1, gn3, gn1, out_new)
    torch.cuda.synchronize()
    assert torch.equal(out_new.contiguous().view(torch.int16), out_old.contiguous().view(torch.int16))
    assert _untouched(buf_n, _view_mask(buf_n, out_new))

    # backward sums of both branches (old: one reduce per branch over g and the stored y)
    old_sums = []
    for y, gn in ((ya, gn3), (yb, gn1)):
        s = torch.zeros((n, 16, 3), dtype=torch.float64, device=DEV)
        be.gn_bwd_reduce_gn(grad, y, gn, s)
        old_sums.append(s)
    new_sums = [torch.zeros((n, 16, 3), dtype=torch.float64, device=DEV) for _ in range(2)]
    be.stem_gn_bwd_sums(x, p3, b3, p1, b1, gn3, gn1, grad, new_sums[0], new_sums[1])
    # bound: fp32 partials of at most a few hundred terms each, then fp64 -> 1e-5 of the sum of |terms|
    gf = grad.double()
    for y, new, old in ((ya, new_sums[0], old_sums[0]), (yb, new_sums[1], old_sums[1])):
        yf = y.double()
        mag = torch.stack([gf.abs().sum((1, 2, 3)), (gf * yf).abs().sum((1, 2, 3)), yf.abs().sum((1, 2, 3))], -1)
        assert ((new - old).abs() <= 1e-5 * mag + 1e-6).all(), (new - old).abs().max()

    # weight and GroupNorm-parameter gradients, from the SAME sums (so every dy is the same bf16 value)
    z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=DEV)
    o_dw3, o_dw1, o_dg, o_db, o_db3, o_db1 = z(27, 1, 16), z(1, 1, 16), z(16), z(16), z(16), z(16)
    dys = []
    for y, gn, s, dw, dbias, kind in ((ya, gn3, old_sums[0], o_dw3, o_db3, K3), (yb, gn1, old_sums[1], o_dw1, o_db1, K1)):
        dy = torch.empty_like(y)
        be.gn_bwd_apply_gn(grad, y, gn, s, dy, o_dg, o_db, dbias)
        be.wgrad(kind, 3, x, dy, dw)
        dys.append(dy)
    n_dw3, n_dw1, n_dg, n_db, n_db3, n_db1 = z(27, 1, 16), z(1, 1, 16), z(16), z(16), z(16), z(16)
    be.stem_gn_bwd(x, p3, b3, p1, b1, gn3, gn1, grad, old_sums[0], old_sums[1], n_dw3, n_dw1, n_dg, n_db, n_db3, n_db1)
    torch.cuda.synchronize()
    # dW: fp32 sums of the same bf16 products in another grouping -> 1e-5 of sum |dy| * max |x| per channel
    xmax = x.abs().max().item()
    for new, old, dy in ((n_dw3, o_dw3, dys[0]), (n_dw1, o_dw1, dys[1])):
        bound = 1e-5 * dy.double().abs().sum((0, 1, 2, 3)) * xmax + 1e-6
        assert ((new - old).double().abs() <= bound.view(1, 1, 16)).all(), (new - old).abs().max()
    # d gamma, d beta, d bias: the same fp64 expressions of the same sums, then fp32 atomics in another order
    for new, old in ((n_dg, o_dg), (n_db, o_db), (n_db3, o_db3), (n_db1, o_db1)):
        torch.testing.assert_close(new, old, rtol=1e-5, atol=1e-5 * old.abs().max().item() + 1e-7)


def test_stem_gn_graph_replay_equals_eager():
    be = _be()
    n, sp = 2, (16, 32, 64)
    x, w3, w1, b3, b1, gamma, beta, s3, s1, grad = _case(n, sp, seed=7)
    vox = sp[0] * sp[1] * sp[2]
    p3 = be.pack_weight(w3, K3, "fwd", torch.bfloat16, 3, vox=vox)
    p1 = be.pack_weight(w1, K1, "fwd", torch.bfloat16, 3, vox=vox)
    st = [torch.zeros((n, 16, 2), dtype=torch.float64, device=DEV) for _ in range(2)]
    sums = [torch.zeros((n, 16, 3), dtype=torch.float64, device=DEV) for _ in range(2)]
    out = torch.empty((n,) + sp + (16,), dtype=torch.bfloat16, device=DEV)
    grads = [torch.zeros(s, dtype=torch.float32, device=DEV) for s in ((27, 1, 16), (1, 1, 16), 16, 16, 16, 16)]
    gn = lambda i, s: (st[i], gamma, beta, s, vox, 8, 1e-5)

    def step():
        for t in st + sums + grads:
            t.zero_()
        be.stem_gn_stats(x, p3, b3, p1, b1, st[0], st[1])
        be.stem_gn_apply(x, p3, b3, p1, b1, gn(0, s3), gn(1, s1), out)
        be.stem_gn_bwd_sums(x, p3, b3, p1, b1, gn(0, s3), gn(1, s1), grad, sums[0], sums[1])
        be.stem_gn_bwd(x, p3, b3, p1, b1, gn(0, s3), gn(1, s1), grad, sums[0], sums[1], *grads)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    eager = [t.clone() for t in [out] + st + sums + grads]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    graph.replay()
    torch.cuda.synchronize()
    replay = [out] + st + sums + grads
    assert torch.equal(replay[0].view(torch.int16), eager[0].view(torch.int16)) or \
        torch.allclose(replay[0].float(), eager[0].float(), rtol=1e-2, atol=1e-2)
    for a, b in zip(replay[1:], eager[1:]):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-5 * b.abs().max().item() + 1e-9)


class _WithoutStemGn:
    """the CUDA backend minus the fused input block: the engine takes the per-branch calls"""

    def __init__(self, inner):
        self.inner = inner

    def __getattr__(self, name):
        if name.startswith("stem_gn"):
            raise AttributeError(name)
        return getattr(self.inner, name)


@pytest.mark.parametrize("arch", ["vnet3d", "resnet3d"])
def test_graphed_step_fused_vs_per_branch(arch):
    import pytorchdeeplearing_b200 as b200
    from pytorchdeeplearing_b200 import runtime
    from pytorchdeeplearing_b200.graphed import GraphedStep
    import oracle

    b200.set_precision("bf16")
    sp = (64, 64, 64) if arch == "vnet3d" else (32, 32, 32)
    x, y = oracle.make_inputs(2, 1, sp, 2, seed=3)
    x, y = x.to(DEV), y.to(DEV)
    if arch == "resnet3d":
        y = torch.tensor([0, 1], device=DEV)

    def run(backend):
        runtime._set_backend_for_testing(backend)
        try:
            torch.manual_seed(0)
            m = (b200.VNet3d(1, 2) if arch == "vnet3d" else b200.ResNet3d(1, 2))
            m.apply(b200.initialize_weights)
            m = m.to(DEV).train()
            lossfn = (b200.MutilDiceLoss if arch == "vnet3d" else b200.MutilCrossEntropyLoss)(torch.ones(2, device=DEV))
            torch.manual_seed(100)
            step = GraphedStep(m, lossfn, x, y, warmup=1)
            loss = float(step())
            torch.cuda.synchronize()
            norms = torch.stack([p.grad.double().norm() for p in m.parameters()])
            dice = float(step.dice) if getattr(step, "dice", None) is not None else None
            return loss, dice, norms, m
        finally:
            runtime._set_backend_for_testing(None)

    be = runtime.cuda_backend()
    l_new, d_new, n_new, m = run(be)
    l_old, d_old, n_old, _ = run(_WithoutStemGn(be))
    assert abs(l_new - l_old) <= 1e-3 * max(1.0, abs(l_old)), (l_new, l_old)
    if d_old is not None:
        assert abs(d_new - d_old) <= 1e-3, (d_new, d_old)
    names = [k for k, _ in m.named_parameters()]
    rel = ((n_new - n_old).abs() / n_old.clamp_min(1e-12)).tolist()
    bad = [(k, r) for k, r in zip(names, rel) if r > 5e-2]
    assert not bad, bad
