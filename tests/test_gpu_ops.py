"""Per-entry-point parity of the sm_90a kernels (through the C ABI) against the test-only
PyTorch statement of the same op (tests/emu_backend.py, CPU fp32/fp64).  `-m gpu`."""
import pytest
import torch

from emu_backend import EmuBackend, K3, K1, DOWN, UP

pytestmark = pytest.mark.gpu

EMU = EmuBackend()


@pytest.fixture(scope="module")
def be():
    from pytorchdeeplearing_b200._abi import CudaBackend
    return CudaBackend()


def dev(t):
    return None if t is None else t.cuda()


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def tol(dtype, k=1.0):
    return (3e-5 if dtype == torch.float32 else 1.2e-2) * k


def rnd(shape, dtype, g, scale=1.0):
    return (torch.randn(shape, generator=g) * scale).to(dtype)


def stem_mma_shape(dtype, cin, sp):
    """the bf16 stem kernels convert the fp32 image to bf16: feed them bf16-representable inputs"""
    return dtype == torch.bfloat16 and cin == 1 and sp[2] % 16 == 0 and sp[1] % 8 == 0


def sliced(n, sp, c, dtype, g, pad):
    """activation view with channel pitch > C when pad"""
    if pad:
        full = rnd((n,) + sp + (c + pad,), dtype, g)
        return full[..., pad // 2: pad // 2 + c]
    return rnd((n,) + sp + (c,), dtype, g)


CONV_CASES = [
    # kind, dims, n, in-spatial, cin, cout
    (K3, 3, 2, (6, 10, 12), 16, 16),
    (K3, 3, 1, (5, 7, 9), 32, 32),
    (K3, 3, 1, (4, 6, 8), 1, 16),
    (K3, 3, 1, (3, 5, 7), 1, 16),            # odd width: one voxel per thread
    (K3, 3, 2, (20, 24, 28), 1, 16),         # > one grid stride of voxels: coordinate carries in the stem wgrad
    (K3, 3, 1, (4, 6, 8), 1, 32),
    (K3, 3, 2, (6, 16, 32), 1, 16),          # bf16: mma.sync stem (W % 16 == 0, H % 8 == 0)
    (K3, 3, 1, (3, 8, 96), 1, 32),
    (K3, 2, 2, (1, 24, 48), 1, 32),
    (K3, 2, 1, (1, 16, 256), 1, 16),         # two tiles along w
    (K1, 3, 1, (4, 8, 16), 1, 16),
    (K3, 2, 3, (1, 40, 56), 1, 32),
    (K3, 3, 1, (4, 6, 8), 3, 16),
    (K3, 3, 1, (4, 4, 8), 64, 48),
    (K3, 2, 2, (1, 12, 20), 16, 32),
    (K3, 2, 1, (1, 16, 16), 1, 16),
    (K1, 3, 2, (4, 6, 8), 32, 16),
    (K1, 3, 1, (4, 6, 8), 16, 2),
    (K1, 3, 1, (4, 6, 8), 16, 5),
    (K1, 3, 1, (4, 6, 8), 1, 16),
    (K1, 2, 2, (1, 8, 8), 16, 1),
    (DOWN, 3, 2, (4, 8, 12), 16, 32),
    (DOWN, 3, 1, (2, 2, 2), 128, 256),
    (DOWN, 2, 1, (1, 8, 12), 16, 32),
    (UP, 3, 2, (2, 4, 6), 32, 16),
    (UP, 3, 1, (1, 1, 1), 256, 128),
    (UP, 2, 2, (1, 4, 6), 32, 16),
]


def out_spatial(kind, dims, sp):
    if kind == DOWN:
        return (sp[0] // 2 if dims == 3 else 1, sp[1] // 2, sp[2] // 2)
    if kind == UP:
        return (sp[0] * 2 if dims == 3 else 1, sp[1] * 2, sp[2] * 2)
    return sp


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind,dims,n,sp,cin,cout", CONV_CASES)
def test_conv_forward(be, dtype, kind, dims, n, sp, cin, cout):
    g = torch.Generator().manual_seed(1)
    k = {K3: 3, K1: 1, DOWN: 2, UP: 2}[kind]
    kk = (k,) * dims
    wshape = ((cin, cout) if kind == UP else (cout, cin)) + kk
    w = torch.randn(wshape, generator=g) * (2.0 / (cin * k ** dims)) ** 0.5
    bias = torch.randn(cout, generator=g) * 0.1
    # network-input style x: fp32 even in bf16 mode when cin is not a channel multiple
    xdt = torch.float32 if cin < 16 else dtype
    x = sliced(n, sp, cin, xdt, g, pad=16 if cin >= 16 else 0)
    if stem_mma_shape(dtype, cin, sp):
        x = x.bfloat16().float()
    osp = out_spatial(kind, dims, sp)
    ydt = torch.float32 if cout < 16 else dtype
    for with_stats, with_addend in ((True, False), (False, True)):
        wp_e = EMU.pack_weight(w, kind, "fwd", dtype, dims)
        wp_c = be.pack_weight(w.cuda(), kind, "fwd", dtype, dims, allow_tc=False)
        assert torch.equal(wp_c.t.cpu().float(), wp_e.float())
        y_e = torch.zeros((n,) + osp + (cout,), dtype=ydt)
        ybuf = torch.zeros((n,) + osp + (cout + 16,), dtype=ydt, device="cuda")
        y_c = ybuf[..., 8:8 + cout]
        st_e = torch.zeros(n, cout, 2, dtype=torch.float64) if with_stats else None
        st_c = dev(st_e.clone()) if with_stats else None
        add = rnd((n,) + osp + (cout,), ydt, g) if with_addend else None
        EMU.conv(kind, dims, x, wp_e, bias, y_e, st_e, add)
        be.conv(kind, dims, x.cuda(), wp_c, bias.cuda(), y_c, st_c, dev(add))
        torch.cuda.synchronize()
        assert rel(y_c, y_e) < tol(dtype)
        assert float(ybuf[..., :8].abs().max()) == 0 and float(ybuf[..., 8 + cout:].abs().max()) == 0
        if with_stats:
            assert rel(st_c, st_e) < 1e-5


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind,dims,n,sp,cin,cout", CONV_CASES)
def test_conv_dgrad_and_wgrad(be, dtype, kind, dims, n, sp, cin, cout):
    """dgrad through b200seg_conv with dgrad-packed weights; wgrad through b200seg_wgrad+unpack;
    both against autograd of the emulated forward."""
    g = torch.Generator().manual_seed(2)
    k = {K3: 3, K1: 1, DOWN: 2, UP: 2}[kind]
    kk = (k,) * dims
    wshape = ((cin, cout) if kind == UP else (cout, cin)) + kk
    w = (torch.randn(wshape, generator=g) * (2.0 / (cin * k ** dims)) ** 0.5)
    osp = out_spatial(kind, dims, sp)
    xdt = torch.float32 if cin < 16 else dtype
    gdt = torch.float32 if cout < 16 else dtype
    x = rnd((n,) + sp + (cin,), xdt, g)
    if stem_mma_shape(dtype, cin, sp):
        x = x.bfloat16().float()
    dy = rnd((n,) + osp + (cout,), gdt, g)
    # reference via autograd in fp64 on the (rounded) operands
    import torch.nn.functional as F
    xr = x.double().permute(0, 4, 1, 2, 3).requires_grad_(True)
    wq = w.to(dtype).double() if kind != UP else w.to(dtype).double()
    wr = wq.clone().requires_grad_(True)
    w5 = wr if dims == 3 else wr.unsqueeze(2)
    if kind == K3:
        o = F.conv3d(xr, w5, None, padding=(1 if dims == 3 else 0, 1, 1))
    elif kind == K1:
        o = F.conv3d(xr, w5, None)
    elif kind == DOWN:
        o = F.conv3d(xr, w5, None, stride=(2 if dims == 3 else 1, 2, 2))
    else:
        o = F.conv_transpose3d(xr, w5, None, stride=(2 if dims == 3 else 1, 2, 2))
    o.backward(dy.double().permute(0, 4, 1, 2, 3))
    dx_ref = xr.grad.permute(0, 2, 3, 4, 1)
    # --- dgrad
    DK = {K3: K3, K1: K1, DOWN: UP, UP: DOWN}[kind]
    wd = be.pack_weight(w.cuda(), kind, "dgrad", dtype, dims, allow_tc=False)
    assert torch.equal(wd.t.cpu().float(), EMU.pack_weight(w, kind, "dgrad", dtype, dims).float())
    if cin >= 16:
        dx = torch.zeros((n,) + sp + (cin,), dtype=dtype, device="cuda")
        be.conv(DK, dims, dy.cuda(), wd, None, dx, None, None)
        torch.cuda.synchronize()
        assert rel(dx, dx_ref) < tol(dtype)
    # --- wgrad
    taps = k ** dims
    if kind == UP:
        dwp = torch.zeros((taps, cout, cin), dtype=torch.float32, device="cuda")
        be.wgrad(DOWN, dims, dy.cuda(), x.cuda(), dwp)
    else:
        dwp = torch.zeros((taps, cin, cout), dtype=torch.float32, device="cuda")
        be.wgrad(kind, dims, x.cuda(), dy.cuda(), dwp)
    gw = torch.zeros(wshape, dtype=torch.float32, device="cuda")
    be.unpack_wgrad(dwp, gw, kind, dims)
    torch.cuda.synchronize()
    assert rel(gw, wr.grad) < 3e-5


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n,sp,c,masked", [(2, (4, 6, 8), 16, True), (1, (3, 5, 7), 32, False),
                                           (2, (1, 8, 8), 64, True), (1, (2, 2, 2), 256, True)])
def test_groupnorm_chain(be, dtype, n, sp, c, masked):
    g = torch.Generator().manual_seed(3)
    y = sliced(n, sp, c, dtype, g, pad=16)
    y2 = rnd((n,) + sp + (c,), dtype, g)
    res = rnd((n,) + sp + (c,), dtype, g)
    gamma = 1 + 0.2 * torch.randn(c, generator=g)
    beta = 0.2 * torch.randn(c, generator=g)
    scale = (torch.rand(n, c, generator=g) > 0.2).float() / 0.8 if masked else None
    vox = sp[0] * sp[1] * sp[2]
    yf = y.double()
    stats = torch.stack([yf.sum((1, 2, 3)), (yf * yf).sum((1, 2, 3))], -1)
    coef_e, mr_e = torch.empty(n, c, 2), torch.empty(n, 8, 2)
    EMU.gn_finalize(stats, gamma, beta, scale, vox, 8, 1e-5, coef_e, mr_e)
    coef_c, mr_c = torch.empty(n, c, 2, device="cuda"), torch.empty(n, 8, 2, device="cuda")
    be.gn_finalize(stats.cuda(), gamma.cuda(), beta.cuda(), dev(scale), vox, 8, 1e-5, coef_c, mr_c)
    assert rel(coef_c, coef_e) < 1e-5 and rel(mr_c, mr_e) < 1e-5
    # apply (all three source forms)
    for use2, useres in ((False, False), (True, False), (False, True)):
        out_e = torch.empty((n,) + sp + (c,), dtype=dtype)
        EMU.apply(y, coef_e, y2 if use2 else None, coef_e if use2 else None, res if useres else None, out_e)
        obuf = torch.zeros((n,) + sp + (2 * c,), dtype=dtype, device="cuda")
        out_c = obuf[..., c:]
        be.apply(y.cuda(), coef_c, dev(y2) if use2 else None, coef_c if use2 else None, dev(res) if useres else None,
                 out_c)
        assert rel(out_c, out_e) < tol(dtype, 0.5)
        assert float(obuf[..., :c].abs().max()) == 0
    # backward chain
    gact = rnd((n,) + sp + (c,), dtype, g)
    sums_e = torch.zeros(n, c, 3, dtype=torch.float64)
    EMU.gn_bwd_reduce(gact, y, coef_e, sums_e)
    sums_c = torch.zeros(n, c, 3, dtype=torch.float64, device="cuda")
    be.gn_bwd_reduce(gact.cuda(), y.cuda(), coef_e.cuda(), sums_c)
    assert rel(sums_c, sums_e) < 1e-5
    c3_e = torch.empty(n, c, 3)
    dg_e, db_e, dbi_e = torch.ones(c), torch.ones(c), torch.zeros(c)
    EMU.gn_bwd_finalize(sums_e, mr_e, gamma, scale, vox, 8, c3_e, dg_e, db_e, dbi_e)
    c3_c = torch.empty(n, c, 3, device="cuda")
    dg_c, db_c, dbi_c = torch.ones(c, device="cuda"), torch.ones(c, device="cuda"), torch.zeros(c, device="cuda")
    be.gn_bwd_finalize(sums_e.cuda(), mr_e.cuda(), gamma.cuda(), dev(scale), vox, 8, c3_c, dg_c, db_c, dbi_c)
    for a, b in ((c3_c, c3_e), (dg_c, dg_e), (db_c, db_e)):
        assert rel(a, b) < 1e-5
    assert (dbi_c.cpu() - dbi_e).abs().max() < 1e-4 * (1 + dbi_e.abs().max())
    dy_e = torch.empty((n,) + sp + (c,), dtype=dtype)
    EMU.gn_bwd_apply(gact, y, coef_e, c3_e, dy_e)
    dy_c = torch.empty((n,) + sp + (c,), dtype=dtype, device="cuda")
    be.gn_bwd_apply(gact.cuda(), y.cuda(), coef_e.cuda(), c3_e.cuda(), dy_c)
    assert rel(dy_c, dy_e) < tol(dtype, 0.5)
    cs_c = torch.zeros(c, device="cuda")
    be.colsum(gact.cuda(), cs_c)
    assert rel(cs_c, gact.double().sum((0, 1, 2, 3))) < 1e-4


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("dims,n,sp,c", [(3, 2, (4, 6, 8), 16), (2, 2, (1, 8, 12), 32), (3, 1, (2, 2, 2), 128)])
def test_pool(be, dtype, dims, n, sp, c):
    g = torch.Generator().manual_seed(4)
    x = torch.relu(sliced(n, sp, c, dtype, g, pad=16))          # ties at zero, like real activations
    osp = (sp[0] // 2 if dims == 3 else 1, sp[1] // 2, sp[2] // 2)
    out_e = torch.empty((n,) + osp + (c,), dtype=dtype)
    EMU.pool_fwd(x, out_e, dims)
    out_c = torch.empty((n,) + osp + (c,), dtype=dtype, device="cuda")
    be.pool_fwd(x.cuda(), out_c, dims)
    assert torch.equal(out_c.cpu().float(), out_e.float())
    go = rnd((n,) + osp + (c,), dtype, g)
    add = rnd((n,) + sp + (c,), dtype, g)
    gx_e = torch.empty((n,) + sp + (c,), dtype=dtype)
    EMU.pool_bwd(x, go, add, gx_e, dims)
    gx_c = torch.empty((n,) + sp + (c,), dtype=dtype, device="cuda")
    be.pool_bwd(x.cuda(), go.cuda(), add.cuda(), gx_c, dims)
    # positions whose window max is 0 are killed by the ReLU mask downstream; compare where x > 0
    m = (x > 0).float()
    assert rel(gx_c.cpu().float() * m, gx_e.float() * m) < tol(dtype, 0.5)


@pytest.mark.parametrize("c", [1, 2, 3, 4, 5, 11])
def test_head_and_losses(be, c):
    g = torch.Generator().manual_seed(5)
    nvox = (2, 5, 6, 7)
    z = 2 * torch.randn(nvox + (c,), generator=g)
    t = (torch.rand(nvox, generator=g) > 0.6).long() if c == 1 else torch.randint(0, c, nvox, generator=g)
    if c > 2:
        t[t == 1] = 0                      # one absent class
    p_e = torch.empty_like(z)
    EMU.head_probs(z, p_e)
    p_c = torch.empty_like(z, device="cuda")
    be.head_probs(z.cuda(), p_c)
    assert (p_c.cpu() - p_e).abs().max() < 2e-6
    alpha = torch.linspace(0.5, 1.5, c)
    for terms in (1, 2, 4, 3, 5, 7):
        for gamma in (2.0, 3.0):
            npart = be.part_size(c)
            part_e = torch.zeros(npart, dtype=torch.float64)
            met_e = torch.zeros(z.shape[0], c, 3, dtype=torch.float64)
            EMU.loss_partials(z, t, gamma, 0.25, part_e, met_e)
            part_c = torch.zeros(npart, dtype=torch.float64, device="cuda")
            met_c = torch.zeros(z.shape[0], c, 3, dtype=torch.float64, device="cuda")
            be.loss_partials(z.cuda(), t.cuda(), gamma, 0.25, part_c, met_c)
            assert rel(part_c, part_e) < 2e-6
            assert torch.equal(met_c.cpu(), met_e)          # counts: exact
            out_e, out_c = torch.empty(2), torch.empty(2, device="cuda")
            EMU.metric_finalize(met_e, out_e)
            be.metric_finalize(met_c, out_c)
            assert (out_c.cpu() - out_e).abs().max() < 1e-6
            met_p = torch.zeros_like(met_c)                 # the same sums from materialised probabilities
            be.metric_partials(p_c, t.cuda(), 0.5, met_p)
            assert torch.equal(met_p.cpu(), met_e)
            nl = 5 if c == 1 else 2 * c + 3
            loss_e, lc_e = torch.empty(()), torch.empty(nl)
            EMU.loss_finalize(part_e, c, terms, alpha, gamma, 0.25, loss_e, lc_e)
            loss_c, lc_c = torch.empty((), device="cuda"), torch.empty(nl, device="cuda")
            be.loss_finalize(part_e.cuda(), c, terms, alpha.cuda(), gamma, 0.25, loss_c, lc_c)
            assert abs(loss_c.item() - loss_e.item()) < 1e-6 * max(1, abs(loss_e.item()))
            assert rel(lc_c, lc_e) < 1e-6
            gs = torch.tensor([0.7])
            dz_e = torch.empty_like(z)
            EMU.loss_bwd(z, t, lc_e, gs, dz_e)
            dz_c = torch.empty_like(z, device="cuda")
            be.loss_bwd(z.cuda(), t.cuda(), lc_e.cuda(), gs.cuda(), dz_c)
            assert (dz_c.cpu() - dz_e).abs().max() < 1e-6 * (1 + dz_e.abs().max()) + 3e-5 * dz_e.abs().max()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("nc,cin", [(1, 16), (2, 16), (4, 16), (3, 32), (8, 16)])
def test_fused_head(be, dtype, nc, cin):
    g = torch.Generator().manual_seed(6)
    n, sp = 2, (3, 5, 8)
    xbuf = rnd((n,) + sp + (cin + 16,), dtype, g)
    x = xbuf[..., 8:8 + cin]
    w = torch.randn(nc, cin, 1, 1, 1, generator=g) * 0.3
    b = torch.randn(nc, generator=g) * 0.1
    lo_e, pr_e = torch.empty((n,) + sp + (nc,)), torch.empty((n,) + sp + (nc,))
    assert EMU.head_fwd(x, w, b, lo_e, pr_e)
    lo_c, pr_c = torch.empty_like(lo_e, device="cuda"), torch.empty_like(pr_e, device="cuda")
    assert be.head_fwd(x.cuda(), w.cuda(), b.cuda(), lo_c, pr_c)
    assert rel(lo_c, lo_e) < 1e-5 and (pr_c.cpu() - pr_e).abs().max() < 1e-5
    dl = torch.randn((n,) + sp + (nc,), generator=g)
    dx_e = torch.empty((n,) + sp + (cin,), dtype=dtype)
    dw_e, db_e = torch.zeros(nc, cin, 1, 1, 1), torch.zeros(nc)
    ok = EMU.head_bwd(x, dl, w, dx_e, dw_e, db_e)
    dx_c = torch.empty((n,) + sp + (cin,), dtype=dtype, device="cuda")
    dw_c, db_c = torch.zeros(nc, cin, 1, 1, 1, device="cuda"), torch.zeros(nc, device="cuda")
    okc = be.head_bwd(x.cuda(), dl.cuda(), w.cuda(), dx_c, dw_c, db_c)
    assert bool(ok) == bool(okc)
    if ok:
        assert rel(dx_c, dx_e) < tol(dtype, 0.5)
        assert rel(dw_c, dw_e) < 1e-5 and rel(db_c, db_e) < 1e-5


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n,sp,c,masked", [(2, (4, 6, 8), 16, True), (1, (3, 5, 7), 32, False),
                                           (2, (1, 8, 8), 64, True), (1, (2, 2, 2), 256, True)])
def test_groupnorm_fused_coefficient_forms(be, dtype, n, sp, c, masked):
    """apply_gn / gn_bwd_reduce_gn / gn_bwd_apply_gn (coefficients derived in-kernel from the statistics)
    against the composition of the unfused statements."""
    g = torch.Generator().manual_seed(31)
    y = sliced(n, sp, c, dtype, g, pad=16)
    y2 = rnd((n,) + sp + (c,), dtype, g)
    res = rnd((n,) + sp + (c,), dtype, g)
    gamma = 1 + 0.2 * torch.randn(c, generator=g)
    beta = 0.2 * torch.randn(c, generator=g)
    scale = (torch.rand(n, c, generator=g) > 0.2).float() / 0.8 if masked else None
    vox = sp[0] * sp[1] * sp[2]

    def stats_of(t):
        tf = t.double()
        return torch.stack([tf.sum((1, 2, 3)), (tf * tf).sum((1, 2, 3))], -1).contiguous()

    gn1 = (stats_of(y), gamma, beta, scale, vox, 8, 1e-5)
    gn2 = (stats_of(y2), gamma, beta, None, vox, 8, 1e-5)
    cu = lambda gn: tuple(v.cuda() if isinstance(v, torch.Tensor) else v for v in gn)
    out_e = torch.empty((n,) + sp + (c,), dtype=dtype)
    EMU.apply_gn(y, gn1, y2, gn2, res, out_e)
    out_c = torch.empty((n,) + sp + (c,), dtype=dtype, device="cuda")
    be.apply_gn(y.cuda(), cu(gn1), y2.cuda(), cu(gn2), res.cuda(), out_c)
    assert rel(out_c, out_e) < tol(dtype, 0.5)
    gact = rnd((n,) + sp + (c,), dtype, g)
    sums_e = torch.zeros(n, c, 3, dtype=torch.float64)
    EMU.gn_bwd_reduce_gn(gact, y, gn1, sums_e)
    sums_c = torch.zeros(n, c, 3, dtype=torch.float64, device="cuda")
    be.gn_bwd_reduce_gn(gact.cuda(), y.cuda(), cu(gn1), sums_c)
    assert rel(sums_c, sums_e) < 1e-5
    dy_e = torch.empty((n,) + sp + (c,), dtype=dtype)
    dg_e, db_e, dbi_e = torch.ones(c), torch.ones(c), torch.zeros(c)
    EMU.gn_bwd_apply_gn(gact, y, gn1, sums_e, dy_e, dg_e, db_e, dbi_e)
    dy_c = torch.empty((n,) + sp + (c,), dtype=dtype, device="cuda")
    dg_c, db_c, dbi_c = torch.ones(c, device="cuda"), torch.ones(c, device="cuda"), torch.zeros(c, device="cuda")
    be.gn_bwd_apply_gn(gact.cuda(), y.cuda(), cu(gn1), sums_e.cuda(), dy_c, dg_c, db_c, dbi_c)
    assert rel(dy_c, dy_e) < tol(dtype, 0.5)
    assert rel(dg_c, dg_e) < 1e-5 and rel(db_c, db_e) < 1e-5
    assert (dbi_c.cpu() - dbi_e).abs().max() < 1e-4 * (1 + dbi_e.abs().max())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n,sp,c,masked", [(2, (24, 24, 24), 64, True), (2, (12, 12, 12), 128, True),
                                           (2, (6, 6, 6), 256, False), (3, (4, 6, 8), 16, True),
                                           (1, (1, 64, 64), 32, True)])
def test_groupnorm_backward_single_launch(be, dtype, n, sp, c, masked):
    """b200seg_gn_bwd_fused_gn (reduce -> grid barrier -> apply in one launch) against the two-launch form"""
    g = torch.Generator().manual_seed(37)
    y = sliced(n, sp, c, dtype, g, pad=16).cuda()
    gact = rnd((n,) + sp + (c,), dtype, g).cuda()
    gamma = (1 + 0.2 * torch.randn(c, generator=g)).cuda()
    beta = (0.2 * torch.randn(c, generator=g)).cuda()
    scale = ((torch.rand(n, c, generator=g) > 0.2).float() / 0.8).cuda() if masked else None
    vox = sp[0] * sp[1] * sp[2]
    yf = y.double()
    stats = torch.stack([yf.sum((1, 2, 3)), (yf * yf).sum((1, 2, 3))], -1).contiguous()
    gn = (stats, gamma, beta, scale, vox, 8, 1e-5)
    dy_a = torch.empty((n,) + sp + (c,), dtype=dtype, device="cuda")
    dy_b = torch.empty_like(dy_a)
    if not be.gn_bwd_fused_ok(gact, y, dy_b):
        assert dtype == torch.float32 and c // 4 > 32      # fp32: more than 32 channel groups per voxel
        pytest.skip("shape stays on the two-launch form")
    sums = torch.zeros(n, c, 3, dtype=torch.float64, device="cuda")
    dg_a, db_a, dbi_a = torch.ones(c, device="cuda"), torch.ones(c, device="cuda"), torch.zeros(c, device="cuda")
    be.gn_bwd_reduce_gn(gact, y, gn, sums)
    be.gn_bwd_apply_gn(gact, y, gn, sums, dy_a, dg_a, db_a, dbi_a)
    for _ in range(3):                       # repeated launches: the one-shot barrier word is fresh each time
        buf = torch.zeros(n * c * 3 + 2, dtype=torch.float64, device="cuda")
        dg_b, db_b, dbi_b = torch.ones(c, device="cuda"), torch.ones(c, device="cuda"), torch.zeros(c, device="cuda")
        be.gn_bwd_fused_gn(gact, y, gn, buf[:n * c * 3].view(n, c, 3), buf[n * c * 3:], dy_b, dg_b, db_b, dbi_b)
        torch.cuda.synchronize()
        assert rel(buf[:n * c * 3].view(n, c, 3), sums) < 1e-5      # fp32 thread partials, different grids
        assert rel(dy_b, dy_a) < tol(dtype, 0.1)
        assert rel(dg_b, dg_a) < 1e-5 and rel(db_b, db_a) < 1e-5
        assert (dbi_b - dbi_a).abs().max() < 1e-4 * (1 + dbi_a.abs().max())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n,sp,c", [(2, (64, 96, 96), 16), (1, (61, 83, 97), 16), (2, (48, 48, 47), 32)])
def test_gn_bwd_reduce_large_streams(be, dtype, n, sp, c):
    """the large-level form of gn_bwd_reduce_gn (four trips of loads in flight, two CTAs per SM) against a direct
    fp64 statement of the three sums; ragged voxel counts exercise the four-trip / two-trip / single tails."""
    g = torch.Generator(device="cuda").manual_seed(5)
    y = torch.randn((n,) + sp + (c,), generator=g, device="cuda").to(dtype)
    ga = torch.randn((n,) + sp + (c,), generator=g, device="cuda").to(dtype)
    gamma = 1 + 0.2 * torch.randn(c, generator=g, device="cuda")
    beta = 0.2 * torch.randn(c, generator=g, device="cuda")
    scale = (torch.rand(n, c, generator=g, device="cuda") > 0.2).float() / 0.8
    vox = sp[0] * sp[1] * sp[2]
    yd = y.double()
    stats = torch.stack([yd.sum((1, 2, 3)), (yd * yd).sum((1, 2, 3))], -1).contiguous()
    sums = torch.zeros(n, c, 3, dtype=torch.float64, device="cuda")
    be.gn_bwd_reduce_gn(ga, y, (stats, gamma, beta, scale, vox, 8, 1e-5), sums)
    # fp64 statement with the SAME fp32 coefficients the kernel derives (mask decisions at y*A + B > 0)
    cpg = c // 8
    sg = stats.view(n, 8, cpg, 2).sum(2)
    m = cpg * vox
    mean = sg[..., 0] / m
    rstd = 1.0 / torch.sqrt((sg[..., 1] / m - mean * mean).clamp_min(0) + 1e-5)
    mean_c, rstd_c = mean.repeat_interleave(cpg, 1), rstd.repeat_interleave(cpg, 1)
    A = (rstd_c * gamma.double() * scale.double()).float()
    B = ((beta.double() - mean_c * rstd_c * gamma.double()) * scale.double()).float()
    mask = (torch.addcmul(B[:, None, None, None, :], y.float(), A[:, None, None, None, :]) > 0).double()
    gm = ga.double() * mask
    ref = torch.stack([gm.sum((1, 2, 3)), (gm * yd).sum((1, 2, 3)), yd.sum((1, 2, 3))], -1)
    torch.cuda.synchronize()
    den = ref.abs().amax(dim=(0, 1), keepdim=True) + 1e-9
    assert ((sums - ref).abs() / den).max() < 2e-5


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_multi_tensor_pack_and_unpack(be, dtype):
    """b200seg_pack_weights_multi / b200seg_unpack_wgrads_multi (tap-contiguous smem-transposed paths and the
    generic path) against the single-tensor entry points, for every operand layout the engine requests."""
    g = torch.Generator().manual_seed(11)
    shapes = [(K3, 3, (32, 16, 3, 3, 3), 128 ** 3), (K3, 3, (16, 16, 3, 3, 3), 128 ** 3), (K3, 3, (64, 64, 3, 3, 3), 24 ** 3),
              (K3, 3, (16, 1, 3, 3, 3), 96 ** 3), (K3, 2, (32, 32, 3, 3), 512 * 512), (K3, 3, (40, 24, 3, 3, 3), 8 ** 3),
              (K1, 3, (32, 32, 1, 1, 1), 96 ** 3), (K1, 3, (2, 16, 1, 1, 1), 96 ** 3),
              (DOWN, 3, (32, 16, 2, 2, 2), 48 ** 3), (DOWN, 2, (64, 32, 2, 2), 64 * 64),
              (UP, 3, (64, 16, 2, 2, 2), 96 ** 3), (UP, 2, (32, 16, 2, 2), 64 * 64)]
    reqs, singles = [], []
    for kind, dims, shp, vox in shapes:
        w = torch.randn(shp, generator=g).cuda()
        for which in ("fwd", "dgrad"):
            reqs.append((w, kind, which, dtype, dims, vox))
    many = be.pack_many(reqs)
    torch.cuda.synchronize()
    for (w, kind, which, dt, dims, vox), pm in zip(reqs, many):
        ps = be.pack_weight(w, kind, which, dt, dims, allow_tc=True, vox=vox)
        assert pm.code == ps.code and pm.t.shape == ps.t.shape
        assert torch.equal(pm.t, ps.t), (kind, which, tuple(w.shape))
    # unpack: [t][k][n] -> parameter layout (n, k, t...)
    items, refs = [], []
    for kind, dims, shp, vox in shapes:
        a, b = shp[0], shp[1]
        t = 1
        for q in shp[2:]:
            t *= q
        dwp = torch.randn((t, b, a), generator=g).cuda()
        grad = torch.zeros(shp, device="cuda")
        ref = torch.zeros(shp, device="cuda")
        be.unpack_wgrad(dwp, ref, kind, dims)
        items.append((dwp, grad))
        refs.append(ref)
    be.unpack_many(items)
    torch.cuda.synchronize()
    for (dwp, grad), ref in zip(items, refs):
        assert torch.equal(grad, ref), tuple(grad.shape)
