"""The LeakyReLU and InstanceNorm (groups = C) forms of the elementwise GroupNorm kernels, and the voxelmorph warp
(csrc/warp3d.cu), on the GPU.

GroupNorm forms.  At the pyramid levels of a 96^3 x 2 network with 16 features (plus one 512-channel level), on
pitched buffers with guard bands, with the exact-operand design of test_gpu_gn_exact.py restated for one group per
channel: statistics chosen so that every mean is a short dyadic and var + eps = 1/4 (rstd = 2 exactly), y and the
residual from {-4 .. 4} / 4, g from {-1, 0, 1} / 8, dyadic gamma and beta, dropout scale 0 or 1.25.  Then A, B, P, Q,
R are short dyadics, fmaf(y, A, B) and fmaf(y, Q, R) are exact, and the LeakyReLU product v * 0.01f is one rounding
-- so apply_gn and gn_bwd_apply_gn (given chosen backward sums) are compared bit for bit with an fp32 restatement in
the kernels' order.  The reductions (gn_bwd_reduce_gn, phase one of gn_bwd_fused_gn) sum non-dyadic fp32 terms in the
kernels' own order and are held to an fp64 reference within 2^-12 of the sum of |terms| (a lost or extra LeakyReLU
factor moves a sum by about the size of its negative part); the fused kernel's dy is checked against
the reference formed from the sums it wrote.

Warp.  Against torch.nn.functional.grid_sample on the GPU at the same fp32 sampling locations (built on the CPU with
the reference's chain, whose divisions are true divisions there): the nearest labels are identical; the trilinear
image is within 32 fp32 units of roundoff of an fp64 trilinear sample at the kernel's fp32 coordinates (relative to
the largest |value|); the d loss / d ddf gradient is held to fp64 autograd of that sampler within 1e-5 of the
gradient's scale.  Cases: the identity warp (ddf = 0, every coordinate an integer: one-sided derivatives), samples
far out of the volume, sizes with s - 1 a power of two (the chain is exact there, so coordinates land exactly on
.5 and exercise round-half-to-even), and non-cubic volumes with three distinct sides."""
import pytest
import torch
import torch.nn.functional as F

from pytorchdeeplearing_b200 import _abi

BF, F32 = torch.bfloat16, torch.float32
EPS = 2.0 ** -10
GUARD = 8            # guard elements on each side of each pitched row
OFF = 8              # channel 0 sits OFF elements into its row (16-byte aligned)
SLOPE = torch.tensor(0.01, dtype=torch.float32)

# (N, spatial, C, dtype): the registration net's levels at 96^3 x 2 with init_features 16 (and 32 for 512 channels)
GN_CASES = {
    "l96": (2, (96, 96, 96), 16, BF), "l48": (2, (48, 48, 48), 32, BF), "l24": (2, (24, 24, 24), 64, BF),
    "l12": (2, (12, 12, 12), 128, BF), "l6": (2, (6, 6, 6), 256, BF), "l6_512": (2, (6, 6, 6), 512, BF),
    "l48_f32": (2, (48, 48, 48), 32, F32), "l6_512_f32": (2, (6, 6, 6), 512, F32),
}


@pytest.fixture(scope="module")
def be():
    from pytorchdeeplearing_b200.runtime import cuda_backend
    return cuda_backend()


# ------------------------------------------------------------------------------------------- GroupNorm operands
def pitched(n, sp, c, dtype, fill=float("nan")):
    """(N, D, H, W, C) view into rows of OFF + C + GUARD elements; everything outside the view is `fill`"""
    ld = OFF + c + GUARD
    buf = torch.full((n,) + tuple(sp) + (ld,), fill, dtype=dtype, device="cuda")
    return buf, buf[..., OFF:OFF + c]


def guards_intact(buf, c):
    return bool(torch.isnan(buf[..., :OFF].float()).all() and torch.isnan(buf[..., OFF + c:].float()).all())


def design(n, sp, c, seed):
    """stats [N][C][2], gamma, beta, scale [N][C], y, y2, res, g (fp64 on the CPU) of the exact design"""
    gen = torch.Generator().manual_seed(seed)
    vox = sp[0] * sp[1] * sp[2]
    mean = (torch.randint(-8, 9, (n, c), generator=gen).double() / 16)
    var = 0.25 - EPS
    stats = torch.stack([mean * vox, (var + mean * mean) * vox], -1)
    gamma = torch.randint(1, 9, (c,), generator=gen).double() / 8
    beta = torch.randint(-8, 9, (c,), generator=gen).double() / 8
    scale = torch.where(torch.rand((n, c), generator=gen) < 0.2, 0.0, 1.25).double()
    ya = lambda: torch.randint(-4, 5, (n,) + tuple(sp) + (c,), generator=gen).double() / 4
    g = torch.randint(-1, 2, (n,) + tuple(sp) + (c,), generator=gen).double() / 8
    return dict(stats=stats, gamma=gamma, beta=beta, scale=scale, y=ya(), y2=ya(), res=ya(), g=g, vox=vox)


def coefs(d, stats=None):
    """A, B [N][C] in fp64 (exact by design), rounded to fp32 as the kernels round them"""
    stats = d["stats"] if stats is None else stats
    vox = d["vox"]
    mean = stats[..., 0] / vox
    var = (stats[..., 1] / vox - mean * mean).clamp_min(0)
    rstd = 1.0 / torch.sqrt(var + EPS)
    A = rstd * d["gamma"] * d["scale"]
    B = (d["beta"] - mean * rstd * d["gamma"]) * d["scale"]
    return A.float(), B.float(), mean, rstd


def leaky(v):
    """torch's LeakyReLU on fp32: v > 0 ? v : v * 0.01f"""
    return torch.where(v > 0, v, v * SLOPE)


def bwd_factor(v, g):
    return torch.where(v > 0, g, g * SLOPE)


def pqr(d, sums, mean, rstd):
    """P, Q, R [N][C] from the backward sums with one channel per group (gn_coef.cuh, in fp64)"""
    sc, ga, m = d["scale"], d["gamma"], float(d["vox"])
    s1, s2 = sums[..., 0] * sc, sums[..., 1] * sc
    m1 = ga * s1 / m
    m2 = ga * rstd * (s2 - mean * s1) / m
    P = rstd * ga * sc
    Q = -rstd * rstd * m2
    R = -rstd * m1 + rstd * rstd * mean * m2
    return P, Q, R, s1, s2, m1, m2


def bc(t, nd=3):
    return t.view(t.shape[0], *([1] * nd), t.shape[1])


def dev_gn(d, groups=None, act=_abi.ACT_LEAKY, stats=None):
    c = d["gamma"].numel()
    st = (d["stats"] if stats is None else stats).cuda().contiguous()
    return (st, d["gamma"].float().cuda(), d["beta"].float().cuda(), d["scale"].float().cuda(), d["vox"],
            c if groups is None else groups, EPS, act)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GN_CASES))
def test_leaky_instance_norm_forms_exact(be, name):
    n, sp, c, dt = GN_CASES[name]
    d = design(n, sp, c, seed=sorted(GN_CASES).index(name))
    A, B, mean, rstd = coefs(d)
    gn = dev_gn(d)
    # ---- apply_gn: leaky(y A + B) + leaky(y2 A + B) + res, fp32, one rounding to the storage type
    bufs = {}
    for k in ("y", "y2", "res", "g"):
        bufs[k] = pitched(n, sp, c, dt)
        bufs[k][1].copy_(d[k].to(dt))
    ob, out = pitched(n, sp, c, dt)
    be.apply_gn(bufs["y"][1], gn, bufs["y2"][1], gn, bufs["res"][1], out)
    pre1 = (d["y"] * bc(A.double()) + bc(B.double()))
    pre2 = (d["y2"] * bc(A.double()) + bc(B.double()))
    assert torch.equal(pre1.float().double(), pre1) and torch.equal(pre2.float().double(), pre2)   # exact by design
    want = ((leaky(pre1.float()) + leaky(pre2.float())) + d["res"].float()).to(dt)
    torch.cuda.synchronize()
    assert guards_intact(ob, c), "apply_gn wrote outside its view"
    assert torch.equal(out.cpu(), want), f"apply_gn: {(out.cpu().float() != want.float()).sum().item()} mismatches"
    # ---- gn_bwd_apply_gn with chosen sums: dy = (g' P) + fmaf(y, Q, R); the parameter gradients of the two samples
    gen = torch.Generator().manual_seed(7)
    a = torch.randint(-4, 5, (n, c), generator=gen).double() / 8
    b_ = torch.randint(-4, 5, (n, c), generator=gen).double() / 8
    s3 = torch.randint(-64, 65, (n, c), generator=gen).double()
    sums = torch.stack([a * d["vox"], b_ * d["vox"], s3], -1)
    P, Q, R, s1, s2, m1, m2 = pqr(d, sums, mean, rstd)
    Pf, Qf, Rf = P.float(), Q.float(), R.float()
    for t in (P, Q, R):
        assert torch.equal(t.float().double(), t)
    dyb, dy = pitched(n, sp, c, dt)
    dgam = torch.zeros(c, device="cuda")
    dbet = torch.zeros(c, device="cuda")
    dbia = torch.zeros(c, device="cuda")
    be.gn_bwd_apply_gn(bufs["g"][1], bufs["y"][1], gn, sums.cuda().contiguous(), dy, dgam, dbet, dbia)
    fy = d["y"] * bc(Q) + bc(R)
    assert torch.equal(fy.float().double(), fy)
    want_dy = (bwd_factor(pre1.float(), d["g"].float()) * bc(Pf) + fy.float()).to(dt)
    vox = float(d["vox"])
    dgam_s = (rstd * (s2 - mean * s1)).float()
    dbia_s = (rstd * d["gamma"] * s1 + (-rstd * rstd * m2) * s3 + R * vox).float()
    torch.cuda.synchronize()
    assert guards_intact(dyb, c), "gn_bwd_apply_gn wrote outside its view"
    assert torch.equal(dy.cpu(), want_dy), f"gn_bwd_apply_gn: {(dy.cpu().float() != want_dy.float()).sum().item()} mismatches"
    # two samples added into zero: the fp32 sum is the same in either order
    assert torch.equal(dbet.cpu(), s1.float()[0] + s1.float()[1])
    assert torch.equal(dgam.cpu(), dgam_s[0] + dgam_s[1])
    assert torch.equal(dbia.cpu(), dbia_s[0] + dbia_s[1])
    # ---- gn_bwd_reduce_gn: sums of g' and g' y (fp32 terms: bounded error) and of y (exact by design)
    got = torch.zeros((n, c, 3), dtype=torch.float64, device="cuda")
    be.gn_bwd_reduce_gn(bufs["g"][1], bufs["y"][1], gn, got)
    gp = bwd_factor(pre1.float(), d["g"].float()).double()
    red = (1, 2, 3)
    want_s = torch.stack([gp.sum(red), (gp * d["y"]).sum(red), d["y"].sum(red)], -1)
    scale_s = torch.stack([gp.abs().sum(red), (gp * d["y"]).abs().sum(red), d["y"].abs().sum(red)], -1)
    err = (got.cpu() - want_s).abs()
    assert torch.equal(got.cpu()[..., 2], want_s[..., 2])
    assert (err <= 2.0 ** -12 * scale_s + 1e-30).all(), f"gn_bwd_reduce_gn: max err {err.max().item():.3e}"
    # ---- gn_bwd_fused_gn (the small levels): its sums as above, its dy from those sums
    if be.gn_bwd_fused_ok(bufs["g"][1], bufs["y"][1], dy):
        fs = torch.zeros(n * c * 3 + 2, dtype=torch.float64, device="cuda")
        fdyb, fdy = pitched(n, sp, c, dt)
        z = [torch.zeros(c, device="cuda") for _ in range(3)]
        be.gn_bwd_fused_gn(bufs["g"][1], bufs["y"][1], gn, fs[:n * c * 3].view(n, c, 3), fs[n * c * 3:], fdy, *z)
        torch.cuda.synchronize()
        assert guards_intact(fdyb, c)
        fsums = fs[:n * c * 3].view(n, c, 3).cpu()
        ferr = (fsums - want_s).abs()
        assert (ferr <= 2.0 ** -12 * scale_s + 1e-30).all(), f"gn_bwd_fused_gn sums: max err {ferr.max().item():.3e}"
        P2, Q2, R2 = pqr(d, fsums, mean, rstd)[:3]
        ref = gp * bc(P2) + d["y"] * bc(Q2) + bc(R2)
        tol = 2.0 ** -20 * (gp.abs() * bc(P2.abs()) + d["y"].abs() * bc(Q2.abs()) + bc(R2.abs())) \
            + (2.0 ** -8 if dt == BF else 2.0 ** -22) * ref.abs() + 1e-30
        ok = (fdy.cpu().double() - ref).abs() <= tol
        assert ok.all(), f"gn_bwd_fused_gn dy: {(~ok).sum().item()} out of bound"


@pytest.mark.gpu
def test_relu_form_unchanged_by_the_act_field(be):
    """a 7-tuple GroupNorm reference (no act) and an explicit ACT_RELU give the same bits as the fp32 restatement"""
    n, sp, c = 2, (24, 24, 24), 64
    d = design(n, sp, c, seed=3)
    yb, y = pitched(n, sp, c, BF)
    y.copy_(d["y"].to(BF))
    outs = []
    for gn in (dev_gn(d, groups=8)[:7], dev_gn(d, groups=8, act=_abi.ACT_RELU)):
        ob, out = pitched(n, sp, c, BF)
        be.apply_gn(y, gn, None, None, None, out)
        outs.append(out.cpu())
    assert torch.equal(outs[0], outs[1])


@pytest.mark.gpu
def test_fused_families_refuse_leaky_on_device(be):
    x = torch.zeros((1, 32, 32, 32, 1), device="cuda")
    out = torch.zeros((1, 32, 32, 32, 16), dtype=BF, device="cuda")
    d = design(1, (32, 32, 32), 16, seed=1)
    gn = dev_gn(d)
    w = torch.zeros(27 * 16, dtype=BF, device="cuda")
    b = torch.zeros(16, device="cuda")
    with pytest.raises(RuntimeError, match="ACT_RELU"):
        be._check(be.lib.b200seg_stem_gn_apply(_abi.C.byref(_abi._desc(x)), w.data_ptr(), b.data_ptr(), w.data_ptr(),
                                               b.data_ptr(), _abi.C.byref(be._gn(gn)), _abi.C.byref(be._gn(gn)),
                                               _abi.C.byref(_abi._desc(out)), 0, None))


# ------------------------------------------------------------------------------------------------------- warp
def chain_coords(ddf):
    """fp32 sampling coordinates (u_D, u_H, u_W) per voxel, (N, D, H, W, 3), by the reference's chain on the CPU, and
    the normalised grid_sample grid (N, D, H, W, 3) in (x, y, z) order"""
    n, _, D, H, W = ddf.shape
    vectors = [torch.arange(0, s) for s in (D, H, W)]
    grid = torch.stack(torch.meshgrid(vectors, indexing="ij")).unsqueeze(0).float()
    new_locs = grid + ddf
    for i, s in enumerate((D, H, W)):
        new_locs[:, i, ...] = 2 * (new_locs[:, i, ...] / (s - 1) - 0.5)
    g = new_locs.permute(0, 2, 3, 4, 1)[..., [2, 1, 0]]
    u = torch.stack([((g[..., 2 - i] + 1) / 2) * (s - 1) for i, s in enumerate((D, H, W))], -1)
    return u, g


def trilinear64(img, u, cell):
    """fp64 trilinear sample of img (N, C, D, H, W) at u (N, D, H, W, 3) in the floor cell `cell` (int64, same shape),
    zero outside; differentiable in u"""
    n, c, D, H, W = img.shape
    out = 0
    f = (u - cell.double())
    for k in range(8):
        o = torch.tensor([(k >> 2) & 1, (k >> 1) & 1, k & 1])         # (z, y, x) offsets
        idx = cell + o
        w = torch.ones_like(u[..., 0])
        for a in range(3):
            w = w * (f[..., a] if o[a] else 1 - f[..., a])
        ok = ((idx >= 0) & (idx < torch.tensor([D, H, W]))).all(-1)
        lin = ((idx[..., 0].clamp(0, D - 1) * H + idx[..., 1].clamp(0, H - 1)) * W + idx[..., 2].clamp(0, W - 1))
        vals = torch.gather(img.reshape(n, c, -1), 2, lin.reshape(n, 1, -1).expand(n, c, -1)).view(n, c, *u.shape[1:4])
        out = out + vals * (w * ok).unsqueeze(1)
    return out


WARP_CASES = {
    "identity_cubic": dict(n=2, sp=(17, 17, 17), ci=1, cl=3, amp=0.0),      # s - 1 = 16: integer coordinates
    "random_noncubic": dict(n=2, sp=(12, 20, 28), ci=1, cl=3, amp=3.0),
    "far_out_of_volume": dict(n=1, sp=(10, 14, 18), ci=2, cl=1, amp=40.0),
    "half_integers": dict(n=2, sp=(17, 33, 65), ci=1, cl=2, amp="half"),
    "registration_96": dict(n=2, sp=(96, 96, 96), ci=1, cl=3, amp=4.0),
}


def warp_inputs(case, seed):
    gen = torch.Generator().manual_seed(seed)
    n, sp, ci, cl, amp = case["n"], case["sp"], case["ci"], case["cl"], case["amp"]
    if amp == "half":
        ddf = torch.randint(-8, 9, (n, 3) + sp, generator=gen).float() / 2
    else:
        ddf = torch.randn((n, 3) + sp, generator=gen) * amp
    img = torch.randn((n, ci) + sp, generator=gen)
    lab = torch.randint(0, 4, (n, cl) + sp, generator=gen).float()
    return ddf, img, lab


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(WARP_CASES))
def test_warp_against_torch(be, name):
    from pytorchdeeplearing_b200 import warp3d
    case = WARP_CASES[name]
    ddf, img, lab = warp_inputs(case, seed=len(name))
    u, g = chain_coords(ddf)
    if case["amp"] == "half":
        assert (u - u.floor() == 0.5).any(), "the design puts coordinates exactly on .5"
    # ---- nearest label: identical to torch's grid_sample on the GPU at the same coordinates
    want_lab = F.grid_sample(lab.cuda(), g.cuda(), align_corners=True, mode="nearest")
    # the head writes ddf channels-last: pass it as such
    ddf_cl = ddf.permute(0, 2, 3, 4, 1).contiguous().cuda().permute(0, 4, 1, 2, 3)
    ddf_cl.requires_grad_(True)
    moved_img, moved_lab = warp3d(img.cuda(), lab.cuda(), ddf_cl)
    assert torch.equal(moved_lab, want_lab), f"labels: {(moved_lab != want_lab).sum().item()} mismatches"
    # ---- trilinear image: within 16 u of the fp64 sample at the kernel's fp32 coordinates
    cell = u.floor().long()
    ref = trilinear64(img.double(), u.double(), cell)
    bound = 32 * 2.0 ** -24 * img.abs().max().item()
    err = (moved_img.detach().cpu().double() - ref).abs().max().item()
    assert err <= bound, f"image: max err {err:.3e} > {bound:.3e}"
    torch_img = F.grid_sample(img.cuda(), g.cuda(), align_corners=True, mode="bilinear")
    assert (moved_img.detach() - torch_img).abs().max().item() <= 2 * bound
    # ---- d loss / d ddf through the image, against fp64 autograd of the sampler in the same cells
    gout = torch.randn(moved_img.shape, generator=torch.Generator().manual_seed(5))
    moved_img.backward(gout.cuda())
    u64 = u.double().requires_grad_(True)
    (trilinear64(img.double(), u64, cell) * gout.double()).sum().backward()
    want_g = u64.grad.permute(0, 4, 1, 2, 3)                    # du / dddf = 1 along each axis
    got_g = ddf_cl.grad.cpu().double()
    scale = want_g.abs().max().item() + 1e-30
    gerr = (got_g - want_g).abs().max().item()
    assert gerr <= 1e-5 * scale, f"ddf gradient: max err {gerr:.3e} (scale {scale:.3e})"
    if case["amp"] == 0.0:
        # the identity warp: the image comes back unchanged, the gradient is the one-sided (forward) difference
        assert torch.equal(moved_img.detach().cpu(), img)
    # ---- the addend form of the backward: + the caller's own gradient on ddf, bit for bit
    field = ddf.permute(0, 2, 3, 4, 1).contiguous().cuda()
    add = torch.randn(field.shape, generator=torch.Generator().manual_seed(9)).cuda()
    g0 = torch.empty_like(field)
    g1 = torch.empty_like(field)
    be.warp3d_bwd(field, img.cuda(), gout.cuda(), None, g0)
    be.warp3d_bwd(field, img.cuda(), gout.cuda(), add, g1)
    assert torch.equal(g1, g0 + add)
    assert torch.equal(g0.permute(0, 4, 1, 2, 3), ddf_cl.grad)


@pytest.mark.gpu
def test_warp_is_deterministic_and_label_path_has_no_gradient(be):
    from pytorchdeeplearing_b200 import warp3d
    ddf, img, lab = warp_inputs(WARP_CASES["random_noncubic"], seed=11)
    d = ddf.cuda().requires_grad_(True)
    mi1, ml1 = warp3d(img.cuda(), lab.cuda(), d)
    mi2, ml2 = warp3d(img.cuda(), lab.cuda(), d)
    assert torch.equal(mi1, mi2) and torch.equal(ml1, ml2)
    assert not ml1.requires_grad
    _, ml = warp3d(None, lab.cuda(), d)
    assert torch.equal(ml, ml1)
    mi, none = warp3d(img.cuda(), None, d)
    assert none is None and torch.equal(mi, mi1)
