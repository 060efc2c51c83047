"""The LeakyReLU and InstanceNorm (groups = C) forms of the elementwise GroupNorm kernels, and the voxelmorph warp
(csrc/warp3d.cu), on the GPU.

GroupNorm forms.  At the pyramid levels of a 96^3 x 2 network with 16 features (plus one 512-channel level, whose
coefficient loops take a second trip over the CTA's 256 threads) and at unaligned / odd channel counts (the VEC = 1
and rounded-grid kernels), on pitched buffers with guard bands, with the exact-operand design of test_gpu_gn_exact.py
restated for one group per channel: statistics chosen so that every mean is a short dyadic and var + eps = 1/4
(rstd = 2 exactly), y and the residual from {-4 .. 4} / 4, g from {-1, 0, 1} / 8, dyadic gamma and beta, dropout
scale 0 or 1.25.  Then A, B, P, Q, R are short dyadics, fmaf(y, A, B) and fmaf(y, Q, R) are exact, and the LeakyReLU
product v * 0.01f is one rounding -- so apply_gn and gn_bwd_apply_gn (given chosen backward sums) are compared bit for
bit with an fp32 restatement in the kernels' order.  Channels with beta = 0 carry y = mean at every eighth voxel,
where v = fmaf(y, A, B) is exactly 0 (as are all v of a dropped channel): the branch test v > 0 is pinned where it
differs from v >= 0.

The reductions (gn_bwd_reduce_gn, phase one of gn_bwd_fused_gn) by channel class, c mod 3:
  0  dense: g everywhere, terms g' = g or fl(0.01f g) -- held to the fp32 chain of the launch geometry, (trips +
     shuffle levels + 2) u of the sum of |terms|, the trips being the voxels one thread walks;
  1  g != 0 only where v > 0: dyadic terms, every partial sum exact;
  2  g = +-1/8 at <= 3 voxels, each with v <= 0 and y = -c for one power of two c per channel: every partial sum is
     J fl(0.01f) 2^k with |J| <= 3, and 3 * 5368709 < 2^24, so it is exact in fp32 in any order.
Classes 1 and 2 (and the sum of y) are compared bit for bit.  The fused kernel's dy is checked against the reference
formed from the sums it wrote.

Warp.  Bit for bit against fp32 restatements at the reference chain's fp32 sampling coordinates (built on the CPU,
whose divisions are true divisions): the nearest labels (label = linear voxel index + 1, so every moved label names
the voxel round-half-to-even picked) and the trilinear image (make_cell's weights and the corner-order fmaf chain,
fmaf emulated exactly); the labels also equal torch's grid_sample on the GPU.  d loss / d ddf is held per element to
(8 ci + 6) u of the sum of its terms' |values| around their fp64 sum (nvcc may contract the products); the addend
form is bit for bit the plain result plus the addend.  Outputs sit in NaN-filled guarded buffers, and the inputs
come back unchanged.  Cases: the identity warp, samples far out of the volume, ties at .5, non-cubic volumes,
extents 2 and 3, coordinates on the cut-offs -2 and s + 1 and on the faces -1, 0, s - 1 and s and next to each,
one to three image channels, and displacements of +-1e38, +-inf and NaN, where torch's CUDA grid_sample and its
autograd give a zero image and a zero gradient."""
import math

import pytest
import torch
import torch.nn.functional as F

from pytorchdeeplearing_b200 import _abi
from test_gpu_gn_exact import E, EW_CASES, SMS, ew_blocks, ew_variants, reduce_staged, required_variants, trip_counts
from test_gpu_gn_exact import vec_ok, vec_width

BF, F32 = torch.bfloat16, torch.float32
EPS = 2.0 ** -10
U = 2.0 ** -24       # fp32 unit roundoff
GUARD = 8            # guard elements on each side of each pitched row
OFF = 8              # channel 0 sits OFF elements into its row (16-byte aligned; 9 takes the VEC = 1 kernels)
SLOPE = torch.tensor(0.01, dtype=torch.float32)

# The cases are EW_CASES of test_gpu_gn_exact.py, run here with LeakyReLU and one group per channel: the registration
# net's levels at 96^3 x 2 with init_features 16, the unaligned (VEC = 1), odd-channel (rounded grid) and ragged
# cases; plus the 512-channel level (init_features 32), which only the InstanceNorm form can take.
LEVELS = {"l96": "vnet96", "l48": "vnet48", "l24": "vnet24", "l12": "vnet12", "l6": "vnet6", "l48_f32": "vnet48_f32"}
SHARED = ("vec1", "vec1_f32", "vec1_c24", "c24", "c24_f32", "c48", "c96", "c192", "c384", "ragged47", "ragged47_f32",
          "ragged61")
GN_CASES = {**{k: EW_CASES[v] for k, v in LEVELS.items()}, **{k: EW_CASES[k] for k in SHARED},
            "l6_512": E(2, (6, 6, 6), 512), "l6_512_f32": E(2, (6, 6, 6), 512, F32)}


def case(name):
    """(N, spatial, C, dtype, offset of channel 0) of one case"""
    cs = GN_CASES[name]
    return cs["n"], cs["sp"], cs["c"], cs["dtype"], cs["off"]


@pytest.fixture(scope="module")
def be():
    from pytorchdeeplearing_b200.runtime import cuda_backend
    return cuda_backend()


# ------------------------------------------------------------------------------------------- GroupNorm operands
def pitched(n, sp, c, dtype, off=OFF, fill=float("nan")):
    """(N, D, H, W, C) view into rows of off + C + GUARD elements; everything outside the view is `fill`"""
    ld = off + c + GUARD
    buf = torch.full((n,) + tuple(sp) + (ld,), fill, dtype=dtype, device="cuda")
    return buf, buf[..., off:off + c]


def guards_intact(buf, c, off=OFF):
    return bool(torch.isnan(buf[..., :off].float()).all() and torch.isnan(buf[..., off + c:].float()).all())


def design(n, sp, c, seed):
    """stats [N][C][2], gamma, beta, scale [N][C], y, y2, res, g (fp64 on the CPU) of the exact design, the channel
    class (c mod 3) and the pre-activation v of the first branch"""
    gen = torch.Generator().manual_seed(seed)
    vox = sp[0] * sp[1] * sp[2]
    mean = (torch.randint(-8, 9, (n, c), generator=gen).double() / 16)
    var = 0.25 - EPS
    stats = torch.stack([mean * vox, (var + mean * mean) * vox], -1)
    gamma = torch.randint(1, 9, (c,), generator=gen).double() / 8
    beta = torch.randint(-8, 9, (c,), generator=gen).double() / 8
    beta[torch.arange(c) % 4 == 3] = 0.0
    scale = torch.where(torch.rand((n, c), generator=gen) < 0.2, 0.0, 1.25).double()
    shape = (n,) + tuple(sp) + (c,)
    ya = lambda: torch.randint(-4, 5, shape, generator=gen).double() / 4
    y, y2, res = ya(), ya(), ya()
    g = torch.randint(-1, 2, shape, generator=gen).double() / 8
    A = 2.0 * gamma * scale
    B = (beta - mean * 2.0 * gamma) * scale
    # v = 0: y = mean in the channels with beta = 0 (then B = -mean A), at every eighth voxel
    j = torch.arange(vox).view(1, *sp, 1)
    zero = (j % 8 == 5) & (beta == 0)
    y = torch.where(zero, bc(mean), y)
    cls = torch.arange(c) % 3
    v = y * bc(A) + bc(B)
    g = torch.where((cls == 1) & (v <= 0), 0.0, g)
    # class 2: g = +-1/8 at three voxels, y = -c there with c the least power of two (>= 1/4) such that v <= 0
    g = torch.where(cls == 2, 0.0, g)
    need = torch.where(A > 0, B / torch.where(A > 0, A, 1.0), 0.0).clamp_min(0.25)
    cpow = 2.0 ** torch.ceil(torch.log2(need))
    yf, gf = y.view(n, vox, c), g.view(n, vox, c)
    for ni in range(n):
        for ch in range(2, c, 3):
            pos = torch.randperm(vox, generator=gen)[:3]
            yf[ni, pos, ch] = -cpow[ni, ch]
            gf[ni, pos, ch] = (torch.randint(0, 2, (3,), generator=gen).double() * 2 - 1) / 8
    v = y * bc(A) + bc(B)
    return dict(stats=stats, gamma=gamma, beta=beta, scale=scale, y=y, y2=y2, res=res, g=g, vox=vox, cls=cls, v=v)


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


def chain_len(name, fused):
    """the fp32 roundings on the way to one (n, c) sum of the dense class: the voxels one thread walks (its serial
    fp32 chain, elementwise.cu ew_blocks and the voxel loops), the shuffle levels of the warp fold, and two for the
    fp64 remainder (at most 2^29 fp64 additions) and the first-order bound's slack"""
    n, sp, c, dt, off = case(name)
    cs = GN_CASES[name]
    V = math.prod(sp)
    G = c // (vec_width(dt) if vec_ok(cs) else 1)
    if fused:
        bx = ew_blocks(V, G, n, 1)[0]
        while bx > 1 and bx * n > SMS:
            bx -= 1
        lanes = min(G, 32)
    else:
        deep = V * G >= SMS * 2 * 256 * 8
        bx = ew_blocks(V, G, n, 2 if deep else 3)[0]
        lanes = G if reduce_staged(cs, True, groups=c) and G < 32 and G & (G - 1) == 0 else 32
    return max(trip_counts(V, bx * 256 // G)) + int(math.log2(32 // lanes)) + 2


def check_sums(got, want, scale, cls, name, what, fused):
    """classes 1, 2 and the sum of y bit for bit; the dense class within its chain bound"""
    got = got.cpu()
    exact = (cls != 0).view(1, -1, 1) & torch.ones_like(got, dtype=torch.bool)
    exact[..., 2] = True
    ne = exact & (got != want)
    if bool(ne.any()):
        idx = tuple(ne.nonzero()[0].tolist())
        raise AssertionError(f"{name} {what}: {int(ne.sum())} exact sums differ; first (n, c, k) = {idx} (class "
                             f"{int(cls[idx[1]])}): got {float(got[idx])!r}, want {float(want[idx])!r}")
    k = chain_len(name, fused)
    bad = ~exact & ~((got - want).abs() <= k * U * scale)
    if bool(bad.any()):
        idx = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{name} {what}: dense sum {idx} off by {float((got - want)[idx]):.3e}, bound "
                             f"{k} u sum|terms| = {float(k * U * scale[idx]):.3e}")


# ------------------------------------------------------------------------------------------------- CPU part
@pytest.mark.parametrize("name", sorted(GN_CASES))
def test_leaky_design_premises(name):
    n, sp, c, dt, off = case(name)
    d = design(n, sp, c, seed=sorted(GN_CASES).index(name))
    v, g, y, cls = d["v"], d["g"], d["y"], d["cls"]
    A, B, _, _ = coefs(d)
    assert torch.equal(A.double(), 2.0 * d["gamma"] * d["scale"])
    # v = 0 exactly with g != 0 in kept channels: the elements where v > 0 and v >= 0 differ
    on = bc(d["scale"] != 0)
    assert bool(((v == 0) & (g != 0) & on).any())
    assert torch.equal(y.to(dt).double(), y)
    # class 1: dyadic terms, sums exact: sum |g| < 2^24 2^-3, sum |g y| < 2^24 2^-7 (y a multiple of 2^-4)
    c1 = cls == 1
    assert bool((v[..., c1][g[..., c1] != 0] > 0).all())
    assert bool((y * 16 == (y * 16).round()).all())
    red = tuple(range(1, len(sp) + 1))
    assert float((g.abs() * (cls == 1)).sum(red).max()) < 2 ** 24 * 2.0 ** -3
    assert float(((g * y).abs() * (cls == 1)).sum(red).max()) < 2 ** 24 * 2.0 ** -7
    # class 2: at most three voxels per (n, c), v <= 0 there, one power of two |y| per (n, c)
    c2 = cls == 2
    g2, y2, v2 = g[..., c2], y[..., c2], v[..., c2]
    nz = g2 != 0
    assert int(nz.sum(red).max()) <= 3
    assert bool((v2[nz] <= 0).all())
    ay = torch.where(nz, y2.abs(), 0.0).amax(red)
    assert bool((torch.where(nz, y2.abs(), bc(ay)) == bc(ay)).all())
    assert bool((torch.log2(ay[ay > 0]) == torch.log2(ay[ay > 0]).round()).all())
    assert 3 * 5368709 < 2 ** 24 and float(SLOPE.double() * 2 ** 29) == 5368709.0
    # the sum of y (exact in any order)
    assert float(y.abs().sum(red).max()) < 2 ** 24 * 2.0 ** -4


def test_leaky_cases_reach_every_variant_of_the_relu_form():
    reached = set().union(*(ew_variants(cs, groups=cs["c"], act=_abi.ACT_LEAKY) for cs in GN_CASES.values()))
    want = required_variants(_abi.ACT_LEAKY)
    assert want <= reached, sorted(want - reached)


def test_sum_checker_rejects_one_ulp_and_a_loose_dense_sum():
    n, c = 2, 6
    want = torch.arange(n * c * 3, dtype=torch.float64).view(n, c, 3) / 8 + 1
    cls = torch.arange(c) % 3
    scale = want.abs()
    check_sums(want.clone(), want, scale, cls, "vec1", "same", False)
    for idx in ((1, 2, 0), (0, 1, 1), (1, 0, 2)):          # class 2, class 1, the sum of y of a dense channel
        got = want.clone()
        got.view(torch.int64)[idx] += 1
        with pytest.raises(AssertionError, match=str(idx).replace("(", r"\(").replace(")", r"\)")):
            check_sums(got, want, scale, cls, "vec1", "one ulp", False)
    got = want.clone()
    got[1, 3, 0] *= 1 + 2.0 ** -12
    with pytest.raises(AssertionError, match="dense sum"):
        check_sums(got, want, scale, cls, "vec1", "2^-12", False)


# ------------------------------------------------------------------------------------------------- GPU part
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GN_CASES))
def test_leaky_instance_norm_forms_exact(be, name):
    n, sp, c, dt, off = case(name)
    d = design(n, sp, c, seed=sorted(GN_CASES).index(name))
    A, B, mean, rstd = coefs(d)
    gn = dev_gn(d)
    # ---- apply_gn: leaky(y A + B) + leaky(y2 A + B) + res, fp32, one rounding to the storage type
    bufs = {}
    for k in ("y", "y2", "res", "g"):
        bufs[k] = pitched(n, sp, c, dt, off)
        bufs[k][1].copy_(d[k].to(dt))
    ob, out = pitched(n, sp, c, dt, off)
    be.apply_gn(bufs["y"][1], gn, bufs["y2"][1], gn, bufs["res"][1], out)
    pre1 = (d["y"] * bc(A.double()) + bc(B.double()))
    pre2 = (d["y2"] * bc(A.double()) + bc(B.double()))
    assert torch.equal(pre1.float().double(), pre1) and torch.equal(pre2.float().double(), pre2)   # exact by design
    want = ((leaky(pre1.float()) + leaky(pre2.float())) + d["res"].float()).to(dt)
    torch.cuda.synchronize()
    assert guards_intact(ob, c, off), "apply_gn wrote outside its view"
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
    dyb, dy = pitched(n, sp, c, dt, off)
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
    assert guards_intact(dyb, c, off), "gn_bwd_apply_gn wrote outside its view"
    assert torch.equal(dy.cpu(), want_dy), f"gn_bwd_apply_gn: {(dy.cpu().float() != want_dy.float()).sum().item()} mismatches"
    # one or two samples added into zero: the fp32 sum is the same in either order
    assert torch.equal(dbet.cpu(), s1.float().sum(0))
    assert torch.equal(dgam.cpu(), dgam_s.sum(0))
    assert torch.equal(dbia.cpu(), dbia_s.sum(0))
    # ---- gn_bwd_reduce_gn: sums of g' and g' y by channel class, and of y (exact by design)
    gp = bwd_factor(pre1.float(), d["g"].float()).double()
    red = (1, 2, 3)
    want_s = torch.stack([gp.sum(red), (gp * d["y"]).sum(red), d["y"].sum(red)], -1)
    scale_s = torch.stack([gp.abs().sum(red), (gp * d["y"]).abs().sum(red), d["y"].abs().sum(red)], -1)
    sb = torch.full((n * c * 3 + 2 * GUARD,), float("nan"), dtype=torch.float64, device="cuda")
    got = sb[GUARD:GUARD + n * c * 3].view(n, c, 3)
    got.zero_()
    be.gn_bwd_reduce_gn(bufs["g"][1], bufs["y"][1], gn, got)
    torch.cuda.synchronize()
    assert bool(sb[:GUARD].isnan().all() and sb[-GUARD:].isnan().all()), "gn_bwd_reduce_gn wrote outside its sums"
    check_sums(got, want_s, scale_s, d["cls"], name, "gn_bwd_reduce_gn", fused=False)
    # ---- gn_bwd_fused_gn (the small levels): its sums as above, its dy from those sums
    if be.gn_bwd_fused_ok(bufs["g"][1], bufs["y"][1], dy):
        fs = torch.zeros(n * c * 3 + 2, dtype=torch.float64, device="cuda")
        fdyb, fdy = pitched(n, sp, c, dt, off)
        z = [torch.zeros(c, device="cuda") for _ in range(3)]
        be.gn_bwd_fused_gn(bufs["g"][1], bufs["y"][1], gn, fs[:n * c * 3].view(n, c, 3), fs[n * c * 3:], fdy, *z)
        torch.cuda.synchronize()
        assert guards_intact(fdyb, c, off)
        fsums = fs[:n * c * 3].view(n, c, 3).cpu()
        check_sums(fsums, want_s, scale_s, d["cls"], name, "gn_bwd_fused_gn sums", fused=True)
        P2, Q2, R2 = pqr(d, fsums, mean, rstd)[:3]
        ref = gp * bc(P2) + d["y"] * bc(Q2) + bc(R2)
        tol = 2.0 ** -20 * (gp.abs() * bc(P2.abs()) + d["y"].abs() * bc(Q2.abs()) + bc(R2.abs())) \
            + (2.0 ** -8 if dt == BF else 2.0 ** -22) * ref.abs() + 1e-30
        ok = (fdy.cpu().double() - ref).abs() <= tol
        assert ok.all(), f"gn_bwd_fused_gn dy: {(~ok).sum().item()} out of bound"
    for k in ("y", "g"):
        assert guards_intact(bufs[k][0], c, off)
        assert torch.equal(bufs[k][1].cpu(), d[k].to(dt)), f"input {k} changed"


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
U32 = 2.0 ** -24          # fp32 unit roundoff
INF = float("inf")


def chain_norm(gi, f, s):
    """the reference's normalised location along one axis of extent s: 2 (loc / (s - 1) - 0.5), loc = grid index gi
    plus displacement f, in fp32"""
    return 2 * ((gi + f) / (s - 1) - 0.5)


def chain_u(gi, f, s):
    """grid_sample's unnormalisation of that location, ((nrm + 1) / 2) (s - 1): the fp32 sampling coordinate"""
    return ((chain_norm(gi, f, s) + 1) / 2) * (s - 1)


def chain_coords(ddf):
    """fp32 sampling coordinates (u_D, u_H, u_W) per voxel, (N, D, H, W, 3), by the reference's chain on the CPU, and
    the normalised grid_sample grid (N, D, H, W, 3) in (x, y, z) order"""
    sp = ddf.shape[2:]
    grid = torch.meshgrid([torch.arange(0, s) for s in sp], indexing="ij")
    nrm = [chain_norm(grid[i], ddf[:, i], s) for i, s in enumerate(sp)]
    u = torch.stack([((nrm[i] + 1) / 2) * (s - 1) for i, s in enumerate(sp)], -1)
    return u, torch.stack(nrm[::-1], -1)


def in_range(u, sp):
    """coord_in_range on every axis: -2 < u < s + 1"""
    return ((u > -2) & (u < torch.tensor(sp, dtype=torch.float32) + 1)).all(-1)


def fmaf32(a, b, c):
    """fmaf on fp32 tensors, exactly: the fp64 product of two fp32 numbers is exact; TwoSum gives the rounding error
    of its fp64 sum with c, and a sum that rounded onto an fp32 midpoint goes to the side that error points to"""
    p = a.double() * b.double()
    c = c.double()
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.float()
    rd = r.double()
    up = torch.nextafter(r, torch.full_like(r, INF))
    dn = torch.nextafter(r, torch.full_like(r, -INF))
    r2 = torch.where((s == (rd + up.double()) / 2) & (e > 0), up, r)
    return torch.where((s == (rd + dn.double()) / 2) & (e < 0), dn, r2)


def cell32(u, sp):
    """make_cell restated in fp32 at the coordinates u (N, D, H, W, 3; (D, H, W) order): whether every coordinate is
    in range, the per-axis factors e = (c0 + 1) - u and w = u - c0 of the floor cell c0 (-4 out of range), and per
    corner in the kernel's order its (z, y, x) offset, index, fp32 weight ((x y) z) and in-volume flag"""
    inr = in_range(u, sp).unsqueeze(-1)
    c0 = torch.where(inr, u.floor(), torch.full_like(u, -4.0))
    e, w = (c0 + 1) - u, u - c0
    corners = []
    for k in range(8):
        o = (k >> 2, (k >> 1) & 1, k & 1)
        fz, fy, fx = (w[..., a] if o[a] else e[..., a] for a in range(3))
        idx = c0.long() + torch.tensor(o)
        ok = ((idx >= 0) & (idx < torch.tensor(sp))).all(-1)
        corners.append((o, idx, (fx * fy) * fz, ok))
    return inr[..., 0], e, w, corners


def gather_vox(vol, idx, ok):
    """vol (N, C, D, H, W) at the voxel indices idx (N, D, H, W, 3), zero where not ok"""
    n, c, D, H, W = vol.shape
    lin = (idx[..., 0].clamp(0, D - 1) * H + idx[..., 1].clamp(0, H - 1)) * W + idx[..., 2].clamp(0, W - 1)
    vals = torch.gather(vol.reshape(n, c, -1), 2, lin.reshape(n, 1, -1).expand(n, c, -1)).view(n, c, *idx.shape[1:4])
    return torch.where(ok.unsqueeze(1), vals, torch.zeros((), dtype=vol.dtype))


def warp_image32(img, u):
    """warp3d_kernel's image: fmaf(value, weight, out) over the in-volume corners in corner order, in fp32"""
    _, e, w, corners = cell32(u, img.shape[2:])
    out = torch.zeros_like(img)
    for _, idx, wt, ok in corners:
        out = torch.where(ok.unsqueeze(1), fmaf32(gather_vox(img, idx, ok), wt.unsqueeze(1), out), out)
    return out


def warp_label_index(u, sp):
    """the linear voxel index nearest sampling picks (round half to even), -1 where the sample is outside"""
    r = torch.where(in_range(u, sp).unsqueeze(-1), u.round(), torch.full_like(u, -1.0)).long()
    ok = ((r >= 0) & (r < torch.tensor(sp))).all(-1)
    lin = (r[..., 0] * sp[1] + r[..., 1]) * sp[2] + r[..., 2]
    return torch.where(ok, lin, -1)


def warp_grad64(img, gout, u):
    """d loss / d ddf (N, D, H, W, 3) as the fp64 sum of warp3d_bwd_kernel's terms -- value x the two other axes'
    fp32 factors of the corner x the output gradient -- and the sum of their |terms|"""
    inr, e, w, corners = cell32(u, img.shape[2:])
    go = gout.double()
    g = torch.zeros(u.shape, dtype=torch.float64)
    mag = torch.zeros(u.shape, dtype=torch.float64)
    for o, idx, _, ok in corners:
        val = gather_vox(img.double(), idx, ok) * go                      # (N, C, D, H, W)
        f = [(w if o[a] else e)[..., a].double() for a in range(3)]
        for a in range(3):
            b, c = [x for x in range(3) if x != a]
            t = torch.where(ok.unsqueeze(1), val * (f[b] * f[c]).unsqueeze(1), torch.zeros((), dtype=torch.float64))
            t = (t if o[a] else -t).sum(1)
            g[..., a] += t
            mag[..., a] += torch.where(ok.unsqueeze(1), (val * (f[b] * f[c]).unsqueeze(1)).abs(),
                                       torch.zeros((), dtype=torch.float64)).sum(1)
    return g, mag


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
        out = out + gather_vox(img, idx, ok) * w.unsqueeze(1)
    return out


def first_diff(ne, got, want, what):
    if bool(ne.any()):
        idx = tuple(ne.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(ne.sum())} of {ne.numel()} differ; first at {idx}: got "
                             f"{float(got[idx])!r}, want {float(want[idx])!r}")


def assert_bits32(got, want, what):
    """fp32 bit for bit (so -0 != +0 and NaN == NaN of the same payload)"""
    got, want = got.cpu().contiguous(), want.cpu().contiguous()
    first_diff(got.view(torch.int32) != want.view(torch.int32), got, want, what)


def assert_grad_within(got, want, mag, ci, what):
    """each element within (8 ci + 6) u of the sum of its |terms|: 8 ci accumulations, two product roundings per
    term and the two of the final scale by (s - 1) / 2 and 2 / (s - 1); no terms -> exactly zero"""
    got = got.cpu().double()
    bound = (8 * ci + 6) * U32 * mag
    bad = ~((got - want).abs() <= bound)
    first_diff(bad, got, want, what + f" (bound (8 ci + 6) u sum|terms|, ci = {ci})")


# the coordinates of the edge designs along an axis of extent s: the coord_in_range cut-offs (-2, s + 1), the
# volume's faces (-1, 0, s - 1, s), each exactly and at the nearest reachable coordinate on either side
def edge_targets(s):
    return [(t, side) for t in (-2, -1, 0, s - 1, s, s + 1) for side in (0, 1, -1)]


def tie_targets(s):
    return [(k + 0.5, 0) for k in range(-2, s + 1)]


NONFINITE = tuple(torch.tensor([1e38, -1e38, INF, -INF, float("nan")]).tolist())      # fp32 values


def ddf_for(gi, targets, s, span=256):
    """fp32 displacements whose chain coordinate at grid index gi is the target exactly (side 0; the nearest
    reachable one if none is) or the nearest reachable coordinate above (side 1) / below (side -1) it, searched
    among target - gi + k 2^-26 (|gi| + |target| + 1), |k| <= span"""
    t = torch.tensor([x for x, _ in targets], dtype=torch.float64)
    side = torch.tensor([sd for _, sd in targets])
    k = torch.arange(-span, span + 1, dtype=torch.float64)
    q = 2.0 ** -26 * (gi.abs() + t.abs() + 1)
    f = ((t - gi).unsqueeze(-1) + k * q.unsqueeze(-1)).float()
    u = chain_u(gi.unsqueeze(-1), f, s).double()
    tt, sd = t.unsqueeze(-1), side.unsqueeze(-1)
    exact = (u == tt).any(-1, keepdim=True)
    hit = torch.where(sd > 0, u > tt, torch.where(sd < 0, u < tt, (u == tt) | ~exact))
    assert bool(hit.any(-1).all()), "no reachable coordinate on the requested side"
    j = torch.where(hit, (u - tt).abs(), torch.full_like(u, INF)).argmin(-1, keepdim=True)
    return f.gather(-1, j).squeeze(-1)


def design_ddf(kind, n, sp, gen):
    """(N, 3, D, H, W) displacements of the edge, tie and non-finite designs"""
    V = sp[0] * sp[1] * sp[2]
    grid = torch.stack(torch.meshgrid([torch.arange(s) for s in sp], indexing="ij")).reshape(3, -1)
    ddf = torch.zeros((n, 3, V))
    if kind == "nonfinite":
        ddf = torch.randn((n, 3, V), generator=gen) * 2
        j = torch.arange(n * V).view(n, V)
        for a in range(3):
            for v, x in enumerate(NONFINITE):
                m = (j % 4 == 1) & ((j // 4) % 3 == a) & ((j // 12) % len(NONFINITE) == v)
                ddf[:, a][m] = x
        return ddf.view((n, 3) + tuple(sp))
    for a, s in enumerate(sp):
        tg = edge_targets(s) if kind == "edges" else tie_targets(s)
        pick = (torch.arange(n * V) + 7 * a) % len(tg)
        gi = grid[a].repeat(n)
        ddf[:, a] = ddf_for(gi, [tg[i] for i in pick.tolist()], s).view(n, V)
    return ddf.view((n, 3) + tuple(sp))


WARP_CASES = {
    "identity_cubic": dict(n=2, sp=(17, 17, 17), ci=1, cl=3, amp=0.0),      # s - 1 = 16: integer coordinates
    "random_noncubic": dict(n=2, sp=(12, 20, 28), ci=1, cl=3, amp=3.0),
    "far_out_of_volume": dict(n=1, sp=(10, 14, 18), ci=2, cl=1, amp=40.0),
    "half_integers": dict(n=2, sp=(17, 33, 65), ci=1, cl=2, amp="half"),
    "registration_96": dict(n=2, sp=(96, 96, 96), ci=1, cl=3, amp=4.0),
    # extents 2 and 3; every coordinate on a cut-off or a face of the volume, or next to one
    "edges_2x3x5": dict(n=2, sp=(2, 3, 5), ci=3, cl=1, amp="edges"),
    "edges_3x9x17": dict(n=2, sp=(3, 9, 17), ci=2, cl=2, amp="edges"),
    # s - 1 not a power of two: ties at .5 reached through the chain's own roundings
    "ties_7x13x6": dict(n=2, sp=(7, 13, 6), ci=1, cl=1, amp="ties"),
    # +-1e38, +-inf and NaN displacements on one axis of every fourth voxel
    "nonfinite": dict(n=2, sp=(4, 5, 6), ci=2, cl=1, amp="nonfinite"),
}


def warp_inputs(case, seed):
    """ddf, image, and labels that name their voxel: label channel k at linear voxel index v is k V + v + 1"""
    gen = torch.Generator().manual_seed(seed)
    n, sp, ci, cl, amp = case["n"], case["sp"], case["ci"], case["cl"], case["amp"]
    if amp == "half":
        ddf = torch.randint(-8, 9, (n, 3) + sp, generator=gen).float() / 2
    elif isinstance(amp, str):
        ddf = design_ddf(amp, n, sp, gen)
    else:
        ddf = torch.randn((n, 3) + sp, generator=gen) * amp
    img = torch.randn((n, ci) + sp, generator=gen)
    V = sp[0] * sp[1] * sp[2]
    lab = (torch.arange(cl * V).float() + 1).view(1, cl, *sp).expand(n, -1, -1, -1, -1).contiguous()
    return ddf, img, lab


def want_labels(lab, u):
    n, cl = lab.shape[:2]
    idx = warp_label_index(u, lab.shape[2:])
    flat = lab.reshape(n, cl, -1)
    picked = torch.gather(flat, 2, idx.clamp_min(0).reshape(n, 1, -1).expand(n, cl, -1)).view(lab.shape)
    return torch.where((idx >= 0).unsqueeze(1), picked, torch.zeros(()))


# ---- CPU part: the restatements and the designs
def test_fmaf32_rounds_once():
    # (1 + 2^-12)^2 = 1 + 2^-11 + 2^-24 is an fp32 midpoint; an addend of +-2^-80 vanishes in the fp64 sum but decides
    # the one rounding of fmaf
    a = torch.tensor([1 + 2.0 ** -12] * 3)
    c = torch.tensor([2.0 ** -80, -2.0 ** -80, 0.0])
    want = torch.tensor([1 + 2.0 ** -11 + 2.0 ** -23, 1 + 2.0 ** -11, 1 + 2.0 ** -11])
    assert torch.equal(fmaf32(a, a, c), want)
    assert torch.equal((a.double() * a.double() + c.double()).float(), torch.full((3,), 1 + 2.0 ** -11))
    gen = torch.Generator().manual_seed(0)
    x, y, z = (torch.randn(10000, generator=gen) for _ in range(3))
    assert torch.equal(fmaf32(x, y, z), torch.addcmul(z.double(), x.double(), y.double()).float())


@pytest.mark.parametrize("name", ["edges_2x3x5", "edges_3x9x17", "ties_7x13x6", "nonfinite"])
def test_warp_designs_reach_their_coordinates(name):
    case = WARP_CASES[name]
    ddf, _, _ = warp_inputs(case, seed=len(name))
    u, _ = chain_coords(ddf)
    for a, s in enumerate(case["sp"]):
        ua = u[..., a]
        if case["amp"] == "edges":
            # s - 1 is a power of two: every target is reached exactly, and a coordinate next to each
            for t in (-2, -1, 0, s - 1, s, s + 1):
                assert bool((ua == t).any()), (a, t)
                assert bool(((ua > t) & (ua < t + 2.0 ** -16)).any()) and bool(((ua < t) & (ua > t - 2.0 ** -16)).any())
        elif case["amp"] == "ties":
            ties = ua[(ua - ua.floor()) == 0.5]
            assert bool((ties >= 0).any()) and ties.unique().numel() >= s - 1, (a, ties.unique())
        else:
            for x in NONFINITE:
                assert bool(((ddf[:, a] == x) | (torch.isnan(ddf[:, a]) & (x != x))).any())


def test_warp_restatements_agree_and_checkers_reject():
    ddf, img, lab = warp_inputs(WARP_CASES["edges_2x3x5"], seed=3)
    ddf = ddf + torch.randn(ddf.shape, generator=torch.Generator().manual_seed(4)) * 0.3
    u, g = chain_coords(ddf)
    # the restated image is a trilinear sample within the roundoff of eight fmaf and the weights
    img32 = warp_image32(img, u)
    ref = trilinear64(img.double(), u.double(), u.floor().long())
    assert ((img32.double() - ref).abs() <= 16 * U32 * img.abs().max()).all()
    # the label restatement is torch's nearest grid_sample on the CPU; the identity warp returns the inputs
    assert torch.equal(want_labels(lab, u), F.grid_sample(lab, g, align_corners=True, mode="nearest"))
    u0, _ = chain_coords(torch.zeros_like(ddf))
    assert torch.equal(warp_image32(img, u0), img) and torch.equal(want_labels(lab, u0), lab)
    # the gradient's term sum against fp64 autograd of the sampler (which differs by the fp32 factors' roundings)
    gout = torch.randn(img.shape, generator=torch.Generator().manual_seed(5))
    want, mag = warp_grad64(img, gout, u)
    u64 = u.double().requires_grad_(True)
    (trilinear64(img.double(), u64, u.floor().long()) * gout.double()).sum().backward()
    assert ((want - u64.grad).abs() <= 1e-5 * (mag + 1)).all()
    # the checkers see one ulp, a wrong label index and a gradient outside its bound
    bad = img32.clone()
    bad.view(torch.int32)[1, 2, 0, 1, 3] += 1
    with pytest.raises(AssertionError, match=r"\(1, 2, 0, 1, 3\)"):
        assert_bits32(bad, img32, "one ulp")
    wl = want_labels(lab, u)
    moved = wl.clone()
    moved[0, 0, 1, 2, 4] += 1 if moved[0, 0, 1, 2, 4] else 2
    with pytest.raises(AssertionError, match=r"\(0, 0, 1, 2, 4\)"):
        assert_bits32(moved, wl, "label index")
    gb = want.float().clone()
    k = tuple((mag > 0).nonzero()[0].tolist())
    gb[k] += float(20 * 8 * U32 * mag[k])
    with pytest.raises(AssertionError, match="bound"):
        assert_grad_within(gb, want, mag, 3, "gradient")


# ---- GPU part
def guarded32(shape, fill=float("nan")):
    """a view of `shape` in the middle of a NaN-filled fp32 buffer -> (buffer, view)"""
    k = 1
    for x in shape:
        k *= x
    buf = torch.full((k + 2 * GUARD,), fill, device="cuda")
    return buf, buf[GUARD:GUARD + k].view(shape)


def guard_ok(buf):
    return bool(torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[-GUARD:]).all())


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(WARP_CASES))
def test_warp_against_torch(be, name):
    from pytorchdeeplearing_b200 import warp3d
    case = WARP_CASES[name]
    ci = case["ci"]
    ddf, img, lab = warp_inputs(case, seed=len(name))
    u, g = chain_coords(ddf)
    if case["amp"] == "half":
        assert (u - u.floor() == 0.5).any(), "the design puts coordinates exactly on .5"
    field = ddf.permute(0, 2, 3, 4, 1).contiguous()
    # ---- one launch into NaN-filled guarded outputs; the inputs come back unchanged
    dfield, dimg, dlab = field.cuda(), img.cuda(), lab.cuda()
    ib, mimg = guarded32(img.shape)
    lb, mlab = guarded32(lab.shape)
    be.warp3d(dfield, dimg, dlab, mimg, mlab)
    torch.cuda.synchronize()
    assert guard_ok(ib) and guard_ok(lb), "warp3d wrote outside its outputs"
    # ---- nearest labels: the voxel round-half-to-even picks, identical to torch's grid_sample on the GPU
    assert_bits32(mlab, want_labels(lab, u), f"{name} labels")
    assert_bits32(mlab, F.grid_sample(dlab, g.cuda(), align_corners=True, mode="nearest"), f"{name} labels (torch)")
    # ---- trilinear image: bit for bit the fp32 cell, weights and corner-order fmaf chain
    assert_bits32(mimg, warp_image32(img, u), f"{name} image")
    torch_img = F.grid_sample(dimg, g.cuda(), align_corners=True, mode="bilinear")
    fin = torch.isfinite(ddf).all(1).cuda().unsqueeze(1)
    assert (mimg - torch_img)[fin.expand_as(mimg)].abs().max().item() <= 64 * U32 * img.abs().max().item()
    # ---- d loss / d ddf: each element within its own terms' bound of their fp64 sum
    gout = torch.randn(img.shape, generator=torch.Generator().manual_seed(5))
    gb, gddf = guarded32(field.shape)
    be.warp3d_bwd(dfield, dimg, gout.cuda(), None, gddf)
    torch.cuda.synchronize()
    assert guard_ok(gb), "warp3d_bwd wrote outside its output"
    want_g, mag = warp_grad64(img, gout, u)
    assert_grad_within(gddf, want_g, mag, ci, f"{name} ddf gradient")
    # ---- the addend form: + the caller's own gradient on ddf, bit for bit
    add = torch.randn(field.shape, generator=torch.Generator().manual_seed(9)).cuda()
    ab, g1 = guarded32(field.shape)
    be.warp3d_bwd(dfield, dimg, gout.cuda(), add, g1)
    torch.cuda.synchronize()
    assert guard_ok(ab)
    assert_bits32(g1, gddf + add, f"{name} addend form")
    for got, want, what in ((dfield, field, "ddf"), (dimg, img, "image"), (dlab, lab, "label")):
        assert_bits32(got, want, f"{name} input {what} changed")
    # ---- the autograd path (ddf channels-last, as the head writes it) gives the same bits
    ddf_cl = field.cuda().permute(0, 4, 1, 2, 3).requires_grad_(True)
    moved_img, moved_lab = warp3d(dimg, dlab, ddf_cl)
    assert torch.equal(moved_img, mimg) and torch.equal(moved_lab, mlab)
    moved_img.backward(gout.cuda())
    assert torch.equal(ddf_cl.grad.permute(0, 2, 3, 4, 1), gddf)
    if case["amp"] == 0.0:
        assert torch.equal(moved_img.detach().cpu(), img)
    if case["amp"] == "nonfinite":
        # torch's CUDA grid_sample and its autograd at the non-finite samples: every corner outside the volume, so
        # the moved image is 0 and d loss / d ddf is 0 (no 0 * inf from the skipped corners)
        gg = g.cuda().requires_grad_(True)
        F.grid_sample(dimg, gg, align_corners=True, mode="bilinear").backward(gout.cuda())
        sm1 = torch.tensor([s - 1 for s in case["sp"]], dtype=torch.float32, device="cuda")
        torch_g = gg.grad[..., [2, 1, 0]] * (2 / sm1)
        for x in NONFINITE:
            sel = (ddf == x).any(1) if x == x else torch.isnan(ddf).any(1)
            assert bool(sel.any())
            got_i, got_g = mimg.permute(0, 2, 3, 4, 1)[sel.cuda()], gddf[sel.cuda()]
            assert bool((got_i == 0).all()) and bool((got_g == 0).all()), f"ddf = {x}: image or gradient not 0"
            assert torch.equal(torch_img.permute(0, 2, 3, 4, 1)[sel.cuda()], got_i), f"ddf = {x}: torch's image differs"
            assert torch.equal(torch_g[sel.cuda()], got_g), f"ddf = {x}: torch's gradient differs"


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
