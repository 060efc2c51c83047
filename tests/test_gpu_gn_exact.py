"""The GroupNorm apply / backward, bias column-sum and max-pool kernels (csrc/elementwise.cu, csrc/gn_coef.cuh)
against independent references, bit for bit where the operands allow it.

1. Exact operand design.  The kernels take the GroupNorm statistics as an input, so the test chooses them: every
   group's mean is a short dyadic and var + eps = 4^-k, with s = mu m and q = (var + mu^2) m per group (m = cpg vox), so
   that s / m and q / m are exact in fp64.  y and the residual come from {-4 .. 4} 2^-2, the upstream gradient g from
   {-1, 0, 1} 2^-3, gamma and beta are short dyadics, the dropout scale is 0 or 1.25 and eps = 2^-10.  Then A, B of
   the forward and P, Q, R of the backward (from chosen sums) are short dyadics: a last-bit error of the device's
   fp64 rsqrt, or another FMA contraction, rounds back to the same fp32 value unless a B, m2 or R nearly cancels,
   which the design asserts does not happen.  Every per-element result (fmaf(y, A, B), the ReLU, the fp32 sums of
   the branches and the residual, (m ? g P : 0) + fmaf(y, Q, R)) is then a dyadic whose every partial sum is exact
   in fp32, asserted from the operands as sum |terms| < 2^24 q for their common quantum q; the outputs are compared
   bit for bit.  No alphabet value of y makes fmaf(y, A, B) zero.  The reductions (sums of g m, g m y, y per (n, c)
   and the bias column sums) stay below 2^24 quanta, so every fp32 partial in any order is exact and the fp64 sums
   must be bit-equal to the reference.
2. Every form of every kernel at the network shapes on guarded, pitched buffers (Guarded), with the host's launch
   rules restated below so that every path variant (VEC = 1, two- and four-trip loops and their tails, staged and
   shared-atomic reductions, rounded grids, the grid cap, the fused backward, the precomputed-coefficient form) is
   asserted to be reached.
3. One ReLU mask from forward to backward: with realistic data, voxels whose y sits next to the threshold -B/A are
   read back from every forward and every backward form and compared voxel by voxel along the engine's pairings
   (engine.py: conv_gn, act, bwd_layer):
       C <= 512: apply_gn  ->  conv_bwdstats + gn_bwd_apply_gn(sum_y_from_stats) | gn_bwd_fused_gn
                               | gn_bwd_reduce_gn + gn_bwd_apply_gn
       C >  512: gn_finalize + apply  ->  gn_bwd_reduce + gn_bwd_finalize + gn_bwd_apply
4. An fp64 autograd oracle of relu(group_norm(y) s) [+ second branch] [+ residual], no emulated backend code.
5. Max-pool forward and backward against torch.max_pool3d and its autograd, ties included.

The CPU part (design preconditions, path coverage, checker sensitivity) runs everywhere; the GPU part is marked
`gpu`."""
import math

import pytest
import torch
import torch.nn.functional as F

from emu_backend import K3
from pytorchdeeplearing_b200._abi import ACT_LEAKY, ACT_RELU
from test_gpu_conv_exact import Guarded, assert_guards, first_mismatch, assert_bitwise
from test_gpu_conv_exact import C as conv_case, GUARD, IN_FILL, OUT_BITS, conv_geometry

SMS = 132                     # H100 SXM
GROUPS = 8                    # engine.GROUPS
EPS = 2.0 ** -10              # exact design; the realistic parts use engine.GN_EPS = 1e-5
U = 2.0 ** -24                # fp32 unit roundoff
Y_ALPHA = torch.arange(-4, 5, dtype=torch.float64) / 4          # y and the residual
G_ALPHA = torch.arange(-1, 2, dtype=torch.float64) / 8          # upstream gradients
BF, F32 = torch.bfloat16, torch.float32


# ---------------------------------------------------------------------------------------------------------- cases
def E(n, sp, c, dtype=BF, off=8):
    """one elementwise case: n samples of spatial size sp with c channels; off = offset of channel 0 in each pitched
    row (8 keeps every view 16-byte aligned; 9 fails vec_ok and takes the VEC = 1 kernels)"""
    return dict(n=n, sp=sp, c=c, dtype=dtype, off=off)


EW_CASES = {
    # the VNet3d levels
    "vnet96": E(2, (96, 96, 96), 16), "vnet96_f32": E(2, (96, 96, 96), 16, F32),
    "vnet48": E(2, (48, 48, 48), 32), "vnet48_f32": E(2, (48, 48, 48), 32, F32),
    "vnet24": E(2, (24, 24, 24), 64), "vnet24_f32": E(2, (24, 24, 24), 64, F32),
    "vnet12": E(2, (12, 12, 12), 128), "vnet12_f32": E(2, (12, 12, 12), 128, F32),
    "vnet6": E(2, (6, 6, 6), 256), "vnet6_f32": E(2, (6, 6, 6), 256, F32),
    # UNet3d, UNet2d (D = 1)
    "unet128": E(1, (128, 128, 128), 16),
    "unet2d512": E(8, (1, 512, 512), 16), "unet2d256": E(8, (1, 256, 256), 32),
    # ragged voxel counts: tails of the two- and four-trip loops
    "ragged61": E(1, (61, 83, 97), 16), "ragged47": E(2, (48, 48, 47), 32), "ragged47_f32": E(2, (48, 48, 47), 32, F32),
    # many samples: grid.y = 500, one block per sample (the grid cap itself is reached by the large cases)
    "samples500": E(500, (1, 16, 8), 16),
    # channel counts whose vector groups are not a power of two (init_features = 24)
    "c24": E(2, (12, 12, 12), 24), "c24_f32": E(2, (12, 12, 12), 24, F32), "c48": E(2, (12, 12, 12), 48),
    "c96": E(2, (12, 12, 12), 96), "c192": E(2, (6, 6, 6), 192), "c384": E(2, (6, 6, 6), 384),
    # wide layers (init_features = 64): the precomputed-coefficient form
    "c768": E(2, (6, 6, 6), 768), "c1024_f32": E(2, (6, 6, 6), 1024, F32),
    # a base offset that fails vec_ok: VEC = 1
    "vec1": E(2, (10, 12, 14), 16, off=9), "vec1_f32": E(2, (10, 12, 14), 32, F32, off=9),
    "vec1_c24": E(1, (9, 10, 11), 24, off=9),
}


# ---------------------------------------------------------------------------------------------------------- launch rules
# elementwise.cu has no query for the variant a launch takes; these restate its host code.
def vec_width(dtype):
    return 8 if dtype == BF else 4


def vec_ok(cs):
    """vec_ok (elementwise.cu:1011): channels, pitch (C + 16) and base address are multiples of 16 bytes"""
    v = vec_width(cs["dtype"])
    return cs["c"] % v == 0 and (cs["c"] + 16) % v == 0 and cs["off"] % v == 0


def ew_blocks(V, G, N, per_sm=8, sms=SMS):
    """ew_blocks (elementwise.cu:1018) -> (blocks per sample, capped)"""
    want = -(-V * G // 1024)
    cap = -(-sms * per_sm // N)
    capped = want > cap
    want = max(1, min(want, cap))
    if 256 % G:
        want = -(-want // G) * G
    return want, capped


def trip_counts(V, vstep):
    """the numbers of voxels the threads of one sample walk with stride vstep"""
    q, r = divmod(V, vstep)
    return ({q + 1} if r else set()) | {q}


def fused_supported(cs, sms=SMS):
    """ew_gn_bwd_fused_supported (elementwise.cu:1181) and the sample bound of b200seg_gn_bwd_fused_supported"""
    if not vec_ok(cs):
        return False
    G = cs["c"] // vec_width(cs["dtype"])
    return (1 <= G <= 256 and G & (G - 1) == 0 and cs["c"] <= 512 and
            cs["n"] * math.prod(cs["sp"]) * cs["c"] <= 4 << 20 and cs["n"] <= sms)


def reduce_staged(cs, gn_form, groups=GROUPS):
    """staged (elementwise.cu:1126-1130): power-of-two vector groups <= 32 and the staging rows fit in 46 KB"""
    C = cs["c"]
    G = C // (vec_width(cs["dtype"]) if vec_ok(cs) else 1)
    groups = groups if gn_form else 1
    full = (3 * C + 2 * C + 4 * groups) * 8 + 5 * C * 4
    return G & (G - 1) == 0 and G <= 32 and full + 8 * 3 * C * 4 <= 46 * 1024


def ew_variants(cs, groups=GROUPS, act=ACT_RELU):
    """the kernel variants the case reaches (labels "kernel:variant") with `groups` GroupNorm groups and activation
    `act`.  The LeakyReLU tail exists only in the fused-coefficient forms (apply_gn, gn_bwd_apply_gn,
    gn_bwd_reduce_gn, gn_bwd_fused_gn; C <= 512): the precomputed-coefficient forms and colsum reach nothing with it"""
    N, V, C = cs["n"], math.prod(cs["sp"]), cs["c"]
    leaky = act == ACT_LEAKY
    if leaky and C > 512:
        return set()
    vec = vec_width(cs["dtype"]) if vec_ok(cs) else 1
    G = C // vec
    out = set()
    tags = [f"vec{vec}"] + (["round_g"] if 256 % G else [])
    # apply / gn_bwd_apply: 3 CTAs per SM, two-trip loop + tail (elementwise.cu:1103, 1166)
    b, capped = ew_blocks(V, G, N, 3)
    cnt = trip_counts(V, b * 256 // G)
    t = tags + (["cap"] if capped else []) + (["tail"] if any(k % 2 for k in cnt) else [])
    for k in ("apply", "bwd_apply"):
        out |= {f"{k}:{x}" for x in t}
    # gn_bwd_reduce: DEEP four-trip loop for large streams (elementwise.cu:1124)
    deep = V * G >= SMS * 2 * 256 * 8
    b, _ = ew_blocks(V, G, N, 2 if deep else 3)
    cnt = trip_counts(V, b * 256 // G)
    t = tags + ["deep" if deep else "shallow"] + (["tail"] if any(k % 2 for k in cnt) else [])
    if deep and any(k % 4 >= 2 for k in cnt):
        t.append("deep_rem2")
    if not leaky:
        t.append("staged" if reduce_staged(cs, False) else "atomic")
    if C <= 512:
        t.append("gn_staged" if reduce_staged(cs, True, groups) else "gn_atomic")
    out |= {f"reduce:{x}" for x in t}
    if fused_supported(cs):
        out.add("fused:" + ("narrow" if G <= 32 else "wide"))
    if not leaky:
        out |= {f"colsum:{x}" for x in tags}
    if C > 512:
        out.add("coef:wide")
    if groups > 256:
        out.add("coef:groups>256")      # gn_coefs' WIDE group loops take a second trip over the 256 threads
    return out


REQUIRED_VARIANTS = {
    "apply:vec8", "apply:vec4", "apply:vec1", "apply:round_g", "apply:cap", "apply:tail",
    "bwd_apply:vec8", "bwd_apply:vec4", "bwd_apply:vec1", "bwd_apply:round_g", "bwd_apply:tail",
    "reduce:vec8", "reduce:vec4", "reduce:vec1", "reduce:deep", "reduce:shallow", "reduce:deep_rem2", "reduce:tail",
    "reduce:staged", "reduce:atomic", "reduce:gn_staged", "reduce:gn_atomic", "reduce:round_g",
    "fused:narrow", "fused:wide", "colsum:vec8", "colsum:vec4", "colsum:vec1", "colsum:round_g", "coef:wide",
}


def required_variants(act):
    """the labels the cases of activation `act` must reach.  LeakyReLU (InstanceNorm, groups = C; the cases of
    test_gpu_gn_act_warp.py): every label of the fused-coefficient forms that the ReLU form requires, and more than
    256 groups (the ReLU form refuses those)"""
    if act == ACT_RELU:
        return REQUIRED_VARIANTS
    return {v for v in REQUIRED_VARIANTS
            if v.split(":")[0] in ("apply", "bwd_apply", "reduce", "fused")
            and v not in ("reduce:staged", "reduce:atomic")} | {"coef:groups>256"}


# ---------------------------------------------------------------------------------------------------------- design
def quantum(*ts):
    """the largest power of two dividing every entry of the fp64 tensors (1 if all are zero)"""
    v = torch.cat([t.reshape(-1) for t in ts]).double()
    v = v[v != 0]
    if v.numel() == 0:
        return 1.0
    e = 40
    while e > -80 and not bool((torch.frac(v / 2.0 ** e) == 0).all()):
        e -= 1
    return 2.0 ** e


def assert_exact_fp32(bound, q, what):
    """a sum whose |terms| add up to at most `bound`, all multiples of q, is exact in fp32 in any order"""
    assert bound < 2 ** 24 * q, f"{what}: sum |terms| {bound!r} is not below 2^24 quanta ({q!r})"


def per_channel(t, cpg):
    return t.repeat_interleave(cpg, -1)


def gn_branch(gen, N, C, vox, drop=True):
    """gamma, beta, scale, per-group mean / rstd and the per-channel statistics of one exact GroupNorm layer; without
    `drop` the scale is 1 everywhere (a layer without Dropout passes no scale)"""
    cpg = C // GROUPS
    mu = torch.randint(-1, 2, (N, GROUPS), generator=gen).double()
    rs = 2.0 ** torch.randint(0, 2, (N, GROUPS), generator=gen).double()
    gamma = torch.randint(2, 7, (C,), generator=gen).double() / 4 * (torch.randint(0, 2, (C,), generator=gen) * 2 - 1)
    beta = torch.randint(-8, 9, (C,), generator=gen).double() / 16
    scale = torch.where(torch.rand((N, C), generator=gen) < 0.2, 0.0, 1.25).double()
    if not drop:
        scale = torch.ones_like(scale)
    mu_c, rs_c = per_channel(mu, cpg), per_channel(rs, cpg)
    for _ in range(64):           # move beta until no alphabet y sits exactly on a threshold
        A = rs_c * gamma * scale
        B = (beta - mu_c * rs_c * gamma) * scale
        bad = (((Y_ALPHA.view(-1, 1, 1) * A + B) == 0).any(0) & (scale != 0)).any(0)
        if not bool(bad.any()):
            break
        beta = beta + bad.double() / 16
    var = 1.0 / (rs * rs) - EPS
    stats = torch.stack([mu_c * vox, (per_channel(var, cpg) + mu_c * mu_c) * vox], -1)
    return dict(mu=mu, rs=rs, mu_c=mu_c, rs_c=rs_c, gamma=gamma, beta=beta, scale=scale, A=A, B=B, stats=stats)


def bwd_coefs(b, sums, vox):
    """P, Q, R (and m1, m2 per channel) of gn_cta_coefs from the given backward sums, in exact fp64"""
    N, C = b["scale"].shape
    cpg = C // GROUPS
    m = float(cpg * vox)
    s, ga, mu, rs = b["scale"], b["gamma"], b["mu_c"], b["rs_c"]
    d2 = ga * sums[..., 0] * s
    d3 = ga * rs * (sums[..., 1] * s - mu * sums[..., 0] * s)
    m1 = per_channel(d2.view(N, GROUPS, cpg).sum(-1) / m, cpg)
    m2 = per_channel(d3.view(N, GROUPS, cpg).sum(-1) / m, cpg)
    P = rs * ga * s
    Q = -rs * rs * m2
    R = -rs * m1 + rs * rs * mu * m2
    return dict(P=P, Q=Q, R=R, m1=m1, m2=m2, d3=d3)


def param_contribs(b, sums, co, vox, s3):
    """per-sample d beta, d gamma, d bias of param_grads_of_sample / gn_bwd_finalize"""
    s, rs, mu = b["scale"], b["rs_c"], b["mu_c"]
    s1, s2 = sums[..., 0] * s, sums[..., 1] * s
    return dict(dbeta=s1, dgamma=rs * (s2 - mu * s1), dbias=rs * b["gamma"] * s1 + co["Q"] * s3 + co["R"] * vox)


def design(cs, seed=0, drop=True):
    """the exact operands of one case (small per-channel tensors; the big ones are drawn on the device)"""
    gen = torch.Generator().manual_seed(seed)
    N, C, vox = cs["n"], cs["c"], math.prod(cs["sp"])
    cpg, m = C // GROUPS, C // GROUPS * vox
    b1, b2 = gn_branch(gen, N, C, vox, drop), gn_branch(gen, N, C, vox, drop)
    a = torch.randint(-1, 2, (N, C), generator=gen).double() / 16
    bb = torch.randint(-1, 2, (N, C), generator=gen).double() / 16
    for _ in range(64):           # nudge a until neither m2 nor R nearly cancels
        sums = torch.stack([a * m, bb * m, torch.randint(-4, 5, (N, C), generator=gen).double() / 4 * vox], -1)
        co = bwd_coefs(b1, sums, vox)
        t2 = per_channel(co["d3"].abs().view(N, GROUPS, cpg).sum(-1) / m, cpg)
        tr = (b1["rs_c"] * co["m1"]).abs() + (b1["rs_c"] ** 2 * b1["mu_c"] * co["m2"]).abs()
        bad = ((co["m2"].abs() <= 2.0 ** -20 * t2) & (t2 > 0)) | ((co["R"].abs() <= 2.0 ** -20 * tr) & (tr > 0))
        if not bool(bad.any()):
            break
        a = a + (bad & (torch.arange(C) % cpg == 0)).double() / 16
    pc = param_contribs(b1, sums, co, vox, sums[..., 2])
    pc_st = param_contribs(b1, sums, co, vox, b1["stats"][..., 0])
    prefill = {k: torch.randint(-3, 4, (C,), generator=gen).double() * quantum(pc[k], pc_st[k]) for k in pc}
    return dict(b1=b1, b2=b2, sums=sums, co=co, pc=pc, pc_st=pc_st, prefill=prefill, vox=vox, m=m)


def check_design(cs, d):
    """every exactness precondition of the case, from its operands and alphabets"""
    N, V, C = cs["n"], math.prod(cs["sp"]), cs["c"]
    y = Y_ALPHA.view(-1, 1, 1)
    for b in (d["b1"], d["b2"]):
        on = b["scale"] != 0
        z = y * b["A"] + b["B"]
        assert not bool(((z == 0) & on).any()), "an alphabet y sits on a ReLU threshold"
        assert bool(((b["A"] == 0) & (b["B"] == 0) | on).all())
        tb = ((b["beta"] * b["scale"]).abs() + (b["mu_c"] * b["rs_c"] * b["gamma"] * b["scale"]).abs())
        assert bool((b["B"].abs() > 2.0 ** -20 * tb)[on].all()), "B nearly cancels"
        # fmaf(y, A, B) and the ReLU outputs are exact
        assert_exact_fp32(float(z.abs().max()), quantum(y * b["A"], b["B"]), "fmaf(y, A, B)")
    # relu(z1) + relu(z2) + res in fp32, and the bf16 / fp32 store of an exact value
    r1 = (Y_ALPHA.view(-1, 1, 1) * d["b1"]["A"] + d["b1"]["B"]).clamp_min(0)
    r2 = (Y_ALPHA.view(-1, 1, 1) * d["b2"]["A"] + d["b2"]["B"]).clamp_min(0)
    assert_exact_fp32(float(r1.max() + r2.max() + Y_ALPHA.abs().max()), quantum(r1, r2, Y_ALPHA), "apply sum")
    # dy = (m ? g P : 0) + fmaf(y, Q, R)
    co = d["co"]
    gP = G_ALPHA.view(-1, 1, 1) * co["P"]
    yQ = Y_ALPHA.view(-1, 1, 1) * co["Q"]
    bound = float(gP.abs().max() + (yQ + co["R"]).abs().max() + yQ.abs().max() + co["R"].abs().max())
    assert_exact_fp32(bound, quantum(gP, yQ, co["R"]), "dy")
    for k in ("P", "Q", "R"):
        assert_exact_fp32(float(co[k].abs().max()), quantum(co[k]), k)
    # parameter gradients: prefill + per-sample contributions in any order.  d bias = ... + R vox needs the bits of
    # the voxel count on top of R's: with an odd count it may not fit, and is then held to its fp32 rounding bound
    inexact = set()
    for tag, pc in (("", d["pc"]), ("from stats ", d["pc_st"])):
        for k, t in pc.items():
            pre = d["prefill"][k]
            if not float((pre.abs() + t.abs().sum(0)).max()) < 2 ** 24 * quantum(pre, t):
                inexact.add(tag + k)
    assert inexact <= ({"dbias", "from stats dbias"} if d["vox"] % 2 else set()), sorted(inexact)
    # reductions per (n, c): sum |g m| < 2^24 2^-3, sum |g m y| < 2^24 2^-5, sum |y| < 2^24 2^-2; colsum over N V
    assert_exact_fp32(V * 2.0 ** -3, 2.0 ** -3, "sum g m")
    assert_exact_fp32(V * 2.0 ** -3, 2.0 ** -5, "sum g m y")
    assert_exact_fp32(V * 1.0, 2.0 ** -2, "sum y")
    assert_exact_fp32(N * V * 2.0 ** -3 + 3 * 2.0 ** -3, 2.0 ** -3, "colsum")
    # the designed statistics are exact in fp64 and give mean = mu, var + eps = 4^-k
    st = d["b1"]["stats"].view(N, GROUPS, C // GROUPS, 2).sum(2)
    assert torch.equal(st[..., 0] / d["m"], d["b1"]["mu"])
    assert torch.equal(st[..., 1] / d["m"] - d["b1"]["mu"] ** 2 + EPS, 1.0 / d["b1"]["rs"] ** 2)
    return inexact


def check_pgrad(got, pre, terms, exact, what):
    """a parameter gradient: prefill + the per-sample terms, bit for bit when the design makes that exact, otherwise
    within the fp32 rounding of each term and of each addition"""
    want = pre + terms.sum(0)
    if exact:
        assert_equal64(got, want, what)
        return
    bound = (terms.shape[0] + 1) * U * (pre.abs() + terms.abs().sum(0))
    _first_bad((got.double().cpu() - want).abs() > bound, got.double().cpu(), want, bound, what)


# ---------------------------------------------------------------------------------------------------------- checkers
def assert_equal64(got, want, what):
    """fp64 (sums) or fp32 (coefficients, parameter gradients) bit for bit, reporting the first index"""
    got, want = got.cpu(), want.cpu().to(got.dtype)
    ne = got != want
    if bool(ne.any()):
        idx = tuple(ne.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(ne.sum())} of {ne.numel()} differ; first at {idx}: got "
                             f"{float(got[idx])!r}, want {float(want[idx])!r}")


def flat(shape, dtype, fill=0.0):
    """a small tensor in the middle of a NaN-filled buffer -> (buffer, view)"""
    n = math.prod(shape)
    buf = torch.full((2 * GUARD + n,), float("nan"), dtype=dtype, device="cuda")
    v = buf[GUARD:GUARD + n].view(shape)
    if torch.is_tensor(fill):
        v.copy_(fill)
    else:
        v.fill_(fill)
    return buf, v


def assert_flat_guards(buf, what):
    assert bool(torch.cat([buf[:GUARD], buf[-GUARD:]]).isnan().all()), f"{what}: guard band written"


def pitched(shape, dtype, fill=None, off=8, device="cuda"):
    """Guarded with channel 0 at offset `off` of each pitched row (ld = C + 16)"""
    return Guarded(shape, dtype, fill=fill, device=device, off=off)


def reset(gb):
    """back to the all-NaN state of a fresh output buffer"""
    ib, pat = OUT_BITS[gb.dtype]
    gb.buf.view(ib).fill_(pat)


def mask_mismatch(fwd, bwd, what):
    """None, or a message naming the first (n, k, c) threshold voxel whose backward mask differs from the forward"""
    ne = fwd != bwd
    if not bool(ne.any()):
        return None
    idx = tuple(ne.nonzero()[0].tolist())
    return (f"{what}: {int(ne.sum())} of {ne.numel()} threshold voxels disagree with the forward mask; first at "
            f"(n, k, c) = {idx}: forward {bool(fwd[idx])}, backward {bool(bwd[idx])}")


def assert_same_mask(fwd, bwd, what):
    msg = mask_mismatch(fwd, bwd, what)
    assert msg is None, msg


def decode_mask(s1, nbits, shift):
    """per-voxel mask bits from sum g m where threshold voxel k carries g = 2^(shift + k) and every other voxel g = 0"""
    v = (s1.double().cpu() / 2.0 ** shift)
    assert bool((v == v.round()).all()) and bool((v >= 0).all()) and bool((v < 2 ** nbits).all()), "undecodable sum"
    iv = v.long()
    return torch.stack([(iv >> k) & 1 for k in range(nbits)], 1).bool()      # (n, k, c)


# ---------------------------------------------------------------------------------------------------------- CPU part
def test_every_kernel_variant_has_a_case():
    reached = set().union(*(ew_variants(c) for c in EW_CASES.values()))
    assert required_variants(ACT_RELU) <= reached, sorted(required_variants(ACT_RELU) - reached)


@pytest.mark.parametrize("name", sorted(EW_CASES))
def test_design_is_exact(name):
    cs = EW_CASES[name]
    check_design(cs, design(cs))


def test_exact_premise_holds_on_the_cpu():
    """the fp32 evaluation of the kernels' expressions on designed operands equals the fp64 one"""
    cs = EW_CASES["c24"]
    d = design(cs)
    b, co = d["b1"], d["co"]
    gen = torch.Generator().manual_seed(9)
    y = Y_ALPHA[torch.randint(0, 9, (cs["n"], 50, cs["c"]), generator=gen)]
    g = G_ALPHA[torch.randint(0, 3, (cs["n"], 50, cs["c"]), generator=gen)]
    A, B = b["A"].unsqueeze(1), b["B"].unsqueeze(1)
    z64 = y * A + B
    z32 = torch.addcmul(B.float(), y.float(), A.float())
    assert torch.equal(z32.double(), z64)
    P, Q, R = (co[k].unsqueeze(1) for k in "PQR")
    dy64 = torch.where(z64 > 0, g * P, 0.0) + y * Q + R
    dy32 = torch.where(z32 > 0, g.float() * P.float(), 0.0) + torch.addcmul(R.float(), y.float(), Q.float())
    assert torch.equal(dy32.double(), dy64)
    assert_bitwise(dy32.bfloat16(), dy64.float().bfloat16(), "bf16 store")


def test_checker_rejects_one_ulp():
    want = (Y_ALPHA[torch.randint(0, 9, (2, 3, 4, 5, 24))] * 3).float().bfloat16()
    got = want.clone()
    got.view(torch.int16)[1, 0, 2, 4, 23] += 1
    with pytest.raises(AssertionError, match=r"\(1, 0, 2, 4, 23\)"):
        assert_bitwise(got, want, "one ulp")
    s = torch.arange(24, dtype=torch.float64).view(2, 4, 3)
    s2 = s.clone()
    s2.view(torch.int64)[1, 2, 0] += 1
    with pytest.raises(AssertionError, match=r"\(1, 2, 0\)"):
        assert_equal64(s2, s, "one ulp of a sum")


def test_checker_rejects_one_flipped_mask_bit():
    fwd = torch.rand(2, 6, 32, generator=torch.Generator().manual_seed(1)) > 0.5
    assert mask_mismatch(fwd, fwd.clone(), "same") is None
    bwd = fwd.clone()
    bwd[1, 4, 17] = ~bwd[1, 4, 17]
    with pytest.raises(AssertionError, match=r"\(1, 4, 17\)"):
        assert_same_mask(fwd, bwd, "flipped")
    # the sums decode: one voxel more or less in sum g m changes one bit
    s1 = (fwd.long() << torch.arange(6).view(1, 6, 1)).sum(1).double() * 2.0 ** 10
    assert torch.equal(decode_mask(s1, 6, 10), fwd)
    s1[1, 17] += 2.0 ** 14
    with pytest.raises(AssertionError, match=r"\(1, 4, 17\)"):
        assert_same_mask(fwd, decode_mask(s1.abs(), 7, 10)[:, :6], "decoded")


@pytest.mark.parametrize("where", ["before", "gap", "after"])
def test_checker_rejects_a_written_guard(where):
    gb = pitched((2, 2, 3, 4, 24), torch.float32, off=9, device="cpu")
    gb.view.copy_(torch.ones(2, 2, 3, 4, 24))
    assert gb.outside_changed() is None
    pos = {"before": GUARD - 1, "gap": GUARD + gb.ld + 8, "after": gb.buf.numel() - GUARD}[where]
    assert not bool(gb.inside[pos])
    gb.buf[pos] = 0.0
    with pytest.raises(AssertionError, match=f"element {pos}"):
        assert_guards(gb, where)
    reset(gb)
    assert gb.outside_changed() is None


# ---------------------------------------------------------------------------------------------------------- GPU part
@pytest.fixture(scope="module")
def be():
    from pytorchdeeplearing_b200._abi import CudaBackend
    return CudaBackend()


def _gn(b, vox, eps=EPS):
    """the GroupNorm reference tuple of the fused-coefficient entry points"""
    return (b["stats"].cuda(), b["gamma"].float().cuda(), b["beta"].float().cuda(), b["scale"].float().cuda(), vox,
            GROUPS, eps)


def _bc(t):
    """(N, C) -> broadcastable over (N, D, H, W, C)"""
    return t.view(t.shape[0], 1, 1, 1, t.shape[1]).cuda()


def _draw(alpha, shape, gen):
    return alpha.cuda()[torch.randint(0, alpha.numel(), shape, generator=gen, device="cuda")]


def _input(x, dtype, off):
    gb = pitched(tuple(x.shape), dtype, fill=IN_FILL, off=off)
    gb.view.copy_(x.to(dtype))
    return gb


def _check_out(gb, want, what):
    assert_bitwise(gb.view, want.float().to(gb.dtype), what)
    assert_guards(gb, what)
    reset(gb)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(EW_CASES))
def test_gn_exact(be, name):
    cs = EW_CASES[name]
    d = design(cs)
    inexact = check_design(cs, d)
    N, sp, C, dt, off = cs["n"], cs["sp"], cs["c"], cs["dtype"], cs["off"]
    vox, shape = d["vox"], (cs["n"],) + cs["sp"] + (cs["c"],)
    b1, b2, co = d["b1"], d["b2"], d["co"]
    narrow = C <= 512                      # the fused-coefficient forms
    gen = torch.Generator(device="cuda").manual_seed(1)
    y1, y2, res = (_draw(Y_ALPHA, shape, gen) for _ in range(3))
    g = _draw(G_ALPHA, shape, gen)
    gy1, gy2, gres, gg = (_input(t, dt, off) for t in (y1, y2, res, g))
    out = pitched(shape, dt, off=off)
    z1 = y1 * _bc(b1["A"]) + _bc(b1["B"])
    z2 = y2 * _bc(b2["A"]) + _bc(b2["B"])

    # gn_finalize: A, B and mean, rstd of the design, bit for bit
    coefs = []
    for b in (b1, b2):
        cbuf, coef = flat((N, C, 2), F32, float("nan"))
        mbuf, mr = flat((N, GROUPS, 2), F32, float("nan"))
        be.gn_finalize(b["stats"].cuda(), b["gamma"].float().cuda(), b["beta"].float().cuda(), b["scale"].float().cuda(),
                       vox, GROUPS, EPS, coef, mr)
        assert_equal64(coef, torch.stack([b["A"], b["B"]], -1), f"{name} gn_finalize coef")
        assert_equal64(mr, torch.stack([b["mu"], b["rs"]], -1), f"{name} gn_finalize mean / rstd")
        assert_flat_guards(cbuf, "coef")
        assert_flat_guards(mbuf, "mr")
        coefs.append((coef, mr))
    (coef1, mr1), (coef2, _) = coefs

    # forward: one branch, two branches, residual, two branches + residual; both coefficient forms
    for two, resid in ((False, False), (True, False), (False, True), (True, True)):
        want = z1.clamp_min(0)
        if two:
            want = want + z2.clamp_min(0)
        if resid:
            want = want + res
        tag = f"{name} apply{' 2 branches' if two else ''}{' + residual' if resid else ''}"
        be.apply(gy1.view, coef1, gy2.view if two else None, coef2 if two else None, gres.view if resid else None,
                 out.view)
        _check_out(out, want, tag)
        if narrow:
            be.apply_gn(gy1.view, _gn(b1, vox), gy2.view if two else None, _gn(b2, vox) if two else None,
                        gres.view if resid else None, out.view)
            _check_out(out, want, tag + " (fused coefficients)")

    # backward with the designed sums: dy = (m ? g P : 0) + y Q + R, parameter gradients added to a prefilled buffer
    sums = d["sums"].cuda()
    dy = torch.where(z1 > 0, g * _bc(co["P"]), 0.0) + y1 * _bc(co["Q"]) + _bc(co["R"])
    pre = {k: v.float() for k, v in d["prefill"].items()}
    pb = {k: flat((C,), F32, pre[k]) for k in pre}
    c3buf, coef3 = flat((N, C, 3), F32, float("nan"))
    be.gn_bwd_finalize(sums, mr1, b1["gamma"].float().cuda(), b1["scale"].float().cuda(), vox, GROUPS, coef3,
                       pb["dgamma"][1], pb["dbeta"][1], pb["dbias"][1])
    assert_equal64(coef3, torch.stack([co["P"], co["Q"], co["R"]], -1), f"{name} gn_bwd_finalize P, Q, R")
    assert_flat_guards(c3buf, "coef3")
    for k in ("dgamma", "dbeta"):
        check_pgrad(pb[k][1], d["prefill"][k], d["pc"][k], k not in inexact, f"{name} gn_bwd_finalize {k} (+=)")
    # gn_bwd_finalize WRITES the bias gradient (the fused forms accumulate it)
    check_pgrad(pb["dbias"][1], torch.zeros(C, dtype=torch.float64), d["pc"]["dbias"], "dbias" not in inexact,
                f"{name} gn_bwd_finalize dbias")
    for k in pb:
        assert_flat_guards(pb[k][0], f"{name} gn_bwd_finalize {k}")
    be.gn_bwd_apply(gg.view, gy1.view, coef1, coef3, out.view)
    _check_out(out, dy, f"{name} gn_bwd_apply")
    if narrow:
        for from_stats, tag in ((False, ""), (True, "from stats ")):
            pb = {k: flat((C,), F32, pre[k]) for k in pre}
            be.gn_bwd_apply_gn(gg.view, gy1.view, _gn(b1, vox), sums, out.view, pb["dgamma"][1], pb["dbeta"][1],
                               pb["dbias"][1], sum_y_from_stats=from_stats)
            what = f"{name} gn_bwd_apply_gn{' (sum y from stats)' if from_stats else ''}"
            _check_out(out, dy, what)
            for k in pb:
                check_pgrad(pb[k][1], d["prefill"][k], (d["pc_st"] if from_stats else d["pc"])[k],
                            tag + k not in inexact, f"{what} {k} (+=)")
                assert_flat_guards(pb[k][0], f"{what} {k}")

    # reductions: sum g m, sum g m y, sum y per (n, c), bit-exact in fp64
    gm = torch.where(z1 > 0, g, 0.0)
    want_s = torch.stack([gm.sum((1, 2, 3)), (gm * y1).sum((1, 2, 3)), y1.sum((1, 2, 3))], -1)
    forms = [("gn_bwd_reduce", lambda s: be.gn_bwd_reduce(gg.view, gy1.view, coef1, s))]
    if narrow:
        forms.append(("gn_bwd_reduce_gn", lambda s: be.gn_bwd_reduce_gn(gg.view, gy1.view, _gn(b1, vox), s)))
    for what, run in forms:
        sbuf, s = flat((N, C, 3), torch.float64)
        run(s)
        assert_equal64(s, want_s, f"{name} {what}")
        assert_flat_guards(sbuf, what)

    # the fused backward: its sums bit-exact, its dy and parameter gradients equal to gn_bwd_apply_gn on those sums
    assert be.gn_bwd_fused_ok(gg.view, gy1.view, out.view) == fused_supported(cs)
    if fused_supported(cs):
        sbuf, s = flat((N, C, 3), torch.float64)
        counter = torch.zeros(4, dtype=torch.int32, device="cuda")
        pf = {k: flat((C,), F32, 0.0) for k in pre}
        be.gn_bwd_fused_gn(gg.view, gy1.view, _gn(b1, vox), s, counter, out.view, pf["dgamma"][1], pf["dbeta"][1],
                           pf["dbias"][1])
        assert_equal64(s, want_s, f"{name} gn_bwd_fused_gn sums")
        assert_flat_guards(sbuf, "fused sums")
        assert_guards(out, f"{name} gn_bwd_fused_gn")
        dy_f = out.view.clone()
        reset(out)
        pa = {k: flat((C,), F32, 0.0) for k in pre}
        be.gn_bwd_apply_gn(gg.view, gy1.view, _gn(b1, vox), s, out.view, pa["dgamma"][1], pa["dbeta"][1],
                           pa["dbias"][1])
        assert_bitwise(dy_f, out.view, f"{name} gn_bwd_fused_gn dy against gn_bwd_apply_gn on its sums")
        reset(out)
        for k in pf:
            # one fp32 atomic per sample: the order of two additions to zero cannot change the sum
            if N <= 2:
                assert_equal64(pf[k][1], pa[k][1], f"{name} gn_bwd_fused_gn {k}")
            else:
                torch.testing.assert_close(pf[k][1], pa[k][1], rtol=N * U, atol=0)
            assert_flat_guards(pf[k][0], f"fused {k}")

    # bias column sums: out[c] += sum over samples and voxels
    cpre = (torch.arange(C) % 7 - 3).double() / 8
    cbuf, cs_out = flat((C,), F32, cpre.float())
    be.colsum(gg.view, cs_out)
    assert_equal64(cs_out, cpre + g.sum((0, 1, 2, 3)).cpu(), f"{name} colsum (+=)")
    assert_flat_guards(cbuf, "colsum")
    torch.cuda.synchronize()
    for gb, what in ((gy1, "y"), (gy2, "y2"), (gres, "residual"), (gg, "g")):
        assert_guards(gb, f"{name} input {what}")


# ---------------------------------------------------------------------------------------------------------- part 3
NTHR = 6          # threshold voxels per (n, c): the three nearest representable y, twice each
SHIFT = 10        # threshold voxel k carries g = 2^(SHIFT + k); every other voxel g = 0


def M(n, sp, c, dtype=BF):
    return dict(n=n, sp=sp, c=c, dtype=dtype)


MASK_CASES = {
    "vnet96": M(2, (96, 96, 96), 16), "vnet48": M(2, (48, 48, 48), 32), "vnet24": M(2, (24, 24, 24), 64),
    "vnet12": M(2, (12, 12, 12), 128), "c256": M(2, (12, 12, 12), 256), "c24": M(2, (16, 16, 16), 24),
    "c768": M(2, (12, 12, 12), 768),
    "vnet96_f32": M(2, (96, 96, 96), 16, F32), "vnet24_f32": M(2, (24, 24, 24), 64, F32),
    "vnet12_f32": M(2, (12, 12, 12), 128, F32), "c256_f32": M(2, (12, 12, 12), 256, F32),
    "c768_f32": M(2, (12, 12, 12), 768, F32),
}


def _neighbours(t, dtype):
    """the representable values of dtype nearest to t (fp64): round(t) and the values one ulp either side"""
    ib = {BF: torch.int16, F32: torch.int32}[dtype]
    r = t.to(dtype)
    up, dn = r.clone(), r.clone()
    up.view(ib).add_(1)
    dn.view(ib).sub_(1)
    return torch.stack([dn, r, up, dn, r, up], 1).double()                  # (n, NTHR, c)


def realistic_layer(n, sp, c, dtype, seed, eps=1e-5):
    """randn data with its own statistics, gamma / beta near (1, 0), a p = 0.2 dropout scale"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    y = torch.randn((n,) + sp + (c,), generator=gen, device="cuda").to(dtype).double()
    stats = torch.stack([y.sum((1, 2, 3)), (y * y).sum((1, 2, 3))], -1).contiguous()
    gamma = (1 + 0.2 * torch.randn(c, generator=gen, device="cuda")).float()
    beta = (0.3 * torch.randn(c, generator=gen, device="cuda")).float()
    scale = ((torch.rand((n, c), generator=gen, device="cuda") > 0.2).float() / 0.8).float()
    return y, stats, gamma, beta, scale, gen


def ulp32(x):
    """the spacing of fp32 values at |x| (normal range)"""
    return 2.0 ** (torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126))) - 23)


def ref_coefs(stats, gamma, beta, scale, vox, eps):
    """A, B as the kernels form them (fp64, rounded to fp32) and mean, rstd per channel in fp64"""
    n, c = stats.shape[:2]
    cpg = c // GROUPS
    st = stats.view(n, GROUPS, cpg, 2).sum(2)
    m = float(cpg * vox)
    mean = st[..., 0] / m
    var = (st[..., 1] / m - mean * mean).clamp_min(0)
    rstd = 1.0 / torch.sqrt(var + float(torch.tensor(eps, dtype=F32)))       # the kernels widen the fp32 eps
    mu_c, rs_c = per_channel(mean, cpg), per_channel(rstd, cpg)
    g64, s64 = gamma.double(), scale.double()
    A = (rs_c * g64 * s64).float().double()
    B = ((beta.double() - mu_c * rs_c * g64) * s64).float().double()
    return A, B, mu_c, rs_c


def threshold_layer(n, sp, c, dtype, seed, eps=1e-5):
    """realistic_layer with the statistics and beta made design inputs, so that -B/A (A, B rounded to fp32) lies
    within a few fp32 ulps of a value y0 of `dtype`: every sample gets the statistics of sample 0 (the threshold then
    depends on the channel only, the dropout scale cancels in -B/A), and beta is moved, a few of its ulps at a time,
    to the value that brings fmaf(y0, A, B) closest to -1, 0 or +1 ulp(B) (cycling over the channels)"""
    y, stats, gamma, beta, scale, gen = realistic_layer(n, sp, c, dtype, seed, eps)
    stats = stats[:1].expand(n, c, 2).contiguous()
    vox = math.prod(sp)
    _, _, mu_c, rs_c = ref_coefs(stats[:1], gamma, beta, torch.ones((1, c), device="cuda"), vox, eps)
    mu, rs, ga, s = mu_c[0], rs_c[0], gamma.double(), 1.25
    A = (rs * ga * s).float().double()
    t = mu - beta.double() / (rs * ga)
    t = torch.where(t.abs() < 1.0 / 16, t + 0.25, t)              # keep y0 away from zero
    y0 = t.to(dtype).double()
    b0 = (rs * ga * (mu - y0)).float().double()
    k = torch.arange(-8, 9, device="cuda", dtype=torch.float64).view(-1, 1)
    bk = (b0 + k * ulp32(b0)).float().double()                   # (17, c) fp32 candidates
    Bk = ((bk - mu * rs * ga) * s).float().double()
    zk = y0 * A + Bk                                               # exact in fp64
    target = ((torch.arange(c, device="cuda") % 3) - 1).double() * ulp32(Bk[8])
    beta = bk.gather(0, (zk - target).abs().argmin(0, keepdim=True))[0].float()
    return y, stats, gamma, beta, scale, gen


def place_thresholds(y, A, B, dtype, gen):
    """write the values of dtype nearest to -B/A into NTHR voxels per (n, c) of y (in place); -> positions (n, NTHR, c)
    and a g that is 2^(SHIFT + k) at threshold voxel k and 0 elsewhere.  Channels with dropout scale 0 keep y.  The
    value nearest to the threshold must give |fmaf(y0, A, B)| <= 4 ulp(B) (threshold_layer)."""
    n, c = A.shape
    V = y[0, ..., 0].numel()
    on = A != 0
    t = torch.where(on, -B / torch.where(on, A, 1.0), 1.0)
    vals = _neighbours(t, dtype)
    assert bool(torch.isfinite(vals).all()) and bool((vals != 0).all())
    z0 = vals[:, 1] * A + B                                        # exact in fp64
    assert bool((z0.abs() <= 4 * ulp32(B))[on].all()), "a threshold voxel is more than 4 ulp(B) from its threshold"
    base = torch.randint(0, V, (n, 1, c), generator=gen, device="cuda")
    pos = (base + torch.arange(NTHR, device="cuda").view(1, -1, 1) * (V // NTHR)) % V
    yf = y.view(n, V, c)
    g = torch.zeros_like(yf)
    keep = yf.gather(1, pos)
    yf.scatter_(1, pos, torch.where(on.unsqueeze(1), vals, keep))
    g.scatter_(1, pos, (2.0 ** (SHIFT + torch.arange(NTHR, device="cuda"))).view(1, -1, 1).expand(n, NTHR, c).double())
    return pos, g.view(y.shape), on


def _gather(t, pos):
    n, c = t.shape[0], t.shape[-1]
    return t.reshape(n, -1, c).gather(1, pos)


def dy_mask(dy, pos, P):
    """mask of the threshold voxels from dy = (m ? g P : 0) + y Q + R with g >= 2^SHIFT there: |dy| > 2^(SHIFT - 1) |P|"""
    v = _gather(dy.double(), pos).abs()
    thr = 2.0 ** (SHIFT - 1) * P.abs().unsqueeze(1)
    return v > thr


def assert_dy_readable(y, pos, sums, gamma, scale, mu_c, rs_c, on, vox):
    """|y Q + R| < 2^(SHIFT - 2) |P| at the threshold voxels (Q, R in fp64 from the backward sums): dy_mask is
    unambiguous"""
    n, C = mu_c.shape
    cpg, m = C // GROUPS, C // GROUPS * vox
    s = sums.double()
    s1, s2 = s[..., 0] * scale.double(), s[..., 1] * scale.double()
    ga = gamma.double()
    m1 = per_channel((ga * s1).view(n, GROUPS, cpg).sum(-1), cpg) / m
    m2 = per_channel((ga * rs_c * (s2 - mu_c * s1)).view(n, GROUPS, cpg).sum(-1), cpg) / m
    Q, R = -rs_c * rs_c * m2, -rs_c * m1 + rs_c * rs_c * mu_c * m2
    side = (_gather(y, pos) * Q.unsqueeze(1) + R.unsqueeze(1)).abs()
    P = (rs_c * ga * scale.double()).abs().unsqueeze(1)
    ok = (side < 2.0 ** (SHIFT - 2) * P) | ~on.unsqueeze(1)
    assert bool(ok.all()), "y Q + R too large to read the mask from dy"


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MASK_CASES))
def test_relu_mask_forward_equals_backward(be, name):
    cs = MASK_CASES[name]
    n, sp, C, dt = cs["n"], cs["sp"], cs["c"], cs["dtype"]
    vox, eps = math.prod(sp), 1e-5
    y, stats, gamma, beta, scale, gen = threshold_layer(n, sp, C, dt, 11)
    A, B, mu_c, rs_c = ref_coefs(stats, gamma, beta, scale, vox, eps)
    pos, g, on = place_thresholds(y, A, B, dt, gen)
    gy, ggb = _input(y, dt, 8), _input(g, dt, 8)
    gn = (stats, gamma, beta, scale, vox, GROUPS, eps)
    out = pitched(gy.view.shape, dt)
    P = rs_c * gamma.double() * scale.double()

    # forward masks: apply_gn and gn_finalize + apply, bit-identical
    cbuf, coef = flat((n, C, 2), F32, float("nan"))
    mbuf, mr = flat((n, GROUPS, 2), F32, float("nan"))
    be.gn_finalize(stats, gamma, beta, scale, vox, GROUPS, eps, coef, mr)
    be.apply(gy.view, coef, None, None, None, out.view)
    fwd_pre = out.view.clone()
    assert_guards(out, f"{name} apply")
    reset(out)
    be.apply_gn(gy.view, gn, None, None, None, out.view)
    assert_bitwise(out.view, fwd_pre, f"{name} apply_gn against gn_finalize + apply")
    assert_guards(out, f"{name} apply_gn")
    reset(out)
    fwd = (_gather(fwd_pre.double(), pos) > 0) & on.unsqueeze(1)
    assert bool(fwd.any()) and not bool(fwd[on.unsqueeze(1).expand_as(fwd)].all()), "thresholds on one side only"

    def sums_mask(s):
        return decode_mask(s[..., 0], NTHR, SHIFT).to(fwd.device) & on.unsqueeze(1)

    def check(bwd, what):
        assert_same_mask(fwd, bwd & on.unsqueeze(1), f"{name} {what}")

    # precomputed-coefficient backward (C > 512): gn_bwd_reduce + gn_bwd_finalize + gn_bwd_apply
    sbuf, s = flat((n, C, 3), torch.float64)
    be.gn_bwd_reduce(ggb.view, gy.view, coef, s)
    check(sums_mask(s), "gn_bwd_reduce")
    assert_dy_readable(y, pos, s, gamma, scale, mu_c, rs_c, on, vox)
    _, c3 = flat((n, C, 3), F32, float("nan"))
    _, dgm = flat((C,), F32)
    _, dbt = flat((C,), F32)
    _, dbi = flat((C,), F32)
    be.gn_bwd_finalize(s, mr, gamma, scale, vox, GROUPS, c3, dgm, dbt, dbi)
    be.gn_bwd_apply(ggb.view, gy.view, coef, c3, out.view)
    check(dy_mask(out.view, pos, P), "gn_bwd_apply")
    assert_guards(out, f"{name} gn_bwd_apply")
    reset(out)
    if C <= 512:
        sbuf, s = flat((n, C, 3), torch.float64)
        be.gn_bwd_reduce_gn(ggb.view, gy.view, gn, s)
        check(sums_mask(s), "gn_bwd_reduce_gn")
        be.gn_bwd_apply_gn(ggb.view, gy.view, gn, s, out.view, dgm, dbt, dbi)
        check(dy_mask(out.view, pos, P), "gn_bwd_apply_gn")
        reset(out)
        if be.gn_bwd_fused_ok(ggb.view, gy.view, out.view):
            sbuf, s = flat((n, C, 3), torch.float64)
            counter = torch.zeros(4, dtype=torch.int32, device="cuda")
            be.gn_bwd_fused_gn(ggb.view, gy.view, gn, s, counter, out.view, dgm, dbt, dbi)
            check(sums_mask(s), "gn_bwd_fused_gn sums")
            check(dy_mask(out.view, pos, P), "gn_bwd_fused_gn")
            assert_guards(out, f"{name} gn_bwd_fused_gn")
            reset(out)
    torch.cuda.synchronize()


# conv_bwdstats folds the first backward pass into the data-gradient epilogue (HALO3 16/32, HALO_WS 64/128 channels):
# with zero weights its output g is the addend, which carries the threshold design
BWDSTATS_CASES = {
    "halo3_c16": conv_case("HALO3", K3, "dgrad", 3, 2, (20, 24, 16), 16, 32, halo=True),
    "halo3_c32": conv_case("HALO3", K3, "dgrad", 3, 2, (48, 48, 48), 32, 32, halo=True),
    "ws_c64": conv_case("HALO_WS", K3, "dgrad", 3, 2, (24, 24, 24), 64, 64, halo=True),
    "ws_c128": conv_case("HALO_WS", K3, "dgrad", 3, 2, (12, 12, 12), 128, 128, halo=True),
}


def bwdstats_masks(be, cs, seed, nudge=False):
    """the forward mask of apply_gn and the backward masks of conv_bwdstats (decoded from its sums) and of
    gn_bwd_apply_gn(sum_y_from_stats) on its sums, at the threshold voxels.  nudge: the backward gets the beta that
    moves B one fp32 ulp up.  -> (forward, [(what, backward)], channels whose B was nudged)"""
    lk, ci, co, xs, ys, wshape = conv_geometry(cs)
    n, vox, eps = cs["n"], math.prod(ys), 1e-5
    y, stats, gamma, beta, scale, gen = threshold_layer(n, ys, co, BF, seed)
    A, B, mu_c, rs_c = ref_coefs(stats, gamma, beta, scale, vox, eps)
    pos, g, on = place_thresholds(y, A, B, BF, gen)
    gf, ga = _input(y, BF, 8), _input(g, BF, 8)
    gx = _input(torch.randn((n,) + xs + (ci,), generator=gen, device="cuda"), BF, 8)
    gyo = pitched((n,) + ys + (co,), BF)
    gn = (stats, gamma, beta, scale, vox, GROUPS, eps)
    beta_b, moved = (beta_one_ulp_up(stats, gamma, beta, vox, eps) if nudge else
                     (beta, torch.zeros(co, dtype=torch.bool, device="cuda")))
    gn_b = (stats, gamma, beta_b, scale, vox, GROUPS, eps)
    wp = be.pack_weight(torch.zeros(wshape, device="cuda"), cs["kind"], "dgrad", BF, 3, vox=10 ** 9)
    assert be.conv_path(lk, 3, gx.view, wp, gyo.view, ga.view) == cs["path"]
    out = pitched(gf.view.shape, BF)
    be.apply_gn(gf.view, gn, None, None, None, out.view)
    fwd = (_gather(out.view.double(), pos) > 0) & on.unsqueeze(1)
    assert bool(fwd.any()) and not bool(fwd[on.unsqueeze(1).expand_as(fwd)].all()), "thresholds on one side only"
    reset(out)
    sbuf, s = flat((n, co, 3), torch.float64)
    be.conv_bwdstats(lk, 3, gx.view, wp, gyo.view, ga.view, gf.view, gn_b, s)
    assert_bitwise(gyo.view, g.float().bfloat16(), f"{cs['path']} g = addend")
    bwd = [("conv_bwdstats", decode_mask(s[..., 0], NTHR, SHIFT).cuda() & on.unsqueeze(1))]
    assert_dy_readable(y, pos, s, gamma, scale, mu_c, rs_c, on, vox)
    _, dgm = flat((co,), F32)
    _, dbt = flat((co,), F32)
    be.gn_bwd_apply_gn(gyo.view, gf.view, gn_b, s, out.view, dgm, dbt, None, sum_y_from_stats=True)
    P = rs_c * gamma.double() * scale.double()
    bwd.append(("gn_bwd_apply_gn (sum y from stats)", dy_mask(out.view, pos, P) & on.unsqueeze(1)))
    torch.cuda.synchronize()
    for gb, what in ((gyo, "g"), (out, "dy"), (gf, "yfwd"), (ga, "addend"), (gx, "dy in")):
        assert_guards(gb, what)
    assert_flat_guards(sbuf, "sums")
    return fwd, bwd, moved


def beta_one_ulp_up(stats, gamma, beta, vox, eps):
    """-> (beta', moved): per channel the nearest beta' above beta whose B (dropout scale 1.25, the statistics every
    sample shares) is the next fp32 value above B, where a step of beta's own ulps reaches it; moved marks those"""
    c = beta.numel()
    _, B, mu_c, rs_c = ref_coefs(stats[:1], gamma, beta, torch.full((1, c), 1.25, device="cuda"), vox, eps)
    mu, rs, ga, b = mu_c[0], rs_c[0], gamma.double(), beta.double()
    k = torch.arange(1, 33, device="cuda", dtype=torch.float64).view(-1, 1)
    bk = (b + k * ulp32(b)).float().double()
    Bk = ((bk - mu * rs * ga) * 1.25).float().double()
    hit = Bk == torch.nextafter(B[0].float(), torch.full((c,), float("inf"), device="cuda")).double()
    moved = hit.any(0)
    first = hit.double().argmax(0, keepdim=True)
    return torch.where(moved, bk.gather(0, first)[0], b).float(), moved


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(BWDSTATS_CASES))
def test_relu_mask_of_conv_bwdstats(be, name):
    fwd, bwd, _ = bwdstats_masks(be, BWDSTATS_CASES[name], 12)
    for what, mask in bwd:
        assert_same_mask(fwd, mask, f"{name} {what}")


def assert_nudge_seen(fwd, bwd, moved, what):
    """the mask check reports the nudge, and only at threshold voxels of channels whose B was moved"""
    msg = mask_mismatch(fwd, bwd, what)
    assert msg is not None, f"{what}: a B one ulp off was not seen"
    with pytest.raises(AssertionError, match="threshold voxels disagree"):
        assert_same_mask(fwd, bwd, what)
    assert bool(moved[(fwd != bwd).any(1).any(0)].all()), f"{what}: a mask moved in a channel whose B did not"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["halo3_c16", "ws_c128"])
def test_mask_check_sees_a_one_ulp_nudge_of_B_in_conv_bwdstats(be, name):
    """bf16: conv_bwdstats and gn_bwd_apply_gn fed a beta that puts B one fp32 ulp up disagree with the forward"""
    fwd, bwd, moved = bwdstats_masks(be, BWDSTATS_CASES[name], 14, nudge=True)
    assert bool(moved.any())
    for what, mask in bwd:
        assert_nudge_seen(fwd, mask, moved, f"{name} nudged B, {what}")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, BF], ids=["f32", "bf16"])
def test_mask_check_sees_a_one_ulp_nudge_of_B(be, dt):
    """the mask comparison reports the threshold voxels when the backward is fed B one ulp larger"""
    n, sp, C = 2, (12, 12, 12), 128
    vox, eps = math.prod(sp), 1e-5
    y, stats, gamma, beta, scale, gen = threshold_layer(n, sp, C, dt, 13)
    A, B, mu_c, rs_c = ref_coefs(stats, gamma, beta, scale, vox, eps)
    pos, g, on = place_thresholds(y, A, B, dt, gen)
    gy, ggb = _input(y, dt, 8), _input(g, dt, 8)
    out = pitched(gy.view.shape, dt)
    _, coef = flat((n, C, 2), F32, float("nan"))
    _, mr = flat((n, GROUPS, 2), F32, float("nan"))
    be.gn_finalize(stats, gamma, beta, scale, vox, GROUPS, eps, coef, mr)
    be.apply(gy.view, coef, None, None, None, out.view)
    fwd = (_gather(out.view.double(), pos) > 0) & on.unsqueeze(1)
    reset(out)
    nudged = coef.clone()
    nudged[..., 1] = torch.nextafter(coef[..., 1], torch.full_like(coef[..., 1], float("inf")))
    moved = torch.ones(C, dtype=torch.bool, device="cuda")
    _, s = flat((n, C, 3), torch.float64)
    be.gn_bwd_reduce(ggb.view, gy.view, nudged, s)
    bwd = decode_mask(s[..., 0], NTHR, SHIFT).cuda() & on.unsqueeze(1)
    assert_nudge_seen(fwd, bwd, moved, "nudged B, gn_bwd_reduce")
    _, c3 = flat((n, C, 3), F32, float("nan"))
    _, dgm = flat((C,), F32)
    _, dbt = flat((C,), F32)
    be.gn_bwd_finalize(s, mr, gamma, scale, vox, GROUPS, c3, dgm, dbt, None)
    be.gn_bwd_apply(ggb.view, gy.view, nudged, c3, out.view)
    P = rs_c * gamma.double() * scale.double()
    assert_nudge_seen(fwd, dy_mask(out.view, pos, P) & on.unsqueeze(1), moved, "nudged B, gn_bwd_apply")


# ---------------------------------------------------------------------------------------------------------- part 4
ORACLE_CASES = {
    "vnet96": (2, (96, 96, 96), 16), "vnet48": (2, (48, 48, 48), 32), "vnet24": (2, (24, 24, 24), 64),
    "vnet12": (2, (12, 12, 12), 128), "vnet6": (2, (6, 6, 6), 256),
    "vnet24_n1": (1, (24, 24, 24), 64), "vnet12_n5": (5, (12, 12, 12), 128), "c768_n5": (5, (6, 6, 6), 768),
}


def _ncdhw(t):
    return t.permute(0, 4, 1, 2, 3)


def _ndhwc(t):
    return t.permute(0, 2, 3, 4, 1)


def _first_bad(bad, got, want, bound, what):
    if bool(bad.any()):
        idx = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} outside the bound; first at {idx}: got "
                             f"{float(got[idx])!r}, fp64 {float(want[idx])!r}, bound {float(bound[idx]):.3g}")


def chain_len(n, sp, c, dtype):
    """fp32 additions a value passes through into a backward sum: its thread's chain (at most twice that of the
    fewest blocks any of the reduce launches starts from: the fused one trims its grid to the SMs), the warp fold,
    one spare"""
    V, G = math.prod(sp), c // vec_width(dtype)
    b = min(ew_blocks(V, G, n, 2)[0], ew_blocks(V, G, n, 1)[0]) // 2
    return -(-V // max(1, b * 256 // G)) + 6


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ORACLE_CASES))
def test_gn_against_fp64_autograd(be, name):
    n, sp, C = ORACLE_CASES[name]
    dt, vox, eps = BF, math.prod(sp), 1e-5
    cpg, m = C // GROUPS, C // GROUPS * math.prod(sp)
    y, stats, gamma, beta, scale, gen = realistic_layer(n, sp, C, dt, 21)
    y2, stats2, gamma2, beta2, scale2, _ = realistic_layer(n, sp, C, dt, 22)
    res = torch.randn(y.shape, generator=gen, device="cuda").to(dt).double()
    g = torch.randn(y.shape, generator=gen, device="cuda").to(dt).double()
    gy, gy2, gres, ggb = (_input(t, dt, 8) for t in (y, y2, res, g))
    out = pitched(gy.view.shape, dt)
    gn1, gn2 = (stats, gamma, beta, scale, vox, GROUPS, eps), (stats2, gamma2, beta2, scale2, vox, GROUPS, eps)
    narrow = C <= 512

    def exact(yy, st, ga, bb, sc):
        """relu(group_norm(y) s) in fp64 with autograd, and the exact per-channel A, B, mean, rstd"""
        mean = st.view(n, GROUPS, cpg, 2).sum(2)[..., 0] / m
        var = st.view(n, GROUPS, cpg, 2).sum(2)[..., 1] / m - mean * mean
        rstd = 1.0 / torch.sqrt(var + eps)
        mu_c, rs_c = per_channel(mean, cpg), per_channel(rstd, cpg)
        A = rs_c * ga.double() * sc.double()
        B = (bb.double() - mu_c * rs_c * ga.double()) * sc.double()
        return mean, rstd, mu_c, rs_c, A, B

    mean, rstd, mu_c, rs_c, A1, B1 = exact(y, stats, gamma, beta, scale)
    _, _, mu2_c, rs2_c, A2, B2 = exact(y2, stats2, gamma2, beta2, scale2)
    # B* = (beta - mean rstd gamma) s may cancel: its rounding is bounded by the uncancelled terms
    B1t = (beta.double().abs() + (mu_c * rs_c * gamma.double()).abs()) * scale.double()
    B2t = (beta2.double().abs() + (mu2_c * rs2_c * gamma2.double()).abs()) * scale2.double()

    # gn_finalize: coef and mean / rstd within one fp32 ulp of fp64
    _, coef = flat((n, C, 2), F32, float("nan"))
    _, mr = flat((n, GROUPS, 2), F32, float("nan"))
    be.gn_finalize(stats, gamma, beta, scale, vox, GROUPS, eps, coef, mr)
    for got, want, extra, what in ((coef[..., 0], A1, 0.0, "A"), (coef[..., 1], B1, 2.0 ** -50 * B1t, "B"),
                                   (mr[..., 0], mean, 0.0, "mean"), (mr[..., 1], rstd, 0.0, "rstd")):
        ulp = torch.where(want == 0, 2.0 ** -149, 2.0 ** (torch.floor(torch.log2(want.abs().clamp_min(2.0 ** -126))) - 23))
        bound = ulp + extra
        _first_bad((got.double() - want).abs() > bound, got.double(), want, bound, f"{name} gn_finalize {what}")

    # forward: one branch; two branches + residual
    t1 = _ncdhw(y).clone()
    ref1 = _ndhwc(F.relu(F.group_norm(t1, GROUPS, gamma.double(), beta.double(), eps) *
                         scale.double().view(n, C, 1, 1, 1)))
    ref2 = _ndhwc(F.relu(F.group_norm(_ncdhw(y2), GROUPS, gamma2.double(), beta2.double(), eps) *
                         scale2.double().view(n, C, 1, 1, 1)))
    e1 = y.abs() * _bc(2 * U * A1.abs()) + _bc(2 * U * B1t) + U * ref1
    e2 = y2.abs() * _bc(2 * U * A2.abs()) + _bc(2 * U * B2t) + U * ref2
    store = 2.0 ** -8
    for two, want, ez in ((False, ref1, e1), (True, ref1 + ref2 + res, e1 + e2)):
        acc = ref1 + (ref2 + res.abs() if two else 0)
        bound = 1.01 * (ez + 2 * U * acc) + store * want.abs()
        forms = [("apply", lambda: be.apply(gy.view, coef, *((gy2.view, _finalized(be, gn2, n, C)) if two else
                                                              (None, None)), gres.view if two else None, out.view))]
        if narrow:
            forms.append(("apply_gn", lambda: be.apply_gn(gy.view, gn1, gy2.view if two else None, gn2 if two else None,
                                                           gres.view if two else None, out.view)))
        for what, run in forms:
            run()
            got = out.view.double()
            _first_bad((got - want).abs() > bound, got, want, bound,
                       f"{name} {what}{' 2 branches + residual' if two else ''}")
            assert_guards(out, f"{name} {what}")
            reset(out)

    # backward of one branch against autograd: dy, d gamma, d beta, d bias (= sum of dy over voxels)
    yq = _ncdhw(y).clone().requires_grad_(True)
    gq = gamma.double().clone().requires_grad_(True)
    bq = beta.double().clone().requires_grad_(True)
    with torch.enable_grad():
        o = F.relu(F.group_norm(yq, GROUPS, gq, bq, eps) * scale.double().view(n, C, 1, 1, 1))
        o.backward(_ncdhw(g))
    dy_ref = _ndhwc(yq.grad)
    dga_ref, dbe_ref, dbi_ref = gq.grad, bq.grad, dy_ref.sum((0, 1, 2, 3))
    # bounds: fp32 sums (chain of L additions) propagate through m1, m2 into Q, R; voxels whose mask is ambiguous
    # within the z bound (part 3 covers them) contribute their |g| to the sums' bound and are not compared
    L = chain_len(n, sp, C, dt)
    z = y * _bc(A1) + _bc(B1)
    amb = z.abs() <= 1.01 * e1
    gm = torch.where(z > 0, g, 0.0)
    red = (1, 2, 3)
    S1, S2 = gm.sum(red), (gm * y).sum(red)
    dS1 = U * L * g.abs().sum(red) + (g.abs() * amb).sum(red)
    dS2 = U * L * (g * y).abs().sum(red) + ((g * y).abs() * amb).sum(red)
    dS3 = U * L * y.abs().sum(red)
    S3 = y.sum(red)
    s64, ga64 = scale.double(), gamma.double()
    dr, dmu = U * rs_c, U * mu_c.abs()
    t1_ = (ga64 * s64 * S1)
    m1 = per_channel(t1_.view(n, GROUPS, cpg).sum(-1), cpg) / m
    t2_ = ga64 * rs_c * s64 * (S2 - mu_c * S1)
    m2 = per_channel(t2_.view(n, GROUPS, cpg).sum(-1), cpg) / m
    gs = (ga64 * s64).abs()
    dm1 = per_channel((gs * dS1).view(n, GROUPS, cpg).sum(-1), cpg) / m
    dm2 = per_channel((gs * (rs_c * (dS2 + mu_c.abs() * dS1 + dmu * S1.abs()) + dr * (S2 - mu_c * S1).abs()))
                      .view(n, GROUPS, cpg).sum(-1), cpg) / m
    P = rs_c * ga64 * s64
    Q = -rs_c * rs_c * m2
    R = -rs_c * m1 + rs_c * rs_c * mu_c * m2
    dQ = 2 * rs_c * dr * m2.abs() + rs_c * rs_c * dm2 + U * Q.abs()
    dR = (dr * m1.abs() + rs_c * dm1 + 2 * rs_c * dr * (mu_c * m2).abs() + rs_c * rs_c * (dmu * m2.abs() + mu_c.abs() * dm2)
          + U * ((rs_c * m1).abs() + (rs_c * rs_c * mu_c * m2).abs()) + U * R.abs())
    dP = dr * gs + U * P.abs()
    e_dy = (g.abs() * _bc(dP) + y.abs() * _bc(dQ) + _bc(dR) +
            2 * U * (g.abs() * _bc(P.abs()) + (y * _bc(Q)).abs() + _bc(R.abs())))
    bound_dy = 1.01 * e_dy + store * dy_ref.abs()
    Nn = n + 1
    tb = s64 * S1
    tg = rs_c * s64 * (S2 - mu_c * S1)
    tbi = rs_c * ga64 * s64 * S1 + Q * S3 + R * vox
    bd_b = (s64.abs() * dS1).sum(0) + Nn * U * tb.abs().sum(0)
    bd_g = (s64.abs() * (dr * (S2 - mu_c * S1).abs() + rs_c * (dS2 + mu_c.abs() * dS1 + dmu * S1.abs()))).sum(0) \
        + Nn * U * tg.abs().sum(0)
    bd_bi = (gs * (dr * S1.abs() + rs_c * dS1) + dQ * S3.abs() + Q.abs() * dS3 + dR * vox).sum(0) \
        + Nn * U * (rs_c * gs * S1.abs() + (Q * S3).abs() + (R * vox).abs()).sum(0)

    def check_bwd(dy_t, dga, dbe, dbi, what):
        got = dy_t.double()
        _first_bad(((got - dy_ref).abs() > bound_dy) & ~amb, got, dy_ref, bound_dy, f"{name} {what} dy")
        for gv, want, bd, k in ((dga, dga_ref, bd_g, "d gamma"), (dbe, dbe_ref, bd_b, "d beta"),
                                (dbi, dbi_ref, bd_bi, "d bias")):
            bd = 1.01 * bd + 1e-30
            _first_bad((gv.double() - want).abs() > bd, gv.double(), want, bd, f"{name} {what} {k}")

    forms = ["precomputed"] + (["reduce_gn", "fused"] if narrow else [])
    for form in forms:
        pg = {k: flat((C,), F32)[1] for k in ("dgamma", "dbeta", "dbias")}
        _, s = flat((n, C, 3), torch.float64)
        if form == "precomputed":
            be.gn_bwd_reduce(ggb.view, gy.view, coef, s)
            _, c3 = flat((n, C, 3), F32, float("nan"))
            be.gn_bwd_finalize(s, mr, gamma, scale, vox, GROUPS, c3, pg["dgamma"], pg["dbeta"], pg["dbias"])
            be.gn_bwd_apply(ggb.view, gy.view, coef, c3, out.view)
        elif form == "reduce_gn":
            be.gn_bwd_reduce_gn(ggb.view, gy.view, gn1, s)
            be.gn_bwd_apply_gn(ggb.view, gy.view, gn1, s, out.view, pg["dgamma"], pg["dbeta"], pg["dbias"])
        else:
            if not be.gn_bwd_fused_ok(ggb.view, gy.view, out.view):
                continue
            counter = torch.zeros(4, dtype=torch.int32, device="cuda")
            be.gn_bwd_fused_gn(ggb.view, gy.view, gn1, s, counter, out.view, pg["dgamma"], pg["dbeta"], pg["dbias"])
        torch.cuda.synchronize()
        check_bwd(out.view, pg["dgamma"], pg["dbeta"], pg["dbias"], form)
        assert_guards(out, f"{name} {form}")
        reset(out)


def _finalized(be, gn, n, C):
    stats, gamma, beta, scale, vox, groups, eps = gn
    coef = torch.empty((n, C, 2), dtype=F32, device="cuda")
    mr = torch.empty((n, groups, 2), dtype=F32, device="cuda")
    be.gn_finalize(stats, gamma, beta, scale, vox, groups, eps, coef, mr)
    return coef


# ---------------------------------------------------------------------------------------------------------- part 5
POOL_CASES = {
    "vnet96": (3, 2, (96, 96, 96), 16, BF, 8), "unet128": (3, 1, (128, 128, 128), 16, BF, 8),
    "unet64": (3, 1, (64, 64, 64), 32, BF, 8), "unet16": (3, 1, (16, 16, 16), 128, BF, 8),
    "unet2d512": (2, 8, (1, 512, 512), 16, BF, 8), "unet2d64": (2, 8, (1, 64, 64), 128, BF, 8),
    "f32": (3, 2, (16, 24, 32), 32, F32, 8), "vec1": (3, 2, (10, 12, 14), 16, BF, 9),
    "vec1_2d": (2, 3, (1, 30, 46), 24, BF, 9),
}


def pool_input(dims, n, sp, c, gen, device="cuda"):
    """ReLU-like values on a coarse grid (ties at zero and between positive values), 30 % of the windows forced to
    2 .. K equal positive maxima, 5 % all zero"""
    kd = 2 if dims == 3 else 1
    K = 4 * kd
    D, H, W = sp
    x = torch.relu(torch.round(torch.randn((n,) + sp + (c,), generator=gen, device=device) * 2) / 2)
    w = x.view(n, D // kd, kd, H // 2, 2, W // 2, 2, c).permute(0, 1, 3, 5, 7, 2, 4, 6).reshape(-1, K).clone()
    M_ = w.shape[0]
    mx = w.max(-1).values
    top = torch.where(mx > 0, mx, 0.5)
    sel = torch.rand(M_, generator=gen, device=device) < 0.3
    t = torch.randint(2, K + 1, (M_,), generator=gen, device=device)
    rank = torch.rand((M_, K), generator=gen, device=device).argsort(-1).argsort(-1)
    w = torch.where(sel.unsqueeze(1) & (rank < t.unsqueeze(1)), top.unsqueeze(1), w)
    w[torch.rand(M_, generator=gen, device=device) < 0.05] = 0
    x = w.view(n, D // kd, H // 2, W // 2, c, kd, 2, 2).permute(0, 1, 5, 2, 6, 3, 7, 4).reshape(n, D, H, W, c)
    return x.double(), w


def pool_ref(dims, x, go):
    """torch.max_pool3d (2 x 2 [x 2]) of x (N,D,H,W,C) float64 and its autograd for the output gradient go ->
    (pooled, gradient w.r.t. x), both (N,D,H,W,C)"""
    k = (2, 2, 2) if dims == 3 else (1, 2, 2)
    xq = _ncdhw(x).contiguous().requires_grad_(True)
    with torch.enable_grad():
        o = F.max_pool3d(xq, k, k)
        o.backward(_ncdhw(go).contiguous())
    return _ndhwc(o.detach()), _ndhwc(xq.grad)


def test_pool_input_has_every_tie_count():
    for dims in (3, 2):
        sp = (8, 8, 8) if dims == 3 else (1, 16, 16)
        _, w = pool_input(dims, 2, sp, 16, torch.Generator().manual_seed(2), device="cpu")
        mx = w.max(-1, keepdim=True).values
        ties = (w == mx).sum(-1)[mx.squeeze(-1) > 0]
        assert set(range(1, w.shape[1] + 1)) <= set(ties.tolist())
        assert bool((mx == 0).any())


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(POOL_CASES))
def test_pool_exact(be, name):
    dims, n, sp, c, dt, off = POOL_CASES[name]
    k = (2, 2, 2) if dims == 3 else (1, 2, 2)
    gen = torch.Generator(device="cuda").manual_seed(7)
    x, _ = pool_input(dims, n, sp, c, gen)
    osp = (sp[0] // k[0], sp[1] // 2, sp[2] // 2)
    go = torch.randint(-8, 9, (n,) + osp + (c,), generator=gen, device="cuda").double() / 8
    add = torch.randint(-8, 9, (n,) + sp + (c,), generator=gen, device="cuda").double() / 16
    want_o, want_g = pool_ref(dims, x, go)
    gx, ggo, gad = _input(x, dt, off), _input(go, dt, off), _input(add, dt, off)
    out = pitched((n,) + osp + (c,), dt, off=off)
    be.pool_fwd(gx.view, out.view, dims)
    _check_out(out, want_o, f"{name} pool_fwd")
    gxo = pitched((n,) + sp + (c,), dt, off=off)
    for addend in (None, gad):
        be.pool_bwd(gx.view, ggo.view, None if addend is None else addend.view, gxo.view, dims)
        want = want_g + (add if addend is not None else 0)
        _check_out(gxo, want, f"{name} pool_bwd{' + addend' if addend is not None else ''}")
    torch.cuda.synchronize()
    for gb, what in ((gx, "x"), (ggo, "g_out"), (gad, "addend")):
        assert_guards(gb, f"{name} {what}")
