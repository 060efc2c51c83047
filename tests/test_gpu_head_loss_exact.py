"""The segmentation head, the fused losses, the per-step accuracy and the Adam step against independent references
(csrc/small_channels.cu, csrc/elementwise.cu head_probs, csrc/train_aux.cu, csrc/loss.cu).  No emulated backend code.

1. Head, bit for bit.  x in {-4..4} 2^-2, w in {-8..8} 2^-5, bias in {-64..64} 2^-7 and dlogits in {-1, 0, 1} 2^-3:
   every logit, dx, dw and db is a multiple of its quantum q with sum |terms| < 2^24 q (asserted from the operands),
   so every fp32 partial sum in any order is exact and the outputs equal fp64 einsum bit for bit (dx rounded once to
   bf16).  x and dx are pitched, guarded views (Guarded).  probs are held to the documented ulp bounds below.
   head_mask must equal mask_logits of head_fwd's logits, head_probs of the logits must equal head_fwd's probs, and
   the loss pass's accuracy sums must equal metric_partials of those probs; p = 0.5 exactly is "off" and argmax takes
   the first of tied maxima.
2. Loss partial sums against fp64: the integer entries (V, class counts, accuracy counts, BAD) exactly, the float
   sums within (per-term bound + chain bound), where the chain bound is 2^-24 L sum |term| with L the number of fp32
   additions per thread (template kernels) or per block (the generic kernel's shared-memory atomics), read from the
   host's sample_grid below; the sums then continue in fp64.
3. Finalize: value, every lcoef and the two accuracy values within 1 fp32 ulp of an fp64 restatement of
   model/losses.py (oracle/losses.py) and model/metric.py, with lcoef = d loss / d (I, P) by fp64 autograd.
4. Loss backward: at the kernel's own lcoef, per element, within a bound propagated from the same ulp table; end to
   end through the b200 loss modules against fp64 autograd of oracle.losses.
5. Adam: bit for bit against a CPU restatement of the kernel's operation order (fmaf evaluated exactly), and against
   torch.optim.Adam / AdamW on CUDA within 2 ulps.

Per-term bounds use the CUDA C++ Programming Guide, "Mathematical Functions", single-precision table (maximum ulp
error over the full range, without fast math): expf 2, logf 1, log1pf 1, powf 4; x / y and sqrtf are correctly
rounded (the library is built with --use_fast_math=false, which keeps -prec-div and -prec-sqrt).

The CPU part (preconditions, path coverage, checker sensitivity) runs without a GPU; the GPU part is marked `gpu`."""
import math

import numpy as np
import pytest
import torch

from test_gpu_conv_exact import Guarded, assert_guards, first_mismatch, assert_bitwise, GUARD, IN_FILL

SMS = 132                       # H100 SXM
U = 2.0 ** -24                  # fp32 unit roundoff
ULP = 2.0 ** -23                # one ulp relative to a normal fp32 value is at most this
ULP_EXPF, ULP_LOGF, ULP_LOG1PF, ULP_POWF = 2, 1, 1, 4
BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64
DICE, CE, FOCAL = 1, 2, 4
SMOOTH, EPS = 1e-5, 1e-7        # model/losses.py:40-41, model/metric.py:148
GAMMAS = (2.0, 3.0, 0.5, 1.0, 0.0)


# ---------------------------------------------------------------------------------------------------------- launch rules
# The library has no query for these; they restate its host code.
def head_blocks(nv, sms=SMS):
    """head_blocks (small_channels.cu:421) and mask_blocks (train_aux.cu:199)"""
    return max(1, min(-(-nv // 256), sms * 8))


def head_bwd_blocks(nv, sms=SMS):
    """head_bwd_cin (small_channels.cu:464)"""
    return head_blocks(nv, sms) // 2 + 1


def head_variant(nc):
    """the NC template of the head forward / head_mask switch (small_channels.cu:436-445, train_aux.cu:215-224):
    nc = 1..7 by value, 8 through `default:`"""
    assert 1 <= nc <= 8
    return nc


def head_bwd_supported(cin, nc):
    """head_bwd_supported (small_channels.cu:482)"""
    return 1 <= nc <= 4 and cin in (16, 32)


def loss_blocks(nvox, sms=SMS):
    """loss_blocks (loss.cu:616)"""
    return max(1, min(-(-nvox // 1024), sms * 8))


def sample_grid(vox, n, sms=SMS):
    """blocks per sample of sample_grid (loss.cu:625)"""
    return max(1, min(-(-vox // 1024), -(-sms * 4 // n)))


def loss_variant(c, ldt):
    """the kernel loss_partials / loss_bwd launch (loss.cu:644-662, 703-720)"""
    if c == 1:
        return "binary_" + ("f32" if ldt == F32 else "i64")
    return f"multi{c}" if c <= 8 else "generic"


def chain_len(vox, n, c):
    """fp32 additions into one partial sum before it is converted to fp64: per-thread trips in the register kernels,
    the block's voxels in the generic kernel (shared-memory atomics)"""
    trips = -(-vox // (sample_grid(vox, n) * 256))
    return trips * 256 if c > 8 else trips


def adam_launch(n, aligned, sms=SMS):
    """adam_step (train_aux.cu:83-87) -> (n4, blocks)"""
    n4 = n >> 2 if aligned else 0
    blocks = max(1, min(-(-((n // 4) if aligned else n) // 256), sms * 8))
    return n4, blocks


def adam_variants(n, aligned):
    n4, blocks = adam_launch(n, aligned)
    v = {"float4" if n4 else "scalar"}
    if n4 and n % 4:
        v.add(f"tail{n % 4}")
    if (n4 if aligned else n) > blocks * 256:
        v.add("grid_stride")
    return v


# ---------------------------------------------------------------------------------------------------------- cases
def H(n, sp, cin, nc, dtype=BF):
    return dict(n=n, sp=sp, cin=cin, nc=nc, dtype=dtype)


HEAD_FWD = {
    "vnet96": H(2, (96, 96, 96), 16, 2), "vnet96_f32": H(2, (96, 96, 96), 16, 2, F32),
    "unet128": H(1, (128, 128, 128), 16, 1), "unet2d512": H(8, (1, 512, 512), 16, 4),
    "vnet96_c32": H(2, (96, 96, 96), 32, 2),
    **{f"ragged_nc{k}": H(2, (23, 37, 41), 16 if k % 2 else 32, k, BF if k % 3 else F32) for k in range(1, 9)},
    "cap_nc8": H(1, (70, 70, 70), 32, 8, F32),
}
HEAD_BWD = {
    "vnet96": H(2, (96, 96, 96), 16, 2), "vnet96_f32": H(2, (96, 96, 96), 16, 2, F32),
    "unet128": H(1, (128, 128, 128), 16, 1), "unet2d512": H(8, (1, 512, 512), 16, 4),
    "vnet96_c32": H(2, (96, 96, 96), 32, 3),
    **{f"ragged_c{ci}_nc{k}_{'bf16' if dt == BF else 'f32'}": H(2, (23, 37, 41), ci, k, dt)
       for ci in (16, 32) for k in (1, 2, 3, 4) for dt in (BF, F32)},
}


def L(n, sp, c, ldt=torch.int64, gamma=2.0):
    return dict(n=n, sp=sp, c=c, ldt=ldt, gamma=gamma)


_ALLC = [(1, torch.int64), (1, F32), (2, None), (3, None), (4, None), (5, None), (6, None), (7, None), (8, None),
         (9, None), (12, None), (33, None)]
LOSS_CASES = {
    "vnet96_c2": L(2, (96, 96, 96), 2), "vnet96_c1": L(2, (96, 96, 96), 1, gamma=0.0),
    "vnet96_c1_soft": L(2, (96, 96, 96), 1, F32, gamma=0.5), "vnet96_c12": L(2, (96, 96, 96), 12, gamma=1.0),
    "unet128_c1": L(1, (128, 128, 128), 1, gamma=3.0), "unet128_c4": L(1, (128, 128, 128), 4, gamma=0.0),
    "unet2d512_c1": L(8, (1, 512, 512), 1, gamma=2.0), "unet2d512_c5": L(8, (1, 512, 512), 5, gamma=0.5),
    **{f"ragged_c{c}{'_soft' if dt == F32 else ''}": L(2, (33, 41, 37), c, dt or torch.int64,
                                                     GAMMAS[i % len(GAMMAS)]) for i, (c, dt) in enumerate(_ALLC)},
    **{f"classifier_c{c}": L(600, (1, 1, 1), c, gamma=g) for c, g in ((1, 2.0), (2, 0.0), (9, 3.0), (33, 0.5))},
    **{f"bigbatch_c{c}": L(600, (1, 16, 256), c, gamma=g) for c, g in ((1, 1.0), (2, 2.0), (33, 0.0))},
}
for _c, _g in ((3, 0.0), (8, 0.0), (9, 0.0), (2, 3.0), (4, 0.5), (1, 0.5)):
    LOSS_CASES[f"gamma_c{_c}_{_g}"] = L(2, (9, 17, 19), _c, gamma=_g)

ADAM_CASES = {       # n, element offset of every slice (0: 16-byte aligned)
    "float4": (4096, 0), "tail1": (4097, 0), "tail2": (4098, 0), "tail3": (4099, 0),
    "unaligned": (1001, 1), "unaligned_short": (3, 3),
    "grid_stride": (SMS * 8 * 256 * 4 * 2 + 5, 0), "grid_stride_unaligned": (SMS * 8 * 256 * 2 + 77, 2),
}


# ---------------------------------------------------------------------------------------------------------- head operands
QX, QW, QB, QG = 2.0 ** -2, 2.0 ** -5, 2.0 ** -7, 2.0 ** -3


def head_operands(cs, seed, device):
    g = torch.Generator(device=device).manual_seed(seed)
    n, sp, cin, nc = cs["n"], cs["sp"], cs["cin"], cs["nc"]
    x = torch.randint(-4, 5, (n,) + sp + (cin,), generator=g, device=device).to(F64) * QX
    w = torch.randint(-8, 9, (nc, cin), generator=g, device=device).to(F64) * QW
    b = torch.randint(-64, 65, (nc,), generator=g, device=device).to(F64) * QB
    return x, w, b


def head_fwd_bound(cin):
    """sum |terms| of one logit from the operand ranges, in quanta QX QW = 2^-7 = QB"""
    return (cin * 1.0 * 0.25 + 0.5) / QB


def head_bwd_bound(nv, cin, nc):
    """dw: nv |dl| |x| <= nv 2^-3 in quanta 2^-5 (plus |dw0| <= 2 2^-1); db: nv 2^-3 + 8 in quanta 2^-3"""
    return (nv * QG * 1.0 + 1.0) / (QG * QX), (nv * QG + 8.0) / QG


def prob_bounds(z, nc):
    """fp64 probabilities of fp64 logits z [..., nc] and the relative bound of the kernels' expressions:
    sigmoid 1/(1 + expf(-z)): expf, one addition, one division; softmax expf(z - mx) / sum: z - mx is exact for the
    grid logits, sum of nc values rounded nc - 1 times, one division (inv = 1/s) and one product."""
    if nc == 1:
        return torch.sigmoid(z), ULP_EXPF * ULP + 2 * U
    return torch.softmax(z, -1), 2 * ULP_EXPF * ULP + (nc + 1) * U


def check_probs(probs, z, nc, what):
    want, rel = prob_bounds(z, nc)
    err = (probs.double() - want).abs()
    tol = want * rel * (1 + 1e-6)
    bad = err > tol
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} probabilities outside the bound; first at {i}: got "
                             f"{float(probs[i])!r}, fp64 {float(want[i])!r}, bound {float(tol[i]):.3g}")


# ---------------------------------------------------------------------------------------------------------- loss reference
def loss_logits(cs, seed, device):
    """full-mantissa logits (N, ..., C) fp32 and labels, with planted confident voxels (1 - pt rounds to 0 in fp32),
    planted tied top-2 logits at C = 2, and labels -1, C and 255 at C > 1; no probability other than an exact tie
    within 1e-5 of the 0.5 threshold"""
    g = torch.Generator(device=device).manual_seed(seed)
    n, sp, c = cs["n"], cs["sp"], cs["c"]
    shape = (n,) + sp
    z = torch.randn(shape + (c,), generator=g, device=device, dtype=F64) * 3
    if cs["ldt"] == F32:
        t = torch.rand(shape, generator=g, device=device, dtype=F64).float()
        t[torch.rand(shape, generator=g, device=device) < 0.3] = 0.0
        t[torch.rand(shape, generator=g, device=device) < 0.3] = 1.0
    else:
        t = torch.randint(0, max(c, 2), shape, generator=g, device=device)
    conf = torch.rand(shape, generator=g, device=device) < 0.05
    if c == 1:
        z[..., 0] = torch.where(conf & (t == 0), torch.full_like(z[..., 0], -20.0), z[..., 0])
        zz = z[..., 0]
        z[..., 0] = torch.where(zz.abs() < 1e-4, torch.where(zz < 0, -1e-4, 1e-4), zz)
    else:
        oh = torch.nn.functional.one_hot(t, c).bool()
        z = torch.where(conf[..., None], torch.where(oh, 12.0, -12.0), z)
        if c == 2:
            tie = torch.rand(shape, generator=g, device=device) < 0.01
            z[..., 1] = torch.where(tie, z[..., 0], z[..., 1])
        for _ in range(3):              # raise the first near class of each such voxel (at C = 2 both are near)
            p = torch.softmax(z.float().double(), -1)
            near = ((p - 0.5).abs() < 1e-5) & (p != 0.5)
            if not bool(near.any()):
                break
            first = torch.nn.functional.one_hot(near.to(torch.uint8).argmax(-1), c).to(F64)
            z = z + first * near.any(-1, keepdim=True).to(F64) * 1e-3
        p = torch.softmax(z.float().double(), -1)
        assert not bool((((p - 0.5).abs() < 1e-5) & (p != 0.5)).any())
        flat = t.view(-1)
        for k, bad in enumerate((-1, c, 255)):
            flat[(k * 7919 + 13) % flat.numel()] = bad
    return z.float(), t


def _sums(v, dims):
    return v.sum(dims)


def loss_reference(z, t, gamma, alpha_f=0.25):
    """fp64 partial sums of loss_partials from the fp32 logits z (N, ..., C) and labels t, with per-element error
    bounds of the kernel's fp32 expressions.  -> dict(part, part_tol (per-term bounds + sum |term|, i.e. the inputs of
    the chain bound), metric, metric_tol (soft targets only), voxel-wise tensors for the backward)"""
    n, c = z.shape[0], z.shape[-1]
    zf = z.reshape(n, -1, c).double()
    vox = zf.shape[1]
    out = dict(vox=vox)
    if c == 1:
        zz, tt = zf[..., 0], t.reshape(n, -1).double()
        p = torch.sigmoid(zz)
        ep = p * (ULP_EXPF * ULP + 2 * U)
        e = torch.exp(-zz.abs())
        sp = torch.log1p(e)
        mzt = zz.clamp_min(0) - zz * tt
        b = mzt + sp
        eb = U * (zz * tt).abs() + U * mzt.abs() + e * ULP_EXPF * ULP + ULP_LOG1PF * ULP * sp + U * b.abs()
        pt = torch.exp(-b)
        ept = pt * (ULP_EXPF * ULP + eb)
        om = 1 - pt
        eom = ept + U * om
        f = alpha_f * om ** gamma * b
        hi = alpha_f * (om + eom) ** gamma * (b + eb) * (1 + ULP_POWF * ULP) * (1 + U) ** 2
        lo = alpha_f * (om - eom).clamp_min(0) ** gamma * (b - eb).clamp_min(0) * (1 - ULP_POWF * ULP) * (1 - U) ** 2
        ef = torch.maximum(hi - f, f - lo)
        terms = [p * tt, p, tt, b, f]
        errs = [ep * tt, ep, torch.zeros_like(p), eb, ef]
        out["part"] = torch.stack([v.sum() for v in terms] + [torch.tensor(float(n * vox), dtype=F64, device=z.device)])
        out["abs"] = torch.stack([v.abs().sum() for v in terms] + [torch.zeros((), dtype=F64, device=z.device)])
        out["err"] = torch.stack([v.sum() for v in errs] + [torch.zeros((), dtype=F64, device=z.device)])
        on = (p > 0.5).double()
        out["metric"] = torch.stack([(on * tt).sum(1), on.sum(1), tt.sum(1)], -1)[:, None, :]
        out.update(p=p, ep=ep, b=b, eb=eb, t=tt, z=zz)
        return out
    tl = t.reshape(n, -1)
    valid = (tl >= 0) & (tl < c)
    ti = tl.clamp(0, c - 1)
    oh = torch.nn.functional.one_hot(ti, c).double() * valid[..., None]
    mx = zf.max(-1, keepdim=True).values
    d = zf - mx
    rel_e = ULP_EXPF * ULP + U * d.abs()
    s = torch.exp(d).sum(-1, keepdim=True)
    eps_s = rel_e.max(-1, keepdim=True).values + (c - 1) * U
    p = torch.softmax(zf, -1)
    rel_p = rel_e + eps_s + 2 * U
    lse = mx + torch.log(s)
    zt = zf.gather(-1, ti[..., None])
    nll = (lse - zt)[..., 0]
    enll = (eps_s * (1 + 1e-6) + ULP_LOGF * ULP * torch.log(s).abs() + U * lse.abs() + U * nll[..., None].abs())[..., 0]
    pt = torch.exp(-nll)
    ept = pt * (ULP_EXPF * ULP + enll)
    om = 1 - pt
    eom = ept + U * om
    f = om ** gamma * nll
    hi = (om + eom) ** gamma * (nll + enll) * (1 + ULP_POWF * ULP) * (1 + U)
    lo = (om - eom).clamp_min(0) ** gamma * (nll - enll).clamp_min(0) * (1 - ULP_POWF * ULP) * (1 - U)
    ef = torch.maximum(hi - f, f - lo)
    vd = valid.double()
    pv = p * vd[..., None]
    I, P, Cn = (pv * oh).sum((0, 1)), pv.sum((0, 1)), oh.sum((0, 1))
    eI, eP = (p * rel_p * oh).sum((0, 1)), (p * rel_p * vd[..., None]).sum((0, 1))
    zero = torch.zeros((), dtype=F64, device=z.device)
    out["part"] = torch.cat([I, P, Cn, torch.stack([(nll * vd).sum(), (f * vd).sum(),
                                                    torch.tensor(float(n * vox), dtype=F64, device=z.device),
                                                    (~valid).sum().double()])])
    out["abs"] = torch.cat([I, P, torch.zeros_like(Cn), torch.stack([(nll.abs() * vd).sum(), (f * vd).sum(), zero,
                                                                     zero])])
    out["err"] = torch.cat([eI, eP, torch.zeros_like(Cn), torch.stack([(enll * vd).sum(), (ef * vd).sum(), zero,
                                                                       zero])])
    on = (p > 0.5).double() * vd[..., None]
    out["metric"] = torch.stack([(on * oh).sum(1), on.sum(1), oh.sum(1)], -1)
    out.update(p=p, rel_p=rel_p, nll=nll, enll=enll, oh=oh, valid=valid, t=ti)
    return out


def integer_slots(c, soft):
    """indices of part that hold exact integers: binary V (and T for int labels); multi class counts, V, BAD"""
    if c == 1:
        return [5] if soft else [2, 5]
    return list(range(2 * c, 3 * c)) + [3 * c + 2, 3 * c + 3]


def check_partials(part, metric, ref, c, chain, soft, what):
    """integer entries exact, float entries within err + gamma_L sum |term| (+ fp64 noise)"""
    want, tol = ref["part"], ref["err"] + (chain * U / (1 - chain * U)) * (ref["abs"] + ref["err"])
    tol = tol * (1 + 1e-6) + 1e-12 * ref["abs"]
    got = part[:want.numel()].double()
    ints = integer_slots(c, soft)
    for i in range(want.numel()):
        if i in ints:
            assert float(got[i]) == float(want[i]), f"{what}: part[{i}] = {float(got[i])!r}, want {float(want[i])!r}"
        else:
            assert abs(float(got[i]) - float(want[i])) <= float(tol[i]), \
                f"{what}: part[{i}] = {float(got[i])!r}, fp64 {float(want[i])!r}, bound {float(tol[i]):.3g}"
    if metric is not None:
        if soft:      # on-counts exact; sums of soft targets within the chain bound
            assert torch.equal(metric[..., 1], ref["metric"][..., 1]), f"{what}: accuracy counts differ"
            mt = ref["metric"][..., [0, 2]]
            assert bool(((metric[..., [0, 2]] - mt).abs() <= chain * 2 * U * mt + 1e-12).all()), f"{what}: metric"
        else:
            ne = metric != ref["metric"]
            if bool(ne.any()):
                i = tuple(ne.nonzero()[0].tolist())
                raise AssertionError(f"{what}: accuracy sum (n, c, k) = {i} is {float(metric[i])!r}, "
                                     f"want {float(ref['metric'][i])!r}")


# ---------------------------------------------------------------------------------------------------------- finalize reference
def finalize_reference(part, c, terms, alpha, gamma, alpha_f):
    """fp64 restatement of model/losses.py (oracle/losses.py: binary_dice / bce / focal, multi_dice / ce / focal) as a
    function of the partial sums; lcoef = d loss / d I and d loss / d P by autograd, then 1/V, (alpha_f)/V, gamma"""
    part = [float(v) for v in part]
    if c == 1:
        I = torch.tensor(part[0], dtype=F64, requires_grad=True)
        P = torch.tensor(part[1], dtype=F64, requires_grad=True)
        T, sb, sf, V = part[2], part[3], part[4], part[5]
        val = torch.zeros((), dtype=F64)
        if terms & DICE:
            val = val + 1.0 - (2.0 * I + SMOOTH) / (P + T + SMOOTH).clamp_min(EPS)
        if terms & CE:
            val = val + sb / V
        if terms & FOCAL:
            val = val + sf / V
        a, b = torch.autograd.grad(val, (I, P)) if terms & DICE else (0.0, 0.0)
        lc = [float(a), float(b), 1.0 / V if terms & CE else 0.0, alpha_f / V if terms & FOCAL else 0.0, gamma]
        return float(val.detach()), lc
    I = torch.tensor(part[:c], dtype=F64, requires_grad=True)
    P = torch.tensor(part[c:2 * c], dtype=F64, requires_grad=True)
    Cn = torch.tensor(part[2 * c:3 * c], dtype=F64)
    snll, sfoc, V, bad = part[3 * c:3 * c + 4]
    present = (Cn > 0).double()
    val = torch.zeros((), dtype=F64)
    if terms & DICE:
        d = ((2.0 * I + SMOOTH) / (Cn + P + SMOOTH)).clamp_min(EPS)
        val = val + (-d * present * torch.as_tensor(alpha, dtype=F64)).sum() / present.sum()
    if terms & CE:
        val = val + snll / V
    if terms & FOCAL:
        val = val + sfoc / V
    if terms & DICE:
        a, b = torch.autograd.grad(val, (I, P))
    else:
        a = b = torch.zeros(c, dtype=F64)
    lc = a.tolist() + b.tolist() + [1.0 / V if terms & CE else 0.0, 1.0 / V if terms & FOCAL else 0.0, gamma]
    return (float("nan") if bad > 0 else float(val.detach())), lc


def metric_reference(metric):
    """model/metric.py dice_coeff / iou_coeff (C == 1), multiclass_dice_coeff and its iou analogue (classes 1..C-1)"""
    m = metric.double()
    dice = (2 * m[..., 0] + SMOOTH) / (m[..., 1] + m[..., 2] + SMOOTH)
    iou = (m[..., 0] + SMOOTH) / (m[..., 1] + m[..., 2] - m[..., 0] + SMOOTH)
    c0 = 0 if m.shape[1] == 1 else 1
    return float(dice[:, c0:].mean(0).mean()), float(iou[:, c0:].mean(0).mean())


def within_ulp(got, want, k=1):
    """|got - want| <= k fp32 ulps of want (NaN only against NaN)"""
    if math.isnan(want):
        return math.isnan(got)
    return abs(got - want) <= k * float(np.spacing(np.float32(abs(want)))) + 1e-45


# ---------------------------------------------------------------------------------------------------------- backward reference
def focal_factor64(ce, gamma):
    """d/dce of (1 - pt)^gamma ce with pt = exp(-ce), in fp64; the om = 0 limits of focal_factor (loss.cu)"""
    pt = torch.exp(-ce)
    om = 1 - pt
    return _ff(om, pt, ce, gamma)


def _ff(om, pt, ce, gamma):
    pos = om > 0
    oms = torch.where(pos, om, torch.ones_like(om))
    f = oms ** gamma + gamma * oms ** (gamma - 1) * pt * ce
    lim = torch.full_like(om, 1.0 if gamma == 0 else 0.0) if gamma != 1 else pt * ce
    return torch.where(pos, f, lim)


def focal_factor_err(ce, ece, gamma):
    """bound on |focal_factor(fp32 ce~) - focal_factor64(ce)| for |ce~ - ce| <= ece: every factor of the closed form
    is monotone in om, pt and ce, so the extremes lie at the corners of their error intervals (om~ is 0 or at least
    2^-24; om~ = 0 takes the limit branch), plus the pow / product roundings"""
    pt = torch.exp(-ce)
    ept = pt * (ULP_EXPF * ULP + ece)
    om = 1 - pt
    eom = ept + U * om
    f0 = _ff(om, pt, ce, gamma)
    lo_om = (om - eom).clamp_min(2.0 ** -24)
    worst = torch.zeros_like(ce)
    for o in (lo_om, om + eom):
        for q in (pt - ept, (pt + ept).clamp_max(1.0)):
            for cc in ((ce - ece).clamp_min(0), ce + ece):
                worst = torch.maximum(worst, (_ff(o, q, cc, gamma) - f0).abs())
    can_zero = (om - eom) < 2.0 ** -24
    lim = torch.full_like(om, 1.0 if gamma == 0 else 0.0) if gamma != 1 else (pt + ept) * (ce + ece)
    worst = torch.where(can_zero, torch.maximum(worst, (lim - f0).abs()), worst)
    return worst + (2 * ULP_POWF * ULP + 5 * U) * (f0.abs() + worst)


def bwd_reference(ref, lc, c, gamma, gs, dlcoef=0.0):
    """fp64 d loss / d logits of the closed forms of loss_bwd at coefficients lc, and a per-element bound of the
    kernel's fp32 evaluation; dlcoef: relative uncertainty of lc itself (end to end)"""
    dev = ref["p"].device
    if c == 1:
        a, b, cs, fs = lc[:4]
        p, ep, t, bce, eb = ref["p"], ref["ep"], ref["t"], ref["b"], ref["eb"]
        q, eq = 1 - p, ep + U * (1 - p)
        A = t * a + b
        t1 = A * p * q
        e1 = A.abs() * (ep * q + p * eq) + (t * a).abs() * 2 * U * p * q + 3 * U * t1.abs()
        F = focal_factor64(bce, gamma)
        eF = focal_factor_err(bce, eb, gamma)
        pmt = p - t
        epmt = ep + U * pmt.abs()
        t2 = cs * pmt
        e2 = abs(cs) * epmt + U * t2.abs()
        t3 = fs * F * pmt
        e3 = abs(fs) * (eF * pmt.abs() + F * epmt) + 2 * U * t3.abs()
        g = t1 + t2 + t3
        mag = t1.abs() + t2.abs() + t3.abs()
        err = gs * (e1 + e2 + e3 + 2 * U * mag) + U * abs(gs * g)
        err = err + dlcoef * gs * mag
        return (g * gs)[..., None], (err * 1.01)[..., None]
    a = torch.tensor(lc[:c], dtype=F64, device=dev)
    b = torch.tensor(lc[c:2 * c], dtype=F64, device=dev)
    cs, fs = lc[2 * c], lc[2 * c + 1]
    p, rel_p, oh, nll, enll = ref["p"], ref["rel_p"], ref["oh"], ref["nll"], ref["enll"]
    ep = p * rel_p
    o = oh * a + b
    dot = (o * p).sum(-1, keepdim=True)
    edot = (o.abs() * ep).sum(-1, keepdim=True) + (c + 1) * U * (o.abs() * p).sum(-1, keepdim=True)
    omd = o - dot
    eomd = U * o.abs() + edot + U * omd.abs()
    t1 = p * omd
    e1 = ep * omd.abs() + p * eomd + U * t1.abs()
    F = focal_factor64(nll, gamma)[..., None]
    eF = focal_factor_err(nll, enll, gamma)[..., None]
    k = cs + fs * F
    ek = abs(fs) * eF + U * abs(fs) * F + U * k.abs()
    pmo = p - oh
    t2 = k * pmo
    e2 = ek * pmo.abs() + k.abs() * (ep + U * pmo.abs()) + U * t2.abs()
    g = t1 + t2
    mag = p * (o.abs() + (o.abs() * p).sum(-1, keepdim=True)) + k.abs() * pmo.abs()
    err = gs * (e1 + e2 + U * (t1.abs() + t2.abs())) + U * (g * gs).abs() + dlcoef * gs * mag
    return g * gs, err * 1.01


def check_dz(dz, want, tol, what, mask=None):
    bad = (dz.double() - want).abs() > tol
    if mask is not None:
        bad = bad & mask
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} gradients outside the bound; first at {i}: "
                             f"got {float(dz[i])!r}, fp64 {float(want[i])!r}, bound {float(tol[i]):.3g}")


# ---------------------------------------------------------------------------------------------------------- Adam restatement
def fmaf(a, b, c):
    """fp32 fmaf(a, b, c), correctly rounded: a b is exact in fp64, the fp64 sum is made round-to-odd from its
    TwoSum error, and one rounding of a round-to-odd value with 53 >= 24 + 2 bits to fp32 is correct"""
    a, b, c = (np.asarray(v, dtype=np.float32).astype(np.float64) for v in (a, b, c))
    prod = a * b
    s = prod + c
    bb = s - prod
    err = (prod - (s - bb)) + (c - bb)
    fix = (err != 0) & ((s.view(np.int64) & 1) == 0)
    s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def adam_tick_ref(state, lr, beta1, beta2):
    st = state.copy()
    t = float(state[0]) + 1.0
    st[0] = np.float32(t)
    st[1] = np.float32(lr / (1.0 - beta1 ** t))
    st[2] = np.float32(math.sqrt(1.0 - beta2 ** t))
    return st


def adam_step_ref(p, g, m, v, state, lr, beta1, beta2, eps, wd, decoupled, gs=None, fp32_constants=False):
    """adam_step_kernel (train_aux.cu) in its operation order.  fp32_constants: the constants as the library computed
    them before they were rounded from double (1.f - beta, 1.f - lr * wd in fp32)"""
    f = np.float32
    step_size, bc2s = f(state[1]), f(state[2])
    if fp32_constants:
        w1, w2, decay = f(1) - f(beta1), f(1) - f(beta2), f(1) - f(lr) * f(wd)
    else:
        w1, w2, decay = f(1.0 - beta1), f(1.0 - beta2), f(1.0 - lr * wd)
    gg = g * f(1.0 if gs is None else gs)
    if decoupled:
        p = p * decay
    else:
        gg = fmaf(f(wd), p, gg)
    m = fmaf(gg - m, w1, m)
    v = fmaf(v, f(beta2), (w2 * gg) * gg)
    denom = np.sqrt(v) / bc2s + f(eps)
    p = fmaf(-step_size, m / denom, p)
    return p, m, v


def ulp_dist(got, want, floor=0.0):
    """|got - want| in fp32 ulps of max(|want|, floor)"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = np.spacing(np.maximum(np.abs(want), floor).astype(np.float32)).astype(np.float64)
    return np.abs(got - want) / scale


def adam_state(n, seed):
    r = np.random.default_rng(seed)
    p = (r.standard_normal(n) * 0.1).astype(np.float32)
    m = (r.standard_normal(n) * 1e-3).astype(np.float32)
    v = (r.random(n) * 1e-5).astype(np.float32)
    return p, m, v, r


def torch_adam(kind, p, g, m, v, t0, lr, wd, device, foreach):
    """one torch.optim step from the state (p, m, v, step t0)"""
    P = torch.nn.Parameter(torch.from_numpy(p.copy()).to(device))
    P.grad = torch.from_numpy(g.copy()).to(device)
    cls = torch.optim.AdamW if kind == "AdamW" else torch.optim.Adam
    opt = cls([P], lr=lr, weight_decay=wd, foreach=foreach)
    opt.state[P] = dict(step=torch.tensor(float(t0)), exp_avg=torch.from_numpy(m.copy()).to(device),
                        exp_avg_sq=torch.from_numpy(v.copy()).to(device))
    opt.step()
    st = opt.state[P]
    return P.detach().cpu().numpy(), st["exp_avg"].cpu().numpy(), st["exp_avg_sq"].cpu().numpy()


# ---------------------------------------------------------------------------------------------------------- CPU part
def test_every_variant_has_a_case():
    assert {head_variant(c["nc"]) for c in HEAD_FWD.values()} == set(range(1, 9))
    assert {(c["nc"], c["cin"], c["dtype"]) for c in HEAD_BWD.values()} >= \
        {(k, ci, dt) for k in range(1, 5) for ci in (16, 32) for dt in (BF, F32)}
    assert any(c["n"] * math.prod(c["sp"]) > SMS * 8 * 256 for c in HEAD_FWD.values())        # grid cap
    assert any(c["n"] * math.prod(c["sp"]) % 256 for c in HEAD_FWD.values())                  # tail block
    assert any(head_bwd_blocks(c["n"] * math.prod(c["sp"])) == SMS * 4 + 1 for c in HEAD_BWD.values())
    got = {loss_variant(c["c"], c["ldt"]) for c in LOSS_CASES.values()}
    assert got == {"binary_f32", "binary_i64", "generic"} | {f"multi{k}" for k in range(2, 9)}
    assert {c["c"] for c in LOSS_CASES.values()} >= {1, 2, 3, 4, 5, 8, 9, 12, 33}
    grids = [(sample_grid(math.prod(c["sp"]), c["n"]), -(-math.prod(c["sp"]) // 1024)) for c in LOSS_CASES.values()]
    assert any(per < want for per, want in grids)                       # capped at the SM budget
    assert any(per == 1 and want > 1 for per, want in grids)           # one block per sample
    assert any(per == want > 1 for per, want in grids)                 # uncapped
    for c in LOSS_CASES.values():
        assert loss_blocks(c["n"] * math.prod(c["sp"])) >= 1
    assert {c["gamma"] for c in LOSS_CASES.values()} == set(GAMMAS)
    for kernels in ((1,), range(2, 9), range(9, 1025)):      # every gamma (2 has its own branch) in every family
        assert {c["gamma"] for c in LOSS_CASES.values() if c["c"] in kernels} == set(GAMMAS)
    variants = set().union(*(adam_variants(n, off == 0) for n, off in ADAM_CASES.values()))
    assert variants == {"float4", "scalar", "tail1", "tail2", "tail3", "grid_stride"}


def test_head_bwd_support_rule():
    for ci in (4, 8, 12, 16, 24, 32, 48, 64):
        for k in range(0, 10):
            assert head_bwd_supported(ci, k) == (1 <= k <= 4 and ci in (16, 32))


@pytest.mark.parametrize("name", sorted(HEAD_FWD))
def test_head_fwd_sums_are_exact(name):
    cs = HEAD_FWD[name]
    assert head_fwd_bound(cs["cin"]) < 2 ** 24


@pytest.mark.parametrize("name", sorted(HEAD_BWD))
def test_head_bwd_sums_are_exact(name):
    cs = HEAD_BWD[name]
    bw, bb = head_bwd_bound(cs["n"] * math.prod(cs["sp"]), cs["cin"], cs["nc"])
    assert bw < 2 ** 24 and bb < 2 ** 24


def test_exact_premise_holds_on_the_cpu():
    cs = H(2, (3, 5, 7), 32, 3)
    x, w, b = head_operands(cs, 0, "cpu")
    z64 = torch.einsum("...k,ck->...c", x, w) + b
    z32 = torch.einsum("...k,ck->...c", x.float(), w.float()) + b.float()
    assert torch.equal(z32.double(), z64)


def test_probability_bound_holds_for_fp32_evaluation():
    """the CPU's fp32 sigmoid / softmax (its own expf) stay inside the bound the GPU test uses"""
    z = torch.linspace(-12, 12, 4001, dtype=F64).reshape(-1, 1)
    z = torch.round(z / QB) * QB
    check_probs(1 / (1 + torch.exp(-z.float())), z, 1, "sigmoid")
    z4 = torch.cat([z, -z, z / 2, z * 0], -1)
    e = torch.exp(z4.float() - z4.float().max(-1, keepdim=True).values)
    check_probs(e * (1 / e.sum(-1, keepdim=True)), z4, 4, "softmax")


@pytest.mark.parametrize("c,soft", [(1, False), (1, True), (3, False), (12, False)])
def test_loss_reference_bounds_hold_for_fp32_evaluation(c, soft):
    """an fp32 evaluation of the kernels' expressions on the CPU stays within the reference bounds"""
    cs = L(2, (3, 11, 13), c, F32 if soft else torch.int64, gamma=0.5)
    z, t = loss_logits(cs, 1, "cpu")
    ref = loss_reference(z, t, cs["gamma"])
    n = z.shape[0]
    zf = z.reshape(n, -1, c)
    if c == 1:
        zz, tt = zf[..., 0], t.reshape(n, -1).float()
        p = 1 / (1 + torch.exp(-zz))
        b = zz.clamp_min(0) - zz * tt + torch.log1p(torch.exp(-zz.abs()))
        f = 0.25 * torch.pow(1 - torch.exp(-b), cs["gamma"]) * b
        got = torch.stack([(p * tt).double().sum(), p.double().sum(), tt.double().sum(), b.double().sum(),
                           f.double().sum(), torch.tensor(float(zz.numel()), dtype=F64)])
    else:
        tl = t.reshape(n, -1)
        ok = (tl >= 0) & (tl < c)
        mx = zf.max(-1, keepdim=True).values
        e = torch.exp(zf - mx)
        s = e.sum(-1, keepdim=True)
        p = e * (1 / s)
        nll = (mx + torch.log(s) - zf.gather(-1, tl.clamp(0, c - 1)[..., None]))[..., 0]
        f = torch.pow(1 - torch.exp(-nll), cs["gamma"]) * nll
        oh = torch.nn.functional.one_hot(tl.clamp(0, c - 1), c).double() * ok[..., None]
        pv = p.double() * ok[..., None]
        got = torch.cat([(pv * oh).sum((0, 1)), pv.sum((0, 1)), oh.sum((0, 1)),
                         torch.stack([(nll.double() * ok).sum(), (f.double() * ok).sum(),
                                      torch.tensor(float(tl.numel()), dtype=F64), (~ok).sum().double()])])
    check_partials(got, None, ref, c, 1, soft, "cpu fp32")


def test_checkers_reject_swapped_classes_and_a_bad_count():
    cs = L(2, (4, 9, 11), 4, gamma=2.0)
    z, t = loss_logits(cs, 2, "cpu")
    ref = loss_reference(z, t, 2.0)
    part = ref["part"].clone()
    check_partials(part, ref["metric"].clone(), ref, 4, 1, False, "exact")
    swapped = part.clone()
    swapped[[4, 5]] = part[[5, 4]]                     # P of classes 0 and 1
    with pytest.raises(AssertionError, match=r"part\[4\]"):
        check_partials(swapped, None, ref, 4, 1, False, "swapped")
    zs = z.clone()
    zs[..., [0, 1]] = z[..., [1, 0]]                   # two class channels of the logits
    with pytest.raises(AssertionError):
        check_partials(loss_reference(zs, t, 2.0)["part"], None, ref, 4, 1, False, "swapped logits")
    bad = part.clone()
    bad[3 * 4 + 3] += 1
    with pytest.raises(AssertionError, match=r"part\[15\]"):
        check_partials(bad, None, ref, 4, 1, False, "BAD + 1")
    assert float(part[15]) == 3.0                      # labels -1, C and 255
    m = ref["metric"].clone()
    m[1, 2, 1] += 1
    with pytest.raises(AssertionError, match="accuracy"):
        check_partials(part, m, ref, 4, 1, False, "metric + 1")


def test_checker_rejects_one_ulp_of_a_logit_and_a_probability():
    z = (torch.arange(-40, 40, dtype=F64) * QB).reshape(4, 5, 4)
    got = z.float()
    got.view(torch.int32)[1, 2, 3] += 1
    with pytest.raises(AssertionError, match=r"\(1, 2, 3\)"):
        assert_bitwise(got, z.float(), "one ulp")
    p = torch.softmax(z, -1).float()
    p.view(torch.int32)[2, 1, 0] += 16                 # 16 ulps: the bound is 4 ulps + 5 u of p
    with pytest.raises(AssertionError, match="probabilities"):
        check_probs(p, z, 4, "probs")


def test_checker_rejects_a_rewritten_guard():
    gb = Guarded((1, 2, 3, 4, 16), F32)
    gb.view.copy_(torch.ones(1, 2, 3, 4, 16))
    pos = GUARD + gb.ld + 30
    assert not bool(gb.inside[pos])
    gb.buf.view(torch.int32)[pos] = 0
    with pytest.raises(AssertionError, match=f"element {pos}"):
        assert_guards(gb, "dx")


def test_focal_factor_limit_at_gamma_zero():
    """at om = 0 the derivative of (1 - pt)^0 ce is 1; the bound tells 1 from the former 0"""
    ce = torch.tensor([1e-11, 2e-9, 1e-3], dtype=F64)
    for gamma in GAMMAS:
        f = focal_factor64(ce, gamma)
        err = focal_factor_err(ce, ce * 4 * U, gamma)
        assert bool((err < 0.5).all())
        if gamma == 0:
            assert torch.equal(f, torch.ones(3, dtype=F64))
            assert bool(((f - 0).abs() > err).all())        # a kernel returning 0 there is rejected


@pytest.mark.parametrize("c,terms", [(1, t) for t in range(1, 8)] + [(3, t) for t in range(1, 8)])
def test_finalize_reference_matches_the_closed_form(c, terms):
    """the autograd lcoef of the restatement equal the closed forms of loss_finalize_kernel (loss.cu:289-336)"""
    part = [30.5, 80.25, 40.0, 50.5, 7.25, 1000.0, 0.0] if c == 1 else \
        [20.0, 5.0, 0.0, 70.0, 30.0, 10.0, 40.0, 0.0, 2000.0, 600.0, 80.0, 1000.0, 0.0]
    val, lc = finalize_reference(part, c, terms, [1.0, 0.5, 2.0][:c], 2.0, 0.25)
    if c == 1 and terms & DICE:
        den = part[1] + part[2] + SMOOTH
        assert math.isclose(lc[0], -2 / den, rel_tol=1e-14)
        assert math.isclose(lc[1], (2 * part[0] + SMOOTH) / den ** 2, rel_tol=1e-14)
    if c == 3 and terms & DICE:
        assert lc[2] == 0 and lc[5] == 0                    # the clamped class (draw < eps) has no gradient
        assert lc[1] == 0 and lc[4] == 0                    # nor has the absent class
        assert lc[0] < 0 < lc[3]
    assert math.isfinite(val)


def test_adam_restatement_matches_torch_cpu_and_the_fp32_constants_do_not():
    """the restatement with torch's constant rounding stays within 2 ulps of CPU torch.optim.AdamW after one step
    from zero moments; with the former fp32 constants exp_avg_sq is off by about 111 ulps and exp_avg by 3"""
    p, _, _, r = adam_state(4096, 5)
    g = (r.standard_normal(4096) * 1e-2).astype(np.float32)
    m0, v0 = np.zeros_like(p), np.zeros_like(p)
    st = adam_tick_ref(np.zeros(4, np.float32), 1e-3, 0.9, 0.999)
    tp, tm, tv = torch_adam("AdamW", p, g, m0, v0, 0, 1e-3, 1e-2, "cpu", False)
    new = adam_step_ref(p, g, m0, v0, st, 1e-3, 0.9, 0.999, 1e-8, 1e-2, True)
    old = adam_step_ref(p, g, m0, v0, st, 1e-3, 0.9, 0.999, 1e-8, 1e-2, True, fp32_constants=True)
    assert ulp_dist(new[1], tm).max() <= 2 and ulp_dist(new[2], tv).max() <= 2
    assert ulp_dist(new[0], tp, 0.05).max() <= 2
    assert np.median(ulp_dist(old[2], tv)) > 100 and np.median(ulp_dist(old[1], tm)) >= 2


def test_fmaf_restatement_rounds_once():
    # 1 + 2^-24 + 2^-60: one rounding goes up, fp64 rounding then fp32 rounding would tie to even (down)
    a, b, c = np.float32(1 + 2 ** -23), np.float32(1 + 2 ** -23), np.float32(-(2 ** -23))
    want = np.float32(1 + 2 ** -23)          # (1 + 2^-23)^2 - 2^-23 = 1 + 2^-23 + 2^-46 -> 1 + 2^-23
    assert fmaf(a, b, c) == want
    x = np.float32(1 + 2 ** -12)
    y = np.float32(1 + 2 ** -12)
    z = np.float32(-(2 ** -11) * (1 + 2 ** -13))
    # x y + z = 1 + 2^-24 - 2^-24 ... exact value 1 + 2^-24 + 2^-24 * (1 - 2^-1)... checked against Fraction
    from fractions import Fraction
    for u, v, w in ((a, b, c), (x, y, z), (np.float32(3.0), np.float32(1 / 3), np.float32(-1.0))):
        exact = Fraction(float(u)) * Fraction(float(v)) + Fraction(float(w))
        got = fmaf(u, v, w)
        lo = np.float32(float(exact))
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        best = min(cands, key=lambda q: (abs(Fraction(float(q)) - exact), int(np.float32(q).view(np.int32)) & 1))
        assert got == best


# ---------------------------------------------------------------------------------------------------------- GPU part
@pytest.fixture(scope="module")
def be():
    from pytorchdeeplearing_b200._abi import CudaBackend
    return CudaBackend()


def _nan(shape, dtype=F32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(HEAD_FWD))
def test_head_fwd_exact(be, name):
    cs = HEAD_FWD[name]
    n, sp, cin, nc, dt = cs["n"], cs["sp"], cs["cin"], cs["nc"], cs["dtype"]
    x, w, b = head_operands(cs, 11, "cuda")
    assert float((x.abs() @ w.abs().T).max() + b.abs().max()) < 2 ** 24 * QB
    gx = Guarded((n,) + sp + (cin,), dt, fill=IN_FILL, device="cuda")
    gx.view.copy_(x.to(dt))
    logits, probs = _nan((n,) + sp + (nc,)), _nan((n,) + sp + (nc,))
    assert be.head_fwd(gx.view, w.float().contiguous(), b.float(), logits, probs)
    want = torch.einsum("...k,ck->...c", x, w) + b
    assert_bitwise(logits, want.float(), f"{name}: logits")
    check_probs(probs, want, nc, f"{name}: probs")
    assert_guards(gx, f"{name}: x")
    p2 = _nan(probs.shape)
    be.head_probs(logits, p2)
    assert_bitwise(p2, probs, f"{name}: head_probs(logits) vs head_fwd probs")
    lg2 = _nan(logits.shape)
    assert be.head_fwd(gx.view, w.float().contiguous(), None, lg2, None)          # no bias, no probs
    assert_bitwise(lg2, (want - b).float(), f"{name}: logits without bias")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(HEAD_BWD))
def test_head_bwd_exact(be, name):
    cs = HEAD_BWD[name]
    n, sp, cin, nc, dt = cs["n"], cs["sp"], cs["cin"], cs["nc"], cs["dtype"]
    assert be.lib.b200seg_head_bwd_supported(cin, nc) == 1
    x, w, _ = head_operands(cs, 12, "cuda")
    g = torch.Generator(device="cuda").manual_seed(13)
    dl = torch.randint(-1, 2, (n,) + sp + (nc,), generator=g, device="cuda").to(F64) * QG
    dw0 = torch.randint(-16, 17, (nc, cin), generator=g, device="cuda").to(F64) * (QG * QX)
    db0 = torch.randint(-64, 65, (nc,), generator=g, device="cuda").to(F64) * QG
    nv = n * math.prod(sp)
    xs, dls = x.reshape(nv, cin), dl.reshape(nv, nc)
    assert float((dls.abs().T @ xs.abs() + dw0.abs()).max()) < 2 ** 24 * QG * QX
    assert float(dls.abs().sum(0).max() + db0.abs().max()) < 2 ** 24 * QG
    gx = Guarded((n,) + sp + (cin,), dt, fill=IN_FILL, device="cuda")
    gx.view.copy_(x.to(dt))
    gdx = Guarded((n,) + sp + (cin,), dt, device="cuda")
    dw, db = dw0.float().contiguous(), db0.float().contiguous()
    assert be.head_bwd(gx.view, dl.float().contiguous(), w.float().contiguous(), gdx.view, dw, db)
    # + 0.0: the kernel's sums start from +0, so a sum of products that are all -0 is +0
    assert_bitwise(gdx.view, (torch.einsum("...c,ck->...k", dl, w) + 0.0).float().to(dt), f"{name}: dx")
    assert_bitwise(dw, (dw0 + dls.T @ xs).float(), f"{name}: dw")
    assert_bitwise(db, (db0 + dls.sum(0)).float(), f"{name}: db")
    assert_guards(gx, f"{name}: x")
    assert_guards(gdx, f"{name}: dx")


@pytest.mark.gpu
def test_head_bwd_supported_matches_the_library(be):
    for ci in (4, 8, 16, 24, 32, 64):
        for k in range(0, 10):
            assert bool(be.lib.b200seg_head_bwd_supported(ci, k)) == head_bwd_supported(ci, k), (ci, k)


@pytest.mark.gpu
@pytest.mark.parametrize("nc", range(1, 9))
@pytest.mark.parametrize("dt", [BF, F32], ids=["bf16", "f32"])
def test_head_mask_and_probs_are_one_expression(be, nc, dt):
    """full-mantissa operands: head_mask = mask_logits(head_fwd logits), head_probs(logits) = head_fwd probs, and
    the loss pass's accuracy sums = metric_partials(probs)"""
    n, sp, cin = 1, (70, 70, 70), 32
    g = torch.Generator(device="cuda").manual_seed(nc)
    x = torch.randn((n,) + sp + (cin,), generator=g, device="cuda").to(dt)
    w = torch.randn(nc, cin, generator=g, device="cuda") * 0.3
    b = torch.randn(nc, generator=g, device="cuda") * 0.1
    logits, probs = _nan((n,) + sp + (nc,)), _nan((n,) + sp + (nc,))
    be.head_fwd(x, w, b, logits, probs)
    mask = torch.full((n,) + sp, 77, dtype=torch.uint8, device="cuda")
    mask2 = mask.clone()
    assert be.head_mask(x, w, b, mask, 0.5)
    be.mask_logits(logits, 0.5, mask2)
    assert torch.equal(mask, mask2), f"nc={nc}: head_mask differs from mask_logits in {int((mask != mask2).sum())}"
    want = ((probs[..., 0] > 0.5) * 255).to(torch.uint8) if nc == 1 else logits.argmax(-1).to(torch.uint8)
    assert torch.equal(mask, want)
    p2 = _nan(probs.shape)
    be.head_probs(logits, p2)
    assert_bitwise(p2, probs, "head_probs")
    labels = torch.randint(0, max(nc, 2), (n,) + sp, generator=g, device="cuda")
    part = torch.zeros(be.part_size(nc), dtype=F64, device="cuda")
    m1 = torch.zeros(n, nc, 3, dtype=F64, device="cuda")
    m2 = torch.zeros_like(m1)
    be.loss_partials(logits, labels, 2.0, 0.25, part, m1)
    be.metric_partials(probs, labels, 0.5, m2)
    assert torch.equal(m1, m2)


@pytest.mark.gpu
def test_head_thresholds_and_ties(be):
    """z = 0 gives p = 0.5 exactly and mask 0 (nc = 1); tied maxima take the first index (nc = 4); tied top-2 logits
    at nc = 2 give p = 0.5 exactly, mask 0 and no 'on' voxel in either accuracy sum"""
    n, sp, cin = 2, (20, 24, 28), 16
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randint(-4, 5, (n,) + sp + (cin,), generator=g, device="cuda").float() * QX
    # nc = 1: w[0][0] = 0.25, bias 0.25 and x row (-1, 0, ..., 0) at planted voxels: z = 0
    w1 = torch.randint(-8, 9, (1, cin), generator=g, device="cuda").float() * QW
    w1[0, 0] = 0.25
    plant = torch.rand((n,) + sp, generator=g, device="cuda") < 0.1
    x1 = torch.where(plant[..., None], torch.zeros_like(x), x)
    x1[..., 0] = torch.where(plant, -1.0, x1[..., 0])
    b1 = torch.tensor([0.25], device="cuda")
    z, p = _nan((n,) + sp + (1,)), _nan((n,) + sp + (1,))
    be.head_fwd(x1, w1, b1, z, p)
    assert bool((z[plant] == 0).all()) and bool((p[plant] == 0.5).all())
    mask = torch.empty((n,) + sp, dtype=torch.uint8, device="cuda")
    be.head_mask(x1, w1, b1, mask, 0.5)
    assert bool((mask[plant] == 0).all())
    assert torch.equal(mask, ((z[..., 0] > 0) * 255).to(torch.uint8))
    # nc = 4: classes 1 and 3 identical -> whenever they are the maximum, argmax is 1
    w4 = torch.randint(-8, 9, (4, cin), generator=g, device="cuda").float() * QW
    w4[3] = w4[1]
    b4 = torch.tensor([0.0, 0.125, -0.25, 0.125], device="cuda")
    z4 = _nan((n,) + sp + (4,))
    be.head_fwd(x, w4, b4, z4, None)
    be.head_mask(x, w4, b4, mask, 0.5)
    top = z4.max(-1).values
    assert bool((z4[..., 1] == z4[..., 3]).all())
    first = torch.where(z4[..., 0] == top, 0, torch.where(z4[..., 1] == top, 1, torch.where(z4[..., 2] == top, 2, 3)))
    assert torch.equal(mask.long(), first) and bool((mask != 3).all()) and bool((mask == 1).any())
    # nc = 2: tied rows -> p = 0.5 exactly, mask 0, 'on' never set
    w2 = w4[:2].clone()
    w2[1] = w2[0]
    b2 = torch.tensor([0.125, 0.125], device="cuda")
    z2, p2 = _nan((n,) + sp + (2,)), _nan((n,) + sp + (2,))
    be.head_fwd(x, w2, b2, z2, p2)
    assert bool((p2 == 0.5).all())
    be.head_mask(x, w2, b2, mask, 0.5)
    assert bool((mask == 0).all())
    labels = torch.randint(0, 2, (n,) + sp, generator=g, device="cuda")
    part = torch.zeros(be.part_size(2), dtype=F64, device="cuda")
    m1 = torch.zeros(n, 2, 3, dtype=F64, device="cuda")
    m2 = torch.zeros_like(m1)
    be.loss_partials(z2, labels, 2.0, 0.25, part, m1)
    be.metric_partials(p2, labels, 0.5, m2)
    assert torch.equal(m1, m2) and bool((m1[..., :2] == 0).all())
    assert torch.equal(m1[..., 2], torch.stack([(labels == c).sum((1, 2, 3)) for c in range(2)], -1).double())


def _run_partials(be, z, t, cs):
    n, c = z.shape[0], z.shape[-1]
    part = torch.zeros(be.part_size(c), dtype=F64, device="cuda")
    metric = torch.zeros(n, c, 3, dtype=F64, device="cuda")
    be.loss_partials(z, t, cs["gamma"], 0.25, part, metric)
    return part, metric


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(LOSS_CASES))
def test_loss_partials_against_fp64(be, name):
    cs = LOSS_CASES[name]
    z, t = loss_logits(cs, 21, "cuda")
    part, metric = _run_partials(be, z, t, cs)
    ref = loss_reference(z, t, cs["gamma"])
    chain = chain_len(ref["vox"], cs["n"], cs["c"])
    check_partials(part, metric, ref, cs["c"], chain, cs["ldt"] == F32, name)
    if cs["c"] > 1:
        assert float(part[3 * cs["c"] + 3]) == 3.0


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(LOSS_CASES))
def test_loss_bwd_at_kernel_lcoef(be, name):
    """dz within the propagated bound of the fp64 closed form at the kernel's own fp32 lcoef, for gscale 1 and 0.7,
    with all three terms and with the focal term alone (the gamma = 0 limit at confidently classified voxels)"""
    cs = LOSS_CASES[name]
    c = cs["c"]
    z, t = loss_logits(cs, 22, "cuda")
    part, _ = _run_partials(be, z, t, cs)
    ref = loss_reference(z, t, cs["gamma"])
    alpha = torch.linspace(0.5, 1.5, c, device="cuda")
    for terms in (DICE | CE | FOCAL, FOCAL):
        loss = torch.empty((), dtype=F32, device="cuda")
        lcoef = _nan((2 * c + 3 if c > 1 else 5,))
        be.loss_finalize(part, c, terms, alpha, cs["gamma"], 0.25, loss, lcoef)
        lc = lcoef.double().tolist()
        for gs in (1.0, 0.7):
            gsc = torch.tensor([gs], dtype=F32, device="cuda")
            dz = _nan(z.shape)
            be.loss_bwd(z, t, lcoef, gsc, dz)
            want, tol = bwd_reference(ref, lc, c, cs["gamma"], float(np.float32(gs)))
            dzr = dz.reshape(want.shape)
            mask = None if c == 1 else ref["valid"][..., None].expand_as(want)
            check_dz(dzr, want, tol, f"{name} terms={terms} gscale={gs}", mask)
            if c > 8:        # the generic kernel zeroes the gradient of a label outside [0, C)
                assert bool((dzr[~ref["valid"]] == 0).all())


def _finalize_cases():
    out = []
    for c in (1, 3):
        for terms in range(1, 8):
            out.append((c, terms, "plain"))
    out += [(3, DICE, "absent"), (3, DICE | CE, "clamp"), (3, DICE | CE | FOCAL, "bad"), (5, DICE | FOCAL, "absent")]
    return out


def _finalize_part(c, kind, seed):
    r = np.random.default_rng(seed)
    if c == 1:
        V = 2 * 96 ** 3
        I, P, T = r.random() * 1e4, r.random() * 3e4, float(r.integers(1000, 30000))
        return [I, P, T, r.random() * V * 0.6, r.random() * V * 0.1, float(V), 0.0]
    V = float(2 * 96 ** 3)
    Cn = r.integers(1000, 100000, c).astype(float)
    P = r.random(c) * 1e5
    I = np.minimum(P, Cn) * r.random(c)
    bad = 0.0
    if kind == "absent":
        Cn[1], I[1] = 0.0, 0.0
    if kind == "clamp":
        I[2], P[2] = 0.0, 5e4               # draw = 1e-5 / (Cn + 5e4 + 1e-5) < 1e-7
    if kind == "bad":
        bad = 3.0
    return list(I) + list(P) + list(Cn) + [r.random() * V * 0.7, r.random() * V * 0.2, V, bad]


@pytest.mark.gpu
@pytest.mark.parametrize("c,terms,kind", _finalize_cases())
def test_loss_finalize_within_one_ulp(be, c, terms, kind):
    part_l = _finalize_part(c, kind, 100 * c + terms)
    part = torch.tensor(part_l, dtype=F64, device="cuda")
    alpha = [0.5 + 0.25 * k for k in range(c)]
    for gamma in (2.0, 0.5):
        loss = _nan(())
        lcoef = _nan((2 * c + 3 if c > 1 else 5,))
        be.loss_finalize(part, c, terms, torch.tensor(alpha, device="cuda"), gamma, 0.25, loss, lcoef)
        val, lc = finalize_reference(part_l, c, terms, [float(np.float32(a)) for a in alpha], gamma, 0.25)
        assert within_ulp(float(loss), val), (kind, terms, float(loss), val)
        for i, (gv, wv) in enumerate(zip(lcoef.tolist(), lc)):
            assert within_ulp(gv, wv), (kind, terms, i, gv, wv)
        if kind == "bad":
            assert math.isnan(float(loss))


@pytest.mark.gpu
@pytest.mark.parametrize("n,c", [(2, 1), (2, 2), (5, 4), (600, 1), (3, 9)])
def test_metric_finalize_within_one_ulp(be, n, c):
    r = np.random.default_rng(n * 10 + c)
    m = np.zeros((n, c, 3))
    m[..., 1] = r.integers(0, 5000, (n, c))
    m[..., 2] = r.integers(0, 5000, (n, c))
    m[..., 0] = np.floor(np.minimum(m[..., 1], m[..., 2]) * r.random((n, c)))
    m[0, 0] = 0                                          # an empty class: dice = 1 by the smoothing
    metric = torch.tensor(m, dtype=F64, device="cuda")
    out = _nan((2,))
    be.metric_finalize(metric, out)
    dice, iou = metric_reference(metric.cpu())
    assert within_ulp(float(out[0]), dice) and within_ulp(float(out[1]), iou), (out.tolist(), dice, iou)


E2E = [("MutilDiceLoss", 2), ("MutilCrossEntropyLoss", 2), ("MutilFocalLoss", 2), ("MutilCrossEntropyDiceLoss", 2),
       ("BinaryDiceLoss", 1), ("BinaryCrossEntropyLoss", 1), ("BinaryFocalLoss", 1),
       ("BinaryCrossEntropyDiceLoss", 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,c", E2E)
def test_loss_modules_against_fp64_autograd(name, c):
    """b200.<Loss> forward and backward at 96^3 x 2 against fp64 autograd of oracle.losses; the bound adds to the
    per-element one the effect of the fp32 rounding of lcoef and of the partial sums it comes from"""
    import oracle
    import pytorchdeeplearing_b200 as b200
    cs = L(2, (96, 96, 96), c, gamma=2.0)
    z, t = loss_logits(cs, 31, "cuda")
    if c > 1:
        t = t.clamp(0, c - 1)
    alpha = torch.tensor([0.75, 1.25], device="cuda")
    mod = getattr(b200, name)(alpha) if name.startswith("Mutil") else getattr(b200, name)()
    zn = z.permute(0, 4, 1, 2, 3).contiguous().requires_grad_(True)
    loss = mod(zn, t)
    loss.backward()
    z64 = zn.detach().double().requires_grad_(True)
    ref_loss = oracle.loss_forward(name, z64, t, alpha.double(), dtype=F64)
    ref_loss.backward()
    ref = loss_reference(z, t, 2.0)
    chain = chain_len(ref["vox"], 2, c)
    eps_sum = float(((ref["err"] + chain * U * ref["abs"]) / ref["part"].abs().clamp_min(1e-300)).max())
    terms = {"Dice": DICE, "CrossEntropy": CE, "Focal": FOCAL, "CrossEntropyDice": CE | DICE}[
        name.replace("Mutil", "").replace("Binary", "").replace("Loss", "")]
    _, lc = finalize_reference(ref["part"].tolist(), c, terms, alpha.double().tolist(), 2.0, 0.25)
    want, tol = bwd_reference(ref, lc, c, 2.0, 1.0, dlcoef=3 * eps_sum + 4 * U)
    got = zn.grad.permute(0, 2, 3, 4, 1).reshape(want.shape)
    auto = z64.grad.permute(0, 2, 3, 4, 1).reshape(want.shape)
    check_dz(got, auto, tol, name)
    rl = float(ref_loss.detach())
    assert abs(float(loss) - rl) <= 3 * eps_sum * (abs(rl) + 1) + U * abs(rl)


def _adam_buffers(n, off, seed):
    p, m, v, r = adam_state(n, seed)
    bufs = []
    for a in (p, (r.standard_normal(n) * 1e-2).astype(np.float32), m, v):
        full = torch.full((n + off + 8,), float("nan"), dtype=F32, device="cuda")
        full[off:off + n] = torch.from_numpy(a).cuda()
        bufs.append(full)
    return bufs, [b[off:off + n] for b in bufs]


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ADAM_CASES))
@pytest.mark.parametrize("decoupled,wd", [(1, 0.0), (1, 1e-2), (0, 0.0), (0, 3e-2)])
@pytest.mark.parametrize("gscale", [None, 0.5])
def test_adam_step_bitwise(be, name, decoupled, wd, gscale):
    n, off = ADAM_CASES[name]
    fulls, (P, G, M, V) = _adam_buffers(n, off, 10 * sorted(ADAM_CASES).index(name) + 2 * decoupled + (wd > 0))
    assert ((P.data_ptr() % 16) == 0) == (off == 0)
    state = torch.zeros(4, dtype=F32, device="cuda")
    gs = None if gscale is None else torch.tensor([gscale], dtype=F32, device="cuda")
    p, m, v = (a.cpu().numpy() for a in (P, M, V))
    st = np.zeros(4, np.float32)
    lr, b1, b2, eps = 1e-3, 0.9, 0.999, 1e-8
    for step in range(3):
        g = (np.random.default_rng(step).standard_normal(n) * 1e-2).astype(np.float32)
        G.copy_(torch.from_numpy(g))
        be.adam_step(P, G, M, V, state, lr, b1, b2, eps, wd, decoupled, gscale=gs, tick=True)
        st = adam_tick_ref(st, lr, b1, b2)
        p, m, v = adam_step_ref(p, g, m, v, st, lr, b1, b2, eps, wd, decoupled, gscale)
        for what, got, want in (("p", P, p), ("exp_avg", M, m), ("exp_avg_sq", V, v)):
            msg = first_mismatch(got.cpu(), torch.from_numpy(want))
            assert msg is None, f"{name} step {step + 1}: {what}: {msg}"
        assert_bitwise(state[:3].cpu(), torch.from_numpy(st[:3]), f"state after {step + 1} ticks")
    for full in fulls:                 # nothing outside the slices was written
        assert bool(full[:off].isnan().all()) and bool(full[off + n:].isnan().all())


@pytest.mark.gpu
def test_adam_per_parameter_calls(be):
    """optim.py's fallback: one tick = 1 call, then tick = 0 calls on unaligned parameter slices, equals one step of
    the restatement over the whole buffer"""
    sizes = [16 * 27, 16, 1, 32 * 16 * 27, 3, 2, 64 * 4, 5]
    n = sum(sizes)
    fulls, (P, G, M, V) = _adam_buffers(n, 0, 3)
    state = torch.tensor([9.0, 0, 0, 0], dtype=F32, device="cuda")
    p, g, m, v = (a.cpu().numpy() for a in (P, G, M, V))
    o = 0
    for k, s in enumerate(sizes):
        be.adam_step(P[o:o + s], G[o:o + s], M[o:o + s], V[o:o + s], state, 1e-3, 0.9, 0.999, 1e-8, 1e-2, True,
                     tick=(k == 0))
        o += s
    st = adam_tick_ref(np.array([9.0, 0, 0, 0], np.float32), 1e-3, 0.9, 0.999)
    p, m, v = adam_step_ref(p, g, m, v, st, 1e-3, 0.9, 0.999, 1e-8, 1e-2, True)
    for what, got, want in (("p", P, p), ("exp_avg", M, m), ("exp_avg_sq", V, v)):
        assert_bitwise(got.cpu(), torch.from_numpy(want), what)
    assert_bitwise(state[:3].cpu(), torch.from_numpy(st[:3]), "state")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["Adam", "AdamW"])
@pytest.mark.parametrize("foreach", [None, False], ids=["default", "single_tensor"])
@pytest.mark.parametrize("t0", [0, 1, 9, 999])
def test_adam_against_torch_cuda(be, kind, foreach, t0):
    """from identical (p, m, v, t) states: one step of torch.optim on CUDA and of the kernel agree within 2 ulps
    (m and v of max(|.|, 2^-126); p of max(|p|, 0.05)).  The remaining differences are the order of v's two roundings
    (v b2 rounded first in torch, fused into the fma here) and whether torch fuses its scalar multiply-adds"""
    n = 100003
    p, m, v, r = adam_state(n, 40 + t0)
    if t0 == 0:
        m, v = np.zeros_like(m), np.zeros_like(v)
    g = (r.standard_normal(n) * 1e-2).astype(np.float32)
    lr, wd = 1e-3, (1e-2 if kind == "AdamW" else 1e-4)
    tp, tm, tv = torch_adam(kind, p, g, m, v, t0, lr, wd, "cuda", foreach)
    P, G, M, V = (torch.from_numpy(a.copy()).cuda() for a in (p, g, m, v))
    state = torch.tensor([float(t0), 0, 0, 0], dtype=F32, device="cuda")
    be.adam_step(P, G, M, V, state, lr, 0.9, 0.999, 1e-8, wd, kind == "AdamW", tick=True)
    dm = ulp_dist(M.cpu().numpy(), tm, 2.0 ** -126)
    dv = ulp_dist(V.cpu().numpy(), tv, 2.0 ** -126)
    dp = ulp_dist(P.cpu().numpy(), tp, 0.05)
    assert dm.max() <= 2, f"exp_avg: {dm.max():.0f} ulps (median {np.median(dm):.1f})"
    assert dv.max() <= 2, f"exp_avg_sq: {dv.max():.0f} ulps (median {np.median(dv):.1f})"
    assert dp.max() <= 2, f"param: {dp.max():.1f} ulps"
