"""The extension losses per element against fp64: the sensitivity-specificity partial sums and backward, the extended
finalize (Jaccard, ELDice, Tversky, SS, MutilELDice), Lovasz-Softmax, the binary Lovasz hinge and SSIM / SSIM3D
(csrc/loss.cu, csrc/lovasz.cu, csrc/ssim.cu).  No emulated backend code.

1. loss_partials_ss: V and T (int64 labels) and the accuracy sums exactly, the float slots within the per-term bound
   plus the fp32 chain bound of sample_grid.  loss_finalize_ext: value and every lcoef within 1 fp32 ulp of an fp64
   restatement of oracle/losses_ext.py as a function of the partial sums (lcoef = d loss / d (I, P) by autograd; for
   SS the fg / bg weights), at designed partial-sum vectors that reach every clamp and NaN branch.  loss_bwd_ss per
   element at the kernel's own lcoef.  The five loss modules end to end against fp64 autograd of the oracle.
2. Lovasz-Softmax: coef bit for bit against a restatement of the kernel's order (stable sort by e descending, ignored
   last, exact integer prefix counts, J_i and J_{i-1} in fp64 in the kernel's expression order: every operation is an
   exact integer step or one correctly rounded division or subtraction, so the fp64 values are reproducible), seg_scale
   and dz bit for bit, and every dz within 4u |g64| of fp64 autograd of oracle.losses_ext.lovasz_softmax: the kernel
   rounds coef, seg_scale and their product to fp32 (3u); the oracle rounds its gradient once to fp32 where the
   errors enter its fp64 dot product (u).
3. Lovasz hinge: coef = fp32((fg ? -gr : gr) (1/nseg)), dz = gs coef and bad bit for bit; dz within 2u |g64| of the
   oracle (the kernel's fp64-then-fp32 rounding, the oracle's single fp32 rounding).
4. SSIM: gaussian_taps equals oracle.ssim.gaussian bit for bit.  A restatement filters x, y, x^2, y^2, xy separably
   in fp64 with the taps widened from fp32 (the window is their exact outer product; the reference's fp32-rounded 3-D
   window is a documented difference and not used).  Bound: one fp32 rounding plus an fp64 term derived here: every
   filtered field is within gamma_{3k+2} of the same filter applied to |field|; those errors, and the local roundings
   of S and of the coefficient formulas written as equivalent field perturbations, go through S and the coefficients
   by forward-mode autograd (first order), then through the adjoint filter.  Kernel and restatement each carry the
   term, so it counts twice.  The CPU part checks the derivation with u = 2^-24 against an fp32 evaluation.

Every workspace is a view of exactly the reported byte count, 512-byte aligned, between whole 512-byte guard blocks;
every output lives in a guarded allocation holding a NaN pattern outside the view; every input is checked unchanged.
The CPU part (restatements against the oracles, bound derivations, case coverage, checker sensitivity) runs without a
GPU; the GPU part is marked `gpu`."""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_conv_exact import Guarded, assert_guards, assert_bitwise, GUARD, IN_FILL
from test_gpu_head_loss_exact import (sample_grid, loss_blocks, chain_len, check_partials, within_ulp, U, ULP,
                                      ULP_EXPF, SMOOTH, EPS, L, loss_logits, loss_reference, bwd_reference,
                                      check_dz, _finalize_part)

F32, F64, I64 = torch.float32, torch.float64, torch.int64
JACCARD, ELDICE, TVERSKY, SS = 8, 16, 32, 64            # include/b200seg.h B200SEG_LOSS_*
U64 = 2.0 ** -53
WS_BLOCK = 512
WS_FILL = 0xA5
K_TILE = 4096                                           # lovasz.cu kTile: the sort and scan tile
IGNORED_KEY = 0xFFFFFFFF


def f32(v):
    return float(np.float32(v))


def gamma64(n):
    return n * U64 / (1 - n * U64)


# ---------------------------------------------------------------------------------------------------------- guards
class GuardedWorkspace:
    """a workspace view of exactly `nbytes`, starting 512-byte aligned after one whole 512-byte guard block and
    followed by at least one whole guard block (the allocation is whole blocks); everything holds WS_FILL"""

    def __init__(self, nbytes, device="cuda"):
        self.n = int(nbytes)
        tail = WS_BLOCK + (-self.n) % WS_BLOCK
        self.buf = torch.full((WS_BLOCK + self.n + tail,), WS_FILL, dtype=torch.uint8, device=device)
        assert self.buf.data_ptr() % WS_BLOCK == 0 or self.buf.device.type == "cpu"
        self.ptr = self.buf.data_ptr() + WS_BLOCK

    def outside_changed(self):
        b = self.buf.cpu()
        for lo, hi in ((0, WS_BLOCK), (WS_BLOCK + self.n, b.numel())):
            ne = (b[lo:hi] != WS_FILL).nonzero()
            if ne.numel():
                return lo + int(ne[0])
        return None


_NAN_BITS = {F32: (torch.int32, 0x7FC00DEF), F64: (torch.int64, 0x7FF8000000000DEF), I64: (I64, -0x5A5A5A5A5A5A5A5B)}


class GuardedOut:
    """a contiguous output view of `shape` with GUARD elements before and after holding a NaN bit pattern (int64: a
    sentinel); `init` fills the view (accumulating outputs start from zero)"""

    def __init__(self, shape, dtype, init=None, device="cuda"):
        n = math.prod(shape)
        self.ib, pat = _NAN_BITS[dtype]
        self.buf = torch.empty(2 * GUARD + n, dtype=dtype, device=device)
        self.buf.view(self.ib).fill_(pat)
        self.n = n
        self.view = self.buf[GUARD:GUARD + n].view(shape)
        if init is not None:
            self.view.fill_(init)
        self.ptr = self.view.data_ptr()
        self.pat = pat

    def outside_changed(self):
        b = self.buf.view(self.ib).cpu()
        for lo, hi in ((0, GUARD), (GUARD + self.n, b.numel())):
            ne = (b[lo:hi] != self.pat).nonzero()
            if ne.numel():
                return lo + int(ne[0])
        return None


def out32(shape):
    """an fp32 output in a Guarded (dense) allocation"""
    g = Guarded((1, 1, 1, 1, max(1, math.prod(shape))), F32, device="cuda", dense=True)
    g.out = g.view.reshape(shape)
    return g


class Inputs:
    """snapshots of the inputs of a call; check() asserts every one is unchanged bit for bit"""

    def __init__(self, **ts):
        self.ts = {k: (v, v.clone()) for k, v in ts.items() if v is not None}

    def check(self, what):
        for k, (v, v0) in self.ts.items():
            a, b = v.detach(), v0
            if a.is_floating_point():
                ib = {F32: torch.int32, F64: torch.int64}[a.dtype]
                a, b = a.contiguous().view(ib), b.contiguous().view(ib)
            assert torch.equal(a, b), f"{what}: input {k} was modified"


def _rc(be, rc, what):
    assert int(rc) == 0, f"{what}: library returned {int(rc)}"


def _stream(be, t):
    dev, st = be._ds(t)
    return dev, st


# ======================================================================================= 1. sensitivity-specificity
def ss_reference(z, t):
    """fp64 partial sums of loss_partials_ss from fp32 logits z (N, ..., 1) and labels t (int64 or fp32 soft), with the
    per-term bounds of the kernel's fp32 expressions: p = 1/(1 + expf(-z)) (ULP_EXPF ulps, one addition, one division),
    d = p - t and d^2 rounded once each, 1 - t rounded for soft labels, each product into an fmaf (exact product)"""
    n = z.shape[0]
    zz, tt = z.reshape(n, -1).double(), t.reshape(n, -1).double()
    p = torch.sigmoid(zz)
    ep = p * (ULP_EXPF * ULP + 2 * U)
    d = p - tt
    ed = ep + U * d.abs()
    d2 = d * d
    ed2 = 2 * d.abs() * ed + ed * ed + U * (d2 + 2 * d.abs() * ed + ed * ed)
    omt = 1 - tt
    eomt = U * omt.abs()
    terms = [p * tt, p, tt, d2 * tt, d2 * omt]
    errs = [ep * tt.abs(), ep, torch.zeros_like(p), ed2 * tt.abs(), ed2 * omt.abs() + (d2 + ed2) * eomt]
    V = torch.tensor(float(zz.numel()), dtype=F64, device=z.device)
    zero = torch.zeros((), dtype=F64, device=z.device)
    on = (p > 0.5).double()
    return dict(vox=zz.shape[1], part=torch.stack([v.sum() for v in terms] + [V]),
                abs=torch.stack([v.abs().sum() for v in terms] + [zero]),
                err=torch.stack([v.sum() for v in errs] + [zero]),
                metric=torch.stack([(on * tt).sum(1), on.sum(1), tt.sum(1)], -1)[:, None, :],
                p=p, ep=ep, t=tt)


def ss_bwd_reference(ref, wf, wb, gs, dwf=0.0, dwb=0.0):
    """fp64 2 (p - t)(wf t + wb (1 - t)) p (1 - p) gs and a per-element bound of loss_bwd_ss_kernel's fp32 evaluation:
    p as above, d = p - t, q = 1 - p, 1 - t (soft) and w = wf t + wb (1 - t) (two products and an addition, possibly
    one fmaf) each rounded once, four products and the gs product; dwf / dwb: uncertainty of wf / wb themselves"""
    p, ep, t = ref["p"], ref["ep"], ref["t"]
    q, eq = 1 - p, ep + U * (1 - p)
    d, ed = p - t, ep + U * (p - t).abs()
    omt = 1 - t
    w = wf * t + wb * omt
    wm = abs(wf) * t.abs() + abs(wb) * omt.abs()
    ew = 3 * U * wm + abs(wb) * U * omt.abs() + dwf * t.abs() + dwb * omt.abs()
    g = 2 * d * w * p * q
    eg = 2 * (w.abs() * (ed * p * q + d.abs() * ep * q + d.abs() * p * eq) + ew * d.abs() * p * q) + 4 * U * g.abs()
    err = abs(gs) * eg + U * (g * gs).abs()
    return g * gs, err * 1.01


SS_CASES = {                # n, spatial, label dtype
    "below_block_n1_i64": (1, (1, 10, 20), I64), "below_block_n5_f32": (5, (1, 7, 11), F32),
    "one_block_n2_i64": (2, (1, 32, 32), I64), "one_block_n1_f32": (1, (1, 16, 64), F32),
    "uncapped_n5_f32": (5, (4, 32, 40), F32), "uncapped_n2_i64": (2, (8, 32, 40), I64),
    "capped_n2_i64": (2, (96, 96, 96), I64), "capped_n1_f32": (1, (96, 96, 96), F32),
    "capped_n5_i64": (5, (32, 64, 64), I64),
}


def ss_grid_kind(n, sp):
    vox = math.prod(sp)
    per, want = sample_grid(vox, n), -(-vox // 1024)
    if vox < 256:
        return "below_block"
    if per < want:
        return "capped"
    return "one_block" if per == 1 else "uncapped"


# ---------------------------------------------------------------------------------------------------------- finalize
def ext_finalize_reference(part, c, terms, alpha=None, gamma=0.0, alpha_f=0.0):
    """fp64 restatement of oracle/losses_ext.py (binary_jaccard / binary_eldice / binary_tversky / binary_ss /
    multi_eldice) as a function of the partial sums.  -> (value, lcoef): lcoef[0..C) and [C..2C) = d loss / d I and
    d loss / d P by autograd (SS: the fg / bg weights r / (s + T) and (1 - r) / (s + V - T)), then zeros.  gamma and
    alpha_f are the fp32 arguments the kernel receives (Tversky: alpha = alpha_f, beta = gamma; SS: r = alpha_f)."""
    part = [float(v) for v in part]
    s = SMOOTH
    if c == 1:
        I = torch.tensor(part[0], dtype=F64, requires_grad=True)
        P = torch.tensor(part[1], dtype=F64, requires_grad=True)
        T, Sf, Sb, V = part[2], part[3], part[4], part[5]
        if terms == SS:
            r = alpha_f
            val = r * Sf / (s + T) + (1 - r) * Sb / (s + V - T)
            return val, [r / (s + T), (1 - r) / (s + V - T), 0.0, 0.0, 0.0]
        if terms == JACCARD:
            val = 1.0 - (I + s) / (P + T - I + s).clamp_min(EPS)
        elif terms == ELDICE:
            dsc = (2.0 * I + s) / (P + T + s).clamp_min(EPS)
            val = torch.clamp(torch.pow(-torch.log(dsc + s), 0.3), 0, 2)
        elif terms == TVERSKY:
            tp, fp, fn = I, P - I, T - I
            val = torch.clamp(1 - (tp + s) / (tp + alpha_f * fp + gamma * fn + s), 0, 2)
        else:
            raise ValueError(terms)
        a, b = torch.autograd.grad(val, (I, P))
        return float(val.detach()), [float(a), float(b), 0.0, 0.0, 0.0]
    assert terms == ELDICE
    I = torch.tensor(part[:c], dtype=F64, requires_grad=True)
    P = torch.tensor(part[c:2 * c], dtype=F64, requires_grad=True)
    Cn = torch.tensor(part[2 * c:3 * c], dtype=F64)
    bad = part[3 * c + 3]
    al = torch.tensor([f32(a) for a in alpha], dtype=F64)
    d = ((2.0 * I + s) / (Cn + P + s)).clamp_min(EPS)
    present = Cn > 0
    dice = d * present.double() * al
    val = torch.clamp(torch.pow(-torch.log(dice + s), 0.3).sum() / torch.count_nonzero(present), 0, 2)
    a, b = torch.autograd.grad(val, (I, P))
    lc = a.tolist() + b.tolist() + [0.0, 0.0, 0.0]
    return (float("nan") if bad > 0 else float(val.detach())), lc


def F1(I, P, T, Sf=0.0, Sb=0.0, V=1e6):
    return [I, P, T, Sf, Sb, V, 0.0]


def FM(I, P, Cn, bad=0.0, V=2.0 * 96 ** 3):
    return list(I) + list(P) + list(Cn) + [0.0, 0.0, V, bad]


def _multi_part(c, kind, seed):
    r = np.random.default_rng(seed)
    Cn = r.integers(1000, 100000, c).astype(float)
    P = r.random(c) * 1e5
    I = np.minimum(P, Cn) * r.random(c)
    bad = 0.0
    if kind == "absent":                 # the present classes well predicted, so that the mean stays below 2
        P = Cn * (1 + 0.05 * r.random(c))
        I = 0.97 * Cn
        Cn[c // 2], I[c // 2] = 0.0, 0.0
    if kind == "clamp":                  # every class missed: each term (-log(~1e-5))^0.3 > 2
        I[:] = 0.0
        Cn[0] = 0.0
    if kind == "bad":
        bad = 2.0
    if kind == "draw_eps":               # one class with draw < eps: no gradient through its clamp_min
        I[-1], P[-1] = 0.0, 5e4
    return FM(I, P, Cn, bad)


# name -> (c, terms, part, alpha, gamma, alpha_f, branch)
FIN_CASES = {
    "jaccard": (1, JACCARD, _finalize_part(1, "plain", 801), None, 0.0, 0.0, "normal"),
    "jaccard_small": (1, JACCARD, F1(0.5, 2.25, 1.0), None, 0.0, 0.0, "normal"),
    "jaccard_u_below_eps": (1, JACCARD, F1(1e-3, 0.0, 0.0), None, 0.0, 0.0, "clamp_min"),
    "eldice": (1, ELDICE, _finalize_part(1, "plain", 802), None, 0.0, 0.0, "normal"),
    "eldice_near_one": (1, ELDICE, F1(990.0, 1000.0, 1000.0), None, 0.0, 0.0, "normal"),
    "eldice_clamp2": (1, ELDICE, F1(0.0, 10.0, 0.0), None, 0.0, 0.0, "clamp"),
    "eldice_nan": (1, ELDICE, F1(1000.0, 1000.0, 1000.0), None, 0.0, 0.0, "nan"),
    "tversky_03_07": (1, TVERSKY, _finalize_part(1, "plain", 803), None, f32(0.7), f32(0.3), "normal"),
    "tversky_asym": (1, TVERSKY, _finalize_part(1, "plain", 804), None, f32(0.15), f32(0.8), "normal"),
    "tversky_clamp0": (1, TVERSKY, F1(100.0, 50.0, 100.0), None, f32(0.7), f32(0.3), "clamp"),
    "ss_r01": (1, SS, _finalize_part(1, "plain", 805), None, 0.0, f32(0.1), "normal"),
    "ss_r05": (1, SS, _finalize_part(1, "plain", 806), None, 0.0, f32(0.5), "normal"),
    "ss_empty_fg": (1, SS, F1(0.0, 300.0, 0.0, 0.0, 120.5, 1000.0), None, 0.0, f32(0.1), "normal"),
}
for _c in (2, 3, 9):
    _al = [0.5 + 0.5 * k / (_c - 1) for k in range(_c)]
    for _kind in ("plain", "absent", "clamp", "bad", "draw_eps"):
        _part = _multi_part(_c, _kind, 900 + 10 * _c + len(_kind))
        FIN_CASES[f"multi_c{_c}_{_kind}"] = (_c, ELDICE, _part, _al, 0.0, 0.0, None)


def finalize_branch(c, terms, part, alpha=None, gamma=0.0, alpha_f=0.0):
    """which branch of loss_finalize_ext_kernel a part vector takes"""
    s = SMOOTH
    if c > 1:
        if part[3 * c + 3] > 0:
            return "nan"
        I, P, Cn = part[:c], part[c:2 * c], part[2 * c:3 * c]
        K = sum(1 for v in Cn if v > 0)
        S = 0.0
        low = False
        for k in range(c):
            draw = (2 * I[k] + s) / (Cn[k] + P[k] + s)
            low |= Cn[k] > 0 and draw < EPS
            dice = max(draw, EPS) * f32(alpha[k]) if Cn[k] > 0 else 0.0
            S += (-math.log(dice + s)) ** 0.3
        if not 0 <= S / K <= 2:
            return "clamp"
        return "clamp_min" if low else ("absent" if K < c else "normal")
    I, P, T = part[:3]
    if terms == JACCARD:
        return "normal" if P + T - I + s >= EPS else "clamp_min"
    if terms == ELDICE:
        dsc = (2 * I + s) / max(P + T + s, EPS)
        if dsc + s >= 1:
            return "nan"
        return "normal" if (-math.log(dsc + s)) ** 0.3 <= 2 and P + T + s >= EPS else "clamp"
    if terms == TVERSKY:
        v = 1 - (I + s) / (I + alpha_f * (P - I) + gamma * (T - I) + s)
        return "normal" if 0 <= v <= 2 else "clamp"
    return "normal"


for _name, _cs in FIN_CASES.items():
    if _cs[6] is None:
        FIN_CASES[_name] = _cs[:6] + (finalize_branch(*_cs[:6]),)


def sensitivity(fn, part, tol):
    """first-order bounds on the change of (value, lcoef) over part +- tol: the sum over slots of the change when one
    slot moves by its bound, times 2 (the step is the bound itself, so curvature over it is included once more)"""
    v0, l0 = fn(part)
    l0 = np.array(l0)
    dv, dl = 0.0, np.zeros_like(l0)
    for j, tj in enumerate(tol):
        if tj <= 0:
            continue
        p2 = list(part)
        p2[j] += tj
        v1, l1 = fn(p2)
        dv += abs(v1 - v0)
        dl += np.abs(np.array(l1) - l0)
    return 2 * dv, 2 * dl


# ======================================================================================= 2. Lovasz-Softmax
def lovasz_segments(z, t, per_image, ignore):
    """(N, vox, C) fp32 logits and (N, vox) labels -> per segment (seg = b C + c): z_c, labels, class, fg, ignored"""
    n, vox, c = z.shape
    if per_image:
        zc = z.permute(0, 2, 1).reshape(n * c, vox)
        lab = t.reshape(n, 1, vox).expand(n, c, vox).reshape(n * c, vox)
        cls = torch.arange(c).repeat(n)
    else:
        zc = z.reshape(n * vox, c).T
        lab = t.reshape(1, -1).expand(c, -1)
        cls = torch.arange(c)
    ign = (lab == ignore) if ignore is not None else torch.zeros_like(lab, dtype=torch.bool)
    fg = lab == cls[:, None]
    return zc.contiguous(), lab, fg, ign


def sorted_grad(keys, fg, gts, drop_first_jp=False):
    """stable ascending sort of the keys (ties in position order), exact integer prefix counts of the sorted
    foreground and gr_i = J_i - J_{i-1} in fp64 in the kernels' expression order; -> (order, gr, fg sorted, valid)"""
    order = torch.sort(keys, dim=1, stable=True).indices
    fgs = fg.gather(1, order).long()
    cum = fgs.cumsum(1)
    j = torch.arange(keys.shape[1], dtype=F64)[None, :]
    g = gts.double()[:, None]
    cf, cp = cum.double(), (cum - fgs).double()
    Ji = 1.0 - (g - cf) / (g + ((j + 1) - cf))
    Jp = 1.0 - (g - cp) / (g + (j - cp))
    if drop_first_jp:
        Jp[:, 0] = 0.0
    valid = keys.gather(1, order) != IGNORED_KEY
    return order, Ji - Jp, fgs, valid


def _keys(e, dropped):
    k = (~e.contiguous().view(torch.int32)).long() & 0x7FFFFFFF
    return torch.where(dropped, torch.full_like(k, IGNORED_KEY), k)


def lovasz_restate(z, t, per_image, ignore, order_fix=None):
    """the kernel's coef [N][vox][C], seg_scale and per-segment sum |e gr|; z (N, vox, C) fp32, t (N, vox) int64 on
    the CPU.  order_fix(order) may rewrite the sort order (checker sensitivity)"""
    n, vox, c = z.shape
    zc, lab, fg, ign = lovasz_segments(z, t, per_image, ignore)
    e = (fg.float() - zc).abs()
    keys = _keys(e, ign)
    fgv = fg & ~ign
    gts = fgv.sum(1)
    order, gr, fgs, valid = sorted_grad(keys, fgv, gts)
    if order_fix is not None:
        order = order_fix(order)
        _, gr, fgs, valid = sorted_grad(keys.gather(1, order), fgv.gather(1, order), gts)
    ok = valid & (gts[:, None] > 0)
    grad = torch.where(ok, gr, torch.zeros_like(gr)).float()
    es = e.gather(1, order).double()
    eg = torch.where(ok, es * gr, torch.zeros_like(gr))
    seg = torch.zeros_like(grad).scatter_(1, order, grad)
    if per_image:
        coef = seg.reshape(n, c, vox).permute(0, 2, 1)
    else:
        coef = seg.T.reshape(n, vox, c)
    nimg = n if per_image else 1
    present = (gts > 0).reshape(nimg, c)
    K = present.sum(1)
    scale = torch.zeros(nimg, c, dtype=F32)
    for b in range(nimg):
        if int(K[b]) > 0:
            w = f32(1.0 / (nimg * int(K[b])))
            scale[b] = torch.where(present[b], torch.tensor(w), torch.tensor(0.0))
    loss = 0.0
    for b in range(nimg):
        if int(K[b]) > 0:
            loss += float(eg.sum(1).reshape(nimg, c)[b].sum()) / int(K[b])
    return dict(coef=coef.contiguous(), scale=scale.reshape(-1), loss=loss / nimg,
                abs=float(eg.abs().sum()), len=keys.shape[1])


def lovasz_dz(z, t, coef, scale, gs, per_image):
    """the kernel's dz = ((gs coef) sgn) seg_scale in fp32, sgn(0) = 0"""
    n, vox, c = z.shape
    fg = (t[..., None] == torch.arange(c)).float()
    d = z - fg
    sg = torch.sign(d)
    sc = scale.reshape(n if per_image else 1, 1, c)
    return ((torch.tensor(gs, dtype=F32) * coef) * sg) * sc


def lovasz_oracle(z, t, per_image, ignore, device="cpu"):
    """fp64 autograd of oracle.losses_ext.lovasz_softmax (NCDHW) -> (value, grad (N, vox, C))"""
    from oracle import losses_ext as ox
    n, vox, c = z.shape
    zo = z.double().permute(0, 2, 1).reshape(n, c, vox, 1, 1).to(device).requires_grad_(True)
    v = ox.lovasz_softmax(zo, t.reshape(n, vox, 1, 1).to(device), per_image=per_image, ignore=ignore, dtype=F64)
    if torch.is_tensor(v) and v.requires_grad:
        v.backward()
        gr = zo.grad.reshape(n, c, vox).permute(0, 2, 1).cpu()
    else:
        gr = torch.zeros(n, vox, c, dtype=F64)
    return float(v.detach() if torch.is_tensor(v) else v), gr


def LZ(n, vox, c, per_image=False, ignore=None, kind="randn", **kw):
    d = dict(n=n, vox=vox, c=c, per_image=per_image, ignore=ignore, kind=kind)
    d.update(kw)
    return d


LOVASZ_CASES = {
    "len1": LZ(1, 1, 3), "len4095": LZ(1, 4095, 3), "len4096": LZ(1, 4096, 3), "len4097": LZ(1, 4097, 3),
    "len3tiles_plus1": LZ(1, 3 * K_TILE + 1, 3),
    "c2": LZ(2, 3000, 2), "c3": LZ(2, 2500, 3, kind="quant"), "c5": LZ(3, 2000, 5, kind="onehot"),
    "c9": LZ(2, 2100, 9), "c1024_short": LZ(2, 37, 1024),
    "per_image_n1": LZ(1, 5000, 3, per_image=True), "per_image_n3": LZ(3, 4097, 4, per_image=True, kind="quant"),
    "ignore_class": LZ(2, 4500, 3, ignore=1), "ignore_255": LZ(2, 4500, 3, ignore=255, kind="outside"),
    "outside_not_ignored": LZ(2, 3000, 3, kind="outside"),
    "per_image_all_ignored": LZ(3, 3000, 3, per_image=True, ignore=2, kind="all_ignored"),
    "absent_classes": LZ(2, 3000, 5, kind="absent"),
    "quantised_ties": LZ(2, 2 * K_TILE + 123, 2, kind="quant"),
    "e_zero": LZ(2, 5000, 3, kind="onehot"),
    "vnet96_c2": LZ(2, 96 ** 3, 2, big=True), "unet_c5": LZ(1, 128 * 112 * 112, 5, big=True),
    "per_image_ignore_48": LZ(2, 48 ** 3, 3, per_image=True, ignore=1, big=True),
}


def lovasz_operands(cs, seed):
    """(N, vox, C) fp32 logits and (N, vox) int64 labels on the CPU.  quant: logits on a 1/8 grid in [0, 1], so long
    runs of equal e cross tile seams; onehot: about a quarter of the voxels carry z_c = fg exactly (e = 0, key
    0x7FFFFFFF); outside: labels 255 and C; absent: classes 1 and 3 never occur; all_ignored: sample 1 is all ignore"""
    g = torch.Generator().manual_seed(seed)
    n, vox, c, kind = cs["n"], cs["vox"], cs["c"], cs["kind"]
    t = torch.randint(0, c, (n, vox), generator=g)
    if kind == "quant":
        z = torch.randint(0, 9, (n, vox, c), generator=g).float() / 8
    else:
        z = torch.randn((n, vox, c), generator=g)
    if kind == "onehot":
        exact = torch.rand((n, vox), generator=g) < 0.25
        oh = F.one_hot(t, c).float()
        z = torch.where(exact[..., None], oh, z)
        z[0, :7] = 0.0                                   # e = 1 for fg, 0 for bg
    if kind in ("outside",):
        sel = torch.rand((n, vox), generator=g)
        t = torch.where(sel < 0.05, torch.full_like(t, 255), torch.where(sel < 0.08, torch.full_like(t, c), t))
    if kind == "absent":
        t = torch.where((t == 1) | (t == 3), torch.zeros_like(t), t)
    if kind == "all_ignored":
        t[1] = cs["ignore"]
    return z.contiguous(), t.contiguous()


def lovasz_tiles(vox, n, per_image):
    ln = vox if per_image else n * vox
    return -(-ln // K_TILE), ln


# ======================================================================================= 3. Lovasz hinge
def hinge_restate(z, t, per_image, ignore):
    """the kernel's coef (as z), loss, bad, per segment sum |relu(e) gr|; z (N, vox) fp32, t (N, vox) int64 (CPU)"""
    n = z.shape[0]
    nseg = n if per_image else 1
    zz, lab = z.reshape(nseg, -1), t.reshape(nseg, -1)
    e = torch.where(lab == 1, 1 - zz, 1 + zz)
    ign = (lab == ignore) if ignore is not None else torch.zeros_like(lab, dtype=torch.bool)
    dropped = ign | (e <= 0)
    keys = _keys(e, dropped)
    fgv = (lab == 1) & ~ign
    gts = fgv.sum(1)
    order, gr, fgs, valid = sorted_grad(keys, fgv & ~dropped, gts, drop_first_jp=True)
    inv = 1.0 / nseg
    d = torch.where(fgs.bool(), -gr, gr) * inv
    d = torch.where(valid, d, torch.zeros_like(d)).float()
    es = e.gather(1, order).double()
    eg = torch.where(valid, es * gr, torch.zeros_like(gr))
    coef = torch.zeros_like(d).scatter_(1, order, d).reshape(z.shape)
    bad = int(((lab != 0) & (lab != 1) & ~ign).sum())
    return dict(coef=coef, loss=float(eg.sum()) / nseg, abs=float(eg.abs().sum()), bad=bad, len=keys.shape[1])


def hinge_oracle(z, t, per_image, ignore, device="cpu"):
    from oracle import lovasz_hinge as oh
    zo = z.double().to(device).requires_grad_(True)
    v = oh.lovasz_hinge(zo, t.to(device), per_image=per_image, ignore=ignore, dtype=F64)
    if torch.is_tensor(v) and v.requires_grad:
        v.backward()
        return float(v.detach()), zo.grad.cpu()
    return float(v), torch.zeros(z.shape, dtype=F64)


HINGE_CASES = {
    "len1": LZ(1, 1, 1), "len4095": LZ(1, 4095, 1), "len4096": LZ(1, 4096, 1), "len4097": LZ(1, 4097, 1),
    "len3tiles_plus1": LZ(1, 3 * K_TILE + 1, 1),
    "e_zero_and_negative": LZ(2, 5000, 1, kind="margins"),
    "gts_zero": LZ(1, 3000, 1, kind="all_bg"),
    "per_image_bg_and_ignored": LZ(3, 4097, 1, per_image=True, ignore=255, kind="bg_ignored"),
    "per_image_n1": LZ(1, 9000, 1, per_image=True),
    "ignore_0": LZ(2, 3000, 1, ignore=0),
    "bad_labels": LZ(2, 3000, 1, kind="bad"),
    "quantised_ties": LZ(2, 2 * K_TILE + 123, 1, kind="quant"),
    "vnet96": LZ(2, 96 ** 3, 1, big=True), "vnet96_per_image": LZ(2, 96 ** 3, 1, per_image=True, big=True),
    "unet128_ignore": LZ(1, 128 ** 3, 1, ignore=255, kind="outside", big=True),
}


def hinge_operands(cs, seed):
    g = torch.Generator().manual_seed(seed)
    n, vox, kind = cs["n"], cs["vox"], cs["kind"]
    t = (torch.rand((n, vox), generator=g) < 0.4).long()
    z = torch.randn((n, vox), generator=g) * 1.5
    if kind == "margins":                       # z = +-1 exactly (e = 0) and confident voxels (e < 0)
        sel = torch.rand((n, vox), generator=g)
        z = torch.where(sel < 0.15, 2.0 * t.float() - 1.0, z)
        z = torch.where((sel > 0.15) & (sel < 0.3), (2.0 * t.float() - 1.0) * 3, z)
    if kind == "quant":
        z = torch.randint(-8, 9, (n, vox), generator=g).float() / 4
    if kind == "all_bg":
        t.zero_()
    if kind == "bg_ignored":
        t[0].zero_()
        t[1] = 255
        t[2, ::7] = 255
    if kind == "bad":
        t[0, 5::97] = 2
        t[1, 11::89] = -1
    if kind == "outside":
        t[t.numel() // 3:].view(-1)[::13] = 255
        t = t.view(n, vox)
    return z.contiguous(), t.contiguous()


# ======================================================================================= 4. SSIM
SS_TW, SS_MAXK, SS_TARGET = 32, 31, 256
SMEM_PREF, SMEM_MAX = 113 * 1024, 226 * 1024
C1, C2 = 0.01 ** 2, 0.03 ** 2


def ssim_smem(bwd, k, kd, th):
    """smem_bytes (ssim.cu)"""
    R, SW, nf = th + k - 1, SS_TW + k - 1, 4 if bwd else 5
    stage = 4 * R * SW * 8 if bwd else 2 * R * SW * 4
    return stage + nf * R * SS_TW * 8 + kd * nf * th * SS_TW * 8


def pick_th(bwd, k, kd):
    """pick_th (ssim.cu)"""
    for lim in (SMEM_PREF, SMEM_MAX):
        for th in (8, 4, 2, 1):
            if ssim_smem(bwd, k, kd, th) <= lim:
                return th
    return 1


def ssim_tiling(dims, n, c, d, h, w, k, bwd):
    """make_geom + tile (ssim.cu) -> (TH, nWT, nHT, Dc, nDC), (Dout, Hout, Wout), kd"""
    P = k // 2
    Dm = d + 2 * P - k + 1 if dims == 3 else 1
    Hm, Wm = h + 2 * P - k + 1, w + 2 * P - k + 1
    kd = k if dims == 3 else 1
    Dout, Hout, Wout = ((d if dims == 3 else 1), h, w) if bwd else (Dm, Hm, Wm)
    TH = pick_th(bwd, k, kd)
    nWT, nHT = -(-Wout // SS_TW), -(-Hout // TH)
    base = nWT * nHT * n * c
    ndc = max(1, min(-(-SS_TARGET // base), -(-Dout // kd)))
    Dc = -(-Dout // ndc)
    return (TH, nWT, nHT, Dc, -(-Dout // Dc)), (Dout, Hout, Wout), kd


def SC(dims, n, c, sp, k, mode, fwd, bwd, rng=1.0, layout="dense", grads="both"):
    return dict(dims=dims, n=n, c=c, sp=sp, k=k, mode=mode, fwd=fwd, bwd=bwd, rng=rng, layout=layout, grads=grads)


# fwd / bwd: the (TH, nWT, nHT, Dc, nDC) each pass must produce
SSIM_CASES = {
    "2d_k11_w31": SC(2, 2, 1, (37, 31), 11, 0, (8, 1, 5, 1, 1), (8, 1, 5, 1, 1)),
    "2d_k2_w32_mode1": SC(2, 2, 2, (20, 31), 2, 1, (8, 1, 3, 1, 1), (8, 1, 3, 1, 1)),
    "2d_k10_w33_mode1": SC(2, 3, 1, (29, 32), 10, 1, (8, 2, 4, 1, 1), (8, 1, 4, 1, 1), rng=255.0),
    "2d_k31_w65_255": SC(2, 1, 2, (40, 65), 31, 0, (8, 3, 5, 1, 1), (4, 3, 10, 1, 1), rng=255.0),
    "2d_k1": SC(2, 1, 3, (17, 40), 1, 1, (8, 2, 3, 1, 1), (8, 2, 3, 1, 1)),
    "2d_k3_cl_slice": SC(2, 2, 3, (26, 45), 3, 0, (8, 2, 4, 1, 1), (8, 2, 4, 1, 1), layout="slice"),
    "3d_k11_mode0": SC(3, 1, 2, (21, 19, 33), 11, 0, (4, 2, 5, 11, 2), (4, 2, 5, 11, 2)),
    "3d_k3_mode2_cl": SC(3, 2, 2, (30, 14, 20), 3, 2, (8, 1, 2, 3, 10), (8, 1, 2, 3, 10), layout="cl"),
    "3d_k15_dout_lt_kd": SC(3, 2, 1, (5, 23, 31), 15, 2, (4, 1, 6, 5, 1), (4, 1, 6, 5, 1)),
    "3d_k2_even_w67": SC(3, 1, 1, (9, 13, 66), 2, 2, (8, 3, 2, 2, 5), (8, 3, 2, 2, 5), rng=255.0),
    "3d_k10_dc_lt_kd": SC(3, 1, 1, (31, 9, 30), 10, 0, (4, 1, 3, 8, 4), (4, 1, 3, 8, 4)),
    "3d_k31_slice": SC(3, 1, 1, (12, 9, 20), 31, 0, (1, 1, 9, 12, 1), (4, 1, 3, 12, 1), layout="slice"),
    "3d_k11_grad1_only": SC(3, 2, 1, (17, 26, 33), 11, 2, (4, 2, 7, 9, 2), (4, 2, 7, 9, 2), grads="x"),
    "3d_k11_grad2_only_255": SC(3, 1, 2, (13, 10, 12), 11, 0, (4, 1, 3, 7, 2), (4, 1, 3, 7, 2), rng=255.0,
                                grads="y"),
    "3d_96_k11": SC(3, 2, 1, (96, 96, 96), 11, 0, (4, 3, 24, 48, 2), (4, 3, 24, 48, 2)),
}


def ssim_maps(dims, d, h, w, k):
    P = k // 2
    return ((d + 2 * P - k + 1) if dims == 3 else 1), h + 2 * P - k + 1, w + 2 * P - k + 1


def ssim_images(cs, seed, device):
    """fp32 (N, C, [D,] H, W) images in [0, rng] in the case's layout: dense, channels-last strides (cl), or a view
    with a storage offset and padded strides (slice).  y is a noisy, locally scaled copy of x with a flat patch"""
    g = torch.Generator(device="cpu").manual_seed(seed)
    dims, n, c, sp = cs["dims"], cs["n"], cs["c"], cs["sp"]
    shape = (n, c) + tuple(sp)
    x = torch.rand(shape, generator=g)
    y = (0.7 * x + 0.3 * torch.rand(shape, generator=g)).clamp(0, 1)
    x.view(-1)[: x.numel() // 9] = 0.5                   # a flat patch: R near C2 there
    x, y = ((v * cs["rng"]).float() for v in (x, y))
    out = []
    for v in (x, y):
        if cs["layout"] == "cl":
            perm = (0, 2, 3, 1) if dims == 2 else (0, 2, 3, 4, 1)
            inv = (0, 3, 1, 2) if dims == 2 else (0, 4, 1, 2, 3)
            v = v.permute(*perm).contiguous().permute(*inv)
        elif cs["layout"] == "slice":
            big = torch.full(tuple(s + 3 for s in shape), IN_FILL, dtype=F32)
            idx = tuple(slice(1, 1 + s) for s in shape)
            big[idx] = v
            v = big[idx]
        out.append(v.to(device))
    return out[0], out[1]


def _filt(t, g, dims):
    """separable zero-padded correlation with the fp64 taps g along W, H and (3-D) D; t (M, 1, D, H, W)"""
    k = g.numel()
    P = k // 2
    t = F.conv3d(t, g.view(1, 1, 1, 1, k), padding=(0, 0, P))
    t = F.conv3d(t, g.view(1, 1, 1, k, 1), padding=(0, P, 0))
    if dims == 3:
        t = F.conv3d(t, g.view(1, 1, k, 1, 1), padding=(P, 0, 0))
    return t


def s_coef(m0, m1, m2, m3, m4):
    """the SSIM map and the four backward coefficients of ssim_filter_kernel's epilogue, from the filtered fields"""
    mu1, mu2 = m0, m1
    s11, s22, s12 = m2 - mu1 * mu1, m3 - mu2 * mu2, m4 - mu1 * mu2
    A, B = 2.0 * mu1 * mu2 + C1, 2.0 * s12 + C2
    Q, R = mu1 * mu1 + mu2 * mu2 + C1, s11 + s22 + C2
    QR = Q * R
    S = A * B / QR
    sq, sr, bq, aq = S / Q, S / R, B / QR, A / QR
    return (S, 2.0 * mu2 * (bq - aq) + 2.0 * mu1 * (sr - sq), 2.0 * mu1 * (bq - aq) + 2.0 * mu2 * (sr - sq), -sr,
            2.0 * aq)


def _coef_mags(m):
    mu1, mu2 = m[0], m[1]
    S, *_ = s_coef(*m)
    Q = mu1 * mu1 + mu2 * mu2 + C1
    R = m[2] - mu1 * mu1 + m[3] - mu2 * mu2 + C2
    A, B = 2 * mu1 * mu2 + C1, 2 * (m[4] - mu1 * mu2) + C2
    sq, sr, bq, aq = (S / Q).abs(), (S / R).abs(), (B / (Q * R)).abs(), (A / (Q * R)).abs()
    return (S.abs(), 2 * mu2.abs() * (bq + aq) + 2 * mu1.abs() * (sr + sq),
            2 * mu1.abs() * (bq + aq) + 2 * mu2.abs() * (sr + sq), sr, 2 * aq)


def ssim_restate(x, y, k, mode, gout, dtype=F64, u=U64):
    """the restatement in `dtype` (F64 for the GPU checks; F32 checks the derivation on the CPU) and the error bound
    of one evaluation with unit roundoff u.  -> dict(value, acc, count, coef [4][map], dx, dy, and their bounds
    dS (map), dcoef, ddx, ddy, dacc: one evaluation's error, first order)"""
    from pytorchdeeplearing_b200.ssim import gaussian_taps
    dims = x.dim() - 2
    n, c = x.shape[:2]
    shp = (n * c, 1) + ((1,) if dims == 2 else ()) + tuple(x.shape[2:])
    g = gaussian_taps(k).to(device=x.device, dtype=dtype)
    X = x.to(dtype).reshape(shp).detach().requires_grad_(True)
    Y = y.to(dtype).reshape(shp).detach().requires_grad_(True)
    fields = [X, Y, X * X, Y * Y, X * Y]
    m = [_filt(f, g, dims) for f in fields]
    S, *cf = s_coef(*m)
    Dm, Hm, Wm = S.shape[2:]
    if mode == 0:
        cnt = float(S.numel())
        s = gout.to(dtype).reshape(()) / cnt
        s = s.expand_as(S)
        red = lambda v: v.sum().reshape(1)                        # noqa: E731
    elif mode == 1:
        cnt = float(c * Hm * Wm)
        s = (gout.to(dtype).reshape(n, 1, 1, 1, 1) / cnt).expand(n, c, 1, 1, 1).reshape(n * c, 1, 1, 1, 1).expand_as(S)
        red = lambda v: v.reshape(n, -1).sum(1)                   # noqa: E731
    else:
        cnt = float(c * Dm * Hm)
        s = (gout.to(dtype).reshape(n, 1, 1, 1, Wm) / cnt).expand(n, c, 1, 1, Wm).reshape(n * c, 1, 1, 1, Wm)
        s = s.expand_as(S)
        red = lambda v: v.reshape(n, c * Dm * Hm, Wm).sum(1)      # noqa: E731
    dx, dy = torch.autograd.grad((s * S).sum(), (X, Y))
    md = [v.detach() for v in m]
    gam = 3 * k + 2
    gk = gam * u / (1 - gam * u)
    with torch.no_grad():
        E = [gk * _filt(f.detach().abs(), g, dims) for f in fields]
        loc = 4 * u * (md[2].abs() + md[0] ** 2 + md[3].abs() + md[1] ** 2 + C2)
        E[2], E[3] = E[2] + loc, E[3] + loc
        E[4] = E[4] + 4 * u * (md[4].abs() + (md[0] * md[1]).abs() + C2)
    outs = [torch.zeros_like(md[0]) for _ in range(5)]
    for j in range(5):
        tan = tuple(E[j] if i == j else torch.zeros_like(md[0]) for i in range(5))
        _, t_out = torch.func.jvp(s_coef, tuple(md), tan)
        for i in range(5):
            outs[i] = outs[i] + t_out[i].abs()
    mags = _coef_mags(md)
    dS = outs[0] + 20 * u * mags[0]
    dcoef = [outs[i] + 20 * u * mags[i] for i in range(1, 5)]
    cfd = [v.detach() for v in cf]
    sd = s.detach()

    def adj(field):
        z0 = torch.zeros(shp, dtype=dtype, device=x.device, requires_grad=True)
        with torch.enable_grad():
            return torch.autograd.grad(_filt(z0, g, dims), z0, grad_outputs=field)[0]

    gk3 = gamma64(3 * k) if u == U64 else 3 * k * u / (1 - 3 * k * u)
    Fv = [adj(sd * v) for v in cfd]
    dF = [adj(sd.abs() * dc + 2 * u * (sd * v).abs()) + gk3 * adj((sd * v).abs()) for v, dc in zip(cfd, dcoef)]
    xd, yd = X.detach(), Y.detach()
    ddx = dF[0] + 2 * xd.abs() * dF[2] + yd.abs() * dF[3] + 3 * u * (Fv[0].abs() + 2 * (xd * Fv[2]).abs()
                                                                     + (yd * Fv[3]).abs())
    ddy = dF[1] + 2 * yd.abs() * dF[2] + xd.abs() * dF[3] + 3 * u * (Fv[1].abs() + 2 * (yd * Fv[2]).abs()
                                                                     + (xd * Fv[3]).abs())
    Sd = S.detach()
    nsum = Sd.numel() // red(Sd).numel()
    acc = red(Sd)
    dacc = red(dS) + nsum * u / (1 - nsum * u) * red(Sd.abs())
    return dict(S=Sd, acc=acc, dacc=dacc, count=cnt, value=acc / cnt, dS=dS,
                coef=torch.stack([v.reshape(-1) for v in cfd]), dcoef=torch.stack([v.reshape(-1) for v in dcoef]),
                dx=dx.reshape(x.shape), dy=dy.reshape(x.shape), ddx=ddx.reshape(x.shape), ddy=ddy.reshape(x.shape),
                maps=(Dm, Hm, Wm))


def check_close(got, want, tol, what):
    """|got - want| <= tol elementwise (NaN nowhere)"""
    got, want, tol = got.double().cpu(), want.double().cpu(), tol.double().cpu()
    bad = ~((got - want).abs() <= tol)
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} outside the bound; first at {i}: got "
                             f"{float(got[i])!r}, want {float(want[i])!r}, bound {float(tol[i]):.3g}")


def ssim_gout(cs, maps, seed, device):
    g = torch.Generator().manual_seed(seed)
    n = cs["n"]
    shape = {0: (1,), 1: (n,), 2: (n, maps[2])}[cs["mode"]]
    return (torch.rand(shape, generator=g) * 1.5 - 0.25).float().to(device)


# ======================================================================================= CPU part
def test_every_variant_has_a_case():
    kinds = {(ss_grid_kind(n, sp), ldt, n) for n, sp, ldt in SS_CASES.values()}
    assert {k for k, _, _ in kinds} == {"below_block", "one_block", "uncapped", "capped"}
    assert {ldt for _, ldt, _ in kinds} == {I64, F32} and {n for _, _, n in kinds} == {1, 2, 5}
    for kind in ("below_block", "capped"):
        assert {ldt for k, ldt, _ in kinds if k == kind} == {I64, F32}
    for n, sp, _ in SS_CASES.values():
        assert loss_blocks(n * math.prod(sp)) >= 1
    branches = {(c, terms, br) for c, terms, part, al, gm, af, br in FIN_CASES.values()}
    assert {br for c, t, br in branches if t == ELDICE and c == 1} == {"normal", "clamp", "nan"}
    assert {br for c, t, br in branches if t == JACCARD} == {"normal", "clamp_min"}
    assert {br for c, t, br in branches if t == TVERSKY} == {"normal", "clamp"}
    assert {br for c, t, br in branches if c > 1} == {"normal", "absent", "clamp", "nan", "clamp_min"}
    assert {c for c, t, br in branches if c > 1} == {2, 3, 9}              # template and generic (C > 8) kernels
    assert {f32(FIN_CASES[k][5]) for k in ("ss_r01", "ss_r05")} == {f32(0.1), f32(0.5)}
    for name, (c, terms, part, al, gm, af, br) in FIN_CASES.items():
        assert finalize_branch(c, terms, part, al, gm, af) == br, name
    # Lovasz: the tile seams, class counts, per_image, ignore forms
    lens = {lovasz_tiles(cs["vox"], cs["n"], cs["per_image"])[1] % K_TILE for cs in LOVASZ_CASES.values()}
    assert {1, K_TILE - 1, 0} <= lens
    assert any(lovasz_tiles(cs["vox"], cs["n"], cs["per_image"])[0] == 4 for cs in LOVASZ_CASES.values())
    assert {cs["c"] for cs in LOVASZ_CASES.values()} >= {2, 3, 5, 9, 1024}
    assert {cs["n"] for cs in LOVASZ_CASES.values() if cs["per_image"]} >= {1, 3}
    assert {cs["ignore"] for cs in LOVASZ_CASES.values()} >= {None, 1, 255}
    assert {cs["kind"] for cs in LOVASZ_CASES.values()} >= {"quant", "onehot", "outside", "absent", "all_ignored"}
    hl = {lovasz_tiles(cs["vox"], cs["n"], cs["per_image"])[1] % K_TILE for cs in HINGE_CASES.values()}
    assert {1, K_TILE - 1, 0} <= hl
    assert {cs["kind"] for cs in HINGE_CASES.values()} >= {"margins", "all_bg", "bg_ignored", "bad", "quant"}
    # SSIM: every tiling the cases claim is the one the library computes, and the tilings cover the seams
    seen = dict(wout=set(), th_rem=set(), k=set(), modes=set(), layouts=set(), grads=set(), rng=set())
    flags = set()
    for name, cs in SSIM_CASES.items():
        d, h, w = (cs["sp"] if cs["dims"] == 3 else (1,) + cs["sp"])
        for bwd, want in ((False, cs["fwd"]), (True, cs["bwd"])):
            got, (Do, Ho, Wo), kd = ssim_tiling(cs["dims"], cs["n"], cs["c"], d, h, w, cs["k"], bwd)
            assert got == want, (name, bwd, got)
            TH, nWT, nHT, Dc, nDC = got
            seen["wout"].add(Wo)
            seen["th_rem"].add((bwd, TH, Ho % TH != 0))
            if nDC > 1 and Do % Dc:
                flags.add("short_last_chunk")
            if cs["dims"] == 3 and Do < kd:
                flags.add("dout_lt_kd")
            if cs["dims"] == 3 and Dc < kd and Do >= kd:
                flags.add("dc_lt_kd")
        seen["k"].add(cs["k"])
        seen["modes"].add((cs["mode"], cs["dims"], cs["n"] * cs["c"] > 1))
        seen["layouts"].add(cs["layout"])
        seen["grads"].add(cs["grads"])
        seen["rng"].add(cs["rng"])
    assert {31, 32, 33, 65} <= seen["wout"]
    for bwd in (False, True):
        ths = {th for b, th, _ in seen["th_rem"] if b == bwd}
        for th in ths - {1}:
            assert (bwd, th, True) in seen["th_rem"], (bwd, th)
    assert flags == {"short_last_chunk", "dout_lt_kd", "dc_lt_kd"}
    assert {1, 2, 3, 10, 11, 15, 31} <= seen["k"]
    assert {(0, 2, True), (0, 3, True), (1, 2, True), (2, 3, True)} <= seen["modes"]
    assert seen["layouts"] == {"dense", "cl", "slice"} and seen["grads"] == {"both", "x", "y"}
    assert seen["rng"] == {1.0, 255.0}
    assert any(cs["sp"] == (96, 96, 96) and cs["k"] == 11 and cs["n"] == 2 for cs in SSIM_CASES.values())


@pytest.mark.parametrize("soft", [False, True])
def test_ss_reference_bounds_hold_for_fp32_evaluation(soft):
    """an fp32 evaluation of loss_partials_ss's expressions on the CPU stays within the reference bounds, and so does
    loss_bwd_ss's expression"""
    cs = L(2, (3, 11, 13), 1, F32 if soft else I64)
    z, t = loss_logits(cs, 4, "cpu")
    ref = ss_reference(z, t)
    zz, tt = z.reshape(2, -1), t.reshape(2, -1).float()
    p = 1 / (1 + torch.exp(-zz))
    d = p - tt
    d2 = d * d
    got = torch.stack([(p * tt).double().sum(), p.double().sum(), tt.double().sum(), (d2 * tt).double().sum(),
                       (d2 * (1 - tt)).double().sum(), torch.tensor(float(zz.numel()), dtype=F64)])
    check_partials(got, None, ref, 1, 1, soft, "cpu fp32")
    wf, wb, gs = f32(0.1 / 3000), f32(0.9 / 40000), f32(0.7)
    g32 = 2 * (p - tt) * (wf * tt + wb * (1 - tt)) * p * (1 - p) * gs
    want, tol = ss_bwd_reference(ref, wf, wb, gs)
    check_dz(g32, want, tol, "cpu fp32 ss backward")


def test_ext_finalize_restatement_matches_the_oracle_and_the_kernel_forms():
    """value of the restatement at the fp64 partial sums equals oracle.losses_ext in fp64, and its lcoef reproduce the
    oracle's autograd gradient through the closed forms the backward kernels evaluate"""
    from oracle import losses_ext as ox
    g = torch.Generator().manual_seed(3)
    z = torch.randn(2, 1, 4, 9, 11, generator=g, dtype=F64) * 2
    for soft in (False, True):
        t = (torch.rand(2, 4, 9, 11, generator=g) < 0.4).double()
        if soft:
            t = torch.rand(2, 4, 9, 11, generator=g, dtype=F64)
        p = torch.sigmoid(z[:, 0])
        part = [float((p * t).sum()), float(p.sum()), float(t.sum()), float(((p - t) ** 2 * t).sum()),
                float(((p - t) ** 2 * (1 - t)).sum()), float(t.numel()), 0.0]
        for terms, fn, kw in ((JACCARD, ox.binary_jaccard, {}), (ELDICE, ox.binary_eldice, {}),
                              (TVERSKY, ox.binary_tversky, dict(alpha=0.3, beta=0.7)),
                              (SS, ox.binary_ss, dict(r=0.1))):
            zz = z.clone().requires_grad_(True)
            v = fn(zz, t, dtype=F64, **kw)
            v.backward()
            val, lc = ext_finalize_reference(part, 1, terms, None, kw.get("beta", 0.0),
                                             kw.get("alpha", kw.get("r", 0.0)))
            assert math.isclose(val, float(v.detach()), rel_tol=1e-12), (terms, soft)
            q = p * (1 - p)
            if terms == SS:
                want = 2 * (p - t) * (lc[0] * t + lc[1] * (1 - t)) * q
            else:
                want = (t * lc[0] + lc[1]) * q
            assert torch.allclose(zz.grad[:, 0], want, rtol=1e-10, atol=1e-14), (terms, soft)
    c = 3
    t = torch.randint(0, c, (2, 4, 9, 11), generator=g)
    t[t == 1] = 0                                        # class 1 absent
    z = torch.randn(2, c, 4, 9, 11, generator=g, dtype=F64)
    alpha = torch.tensor([0.5, 0.875, 1.25])
    zz = z.clone().requires_grad_(True)
    v = ox.multi_eldice(zz, t, alpha, dtype=F64)
    v.backward()
    p = torch.softmax(z, 1)
    oh = F.one_hot(t, c).permute(0, 4, 1, 2, 3).double()
    part = ((p * oh).sum((0, 2, 3, 4)).tolist() + p.sum((0, 2, 3, 4)).tolist() + oh.sum((0, 2, 3, 4)).tolist()
            + [0.0, 0.0, float(t.numel()), 0.0])
    val, lc = ext_finalize_reference(part, c, ELDICE, alpha.tolist())
    assert math.isclose(val, float(v.detach()), rel_tol=1e-12)
    a, b = torch.tensor(lc[:c], dtype=F64), torch.tensor(lc[c:2 * c], dtype=F64)
    o = oh * a.view(1, c, 1, 1, 1) + b.view(1, c, 1, 1, 1)
    want = p * (o - (o * p).sum(1, keepdim=True))
    assert torch.allclose(zz.grad, want, rtol=1e-10, atol=1e-14)


def test_ext_finalize_branches_of_the_restatement():
    """the clamped cases have no gradient, the NaN cases a NaN value; the SS weights are the fg / bg weights"""
    for name, (c, terms, part, al, gm, af, br) in FIN_CASES.items():
        val, lc = ext_finalize_reference(part, c, terms, al, gm, af)
        if br == "nan":
            assert math.isnan(val), name
        else:
            assert math.isfinite(val), name
        if br == "clamp":
            assert all(v == 0.0 for v in lc), name
        if br == "clamp_min" and c == 1:
            assert lc[1] == 0.0 and lc[0] != 0.0, name
        if br == "clamp_min" and c > 1:
            assert lc[c - 1] == 0.0 and lc[2 * c - 1] == 0.0, name
        if br == "absent":
            k = c // 2
            assert lc[k] == 0.0 and lc[c + k] == 0.0, name


@pytest.mark.parametrize("name", ["c3", "len4097", "per_image_n3", "ignore_255", "per_image_all_ignored",
                                  "absent_classes", "e_zero", "c1024_short"])
def test_lovasz_restatement_matches_the_oracle(name):
    """coef seg_scale sgn of the restatement within 4u of fp64 autograd of oracle.losses_ext.lovasz_softmax, and the
    loss within the fp64 chain term"""
    cs = dict(LOVASZ_CASES[name])
    if cs["c"] == 1024:
        cs["vox"] = 5
    z, t = lovasz_operands(cs, 7)
    r = lovasz_restate(z, t, cs["per_image"], cs["ignore"])
    dz = lovasz_dz(z, t, r["coef"], r["scale"], 1.0, cs["per_image"])
    v, go = lovasz_oracle(z, t, cs["per_image"], cs["ignore"])
    check_close(dz, go, 4 * U * go.abs() + 1e-300, name)
    assert abs(r["loss"] - v) <= gamma64(2 * r["len"] + 8) * r["abs"] + 1e-300


@pytest.mark.parametrize("name", ["len4097", "e_zero_and_negative", "gts_zero", "per_image_bg_and_ignored",
                                  "ignore_0", "quantised_ties"])
def test_hinge_restatement_matches_the_oracle(name):
    cs = HINGE_CASES[name]
    z, t = hinge_operands(cs, 8)
    r = hinge_restate(z, t, cs["per_image"], cs["ignore"])
    v, go = hinge_oracle(z, t, cs["per_image"], cs["ignore"])
    check_close(r["coef"], go, 2 * U * go.abs() + 1e-300, name)
    assert abs(r["loss"] - v) <= gamma64(2 * r["len"] + 8) * r["abs"] + 1e-300
    if name == "gts_zero":
        nz = r["coef"].nonzero()
        assert nz.shape[0] == 1 and float(r["coef"][tuple(nz[0])]) == 1.0


def test_ssim_taps_equal_the_oracle_window():
    from oracle.ssim import gaussian
    from pytorchdeeplearing_b200.ssim import gaussian_taps
    for k in range(1, SS_MAXK + 1):
        assert_bitwise(gaussian_taps(k), gaussian(k), f"taps k={k}")


@pytest.mark.parametrize("dims,k,mode", [(2, 11, 0), (2, 2, 1), (3, 3, 2), (3, 10, 0), (3, 1, 2)])
def test_ssim_restatement_matches_the_oracle(monkeypatch, dims, k, mode):
    """the separable fp64 restatement equals oracle.ssim.ssim in fp64 with its window rebuilt in fp64 from the fp32
    taps: value and autograd gradients"""
    import oracle.ssim as os_
    from pytorchdeeplearing_b200.ssim import gaussian_taps

    def window64(ws, dm):
        gg = gaussian_taps(ws).double()
        w2 = gg[:, None] * gg[None, :]
        return w2 if dm == 2 else gg[:, None, None] * w2[None]
    monkeypatch.setattr(os_, "window", window64)
    cs = SC(dims, 2, 2, (9, 12) if dims == 2 else (7, 8, 10), k, mode, None, None)
    x, y = ssim_images(cs, 5, "cpu")
    Dm, Hm, Wm = ssim_maps(dims, *((1,) + cs["sp"] if dims == 2 else cs["sp"]), k)
    gout = ssim_gout(cs, (Dm, Hm, Wm), 6, "cpu")
    r = ssim_restate(x, y, k, mode, gout)
    x64, y64 = x.double().requires_grad_(True), y.double().requires_grad_(True)
    v = os_.ssim(x64, y64, k, size_average=(mode == 0), dims=dims, dtype=F64)
    (v * gout.double().reshape(v.shape)).sum().backward()
    assert torch.allclose(r["value"].reshape(v.shape), v.detach(), rtol=1e-13, atol=1e-15)
    assert torch.allclose(r["dx"], x64.grad, rtol=1e-11, atol=1e-15)
    assert torch.allclose(r["dy"], y64.grad, rtol=1e-11, atol=1e-15)


@pytest.mark.parametrize("dims,k,mode,rng", [(2, 11, 0, 1.0), (2, 2, 1, 255.0), (3, 3, 2, 1.0), (3, 10, 0, 255.0)])
def test_ssim_bound_holds_for_fp32_evaluation(dims, k, mode, rng):
    """the derivation with u = 2^-24 bounds an fp32 evaluation of the restatement against the fp64 one (value, acc,
    coef, dx, dy); and with u = 2^-53 the fp64 term stays below 1/4 fp32 ulp at 99% of the 0-1 gradients"""
    cs = SC(dims, 2, 2, (21, 26) if dims == 2 else (9, 11, 14), k, mode, None, None, rng=rng)
    x, y = ssim_images(cs, 9, "cpu")
    Dm, Hm, Wm = ssim_maps(dims, *((1,) + cs["sp"] if dims == 2 else cs["sp"]), k)
    gout = ssim_gout(cs, (Dm, Hm, Wm), 10, "cpu")
    r64 = ssim_restate(x, y, k, mode, gout)
    r32 = ssim_restate(x, y, k, mode, gout, dtype=F32, u=U)
    check_close(r32["acc"], r64["acc"], r32["dacc"] * 1.01, "fp32 acc")
    check_close(r32["coef"], r64["coef"], r32["dcoef"] * 1.01 + 1e-30, "fp32 coef")
    check_close(r32["dx"], r64["dx"], r32["ddx"] * 1.01 + 1e-30, "fp32 dx")
    check_close(r32["dy"], r64["dy"], r32["ddy"] * 1.01 + 1e-30, "fp32 dy")
    if rng == 1.0:
        quarter = 0.25 * U * r64["dx"].abs()
        assert float((2 * r64["ddx"] <= quarter).double().mean()) >= 0.99


def test_checkers_catch_planted_faults():
    # one ulp of one element of coef / dz / dx
    cs = LOVASZ_CASES["len4097"]
    z, t = lovasz_operands(cs, 7)
    r = lovasz_restate(z, t, False, None)
    bad = r["coef"].clone()
    i = int(bad.reshape(-1).abs().argmax())
    bad.view(-1).view(torch.int32)[i] += 1
    with pytest.raises(AssertionError, match="differ"):
        assert_bitwise(bad, r["coef"], "coef")
    dz = lovasz_dz(z, t, r["coef"], r["scale"], 0.7, False)
    bdz = dz.clone()
    bdz.view(-1).view(torch.int32)[i] -= 1
    with pytest.raises(AssertionError, match="differ"):
        assert_bitwise(bdz, dz, "dz")
    # two tied elements (one foreground, one background) swapped in the sort order
    n = 64
    zq = torch.full((1, n, 2), 0.25)
    tq = torch.zeros(1, n, dtype=I64)
    tq[0, ::2] = 1
    zq[0, ::2, 1] = 0.75                                 # class 1: fg e = |1 - 0.75| = 0.25, bg e = 0.25: all tied
    good = lovasz_restate(zq, tq, False, None)

    def swap(order):
        o = order.clone()
        o[1, [3, 4]] = o[1, [4, 3]]
        return o
    wrong = lovasz_restate(zq, tq, False, None, order_fix=swap)
    with pytest.raises(AssertionError, match="differ"):
        assert_bitwise(wrong["coef"], good["coef"], "swapped ties")
    # one ulp of dx in the SSIM check
    sc = SC(2, 1, 1, (14, 15), 3, 0, None, None)
    x, y = ssim_images(sc, 1, "cpu")
    gout = ssim_gout(sc, ssim_maps(2, 1, 14, 15, 3), 2, "cpu")
    rs = ssim_restate(x, y, 3, 0, gout)
    dx = rs["dx"].float()
    check_close(dx, rs["dx"], U * rs["dx"].abs() + 2 * rs["ddx"] * (1 + U), "dx")
    j = int(rs["dx"].reshape(-1).abs().argmax())
    dx.view(-1).view(torch.int32)[j] += 2                # beyond one rounding of the largest element
    with pytest.raises(AssertionError, match="outside the bound"):
        check_close(dx, rs["dx"], U * rs["dx"].abs() + 2 * rs["ddx"] * (1 + U), "dx")
    # one byte of the guard after a workspace, and one element after an output
    ws = GuardedWorkspace(1000, device="cpu")
    assert ws.outside_changed() is None
    ws.buf[WS_BLOCK + 1000] = 0
    with pytest.raises(AssertionError, match=f"element {WS_BLOCK + 1000}"):
        assert_guards(ws, "workspace")
    go = GuardedOut((3, 5), F64, init=0.0, device="cpu")
    go.buf[GUARD + 15] = 0.0
    with pytest.raises(AssertionError, match=f"element {GUARD + 15}"):
        assert_guards(go, "coef")


# ======================================================================================= GPU part
@pytest.fixture(scope="module")
def be():
    from pytorchdeeplearing_b200 import runtime
    return runtime.get_backend(torch.zeros(1, device="cuda"))


def _ss_partials(be, z, t):
    n = z.shape[0]
    part = GuardedOut((be.part_size(1),), F64, init=0.0)
    metric = GuardedOut((n, 1, 3), F64, init=0.0)
    ins = Inputs(z=z, t=t)
    dev, st = _stream(be, z)
    _rc(be, be.lib.b200seg_loss_partials_ss(z.data_ptr(), t.data_ptr(), be._label_dtype(t), n, z.numel() // n,
                                            part.ptr, metric.ptr, dev, st), "loss_partials_ss")
    torch.cuda.synchronize()
    ins.check("loss_partials_ss")
    assert_guards(part, "part")
    assert_guards(metric, "metric")
    return part.view, metric.view


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SS_CASES))
def test_loss_partials_ss_against_fp64(be, name):
    n, sp, ldt = SS_CASES[name]
    z, t = loss_logits(L(n, sp, 1, ldt), 41, "cuda")
    part, metric = _ss_partials(be, z, t)
    ref = ss_reference(z, t)
    check_partials(part, metric.cpu(), {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in ref.items()}, 1,
                   chain_len(ref["vox"], n, 1), ldt == F32, name)
    assert float(part[6]) == 0.0


def _finalize(be, part_l, c, terms, alpha, gamma, alpha_f):
    part = torch.tensor(part_l, dtype=F64, device="cuda")
    al = torch.tensor(alpha if alpha is not None else [1.0] * c, dtype=F32, device="cuda")
    loss, lcoef = out32(()), out32((2 * c + 3 if c > 1 else 5,))
    ins = Inputs(part=part, alpha=al)
    dev, st = _stream(be, part)
    _rc(be, be.lib.b200seg_loss_finalize(part.data_ptr(), c, terms, al.data_ptr(), ctypes.c_float(gamma),
                                         ctypes.c_float(alpha_f), loss.out.data_ptr(), lcoef.out.data_ptr(), dev, st),
        "loss_finalize")
    torch.cuda.synchronize()
    ins.check("loss_finalize")
    assert_guards(loss, "loss")
    assert_guards(lcoef, "lcoef")
    return float(loss.out), lcoef.out.double().tolist(), lcoef.out


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FIN_CASES))
def test_loss_finalize_ext_within_one_ulp(be, name):
    c, terms, part, alpha, gamma, alpha_f, br = FIN_CASES[name]
    loss, lc, _ = _finalize(be, part, c, terms, alpha, gamma, alpha_f)
    val, want = ext_finalize_reference(part, c, terms, alpha, gamma, alpha_f)
    assert within_ulp(loss, val), (name, loss, val)
    if br == "nan" and c == 1:
        # dsc + s >= 1: torch's clamp passes no gradient to the NaN, but its pow backward then multiplies that zero
        # by NaN; the kernel writes zero coefficients
        assert all(v == 0.0 for v in lc), (name, lc)
        return
    for i, (gv, wv) in enumerate(zip(lc, want)):
        assert within_ulp(gv, wv), (name, i, gv, wv)
    if br == "clamp":
        assert all(v == 0.0 for v in lc[:2 * c]), name


@pytest.mark.gpu
@pytest.mark.parametrize("soft", [False, True], ids=["hard", "soft"])
@pytest.mark.parametrize("n,sp", [(2, (96, 96, 96)), (5, (7, 33, 41)), (1, (1, 10, 20))])
def test_loss_bwd_ss_at_kernel_lcoef(be, n, sp, soft):
    z, t = loss_logits(L(n, sp, 1, F32 if soft else I64), 42, "cuda")
    part, _ = _ss_partials(be, z, t)
    ref = ss_reference(z, t)
    for r in (f32(0.1), f32(0.5)):
        _, lc, lcoef = _finalize(be, part.tolist(), 1, SS, None, 0.0, r)
        for gs in (1.0, 0.7):
            gsc = torch.tensor([gs], dtype=F32, device="cuda")
            dz = out32(z.shape)
            ins = Inputs(z=z, t=t, lcoef=lcoef, gs=gsc)
            dev, st = _stream(be, z)
            _rc(be, be.lib.b200seg_loss_bwd_ss(z.data_ptr(), t.data_ptr(), be._label_dtype(t), z.numel(),
                                               lcoef.data_ptr(), gsc.data_ptr(), dz.out.data_ptr(), dev, st), "bwd_ss")
            torch.cuda.synchronize()
            ins.check("loss_bwd_ss")
            assert_guards(dz, "dz")
            want, tol = ss_bwd_reference(ref, lc[0], lc[1], f32(gs))
            check_dz(dz.out.reshape(want.shape), want, tol, f"ss bwd r={r} gs={gs}")


E2E_EXT = [("BinaryJaccardLoss", JACCARD), ("BinaryELDiceLoss", ELDICE), ("BinaryTverskyLoss", TVERSKY),
           ("BinarySSLoss", SS)]


def _dev_logits(z, channels_last):
    if channels_last:
        z = z.permute(0, 2, 3, 4, 1).contiguous().permute(0, 4, 1, 2, 3)
    return z.detach().requires_grad_(True)


@pytest.mark.gpu
@pytest.mark.parametrize("channels_last", [False, True], ids=["ncdhw", "ndhwc"])
@pytest.mark.parametrize("name,terms", E2E_EXT)
def test_binary_ext_modules_against_fp64_autograd(name, terms, channels_last):
    """b200.<Loss> at 2x1x96^3 against fp64 autograd of oracle.losses_ext: per element within the backward bound at
    the fp64 lcoef plus the effect of the lcoef's own error (the partial sums' bounds through the finalize, first
    order, and its fp32 rounding); the value within the same propagated bound"""
    import pytorchdeeplearing_b200 as b200
    from oracle import losses_ext as ox
    z, t = loss_logits(L(2, (96, 96, 96), 1), 43, "cuda")
    zn = _dev_logits(z.permute(0, 4, 1, 2, 3), channels_last)
    mod = getattr(b200, name)()
    loss = mod(zn, t)
    loss.backward()
    z64 = zn.detach().double().requires_grad_(True)
    fn = {JACCARD: ox.binary_jaccard, ELDICE: ox.binary_eldice, TVERSKY: ox.binary_tversky, SS: ox.binary_ss}[terms]
    # the oracle at the fp32 parameters the kernel receives (its fp64 0.3 / 0.7 / 0.1 differ by one fp32 rounding)
    kw = dict(alpha=f32(mod.alpha), beta=f32(mod.beta)) if terms == TVERSKY else \
        (dict(r=f32(mod.r)) if terms == SS else {})
    v64 = fn(z64, t, dtype=F64, **kw)
    v64.backward()
    gamma, alpha_f = (f32(mod.beta), f32(mod.alpha)) if terms == TVERSKY else (0.0, f32(mod.r) if terms == SS else 0.0)
    ref = ss_reference(z, t) if terms == SS else loss_reference(z, t, 2.0)
    chain = chain_len(ref["vox"], 2, 1)
    tol = (ref["err"] + chain * U / (1 - chain * U) * (ref["abs"] + ref["err"])).tolist()
    part = ref["part"].tolist() + [0.0]
    fn_part = lambda p: ext_finalize_reference(p, 1, terms, None, gamma, alpha_f)      # noqa: E731
    val, lc = fn_part(part)
    dv, dl = sensitivity(fn_part, part, tol + [0.0])
    da, db = dl[0] + U * abs(lc[0]), dl[1] + U * abs(lc[1])
    if terms == SS:
        want, btol = ss_bwd_reference(ref, lc[0], lc[1], 1.0, da, db)
        want, btol = want.reshape(-1), btol.reshape(-1)
    else:
        want, btol = bwd_reference(ref, lc, 1, 2.0, 1.0)
        p = ref["p"]
        btol = (btol[..., 0] + (ref["t"].abs() * da + db) * p * (1 - p) * 1.01).reshape(-1)
    got = zn.grad.permute(0, 2, 3, 4, 1).reshape(-1)
    auto = z64.grad.permute(0, 2, 3, 4, 1).reshape(-1)
    assert float((auto - want.reshape(-1)).abs().max()) <= 1e-12 * float(want.abs().max()) + 1e-300
    check_dz(got, auto, btol + 1e-13 * auto.abs(), name)
    v = float(v64.detach())
    assert abs(float(loss) - v) <= dv + U * abs(v) + 1e-12 * abs(v), (float(loss), v, dv)


@pytest.mark.gpu
@pytest.mark.parametrize("channels_last", [False, True], ids=["ncdhw", "ndhwc"])
@pytest.mark.parametrize("c", [3, 9])
def test_mutil_eldice_module_against_fp64_autograd(c, channels_last):
    import pytorchdeeplearing_b200 as b200
    from oracle import losses_ext as ox
    g = torch.Generator(device="cuda").manual_seed(44 + c)
    sp = (128, 112, 112)
    z = (torch.randn((1,) + sp + (c,), generator=g, device="cuda") * 3).float()
    t = torch.randint(0, c, (1,) + sp, generator=g, device="cuda")
    t[t == 1] = 0                                        # an absent class
    alpha = torch.tensor([0.5 + 0.25 * k for k in range(c)], device="cuda")
    zn = _dev_logits(z.permute(0, 4, 1, 2, 3), channels_last)
    mod = b200.MutilELDiceLoss(alpha)
    loss = mod(zn, t)
    loss.backward()
    z64 = zn.detach().double().requires_grad_(True)
    v64 = ox.multi_eldice(z64, t, alpha.double(), dtype=F64)
    v64.backward()
    ref = loss_reference(z, t, 2.0)
    chain = chain_len(ref["vox"], 1, c)
    tol = (ref["err"] + chain * U / (1 - chain * U) * (ref["abs"] + ref["err"])).tolist()
    part = ref["part"].tolist()
    fn_part = lambda p: ext_finalize_reference(p, c, ELDICE, alpha.tolist())            # noqa: E731
    val, lc = fn_part(part)
    dv, dl = sensitivity(fn_part, part, tol)
    want, btol = bwd_reference(ref, lc, c, 2.0, 1.0)
    da = torch.tensor(dl[:c] + U * np.abs(lc[:c]), dtype=F64, device="cuda")
    db = torch.tensor(dl[c:2 * c] + U * np.abs(lc[c:2 * c]), dtype=F64, device="cuda")
    do = ref["oh"] * da + db
    p = ref["p"]
    btol = btol + p * (do + (do * p).sum(-1, keepdim=True)) * 1.01
    got = zn.grad.permute(0, 2, 3, 4, 1).reshape(want.shape)
    auto = z64.grad.permute(0, 2, 3, 4, 1).reshape(want.shape)
    check_dz(got, auto, btol + 1e-13 * auto.abs(), f"MutilELDice c={c}")
    v = float(v64.detach())
    assert abs(float(loss) - v) <= dv + U * abs(v) + 1e-12 * abs(v), (float(loss), v, dv)


# ---------------------------------------------------------------------------------------------------------- Lovasz
def _lovasz_call(be, z, t, cs):
    n, vox, c = z.shape
    pi = 1 if cs["per_image"] else 0
    nb = int(be.lib.b200seg_lovasz_workspace(n, vox, c, pi))
    ws = GuardedWorkspace(nb)
    loss, coef, scale = out32(()), out32((n, vox, c)), out32(((n if pi else 1) * c,))
    ins = Inputs(z=z, t=t)
    dev, st = _stream(be, z)
    ig = cs["ignore"]
    _rc(be, be.lib.b200seg_lovasz_fwd(z.data_ptr(), t.data_ptr(), n, vox, c, pi, 0 if ig is None else 1,
                                      0 if ig is None else int(ig), ws.ptr, nb, loss.out.data_ptr(),
                                      coef.out.data_ptr(), scale.out.data_ptr(), dev, st), "lovasz_fwd")
    torch.cuda.synchronize()
    ins.check("lovasz_fwd")
    for gb, what in ((ws, "workspace"), (loss, "loss"), (coef, "coef"), (scale, "seg_scale")):
        assert_guards(gb, what)
    return loss.out, coef.out, scale.out


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(LOVASZ_CASES))
def test_lovasz_exact(be, name):
    cs = LOVASZ_CASES[name]
    z, t = lovasz_operands(cs, 51)
    zc, tc = z.cuda(), t.cuda()
    loss, coef, scale = _lovasz_call(be, zc, tc, cs)
    r = lovasz_restate(z, t, cs["per_image"], cs["ignore"])
    assert_bitwise(coef.cpu(), r["coef"], f"{name}: coef")
    assert_bitwise(scale.cpu(), r["scale"], f"{name}: seg_scale")
    n, vox, c = z.shape
    for gs in (1.0, 0.7):
        gsc = torch.tensor([gs], dtype=F32, device="cuda")
        dz = out32(z.shape)
        ins = Inputs(z=zc, t=tc, coef=coef, scale=scale, gs=gsc)
        dev, st = _stream(be, zc)
        _rc(be, be.lib.b200seg_lovasz_bwd(zc.data_ptr(), tc.data_ptr(), n, vox, c, 1 if cs["per_image"] else 0,
                                          coef.data_ptr(), scale.data_ptr(), gsc.data_ptr(), dz.out.data_ptr(), dev,
                                          st), "lovasz_bwd")
        torch.cuda.synchronize()
        ins.check("lovasz_bwd")
        assert_guards(dz, "dz")
        assert_bitwise(dz.out.cpu(), lovasz_dz(z, t, r["coef"], r["scale"], gs, cs["per_image"]), f"{name}: dz")
        if gs == 1.0:
            dz1 = dz.out.cpu()
    dev = "cuda" if cs.get("big") else "cpu"
    v, go = lovasz_oracle(z, t, cs["per_image"], cs["ignore"], dev)
    check_close(dz1, go, 4 * U * go.abs() + 1e-300, f"{name}: dz vs fp64 oracle")
    fp64 = 2 * gamma64(r["len"] + 2 * lovasz_tiles(vox, n, cs["per_image"])[0] + 8) * r["abs"]
    assert within_ulp(float(loss), v) or abs(float(loss) - v) <= float(np.spacing(np.float32(abs(v)))) + fp64, \
        (name, float(loss), v)


@pytest.mark.gpu
@pytest.mark.parametrize("nseg,ln", [(1, 1), (3, 4095), (2, 4097), (1, 3 * K_TILE + 1)])
def test_radix_sort_workspace_is_exact(be, nseg, ln):
    """the sort alone in an exact-size guarded workspace: the result is torch's stable sort"""
    g = torch.Generator().manual_seed(nseg * ln)
    keys = torch.randint(0, 6, (nseg, ln), generator=g).int() * 0x01010101
    vals = torch.arange(nseg * ln, dtype=torch.int32).reshape(nseg, ln)
    kc, vc = keys.cuda(), vals.cuda()
    nb = int(be.lib.b200seg_radix_sort_workspace(nseg, ln))
    ws = GuardedWorkspace(nb)
    ko, vo = GuardedOut((nseg, ln), F32), GuardedOut((nseg, ln), F32)
    ins = Inputs(k=kc, v=vc)
    dev, st = _stream(be, kc)
    _rc(be, be.lib.b200seg_radix_sort_pairs(kc.data_ptr(), vc.data_ptr(), ko.ptr, vo.ptr, nseg, ln, ws.ptr, nb, dev,
                                            st), "radix_sort")
    torch.cuda.synchronize()
    ins.check("radix_sort")
    for gb, what in ((ws, "workspace"), (ko, "keys"), (vo, "vals")):
        assert_guards(gb, what)
    s = torch.sort(keys.long() & 0xFFFFFFFF, dim=1, stable=True)
    assert torch.equal(ko.view.cpu().view(torch.int32).long() & 0xFFFFFFFF, s.values)
    assert torch.equal(vo.view.cpu().view(torch.int32), torch.gather(vals, 1, s.indices))


# ---------------------------------------------------------------------------------------------------------- hinge
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(HINGE_CASES))
def test_lovasz_hinge_exact(be, name):
    cs = HINGE_CASES[name]
    z, t = hinge_operands(cs, 61)
    zc, tc = z.cuda(), t.cuda()
    n, vox = z.shape
    pi = 1 if cs["per_image"] else 0
    nb = int(be.lib.b200seg_lovasz_hinge_workspace(n, vox, pi))
    ws = GuardedWorkspace(nb)
    loss, coef, bad = out32(()), out32((n, vox)), GuardedOut((1,), I64)
    ins = Inputs(z=zc, t=tc)
    dev, st = _stream(be, zc)
    ig = cs["ignore"]
    _rc(be, be.lib.b200seg_lovasz_hinge_fwd(zc.data_ptr(), tc.data_ptr(), n, vox, pi, 0 if ig is None else 1,
                                            0 if ig is None else int(ig), ws.ptr, nb, loss.out.data_ptr(),
                                            coef.out.data_ptr(), bad.ptr, dev, st), "hinge_fwd")
    torch.cuda.synchronize()
    ins.check("hinge_fwd")
    for gb, what in ((ws, "workspace"), (loss, "loss"), (coef, "coef"), (bad, "bad")):
        assert_guards(gb, what)
    r = hinge_restate(z, t, cs["per_image"], ig)
    assert_bitwise(coef.out.cpu(), r["coef"], f"{name}: coef")
    assert int(bad.view[0]) == r["bad"]
    gsc = torch.tensor([0.7], dtype=F32, device="cuda")
    dz = out32((n, vox))
    ins = Inputs(coef=coef.out, gs=gsc)
    _rc(be, be.lib.b200seg_lovasz_hinge_bwd(coef.out.data_ptr(), n * vox, gsc.data_ptr(), dz.out.data_ptr(), dev, st),
        "hinge_bwd")
    torch.cuda.synchronize()
    ins.check("hinge_bwd")
    assert_guards(dz, "dz")
    assert_bitwise(dz.out.cpu(), torch.tensor(0.7, dtype=F32) * r["coef"], f"{name}: dz")
    if name == "gts_zero":
        nz = coef.out.cpu().nonzero()
        assert nz.shape[0] == 1 and float(coef.out.cpu()[tuple(nz[0])]) == 1.0
    if r["bad"]:
        return                                           # the oracle reads labels other than 0 / 1 as weights
    v, go = hinge_oracle(z, t, cs["per_image"], ig, "cuda" if cs.get("big") else "cpu")
    check_close(coef.out.cpu(), go, 2 * U * go.abs() + 1e-300, f"{name}: coef vs fp64 oracle")
    fp64 = 2 * gamma64(r["len"] + 2 * lovasz_tiles(vox, n, cs["per_image"])[0] + 8) * r["abs"]
    assert within_ulp(float(loss.out), v) or \
        abs(float(loss.out) - v) <= float(np.spacing(np.float32(abs(v)))) + fp64, (name, float(loss.out), v)


# ---------------------------------------------------------------------------------------------------------- SSIM
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SSIM_CASES))
def test_ssim_against_fp64_restatement(be, name):
    from pytorchdeeplearing_b200.ssim import gaussian_taps
    cs = SSIM_CASES[name]
    dims, n, c, k, mode = cs["dims"], cs["n"], cs["c"], cs["k"], cs["mode"]
    x, y = ssim_images(cs, 71, "cuda")
    d, h, w = cs["sp"] if dims == 3 else (1,) + cs["sp"]
    maps = ssim_maps(dims, d, h, w, k)
    gout = ssim_gout(cs, maps, 72, "cuda")
    r = ssim_restate(x, y, k, mode, gout)
    geom, sx = be._ssim_geom(x)
    _, sy = be._ssim_geom(y)
    nmap = n * c * math.prod(maps)
    nb = int(be.lib.b200seg_ssim_workspace(*geom, k))
    ws = GuardedWorkspace(nb)
    coef = GuardedOut((4, nmap), F64)
    taps = gaussian_taps(k)
    tp = (ctypes.c_float * k)(*taps.tolist())
    ins = Inputs(x=x, y=y, gout=gout)
    dev, st = _stream(be, x)
    _rc(be, be.lib.b200seg_ssim_fwd(dims, x.data_ptr(), ctypes.cast(sx, ctypes.c_void_p), y.data_ptr(),
                                    ctypes.cast(sy, ctypes.c_void_p), *geom[1:], k, ctypes.cast(tp, ctypes.c_void_p),
                                    coef.ptr, ws.ptr, nb, dev, st), "ssim_fwd")
    nacc = {0: 2, 1: n, 2: n * maps[2]}[mode]
    nval = {0: 1, 1: n, 2: n * maps[2]}[mode]
    acc, value = GuardedOut((nacc,), F64), out32((nval,))
    _rc(be, be.lib.b200seg_ssim_finalize(*geom, k, int(mode == 0), 1, ws.ptr, nb, acc.ptr, value.out.data_ptr(), dev,
                                         st), "ssim_finalize")
    gx = out32(tuple(x.shape)) if cs["grads"] in ("both", "x") else None
    gy = out32(tuple(x.shape)) if cs["grads"] in ("both", "y") else None
    _rc(be, be.lib.b200seg_ssim_bwd(dims, x.data_ptr(), ctypes.cast(sx, ctypes.c_void_p), y.data_ptr(),
                                    ctypes.cast(sy, ctypes.c_void_p), *geom[1:], k, ctypes.cast(tp, ctypes.c_void_p),
                                    coef.ptr, int(mode == 0), gout.data_ptr(), acc.ptr,
                                    gx.out.data_ptr() if gx else None, gy.out.data_ptr() if gy else None, dev, st),
        "ssim_bwd")
    torch.cuda.synchronize()
    ins.check("ssim")
    for gb, what in ((ws, "workspace"), (coef, "coef"), (acc, "acc"), (value, "value"), (gx, "dx"), (gy, "dy")):
        if gb is not None:
            assert_guards(gb, what)
    check_close(coef.view, r["coef"], 2 * r["dcoef"] * 1.01 + 1e-300, f"{name}: coef")
    got_acc = acc.view[:1] if mode == 0 else acc.view
    check_close(got_acc, r["acc"].reshape(-1), 2 * r["dacc"].reshape(-1) * 1.01 + 1e-300, f"{name}: acc")
    if mode == 0:
        assert float(acc.view[1]) == r["count"]
    want_v = r["value"].reshape(-1)
    check_close(value.out, want_v, U * want_v.abs() + 2 * r["dacc"].reshape(-1) / r["count"] * 1.01 + 1e-45,
                f"{name}: value")
    for gb, key in ((gx, "dx"), (gy, "dy")):
        if gb is not None:
            wv = r[key].reshape(-1)
            check_close(gb.out.reshape(-1), wv, U * wv.abs() + 2 * r["d" + key].reshape(-1) * (1 + U) + 1e-45,
                        f"{name}: {key}")
