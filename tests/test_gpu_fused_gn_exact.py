"""The fused input block (csrc/stem_gn.cu) and the fused first layer of up_tr32 (csrc/up_gn.cu) against independent
fp64 references, bit for bit where the operands allow it.

1. Exact design.  Both kernel families recompute a convolution they never store, then apply one GroupNorm, dropout and
   ReLU.  The statistics and the backward sums are inputs to APPLY, BSUMS and BWD, so the test chooses them as
   test_gpu_gn_exact.py does (dyadic means, var + eps = 4^-k, short dyadic gamma, dropout scale 0 or 1.25); beta is an
   odd multiple of 2^-9, moved by 2^-8 in any channel where some y still sits on -B/A (off_thresholds).  The convolution
   operands come from grids (grid()): the stem image from {-16 .. 16} 2^-2 (or an fp32 image with full mantissas that
   the kernel rounds to bf16), the 3x3x3 weights from {-8 .. 8} 2^-5, the 1x1x1 weights from {-32 .. 32} 2^-5, the
   up_tr32 input from {-4 .. 4} 2^-2 and its weights from {-16 .. 16} 2^-5, biases from {-16 .. 16} 2^-7.  Then the
   fp32 conv output is exact, and so is every fmaf(y, A, B), ReLU sum and dy = (m ? g P : 0) + fmaf(y, Q, R).  Every
   such precondition is asserted from the actual operands as sum |terms| < 2^24 q for the terms' common quantum q.
   |y| >= 2 occurs, so the bf16 rounding of y meets exact ties, and so does the bf16 rounding of dy in the dense
   cases; the test counts them and asserts there are some, so round-to-nearest-even is told apart from truncation.
   The statistics and backward-sum partials are fp32 per CTA and sample, then fp64: their bound comes from the
   kernels' tile walk, restated below (stem_walk, up_walk).  The stem statistics use a second, coarse operand set
   (x from {-2 .. 2}, w from {-2 .. 2} 2^-2, biases from {-4 .. 4} 2^-2) whose squares stay below 2^24 quanta at the
   network shapes; the full-mantissa image is held to the fp32 chain bound of check_stats, and so are its backward
   sums and weight gradients.  The weight gradients at the large shapes run with backward sums of zero (m1 = m2 = 0,
   so Q = R = 0) and a sparse g, and are exact.  The dense Q, R form (cases marked dense) is exact in APPLY, BSUMS and
   the parameter gradients; its dy is dense, so the weight gradients (and up_tr32's dx) are held to the fp32 chain
   bounds stated in stem_dw_chain / up_dw_chain (dx: 128 products and one bf16 rounding).
2. Every pass at the network and edge shapes, on guarded, pitched buffers: the output goes into one half of a
   32-channel buffer whose other half and guard bands keep a NaN pattern; g is read from one half of a concat
   gradient whose other half holds the large finite sentinel IN_FILL; weight and parameter gradients are added onto
   nonzero prefills.  The rejected arguments return B200SEG_EINVAL, launch nothing and write nothing.
3. One ReLU mask from forward to backward (test_relu_mask_forward_equals_backward_and_z0_is_masked): beta puts
   fmaf(y0, A, B) at exactly -1 ulp(B), 0 or +1 ulp(B) for a y0 that occurs at NTHR planted voxels per (n, c), where g
   is a distinct power of two (zero elsewhere).  APPLY's zero / nonzero output is the forward mask, BSUMS's sum g m is
   decoded bit by bit, and BWD's exact weight (and data) gradient must equal the fp64 reference built from the
   forward mask; z = 0 is masked in every pass.
4. The whole block against fp64 torch autograd (test_block_against_fp64_autograd): the kernels' own passes chained
   with realistic data and GN_EPS = 1e-5 at 2 x 96^3 (stem) and 2 x 48^3 (up_tr32), with the bounds derived in
   oracle_bounds.

The CPU part (design preconditions for 132 and 114 SMs, tile-walk coverage, checker sensitivity) runs everywhere; the
GPU part is marked `gpu`."""
import functools
import math

import pytest
import torch
import torch.nn.functional as F

from emu_backend import K3, K1, DOWN, UP
from test_gpu_conv_exact import Guarded, assert_bitwise, assert_guards, first_mismatch, grid, ref_wgrad, check_stats
from test_gpu_conv_exact import GUARD, IN_FILL
from test_gpu_gn_exact import quantum, assert_exact_fp32, gn_branch, bwd_coefs, param_contribs, assert_equal64
from test_gpu_gn_exact import check_pgrad, decode_mask, assert_same_mask, flat, assert_flat_guards
from test_gpu_gn_exact import per_channel, ulp32, GROUPS, EPS, U

BF, F32 = torch.bfloat16, torch.float32
C = 16                        # output channels of both fused families
CI = 32                       # up_tr32's input channels
# the (channel pitch, channel offset) layouts the exact tests run the fused kernels' outputs and upstream gradients at.
# They include the networks' own: VNet3d's input block writes the skip half of a 32-channel concat and ResNet3d's a
# contiguous buffer; its g arrives contiguous from the next layer's data gradient; up_tr32 writes the left half of its
# concat, reads the left half of the concat gradient and writes a contiguous dx.  (CI + 16, None): the case's dx_off.
LAYOUTS = {"stem_gn out": ((C + 16, 16), (C, 0)), "stem_gn g": ((C + 16, 0), (C, 0)),
           "up_gn out": ((C + 16, 0),), "up_gn g": ((C + 16, 0),), "up_gn dx": ((CI + 16, None), (CI, 0))}
SM_TH = 8                     # stem tile rows (stem_mma.cuh:10)
PW_TILE, UB_TILE = 512, 128   # up_gn tiles (pw_mma.cuh:11, up_gn.cu:33)
EINVAL = -1                   # B200SEG_EINVAL (include/b200seg.h)
SMS_CHECKED = (132, 114)      # H100 SXM, H100 PCIe


# ---------------------------------------------------------------------------------------------------------- launch rules
def stem_tile_width(W):
    """stem_tile_width (stem_mma.cuh:103): the widest multiple of 16 up to 128 that divides W, or 0"""
    for c in (128, 112, 96, 80, 64, 48, 32, 16):
        if W % c == 0:
            return c
    return 0


def stem_walk(n, sp, sms, bwd):
    """the stem's tile walk: tiles of 8 rows x TW columns of one (n, d) slice (stem_mma_geom, stem_mma.cuh:110), the
    grid min(tiles, 2 SMs) (stem_grid, stem_mma.cuh:131) or min(tiles, SMs) for BWD (stem_gn.cu:507), and
    ceil(tiles / grid) consecutive tiles per CTA (stem_gn.cu:221)"""
    D, H, W = sp
    tw = stem_tile_width(W)
    tps = D * (H // SM_TH) * (W // tw)
    tiles = n * tps
    g = min(tiles, sms if bwd else 2 * sms)
    return dict(tw=tw, tiles_w=W // tw, tiles=tiles, tps=tps, grid=g, tpc=-(-tiles // g))


def up_walk(n, sp, sms, bwd):
    """up_gn's walk: 512-voxel coarse tiles (128 in BWD, up_gn.cu:368), the grid min(tiles, SMs) (ug_launch,
    up_gn.cu:547) and ceil(tiles / grid) consecutive tiles per CTA (up_gn.cu:198, 369)"""
    V = math.prod(sp)
    tile = UB_TILE if bwd else PW_TILE
    tiles = n * V // tile
    g = min(tiles, sms)
    return dict(tiles=tiles, tps=V // tile, grid=g, tpc=-(-tiles // g), tile=tile)


def crosses_samples(w):
    """does some CTA's tile range hold tiles of two samples?"""
    t = torch.arange(w["tiles"])
    cta, smp = t // w["tpc"], t // w["tps"]
    first = torch.zeros(w["grid"], dtype=torch.long).index_reduce_(0, cta, smp, "amin", include_self=False)
    last = torch.zeros(w["grid"], dtype=torch.long).index_reduce_(0, cta, smp, "amax", include_self=False)
    return bool((first != last).any())


def walk_max(tile_sums, w):
    """max over (CTA, sample) of the per-tile sums of |terms| that one CTA folds for one sample: the largest value an
    fp32 partial of the statistics or backward sums can reach"""
    t = torch.arange(w["tiles"], device=tile_sums.device)
    n = w["tiles"] // w["tps"]
    key = (t // w["tpc"]) * n + t // w["tps"]
    acc = torch.zeros((w["grid"] * n, tile_sums.shape[1]), dtype=tile_sums.dtype, device=tile_sums.device)
    return float(acc.index_add_(0, key, tile_sums).max())


def stem_tile_sums(v, tw):
    """(N, D, H, W, C) -> (tiles, C) in the stem's tile order"""
    N, D, H, W, c = v.shape
    return v.reshape(N, D, H // SM_TH, SM_TH, W // tw, tw, c).sum((3, 5)).reshape(-1, c)


def up_tile_sums(v, tile):
    """fine (N, 2D, 2H, 2W, C) -> (tiles, C): the 8 fine voxels of each coarse voxel, tile coarse voxels per tile"""
    N, fd, fh, fw, c = v.shape
    cv = v.reshape(N, fd // 2, 2, fh // 2, 2, fw // 2, 2, c).sum((2, 4, 6)).reshape(-1, c)
    return cv.reshape(-1, tile, c).sum(1)


# ---------------------------------------------------------------------------------------------------------- cases
def S(n, sp, **kw):
    """one stem case.  n: samples, or a function of the SM count.  flags: x_full (fp32 image with full mantissas),
    bias (False: null b3, b1, db3 and db1), dense (nonzero backward sums: dense Q, R; otherwise Q = R = 0 with a sparse g)"""
    d = dict(n=n, sp=sp, x_full=False, bias=True, dense=False)
    d.update(kw)
    return d


STEM_CASES = {
    "vnet96": S(2, (96, 96, 96)),                          # the benchmark; TW 96
    "tw112": S(1, (128, 112, 112)),                        # TW 112
    "resnet32": S(2, (32, 32, 32)),
    "d1": S(1, (1, 8, 16), dense=True),                    # both neighbour planes are padding; TW 16, one tile
    "tw128_two_tiles": S(3, (2, 16, 256)),                 # TW 128, two tiles across W
    "tw48_three_tiles": S(2, (5, 24, 144)),                # TW 48, three tiles across W
    "cross_samples": S(300, (1, 8, 16)),                   # CTAs cross samples in every pass
    "fewer_tiles_than_sms": S(1, (4, 16, 32)),
    "sms_plus_one": S(lambda s: s + 1, (1, 8, 16)),
    "two_sms_plus_one": S(lambda s: 2 * s + 1, (1, 8, 16)),
    "dense_small": S(2, (2, 8, 16), dense=True),
    "x_full": S(2, (4, 16, 32), x_full=True),
    "null_bias": S(2, (2, 8, 16), bias=False, dense=True),
}


def Up(n, sp, **kw):
    """one up_tr32 case (coarse shape).  flags: x_off (channel offset of x in its 48-channel buffer), dx_off (of dx;
    2 = 4-byte aligned only), bias, dense"""
    d = dict(n=n, sp=sp, x_off=8, dx_off=8, bias=True, dense=False)
    d.update(kw)
    return d


UP_CASES = {
    "vnet48": Up(2, (48, 48, 48)),                         # the benchmark
    "c32": Up(1, (32, 32, 32)),
    "v512": Up(16, (8, 4, 16)),                            # V = 512, the smallest fused size
    "v512_dense": Up(16, (8, 4, 16), dense=True),
    "cross_samples": Up(300, (8, 4, 16)),
    "w48": Up(6, (4, 8, 48)),                              # three 16-voxel groups per row
    "d9": Up(3, (9, 16, 32)),
    "x_offset16": Up(8, (8, 8, 16), x_off=16, dense=True),
    "null_bias": Up(8, (8, 8, 16), bias=False, dense=True),
    "dx_align4": Up(8, (8, 8, 16), dx_off=2),
}

G_RHO = 0.02                  # density of g where Q = R = 0


def shape_of(cs, sms):
    return (cs["n"](sms) if callable(cs["n"]) else cs["n"]), cs["sp"]


# ---------------------------------------------------------------------------------------------------------- design
def ties(v):
    """how many of the exact fp32 values v lie exactly half-way between two bf16 values"""
    return int(((v.float().view(torch.int32) & 0xFFFF) == 0x8000).sum())


def qof(t):
    return quantum(torch.unique(t).cpu())


def bf(t):
    """round-to-nearest-even to bf16 of exact fp32 values, back in fp64"""
    return t.float().bfloat16().double()


def branch(gen, N, vox):
    """gn_branch with beta an odd multiple of 2^-9"""
    b = gn_branch(gen, N, C, vox)
    b["beta"] = (torch.randint(-8, 8, (C,), generator=gen) * 2 + 1).double() / 512
    b["A"] = b["rs_c"] * b["gamma"] * b["scale"]
    b["B"] = (b["beta"] - b["mu_c"] * b["rs_c"] * b["gamma"]) * b["scale"]
    return b


def off_thresholds(b, y):
    """move beta by 2^-8 in the channels where some y of a live channel sits exactly on -B/A, until none does"""
    for _ in range(64):
        z = y * _bc(b["A"], y.device) + _bc(b["B"], y.device)
        hit = ((z == 0) & (_bc(b["scale"], y.device) != 0)).reshape(-1, C).any(0).cpu()
        if not bool(hit.any()):
            return
        b["beta"] = b["beta"] + hit.double() / 256
        b["B"] = (b["beta"] - b["mu_c"] * b["rs_c"] * b["gamma"]) * b["scale"]


def bwd_sums(gen, b, vox, dense):
    """designed backward sums [N][C][3]; dense=False: sum g m = sum g m y = 0, so m1 = m2 = 0 and Q = R = 0"""
    N = b["scale"].shape[0]
    m = (C // GROUPS) * vox
    s3 = torch.randint(-4, 5, (N, C), generator=gen).double() / 4 * vox
    a = torch.randint(-1, 2, (N, C), generator=gen).double() / 16 if dense else torch.zeros(N, C, dtype=torch.float64)
    bb = torch.randint(-1, 2, (N, C), generator=gen).double() / 16 if dense else torch.zeros(N, C, dtype=torch.float64)
    for _ in range(64):           # nudge a until neither m2 nor R nearly cancels
        sums = torch.stack([a * m, bb * m, s3], -1)
        co = bwd_coefs(b, sums, vox)
        t2 = per_channel(co["d3"].abs().view(N, GROUPS, -1).sum(-1) / m, C // GROUPS)
        tr = (b["rs_c"] * co["m1"]).abs() + (b["rs_c"] ** 2 * b["mu_c"] * co["m2"]).abs()
        bad = ((co["m2"].abs() <= 2.0 ** -20 * t2) & (t2 > 0)) | ((co["R"].abs() <= 2.0 ** -20 * tr) & (tr > 0))
        if not bool(bad.any()):
            break
        a = a + (bad & (torch.arange(C) % (C // GROUPS) == 0)).double() / 16
        bb = bb + (bad & (torch.arange(C) % (C // GROUPS) == 1)).double() / 16
    else:
        raise AssertionError("m2 or R nearly cancels in the designed backward sums")
    return sums, co


def _gen_g(gen, shape, dense, device):
    g = torch.randint(-1, 2, shape, generator=gen).double() / 8
    if not dense:
        g = g * (torch.rand(shape, generator=gen) < G_RHO).double()
    return g.to(device)


def _ncdhw(t):
    return t.permute(0, 4, 1, 2, 3)


def _ndhwc(t):
    return t.permute(0, 2, 3, 4, 1)


def _bc(t, dev):
    return t.to(dev).view(t.shape[0], 1, 1, 1, t.shape[1])


def stem_conv(x, w3, w1, b3, b1):
    """fp64 stem outputs (N, D, H, W, 16) of both branches, from weights in parameter layout"""
    xa = _ncdhw(x)
    ya = _ndhwc(F.conv3d(xa, w3, None, padding=1))
    yb = _ndhwc(F.conv3d(xa, w1))
    if b3 is not None:
        ya, yb = ya + b3, yb + b1
    return ya, yb


def up_conv(x, w, b):
    y = _ndhwc(F.conv_transpose3d(_ncdhw(x), w, None, stride=2))
    return y + b if b is not None else y


def gn_side(b, y, g, sums, co, dev):
    """per-element references of one branch: z, the mask, relu(z), dy (exact) and the BSUMS sums"""
    A, B = _bc(b["A"], dev), _bc(b["B"], dev)
    z = y * A + B
    m = z > 0
    dy = torch.where(m, g * _bc(co["P"], dev), 0.0) + y * _bc(co["Q"], dev) + _bc(co["R"], dev)
    gm = torch.where(m, g, 0.0)
    red = (1, 2, 3)
    s = torch.stack([gm.sum(red), (gm * y).sum(red), y.sum(red)], -1)
    return dict(z=z, m=m, relu=z.clamp_min(0), dy=dy, sums=s, gm=gm)


def check_side(b, co, y, g, side, what):
    """the per-element exactness preconditions of one branch"""
    on = _bc(b["scale"], y.device) != 0
    assert not bool(((side["z"] == 0) & on).any()), f"{what}: a y of a live channel sits on a ReLU threshold"
    tb = (b["beta"] * b["scale"]).abs() + (b["mu_c"] * b["rs_c"] * b["gamma"] * b["scale"]).abs()
    assert bool((b["B"].abs() > 2.0 ** -20 * tb)[b["scale"] != 0].all()), f"{what}: B nearly cancels"
    qy = qof(y)
    qz = min(qy * quantum(b["A"]), quantum(b["B"]))
    assert_exact_fp32(float((y.abs() * _bc(b["A"].abs(), y.device) + _bc(b["B"].abs(), y.device)).max()), qz,
                      f"{what} fmaf(y, A, B)")
    qd = min(qof(g) * quantum(co["P"]), qy * quantum(co["Q"]), quantum(co["R"]))
    dev = y.device
    bound = (g.abs() * _bc(co["P"].abs(), dev) + y.abs() * _bc(co["Q"].abs(), dev) + _bc(co["R"].abs(), dev)).max()
    assert_exact_fp32(float(bound), qd, f"{what} dy")
    return qz, qd


def pgrad_exact(pre, terms):
    return float((pre.abs() + terms.abs().sum(0)).max()) < 2 ** 24 * quantum(pre, terms)


@functools.lru_cache(maxsize=1)
def stem_design(name, n, device="cpu", seed=0):
    """the operands and fp64 references of one stem case (everything but the tile-walk bounds)"""
    cs = STEM_CASES[name]
    sp = cs["sp"]
    vox = math.prod(sp)
    gen = torch.Generator().manual_seed(seed)
    x = grid((n,) + sp + (1,), 16, 2, gen)
    if cs["x_full"]:
        mag = torch.rand(x.shape, generator=gen, dtype=torch.float64) * (4 - 0.125) + 0.125
        x = (mag * (torch.randint(0, 2, x.shape, generator=gen).double() * 2 - 1)).float().double()
    w3, w1 = grid((C, 1, 3, 3, 3), 8, 5, gen), grid((C, 1, 1, 1, 1), 32, 5, gen)
    b3, b1 = (grid((C,), 16, 7, gen), grid((C,), 16, 7, gen)) if cs["bias"] else (None, None)
    # the coarse operand set of the statistics
    xs = torch.randint(-2, 3, x.shape, generator=gen).double()
    ws3 = torch.randint(-2, 3, w3.shape, generator=gen).double() / 4
    ws1 = torch.randint(-2, 3, w1.shape, generator=gen).double() / 4
    bs3, bs1 = (torch.randint(-4, 5, (C,), generator=gen).double() / 4 for _ in range(2))
    g = _gen_g(gen, (n,) + sp + (C,), cs["dense"], device)
    br = [branch(gen, n, vox) for _ in range(2)]
    sc = [bwd_sums(gen, b, vox, cs["dense"]) for b in br]
    dev = torch.device(device)
    x, xs = x.to(dev), xs.to(dev)
    xk = bf(x)
    mv = lambda t: None if t is None else t.to(dev)
    ya_raw, yb_raw = stem_conv(xk, mv(w3), mv(w1), mv(b3), mv(b1))
    sa_raw, sb_raw = stem_conv(xs, mv(ws3), mv(ws1), mv(bs3), mv(bs1))
    ys = [bf(ya_raw), bf(yb_raw)]
    for b, y in zip(br, ys):
        off_thresholds(b, y)
    sides =[gn_side(b, y, g, s[0], s[1], dev) for b, y, s in zip(br, ys, sc)]
    pcs = [param_contribs(b, s[0], s[1], vox, s[0][..., 2]) for b, s in zip(br, sc)]
    terms = {k: torch.cat([pcs[0][k], pcs[1][k]]) for k in ("dgamma", "dbeta")}
    terms["db3"], terms["db1"] = pcs[0]["dbias"], pcs[1]["dbias"]
    prefill = {k: torch.randint(-3, 4, (C,), generator=gen).double() * quantum(t) for k, t in terms.items()}
    dys = [bf(s["dy"]) for s in sides]
    ws3_ = dict(kind=K3, dims=3, ca=1, cb=C)
    ws1_ = dict(kind=K1, dims=3, ca=1, cb=C)
    dw3 = ref_wgrad(ws3_, xk, dys[0])
    dw1 = ref_wgrad(ws1_, xk, dys[1])
    dw3_abs = ref_wgrad(ws3_, xk.abs(), dys[0].abs())
    dw1_abs = ref_wgrad(ws1_, xk.abs(), dys[1].abs())
    q_dw = [qof(xk) * min(qof(g) * quantum(s[1]["P"]), qof(y) * quantum(s[1]["Q"]), quantum(s[1]["R"]))
            for s, y in zip(sc, ys)]
    dw_pre = [torch.randint(-3, 4, t.shape, generator=gen).double().to(dev) * q for t, q in ((dw3, q_dw[0]),
                                                                                           (dw1, q_dw[1]))]
    return dict(cs=cs, n=n, sp=sp, vox=vox, x=x, xk=xk, w3=w3, w1=w1, b3=b3, b1=b1, xs=xs, ws3=ws3, ws1=ws1, bs3=bs3,
                bs1=bs1, g=g, br=br, sc=sc, ya_raw=ya_raw, yb_raw=yb_raw, sa_raw=sa_raw, sb_raw=sb_raw, ys=ys,
                sides=sides, terms=terms, prefill=prefill, dys=dys, dw=[dw3, dw1], dw_abs=[dw3_abs, dw1_abs],
                q_dw=q_dw, dw_pre=dw_pre)


def check_stem_design(d, sms):
    """every exactness precondition of a stem case; -> the set of comparisons that are held to a bound instead"""
    cs, n, sp = d["cs"], d["n"], d["sp"]
    inexact = set()
    w = stem_walk(n, sp, sms, False)
    xk = d["xk"]
    # the fp32 conv outputs (both operand sets)
    for raw, xx, ww, bb, what in ((d["ya_raw"], xk, d["w3"], d["b3"], "y3"), (d["yb_raw"], xk, d["w1"], d["b1"], "y1"),
                                  (d["sa_raw"], d["xs"], d["ws3"], d["bs3"], "stats y3"),
                                  (d["sb_raw"], d["xs"], d["ws1"], d["bs1"], "stats y1")):
        dev = raw.device
        ab = F.conv3d(_ncdhw(xx.abs()), ww.abs().to(dev), None, padding=ww.shape[-1] // 2)
        bound = float(ab.max()) + (float(bb.abs().max()) if bb is not None else 0.0)
        q = qof(xx) * quantum(ww) if bb is None else min(qof(xx) * quantum(ww), quantum(bb))
        assert_exact_fp32(bound, q, what)
        if what.startswith("stats"):
            # statistics partials per CTA and sample: sum y and sum y^2
            assert_exact_fp32(walk_max(stem_tile_sums(raw.abs(), w["tw"]), w), q, what + " sum")
            assert_exact_fp32(walk_max(stem_tile_sums(raw * raw, w["tw"]), w), q * q, what + " sum of squares")
    # both rounding points meet ties
    assert ties(d["ya_raw"]) + ties(d["yb_raw"]) > 0, "no bf16 tie of y"
    if cs["dense"]:
        assert sum(ties(s["dy"]) for s in d["sides"]) > 0, "no bf16 tie of dy"
    qz = []
    for i, (b, s, y, side) in enumerate(zip(d["br"], d["sc"], d["ys"], d["sides"])):
        qz.append(check_side(b, s[1], y, d["g"], side, f"branch {i}")[0])
        # BSUMS partials per CTA and sample
        qg, qy = qof(d["g"]), qof(y)
        for t, q, k in ((side["gm"].abs(), qg, "sum g m"), ((side["gm"] * y).abs(), qg * qy, "sum g m y"),
                        (y.abs(), qy, "sum y")):
            if cs["x_full"] and not walk_max(stem_tile_sums(t, w["tw"]), w) < 2 ** 24 * q:
                inexact.add("bsums")          # y has the quantum of the full-mantissa image: held to a chain bound
                continue
            assert_exact_fp32(walk_max(stem_tile_sums(t, w["tw"]), w), q, f"branch {i} {k}")
        # the weight gradient: every fp32 partial is part of prefill + sum |x dy|
        if not float((d["dw_pre"][i].abs() + d["dw_abs"][i]).max()) < 2 ** 24 * d["q_dw"][i]:
            inexact.add(f"dw{i}")
    # relu(z3) + relu(z1)
    tot = d["sides"][0]["relu"] + d["sides"][1]["relu"]
    assert_exact_fp32(float(tot.max()), min(qz), "apply sum")
    for k, t in d["terms"].items():
        if not pgrad_exact(d["prefill"][k], t):
            inexact.add(k)
    return inexact


@functools.lru_cache(maxsize=1)
def up_design(name, n, device="cpu", seed=0):
    cs = UP_CASES[name]
    sp = cs["sp"]
    fine = tuple(2 * s for s in sp)
    vox = math.prod(fine)
    gen = torch.Generator().manual_seed(seed)
    dev = torch.device(device)
    x = grid((n,) + sp + (CI,), 4, 2, gen).to(dev)
    w = grid((CI, C, 2, 2, 2), 16, 5, gen)
    b = grid((C,), 16, 7, gen) if cs["bias"] else None
    # the coarse operand set of the statistics
    xs = torch.randint(-1, 2, x.shape, generator=gen).double().to(dev)
    ws = torch.randint(-1, 2, w.shape, generator=gen).double() / 4
    bs = torch.randint(-2, 3, (C,), generator=gen).double() / 4
    s_raw = up_conv(xs, ws.to(dev), bs.to(dev))
    g = _gen_g(gen, (n,) + fine + (C,), cs["dense"], device)
    br = branch(gen, n, vox)
    sums, co = bwd_sums(gen, br, vox, cs["dense"])
    y_raw = up_conv(x, w.to(dev), None if b is None else b.to(dev))
    y = bf(y_raw)
    off_thresholds(br, y)
    side = gn_side(br, y, g, sums, co, dev)
    pc = param_contribs(br, sums, co, vox, sums[..., 2])
    terms = {"dgamma": pc["dgamma"], "dbeta": pc["dbeta"], "dbias": pc["dbias"]}
    prefill = {k: torch.randint(-3, 4, (C,), generator=gen).double() * quantum(t) for k, t in terms.items()}
    dy = bf(side["dy"])
    wsd = dict(kind=DOWN, dims=3, ca=C, cb=CI)
    dw, dw_abs = ref_wgrad(wsd, dy, x), ref_wgrad(wsd, dy.abs(), x.abs())
    wd = w.to(dev)
    dx_raw = _ndhwc(F.conv3d(_ncdhw(dy), wd, None, stride=2))
    dx_abs = _ndhwc(F.conv3d(_ncdhw(dy.abs()), wd.abs(), None, stride=2))
    q_dy = min(qof(g) * quantum(co["P"]), qof(y) * quantum(co["Q"]), quantum(co["R"]))
    q_dw = qof(x) * q_dy
    dw_pre = torch.randint(-3, 4, dw.shape, generator=gen).double().to(dev) * q_dw
    return dict(cs=cs, n=n, sp=sp, fine=fine, vox=vox, x=x, w=w, b=b, xs=xs, ws=ws, bs=bs, s_raw=s_raw, g=g, br=br, sums=sums, co=co, y_raw=y_raw, y=y,
                side=side, terms=terms, prefill=prefill, dy=dy, dw=dw, dw_abs=dw_abs, dx_raw=dx_raw, dx_abs=dx_abs,
                q_dy=q_dy, q_dw=q_dw, dw_pre=dw_pre)


def stem_dw_chain(n, sp, sms):
    """fp32 additions into one dW entry of stem_gn_bwd: per warp, TW / 16 groups per tile over the CTA's tiles, each
    an mma.sync of 16 products (counted as 16 roundings), the fold of 8 warps, then one atomic per CTA"""
    w = stem_walk(n, sp, sms, True)
    return w["tpc"] * w["tw"] // 16 * 16 + 8 + w["grid"] + 1


def up_dw_chain(n, sp, sms):
    """fp32 additions into one dW entry of up_gn_bwd: per CTA, 8 groups per 128-voxel tile, each an mma.sync of 16
    products (counted as 16 roundings), then one atomic per CTA"""
    w = up_walk(n, sp, sms, True)
    return w["tpc"] * 8 * 16 + w["grid"] + 1


def check_up_design(d, sms):
    cs, n, sp = d["cs"], d["n"], d["sp"]
    inexact = set()
    x, y = d["x"], d["y"]
    dev = x.device
    ab = up_conv(x.abs(), d["w"].abs().to(dev), None)
    bound = float(ab.max()) + (float(d["b"].abs().max()) if d["b"] is not None else 0.0)
    q = qof(x) * quantum(d["w"])
    if d["b"] is not None:
        q = min(q, quantum(d["b"]))
    assert_exact_fp32(bound, q, "y")
    w = up_walk(n, sp, sms, False)
    raw = d["s_raw"]
    qs = min(qof(d["xs"]) * quantum(d["ws"]), quantum(d["bs"]))
    assert_exact_fp32(float(up_conv(d["xs"].abs(), d["ws"].abs().to(dev), None).max() + d["bs"].abs().max()), qs,
                      "stats y")
    assert_exact_fp32(walk_max(up_tile_sums(raw.abs(), PW_TILE), w), qs, "stats sum")
    assert_exact_fp32(walk_max(up_tile_sums(raw * raw, PW_TILE), w), qs * qs, "stats sum of squares")
    assert ties(d["y_raw"]) > 0, "no bf16 tie of y"
    if cs["dense"]:
        assert ties(d["side"]["dy"]) > 0, "no bf16 tie of dy"
    check_side(d["br"], d["co"], y, d["g"], d["side"], "up")
    qg, qy = qof(d["g"]), qof(y)
    side = d["side"]
    for t, qq, k in ((side["gm"].abs(), qg, "sum g m"), ((side["gm"] * y).abs(), qg * qy, "sum g m y"),
                     (y.abs(), qy, "sum y")):
        assert_exact_fp32(walk_max(up_tile_sums(t, PW_TILE), w), qq, k)
    if cs["dense"] and not float(d["dx_abs"].max()) < 2 ** 24 * d["q_dy"] * quantum(d["w"]):
        inexact.add("dx")         # dense dy: held to the fp32 chain of 128 products and one bf16 rounding
    else:
        assert_exact_fp32(float(d["dx_abs"].max()), d["q_dy"] * quantum(d["w"]), "dx")
    if not float((d["dw_pre"].abs() + d["dw_abs"]).max()) < 2 ** 24 * d["q_dw"]:
        inexact.add("dw")
    for k, t in d["terms"].items():
        if not pgrad_exact(d["prefill"][k], t):
            inexact.add(k)
    return inexact


# ---------------------------------------------------------------------------------------------------------- CPU part
@pytest.mark.parametrize("name", sorted(STEM_CASES))
def test_stem_design_is_exact(name):
    """the preconditions hold for 132 and 114 SMs; only a dense case's dW may be held to its fp32 chain bound"""
    for sms in SMS_CHECKED:
        n, _ = shape_of(STEM_CASES[name], sms)
        inexact = check_stem_design(stem_design(name, n), sms)
        cs = STEM_CASES[name]
        allowed = ({"dw0", "dw1"} if cs["dense"] or cs["x_full"] else set()) | ({"bsums"} if cs["x_full"] else set())
        assert inexact <= allowed, (name, sms, sorted(inexact))


@pytest.mark.parametrize("name", sorted(UP_CASES))
def test_up_design_is_exact(name):
    """the preconditions hold for 132 and 114 SMs; only a dense case's dW is held to its fp32 chain bound"""
    for sms in SMS_CHECKED:
        inexact = check_up_design(up_design(name, UP_CASES[name]["n"]), sms)
        assert inexact <= ({"dw", "dx"} if UP_CASES[name]["dense"] else set()), (name, sms, sorted(inexact))


def test_every_listed_shape_reaches_its_walk():
    for sms in SMS_CHECKED:
        def st(name, bwd=False):
            n, sp = shape_of(STEM_CASES[name], sms)
            return stem_walk(n, sp, sms, bwd)
        assert st("vnet96")["tw"] == 96 and st("tw112")["tw"] == 112
        assert st("d1")["tw"] == 16 and st("d1")["tiles"] == 1 and STEM_CASES["d1"]["sp"][0] == 1
        assert st("tw128_two_tiles")["tw"] == 128 and st("tw128_two_tiles")["tiles_w"] == 2
        assert st("tw48_three_tiles")["tw"] == 48 and st("tw48_three_tiles")["tiles_w"] == 3
        assert crosses_samples(st("cross_samples")) and crosses_samples(st("cross_samples", True))
        assert st("cross_samples", True)["tpc"] >= 3
        assert st("fewer_tiles_than_sms")["tiles"] < sms and st("fewer_tiles_than_sms", True)["grid"] < sms
        a, ab = st("sms_plus_one"), st("sms_plus_one", True)
        assert a["tiles"] == sms + 1 and ab["grid"] == sms and ab["tpc"] == 2 and ab["tiles"] % ab["tpc"]
        a = st("two_sms_plus_one")
        assert a["tiles"] == 2 * sms + 1 and a["grid"] == 2 * sms and a["tpc"] == 2
        # every stem case is a shape the kernels take
        for cs in STEM_CASES.values():
            n, (D, H, W) = shape_of(cs, sms)
            assert H % SM_TH == 0 and stem_tile_width(W) > 0

        def up(name, bwd=False):
            cs = UP_CASES[name]
            return up_walk(cs["n"], cs["sp"], sms, bwd)
        assert math.prod(UP_CASES["v512"]["sp"]) == 512 and up("v512")["tiles"] < sms
        assert crosses_samples(up("cross_samples")) and crosses_samples(up("cross_samples", True))
        assert UP_CASES["w48"]["sp"][2] // 16 == 3
        for cs in UP_CASES.values():
            n, (D, H, W) = cs["n"], cs["sp"]
            assert W % 16 == 0 and (D * H * W) % PW_TILE == 0 and 8 * n * D * H * W >= 65536


def test_checkers_reject_one_ulp_and_a_rewritten_guard():
    d = stem_design("dense_small", 2)
    want = (d["sides"][0]["relu"] + d["sides"][1]["relu"]).float().bfloat16()
    got = want.clone()
    got.view(torch.int16)[1, 1, 3, 5, 9] += 1
    with pytest.raises(AssertionError, match=r"\(1, 1, 3, 5, 9\)"):
        assert_bitwise(got, want, "one ulp")
    gb = Guarded(tuple(want.shape), BF, off=16)
    gb.view.copy_(want)
    assert gb.outside_changed() is None
    gb.buf.view(torch.int16)[GUARD + 3] = 0          # the other half of the 32-channel row
    with pytest.raises(AssertionError, match=f"element {GUARD + 3}"):
        assert_guards(gb, "left half")


def test_checker_rejects_one_flipped_mask_bit():
    fwd = torch.rand(2, 6, C, generator=torch.Generator().manual_seed(1)) > 0.5
    s1 = (fwd.long() << torch.arange(6).view(1, 6, 1)).sum(1).double()
    assert torch.equal(decode_mask(s1, 6, 0), fwd)
    s1[1, 5] += 4.0 if not bool(fwd[1, 2, 5]) else -4.0
    with pytest.raises(AssertionError, match=r"\(1, 2, 5\)"):
        assert_same_mask(fwd, decode_mask(s1, 6, 0), "flipped")


def test_checker_rejects_a_tile_moved_to_the_next_sample():
    d = stem_design("dense_small", 2)
    raw = d["sa_raw"]
    want = torch.stack([raw.sum((1, 2, 3)), (raw * raw).sum((1, 2, 3))], -1)
    tile = raw[0, 1, 0:8, 0:16]
    moved = want.clone()
    moved[0, :, 0] -= tile.sum((0, 1))
    moved[1, :, 0] += tile.sum((0, 1))
    assert_equal64(want.clone(), want, "same")
    with pytest.raises(AssertionError, match="differ"):
        assert_equal64(moved, want, "moved tile")


@pytest.mark.parametrize("what", ["swapped taps", "exchanged planes"])
def test_checker_rejects_a_wrong_tap_order(what):
    """two 3x3x3 taps exchanged, or the d - 1 and d + 1 image planes exchanged (the halo staging), change the output"""
    d = stem_design("dense_small", 2)
    w3 = d["w3"].clone()
    if what == "swapped taps":
        w3[..., 0, 0, 0], w3[..., 1, 2, 2] = d["w3"][..., 1, 2, 2], d["w3"][..., 0, 0, 0]
    else:
        w3 = w3.flip(2)
    ya, _ = stem_conv(d["xk"], w3, d["w1"], d["b3"], d["b1"])
    b = d["br"][0]
    za = bf(ya) * _bc(b["A"], "cpu") + _bc(b["B"], "cpu")
    got = (za.clamp_min(0) + d["sides"][1]["relu"]).float().bfloat16()
    want = (d["sides"][0]["relu"] + d["sides"][1]["relu"]).float().bfloat16()
    assert first_mismatch(got, want) is not None


def test_checker_rejects_a_chunk_in_the_neighbouring_run():
    """one 16-byte chunk (8 channels of one fine voxel) of up_gn's APPLY stage stored into the next fine row"""
    d = up_design("v512", 16)
    want = d["side"]["relu"].float().bfloat16()
    nz = (want[:, :, 0::2, :, :8].float().abs().sum(-1) > 0).nonzero()
    n, fd, fh, fw = nz[0].tolist()
    fh *= 2
    got = want.clone()
    got[n, fd, fh + 1, fw, :8] = want[n, fd, fh, fw, :8]
    assert not torch.equal(got.float(), want.float())
    with pytest.raises(AssertionError, match="differ"):
        assert_bitwise(got, want, "moved chunk")


# ---------------------------------------------------------------------------------------------------------- GPU part
@pytest.fixture(scope="module")
def be():
    from pytorchdeeplearing_b200._abi import CudaBackend
    return CudaBackend()


def device_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _gn(b, vox, stats=None, eps=EPS):
    return ((b["stats"] if stats is None else stats).cuda(), b["gamma"].float().cuda(), b["beta"].float().cuda(),
            b["scale"].float().cuda(), vox, GROUPS, eps)


def _at(c, layout, off=None):
    """Guarded's arguments for a (pitch, offset) layout of c channels"""
    ld, o = layout
    assert ld in (c, c + 16)
    return dict(dense=True) if ld == c else dict(off=off if o is None else o)


def _f(t):
    return None if t is None else t.float().cuda()


def _stem_packs(be, w3, w1):
    return (be.pack_weight(w3.float().cuda(), K3, "fwd", BF, 3), be.pack_weight(w1.float().cuda(), K1, "fwd", BF, 3))


def _up_pack(be, w):
    return be.pack_weight(w.float().cuda(), UP, "fwd", BF, 3, vox=10 ** 9)


def _check_dw(got, want, pre, absum, exact, chain, what):
    full = pre + want
    if exact:
        assert_equal64(got, full, what)
        return
    bound = chain * U * (pre.abs() + absum)
    bad = (got.double() - full).abs() > bound
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} entries outside the fp32 chain bound"


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(STEM_CASES))
def test_stem_gn_exact(be, name):
    sms = device_sms()
    cs = STEM_CASES[name]
    n, sp = shape_of(cs, sms)
    d = stem_design(name, n, "cuda")
    inexact = check_stem_design(d, sms)
    vox = d["vox"]
    shape = (n,) + sp + (C,)
    gx = Guarded((n,) + sp + (1,), F32, fill=IN_FILL, device="cuda", dense=True)
    assert be.stem_gn_ok(gx.view, C, 3)
    walk = stem_walk(n, sp, sms, False)
    assert walk["tw"] == stem_tile_width(sp[2])
    p3, p1 = _stem_packs(be, d["ws3"], d["ws1"])

    # STATS of the unrounded conv output (coarse operand set): bit-equal fp64; the full-mantissa image: chain bound
    gx.view.copy_(d["xs"].float())
    sbuf = [flat((n, C, 2), torch.float64) for _ in range(2)]
    be.stem_gn_stats(gx.view, p3, _f(d["bs3"]), p1, _f(d["bs1"]), sbuf[0][1], sbuf[1][1])
    for (buf, got), raw, k in zip(sbuf, (d["sa_raw"], d["sb_raw"]), ("3x3x3", "1x1x1")):
        assert_equal64(got, torch.stack([raw.sum((1, 2, 3)), (raw * raw).sum((1, 2, 3))], -1), f"{name} stats {k}")
        assert_flat_guards(buf, "stats")
    p3, p1 = _stem_packs(be, d["w3"], d["w1"])
    b3, b1 = _f(d["b3"]), _f(d["b1"])
    gx.view.copy_(d["x"].float())
    if cs["x_full"]:
        sbuf = [flat((n, C, 2), torch.float64) for _ in range(2)]
        be.stem_gn_stats(gx.view, p3, b3, p1, b1, sbuf[0][1], sbuf[1][1])
        chain = 2 * walk["tpc"] * walk["tw"] // 16 + 6
        for (_, got), raw, k in zip(sbuf, (d["ya_raw"], d["yb_raw"]), ("3x3x3", "1x1x1")):
            check_stats(got.cpu(), raw.cpu(), chain, f"{name} stats {k} (full mantissas)")

    # APPLY into the right half of a 32-channel buffer, and into a contiguous one
    gna, gnb = _gn(d["br"][0], vox), _gn(d["br"][1], vox)
    for lay in LAYOUTS["stem_gn out"]:
        out = Guarded(shape, BF, device="cuda", **_at(C, lay))
        be.stem_gn_apply(gx.view, p3, b3, p1, b1, gna, gnb, out.view)
        assert_bitwise(out.view, (d["sides"][0]["relu"] + d["sides"][1]["relu"]).float().bfloat16(),
                       f"{name} apply {lay}")
        assert_guards(out, f"{name} apply {lay}")
    for lay in LAYOUTS["stem_gn g"]:
        _stem_backward(be, name, cs, d, inexact, n, sp, sms, walk, gx, p3, b3, p1, b1, gna, gnb, lay)


def _stem_backward(be, name, cs, d, inexact, n, sp, sms, walk, gx, p3, b3, p1, b1, gna, gnb, lay):
    """BSUMS and BWD of one stem case with g at layout `lay` (a concat-gradient half: the other half holds IN_FILL)"""
    shape = (n,) + sp + (C,)
    name = f"{name} g {lay}"
    gg = Guarded(shape, BF, fill=IN_FILL, device="cuda", **_at(C, lay))
    gg.view.copy_(d["g"].bfloat16())
    sums = [flat((n, C, 3), torch.float64) for _ in range(2)]
    be.stem_gn_bwd_sums(gx.view, p3, b3, p1, b1, gna, gnb, gg.view, sums[0][1], sums[1][1])
    for i in range(2):
        side, y = d["sides"][i], d["ys"][i]
        if "bsums" in inexact:
            # fp32 chain of the lane partials (as for the statistics) on sum |terms|
            red = (1, 2, 3)
            mag = torch.stack([side["gm"].abs().sum(red), (side["gm"] * y).abs().sum(red), y.abs().sum(red)], -1)
            bad = (sums[i][1] - side["sums"]).abs() > (2 * walk["tpc"] * walk["tw"] // 16 + 6) * U * mag
            assert not bool(bad.any()), f"{name} bwd sums branch {i} outside the fp32 chain bound"
        else:
            assert_equal64(sums[i][1], side["sums"], f"{name} bwd sums branch {i}")
        assert_flat_guards(sums[i][0], "sums")

    # BWD from the designed sums: both stem weight gradients, d gamma, d beta, both bias gradients, onto prefills
    dwb = [flat(tuple(t.shape), F32, t.float()) for t in d["dw_pre"]]
    pb = {k: flat((C,), F32, v.float()) for k, v in d["prefill"].items()}
    null = not cs["bias"]
    be.stem_gn_bwd(gx.view, p3, b3, p1, b1, gna, gnb, gg.view, d["sc"][0][0].cuda(), d["sc"][1][0].cuda(),
                   dwb[0][1], dwb[1][1], pb["dgamma"][1], pb["dbeta"][1], None if null else pb["db3"][1],
                   None if null else pb["db1"][1])
    torch.cuda.synchronize()
    for i in range(2):
        _check_dw(dwb[i][1], d["dw"][i], d["dw_pre"][i], d["dw_abs"][i], f"dw{i}" not in inexact,
                  stem_dw_chain(n, sp, sms), f"{name} dW branch {i}")
        assert_flat_guards(dwb[i][0], "dw")
    for k in ("dgamma", "dbeta", "db3", "db1"):
        if null and k in ("db3", "db1"):
            # a bias gradient passed as null: the buffer that would have held it is untouched
            assert_equal64(pb[k][1], d["prefill"][k], f"{name} null {k} unwritten")
        else:
            check_pgrad(pb[k][1], d["prefill"][k], d["terms"][k], k not in inexact, f"{name} {k} (+=)")
        assert_flat_guards(pb[k][0], k)
    for gb, what in ((gx, "x"), (gg, "g")):
        assert_guards(gb, f"{name} {what}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(UP_CASES))
def test_up_gn_exact(be, name):
    sms = device_sms()
    cs = UP_CASES[name]
    n, sp = cs["n"], cs["sp"]
    d = up_design(name, n, "cuda")
    inexact = check_up_design(d, sms)
    vox, fine = d["vox"], d["fine"]
    gx = Guarded((n,) + sp + (CI,), BF, fill=IN_FILL, device="cuda", off=cs["x_off"])
    gx.view.copy_(d["xs"].bfloat16())
    ws = _up_pack(be, d["ws"])
    assert be.up_gn_ok(gx.view, ws, C, 3)
    sbuf, st = flat((n, C, 2), torch.float64)
    be.up_gn_stats(gx.view, ws, _f(d["bs"]), st)
    raw = d["s_raw"]
    assert_equal64(st, torch.stack([raw.sum((1, 2, 3)), (raw * raw).sum((1, 2, 3))], -1), f"{name} stats")
    assert_flat_guards(sbuf, "stats")
    gx.view.copy_(d["x"].bfloat16())
    wf = _up_pack(be, d["w"])
    b = _f(d["b"])

    gn = _gn(d["br"], vox)
    out = Guarded((n,) + fine + (C,), BF, device="cuda", off=0)
    be.up_gn_apply(gx.view, wf, b, gn, out.view)
    assert_bitwise(out.view, d["side"]["relu"].float().bfloat16(), f"{name} apply")
    assert_guards(out, f"{name} apply")

    gg = Guarded((n,) + fine + (C,), BF, fill=IN_FILL, device="cuda", off=0)
    gg.view.copy_(d["g"].bfloat16())
    sb, s = flat((n, C, 3), torch.float64)
    be.up_gn_bwd_sums(gx.view, wf, b, gn, gg.view, s)
    assert_equal64(s, d["side"]["sums"], f"{name} bwd sums")
    assert_flat_guards(sb, "sums")

    for lay in LAYOUTS["up_gn dx"]:
        _up_backward(be, f"{name} dx {lay}", cs, d, inexact, n, sp, sms, gx, wf, b, gn, gg, lay)


def _up_backward(be, name, cs, d, inexact, n, sp, sms, gx, wf, b, gn, gg, lay):
    """BWD of one up_tr32 case with dx at layout `lay`"""
    dwb, dw = flat((8, C, CI), F32, d["dw_pre"].float())
    pb = {k: flat((C,), F32, v.float()) for k, v in d["prefill"].items()}
    gdx = Guarded((n,) + sp + (CI,), BF, device="cuda", **_at(CI, lay, cs["dx_off"]))
    be.up_gn_bwd(gx.view, wf, b, gn, gg.view, d["sums"].cuda(), dw, gdx.view, pb["dgamma"][1], pb["dbeta"][1],
                 None if not cs["bias"] else pb["dbias"][1])
    torch.cuda.synchronize()
    if "dx" in inexact:
        got = gdx.view.double()
        # each dx value is an fp32 chain of 8 taps x 16 channels = 128 products (counted as 128 roundings of at
        # most U sum |terms| each, plus 2 spare), then one bf16 round-to-nearest-even of the fp32 value v: half an
        # ulp, and an ulp of bf16's 8-bit significand is at most 2^-7 |v|, so |bf16(v) - v| <= 2^-8 |v| (the tie
        # v = 1 + 2^-8 rounds to 1: an error of 2^-8 / (1 + 2^-8) relative), and |v| <= |dx| + the chain error
        chain = 130 * U * d["dx_abs"]
        bound = 2.0 ** -8 * (d["dx_raw"].abs() + chain) + chain
        bad = (got - d["dx_raw"]).abs() > bound
        assert not bool(bad.any()), f"{name} dx: {int(bad.sum())} values outside one bf16 rounding + the fp32 chain"
    else:
        assert_bitwise(gdx.view, d["dx_raw"].float().bfloat16(), f"{name} dx")
    assert_guards(gdx, f"{name} dx")
    _check_dw(dw, d["dw"], d["dw_pre"], d["dw_abs"], "dw" not in inexact, up_dw_chain(n, sp, sms), f"{name} dW")
    assert_flat_guards(dwb, "dw")
    for k in ("dgamma", "dbeta", "dbias"):
        if k == "dbias" and not cs["bias"]:
            assert_equal64(pb[k][1], d["prefill"][k], f"{name} null dbias unwritten")
        else:
            check_pgrad(pb[k][1], d["prefill"][k], d["terms"][k], k not in inexact, f"{name} {k} (+=)")
        assert_flat_guards(pb[k][0], k)
    for gb_, what in ((gx, "x"), (gg, "g")):
        assert_guards(gb_, f"{name} {what}")


@pytest.mark.gpu
def test_stats_are_of_the_unrounded_conv_output(be):
    """STATS sums y and y^2 of the fp32 conv output BEFORE its bf16 rounding (the stored y, which APPLY, BSUMS and
    BWD recompute, is rounded): the convention of the stem and pointwise epilogues.  The case is chosen so that the
    two conventions give different sums, and both families must match the unrounded one bit for bit."""
    d = stem_design("dense_small", 2, "cuda")
    sms = device_sms()
    check_stem_design(d, sms)
    w = stem_walk(2, d["sp"], sms, False)
    for raw in (d["ya_raw"], d["yb_raw"]):
        q = qof(raw)
        assert_exact_fp32(walk_max(stem_tile_sums(raw.abs(), w["tw"]), w), q, "sum y")
        assert_exact_fp32(walk_max(stem_tile_sums(raw * raw, w["tw"]), w), q * q, "sum y^2")
    gx = Guarded((2,) + d["sp"] + (1,), F32, fill=IN_FILL, device="cuda", dense=True)
    gx.view.copy_(d["x"].float())
    p3, p1 = _stem_packs(be, d["w3"], d["w1"])
    s3, s1 = torch.zeros((2, C, 2), dtype=torch.float64, device="cuda"), torch.zeros((2, C, 2), dtype=torch.float64,
                                                                                       device="cuda")
    be.stem_gn_stats(gx.view, p3, _f(d["b3"]), p1, _f(d["b1"]), s3, s1)
    for got, raw in ((s3, d["ya_raw"]), (s1, d["yb_raw"])):
        want = torch.stack([raw.sum((1, 2, 3)), (raw * raw).sum((1, 2, 3))], -1)
        rounded = torch.stack([bf(raw).sum((1, 2, 3)), (bf(raw) ** 2).sum((1, 2, 3))], -1)
        assert not torch.equal(want, rounded)
        assert_equal64(got, want, "stem stats")
    # up_tr32: x nonzero at one coarse voxel per sample, so sum y^2 of tie-rich y stays below 2^24 quanta over the
    # 512-voxel tiles (elsewhere y is the bias)
    u = up_sparse_stats_design("cuda")
    w_ = up_walk(u["n"], u["sp"], sms, False)
    raw = u["y_raw"]
    assert ties(raw) > 0
    assert_exact_fp32(walk_max(up_tile_sums(raw.abs(), PW_TILE), w_), u["q"], "up sum y")
    assert_exact_fp32(walk_max(up_tile_sums(raw * raw, PW_TILE), w_), u["q"] ** 2, "up sum y^2")
    gxu = Guarded((u["n"],) + u["sp"] + (CI,), BF, fill=IN_FILL, device="cuda")
    gxu.view.copy_(u["x"].bfloat16())
    wu = _up_pack(be, u["w"])
    assert be.up_gn_ok(gxu.view, wu, C, 3)
    st = torch.zeros((u["n"], C, 2), dtype=torch.float64, device="cuda")
    be.up_gn_stats(gxu.view, wu, _f(u["b"]), st)
    want = torch.stack([raw.sum((1, 2, 3)), (raw * raw).sum((1, 2, 3))], -1)
    rounded = torch.stack([bf(raw).sum((1, 2, 3)), (bf(raw) ** 2).sum((1, 2, 3))], -1)
    assert not torch.equal(want, rounded)
    assert_equal64(st, want, "up stats")


def up_sparse_stats_design(device):
    """16 x (8, 4, 16) coarse, x from {-4 .. 4} 2^-2 at one coarse voxel per sample and 0 elsewhere"""
    gen = torch.Generator().manual_seed(5)
    n, sp = 16, (8, 4, 16)
    V = math.prod(sp)
    x = torch.zeros((n, V, CI), dtype=torch.float64)
    x[torch.arange(n), torch.randint(0, V, (n,), generator=gen)] = grid((n, CI), 4, 2, gen)
    x = x.view((n,) + sp + (CI,)).to(device)
    w, b = grid((CI, C, 2, 2, 2), 16, 5, gen), grid((C,), 16, 7, gen)
    y_raw = up_conv(x, w.to(device), b.to(device))
    return dict(n=n, sp=sp, x=x, w=w, b=b, y_raw=y_raw, q=min(qof(x) * quantum(w), quantum(b)))


def test_up_sparse_stats_design_meets_ties_and_bounds():
    u = up_sparse_stats_design("cpu")
    raw = u["y_raw"]
    assert ties(raw) > 0
    for sms in SMS_CHECKED:
        w_ = up_walk(u["n"], u["sp"], sms, False)
        assert_exact_fp32(walk_max(up_tile_sums(raw * raw, PW_TILE), w_), u["q"] ** 2, "up sum y^2")
    assert not torch.equal(raw.sum((1, 2, 3)), bf(raw).sum((1, 2, 3))) or \
        not torch.equal((raw * raw).sum((1, 2, 3)), (bf(raw) ** 2).sum((1, 2, 3)))


# ---------------------------------------------------------------------------------------------------------- rejections
def _nan_bufs(*shapes):
    return [torch.full(s, float("nan"), dtype=torch.float64 if len(s) == 3 else F32, device="cuda") for s in shapes]


def _strided(shape, ld, off, dtype=BF):
    n, dd, h, w, c = shape
    buf = torch.full((n * dd * h * w * ld + 64,), float("nan"), dtype=dtype, device="cuda")
    return buf, buf.as_strided(shape, (dd * h * w * ld, h * w * ld, w * ld, ld, 1), off)


def _expect_einval(be, fn, bufs, what):
    before = [b.clone() for b in bufs]
    count = be.launch_count
    with pytest.raises(RuntimeError, match=f"libb200seg error {EINVAL}"):
        fn()
    torch.cuda.synchronize()
    assert be.launch_count == count, what
    for b0, b1 in zip(before, bufs):
        assert torch.equal(b0.view(torch.int8), b1.view(torch.int8)), f"{what}: an output was written"


@pytest.mark.gpu
def test_stem_gn_rejects_bad_arguments(be):
    gen = torch.Generator().manual_seed(3)
    w3, w1 = grid((C, 1, 3, 3, 3), 8, 5, gen), grid((C, 1, 1, 1, 1), 32, 5, gen)
    p3, p1 = _stem_packs(be, w3, w1)
    b = torch.zeros(C, device="cuda")
    n, sp = 2, (2, 8, 16)
    vox = math.prod(sp)
    br = branch(gen, n, vox)
    good_x = torch.zeros((n,) + sp + (1,), device="cuda")
    st3, st1, su3, su1 = _nan_bufs((n, C, 2), (n, C, 2), (n, C, 3), (n, C, 3))
    dws = _nan_bufs((27, 1, C), (1, 1, C), (C,), (C,), (C,), (C,))
    _, good_o = _strided((n,) + sp + (C,), 32, 16)
    _, good_g = _strided((n,) + sp + (C,), 32, 0)

    def passes(x, gn, o, g, gn_b=None):
        gn_b = gn if gn_b is None else gn_b
        return [("stats", lambda: be.stem_gn_stats(x, p3, b, p1, b, st3, st1), [st3, st1]),
                ("apply", lambda: be.stem_gn_apply(x, p3, b, p1, b, gn, gn_b, o), [o]),
                ("bwd_sums", lambda: be.stem_gn_bwd_sums(x, p3, b, p1, b, gn, gn_b, g, su3, su1), [su3, su1]),
                ("bwd", lambda: be.stem_gn_bwd(x, p3, b, p1, b, gn, gn_b, g, su3.nan_to_num(0), su1.nan_to_num(0),
                                               *dws), dws)]
    gn = _gn(br, vox)
    cases = []
    for bad_sp, what in (((2, 12, 16), "H % 8"), ((2, 8, 24), "W not a multiple of 16")):
        x = torch.zeros((n,) + bad_sp + (1,), device="cuda")
        assert not be.stem_gn_ok(x, C, 3)
        _, o = _strided((n,) + bad_sp + (C,), 32, 16)
        _, g = _strided((n,) + bad_sp + (C,), 32, 0)
        cases += [(what + " " + p, f, bufs) for p, f, bufs in passes(x, _gn(br, math.prod(bad_sp)), o, g)]
    f32o = torch.full((n,) + sp + (C,), float("nan"), device="cuda")
    _, mis = _strided((n,) + sp + (C,), 32, 4)
    _, ld20 = _strided((n,) + sp + (C,), 20, 0)
    for o, what in ((f32o, "fp32 output"), (mis, "misaligned output"), (ld20, "ld % 8")):
        cases.append((what, passes(good_x, gn, o, good_g)[1][1], [o]))
    for g, what in ((mis, "misaligned gradient"), (ld20, "gradient ld % 8")):
        cases += [(what + " " + p, f, bufs) for p, f, bufs in passes(good_x, gn, good_o, g)[2:]]
    for bad_gn, what in ((_gn(br, vox)[:5] + (4, EPS), "groups = 4"), (_gn(br, vox + 1), "gn.vox")):
        for gn_a, gn_b in ((bad_gn, gn), (gn, bad_gn)):
            cases += [(what + " " + p, f, bufs) for p, f, bufs in passes(good_x, gn_a, good_o, good_g, gn_b)[1:]]
    for what, fn, bufs in cases:
        _expect_einval(be, fn, bufs, what)


@pytest.mark.gpu
def test_up_gn_rejects_bad_arguments(be):
    gen = torch.Generator().manual_seed(4)
    w = grid((CI, C, 2, 2, 2), 16, 5, gen)
    wf = _up_pack(be, w)
    b = torch.zeros(C, device="cuda")
    n, sp = 8, (8, 8, 16)
    fine = tuple(2 * s for s in sp)
    vox = math.prod(fine)
    br = branch(gen, n, vox)
    gn = _gn(br, vox)
    x = torch.zeros((n,) + sp + (CI,), dtype=BF, device="cuda")
    assert be.up_gn_ok(x, wf, C, 3)
    st, su = _nan_bufs((n, C, 2), (n, C, 3))
    dws = _nan_bufs((8, C, CI), (C,), (C,), (C,))
    _, good_o = _strided((n,) + fine + (C,), 32, 0)
    _, good_dx = _strided((n,) + sp + (CI,), 48, 8)

    def passes(xx, g_, o, g, dx):
        return [("stats", lambda: be.up_gn_stats(xx, wf, b, st), [st]),
                ("apply", lambda: be.up_gn_apply(xx, wf, b, g_, o), [o]),
                ("bwd_sums", lambda: be.up_gn_bwd_sums(xx, wf, b, g_, g, su), [su]),
                ("bwd", lambda: be.up_gn_bwd(xx, wf, b, g_, g, su.nan_to_num(0), dws[0], dx, *dws[1:]), dws + [dx])]
    cases = []
    for bad_sp, what in (((8, 8, 24), "W not a multiple of 16"), ((8, 8, 8), "W = 8")):
        xb = torch.zeros((n,) + bad_sp + (CI,), dtype=BF, device="cuda")
        assert not be.up_gn_ok(xb, wf, C, 3)
        fb = tuple(2 * s for s in bad_sp)
        _, o = _strided((n,) + fb + (C,), 32, 0)
        _, dx = _strided((n,) + bad_sp + (CI,), 48, 8)
        cases += [(what + " " + p, f, bb) for p, f, bb in passes(xb, _gn(br, math.prod(fb)), o, o, dx)]
    f32o = torch.full((n,) + fine + (C,), float("nan"), device="cuda")
    _, mis = _strided((n,) + fine + (C,), 32, 4)
    _, ld20 = _strided((n,) + fine + (C,), 20, 0)
    for o, what in ((f32o, "fp32 output"), (mis, "misaligned output"), (ld20, "ld % 8")):
        cases.append((what, passes(x, gn, o, good_o, good_dx)[1][1], [o]))
    for g, what in ((mis, "misaligned gradient"), (ld20, "gradient ld % 8")):
        cases += [(what + " " + p, f, bb) for p, f, bb in passes(x, gn, good_o, g, good_dx)[2:]]
    for bad_gn, what in ((gn[:5] + (4, EPS), "groups = 4"), (_gn(br, vox // 8), "gn.vox of the coarse grid")):
        cases += [(what + " " + p, f, bb) for p, f, bb in passes(x, bad_gn, good_o, good_o, good_dx)[1:]]
    _, dx16 = _strided((n,) + sp + (C,), 48, 8)
    _, dx_mis = _strided((n,) + sp + (CI,), 48, 1)
    for dx, what in ((dx16, "dx with 16 channels"), (dx_mis, "dx 2-byte aligned")):
        cases.append((what, passes(x, gn, good_o, good_o, dx)[3][1], dws + [dx]))
    for what, fn, bufs in cases:
        _expect_einval(be, fn, bufs, what)


class _Counting:
    """the CUDA backend, counting the fused calls and the forward transposed convolutions (kind UP with statistics:
    a data gradient of a strided convolution is also of kind UP, but has none)"""

    def __init__(self, inner):
        self.inner = inner
        self.calls = {}

    def __getattr__(self, name):
        fn = getattr(self.inner, name)
        if not callable(fn) or not (name.startswith(("stem_gn_", "up_gn_")) or name == "conv"):
            return fn

        def wrapped(*a, **k):
            key = "conv UP" if name == "conv" and a[0] == UP and a[6] is not None else name
            self.calls[key] = self.calls.get(key, 0) + 1
            return fn(*a, **k)
        return wrapped


def _vnet_step_calls(be, sp):
    """one eager bf16 VNet3d(1, 2) training step at 1 x sp -> the counted backend calls"""
    import oracle
    import pytorchdeeplearing_b200 as b200
    from pytorchdeeplearing_b200 import runtime
    b200.set_precision("bf16")
    x, y = oracle.make_inputs(1, 1, sp, 2, seed=3)
    cb = _Counting(be)
    runtime._set_backend_for_testing(cb)
    try:
        torch.manual_seed(0)
        m = b200.VNet3d(1, 2)
        m.apply(b200.initialize_weights)
        m = m.cuda().train()
        logits, _ = m(x.cuda())
        b200.MutilDiceLoss(torch.ones(2, device="cuda"))(logits, y.cuda()).backward()
        torch.cuda.synchronize()
        assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in m.parameters())
    finally:
        runtime._set_backend_for_testing(None)
    return cb.calls


@pytest.mark.gpu
def test_up_gn_not_taken_at_128x112x112(be):
    """1 x 128 x 112 x 112: the coarse grid of up_tr32 is 64 x 56 x 56 and W = 56 is not a multiple of 16, so the
    fused layer is refused and a VNet3d training step takes the per-layer calls for it (the input block still runs
    fused).  At 64^3 the same step takes the fused layer: the counting sees both."""
    x = torch.zeros((1, 64, 56, 56, CI), dtype=BF, device="cuda")
    wf = be.pack_weight(torch.zeros((CI, C, 2, 2, 2), device="cuda"), UP, "fwd", BF, 3, vox=128 * 112 * 112)
    assert not be.up_gn_ok(x, wf, C, 3)
    calls = _vnet_step_calls(be, (128, 112, 112))
    assert not any(k.startswith("up_gn_") and not k.endswith("_ok") for k in calls), calls
    assert calls.get("stem_gn_apply", 0) == 1, calls
    fused = _vnet_step_calls(be, (64, 64, 64))
    assert fused.get("up_gn_apply", 0) == 1 and fused.get("up_gn_bwd", 0) == 1, fused
    # the per-layer form runs one more forward transposed convolution than the fused step: up_tr32's
    assert calls.get("conv UP", 0) == fused.get("conv UP", 0) + 1, (calls, fused)


# ---------------------------------------------------------------------------------------------------------- part 3
NTHR = 6          # planted threshold voxels per (n, c); planted voxel k carries g = 2^k, every other voxel g = 0


def shared_gn(gen, N, vox, on):
    """an exact GroupNorm reference whose statistics every sample shares (so -B/A depends on the channel only), with
    dropout scale 1.25 (on) or 0 (off: A = B = 0, the branch contributes nothing)"""
    b = gn_branch(gen, 1, C, vox)
    for k in ("mu", "rs", "mu_c", "rs_c", "stats"):
        b[k] = b[k].expand((N,) + tuple(b[k].shape[1:])).contiguous()
    b["scale"] = torch.full((N, C), 1.25 if on else 0.0, dtype=torch.float64)
    b["A"] = b["rs_c"] * b["gamma"] * b["scale"]
    b["B"] = (b["beta"] - b["mu_c"] * b["rs_c"] * b["gamma"]) * b["scale"]
    return b


def pick_y0(y, gen):
    """per channel the value y0 (|y0| >= 1/4 where there is one, else nonzero) of y (N, ..., C) that occurs most often in its rarest sample, and NTHR
    voxels of every sample that hold it -> y0 (C,), positions (N, NTHR, C)"""
    N = y.shape[0]
    yf = y.reshape(N, -1, C)
    y0 = torch.empty(C, dtype=torch.float64)
    pos = torch.empty((N, NTHR, C), dtype=torch.long)
    for c in range(C):
        u = torch.unique(yf[..., c])
        u = u[u.abs() >= 0.25] if bool((u.abs() >= 0.25).any()) else u[u != 0]     # a zero 1x1x1 weight: y = bias
        assert u.numel() > 0, f"channel {c}: y is zero everywhere"
        cnt = (yf[..., c].unsqueeze(-1) == u).sum(1).min(0).values
        best = int(cnt.argmax())
        assert int(cnt[best]) >= NTHR, f"channel {c}: no value of y occurs {NTHR} times in every sample"
        y0[c] = float(u[best])
        for n in range(N):
            idx = (yf[n, :, c] == u[best]).nonzero()[:, 0].cpu()
            pos[n, :, c] = idx[torch.randperm(idx.numel(), generator=gen)[:NTHR]]
    return y0, pos


def threshold_beta(b, y0):
    """beta per channel (fp32) such that z0 = y0 A + B, with B rounded to fp32 as gn_cta_coefs rounds it, is exactly
    -1 ulp(B), 0 or +1 ulp(B) (cls = -1, 0, +1).  The classes are tried in an order that rotates over the channels;
    a channel takes the first one some fp32 beta reaches.  Sets beta and B of b -> z0, cls"""
    A, mu, rs, ga = b["A"][0], b["mu_c"][0], b["rs_c"][0], b["gamma"]
    Bs = -y0 * A
    assert torch.equal(Bs.float().double(), Bs), "y0 A is not an fp32 value"
    k = torch.arange(-64, 65, dtype=torch.float64).view(-1, 1)
    cls = torch.full((C,), 2, dtype=torch.long)
    beta = torch.zeros(C, dtype=torch.float64)
    for r in range(3):
        for c in range(C):
            want = (c + r) % 3 - 1
            if cls[c] != 2:
                continue
            Bt = Bs[c] if want == 0 else torch.nextafter(Bs[c].float(), torch.tensor(want * float("inf"))).double()
            b0 = (Bt / 1.25 + mu[c] * rs[c] * ga[c]).float().double()
            bk = (b0 + k[:, 0] * ulp32(b0.view(1))).float().double()
            hit = ((bk - mu[c] * rs[c] * ga[c]) * 1.25).float().double() == Bt
            if bool(hit.any()):
                cls[c], beta[c] = want, bk[int(hit.double().argmax())]
    assert bool((cls != 2).all()), "a channel whose B cannot be placed within one ulp of -y0 A"
    b["beta"] = beta
    b["B"] = ((beta - b["mu_c"] * b["rs_c"] * ga) * b["scale"]).float().double()
    z0 = y0 * A + b["B"][0]
    assert torch.equal(torch.sign(z0), cls.double()) and bool((z0.abs() <= ulp32(Bs) * 1.0001).all())
    return z0, cls


def mask_design(family, branch_on, device="cpu", seed=7):
    """operands of the planted-threshold test: the GroupNorm of branch `branch_on` has -B/A within one fp32 ulp of a
    y0 that occurs at NTHR planted voxels per (n, c); the other stem branch is switched off by a zero dropout scale"""
    gen = torch.Generator().manual_seed(seed)
    dev = torch.device(device)
    if family == "stem":
        n, sp = 2, (8, 16, 32)
        x = grid((n,) + sp + (1,), 16, 2, gen)
        w3, w1 = grid((C, 1, 3, 3, 3), 8, 5, gen), grid((C, 1, 1, 1, 1), 32, 5, gen)
        b3, b1 = grid((C,), 16, 7, gen), grid((C,), 16, 7, gen)
        ys = [bf(t) for t in stem_conv(x.to(dev), w3.to(dev), w1.to(dev), b3.to(dev), b1.to(dev))]
        ops = dict(x=x, w3=w3, w1=w1, b3=b3, b1=b1)
        vox = math.prod(sp)
    else:
        n, sp = 8, (8, 8, 16)
        x = grid((n,) + sp + (CI,), 4, 2, gen)
        w, b = grid((CI, C, 2, 2, 2), 16, 5, gen), grid((C,), 16, 7, gen)
        ys = [bf(up_conv(x.to(dev), w.to(dev), b.to(dev)))]
        ops = dict(x=x, w=w, b=b)
        vox = 8 * math.prod(sp)
    brs = [shared_gn(gen, n, vox, i == branch_on) for i in range(len(ys))]
    y = ys[branch_on]
    y0, pos = pick_y0(y, gen)
    z0, cls = threshold_beta(brs[branch_on], y0)
    for i, b in enumerate(brs):
        if i != branch_on:
            b["beta"], b["gamma"] = brs[branch_on]["beta"], brs[branch_on]["gamma"]
            b["A"] = b["B"] = torch.zeros(n, C, dtype=torch.float64)
    g = torch.zeros((n, y[0, ..., 0].numel(), C), dtype=torch.float64)
    g.scatter_(1, pos, (2.0 ** torch.arange(NTHR, dtype=torch.float64)).view(1, -1, 1).expand(n, NTHR, C).contiguous())
    g = g.view(y.shape).to(dev)
    # the fp32 z (y A + B is exact in fp64) and the references of APPLY and BSUMS
    sides = []
    for yy, b in zip(ys, brs):
        z = (yy * _bc(b["A"], dev) + _bc(b["B"], dev)).float().double()
        gm = torch.where(z > 0, g, 0.0)
        red = (1, 2, 3)
        sides.append(dict(z=z, relu=z.clamp_min(0),
                          sums=torch.stack([gm.sum(red), (gm * yy).sum(red), yy.sum(red)], -1)))
    return dict(family=family, n=n, sp=sp, vox=vox, ys=ys, brs=brs, y0=y0, pos=pos, z0=z0, cls=cls, g=g,
                sides=sides, on=branch_on, **ops)


@pytest.mark.parametrize("family,branch_on", [("stem", 0), ("stem", 1), ("up", 0)])
def test_mask_design_plants_every_threshold_class(family, branch_on):
    """from the operands: at the planted voxels fmaf(y0, A, B) is -1 ulp(B), exactly 0 or +1 ulp(B), each in some
    channel; g there is a distinct power of two, so sum g m decodes the mask bit by bit"""
    d = mask_design(family, branch_on)
    z = d["sides"][branch_on]["z"]
    n = d["n"]
    zp = z.reshape(n, -1, C).gather(1, d["pos"])
    assert torch.equal(zp, d["z0"].view(1, 1, C).expand_as(zp))
    assert set(d["cls"].tolist()) == {-1, 0, 1} and bool((d["z0"] == 0).any())
    gp = d["g"].reshape(n, -1, C).gather(1, d["pos"])
    assert torch.equal(gp, (2.0 ** torch.arange(NTHR)).view(1, -1, 1).expand_as(gp).double())
    assert torch.equal(decode_mask(d["sides"][branch_on]["sums"][..., 0], NTHR, 0),
                       (d["cls"] > 0).view(1, 1, C).expand(n, NTHR, C))


@pytest.mark.gpu
@pytest.mark.parametrize("family,branch_on", [("stem", 0), ("stem", 1), ("up", 0)])
def test_relu_mask_forward_equals_backward_and_z0_is_masked(be, family, branch_on):
    """APPLY, BSUMS and BWD recompute y and the mask in separate launches.  At the planted voxels (z = -1 ulp, 0,
    +1 ulp of B): APPLY's zero / nonzero output is the forward mask; BSUMS's sum g m decodes the backward mask bit by
    bit; BWD's weight gradient (and up_tr32's data gradient), from backward sums with m1 = m2 = 0 (Q = R = 0, so
    dy = m g P exactly), must equal the fp64 reference built from the FORWARD mask.  z = 0 exactly is masked in every
    pass, as torch's ReLU backward does."""
    d = mask_design(family, branch_on, "cuda")
    n, sp, vox, pos = d["n"], d["sp"], d["vox"], d["pos"].cuda()
    gns = [_gn(b, vox) for b in d["brs"]]
    side = d["sides"][branch_on]
    fine = d["ys"][0].shape[1:4]
    out = Guarded((n,) + tuple(fine) + (C,), BF, device="cuda", off=16 if family == "stem" else 0)
    gg = Guarded((n,) + tuple(fine) + (C,), BF, fill=IN_FILL, device="cuda", off=0)
    gg.view.copy_(d["g"].bfloat16())
    if family == "stem":
        gx = Guarded((n,) + sp + (1,), F32, fill=IN_FILL, device="cuda", dense=True)
        gx.view.copy_(d["x"].float())
        p3, p1 = _stem_packs(be, d["w3"], d["w1"])
        b3, b1 = _f(d["b3"]), _f(d["b1"])
        be.stem_gn_apply(gx.view, p3, b3, p1, b1, gns[0], gns[1], out.view)
    else:
        gx = Guarded((n,) + sp + (CI,), BF, fill=IN_FILL, device="cuda")
        gx.view.copy_(d["x"].bfloat16())
        wf = _up_pack(be, d["w"])
        be.up_gn_apply(gx.view, wf, _f(d["b"]), gns[0], out.view)
    want = sum(s["relu"] for s in d["sides"]).float().bfloat16()
    assert_bitwise(out.view, want, f"{family} apply")
    assert_guards(out, f"{family} apply")
    fwd = out.view.double().reshape(n, -1, C).gather(1, pos) > 0                # (n, NTHR, c)
    expect = (d["cls"] > 0).cuda().view(1, 1, C).expand_as(fwd)
    assert_same_mask(expect, fwd, f"{family} forward mask (z = 0 and -1 ulp masked, +1 ulp passed)")

    # BSUMS
    sums = [flat((n, C, 3), torch.float64) for _ in d["brs"]]
    if family == "stem":
        be.stem_gn_bwd_sums(gx.view, p3, b3, p1, b1, gns[0], gns[1], gg.view, sums[0][1], sums[1][1])
    else:
        be.up_gn_bwd_sums(gx.view, wf, _f(d["b"]), gns[0], gg.view, sums[0][1])
    assert_same_mask(fwd, decode_mask(sums[branch_on][1][..., 0], NTHR, 0).cuda(), f"{family} bwd sums mask")
    for i, s in enumerate(d["sides"]):
        assert_equal64(sums[i][1], s["sums"], f"{family} bwd sums branch {i}")
        assert_flat_guards(sums[i][0], "sums")

    # BWD from sums with m1 = m2 = 0: dy = m g P, built here from the forward mask
    bsums = [torch.stack([torch.zeros_like(s["sums"][..., 0]), torch.zeros_like(s["sums"][..., 0]),
                          s["sums"][..., 2]], -1) for s in d["sides"]]
    b = d["brs"][branch_on]
    P = _bc(b["rs_c"] * b["gamma"] * b["scale"], "cuda")
    mfwd = torch.zeros((n, d["g"][0, ..., 0].numel(), C), dtype=torch.bool, device="cuda")
    mfwd.scatter_(1, pos, fwd)
    dy = torch.where(mfwd.view(d["g"].shape), d["g"] * P, 0.0)
    assert torch.equal(bf(dy), dy)
    pg = [flat((C,), F32, 0.0) for _ in range(4)]
    if family == "stem":
        dws = [flat((27, 1, C), F32, 0.0), flat((1, 1, C), F32, 0.0)]
        be.stem_gn_bwd(gx.view, p3, b3, p1, b1, gns[0], gns[1], gg.view, bsums[0].cuda(), bsums[1].cuda(),
                       dws[0][1], dws[1][1], *(t[1] for t in pg))
        xk = bf(d["x"].cuda())
        kind = (K3, K1)[branch_on]
        want_dw = ref_wgrad(dict(kind=kind, dims=3, ca=1, cb=C), xk, dy)
        assert_equal64(dws[branch_on][1], want_dw, f"stem dW branch {branch_on} from the forward mask")
        assert float(dws[1 - branch_on][1].abs().max()) == 0.0, "the switched-off branch has a weight gradient"
    else:
        dwb, dw = flat((8, C, CI), F32, 0.0)
        gdx = Guarded((n,) + sp + (CI,), BF, device="cuda")
        be.up_gn_bwd(gx.view, wf, _f(d["b"]), gns[0], gg.view, bsums[0].cuda(), dw, gdx.view, *(t[1] for t in pg[:3]))
        xc = d["x"].cuda()
        assert_equal64(dw, ref_wgrad(dict(kind=DOWN, dims=3, ca=C, cb=CI), dy, xc), "up dW from the forward mask")
        dx = _ndhwc(F.conv3d(_ncdhw(dy), d["w"].cuda(), None, stride=2))
        assert_bitwise(gdx.view, dx.float().bfloat16(), "up dx from the forward mask")
        assert_guards(gdx, "up dx")
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------- part 4
GN_EPS = 1e-5     # engine.GN_EPS


def _gsum(t, n):
    """(n, C) per channel -> per group sum, back per channel"""
    return per_channel(t.view(n, GROUPS, -1).sum(-1), C // GROUPS)


def oracle_bounds(yr, T, K, gamma, beta, scale, g, vox, L):
    """fp64 reference quantities of one GroupNorm branch relu(GN(yr) s) and the bounds of what the kernels compute.

    yr: the exact conv output (of the bf16-rounded x and w), T: its sum |terms|, K: terms per output.  The kernel's
    fp32 y is within K U T of yr and the stored y within e_y = 2^-8 |yr| + 2 K U T.  Its statistics are fp32 chains
    of at most L additions per CTA, so the group sums are within dS = sum (K U T + L U |yr|) (and 2 |yr| K U T +
    L U yr^2 for the squares), which bounds the fp64 mean (dmu), var (+ the fp32 widening of eps) and
    rstd (dr = rs^3 dvar / 2, to first order with 1 % slack).  A, B are rounded once to fp32 from them: dA, dB.  Then
    fmaf(y, A, B) is within ez = |A| e_y + dA |yr| + dB + 2 U (|A yr| + |B|) of the exact z; voxels with |z| <= ez
    have an ambiguous mask and add |g| to the backward sums' bounds.  The backward sums (fp32 chains of L, of the
    stored y) bound m1, m2 and through them P, Q, R (dP, dQ, dR) as in test_gpu_gn_exact.py; dy is then within
    e_dy of the exact gradient before its bf16 rounding."""
    n = yr.shape[0]
    dev = yr.device
    cpg, m = C // GROUPS, float(C // GROUPS * vox)
    red = (1, 2, 3)
    e_y = 2.0 ** -8 * yr.abs() + 2 * K * U * T
    S1e = (K * U * T + L * U * yr.abs()).sum(red)
    S2e = (2 * yr.abs() * K * U * T + L * U * yr * yr).sum(red)
    st = torch.stack([yr.sum(red), (yr * yr).sum(red)], -1)
    mu = _gsum(st[..., 0], n) / m
    var = _gsum(st[..., 1], n) / m - mu * mu
    rs = 1.0 / torch.sqrt(var + GN_EPS)
    dmu = _gsum(S1e, n) / m
    dvar = _gsum(S2e, n) / m + 2 * mu.abs() * dmu + abs(float(torch.tensor(GN_EPS, dtype=F32)) - GN_EPS)
    dr = 1.01 * 0.5 * rs ** 3 * dvar + U * rs
    ga, be_, s = gamma.double().to(dev), beta.double().to(dev), scale.double().to(dev)
    A = rs * ga * s
    B = (be_ - mu * rs * ga) * s
    dA = (ga * s).abs() * dr + U * A.abs()
    dB = (ga * s).abs() * (mu.abs() * dr + rs * dmu) + 2 * U * ((be_ * s).abs() + (mu * rs * ga * s).abs())
    z = yr * _bc(A, dev) + _bc(B, dev)
    ez = _bc(A.abs(), dev) * e_y + _bc(dA, dev) * yr.abs() + _bc(dB, dev) + 2 * U * (
        (yr * _bc(A, dev)).abs() + _bc(B.abs(), dev))
    amb = z.abs() <= 1.01 * ez
    gm = torch.where(z > 0, g, 0.0)
    S1, S2, S3 = gm.sum(red), (gm * yr).sum(red), yr.sum(red)
    dS1 = L * U * g.abs().sum(red) + (g.abs() * amb).sum(red)
    dS2 = L * U * (g * yr).abs().sum(red) + (g.abs() * e_y).sum(red) + ((g * yr).abs() * amb).sum(red)
    dS3 = L * U * yr.abs().sum(red) + e_y.sum(red)
    gs = (ga * s).abs()
    m1 = _gsum(ga * s * S1, n) / m
    m2 = _gsum(ga * rs * s * (S2 - mu * S1), n) / m
    dm1 = _gsum(gs * dS1, n) / m
    dm2 = _gsum(gs * (rs * (dS2 + mu.abs() * dS1 + dmu * S1.abs()) + dr * (S2 - mu * S1).abs()), n) / m
    P, Q, R = rs * ga * s, -rs * rs * m2, -rs * m1 + rs * rs * mu * m2
    dP = dr * gs + U * P.abs()
    dQ = 2 * rs * dr * m2.abs() + rs * rs * dm2 + U * Q.abs()
    dR = (dr * m1.abs() + rs * dm1 + 2 * rs * dr * (mu * m2).abs() + rs * rs * (dmu * m2.abs() + mu.abs() * dm2)
          + U * ((rs * m1).abs() + (rs * rs * mu * m2).abs()) + U * R.abs())
    e_dy = (g.abs() * _bc(dP, dev) + yr.abs() * _bc(dQ, dev) + _bc(dR, dev) + e_y * _bc(Q.abs(), dev)
            + 2 * U * (g.abs() * _bc(P.abs(), dev) + (yr * _bc(Q, dev)).abs() + _bc(R.abs(), dev))
            + amb * g.abs() * _bc(P.abs(), dev))
    # per-sample parameter terms (fp64 from the sums, one fp32 rounding each, fp32 atomics)
    tb, tg = s * S1, rs * s * (S2 - mu * S1)
    tbi = rs * ga * s * S1 + Q * S3 + R * vox
    bd = dict(dbeta=(s.abs() * dS1).sum(0), dgamma=(s.abs() * (dr * (S2 - mu * S1).abs() + rs * (
        dS2 + mu.abs() * dS1 + dmu * S1.abs()))).sum(0),
        dbias=(gs * (dr * S1.abs() + rs * dS1) + dQ * S3.abs() + Q.abs() * dS3 + dR * vox).sum(0))
    mag = dict(dbeta=tb.abs().sum(0), dgamma=tg.abs().sum(0), dbias=(rs * gs * S1.abs() + (Q * S3).abs() +
                                                                     (R * vox).abs()).sum(0))
    return dict(ez=ez, e_dy=e_dy, bd=bd, mag=mag)


def _within(got, want, bound, what):
    bad = (got.double() - want).abs() > bound
    if bool(bad.any()):
        idx = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} outside the bound; first at {idx}: got "
                             f"{float(got[idx])!r}, fp64 {float(want[idx])!r}, bound {float(bound[idx]):.3g}")


def _wg_abs(kind, a, b):
    return ref_wgrad(dict(kind=kind, dims=3, ca=a.shape[-1], cb=b.shape[-1]), a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["stem", "up"])
def test_block_against_fp64_autograd(be, family):
    """The kernels' own passes chained (STATS -> APPLY -> BSUMS -> BWD) with realistic data and GN_EPS = 1e-5,
    against torch fp64 autograd of the functional block:
        stem (2 x 96^3):        relu(GN(conv3d(x, w3) + b3) s3) + relu(GN(conv3d(x, w1) + b1) s1), one gamma, beta
        up (2 x 48^3 coarse):   relu(GN(conv_transpose3d(x, w) + b) s)
    The restatement rounds where the library is specified to round: x and w to bf16 (the reference convolves the
    rounded values).  The bounds (oracle_bounds) follow from the fp32 chains and from the rounding of the stored y,
    the coefficients, dy (2^-8 relative: bf16) and the outputs (2^-8 relative).  dW: sum over voxels of |x| times the
    dy bound, plus the fp32 chain of stem_dw_chain / up_dw_chain; dx: the same over its 128 products, plus one bf16
    rounding; d gamma, d beta, d bias: the propagated sum bounds plus (2N + 1) U sum |terms| of the atomics."""
    sms = device_sms()
    gen = torch.Generator().manual_seed(31)
    r = lambda *sh, sc=1.0: (torch.randn(*sh, generator=gen, dtype=torch.float64) * sc).cuda()
    gamma, beta = (1 + 0.2 * r(C)).float(), (0.1 * r(C)).float()
    if family == "stem":
        n, sp = 2, (96, 96, 96)
        fine, vox = sp, math.prod(sp)
        x = r(n, *sp, 1, sc=2.0).float()
        ws = [r(C, 1, 3, 3, 3, sc=0.3).float(), r(C, 1, 1, 1, 1, sc=0.5).float()]
        bs = [(0.1 * r(C)).float(), (0.1 * r(C)).float()]
        kinds, Ks = (K3, K1), (28, 2)
        walk = stem_walk(n, sp, sms, False)
        L = 2 * walk["tpc"] * walk["tw"] // 16 + 6
    else:
        n, sp = 2, (48, 48, 48)
        fine = tuple(2 * v for v in sp)
        vox = math.prod(fine)
        x = r(n, *sp, CI).bfloat16()
        ws = [r(CI, C, 2, 2, 2, sc=0.1).float()]
        bs = [(0.1 * r(C)).float()]
        Ks = (33,)
        walk = up_walk(n, sp, sms, False)
        L = walk["tpc"] * 64 + 6
    nb = len(ws)
    scales = [((torch.rand(n, C, generator=gen) > 0.2).double() * 1.25).float().cuda() for _ in range(nb)]
    g = r(n, *fine, C).bfloat16()

    # fp64 autograd reference on the bf16-rounded x and w
    xk = bf(x.double())
    wq = [bf(w.double()).requires_grad_(True) for w in ws]
    bq = [b.double().requires_grad_(True) for b in bs]
    gq, btq = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    with torch.enable_grad():
        if family == "stem":
            yr = [F.conv3d(_ncdhw(xk), wq[0], bq[0], padding=1), F.conv3d(_ncdhw(xk), wq[1], bq[1])]
        else:
            xq = xk.clone().requires_grad_(True)
            yr = [F.conv_transpose3d(_ncdhw(xq), wq[0], bq[0], stride=2)]
        for t in yr:
            t.retain_grad()
        o = sum(F.relu(F.group_norm(t, GROUPS, gq, btq, GN_EPS) * sc.double().view(n, C, 1, 1, 1))
                for t, sc in zip(yr, scales))
        o.backward(_ncdhw(g.double()))
    ref_out = _ndhwc(o.detach())
    yrs = [_ndhwc(t.detach()) for t in yr]
    dys = [_ndhwc(t.grad) for t in yr]
    if family == "stem":
        Ts = [_ndhwc(F.conv3d(_ncdhw(xk.abs()), w.detach().abs(), b.detach().abs(), padding=w.shape[-1] // 2))
              for w, b in zip(wq, bq)]
    else:
        Ts = [up_conv(xk.abs(), wq[0].detach().abs(), bq[0].detach().abs())]
    gd = g.double()
    obs = [oracle_bounds(yy, T, K, gamma, beta, sc, gd, vox, L) for yy, T, K, sc in zip(yrs, Ts, Ks, scales)]

    # the kernels' chain
    stats = [torch.zeros((n, C, 2), dtype=torch.float64, device="cuda") for _ in range(nb)]
    sums = [torch.zeros((n, C, 3), dtype=torch.float64, device="cuda") for _ in range(nb)]
    gns = [(st, gamma, beta, sc, vox, GROUPS, GN_EPS) for st, sc in zip(stats, scales)]
    out = Guarded((n,) + fine + (C,), BF, device="cuda", off=16 if family == "stem" else 0)
    gg = Guarded((n,) + fine + (C,), BF, fill=IN_FILL, device="cuda", off=0)
    gg.view.copy_(g)
    pg = {k: torch.zeros(C, device="cuda") for k in ("dgamma", "dbeta", "db0", "db1")}
    dws = ([torch.zeros((27, 1, C), device="cuda"), torch.zeros((1, 1, C), device="cuda")] if family == "stem" else
           [torch.zeros((8, C, CI), device="cuda")])
    if family == "stem":
        p3, p1 = _stem_packs(be, ws[0], ws[1])
        be.stem_gn_stats(x, p3, bs[0], p1, bs[1], stats[0], stats[1])
        be.stem_gn_apply(x, p3, bs[0], p1, bs[1], gns[0], gns[1], out.view)
        be.stem_gn_bwd_sums(x, p3, bs[0], p1, bs[1], gns[0], gns[1], gg.view, sums[0], sums[1])
        be.stem_gn_bwd(x, p3, bs[0], p1, bs[1], gns[0], gns[1], gg.view, sums[0], sums[1], dws[0], dws[1],
                       pg["dgamma"], pg["dbeta"], pg["db0"], pg["db1"])
        dw_chain = stem_dw_chain(n, sp, sms)
    else:
        wf = _up_pack(be, ws[0])
        be.up_gn_stats(x, wf, bs[0], stats[0])
        be.up_gn_apply(x, wf, bs[0], gns[0], out.view)
        be.up_gn_bwd_sums(x, wf, bs[0], gns[0], gg.view, sums[0])
        gdx = Guarded((n,) + sp + (CI,), BF, device="cuda")
        be.up_gn_bwd(x, wf, bs[0], gns[0], gg.view, sums[0], dws[0], gdx.view, pg["dgamma"], pg["dbeta"], pg["db0"])
        dw_chain = up_dw_chain(n, sp, sms)
    torch.cuda.synchronize()

    # forward: the sum of the branches' z bounds, the fp32 branch sum, one bf16 rounding
    E = sum(ob["ez"] for ob in obs) + U * ref_out.abs()
    _within(out.view, ref_out, 2.0 ** -8 * (ref_out.abs() + E) + E, f"{family} apply")
    assert_guards(out, f"{family} apply")
    # weight gradients (dW[t][ci][co] layouts of ref_wgrad) against autograd
    for i, (ob, dy) in enumerate(zip(obs, dys)):
        Edy = ob["e_dy"] + 2.0 ** -8 * (dy.abs() + ob["e_dy"])
        if family == "stem":
            kind = kinds[i]
            want = wq[i].grad.reshape(C, 1, -1).permute(2, 1, 0)
            bound = _wg_abs(kind, xk.abs(), Edy) + dw_chain * U * _wg_abs(kind, xk.abs(), dy.abs() + Edy)
        else:
            want = wq[0].grad.reshape(CI, C, -1).permute(2, 1, 0)
            bound = _wg_abs(DOWN, Edy, xk.abs()) + dw_chain * U * _wg_abs(DOWN, dy.abs() + Edy, xk.abs())
            wa = wq[0].detach().abs()
            edx = _ndhwc(F.conv3d(_ncdhw(Edy), wa, None, stride=2))
            chain = 130 * U * _ndhwc(F.conv3d(_ncdhw(dy.abs() + Edy), wa, None, stride=2))
            dxr = xq.grad
            _within(gdx.view, dxr, edx + chain + 2.0 ** -8 * (dxr.abs() + edx + chain), "up dx")
            assert_guards(gdx, "up dx")
        _within(dws[i], want, 1.01 * bound + 1e-30, f"{family} dW branch {i}")
    # d gamma, d beta (both branches), d bias (per branch)
    Nn = nb * n + 1
    for k, want in (("dgamma", gq.grad), ("dbeta", btq.grad)):
        bound = sum(ob["bd"][k] + Nn * U * ob["mag"][k] for ob in obs)
        _within(pg[k], want, 1.01 * bound + 1e-30, f"{family} {k}")
    for i, ob in enumerate(obs):
        _within(pg[f"db{i}"], bq[i].grad, 1.01 * (ob["bd"]["dbias"] + Nn * U * ob["mag"]["dbias"]) + 1e-30,
                f"{family} d bias {i}")
