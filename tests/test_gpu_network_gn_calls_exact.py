"""Every GroupNorm, activation, upsample and head call a training step of the networks makes, replayed bit for bit
against fp64 at the buffer layouts the engine hands the kernels.

test_gpu_gn_exact.py, test_gpu_unet3dthin.py and test_gpu_resnet.py run these kernels on synthetic layouts (pitch
C + 16, contiguous guarded buffers) or hold them to norm-wise tolerances.  The networks hand them other views: the
halves of a [up | skip] concat (pitch 2C at channel offset 0 or C) as outputs and as upstream gradients, parameter-
gradient views inside the one flat gradient bucket, fp64 sums from the engine's zero arena, and ResNet2d's batch of
128, where the fused GroupNorm backward runs at exactly its size limit.  This file records what the engine launches
and replays it (the record-and-rebuild machinery is test_gpu_network_calls_exact.py's).

1. Record.  `Recorder` with `ops=OPS` and `hook=record_call`: per tensor operand its sizes, strides, storage offset,
   storage length, dtype and address mod 512 (trec); per GroupNorm descriptor its tensors and its structure (vox,
   groups, whether a dropout scale is present), never its values; the `sum_y_from_stats` flag.
2. Replay.  Every unique call runs again with each tensor rebuilt at its recorded layout (Rebuilt), the tensors of
   the GroupNorm descriptors and the head weights included: inputs hold IN_FILL outside the view, outputs the NaN
   pattern.  Only layouts, shapes, dtypes, optional operands and flags come from the recording; the values come from
   the exact designs (test_gpu_gn_exact.design, eps = 2^-10; the head grids of test_gpu_head_loss_exact; the
   upsample grids of test_gpu_unet3dthin).  Outputs must equal fp64 bit for bit, nothing outside an output view may
   change and no input may change.  Parameter gradients are added (+=) into a prefilled view at its recorded
   position in a rebuilt copy of the whole flat gradient bucket: the view must equal prefill + contributions and
   every other element of the bucket (the neighbouring parameters' gradients) must keep its bits.
   The coefficient forms (COEF_FORMS) are recorded but not replayed: only layers wider than 512 channels take them
   and none of these networks has one.  stem_gn_* / up_gn_* are not replayed either: every output, upstream
   gradient and dx layout the networks hand them must be one that test_gpu_fused_gn_exact.py runs them at (LAYOUTS).
3. The fused GroupNorm backward adds one fp32 atomic per sample to each parameter gradient, in any order.  For
   N > 2 its operands (fused_operands: y antisymmetric in voxel halves, so that sum y = 0 per (n, c); a sparse g)
   make every per-sample contribution and every partial sum of them a multiple of one quantum below 2^24 quanta
   (fused_exact, asserted for ResNet2d's batch of 128 in the CPU part and again on every replay), so its parameter
   gradients are compared with fp64 bit for bit; a call with N > 2 and no exact design fails.  For N <= 2, y is
   drawn freely (sum y and the Q sum-y term of d bias are nonzero); where that or a voxel count that is not a power
   of two (m1 = sum / (cpg vox) rounds in fp64) leaves no exact design, the parameter gradients, from a zero prefill
   where two atomics commute, must equal gn_bwd_apply_gn's on the same sums.  Its sums are compared with fp64, its
   dy with gn_bwd_apply_gn on them, and its barrier counter must hold the grid size afterwards.
4. Classifier head (cls_head_fwd / _bwd).  x in {-4..4} 2^-2, so the fp32 voxel sum is exact; pooled is one fp32
   multiply of that sum by fp32(1/vox) and is compared bit for bit.  Where vox is a power of two every output is
   exact and compared bit for bit; otherwise each element is held to the fixed-order fmaf chain bound
   (terms + 1) u sum |terms| (CLS_BOUND names those outputs).  dx must equal dp (read back from `work`) rounded to
   the dtype at every voxel.

The CPU part records small steps on the emulated backend (tests/emu_backend.py) and checks the recorder, the rebuilt
layouts, the design preconditions and the checkers; the GPU part is marked `gpu`."""
import math
import time
from collections import namedtuple

import pytest
import torch

from test_gpu_conv_exact import IN_FILL
from test_gpu_fused_gn_exact import LAYOUTS as FUSED_GN_LAYOUTS
from test_gpu_gn_exact import (EPS, G_ALPHA, GROUPS, U, Y_ALPHA, bwd_coefs, check_design, design, ew_blocks,
                               fused_supported, param_contribs, quantum)
from test_gpu_head_loss_exact import QB, QG, QW, QX, check_probs, head_bwd_bound, head_fwd_bound
from test_gpu_network_calls_exact import (DTYPES, FILL_BITS, WORKLOADS, Rebuilt, check_in, pitch, record_step, trec,
                                          unique_calls)
from test_gpu_unet3dthin import up2_ref, up2t_ref

# the recorded entry points: positional argument roles
ARGS = {
    "gn_finalize": "stats gamma beta scale vox groups eps coef mr",
    "apply": "y1 c1 y2 c2 res out",
    "apply_gn": "y1 gn1 y2 gn2 res out",
    "gn_bwd_reduce": "g y coef sums",
    "gn_bwd_reduce_gn": "g y gn sums",
    "gn_bwd_apply": "g y coef coef3 dy",
    "gn_bwd_apply_gn": "g y gn sums dy dgamma dbeta dbias sum_y_from_stats",
    "gn_bwd_fused_gn": "g y gn sums counter dy dgamma dbeta dbias",
    "gn_bwd_finalize": "sums mr gamma scale vox groups coef3 dgamma dbeta dbias",
    "colsum": "dy out",
    "upsample_add": "a e s",
    "upsample_bwd": "g_s g_a",
    "head_fwd": "x w bias logits probs",
    "head_bwd": "x dlogits w dx dw db",
    "head_probs": "logits probs",
    "head_mask": "x w bias mask threshold",
    "mask_logits": "logits threshold mask",
    "cls_head_fwd": "x w1 b1 w2 b2 pooled hidden logits",
    "cls_head_bwd": "dlogits pooled hidden w1 w2 work dx dw1 db1 dw2 db2",
    "stem_gn_apply": "x w3 b3 w1 b1 gn3 gn1 out",
    "stem_gn_bwd_sums": "x w3 b3 w1 b1 gn3 gn1 g sums3 sums1",
    "stem_gn_bwd": "x w3 b3 w1 b1 gn3 gn1 g sums3 sums1 dw3 dw1 dgamma dbeta db3 db1",
    "up_gn_apply": "x wpk bias gn out",
    "up_gn_bwd_sums": "x wpk bias gn g sums",
    "up_gn_bwd": "x wpk bias gn g sums dw dx dgamma dbeta dbias",
}
OPS = tuple(ARGS)
FAMILY = {**{op: "gn_fwd" for op in ("gn_finalize", "apply", "apply_gn")},
          **{op: "gn_bwd" for op in OPS if op.startswith("gn_bwd") or op == "colsum"},
          "upsample_add": "upsample", "upsample_bwd": "upsample",
          **{op: "head" for op in ("head_fwd", "head_bwd", "head_probs", "head_mask", "mask_logits", "cls_head_fwd",
                                   "cls_head_bwd")},
          **{op: "fused_gn" for op in OPS if op.startswith(("stem_gn", "up_gn"))}}
# the coefficient forms (gn_finalize + apply, gn_bwd_reduce + gn_bwd_finalize + gn_bwd_apply): recorded, but only layers
# wider than 512 channels take them (engine.conv_gn) and none of these networks has one; test_gpu_gn_exact.py holds them
COEF_FORMS = {"gn_finalize", "apply", "gn_bwd_reduce", "gn_bwd_finalize", "gn_bwd_apply"}
NOT_IN_TRAINING = {"head_mask", "mask_logits"}     # the inference form of the head (engine.head, mask_threshold set)
SMS = 132                                          # H100 SXM (the CPU part; the GPU part reads the device's)

# cls_head outputs held to the fmaf chain bound instead of bit for bit, with the reason: at a voxel count that is not
# a power of two, pooled carries the rounding of fp32(1/vox), and hidden, logits and the two weight gradients that
# read pooled / hidden inherit it; every other output (dh, dp, db1, db2, dx) stays bit for bit
CLS_BOUND = {"hidden", "logits", "dw1", "dw2"}

TABLE = {**WORKLOADS,
         "unet3dthin_96": ("UNet3dthin", (1, 2), 2, (96, 96, 96)),
         "unet3dthin_128x112": ("UNet3dthin", (1, 2), 1, (128, 112, 112))}
CPU_TABLE = {"vnet3d_32": ("VNet3d", (1, 2), 2, (32, 32, 32)),
             "unet2d_64": ("UNet2d", (1, 1), 2, (64, 64)),
             "resnet3d_32": ("ResNet3d", (1, 4), 2, (32, 32, 32)),
             "resnet2d_32": ("ResNet2d", (1, 10), 4, (32, 32)),
             "unet3dthin_32": ("UNet3dthin", (1, 2), 1, (32, 32, 32))}

GnRec = namedtuple("GnRec", "stats gamma beta scale vox groups has_scale")
Sig = namedtuple("Sig", "op args")                 # args: ((role, TRec | GnRec | int | bool | None), ...)


# ---------------------------------------------------------------------------------------------------------- record
def _rec_arg(v):
    if torch.is_tensor(v):
        return trec(v)
    if isinstance(v, tuple):                       # a GroupNorm descriptor, by structure
        stats, gamma, beta, scale, vox, groups, _ = v
        return GnRec(trec(stats), trec(gamma), trec(beta), trec(scale), vox, groups, scale is not None)
    if isinstance(v, (bool, int)) and not isinstance(v, float):
        return v
    return None                                     # eps, threshold: values, not layout


def record_call(rec, op, a, k):
    names = ARGS[op].split()
    vals = dict(zip(names, a))
    vals.update(k)
    args = tuple((r, _rec_arg(vals.get(r))) for r in names)
    return {"sig": Sig(op, args), "tag": rec.tag, "weight": None}


def record(backend, workload, precision, device, table=TABLE):
    return record_step(backend, workload, precision, device, table, ops=OPS, hook=record_call)


# ---------------------------------------------------------------------------------------------------------- designs
def fused_operands(n, sp, c, dtype_name):
    """y, g of a fused GroupNorm backward (CPU, seeded by the shape); g from G_ALPHA at one voxel in eight.  For N > 2
    y is antisymmetric in the two voxel halves of each (n, c): sum y = 0, so the Q sum-y term of d bias, whose quantum
    is far below the others', vanishes and the batch's parameter gradients stay exact.  For N <= 2, where the
    parameter gradients are also compared with gn_bwd_apply_gn's, y is drawn freely, so the kernel's third sum (sum y)
    and that term are nonzero."""
    V = math.prod(sp)
    gen = torch.Generator().manual_seed(n * 1000003 + V * 101 + c)
    if n > 2:
        assert V % 2 == 0
        half = Y_ALPHA[torch.randint(0, 9, (n, V // 2, c), generator=gen)]
        y = torch.cat([half, -half], 1)
    else:
        y = Y_ALPHA[torch.randint(0, 9, (n, V, c), generator=gen)]
    g = G_ALPHA[torch.randint(0, 3, (n, V, c), generator=gen)] * (torch.rand((n, V, c), generator=gen) < 0.125)
    shape = (n,) + tuple(sp) + (c,)
    return y.view(shape), g.view(shape)


def bwd_sums(y, g, A, B):
    """sum g m, sum g m y, sum y per (n, c) in fp64, m = [fmaf(y, A, B) > 0]"""
    n, c = A.shape
    z = y * A.view(n, 1, 1, 1, c) + B.view(n, 1, 1, 1, c)
    gm = torch.where(z > 0, g, 0.0)
    return torch.stack([gm.sum((1, 2, 3)), (gm * y).sum((1, 2, 3)), y.sum((1, 2, 3))], -1)


def fused_exact(b, sums, vox, prefill):
    """the per-sample d gamma, d beta, d bias of sums and whether each is exact in any order: -> (contributions,
    {name: (sum |terms| in quanta)})"""
    co = bwd_coefs(b, sums, vox)
    pc = param_contribs(b, sums, co, vox, sums[..., 2])
    quanta = {}
    for k, t in pc.items():
        q = quantum(prefill[k], t)
        quanta[k] = float((prefill[k].abs() + t.abs().sum(0)).max()) / q
    return pc, quanta


def fused_prefill(b, sums, vox, seed):
    co = bwd_coefs(b, sums, vox)
    pc = param_contribs(b, sums, co, vox, sums[..., 2])
    gen = torch.Generator().manual_seed(seed)
    return {k: torch.randint(-3, 4, t.shape[1:], generator=gen).double() * quantum(t) for k, t in pc.items()}


def fused_design(n, sp, c, has_scale, dtype_name):
    """everything of one fused replay that does not need a GPU"""
    cs = dict(n=n, sp=tuple(sp), c=c, dtype=DTYPES[dtype_name], off=8)
    d = design(cs, drop=has_scale)
    y, g = fused_operands(n, sp, c, dtype_name)
    sums = bwd_sums(y, g, d["b1"]["A"], d["b1"]["B"])
    pre = fused_prefill(d["b1"], sums, d["vox"], n + c)
    pc, quanta = fused_exact(d["b1"], sums, d["vox"], pre)
    return dict(d=d, y=y, g=g, sums=sums, pre=pre, pc=pc, quanta=quanta)


def cls_operands(n, c, hd, k, gen):
    x_alpha = torch.arange(-4, 5, dtype=torch.float64) * QX
    dev = gen.device
    w1 = torch.randint(-8, 9, (hd, c), generator=gen, device=dev).double() * QW
    b1 = torch.randint(-64, 65, (hd,), generator=gen, device=dev).double() * QB
    w2 = torch.randint(-8, 9, (k, hd), generator=gen, device=dev).double() * QW
    b2 = torch.randint(-64, 65, (k,), generator=gen, device=dev).double() * QB
    dl = torch.randint(-1, 2, (n, k), generator=gen, device=dev).double() * QG
    return x_alpha.to(dev), w1, b1, w2, b2, dl


def pooled_model(S, vox):
    """the kernel's mean: one IEEE fp32 multiply of the (exact) fp32 voxel sum by fp32(1/vox)"""
    inv = torch.tensor(1.0 / vox, dtype=torch.float32, device=S.device)
    return (S.float() * inv).double()


def chain(terms, extra=None):
    """sums over the last axis (+ extra): fp64 value, fixed-order fmaf chain bound (terms + 1) u sum |terms|, and
    sum |terms|"""
    want = terms.sum(-1) + (0 if extra is None else extra) + 0.0          # + 0.0: an all-zero sum is +0
    mag = terms.abs().sum(-1) + (0 if extra is None else extra.abs())
    return want, (terms.shape[-1] + 1) * U * mag, mag


# ---------------------------------------------------------------------------------------------------------- checks
def mismatch(got, want, what):
    """None, or a message naming the first index whose bits differ (got in its own dtype, want rounded to it)"""
    want = want.to(got.dtype)
    ib = FILL_BITS[got.dtype][0]
    ne = got.contiguous().view(ib) != want.contiguous().view(ib)
    if not bool(ne.any()):
        return None
    idx = tuple(ne.nonzero()[0].tolist())
    return (f"{what}: {int(ne.sum())} of {ne.numel()} differ; first at {idx}: got {float(got[idx])!r}, want "
            f"{float(want[idx])!r}")


def out_msgs(rb, want, what):
    """an output view bit for bit, then nothing outside it changed"""
    m = mismatch(rb.view, want, f"{what}: inside the view")
    pos = rb.changed()
    return [m, None if pos is None else f"{what}: written outside the view: {pos}"]


def bound_msg(got, want, tol, what):
    bad = (got.double() - want).abs() > tol
    if not bool(bad.any()):
        return None
    i = tuple(bad.nonzero()[0].tolist())
    return (f"{what}: {int(bad.sum())} of {bad.numel()} outside the chain bound; first at {i}: got {float(got[i])!r}, "
            f"fp64 {float(want[i])!r}, bound {float(tol[i]):.3g}")


def exact_ok(mag, q):
    return float(mag.max()) < 2 ** 24 * q


class Log:
    def __init__(self, label, sms=SMS):
        self.label, self.failures, self.forms, self.sms = label, [], set(), sms

    def fail(self, sig, tags, msg):
        self.failures.append(f"{self.label} {sig.op} tags={','.join(tags)}: {msg}")


# ---------------------------------------------------------------------------------------------------------- replay
def _draw(alpha, shape, gen):
    return alpha.to(gen.device)[torch.randint(0, alpha.numel(), shape, generator=gen, device=gen.device)]


def _bc(t):
    return t.view(t.shape[0], 1, 1, 1, t.shape[1]).cuda()


def _gn_in(b, gnr):
    """a GroupNorm descriptor with its statistics, gamma, beta and scale rebuilt at their recorded layouts -> (the
    descriptor, the rebuilt inputs)"""
    parts = [_in(gnr.stats, b["stats"].cuda()), _in(gnr.gamma, b["gamma"].cuda()), _in(gnr.beta, b["beta"].cuda()),
             _in(gnr.scale, b["scale"].cuda()) if gnr.has_scale else None]
    desc = (parts[0].view, parts[1].view, parts[2].view, _v(parts[3]), gnr.vox, GROUPS, EPS)
    return desc, [p for p in parts if p is not None]


def _inputs_unchanged(rbs, what):
    return [check_in(rb, f"{what} {i}") for i, rb in enumerate(rbs)]


def _pgrad(r, pre):
    """a parameter-gradient view rebuilt in its flat bucket: IN_FILL around it (the neighbours), prefill inside"""
    return Rebuilt(r, IN_FILL).set(pre.view(r.sizes)).snapshot()


def _in(r, v):
    return None if r is None else Rebuilt(r, IN_FILL).set(v).snapshot()


def _out(r):
    return None if r is None else Rebuilt(r).snapshot()


def _v(rb):
    return None if rb is None else rb.view


def _design_for(yr, gnr, drop):
    cs = dict(n=yr.sizes[0], sp=yr.sizes[1:4], c=yr.sizes[-1], dtype=DTYPES[yr.dtype], off=8)
    d = design(cs, drop=drop)
    inexact = check_design(cs, d)
    if gnr is not None:
        assert gnr.vox == d["vox"] and gnr.groups == GROUPS, "descriptor does not match the operand"
    return cs, d, inexact


def replay_gn_fwd(be, sig, gen, log):
    A = dict(sig.args)
    if sig.op in COEF_FORMS:
        return [f"{sig.op} has no replay here: only layers wider than 512 channels take it (test_gpu_gn_exact.py)"]
    msgs = []
    yr, y2r, rr, outr = A["y1"], A["y2"], A["res"], A["out"]
    g1, g2 = A["gn1"], A["gn2"]
    drop = g1.has_scale
    if g2 is not None and g2.has_scale != drop:
        return ["the two branches differ in having a dropout scale"]
    _, d, _ = _design_for(yr, g1, drop)
    b1, b2 = d["b1"], d["b2"]
    y1 = _draw(Y_ALPHA, yr.sizes, gen)
    y2 = _draw(Y_ALPHA, yr.sizes, gen) if y2r is not None else None
    res = _draw(Y_ALPHA, yr.sizes, gen) if rr is not None else None
    ry1, ry2, rres, rout = _in(yr, y1), _in(y2r, y2), _in(rr, res), _out(outr)
    want = (y1 * _bc(b1["A"]) + _bc(b1["B"])).clamp_min(0)
    if y2 is not None:
        want = want + (y2 * _bc(b2["A"]) + _bc(b2["B"])).clamp_min(0)
    if res is not None:
        want = want + res
    gn1, ins = _gn_in(b1, g1)
    gn2, ins2 = _gn_in(b2, g2) if y2 is not None else (None, [])
    be.apply_gn(ry1.view, gn1, _v(ry2), gn2, _v(rres), rout.view)
    torch.cuda.synchronize()
    log.forms.add(f"{sig.op}:{'2' if y2 is not None else '1'}{'+res' if res is not None else ''}"
                  f"{'' if drop else ':noscale'}")
    msgs += out_msgs(rout, want, "out")
    for rb, what in ((ry1, "y1"), (ry2, "y2"), (rres, "res")):
        if rb is not None:
            msgs.append(check_in(rb, what))
    return msgs + _inputs_unchanged(ins, "gn1 operand") + _inputs_unchanged(ins2, "gn2 operand")


def _pgrad_checks(A, pre, contrib, inexact, tag):
    """the dgamma / dbeta / dbias views: prefill + contributions"""
    msgs, out = [], {}
    for k in ("dgamma", "dbeta", "dbias"):
        if A.get(k) is not None:
            out[k] = _pgrad(A[k], pre[k].float().cuda())

    def check():
        for k, rb in out.items():
            if tag + k in inexact:
                msgs.append(f"{k}: the design does not make it exact")
                continue
            want = pre[k] + contrib[k].sum(0)
            msgs.extend(out_msgs(rb, want.float().view(rb.r.sizes).cuda(), k))
        return msgs
    return out, check


def replay_gn_bwd(be, sig, gen, log):
    A = dict(sig.args)
    op = sig.op
    if op in COEF_FORMS:
        return [f"{op} has no replay here: only layers wider than 512 channels take it (test_gpu_gn_exact.py)"]
    if op == "colsum":
        dr, outr = A["dy"], A["out"]
        g = _draw(G_ALPHA, dr.sizes, gen)
        cpre = (torch.arange(outr.sizes[0]) % 7 - 3).double() / 8
        rg, ro = _in(dr, g), _pgrad(outr, cpre.float().cuda())
        be.colsum(rg.view, ro.view)
        torch.cuda.synchronize()
        log.forms.add("colsum")
        return out_msgs(ro, (cpre.cuda() + g.sum((0, 1, 2, 3))).float(), "bias (+=)") + [check_in(rg, "dy")]
    gr, yr, gnr = A["g"], A["y"], A["gn"]
    if op == "gn_bwd_fused_gn":
        return replay_fused(be, sig, A, log)
    _, d, inexact = _design_for(yr, gnr, gnr.has_scale)
    b1, co = d["b1"], d["co"]
    y = _draw(Y_ALPHA, yr.sizes, gen)
    g = _draw(G_ALPHA, gr.sizes, gen)
    ry, rg = _in(yr, y), _in(gr, g)
    gn, ins = _gn_in(b1, gnr)
    msgs = []
    if op == "gn_bwd_reduce_gn":
        rs = _out(A["sums"])
        rs.view.zero_()
        rs.snapshot()
        be.gn_bwd_reduce_gn(rg.view, ry.view, gn, rs.view)
        torch.cuda.synchronize()
        log.forms.add(op)
        msgs += out_msgs(rs, bwd_sums(y, g, b1["A"].cuda(), b1["B"].cuda()), "sums")
    else:
        z = y * _bc(b1["A"]) + _bc(b1["B"])
        want = torch.where(z > 0, g * _bc(co["P"]), 0.0) + y * _bc(co["Q"]) + _bc(co["R"])
        rdy = _out(A["dy"])
        fs = A["sum_y_from_stats"]
        tag = "from stats " if fs else ""
        rsum = _in(A["sums"], d["sums"].cuda())
        ins.append(rsum)
        pg, check = _pgrad_checks(A, d["prefill"], d["pc_st"] if fs else d["pc"], inexact, tag)
        be.gn_bwd_apply_gn(rg.view, ry.view, gn, rsum.view, rdy.view, pg["dgamma"].view, pg["dbeta"].view,
                           pg["dbias"].view if "dbias" in pg else None, sum_y_from_stats=fs)
        torch.cuda.synchronize()
        log.forms.add(f"{op}{':from_stats' if fs else ''}")
        msgs += out_msgs(rdy, want, "dy") + check()
    msgs += [check_in(ry, "y"), check_in(rg, "g")] + _inputs_unchanged(ins, "gn operand")
    return msgs


def fused_grid(n, V, c, dtype, sms):
    """the CTAs of gn_bwd_fused_gn (elementwise.cu:1212-1215): all co-resident, at most one per SM -- the value the
    grid barrier leaves in the counter word"""
    G = c // (8 if dtype == torch.bfloat16 else 4)
    bx = ew_blocks(V, G, n, 1, sms)[0]
    while bx > 1 and bx * n > sms:
        bx -= 1
    if 256 % G:
        bx = bx // G * G
    return bx * n


def replay_fused(be, sig, A, log):
    gr, yr, gnr = A["g"], A["y"], A["gn"]
    n, sp, c = yr.sizes[0], yr.sizes[1:4], yr.sizes[-1]
    fd = fused_design(n, sp, c, gnr.has_scale, yr.dtype)
    d, b1 = fd["d"], fd["d"]["b1"]
    check_design(dict(n=n, sp=sp, c=c, dtype=DTYPES[yr.dtype], off=8), d)
    exact = all(q < 2 ** 24 for q in fd["quanta"].values())
    if not exact and n > 2:
        return [f"no exact design: d {k} has sum |terms| {q:.3g} quanta, not below 2^24"
                for k, q in fd["quanta"].items() if q >= 2 ** 24]
    msgs = []
    y, g = fd["y"].cuda(), fd["g"].cuda()
    ry, rg = _in(yr, y), _in(gr, g)
    rs, rc, rdy = _out(A["sums"]), _out(A["counter"]), _out(A["dy"])
    for rb in (rs, rc):
        rb.view.zero_()
        rb.snapshot()
    # exact design: prefill + contributions against fp64.  Otherwise (N <= 2 at a voxel count that is not a power of
    # two, where m1 = sum / (cpg vox) rounds in fp64): against gn_bwd_apply_gn on the same sums from a zero prefill,
    # where the order of the two per-sample atomics cannot change the sum
    pre = fd["pre"] if exact else {k: torch.zeros_like(v) for k, v in fd["pre"].items()}
    pg, check = _pgrad_checks(A, pre, fd["pc"], set(), "")
    gnt, ins = _gn_in(b1, gnr)
    assert be.gn_bwd_fused_ok(rg.view, ry.view, rdy.view)
    be.gn_bwd_fused_gn(rg.view, ry.view, gnt, rs.view, rc.view, rdy.view, pg["dgamma"].view, pg["dbeta"].view,
                       pg["dbias"].view if "dbias" in pg else None)
    torch.cuda.synchronize()
    log.forms.add("gn_bwd_fused_gn" + (":n>2" if n > 2 else "") + ("" if exact else ":sum_y"))
    msgs += out_msgs(rs, fd["sums"].cuda(), "sums")
    pos = rc.changed()
    if pos is not None:
        msgs.append(f"counter: written outside its words: {pos}")
    word = rc.view.view(torch.int32)
    grid = fused_grid(n, math.prod(sp), c, DTYPES[yr.dtype], log.sms)
    if int(word[0]) != grid or bool((word[1:] != 0).any()):
        msgs.append(f"counter words {word.tolist()}: the barrier should leave the grid size {grid} in the first")
    # dy against the two-pass apply on the fused kernel's own sums, at the same layout
    rdy2 = _out(A["dy"])
    two = {k: torch.zeros(c, device="cuda") for k in ("dgamma", "dbeta", "dbias")}
    be.gn_bwd_apply_gn(rg.view, ry.view, gnt, rs.view.clone(), rdy2.view, two["dgamma"], two["dbeta"],
                       two["dbias"] if "dbias" in pg else None)
    torch.cuda.synchronize()
    msgs.append(mismatch(rdy.view, rdy2.view, "dy against gn_bwd_apply_gn on the fused sums"))
    pos = rdy.changed()
    msgs.append(None if pos is None else f"dy: written outside the view: {pos}")
    if exact:
        msgs += check()
    else:
        for k, rb in pg.items():
            msgs.append(mismatch(rb.view, two[k].view(rb.r.sizes), f"{k} against gn_bwd_apply_gn on the fused sums"))
            pos = rb.changed()
            msgs.append(None if pos is None else f"{k}: written outside the view: {pos}")
    msgs += [check_in(ry, "y"), check_in(rg, "g")] + _inputs_unchanged(ins, "gn operand")
    return msgs


def replay_upsample(be, sig, gen, log):
    A = dict(sig.args)
    if sig.op == "upsample_add":
        ar, er, sr = A["a"], A["e"], A["s"]
        a = torch.randint(-8, 9, ar.sizes, generator=gen, device="cuda").double() / 8
        e = torch.randint(-8, 9, er.sizes, generator=gen, device="cuda").double() / 8
        ra, re_, rs = _in(ar, a), _in(er, e), _out(sr)
        be.upsample_add(ra.view, re_.view, rs.view)
        torch.cuda.synchronize()
        log.forms.add(f"upsample_add:{ar.sizes[1:]}")
        return out_msgs(rs, up2_ref(a) + e, "s") + [check_in(ra, "a"), check_in(re_, "e")]
    gsr, gar = A["g_s"], A["g_a"]
    gs = torch.randint(-8, 9, gsr.sizes, generator=gen, device="cuda").double() / 8
    rg, ra = _in(gsr, gs), _out(gar)
    be.upsample_bwd(rg.view, ra.view)
    torch.cuda.synchronize()
    log.forms.add(f"upsample_bwd:{gar.sizes[1:]}")
    return out_msgs(ra, up2t_ref(gs), "g_a") + [check_in(rg, "g_s")]


def replay_head(be, sig, gen, log):
    A = dict(sig.args)
    op = sig.op
    if op in NOT_IN_TRAINING:
        return [f"{op} is the inference form of the head: a training step does not launch it"]
    if op == "head_probs":
        lr, pr = A["logits"], A["probs"]
        z = torch.randint(-64, 65, lr.sizes, generator=gen, device="cuda").double() * QB
        rl, rp = _in(lr, z), _out(pr)
        be.head_probs(rl.view, rp.view)
        torch.cuda.synchronize()
        log.forms.add(op)
        try:
            check_probs(rp.view, z, lr.sizes[-1], "probs")
        except AssertionError as e:
            return [str(e)]
        pos = rp.changed()
        return [None if pos is None else f"probs: written outside the view: {pos}", check_in(rl, "logits")]
    if op in ("head_fwd", "head_bwd"):
        return replay_seg_head(be, op, A, gen, log)
    return replay_cls_head(be, op, A, gen, log)


def replay_seg_head(be, op, A, gen, log):
    xr, wr = A["x"], A["w"]
    nc, cin = wr.sizes[0], xr.sizes[-1]
    nv = math.prod(xr.sizes[:4])
    x = torch.randint(-4, 5, xr.sizes, generator=gen, device="cuda").double() * QX
    w = torch.randint(-8, 9, wr.sizes, generator=gen, device="cuda").double() * QW
    rx, rw = _in(xr, x), _in(wr, w)
    w2 = w.reshape(nc, cin)
    msgs = []
    if op == "head_fwd":
        assert head_fwd_bound(cin) < 2 ** 24
        b = torch.randint(-64, 65, (nc,), generator=gen, device="cuda").double() * QB
        rl, rp, rb = _out(A["logits"]), _out(A["probs"]), _in(A["bias"], b)
        ok = be.head_fwd(rx.view, rw.view, _v(rb), rl.view, _v(rp))
        torch.cuda.synchronize()
        if not ok:
            return ["head_fwd declined a call it took in the recorded step"]
        z = torch.einsum("ndhwk,ck->ndhwc", x, w2) + (b if A["bias"] is not None else 0)
        log.forms.add(f"head_fwd:nc{nc}")
        msgs += out_msgs(rl, z, "logits")
        if rp is not None:
            try:
                check_probs(rp.view, z, nc, "probs")
            except AssertionError as e:
                msgs.append(str(e))
            pos = rp.changed()
            msgs.append(None if pos is None else f"probs: written outside the view: {pos}")
        if rb is not None:
            msgs.append(check_in(rb, "bias"))
    else:
        bw, bb = head_bwd_bound(nv, cin, nc)
        assert bw < 2 ** 24 and bb < 2 ** 24
        dl = torch.randint(-1, 2, A["dlogits"].sizes, generator=gen, device="cuda").double() * QG
        rdl, rdx = _in(A["dlogits"], dl), _out(A["dx"])
        pre_w = torch.randint(-2, 3, A["dw"].sizes, generator=gen, device="cuda").double() / 4
        pre_b = torch.randint(-8, 9, A["db"].sizes, generator=gen, device="cuda").double() * QG
        rdw, rdb = _pgrad(A["dw"], pre_w.float()), _pgrad(A["db"], pre_b.float())
        ok = be.head_bwd(rx.view, rdl.view, rw.view, rdx.view, rdw.view, rdb.view)
        torch.cuda.synchronize()
        if not ok:
            return ["head_bwd declined a call it took in the recorded step"]
        log.forms.add(f"head_bwd:nc{nc}")
        msgs += out_msgs(rdx, torch.einsum("ndhwc,ck->ndhwk", dl, w2) + 0.0, "dx")     # + 0.0: a zero sum is +0
        msgs += out_msgs(rdw, pre_w + torch.einsum("ndhwc,ndhwk->ck", dl, x).reshape(pre_w.shape), "dw (+=)")
        msgs += out_msgs(rdb, pre_b + dl.sum((0, 1, 2, 3)), "db (+=)")
        msgs.append(check_in(rdl, "dlogits"))
    msgs += [check_in(rx, "x"), check_in(rw, "w")]
    return msgs


def cls_blocks(n, vox, c, sms=SMS):
    """the broadcast dx blocks of cls_head_bwd (cls_head.cu:183-185) -> (blocks, capped)"""
    bb = -(-n * vox * c // 256)
    return min(bb, 8 * sms), bb > 8 * sms


def replay_cls_head(be, op, A, gen, log):
    """both cls_head calls of one step run together: the forward's pooled / hidden feed the backward"""
    wrs = {r: A[r] for r in ("w1", "b1", "w2", "b2", "dlogits") if r in A}
    if op == "cls_head_fwd":
        return cls_case(be, A["x"], wrs, {r: A[r] for r in ("pooled", "hidden", "logits")}, None, None, None, gen,
                        log, op)
    # the backward's x (its forward's input, replayed at dx's layout: the forward call checks its own)
    return cls_case(be, A["dx"], wrs, {r: A[r] for r in ("pooled", "hidden")}, A["dx"],
                    {r: A[r] for r in ("dw1", "db1", "dw2", "db2")}, A["work"], gen, log, op)


def cls_case(be, xr, wrs, outs, dxr, gr, workr, gen, log, op):
    """one classifier-head replay: forward at xr's layout (the weights at wrs') and, when dxr is given, the backward
    into dxr / the gradient views gr.  The forward's outputs are checked when its own recorded layouts are given
    (op == cls_head_fwd)."""
    n, c = xr.sizes[0], xr.sizes[-1]
    hd, k = wrs["w1"].sizes[0], wrs["w2"].sizes[0]
    vox = math.prod(xr.sizes[1:4])
    exact = vox & (vox - 1) == 0
    x_alpha, w1, b1, w2, b2, dl = cls_operands(n, c, hd, k, gen)
    x = _draw(x_alpha, xr.sizes, gen)
    rx = _in(xr, x)
    # the backward's own call takes no biases: its forward gets contiguous ones
    rw = {r: _in(wrs[r] if r in wrs else trec(v.float()), v) for r, v in (("w1", w1), ("b1", b1), ("w2", w2),
                                                                         ("b2", b2))}
    msgs = []
    fwd_rec = op == "cls_head_fwd"
    rp, rh = _out(outs["pooled"]), _out(outs["hidden"])
    rl = _out(outs["logits"]) if fwd_rec else None
    logits_t = rl.view if rl is not None else torch.empty((n, k), device="cuda")
    be.cls_head_fwd(rx.view, rw["w1"].view, rw["b1"].view, rw["w2"].view, rw["b2"].view, rp.view, rh.view, logits_t)
    torch.cuda.synchronize()
    S = x.reshape(n, -1, c).sum(1)
    assert float(x.abs().reshape(n, -1, c).sum(1).max()) < 2 ** 24 * QX, "the voxel sum is not exact in fp32"
    pooled = pooled_model(S, vox)
    msgs += out_msgs(rp, pooled, "pooled")
    if exact:
        assert torch.equal(pooled, S / vox)
    # hidden = relu(W1 pooled + b1); logits = W2 hidden + b2 (from the kernel's own pooled / hidden, checked above)
    t1 = w1.unsqueeze(0) * pooled.unsqueeze(1)                         # (n, hd, c)
    h_want, h_tol, h_mag = chain(t1, b1)
    h_want = h_want.clamp_min(0)                                       # |relu(a) - relu(b)| <= |a - b|
    hidden = rh.view.double()
    t2 = w2.unsqueeze(0) * hidden.unsqueeze(1)                         # (n, k, hd)
    checks = [("hidden", rh, h_want, h_tol, h_mag, QW * QX / vox)]
    if fwd_rec:
        checks.append(("logits", rl, *chain(t2, b2), QW * QW * QX / vox))
    if dxr is not None:
        rwork, rdx, rdl = _out(workr), _out(dxr), _in(wrs["dlogits"], dl)
        pg = {kk: Rebuilt(r, IN_FILL).snapshot() for kk, r in gr.items()}     # written: the neighbours stay
        for rb, what in ((rp, "pooled"), (rh, "hidden")):                     # the forward's outputs, now inputs
            pos = rb.changed()
            msgs.append(None if pos is None else f"{what}: written outside the view: {pos}")
            rb.snapshot()
        be.cls_head_bwd(rdl.view, rp.view, rh.view, rw["w1"].view, rw["w2"].view, rwork.view, rdx.view,
                        pg["dw1"].view, pg["db1"].view, pg["dw2"].view, pg["db2"].view)
        torch.cuda.synchronize()
        msgs += [check_in(rp, "pooled"), check_in(rh, "hidden"), check_in(rdl, "dlogits")]
        work = rwork.view.reshape(-1)
        dh_got, dp_got = work[:n * hd].view(n, hd), work[n * hd:].view(n, c)
        dh = torch.where(hidden > 0, dl @ w2 + 0.0, 0.0)                 # exact: grid operands; a zero sum is +0
        dsum = dh @ w1 + 0.0                                              # exact: grid operands
        assert exact_ok((dh.abs() @ w1.abs()), QG * QW * QW), "W1^T dh is not exact in fp32"
        dp = pooled_model(dsum, vox)
        msgs.append(mismatch(dh_got, dh, "dh (work)"))
        msgs.append(mismatch(dp_got, dp, "dp (work)"))
        bc = dp_got.view(n, 1, 1, 1, c).expand(dxr.sizes)
        msgs += out_msgs(rdx, bc.double(), "dx (the dtype of dp from work)")
        t_w1 = dh.t().unsqueeze(1) * pooled.t().unsqueeze(0)               # (hd, c, n)
        t_w2 = dl.t().unsqueeze(1) * hidden.t().unsqueeze(0)               # (k, hd, n)
        checks += [("dw1", pg["dw1"], *chain(t_w1), QG * QW * QX / vox),
                   ("dw2", pg["dw2"], *chain(t_w2), QG * QW * QX / vox)]
        msgs.append(mismatch(pg["db1"].view, dh.sum(0) + 0.0, "db1"))
        msgs.append(mismatch(pg["db2"].view, dl.sum(0) + 0.0, "db2"))
        for kk in ("db1", "db2"):
            pos = pg[kk].changed()
            msgs.append(None if pos is None else f"{kk}: written outside the view: {pos}")
    for what, rb, want, tol, mag, q in checks:
        if exact:
            assert exact_ok(mag, q), f"{what}: the design is not exact"
            msgs += out_msgs(rb, want, what)
        else:
            assert what in CLS_BOUND
            msgs.append(bound_msg(rb.view, want, tol, what))
            pos = rb.changed()
            msgs.append(None if pos is None else f"{what}: written outside the view: {pos}")
    msgs.append(check_in(rx, "x"))
    msgs += [check_in(rb, f"{r} (the weights)") for r, rb in rw.items()]
    log.forms.add(f"{op}:{'exact' if exact else 'bound'}" + (":capped" if dxr is not None and cls_blocks(
        n, vox, c, log.sms)[1] else ""))
    return msgs


def replay_fused_gn_layout(be, sig, gen, log):
    """stem_gn_* / up_gn_*: not replayed here.  test_gpu_fused_gn_exact.py runs them bit for bit at the layouts in its
    LAYOUTS; every output and upstream gradient the networks hand them must be one of those"""
    A = dict(sig.args)
    fam = "stem_gn" if sig.op.startswith("stem_gn") else "up_gn"
    msgs = []
    for role in ("out", "g", "dx"):
        r = A.get(role)
        if r is None:
            continue
        ld, off = pitch(r)
        allowed = {(l, o) for l, o in FUSED_GN_LAYOUTS[f"{fam} {role}"] if o is not None}
        if not any(ld == l and (o is None or off == o) for l, o in FUSED_GN_LAYOUTS[f"{fam} {role}"]):
            msgs.append(f"{role} at (ld, offset) = ({ld}, {off}): test_gpu_fused_gn_exact.py runs {fam} at {allowed}")
        log.forms.add(f"{fam} {role} ({ld}, {off})")
    return msgs


REPLAY = {"gn_fwd": replay_gn_fwd, "gn_bwd": replay_gn_bwd, "upsample": replay_upsample, "head": replay_head,
          "fused_gn": replay_fused_gn_layout}


# ---------------------------------------------------------------------------------------------------------- facts
def _level(sig):
    r = dict(sig.args).get("y")
    return None if r is None else (r.sizes[0], math.prod(r.sizes[1:4]), r.sizes[-1])


def required_facts(family, workload, precision, sigs, sms=SMS):
    """what the replays of a family must include: -> [(description, holds)]"""
    facts = []
    A = [(s, dict(s.args)) for s in sigs]
    if (workload, precision, family) == ("vnet3d_96", "bf16", "fused_gn"):
        for op in ("stem_gn_apply", "stem_gn_bwd", "up_gn_apply", "up_gn_bwd"):
            facts.append((f"a {op} call", any(s.op == op for s in sigs)))
    if (workload, precision, family) == ("vnet3d_96", "bf16", "gn_fwd"):
        facts.append(("an apply_gn writing the left half of a concat (ld = 2C, offset 0)",
                      any(s.op == "apply_gn" and pitch(a["out"]) == (2 * a["out"].sizes[-1], 0) for s, a in A)))
    if (workload, precision, family) == ("vnet3d_96", "bf16", "gn_bwd"):
        facts.append(("a GroupNorm backward whose g is a concat-gradient half",
                      any("g" in a and a["g"] is not None and pitch(a["g"])[0] == 2 * a["g"].sizes[-1] for s, a in A)))
        facts.append(("a gn_bwd_apply_gn with sum_y_from_stats",
                      any(s.op == "gn_bwd_apply_gn" and a["sum_y_from_stats"] for s, a in A)))
    if workload == "resnet2d_64" and family == "gn_bwd":
        fused = [s for s in sigs if s.op == "gn_bwd_fused_gn"]
        facts.append(("a gn_bwd_fused_gn with N = 128", any(_level(s)[0] == 128 for s in fused)))
        big = [s for s in sigs if s.op in ("gn_bwd_reduce_gn", "gn_bwd_apply_gn") and _level(s)[1] == 64 * 64]
        facts.append(("a reduce + apply backward at 64^2 (over the fused limit)",
                      {s.op for s in big} == {"gn_bwd_reduce_gn", "gn_bwd_apply_gn"}))
        at32 = [(s, a) for s, a in A if s.op.startswith("gn_bwd") and "y" in a and _level(s)[1] == 32 * 32]
        ok32 = bool(at32)
        for s, a in at32:
            cs = dict(n=128, sp=a["y"].sizes[1:4], c=a["y"].sizes[-1], dtype=DTYPES[a["y"].dtype],
                      off=pitch(a["y"])[1])
            form = s.op == "gn_bwd_fused_gn"
            from_stats = s.op == "gn_bwd_apply_gn" and a["sum_y_from_stats"]
            if not from_stats and s.op != "gn_bwd_reduce_gn" and form != fused_supported(cs):
                ok32 = False
        facts.append(("every GroupNorm backward at 32^2 (n vox C = 4 << 20) takes the form fused_supported says",
                      ok32))
        if precision == "fp32":
            facts.append(("the fused form at 32^2 in fp32", any(_level(s)[1] == 32 * 32 for s in fused)))
    if workload == "resnet2d_64" and family == "head":
        facts.append(("a cls_head_bwd whose dx block count is capped at 8 SMs",
                      any(s.op == "cls_head_bwd" and cls_blocks(a["dx"].sizes[0], math.prod(a["dx"].sizes[1:4]),
                                                                a["dx"].sizes[-1], sms)[1] for s, a in A)))
    if workload.startswith("unet3dthin") and family == "upsample":
        n, sp = TABLE[workload][2], TABLE[workload][3]
        levels = {tuple(s // 2 ** i for s in sp) for i in range(1, 5)}
        for op, role in (("upsample_add", "a"), ("upsample_bwd", "g_a")):
            got = {a[role].sizes[1:4] for s, a in A if s.op == op}
            facts.append((f"{op} at every level", got == levels))
    return facts


# ---------------------------------------------------------------------------------------------------------- CPU part
_CPU_RECORDINGS = {}


def _cpu_recording(workload):
    if workload not in _CPU_RECORDINGS:
        torch.set_num_threads(max(1, min(8, torch.get_num_threads())))
        from emu_backend import EmuBackend
        _CPU_RECORDINGS[workload] = record(EmuBackend(), workload, "fp32", "cpu", CPU_TABLE)
    return _CPU_RECORDINGS[workload]


def _gn_layers(m, names):
    return [nm[:-len(".weight")] for nm in names if nm.endswith(".weight") and dict(m.named_parameters())[nm].dim() == 1
            and not nm.startswith("fc_layers")]


@pytest.mark.parametrize("workload", sorted(CPU_TABLE))
def test_call_counts_follow_the_layer_program(workload):
    """one GroupNorm backward apply per GroupNorm'd conv layer, i.e. per forward activation branch; the backward of
    every GroupNorm parameter pair, found by its position in the flat gradient bucket; one head forward and backward;
    for UNet3dthin one upsample_add and one upsample_bwd per decoder"""
    calls, names, m = _cpu_recording(workload)
    ops = [c["sig"].op for c in calls]
    args = [dict(c["sig"].args) for c in calls]
    branches = sum(1 + (a["y2"] is not None) for c, a in zip(calls, args) if c["sig"].op == "apply_gn")
    applies = [a for c, a in zip(calls, args) if c["sig"].op == "gn_bwd_apply_gn"]
    assert len(applies) == branches
    # every apply without sums from the forward statistics has its own reduce (the emulated backend has no fused form)
    assert ops.count("gn_bwd_reduce_gn") == sum(not a["sum_y_from_stats"] for a in applies)
    params = dict(m.named_parameters())
    off, o = {}, 0
    for nm in names:
        off[nm] = o
        o += params[nm].numel()
    gn = {off[nm] for nm in names if nm.endswith(".weight") and params[nm].dim() == 1 and not nm.startswith("fc_")}
    assert {a["dgamma"].offset for a in applies} == gn
    assert all(a["dbeta"].offset == a["dgamma"].offset + a["dgamma"].sizes[0] for a in applies)
    assert not {"gn_finalize", "apply", "gn_bwd_reduce", "gn_bwd_apply", "gn_bwd_finalize"} & set(ops)   # C <= 512
    resnet = workload.startswith("resnet")
    assert ops.count("cls_head_fwd") == ops.count("cls_head_bwd") == (1 if resnet else 0)
    assert ops.count("head_fwd") == ops.count("head_bwd") == (0 if resnet else 1)
    assert not NOT_IN_TRAINING & set(ops)
    thin = workload.startswith("unet3dthin")
    assert ops.count("upsample_add") == ops.count("upsample_bwd") == (4 if thin else 0)


def test_skip_halves_arrive_as_concat_views():
    """VNet3d: the up transitions' GroupNorm activations write the left half of their concat, the input block writes
    the skip half at offset C, and the concat convolutions' GroupNorm backward reads a concat-gradient half"""
    calls, _, _ = _cpu_recording("vnet3d_32")
    outs = [pitch(dict(c["sig"].args)["out"]) + (dict(c["sig"].args)["out"].sizes[-1],) for c in calls
            if c["sig"].op == "apply_gn"]
    assert sum(ld == 2 * co and off == 0 for ld, off, co in outs) == 4
    assert sum(ld == 2 * co and off == co for ld, off, co in outs) == 4      # in_tr + the three last down ops
    gs = [dict(c["sig"].args)["g"] for c in calls if c["sig"].op in ("gn_bwd_reduce_gn", "gn_bwd_apply_gn")]
    assert sum(pitch(g)[0] == 2 * g.sizes[-1] for g in gs) >= 4


def test_parameter_gradients_are_views_of_one_bucket():
    calls, names, m = _cpu_recording("vnet3d_32")
    total = sum(p.numel() for p in m.parameters())
    for c in calls:
        if c["sig"].op == "gn_bwd_apply_gn":
            A = dict(c["sig"].args)
            for k in ("dgamma", "dbeta", "dbias"):
                assert A[k].storage == total and A[k].strides == (1,), (k, A[k])
            assert A["dbeta"].offset == A["dgamma"].offset + A["dgamma"].sizes[0]


@pytest.mark.parametrize("workload", sorted(CPU_TABLE))
def test_rebuilt_views_keep_the_recorded_layout(workload):
    calls, _, _ = _cpu_recording(workload)
    seen = set()
    for sig in unique_calls(calls):
        for _, r in sig.args:
            rs = [x for x in (r if isinstance(r, tuple) and hasattr(r, "has_scale") else (r,))]
            for x in rs:
                if not hasattr(x, "sizes") or x in seen or x.dtype not in DTYPES:
                    continue
                seen.add(x)
                rb = Rebuilt(x, fill=IN_FILL, device="cpu")
                assert tuple(rb.view.shape) == x.sizes and tuple(rb.view.stride()) == x.strides
                assert rb.view.storage_offset() == rb.s0 + x.offset and rb.view.data_ptr() % 512 == x.align
    assert seen


def test_upsample_levels_recorded():
    calls, _, _ = _cpu_recording("unet3dthin_32")
    got = {dict(c["sig"].args)["a"].sizes[1:4] for c in calls if c["sig"].op == "upsample_add"}
    assert got == {(16, 16, 16), (8, 8, 8), (4, 4, 4), (2, 2, 2)}


FUSED_N128 = [(128, (1, 32, 32), 32), (128, (1, 16, 16), 64), (128, (1, 8, 8), 128), (128, (1, 4, 4), 256)]


@pytest.mark.parametrize("n,sp,c", FUSED_N128, ids=lambda v: str(v))
@pytest.mark.parametrize("has_scale", [True, False])
def test_fused_design_makes_the_batch_of_128_exact(n, sp, c, has_scale):
    """ResNet2d's fused levels: every per-sample parameter-gradient contribution and every partial sum of them is a
    multiple of one quantum, below 2^24 quanta, so the fp32 atomics are exact in any order"""
    cs = dict(n=n, sp=sp, c=c, dtype=torch.bfloat16, off=0)
    assert fused_supported(cs) == (n * math.prod(sp) * c <= 4 << 20)
    fd = fused_design(n, sp, c, has_scale, "bfloat16")
    assert bool((fd["sums"][..., 2] == 0).all())
    for k, q in fd["quanta"].items():
        assert q < 2 ** 24, (k, q)
    # and the fp32 sum of the rounded per-sample contributions in a shuffled order equals fp64
    for k, t in fd["pc"].items():
        perm = torch.randperm(n, generator=torch.Generator().manual_seed(3))
        acc = fd["pre"][k].float()
        for i in perm.tolist():
            acc = acc + t[i].float()
        assert torch.equal(acc.double(), fd["pre"][k] + t.sum(0)), k


@pytest.mark.parametrize("workload", ["resnet2d_32", "vnet3d_32"])
def test_gn_design_holds_at_recorded_shapes(workload):
    calls, _, _ = _cpu_recording(workload)
    for sig in unique_calls(calls):
        A = dict(sig.args)
        if sig.op in ("apply_gn", "gn_bwd_apply_gn", "gn_bwd_reduce_gn"):
            r = A["y1"] if "y1" in A else A["y"]
            gnr = A["gn1"] if "gn1" in A else A["gn"]
            cs = dict(n=r.sizes[0], sp=r.sizes[1:4], c=r.sizes[-1], dtype=torch.float32, off=0)
            assert check_design(cs, design(cs, drop=gnr.has_scale)) == set()


def test_cls_head_design_is_exact_at_resnet2d():
    """the ResNet2d head at 128 x 4 x 4 x 256 -> 128 -> 10: every sum of the forward and backward is exact"""
    gen = torch.Generator().manual_seed(0)
    n, vox, c, hd, k = 128, 16, 256, 128, 10
    x_alpha, w1, b1, w2, b2, dl = cls_operands(n, c, hd, k, gen)
    x = x_alpha[torch.randint(0, 9, (n, vox, c), generator=gen)]
    p = pooled_model(x.sum(1), vox)
    assert torch.equal(p, x.sum(1) / vox)
    h = (p @ w1.t() + b1).clamp_min(0)
    assert exact_ok(p.abs() @ w1.abs().t() + b1.abs(), QW * QX / vox)
    assert exact_ok(h @ w2.abs().t() + b2.abs(), QW * QW * QX / vox)
    dh = torch.where(h > 0, dl @ w2, 0.0)
    assert exact_ok(dh.abs() @ w1.abs(), QG * QW * QW)
    assert exact_ok(dh.abs().t() @ p.abs(), QG * QW * QX / vox)
    assert exact_ok(dl.abs().t() @ h, QG * QW * QX / vox)
    # fp32 evaluation equals fp64
    hf = torch.relu(p.float() @ w1.float().t() + b1.float())
    assert torch.equal(hf.double(), h)


def test_cls_blocks_cap_at_resnet2d():
    assert cls_blocks(128, 16, 256) == (8 * SMS, True)
    assert not cls_blocks(2, 216, 256)[1]


# the checkers
def _half_rec():
    calls, _, _ = _cpu_recording("vnet3d_32")
    c = next(c for c in calls if c["sig"].op == "apply_gn" and pitch(dict(c["sig"].args)["out"])[1] == 0
             and pitch(dict(c["sig"].args)["out"])[0] == 2 * dict(c["sig"].args)["out"].sizes[-1])
    return dict(c["sig"].args)["out"]._replace(dtype="bfloat16", align=0)


def _want(r):
    g = torch.Generator().manual_seed(9)
    return (Y_ALPHA[torch.randint(0, 9, r.sizes, generator=g)] * 3).float().bfloat16()


def test_checker_reports_one_ulp():
    r = _half_rec()
    rb = Rebuilt(r, device="cpu").snapshot()
    want = _want(r)
    rb.view.copy_(want)
    assert out_msgs(rb, want, "exact") == [None, None]
    rb.view.view(torch.int16)[1, 1, 2, 3, 7] += 1
    assert "(1, 1, 2, 3, 7)" in out_msgs(rb, want, "one ulp")[0]


def test_checker_reports_a_bit_in_the_other_concat_half():
    r = _half_rec()
    rb = Rebuilt(r, device="cpu").snapshot()
    want = _want(r)
    rb.view.copy_(want)
    ld, off = pitch(r)
    assert off == 0 and ld == 2 * r.sizes[-1]
    rb.buf.view(torch.int16)[rb.s0 + r.offset + 5 * ld + r.sizes[-1] + 3] ^= 1     # channel 3 of row 5's skip half
    m = out_msgs(rb, want, "other half")
    assert m[0] is None and "outside the view" in m[1] and "other concat half" in m[1]


def test_checker_reports_a_bit_in_a_neighbouring_parameter_gradient():
    calls, _, _ = _cpu_recording("vnet3d_32")
    A = next(dict(c["sig"].args) for c in calls if c["sig"].op == "gn_bwd_apply_gn")
    r = A["dgamma"]
    pre = torch.arange(r.sizes[0], dtype=torch.float32) / 8
    rb = _pgrad_cpu(r, pre)
    rb.view.add_(1.0)
    assert out_msgs(rb, pre.double() + 1, "dgamma") == [None, None]
    rb.buf.view(torch.int32)[rb.s0 + r.offset + r.sizes[0]] ^= 1            # the first element of d beta
    m = out_msgs(rb, pre.double() + 1, "dgamma")
    assert m[0] is None and "outside the view" in m[1]


def _pgrad_cpu(r, pre):
    return Rebuilt(r, IN_FILL, device="cpu").set(pre.view(r.sizes)).snapshot()


def test_checker_reports_a_read_of_the_other_halfs_in_fill():
    """a kernel that reads the last channel one past its half (channel C: the first of the other half, which holds
    IN_FILL) and every other channel correctly: the one stray read is reported"""
    r = _half_rec()._replace(dtype="float32")
    rin = Rebuilt(r, IN_FILL, device="cpu")
    y = Y_ALPHA[torch.randint(0, 9, r.sizes, generator=torch.Generator().manual_seed(2))] + 2.0      # all positive
    rin.set(y)
    c = r.sizes[-1]
    out = Rebuilt(r, device="cpu").snapshot()
    out.view.copy_(y)
    assert out_msgs(out, y, "exact") == [None, None]
    past = rin.buf.as_strided(r.sizes[:-1], r.strides[:-1], rin.s0 + r.offset + c)     # channel C of every row
    assert bool((past == IN_FILL).all())
    out.view[..., c - 1] = past
    m = out_msgs(out, y, "stray read")[0]
    assert m is not None and f"{c - 1})" in m and f"{math.prod(r.sizes[:-1])} of" in m


def test_checker_reports_a_cls_dx_one_ulp_off_at_one_voxel():
    n, sp, c = 3, (5, 7, 3), 37
    r = trec(torch.empty((n,) + sp + (48,), dtype=torch.bfloat16)[..., :c])
    rb = Rebuilt(r, device="cpu").snapshot()
    dp = torch.randint(-64, 65, (n, c), generator=torch.Generator().manual_seed(4)).float() / 64
    want = dp.view(n, 1, 1, 1, c).expand(r.sizes).double()
    rb.view.copy_(want.to(torch.bfloat16))
    assert out_msgs(rb, want, "dx") == [None, None]
    rb.view.view(torch.int16)[2, 4, 6, 1, 36] += 1
    assert "(2, 4, 6, 1, 36)" in out_msgs(rb, want, "dx")[0]


def test_chain_bound_rejects_one_ulp_beyond_it():
    terms = torch.tensor([[1.0, 2.0 ** -30, -1.0]], dtype=torch.float64)
    want, tol, _ = chain(terms)
    assert bound_msg(want.float() + 0.0, want, tol, "ok") is None
    assert bound_msg(want.float() + 2.0 ** -20, want, tol, "off") is not None


# ---------------------------------------------------------------------------------------------------------- GPU part
@pytest.fixture(scope="module")
def be():
    from pytorchdeeplearing_b200._abi import CudaBackend
    return CudaBackend()


_RECORDINGS = {}


def _recording(be, workload, precision):
    key = (workload, precision)
    if key not in _RECORDINGS:
        calls, _, m = record(be, workload, precision, "cuda")
        del m
        _RECORDINGS[key] = calls
    return _RECORDINGS[key]


GPU_CASES = [(w, p, f) for w in TABLE for p in ("bf16", "fp32") for f in ("gn_fwd", "gn_bwd", "head", "upsample")
             if f != "upsample" or w.startswith("unet3dthin")]
GPU_CASES += [(w, "bf16", "fused_gn") for w in ("vnet3d_96", "vnet3d_128x112", "resnet3d_96")]


@pytest.mark.gpu
@pytest.mark.parametrize("workload,precision,family", GPU_CASES, ids=["-".join(c) for c in GPU_CASES])
def test_network_gn_calls_exact(be, workload, precision, family):
    t0 = time.time()
    calls = _recording(be, workload, precision)
    uniq = {s: tags for s, tags in unique_calls(calls).items() if FAMILY[s.op] == family}
    n_rec = sum(FAMILY[c["sig"].op] == family for c in calls)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    log = Log(f"{workload} {precision}", sms)
    gen = torch.Generator(device="cuda")
    for i, (sig, tags) in enumerate(uniq.items()):
        gen.manual_seed(1000 + i)
        try:
            for m in REPLAY[family](be, sig, gen, log):
                if m is not None:
                    log.fail(sig, tags, m)
        except AssertionError as e:
            log.fail(sig, tags, f"{e}")
        torch.cuda.empty_cache()
    for what, holds in required_facts(family, workload, precision, list(uniq), sms):
        if not holds:
            log.failures.append(f"{log.label} {family}: no replayed call has {what}")
    print(f"\n{workload:18s} {precision:5s} {family:8s} recorded {n_rec:4d} unique {len(uniq):3d} "
          f"forms {','.join(sorted(log.forms)) or '-'} failures {len(log.failures)} ({time.time() - t0:.1f} s)")
    assert not log.failures, "\n".join(log.failures)


CLS_SYNTHETIC = [(3, (5, 7, 3), 37, 19, 1, 40), (1, (1, 1, 1), 1, 1, 1, 1), (128, (1, 4, 4), 256, 128, 10, 256),
                 (2, (6, 6, 6), 256, 128, 4, 264)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("n,sp,c,hd,k,ld", CLS_SYNTHETIC, ids=lambda v: str(v))
def test_cls_head_synthetic_shapes_exact(be, dtype, n, sp, c, hd, k, ld):
    """the odd shapes of test_gpu_resnet.py (C = 37, Hd = 19, K = 1; 1 x 1 x 1) and the two networks' heads, on a
    pitched x and a dx with a pitch gap, under the same exact checks"""
    dt = DTYPES[dtype]
    xr = trec(torch.empty((n,) + sp + (ld,), dtype=dt, device="cuda")[..., :c])
    dxr = trec(torch.empty((n,) + sp + (ld + 8,), dtype=dt, device="cuda")[..., :c])
    bucket = torch.empty(hd * c + hd + k * hd + k + 5, device="cuda")
    o = [2, 2 + hd * c, 2 + hd * c + hd, 2 + hd * c + hd + k * hd]
    gr = {"dw1": trec(bucket[o[0]:o[1]].view(hd, c)), "db1": trec(bucket[o[1]:o[2]]),
          "dw2": trec(bucket[o[2]:o[3]].view(k, hd)), "db2": trec(bucket[o[3]:o[3] + k])}
    params = torch.empty(hd * c + hd + k * hd + k + 5, device="cuda")         # the weights: views of one bucket
    wrs = {"w1": trec(params[o[0]:o[1]].view(hd, c)), "b1": trec(params[o[1]:o[2]]),
           "w2": trec(params[o[2]:o[3]].view(k, hd)), "b2": trec(params[o[3]:o[3] + k]),
           "dlogits": trec(torch.empty((n, k), device="cuda"))}
    small = {kk: trec(torch.empty(s, device="cuda")) for kk, s in (("pooled", (n, c)), ("hidden", (n, hd)),
                                                                   ("logits", (n, k)))}
    log = Log(f"cls {n}x{sp}x{c}", torch.cuda.get_device_properties(0).multi_processor_count)
    gen = torch.Generator(device="cuda").manual_seed(5)
    msgs = cls_case(be, xr, wrs, small, None, None, None, gen, log, "cls_head_fwd")
    msgs += cls_case(be, xr, wrs, small, dxr, gr, trec(torch.empty(n * (hd + c), device="cuda")), gen, log,
                     "cls_head_bwd")
    msgs = [m for m in msgs if m is not None]
    assert not msgs, "\n".join(msgs)
