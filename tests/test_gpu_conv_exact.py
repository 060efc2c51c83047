"""Every convolution and weight-gradient kernel against an fp64 reference, bit for bit.

The operands are chosen so that every fp32 sum a kernel can form is exact: x is an integer in [-4, 4] times 2^-2, w an
integer in [-8, 8] times 2^-5, bias and addend integers times 2^-7, so every product and partial sum is a multiple of
q = 2^-7.  Each case asserts, from its actual operands, that sum |terms| < 2^20 q for every output: then every partial
sum in any order is a multiple of q below 2^24 q, exactly representable in fp32, and the kernel's fp32 value cannot
depend on summation order, split-K, tile shape or the tensor-core accumulator.  Its bf16 store must therefore equal
the fp64 reference rounded to nearest even, bit for bit.  Weight gradients use a, b in {-1, 0, 1} * 2^k under the same
kind of precondition.

The reference works from the weights in parameter layout (F.conv3d / F.conv_transpose3d, autograd for the weight
gradient); it does not go through any packing code.  Every input and output is a channel-pitched view inside one
larger allocation: input gaps and guard bands hold a large finite sentinel (reading one with a nonzero weight
destroys exactness), output gaps and guards a NaN bit pattern that must survive the launch.  Each case also asserts
which kernel family the library dispatches it to (CudaBackend.conv_path / wgrad_path).

The CPU part at the top (precondition bounds, path coverage, sensitivity of the checkers) runs without a GPU; the
GPU tests are marked `gpu`."""
import math

import pytest
import torch
import torch.nn.functional as F

from emu_backend import K3, K1, DOWN, UP

Q = 2.0 ** -7
SMS = 132                     # H100 SXM: the grid size of the persistent kernels
GUARD = 64                    # guard elements before and after every buffer
IN_FILL = 2.0 ** 60           # finite input sentinel: any product with a nonzero weight breaks exactness
OUT_BITS = {torch.bfloat16: (torch.int16, 0x7FC1), torch.float32: (torch.int32, 0x7FC00DEF)}   # NaN payloads
CONV_PATHS = ("PW_MMA", "TC", "HALO2D", "HALO3", "HALO_WS", "STEM_MMA", "STEM", "SMALLCIN", "GENERIC")
WGRAD_PATHS = ("HALO_MMA", "TC", "STEM_MMA", "STEM", "SMALLCIN", "GENERIC")
DGRAD_KIND = {K3: K3, K1: K1, DOWN: UP, UP: DOWN}    # kind of the data-gradient conv of a layer of each kind


# ---------------------------------------------------------------------------------------------------------- cases
def C(path, kind, which, dims, n, sp, cin, cout, **kw):
    """one conv case.  (kind, cin, cout) describe the LAYER (weights in parameter layout); which = "dgrad" runs its
    data gradient, so the conv maps cout -> cin channels.  sp is the fine (full-resolution) spatial size.
    flags: halo (pack for the halo kernels), stats, addend, bias, dtype ("bf16" | "f32"), x_f32 (fp32 input),
    x_full (fp32 input with full mantissas, rounded to bf16 by the kernel), x_dense (unpitched input), ksplit,
    bwdstats"""
    d = dict(path=path, kind=kind, which=which, dims=dims, n=n, sp=sp, cin=cin, cout=cout, halo=False, stats=True,
             addend=True, bias=True, dtype="bf16", x_f32=False, x_full=False, x_dense=False, ksplit=None,
             bwdstats=False)
    d.update(kw)
    return d


CONV_CASES = {
    # HALO3: 3-D halo-staged 16/32 channels.  The VNet 96^3 level keeps statistics out: its fp32 chain bound (below)
    # is within 100x of one slice tile's share of a channel sum there, so a statistics error could hide in it.
    "halo3_vnet96": C("HALO3", K3, "fwd", 3, 2, (96, 96, 96), 16, 16, halo=True, stats=False),
    "halo3_vnet96_dgrad": C("HALO3", K3, "dgrad", 3, 2, (96, 96, 96), 16, 16, halo=True, stats=False),
    "halo3_vnet48": C("HALO3", K3, "fwd", 3, 2, (48, 48, 48), 32, 32, halo=True),
    "halo3_vnet48_dgrad": C("HALO3", K3, "dgrad", 3, 2, (48, 48, 48), 32, 32, halo=True),
    "halo3_d1": C("HALO3", K3, "fwd", 3, 2, (1, 40, 24), 16, 32, halo=True),
    "halo3_d2": C("HALO3", K3, "dgrad", 3, 3, (2, 33, 20), 16, 32, halo=True),
    "halo3_ragged_hw": C("HALO3", K3, "fwd", 3, 1, (10, 37, 29), 32, 32, halo=True),
    "halo3_cross_cols_samples": C("HALO3", K3, "fwd", 3, 2, (50, 20, 12), 16, 16, halo=True),
    "halo3_many_samples_per_cta": C("HALO3", K3, "fwd", 3, 500, (1, 16, 8), 16, 16, halo=True),
    "halo3_fewer_tiles_than_sms": C("HALO3", K3, "fwd", 3, 1, (5, 16, 16), 32, 16, halo=True),
    "halo3_sms_plus_one_tiles": C("HALO3", K3, "fwd", 3, 1, (SMS + 1, 16, 8), 16, 16, halo=True),
    "halo3_bwdstats_c16": C("HALO3", K3, "dgrad", 3, 2, (20, 24, 16), 16, 32, halo=True, bwdstats=True),
    "halo3_bwdstats_c32": C("HALO3", K3, "dgrad", 3, 2, (13, 20, 12), 32, 16, halo=True, bwdstats=True),
    # HALO_WS: weight-streaming, 64/128 input channels, Cout 64..256
    "ws_unet16_128_256": C("HALO_WS", K3, "fwd", 3, 2, (16, 16, 16), 128, 256, halo=True),
    "ws_unet16_dgrad_128_256": C("HALO_WS", K3, "dgrad", 3, 2, (16, 16, 16), 256, 128, halo=True),
    "ws_vnet24": C("HALO_WS", K3, "fwd", 3, 2, (24, 24, 24), 64, 64, halo=True),
    "ws_vnet24_dgrad": C("HALO_WS", K3, "dgrad", 3, 2, (24, 24, 24), 64, 64, halo=True),
    "ws_vnet12": C("HALO_WS", K3, "fwd", 3, 2, (12, 12, 12), 128, 128, halo=True),
    "ws_vnet12_dgrad": C("HALO_WS", K3, "dgrad", 3, 2, (12, 12, 12), 128, 128, halo=True),
    "ws_cout192": C("HALO_WS", K3, "fwd", 3, 1, (6, 20, 12), 64, 192, halo=True),
    "ws_d1": C("HALO_WS", K3, "fwd", 3, 2, (1, 24, 16), 128, 64, halo=True),
    "ws_d2": C("HALO_WS", K3, "fwd", 3, 3, (2, 20, 12), 64, 128, halo=True),
    "ws_nacc2_one_short_item": C("HALO_WS", K3, "fwd", 3, 3, (7, 16, 8), 64, 64, halo=True),
    "ws_nacc2_odd_segments": C("HALO_WS", K3, "fwd", 3, 2, (199, 16, 8), 64, 64, halo=True),
    "ws_cross_groups_samples": C("HALO_WS", K3, "fwd", 3, 2, (13, 20, 12), 128, 128, halo=True),
    "ws_cross_groups_256": C("HALO_WS", K3, "fwd", 3, 2, (9, 12, 20), 64, 256, halo=True),
    "ws_bwdstats_64_128": C("HALO_WS", K3, "dgrad", 3, 2, (10, 20, 12), 128, 64, halo=True, bwdstats=True),
    "ws_bwdstats_unet16": C("HALO_WS", K3, "dgrad", 3, 2, (16, 16, 16), 256, 128, halo=True, bwdstats=True),
    # HALO2D: 3x3 halo-staged, ragged H and W
    "halo2d": C("HALO2D", K3, "fwd", 2, 1, (1, 131, 141), 16, 32, halo=True),
    "halo2d_dgrad": C("HALO2D", K3, "dgrad", 2, 2, (1, 130, 129), 16, 32, halo=True),
    # TC: wgmma + TMA implicit GEMM
    "tc_k3": C("TC", K3, "fwd", 3, 2, (6, 6, 6), 64, 32),
    "tc_k3_dgrad": C("TC", K3, "dgrad", 3, 2, (6, 6, 6), 64, 32),
    "tc_k3_2d": C("TC", K3, "fwd", 2, 1, (1, 24, 40), 32, 64),
    "tc_k3_2d_dgrad": C("TC", K3, "dgrad", 2, 1, (1, 24, 40), 32, 64),
    "tc_k1": C("TC", K1, "fwd", 3, 2, (8, 8, 8), 32, 16),
    "tc_k1_dgrad": C("TC", K1, "dgrad", 3, 2, (8, 8, 8), 32, 16),
    "tc_down": C("TC", DOWN, "fwd", 3, 2, (12, 12, 12), 32, 64),
    "tc_down_dgrad": C("TC", DOWN, "dgrad", 3, 2, (12, 12, 12), 32, 64),
    "tc_up": C("TC", UP, "fwd", 3, 2, (12, 12, 12), 64, 32),
    "tc_up_dgrad": C("TC", UP, "dgrad", 3, 2, (12, 12, 12), 64, 32),
    "tc_ragged": C("TC", K3, "fwd", 3, 1, (3, 5, 7), 128, 64),
    "tc_splitk_auto": C("TC", K3, "fwd", 3, 2, (6, 6, 6), 256, 256, ksplit=None),
    "tc_splitk_off": C("TC", K3, "fwd", 3, 2, (6, 6, 6), 256, 256, ksplit="0"),
    "tc_splitk_3": C("TC", K3, "fwd", 3, 2, (6, 6, 6), 256, 256, ksplit="3"),
    "tc_splitk_down": C("TC", DOWN, "fwd", 3, 2, (12, 12, 12), 128, 256),
    # PW_MMA: register-level 1x1x1 / transposed conv at >= 65536 voxels
    "pw_k1": C("PW_MMA", K1, "fwd", 3, 2, (32, 32, 32), 32, 16),
    "pw_k1_three_samples": C("PW_MMA", K1, "fwd", 3, 3, (16, 32, 64), 64, 32),
    "pw_k1_2d_dgrad": C("PW_MMA", K1, "dgrad", 2, 1, (1, 256, 256), 32, 32),
    "pw_up": C("PW_MMA", UP, "fwd", 3, 2, (32, 32, 32), 32, 16),
    # one input channel, small input channel counts, everything else
    "stem_mma_f32_image": C("STEM_MMA", K3, "fwd", 3, 2, (8, 16, 32), 1, 16, x_full=True, x_dense=True,
                            addend=False, stats=False),
    "stem_mma_k1": C("STEM_MMA", K1, "fwd", 3, 2, (4, 16, 32), 1, 32, x_dense=True, addend=False, stats=False),
    "stem_bf16": C("STEM", K3, "fwd", 3, 2, (6, 10, 12), 1, 32, addend=False, stats=False),
    "stem_f32": C("STEM", K3, "fwd", 3, 2, (6, 10, 12), 1, 16, dtype="f32", addend=False, stats=False),
    "smallcin_bf16": C("SMALLCIN", K3, "fwd", 3, 2, (6, 10, 12), 3, 16, addend=False, stats=False),
    "smallcin_k1": C("SMALLCIN", K1, "fwd", 3, 1, (5, 9, 11), 4, 24, addend=False, stats=False),
    "generic_bf16": C("GENERIC", K3, "fwd", 3, 2, (5, 6, 7), 8, 8, stats=False),
    "generic_f32": C("GENERIC", K3, "fwd", 3, 2, (5, 6, 7), 16, 16, dtype="f32", stats=False),
    "generic_up_f32": C("GENERIC", UP, "fwd", 3, 1, (6, 8, 10), 16, 8, dtype="f32", stats=False),
    # an fp32 input to a tensor-core-packed layer: the weights are re-packed for the CUDA-core kernels
    "generic_repack_f32_input": C("GENERIC", K3, "fwd", 3, 1, (4, 6, 8), 16, 16, x_f32=True, addend=False,
                                  stats=False),
}


def W(path, kind, dims, n, sp, ca, cb, **kw):
    """one weight-gradient case: dwp[t][ca][cb] += sum a[n, o*s + t - p, ca] * b[n, o, cb]; sp is b's spatial size.
    flags: a_dtype / b_dtype ("bf16" | "f32"), a_dense (unpitched a)"""
    d = dict(path=path, kind=kind, dims=dims, n=n, sp=sp, ca=ca, cb=cb, a_dtype="bf16", b_dtype="bf16", a_dense=False)
    d.update(kw)
    return d


WGRAD_CASES = {
    "wg_halo_mma": W("HALO_MMA", K3, 3, 2, (8, 64, 64), 16, 32),
    "wg_halo_mma_32": W("HALO_MMA", K3, 3, 1, (8, 64, 64), 32, 16),
    "wg_tc_k3": W("TC", K3, 3, 2, (6, 6, 6), 64, 32),
    "wg_tc_k3_2d": W("TC", K3, 2, 1, (1, 24, 40), 32, 64),
    "wg_tc_k1": W("TC", K1, 3, 2, (8, 8, 8), 32, 16),
    "wg_tc_down": W("TC", DOWN, 3, 2, (6, 6, 6), 32, 64),
    "wg_tc_256": W("TC", K3, 3, 2, (6, 6, 6), 256, 256),
    "wg_stem_mma": W("STEM_MMA", K3, 3, 2, (8, 16, 32), 1, 16, a_dtype="f32", a_dense=True),
    "wg_stem": W("STEM", K3, 3, 2, (6, 10, 12), 1, 32),
    "wg_smallcin": W("SMALLCIN", K3, 3, 2, (6, 10, 12), 3, 16),
    "wg_generic_f32": W("GENERIC", K3, 3, 2, (5, 6, 7), 8, 8, a_dtype="f32", b_dtype="f32"),
}


# ---------------------------------------------------------------------------------------------------------- geometry
def _k(kind, dims):
    if kind == K3:
        return (3, 3, 3) if dims == 3 else (1, 3, 3)
    if kind == K1:
        return (1, 1, 1)
    return (2, 2, 2) if dims == 3 else (1, 2, 2)


def _coarse(sp, dims):
    return (sp[0] // 2 if dims == 3 else sp[0], sp[1] // 2, sp[2] // 2)


def conv_geometry(cs):
    """-> (library kind, x channels, y channels, x spatial, y spatial, weight parameter shape)"""
    kind, dims, sp = cs["kind"], cs["dims"], cs["sp"]
    fine, coarse = sp, (_coarse(sp, dims) if kind in (DOWN, UP) else sp)
    k = _k(kind, dims)[3 - dims:]
    wshape = ((cs["cin"], cs["cout"]) if kind == UP else (cs["cout"], cs["cin"])) + k
    if cs["which"] == "fwd":
        xs, ys = {DOWN: (fine, coarse), UP: (coarse, fine)}.get(kind, (sp, sp))
        return kind, cs["cin"], cs["cout"], xs, ys, wshape
    xs, ys = {DOWN: (coarse, fine), UP: (fine, coarse)}.get(kind, (sp, sp))
    return DGRAD_KIND[kind], cs["cout"], cs["cin"], xs, ys, wshape


def ref_conv(cs, x, w, bias, addend):
    """fp64 reference of the conv a case runs: x (N,D,H,W,C) float64, w in parameter layout.  The data gradient is the
    true gradient of the layer (conv_transpose3d of the forward conv and vice versa).  -> (conv + bias, + addend)"""
    kind, dims = cs["kind"], cs["dims"]
    k = _k(kind, dims)
    w5 = w.reshape(w.shape[:2] + k)
    pad = (k[0] // 2, k[1] // 2, k[2] // 2) if kind == K3 else 0
    stride = k if kind in (DOWN, UP) else 1
    xin = x.permute(0, 4, 1, 2, 3)
    transpose = (kind == UP) == (cs["which"] == "fwd")
    if transpose:
        out = F.conv_transpose3d(xin, w5, None, stride=stride, padding=pad)
    else:
        out = F.conv3d(xin, w5, None, stride=stride, padding=pad)
    out = out.permute(0, 2, 3, 4, 1)
    if bias is not None:
        out = out + bias
    return out, (out + addend if addend is not None else out)


def ref_wgrad(ws, a, b):
    """dwp[t][ca][cb] from autograd of the layer conv y = conv(a, W) with dL/dy = b (parameter layout (cb, ca, k))"""
    kind, dims = ws["kind"], ws["dims"]
    k = _k(kind, dims)
    w0 = torch.zeros((ws["cb"], ws["ca"]) + k, dtype=torch.float64, device=a.device, requires_grad=True)
    pad = (k[0] // 2, k[1] // 2, k[2] // 2) if kind == K3 else 0
    stride = k if kind == DOWN else 1
    with torch.enable_grad():
        y = F.conv3d(a.permute(0, 4, 1, 2, 3), w0, None, stride=stride, padding=pad)
        y.backward(b.permute(0, 4, 1, 2, 3))
    return w0.grad.reshape(ws["cb"], ws["ca"], -1).permute(2, 1, 0).contiguous()


def wgrad_a_spatial(ws):
    sp = ws["sp"]
    if ws["kind"] == DOWN:
        return (sp[0] * 2 if ws["dims"] == 3 else sp[0], sp[1] * 2, sp[2] * 2)
    return sp


# ---------------------------------------------------------------------------------------------------------- operands
def grid(shape, k, e, gen):
    """integers in [-k, k] times 2^-e (bf16-exact for k <= 256), on the generator's device"""
    return torch.randint(-k, k + 1, shape, generator=gen, device=gen.device).double() * 2.0 ** -e


def conv_operands(cs, seed=0):
    g = torch.Generator().manual_seed(seed)
    _, ci, co, xs, ys, wshape = conv_geometry(cs)
    n = cs["n"]
    x = grid((n,) + xs + (ci,), 4, 2, g)
    if cs["x_full"]:
        # an fp32 image with full mantissas, |x| in [1/8, 4]: after RNE to bf16 a multiple of 2^-10
        mag = torch.rand((n,) + xs + (ci,), generator=g, dtype=torch.float64) * (4 - 0.125) + 0.125
        sign = torch.randint(0, 2, mag.shape, generator=g).double() * 2 - 1
        x = (mag * sign).float().double()
    w = grid(wshape, 8, 5, g)
    bias = grid((co,), 16, 7, g) if cs["bias"] else None
    addend = grid((n,) + ys + (co,), 128, 7, g) if cs["addend"] else None
    return x, w, bias, addend


def exact_bound(cs, x, w, bias, addend):
    """max over outputs of sum |terms| (products + bias + addend), on the values the kernel multiplies"""
    xk = x.float().bfloat16().double() if cs["x_full"] else x
    _, s = ref_conv(cs, xk.abs(), w.abs(), None if bias is None else bias.abs(),
                    None if addend is None else addend.abs())
    return float(s.max())


def conv_quantum(cs):
    return 2.0 ** -15 if cs["x_full"] else Q      # bf16(x) for |x| >= 1/8 is a multiple of 2^-10, w of 2^-5


def analytic_bound(cs):
    """a cheap upper bound of exact_bound from the operand ranges alone"""
    _, ci, _, _, _, wshape = conv_geometry(cs)
    taps = math.prod(wshape[2:])
    if cs["kind"] == UP and cs["which"] == "fwd" or cs["kind"] == DOWN and cs["which"] == "dgrad":
        taps = 1                                       # each fine output sees one tap of each coarse input
    return taps * ci * 4.0 * 0.25 + (16 * Q if cs["bias"] else 0) + (128 * Q if cs["addend"] else 0)


def wgrad_operands(ws, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = torch.randint(-1, 2, (ws["n"],) + wgrad_a_spatial(ws) + (ws["ca"],), generator=g).double()
    b = torch.randint(-1, 2, (ws["n"],) + ws["sp"] + (ws["cb"],), generator=g).double() * 0.5
    return a, b


def wgrad_bound(ws):
    """sum |a b| per weight entry is at most the number of output voxels times max |a| max |b|"""
    return ws["n"] * math.prod(ws["sp"]) * 1.0 * 0.5


# ---------------------------------------------------------------------------------------------------------- checkers
def first_mismatch(got, want):
    """None, or a message naming the first (n, d, h, w, c) where the bit patterns of got and want differ"""
    ib = {torch.bfloat16: torch.int16, torch.float32: torch.int32}[want.dtype]
    ne = got.contiguous().view(ib) != want.contiguous().view(ib)
    if not bool(ne.any()):
        return None
    idx = tuple(ne.nonzero()[0].tolist())
    return (f"{int(ne.sum())} of {ne.numel()} elements differ; first at (n, d, h, w, c) = {idx}: "
            f"got {float(got[idx])!r}, want {float(want[idx])!r}")


def assert_bitwise(got, want, what):
    msg = first_mismatch(got, want)
    assert msg is None, f"{what}: {msg}"


def stats_chain(path, n, ys, cout, up=False, kind=K3, dims=3, sms=SMS):
    """L: an upper bound on the number of fp32 additions any value passes through on its way into a [n][c] statistic.
    HALO3 / HALO_WS (conv_halo.cu, conv_halo_ws.cu): a per-thread chain over the slices of one column segment (<= D),
    a 5-level warp butterfly, then one addition into the warp's shared-memory row per segment of the CTA's range
    (<= units per CTA); the four warp rows and the flushes are added in fp64.  TC / PW_MMA (conv_tc.cu, pw_mma.cu):
    a per-tile butterfly, then one addition per tile into the warp's row (<= tiles per sample).  PW_MMA (pw_mma.cu):
    a per-thread chain of 8 additions per tap per 512-voxel tile of the CTA's range (2 CTAs per SM, 1 for UP), a
    3-level butterfly; the eight warp rows are added in fp64.
    GENERIC (conv_generic.cu:186-216): each thread adds the (at most) 4 rows it owns of one output column in fp32
    (s += v, q = fmaf(v, v, q)); the BM/4 row partials of a CTA and the CTAs' atomics are fp64.
    STEM (stem.cu:99-128, grid stem.cu:253-259): a per-thread fp32 chain over its VPT voxels of every item of its
    grid-stride range (grid <= 2 SMs / N CTAs per sample, 256 threads), then a 5-level warp butterfly; the 8 warp
    rows and the atomics are fp64.  SMALLCIN (small_channels.cu:77-103, grid :347-350): the same with one voxel per
    item and a grid of <= 8 SMs / N CTAs per sample.  STEM_MMA (stem_mma.cu:74-99, 146-153, grid stem_mma.cuh:131):
    two fp32 additions per 16-column segment of each 8-row tile of the CTA's range (tiles * segments per sample =
    D H/8 W/16, <= 8 segments per tile, one CTA per tile up to 2 SMs), flushed at each new sample, then a 3-level
    butterfly; the 8 warp rows and the atomics are fp64."""
    d, h, w = ys
    if path in ("HALO3", "HALO_WS"):
        units = n * d * -(-h // 16) * -(-w // 8) * (cout // 64 if path == "HALO_WS" else 1)
        return d + 6 + -(-units // min(units, sms))
    if path == "PW_MMA":
        taps = 8 if up else 1
        tiles = n * d * h * w // taps // 512
        return -(-tiles // min(tiles, sms * (1 if up else 2))) * 8 * taps + 4
    if path == "GENERIC":
        return 4
    if path == "STEM":
        vpt = 2 if (kind == K1 or dims == 2) and w % 2 == 0 else 1
        items = d * h * (w // vpt)
        grid_ = min(-(-items // 256), -(-2 * sms // n))
        return vpt * -(-items // (grid_ * 256)) + 5
    if path == "SMALLCIN":
        v = d * h * w
        grid_ = min(-(-v // 256), -(-8 * sms // n))
        return -(-v // (grid_ * 256)) + 5
    if path == "STEM_MMA":
        segs = n * d * (h // 8) * (w // 16)
        return 2 * (-(-segs // (2 * sms)) + 8) + 3
    return 6 + -(-d * h * w // 64)


def tiles_per_sample(ys):
    d, h, w = ys
    return d * -(-h // 16) * -(-w // 8)


def check_stats(got, v, chain, what):
    """got [N][C][2] against fp64 {sum v, sum v^2} of the exact fp32 values v (N,D,H,W,C), per (n, c), with the
    absolute bound 2^-24 L sum|v| (resp. sum v^2) of an fp32 chain of at most L additions"""
    dims = tuple(range(1, v.dim() - 1))
    want = torch.stack([v.sum(dims), (v * v).sum(dims)], -1)
    tol = torch.stack([v.abs().sum(dims), (v * v).sum(dims)], -1) * (2.0 ** -24 * chain)
    bad = (got.double() - want).abs() > tol
    if bool(bad.any()):
        n, c, k = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: statistic {'sum' if k == 0 else 'sum of squares'} of (n, c) = ({n}, {c}) is "
                             f"{float(got[n, c, k])!r}, fp64 {float(want[n, c, k])!r}, bound {float(tol[n, c, k]):.3g}")


class Guarded:
    """an (N, D, H, W, C) view with channel pitch ld = C + 16 (C at offset `off` <= 16 in each row, 8 by default;
    ld = C with dense=True) in the middle of one allocation with GUARD elements before and after.  Everything outside
    the view holds `fill` (a float) or the NaN bit pattern of the dtype (fill=None)."""

    def __init__(self, shape, dtype, fill=None, device="cpu", dense=False, off=8):
        n, d, h, w, c = shape
        assert 0 <= off <= 16
        self.ld, self.off = (c, 0) if dense else (c + 16, off)
        rows = n * d * h * w
        self.dtype = dtype
        buf = torch.empty(2 * GUARD + rows * self.ld, dtype=dtype)
        if fill is None:
            ib, pat = OUT_BITS[dtype]
            buf.view(ib).fill_(pat)
        else:
            buf.fill_(fill)
        self.buf = buf.to(device)
        self.inside = torch.zeros(buf.numel(), dtype=torch.bool)
        self.inside[GUARD:GUARD + rows * self.ld].view(rows, self.ld)[:, self.off:self.off + c] = True
        self.view = self.buf[GUARD:GUARD + rows * self.ld].view(n, d, h, w, self.ld)[..., self.off:self.off + c]
        self.outside0 = buf[~self.inside].clone()

    def outside_changed(self):
        """None, or the first buffer index outside the view whose bits changed"""
        ib = OUT_BITS[self.dtype][0]
        now = self.buf.cpu()[~self.inside].view(ib)
        ne = now != self.outside0.view(ib)
        if not bool(ne.any()):
            return None
        return int(torch.nonzero(~self.inside)[int(ne.nonzero()[0])])


def assert_guards(g, what):
    pos = g.outside_changed()
    assert pos is None, f"{what}: element {pos} outside the view (guard band or pitch gap) was written"


# ---------------------------------------------------------------------------------------------------------- CPU part
def test_every_kernel_family_has_a_case():
    assert set(c["path"] for c in CONV_CASES.values()) == set(CONV_PATHS)
    assert set(c["path"] for c in WGRAD_CASES.values()) == set(WGRAD_PATHS)


def test_library_path_names_match():
    from pytorchdeeplearing_b200 import _abi
    assert _abi.CONV_PATHS == CONV_PATHS and _abi.WGRAD_PATHS == WGRAD_PATHS


@pytest.mark.parametrize("name", sorted(CONV_CASES))
def test_conv_case_sums_are_exact_in_fp32(name):
    """sum |terms| < 2^20 q for every case, from the operand ranges (the GPU test repeats it on the operands)"""
    cs = CONV_CASES[name]
    assert analytic_bound(cs) < 2 ** 20 * conv_quantum(cs)
    if cs["stats"] or cs["bwdstats"]:
        _, _, co, _, ys, _ = conv_geometry(cs)
        # the statistics bound stays 100x below one slice tile's share of a channel sum
        chain = stats_chain(cs["path"], cs["n"], ys, co, cs["kind"] == UP)
        assert chain * tiles_per_sample(ys) * 2.0 ** -24 * 100 <= 1, name


@pytest.mark.parametrize("name", sorted(WGRAD_CASES))
def test_wgrad_case_sums_are_exact_in_fp32(name):
    # two accumulating calls: the sum of both stays exact
    assert 2 * wgrad_bound(WGRAD_CASES[name]) < 2 ** 24 * 0.5


def test_exact_premise_holds_on_the_cpu():
    """an fp32 conv of grid operands equals the fp64 one, and so do their bf16 roundings"""
    cs = CONV_CASES["ws_vnet12"]
    x, w, bias, addend = conv_operands(cs)
    _, y = ref_conv(cs, x, w, bias, addend)
    _, y32 = ref_conv(cs, x.float(), w.float(), bias.float(), addend.float())
    assert torch.equal(y32.double(), y)
    assert exact_bound(cs, x, w, bias, addend) < 2 ** 20 * Q
    assert_bitwise(y32.bfloat16(), y.float().bfloat16(), "bf16")


def test_checker_rejects_one_ulp():
    g = torch.Generator().manual_seed(3)
    want = grid((2, 3, 4, 5, 16), 200, 4, g).float().bfloat16()
    got = want.clone()
    got.view(torch.int16)[1, 2, 3, 4, 7] += 1
    with pytest.raises(AssertionError, match=r"\(1, 2, 3, 4, 7\)"):
        assert_bitwise(got, want, "one ulp")
    assert_bitwise(want.clone(), want, "equal")


def test_checker_rejects_a_tile_moved_to_the_next_sample():
    g = torch.Generator().manual_seed(4)
    ys = (8, 32, 16)
    v = grid((2,) + ys + (32,), 120, 7, g)
    chain = stats_chain("HALO3", 2, ys, 32)
    assert chain * tiles_per_sample(ys) * 2.0 ** -24 * 100 <= 1
    exact = torch.stack([v.sum((1, 2, 3)), (v * v).sum((1, 2, 3))], -1)
    check_stats(exact.clone(), v, chain, "exact")
    tile = v[0, 5, 16:32, 8:16]                     # one 16 x 8 slice tile of sample 0
    moved = exact.clone()
    moved[0, :, 0] -= tile.sum((0, 1))
    moved[0, :, 1] -= (tile * tile).sum((0, 1))
    moved[1, :, 0] += tile.sum((0, 1))
    moved[1, :, 1] += (tile * tile).sum((0, 1))
    with pytest.raises(AssertionError, match="statistic"):
        check_stats(moved, v, chain, "moved tile")


@pytest.mark.parametrize("where", ["before", "gap", "after"])
def test_checker_rejects_a_rewritten_guard(where):
    gb = Guarded((2, 2, 3, 4, 16), torch.bfloat16)
    gb.view.copy_(torch.ones(2, 2, 3, 4, 16))
    assert gb.outside_changed() is None
    pos = {"before": GUARD - 1, "gap": GUARD + gb.ld + 26, "after": gb.buf.numel() - GUARD}[where]
    assert not bool(gb.inside[pos])
    gb.buf.view(torch.int16)[pos] = 0             # a stray store of zero
    with pytest.raises(AssertionError, match=f"element {pos}"):
        assert_guards(gb, where)


# ---------------------------------------------------------------------------------------------------------- GPU part
@pytest.fixture(scope="module")
def be():
    from pytorchdeeplearing_b200._abi import CudaBackend
    return CudaBackend()


def _dt(s):
    return torch.float32 if s == "f32" else torch.bfloat16


def _run_conv(be, cs, w_packed_from, x, bias, addend, want_stats):
    """launch one conv on guarded buffers -> (y Guarded, x Guarded, stats (cuda) or None, stats Guarded)"""
    lk, ci, co, xs, ys, _ = conv_geometry(cs)
    n, dims = cs["n"], cs["dims"]
    xdt = torch.float32 if (cs["x_f32"] or cs["x_full"] or cs["dtype"] == "f32") else torch.bfloat16
    ydt = _dt(cs["dtype"])
    gx = Guarded((n,) + xs + (ci,), xdt, fill=IN_FILL, device="cuda", dense=cs["x_dense"])
    gx.view.copy_(x.to(xdt))
    ga = None
    if addend is not None:
        ga = Guarded((n,) + ys + (co,), ydt, fill=IN_FILL, device="cuda")
        ga.view.copy_(addend.to(ydt))
    gy = Guarded((n,) + ys + (co,), ydt, device="cuda")
    gs = None
    if want_stats:
        gs = torch.full((2 * GUARD + n * co * 2,), float("nan"), dtype=torch.float64, device="cuda")
        gs[GUARD:GUARD + n * co * 2] = 0
    wp = be.pack_weight(w_packed_from.float().cuda(), cs["kind"], cs["which"], _dt(cs["dtype"]), dims,
                        vox=10 ** 9 if cs["halo"] else None)
    xv, yv, av = gx.view, gy.view, None if ga is None else ga.view
    assert be.conv_path(lk, dims, xv, wp, yv, av) == cs["path"]
    st = None if gs is None else gs[GUARD:GUARD + n * co * 2].view(n, co, 2)
    be.conv(lk, dims, xv, wp, None if bias is None else bias.float().cuda(), yv, st, av)
    torch.cuda.synchronize()
    return gy, gx, ga, gs


def _check_stats_guard(gs, what):
    out = torch.cat([gs[:GUARD], gs[-GUARD:]]).cpu()
    assert bool(out.isnan().all()), f"{what}: statistics guard band written"


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(n for n, c in CONV_CASES.items() if not c["bwdstats"]))
def test_conv_exact(be, monkeypatch, name):
    cs = CONV_CASES[name]
    if cs["ksplit"] is not None:
        monkeypatch.setenv("B200SEG_TC_KSPLIT", cs["ksplit"])
    x, w, bias, addend = conv_operands(cs)
    assert exact_bound(cs, x, w, bias, addend) < 2 ** 20 * conv_quantum(cs)
    xk = x.float().bfloat16().double() if cs["x_full"] else x
    v, y = ref_conv(cs, xk, w, bias, addend)
    want = y.float().to(_dt(cs["dtype"]))
    gy, gx, ga, gs = _run_conv(be, cs, w, x, bias, addend, cs["stats"])
    assert_bitwise(gy.view.cpu(), want, name)
    assert_guards(gy, name)
    assert_guards(gx, name + " input")
    if ga is not None:
        assert_guards(ga, name + " addend")
    if cs["stats"]:
        _, _, co, _, ys, _ = conv_geometry(cs)
        _check_stats_guard(gs, name)
        chain = stats_chain(cs["path"], cs["n"], ys, co, cs["kind"] == UP)
        check_stats(gs[GUARD:-GUARD].view(cs["n"], co, 2).cpu(), v, chain, name)


@pytest.mark.gpu
def test_conv_exact_sees_swapped_taps(be):
    """the exact comparison reports weights packed with two taps exchanged (a wrong result, not a fault)"""
    cs = CONV_CASES["ws_vnet12"]
    x, w, bias, addend = conv_operands(cs)
    _, y = ref_conv(cs, x, w, bias, addend)
    ws = w.clone()
    ws[:, :, 0, 0, 0], ws[:, :, 2, 2, 2] = w[:, :, 2, 2, 2], w[:, :, 0, 0, 0]
    gy, *_ = _run_conv(be, cs, ws, x, bias, addend, False)
    assert first_mismatch(gy.view.cpu(), y.float().bfloat16()) is not None


def bwdstats_want(g_bf, yf, stats, gamma, beta, scale, groups, eps, chain):
    """fp64 {sum g m, sum g m yfwd} per (n, c) and their bounds (s0, t0, s1, t1).  m is the ReLU mask from A, B derived
    in fp64 as the kernels' load_coefs does (group mean / rstd from the statistics, rounded to fp32); scale None is
    no dropout.  The bound is an fp32 chain of at most `chain` additions plus every term whose z is within 2^-20 of
    the threshold (there the fp32 fmaf may take either side)."""
    n, co = yf.shape[0], yf.shape[-1]
    vox = yf[0, ..., 0].numel()
    cpg = co // groups
    st = stats.view(n, groups, cpg, 2).sum(2)
    m_ = float(cpg * vox)
    mean = st[..., 0] / m_
    var = (st[..., 1] / m_ - mean * mean).clamp_min(0)
    rstd = 1.0 / torch.sqrt(var + eps)
    mean_c, rstd_c = mean.repeat_interleave(cpg, 1), rstd.repeat_interleave(cpg, 1)
    s = 1.0 if scale is None else scale.double()
    A = (rstd_c * gamma.double() * s).float().double().view(n, 1, 1, 1, co)
    B = ((beta.double() - mean_c * rstd_c * gamma.double()) * s).float().double().view(n, 1, 1, 1, co)
    z = yf * A + B
    amb = z.abs() <= 2.0 ** -20 * ((yf * A).abs() + B.abs())
    m = (z > 0).double()
    gd = g_bf.double()
    s0, s1 = (gd * m).sum((1, 2, 3)), (gd * m * yf).sum((1, 2, 3))
    t0 = 2.0 ** -24 * chain * gd.abs().sum((1, 2, 3)) + (gd.abs() * amb).sum((1, 2, 3))
    t1 = 2.0 ** -24 * chain * (gd * yf).abs().sum((1, 2, 3)) + ((gd * yf).abs() * amb).sum((1, 2, 3))
    return s0, t0, s1, t1


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(n for n, c in CONV_CASES.items() if c["bwdstats"]))
def test_conv_bwdstats_exact(be, name):
    """g = conv(dy) + addend bit for bit, and sums[n][c] = {sum g m, sum g m yfwd} against fp64 (m the ReLU mask from
    A, B derived in fp64 as the kernels' load_coefs does); sums[..., 2] untouched"""
    cs = CONV_CASES[name]
    lk, ci, co, xs, ys, _ = conv_geometry(cs)
    n = cs["n"]
    x, w, _, addend = conv_operands(cs)
    assert exact_bound(cs, x, w, None, addend) < 2 ** 20 * Q
    _, gref = ref_conv(cs, x, w, None, addend)
    g_bf = gref.float().bfloat16()
    gen = torch.Generator().manual_seed(5)
    yfwd = torch.randn((n,) + ys + (co,), generator=gen).bfloat16()
    yf = yfwd.double()
    stats = torch.stack([yf.sum((1, 2, 3)), (yf * yf).sum((1, 2, 3))], -1).contiguous()
    gamma = (1 + 0.2 * torch.randn(co, generator=gen)).float()
    beta = (0.3 * torch.randn(co, generator=gen)).float()
    scale = ((torch.rand((n, co), generator=gen) > 0.2).float() / 0.8).float()
    groups, eps, vox = 8, 1e-5, math.prod(ys)
    chain = stats_chain(cs["path"], n, ys, co)
    s0, t0, s1, t1 = bwdstats_want(g_bf, yf, stats, gamma, beta, scale, groups, eps, chain)

    gx = Guarded((n,) + xs + (ci,), torch.bfloat16, fill=IN_FILL, device="cuda")
    gx.view.copy_(x.bfloat16())
    ga = Guarded((n,) + ys + (co,), torch.bfloat16, fill=IN_FILL, device="cuda")
    ga.view.copy_(addend.bfloat16())
    gf = Guarded((n,) + ys + (co,), torch.bfloat16, fill=IN_FILL, device="cuda")
    gf.view.copy_(yfwd)
    gy = Guarded((n,) + ys + (co,), torch.bfloat16, device="cuda")
    wp = be.pack_weight(w.float().cuda(), cs["kind"], "dgrad", torch.bfloat16, 3, vox=10 ** 9)
    assert be.conv_path(lk, 3, gx.view, wp, gy.view, ga.view) == cs["path"]
    gn = (stats.cuda(), gamma.cuda(), beta.cuda(), scale.cuda(), vox, groups, eps)
    sums = torch.zeros(n, co, 3, dtype=torch.float64, device="cuda")
    assert be.conv_bwdstats_ok(lk, 3, gx.view, wp, gy.view, ga.view, gf.view) or co == 16
    be.conv_bwdstats(lk, 3, gx.view, wp, gy.view, ga.view, gf.view, gn, sums)
    gplain = Guarded((n,) + ys + (co,), torch.bfloat16, device="cuda")
    be.conv(lk, 3, gx.view, wp, None, gplain.view, None, ga.view)
    torch.cuda.synchronize()
    assert_bitwise(gy.view.cpu(), g_bf, name)
    assert_bitwise(gplain.view.cpu(), g_bf, name + " plain conv")
    for gg, what in ((gy, "g"), (gx, "dy"), (ga, "addend"), (gf, "yfwd"), (gplain, "plain g")):
        assert_guards(gg, f"{name} {what}")
    sums = sums.cpu()
    assert float(sums[..., 2].abs().max()) == 0.0
    for k, (want, tol) in enumerate(((s0, t0), (s1, t1))):
        bad = (sums[..., k] - want).abs() > tol
        if bool(bad.any()):
            nn_, c = bad.nonzero()[0].tolist()
            raise AssertionError(f"{name}: sums[{nn_}][{c}][{k}] = {float(sums[nn_, c, k])!r}, fp64 "
                                 f"{float(want[nn_, c])!r}, bound {float(tol[nn_, c]):.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(WGRAD_CASES))
def test_wgrad_exact(be, name):
    ws = WGRAD_CASES[name]
    a, b = wgrad_operands(ws)
    bound = ref_wgrad(ws, a.abs(), b.abs())
    assert 2 * float(bound.max()) < 2 ** 24 * 0.5
    want = ref_wgrad(ws, a, b).float()
    adt, bdt = _dt(ws["a_dtype"]), _dt(ws["b_dtype"])
    ga = Guarded(a.shape, adt, fill=IN_FILL, device="cuda", dense=ws["a_dense"])
    ga.view.copy_(a.to(adt))
    gb = Guarded(b.shape, bdt, fill=IN_FILL, device="cuda")
    gb.view.copy_(b.to(bdt))
    T = want.shape[0]
    buf = torch.full((2 * GUARD + want.numel(),), float("nan"), device="cuda")
    buf[GUARD:-GUARD] = 0
    dwp = buf[GUARD:-GUARD].view(want.shape)
    assert be.wgrad_path(ws["kind"], ws["dims"], ga.view, gb.view) == ws["path"]
    be.wgrad(ws["kind"], ws["dims"], ga.view, gb.view, dwp)
    torch.cuda.synchronize()
    assert T == math.prod(_k(ws["kind"], ws["dims"]))
    assert_bitwise(dwp.cpu().view(T, ws["ca"], ws["cb"], 1, 1), want.view(T, ws["ca"], ws["cb"], 1, 1), name)
    be.wgrad(ws["kind"], ws["dims"], ga.view, gb.view, dwp)      # accumulates
    torch.cuda.synchronize()
    assert_bitwise(dwp.cpu().view(T, ws["ca"], ws["cb"], 1, 1), (2 * want).view(T, ws["ca"], ws["cb"], 1, 1),
                   name + " (second call)")
    assert bool(torch.cat([buf[:GUARD], buf[-GUARD:]]).isnan().all()), f"{name}: dwp guard band written"
    assert_guards(ga, name + " a")
    assert_guards(gb, name + " b")
