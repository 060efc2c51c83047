"""wgmma + TMA convolution path (bf16) against the test-only PyTorch statement of the op:
forward and data-gradient forms, 3x3x3 / 3x3 / 1x1, ragged volumes (box overhang), channel-pitched
(concat-slice) inputs and outputs, fused GroupNorm statistics, fused residual addend.  `-m gpu`."""
import pytest
import torch

from emu_backend import EmuBackend, K3, K1, DOWN, UP

pytestmark = pytest.mark.gpu
EMU = EmuBackend()


@pytest.fixture(scope="module")
def be():
    from pytorchdeeplearing_b200._abi import CudaBackend
    b = CudaBackend()
    assert b.use_tc
    return b


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


TC_CASES = [
    # kind, dims, n, spatial, cin, cout
    (K3, 3, 1, (8, 8, 16), 16, 16),
    (K3, 3, 2, (8, 16, 16), 32, 32),
    (K3, 3, 1, (4, 8, 8), 64, 64),
    (K3, 3, 1, (4, 4, 8), 128, 128),
    (K3, 3, 1, (2, 2, 2), 256, 256),      # heavy overhang, 4 k-blocks per tap
    (K3, 3, 2, (6, 6, 6), 64, 32),        # ragged: no box divides the volume
    (K3, 3, 1, (12, 12, 12), 16, 48),
    (K3, 2, 2, (1, 32, 32), 16, 16),
    (K3, 2, 1, (1, 24, 40), 32, 64),
    (K1, 3, 2, (8, 8, 8), 32, 16),
    (K1, 3, 1, (4, 12, 12), 256, 128),
    (K1, 2, 2, (1, 16, 16), 64, 32),
    # >= 65536 voxels: the register-level mma.sync pointwise kernel (pw_mma.cu)
    (K1, 3, 2, (32, 32, 32), 32, 16),
    (K1, 3, 1, (32, 32, 64), 16, 32),
    (K1, 3, 3, (16, 32, 64), 64, 32),     # three samples: statistics flushed per sample
    (K1, 2, 1, (1, 256, 256), 32, 32),
]


@pytest.mark.parametrize("kind,dims,n,sp,cin,cout", TC_CASES)
@pytest.mark.parametrize("which", ["fwd", "dgrad"])
def test_tc_conv_matches_emulation(be, kind, dims, n, sp, cin, cout, which):
    g = torch.Generator().manual_seed(7)
    k = 3 if kind == K3 else 1
    w = torch.randn((cout, cin) + (k,) * dims, generator=g) * (2.0 / (cin * k ** dims)) ** 0.5
    dt = torch.bfloat16
    if which == "fwd":
        ci, co = cin, cout
    else:
        ci, co = cout, cin                 # dgrad: dy (Cout ch) -> dx (Cin ch)
    bias = torch.randn(co, generator=g) * 0.1
    xbuf = (torch.randn((n,) + sp + (ci + 16,), generator=g)).to(dt)
    x = xbuf[..., 8:8 + ci]                # channel-pitched view (concat slice)
    if not be.lib.b200seg_conv_tc_eligible(kind, ci, co):
        pytest.skip("shape not on the wgmma path")
    wp_c = be.pack_weight(w.cuda(), kind, which, dt, dims)
    assert wp_c.code == 2, "expected the wgmma layout"
    wp_e = EMU.pack_weight(w, kind, which, dt, dims)
    for with_stats, with_addend, with_bias in ((True, False, True), (False, True, False)):
        y_e = torch.zeros((n,) + sp + (co,), dtype=dt)
        ybuf = torch.zeros((n,) + sp + (co + 32,), dtype=dt, device="cuda")
        y_c = ybuf[..., 16:16 + co]
        st_e = torch.zeros(n, co, 2, dtype=torch.float64) if with_stats else None
        st_c = st_e.clone().cuda() if with_stats else None
        add = torch.randn((n,) + sp + (co,), generator=g).to(dt) if with_addend else None
        b_ = bias if with_bias else None
        EMU.conv(kind, dims, x, wp_e, b_, y_e, st_e, add)
        be.conv(kind, dims, x.cuda(), wp_c, b_.cuda() if with_bias else None, y_c, st_c,
                add.cuda() if with_addend else None)
        torch.cuda.synchronize()
        assert rel(y_c, y_e) < 6e-3, rel(y_c, y_e)
        assert float(ybuf[..., :16].abs().max()) == 0 and float(ybuf[..., 16 + co:].abs().max()) == 0
        if with_stats:
            assert rel(st_c, st_e) < 1e-4, rel(st_c, st_e)


def test_tc_conv_large_volume_many_tiles(be):
    """more tiles than SMs -> persistent loop, both accumulator stages, stage ring wrap-around"""
    g = torch.Generator().manual_seed(8)
    n, sp, c = 2, (48, 48, 48), 32
    dt = torch.bfloat16
    w = torch.randn((c, c, 3, 3, 3), generator=g) * (2.0 / (c * 27)) ** 0.5
    x = torch.randn((n,) + sp + (c,), generator=g).to(dt)
    wp_c = be.pack_weight(w.cuda(), K3, "fwd", dt, 3)
    wp_e = EMU.pack_weight(w, K3, "fwd", dt, 3)
    y_e = torch.zeros((n,) + sp + (c,), dtype=dt)
    st_e = torch.zeros(n, c, 2, dtype=torch.float64)
    EMU.conv(K3, 3, x, wp_e, None, y_e, st_e, None)
    y_c = torch.zeros((n,) + sp + (c,), dtype=dt, device="cuda")
    st_c = torch.zeros(n, c, 2, dtype=torch.float64, device="cuda")
    be.conv(K3, 3, x.cuda(), wp_c, None, y_c, st_c, None)
    torch.cuda.synchronize()
    assert rel(y_c, y_e) < 6e-3
    assert rel(st_c, st_e) < 1e-4
    # determinism of the statistics path (fixed-order reductions; fp64 atomics differ at 1e-16)
    y2 = torch.zeros_like(y_c)
    be.conv(K3, 3, x.cuda(), wp_c, None, y2, None, None)
    assert torch.equal(y2, y_c)


@pytest.mark.parametrize("kind,n,sp,cin,cout", [
    (K3, 2, (6, 6, 6), 256, 256),         # VNet3d bottom level: 6 voxel tiles, 108 k-blocks -> 6 ranges of 18
    (K3, 1, (3, 5, 7), 256, 256),         # ragged, one sample
    (K3, 2, (12, 12, 12), 128, 64),
    (DOWN, 2, (6, 6, 6), 128, 256),       # 2x2x2 stride 2: 16 k-blocks
    (K3, 3, (4, 4, 4), 64, 256),          # three samples: statistics flushed per sample by the finishing CTAs only
])
def test_tc_conv_split_k_equals_unsplit(be, monkeypatch, kind, n, sp, cin, cout):
    """deep levels cut the (tap, channel-block) loop over several CTAs (conv_tc.cu: ksplit): same result as the
    unsplit kernel up to fp32 summation order (bf16 outputs differ by at most one rounding), independent of
    which range finishes last (bit-identical across launches), counters left clean for the next launch."""
    g = torch.Generator().manual_seed(31)
    dt = torch.bfloat16
    k = 3 if kind == K3 else 2
    w = torch.randn((cout, cin) + (k,) * 3, generator=g) * (2.0 / (cin * k ** 3)) ** 0.5
    isp = sp if kind == K3 else tuple(2 * v for v in sp)
    x = torch.randn((n,) + isp + (cin,), generator=g).to(dt).cuda()
    bias = (torch.randn(cout, generator=g) * 0.1).cuda()
    add = torch.randn((n,) + sp + (cout,), generator=g).to(dt).cuda()
    wp = be.pack_weight(w.cuda(), kind, "fwd", dt, 3)
    assert wp.code == 2

    def run():
        y = torch.zeros((n,) + sp + (cout,), dtype=dt, device="cuda")
        st = torch.zeros(n, cout, 2, dtype=torch.float64, device="cuda")
        be.conv(kind, 3, x, wp, bias, y, st, add)
        torch.cuda.synchronize()
        return y, st

    monkeypatch.setenv("B200SEG_TC_KSPLIT", "0")
    y0, st0 = run()
    monkeypatch.delenv("B200SEG_TC_KSPLIT")
    y1, st1 = run()
    d = (y1.float() - y0.float()).abs()
    assert float((d / (y0.float().abs() + 1e-2)).max()) < 1.0 / 64, "more than one bf16 rounding apart"
    assert rel(y1, y0) < 1e-3 and rel(st1, st0) < 1e-5
    for _ in range(12):                   # back-to-back launches reuse the slabs and the counters
        y2, st2 = run()
        assert torch.equal(y2, y1)
        assert rel(st2, st1) < 1e-12
    monkeypatch.setenv("B200SEG_TC_KSPLIT", "3")
    y3, _ = run()
    assert rel(y3, y0) < 1e-3


WG_CASES = [
    # kind, dims, n, spatial, ka (x channels), kb (dy channels)
    (K3, 3, 1, (8, 8, 16), 16, 16),
    (K3, 3, 2, (8, 16, 16), 32, 32),
    (K3, 3, 1, (8, 8, 8), 64, 64),
    (K3, 3, 1, (4, 4, 8), 128, 128),
    (K3, 3, 1, (2, 4, 4), 256, 256),
    (K3, 3, 2, (6, 6, 6), 32, 16),        # ragged volume; UNet decoder shape 2C -> C
    (K3, 2, 2, (1, 32, 32), 16, 16),
    (K3, 2, 1, (1, 24, 40), 64, 32),
    (K1, 3, 2, (8, 8, 8), 32, 16),
    (K1, 3, 1, (4, 12, 12), 256, 128),
    (K3, 3, 2, (24, 24, 24), 32, 32),     # more voxel tiles than one CTA chunk
    # >= 32768 voxels per sample with 16/32 channels: the halo-tile mma.sync weight gradient (wgrad_halo_mma.cu)
    (K3, 3, 1, (32, 32, 32), 16, 16),     # W % 32 == 0: 32-wide tiles
    (K3, 3, 2, (24, 40, 48), 16, 16),     # 16-wide tiles, several tiles per CTA, two samples
    (K3, 3, 1, (32, 32, 32), 32, 32),     # one (kd, kh) tap row per warp
    (K3, 3, 1, (16, 48, 48), 32, 16),
    (K3, 3, 1, (16, 48, 64), 16, 32),
]


@pytest.mark.parametrize("kind,dims,n,sp,ka,kb", WG_CASES)
def test_tc_wgrad_matches_emulation(be, kind, dims, n, sp, ka, kb):
    g = torch.Generator().manual_seed(9)
    dt = torch.bfloat16
    abuf = torch.randn((n,) + sp + (ka + 16,), generator=g).to(dt)
    a = abuf[..., 8:8 + ka]                    # pitched view
    b = torch.randn((n,) + sp + (kb,), generator=g).to(dt)
    taps = (27 if dims == 3 else 9) if kind == K3 else 1
    dw_e = torch.zeros(taps, ka, kb)
    EMU.wgrad(kind, dims, a, b, dw_e)
    dw_c = torch.zeros(taps, ka, kb, device="cuda")
    be.wgrad(kind, dims, a.cuda(), b.cuda(), dw_c)
    torch.cuda.synchronize()
    assert rel(dw_c, dw_e) < 2e-5, rel(dw_c, dw_e)
    # accumulation semantics (+=)
    be.wgrad(kind, dims, a.cuda(), b.cuda(), dw_c)
    torch.cuda.synchronize()
    assert rel(dw_c, 2 * dw_e) < 2e-5


RESAMPLE_CASES = [
    # kind, dims, n, INPUT spatial, cin, cout
    (DOWN, 3, 2, (8, 16, 16), 16, 32),
    (DOWN, 3, 1, (8, 8, 16), 64, 128),
    (DOWN, 3, 1, (4, 4, 4), 128, 256),
    (DOWN, 3, 2, (12, 12, 12), 32, 64),       # ragged
    (DOWN, 2, 2, (1, 32, 48), 16, 32),
    (UP, 3, 2, (4, 8, 8), 32, 16),
    (UP, 3, 1, (4, 4, 8), 128, 64),           # 8*64 = 512 columns -> 2 column groups
    (UP, 3, 1, (2, 2, 2), 256, 128),          # 4 column groups
    (UP, 3, 2, (6, 6, 6), 64, 32),            # ragged
    (UP, 2, 2, (1, 16, 24), 32, 16),
    (UP, 2, 1, (1, 8, 8), 256, 128),
    # fine volume >= 65536 voxels, Cin*Cout <= 512: the register-level mma.sync transposed conv (pw_mma.cu)
    (UP, 3, 2, (16, 16, 32), 32, 16),
    (UP, 3, 1, (8, 32, 32), 16, 32),
    (UP, 2, 1, (1, 128, 128), 32, 16),
]


def _out_sp(kind, dims, sp):
    if kind == DOWN:
        return (sp[0] // 2 if dims == 3 else 1, sp[1] // 2, sp[2] // 2)
    return (sp[0] * 2 if dims == 3 else 1, sp[1] * 2, sp[2] * 2)


@pytest.mark.parametrize("kind,dims,n,sp,cin,cout", RESAMPLE_CASES)
def test_tc_down_up_forward_dgrad_wgrad(be, kind, dims, n, sp, cin, cout):
    """k2s2 conv / transposed conv on the wgmma path: forward, data gradient (the opposite form) and
    weight gradient (strided TMA gather), all against the emulation."""
    g = torch.Generator().manual_seed(11)
    dt = torch.bfloat16
    kk = (2,) * dims
    wshape = ((cin, cout) if kind == UP else (cout, cin)) + kk
    w = torch.randn(wshape, generator=g) * (2.0 / (cin * 2 ** dims)) ** 0.5
    bias = torch.randn(cout, generator=g) * 0.1
    osp = _out_sp(kind, dims, sp)
    xbuf = torch.randn((n,) + sp + (cin + 16,), generator=g).to(dt)
    x = xbuf[..., 8:8 + cin]
    # ---- forward (+ stats)
    wp_c = be.pack_weight(w.cuda(), kind, "fwd", dt, dims)
    assert wp_c.code == 2
    wp_e = EMU.pack_weight(w, kind, "fwd", dt, dims)
    y_e = torch.zeros((n,) + osp + (cout,), dtype=dt)
    st_e = torch.zeros(n, cout, 2, dtype=torch.float64)
    EMU.conv(kind, dims, x, wp_e, bias, y_e, st_e, None)
    ybuf = torch.zeros((n,) + osp + (cout + 32,), dtype=dt, device="cuda")
    y_c = ybuf[..., 16:16 + cout]
    st_c = torch.zeros(n, cout, 2, dtype=torch.float64, device="cuda")
    be.conv(kind, dims, x.cuda(), wp_c, bias.cuda(), y_c, st_c, None)
    torch.cuda.synchronize()
    assert rel(y_c, y_e) < 6e-3, rel(y_c, y_e)
    assert rel(st_c, st_e) < 1e-4
    assert float(ybuf[..., :16].abs().max()) == 0 and float(ybuf[..., 16 + cout:].abs().max()) == 0
    # ---- data gradient (+ addend)
    dy = torch.randn((n,) + osp + (cout,), generator=g).to(dt)
    add = torch.randn((n,) + sp + (cin,), generator=g).to(dt)
    DK = UP if kind == DOWN else DOWN
    wd_c = be.pack_weight(w.cuda(), kind, "dgrad", dt, dims)
    assert wd_c.code == 2
    wd_e = EMU.pack_weight(w, kind, "dgrad", dt, dims)
    dx_e = torch.zeros((n,) + sp + (cin,), dtype=dt)
    EMU.conv(DK, dims, dy, wd_e, None, dx_e, None, add)
    dx_c = torch.zeros((n,) + sp + (cin,), dtype=dt, device="cuda")
    be.conv(DK, dims, dy.cuda(), wd_c, None, dx_c, None, add.cuda())
    torch.cuda.synchronize()
    assert rel(dx_c, dx_e) < 6e-3, rel(dx_c, dx_e)
    # ---- weight gradient (DOWN-type gather on the fine side)
    taps = 2 ** dims
    fine, coarse = (x, dy) if kind == DOWN else (dy, x)
    dw_e = torch.zeros(taps, fine.shape[-1], coarse.shape[-1])
    EMU.wgrad(DOWN, dims, fine, coarse, dw_e)
    dw_c = torch.zeros(taps, fine.shape[-1], coarse.shape[-1], device="cuda")
    be.wgrad(DOWN, dims, fine.cuda().contiguous(), coarse.cuda().contiguous(), dw_c)
    torch.cuda.synchronize()
    assert rel(dw_c, dw_e) < 2e-5, rel(dw_c, dw_e)


HALO_CASES = [
    # dims, n, spatial, cin, cout
    (3, 1, (6, 32, 16), 16, 16),
    (3, 2, (5, 16, 24), 32, 32),
    (3, 1, (4, 20, 12), 32, 16),          # ragged in h and w (tile overhang), UNet decoder 2C -> C
    (3, 1, (3, 16, 8), 16, 32),
    (2, 2, (1, 32, 32), 16, 16),
    (2, 1, (1, 48, 40), 32, 32),
    (3, 2, (40, 48, 48), 16, 16),         # more items than one CTA pass, d chunking
]


@pytest.mark.parametrize("dims,n,sp,cin,cout", HALO_CASES)
@pytest.mark.parametrize("which", ["fwd", "dgrad"])
def test_halo_conv_matches_emulation(be, dims, n, sp, cin, cout, which):
    g = torch.Generator().manual_seed(13)
    dt = torch.bfloat16
    w = torch.randn((cout, cin) + (3,) * dims, generator=g) * (2.0 / (cin * 3 ** dims)) ** 0.5
    ci, co = (cin, cout) if which == "fwd" else (cout, cin)
    bias = torch.randn(co, generator=g) * 0.1
    xbuf = torch.randn((n,) + sp + (ci + 16,), generator=g).to(dt)
    x = xbuf[..., 8:8 + ci]
    wp_c = be.pack_weight(w.cuda(), K3, which, dt, dims, vox=10 ** 9)
    assert wp_c.code == 3, "expected the halo layout"
    wp_e = EMU.pack_weight(w, K3, which, dt, dims)
    for with_stats, with_addend in ((True, False), (False, True)):
        y_e = torch.zeros((n,) + sp + (co,), dtype=dt)
        ybuf = torch.zeros((n,) + sp + (co + 32,), dtype=dt, device="cuda")
        y_c = ybuf[..., 16:16 + co]
        st_e = torch.zeros(n, co, 2, dtype=torch.float64) if with_stats else None
        st_c = st_e.clone().cuda() if with_stats else None
        add = torch.randn((n,) + sp + (co,), generator=g).to(dt) if with_addend else None
        EMU.conv(K3, dims, x, wp_e, bias, y_e, st_e, add)
        be.conv(K3, dims, x.cuda(), wp_c, bias.cuda(), y_c, st_c, add.cuda() if with_addend else None)
        torch.cuda.synchronize()
        assert rel(y_c, y_e) < 6e-3, rel(y_c, y_e)
        assert float(ybuf[..., :16].abs().max()) == 0 and float(ybuf[..., 16 + co:].abs().max()) == 0
        if with_stats:
            assert rel(st_c, st_e) < 1e-4


HALO_WS_CASES = [
    # n, spatial, cin, cout
    (2, (24, 24, 24), 64, 64),            # the VNet level (6 column tiles, 6 d-chunks of 4, 2 channel groups)
    (1, (6, 16, 8), 64, 64),              # one column, ragged d chunk (6 = 4 + 2)
    (1, (5, 20, 12), 64, 64),             # tile overhang in h and w, one channel group
    (2, (12, 12, 12), 128, 128),          # the 12^3 level: 2-slice items, 4 channel groups
    (1, (3, 8, 8), 128, 64),              # one-slice items
    (1, (7, 16, 16), 64, 128),            # more items than fit one pass per CTA is not needed; 4 groups
]


@pytest.mark.parametrize("n,sp,cin,cout", HALO_WS_CASES)
@pytest.mark.parametrize("which", ["fwd", "dgrad"])
def test_halo_ws_conv_matches_emulation(be, n, sp, cin, cout, which):
    """weight-streaming halo kernel (64/128 input channels) against the emulated conv"""
    g = torch.Generator().manual_seed(17)
    dt = torch.bfloat16
    w = torch.randn((cout, cin, 3, 3, 3), generator=g) * (2.0 / (cin * 27)) ** 0.5
    ci, co = (cin, cout) if which == "fwd" else (cout, cin)
    if ci not in (64, 128):
        pytest.skip("data-gradient form has an input channel count the kernel does not take")
    bias = torch.randn(co, generator=g) * 0.1
    xbuf = torch.randn((n,) + sp + (ci + 16,), generator=g).to(dt)
    x = xbuf[..., 8:8 + ci]
    wp_c = be.pack_weight(w.cuda(), K3, which, dt, 3, vox=10 ** 9)
    assert wp_c.code == 4, "expected the grouped weight-streaming layout"
    wp_e = EMU.pack_weight(w, K3, which, dt, 3)
    many = be.pack_many([(w.cuda(), K3, which, dt, 3, 10 ** 9)])[0]
    torch.cuda.synchronize()
    assert many.code == 4 and torch.equal(many.t, wp_c.t)
    for with_stats, with_addend in ((True, False), (False, True)):
        y_e = torch.zeros((n,) + sp + (co,), dtype=dt)
        ybuf = torch.zeros((n,) + sp + (co + 32,), dtype=dt, device="cuda")
        y_c = ybuf[..., 16:16 + co]
        st_e = torch.zeros(n, co, 2, dtype=torch.float64) if with_stats else None
        st_c = st_e.clone().cuda() if with_stats else None
        add = torch.randn((n,) + sp + (co,), generator=g).to(dt) if with_addend else None
        EMU.conv(K3, 3, x, wp_e, bias, y_e, st_e, add)
        be.conv(K3, 3, x.cuda(), wp_c, bias.cuda(), y_c, st_c, add.cuda() if with_addend else None)
        torch.cuda.synchronize()
        assert rel(y_c, y_e) < 6e-3, rel(y_c, y_e)
        assert float(ybuf[..., :16].abs().max()) == 0 and float(ybuf[..., 16 + co:].abs().max()) == 0
        if with_stats:
            assert rel(st_c, st_e) < 1e-4


@pytest.mark.parametrize("n,sp,cin,cout,with_addend,with_scale", [
    (2, (12, 32, 24), 16, 16, True, True),
    (1, (9, 20, 12), 32, 32, False, False),       # ragged tile, one CTA per SM variant
    (2, (40, 48, 48), 32, 16, True, True),        # more items than CTAs, both samples, ring wrap
    (1, (6, 16, 8), 16, 32, True, False),
    (2, (24, 24, 24), 64, 64, True, True),        # weight-streaming halo kernel (two accumulators per item)
    (2, (12, 12, 12), 128, 128, True, True),      # weight-streaming halo kernel, one 64-column group at a time
    (1, (7, 10, 13), 64, 64, False, False),       # ragged
    (2, (6, 12, 12), 128, 128, False, True),
])
def test_conv_bwdstats_equals_conv_plus_reduce(be, n, sp, cin, cout, with_addend, with_scale):
    """b200seg_conv_bwdstats: the data-gradient conv whose epilogue accumulates the GroupNorm-backward sums of the
    layer behind its output == b200seg_conv followed by b200seg_gn_bwd_reduce_gn (sums [..][0:2]; [2] untouched)."""
    g = torch.Generator().manual_seed(21)
    dt = torch.bfloat16
    w = torch.randn((cin, cout, 3, 3, 3), generator=g) * (2.0 / (cin * 27)) ** 0.5     # conv (Co=cin.. ) dgrad form
    dy = torch.randn((n,) + sp + (cin,), generator=g).to(dt).cuda()                      # gradient of the consumer layer
    wp = be.pack_weight(w.cuda(), K3, "dgrad", dt, 3, vox=10 ** 9)                       # dgrad: cin(out ch of fwd) -> cout
    assert wp.code == (3 if cin <= 32 else 4)
    yfwd = torch.randn((n,) + sp + (cout,), generator=g).to(dt).cuda()                   # raw conv output of the producer
    add = torch.randn((n,) + sp + (cout,), generator=g).to(dt).cuda() if with_addend else None
    yf = yfwd.float()
    stats = torch.stack([yf.sum((1, 2, 3)).double(), (yf * yf).sum((1, 2, 3)).double()], -1).contiguous()
    gamma = (1 + 0.2 * torch.randn(cout, generator=g)).cuda()
    beta = (0.3 * torch.randn(cout, generator=g)).cuda()
    scale = (torch.rand((n, cout), generator=g) > 0.2).float().div(0.8).cuda() if with_scale else None
    vox = sp[0] * sp[1] * sp[2]
    gn = (stats, gamma, beta, scale, vox, 8, 1e-5)
    # reference: two launches
    g_ref = torch.empty((n,) + sp + (cout,), dtype=dt, device="cuda")
    be.conv(K3, 3, dy, wp, None, g_ref, None, add)
    sums_ref = torch.zeros(n, cout, 3, dtype=torch.float64, device="cuda")
    be.gn_bwd_reduce_gn(g_ref, yfwd, gn, sums_ref)
    # fused
    g_out = torch.empty_like(g_ref)
    if cout != 16:
        assert be.conv_bwdstats_ok(K3, 3, dy, wp, g_out, add, yfwd)
    else:   # 16 output channels: the engine does not pick the fused form (measured slower); the kernel must be right
        assert not be.conv_bwdstats_ok(K3, 3, dy, wp, g_out, add, yfwd)
    sums = torch.zeros(n, cout, 3, dtype=torch.float64, device="cuda")
    be.conv_bwdstats(K3, 3, dy, wp, g_out, add, yfwd, gn, sums)
    torch.cuda.synchronize()
    assert torch.equal(g_out, g_ref)
    assert float(sums[..., 2].abs().max()) == 0.0
    scale_ = sums_ref[..., 0:2].abs().max(dim=0, keepdim=True).values + 1e-9
    assert ((sums[..., 0:2] - sums_ref[..., 0:2]).abs() / scale_).max() < 2e-5
    # the apply pass with sum y taken from the forward statistics == the apply pass on the three-sum buffer
    outs = []
    for s_, flag in ((sums_ref, False), (sums, True)):
        dyo = torch.empty_like(g_ref)
        dg, db, dbi = (torch.zeros(cout, device="cuda") for _ in range(3))
        be.gn_bwd_apply_gn(g_out, yfwd, gn, s_, dyo, dg, db, dbi, sum_y_from_stats=flag)
        outs.append((dyo.float(), dg, db, dbi))
    torch.cuda.synchronize()
    assert rel(outs[1][0], outs[0][0]) < 1e-3
    for a, b in zip(outs[1][1:], outs[0][1:]):
        assert (a - b).abs().max() < 2e-4 * (1 + b.abs().max())
