"""conv_halows_kernel (64/128 input channels, streamed weights) at the VNet shapes and at shapes whose per-CTA ranges
of (slice tile, channel group) units start and end in the middle of a column and cross channel groups and samples,
against the emulated conv (statistics per sample), and the fused GroupNorm-backward sums against conv + reduce.
The GPU tests are marked `gpu`; the work-split model at the top runs on the CPU."""
import pytest
import torch

from emu_backend import EmuBackend, K3

EMU = EmuBackend()
NT, TW, TH = 64, 8, 16


def ws_units(n, sp, cout):
    d, h, w = sp
    return n * -(-h // TH) * -(-w // TW) * (cout // NT) * d


def ws_segments(n, sp, cout, grid, b):
    """the column segments (n, ih, iw, g, d0, nd) of CTA b's range, as ws_range / ws_segment walk them"""
    d, h, w = sp
    th, tw, ng = -(-h // TH), -(-w // TW), cout // NT
    t = ws_units(n, sp, cout)
    u, end = t * b // grid, t * (b + 1) // grid
    segs = []
    while u < end:
        d0, c = u % d, u // d
        g, c = c % ng, c // ng
        iw, c = c % tw, c // tw
        ih, s = c % th, c // th
        nd = min(d - d0, end - u)
        segs.append((s, ih, iw, g, d0, nd))
        u += nd
    return segs


SPLIT_CASES = [
    # n, spatial (d, h, w), cin, cout
    (2, (24, 24, 24), 64, 64),       # VNet 64-channel level: 288 units on 132 SMs
    (2, (12, 12, 12), 128, 128),     # VNet 128-channel level: 96 units, two channel groups
    (3, (50, 16, 8), 64, 64),        # one column per sample: ranges of 1-2 slices cross sample boundaries
    (2, (13, 20, 12), 128, 128),     # 2 x 2 ragged columns, ranges cross columns, channel groups and samples
    (2, (10, 20, 12), 64, 128),      # Cout > NT at 64 input channels (dgrad: 128 -> 64)
]


@pytest.mark.parametrize("n,sp,cin,cout", SPLIT_CASES)
@pytest.mark.parametrize("grid", [132, 7])
def test_halo_ws_split_covers_every_unit_once(n, sp, cin, cout, grid):
    """the even split: every output (slice, channel group) belongs to exactly one segment of one CTA, a segment stays
    in one column and channel group, and the items of NACC slices cover each segment"""
    nacc = 2 if cin == 64 else 1
    grid = min(grid, ws_units(n, sp, cout))
    seen = set()
    sizes = []
    for b in range(grid):
        segs = ws_segments(n, sp, cout, grid, b)
        sizes.append(sum(s[5] for s in segs))
        for (s, ih, iw, g, d0, nd) in segs:
            assert 1 <= nd and d0 + nd <= sp[0]
            items = [min(nacc, nd - o0) for o0 in range(0, nd, nacc)]
            assert sum(items) == nd and all(k == nacc for k in items[:-1])
            for dd in range(d0, d0 + nd):
                key = (s, ih, iw, g, dd)
                assert key not in seen
                seen.add(key)
    assert len(seen) == ws_units(n, sp, cout)
    assert max(sizes) - min(sizes) <= 1


@pytest.fixture(scope="module")
def be():
    from pytorchdeeplearing_b200._abi import CudaBackend
    return CudaBackend()


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


@pytest.mark.gpu
@pytest.mark.parametrize("n,sp,cin,cout", SPLIT_CASES)
@pytest.mark.parametrize("which", ["fwd", "dgrad"])
def test_halo_ws_split_matches_emulation(be, n, sp, cin, cout, which):
    g = torch.Generator().manual_seed(37)
    dt = torch.bfloat16
    w = torch.randn((cout, cin, 3, 3, 3), generator=g) * (2.0 / (cin * 27)) ** 0.5
    ci, co = (cin, cout) if which == "fwd" else (cout, cin)
    bias = torch.randn(co, generator=g) * 0.1
    x = torch.randn((n,) + sp + (ci,), generator=g).to(dt)
    add = torch.randn((n,) + sp + (co,), generator=g).to(dt)
    wp_c = be.pack_weight(w.cuda(), K3, which, dt, 3, vox=10 ** 9)
    assert wp_c.code == 4, "expected the grouped weight-streaming layout"
    wp_e = EMU.pack_weight(w, K3, which, dt, 3)
    y_e = torch.zeros((n,) + sp + (co,), dtype=dt)
    st_e = torch.zeros(n, co, 2, dtype=torch.float64)
    EMU.conv(K3, 3, x, wp_e, bias, y_e, st_e, add)
    outs = []
    for _ in range(2):
        y_c = torch.zeros((n,) + sp + (co,), dtype=dt, device="cuda")
        st_c = torch.zeros(n, co, 2, dtype=torch.float64, device="cuda")
        be.conv(K3, 3, x.cuda(), wp_c, bias.cuda(), y_c, st_c, add.cuda())
        torch.cuda.synchronize()
        outs.append((y_c, st_c))
    y_c, st_c = outs[0]
    assert rel(y_c, y_e) < 6e-3, rel(y_c, y_e)
    # per sample, so that statistics flushed into the wrong sample show
    for s in range(n):
        assert rel(st_c[s], st_e[s]) < 1e-4, (s, rel(st_c[s], st_e[s]))
    # a second run gives the same outputs bit for bit; the statistics add per-CTA partials with fp64 atomics
    assert torch.equal(outs[1][0], y_c)
    assert torch.allclose(outs[1][1], st_c, rtol=1e-12, atol=0.0)


@pytest.mark.gpu
@pytest.mark.parametrize("n,sp,cin,cout", [(2, (24, 24, 24), 64, 64), (2, (12, 12, 12), 128, 128),
                                           (3, (50, 16, 8), 64, 64), (2, (13, 20, 12), 128, 128),
                                           (2, (10, 20, 12), 128, 64), (2, (9, 12, 20), 64, 128)])
def test_halo_ws_split_bwdstats(be, n, sp, cin, cout):
    # dgrad weights of a cout -> cin forward layer: this conv maps cin -> cout channels
    g = torch.Generator().manual_seed(41)
    dt = torch.bfloat16
    w = torch.randn((cin, cout, 3, 3, 3), generator=g) * (2.0 / (cin * 27)) ** 0.5
    dy = torch.randn((n,) + sp + (cin,), generator=g).to(dt).cuda()
    wp = be.pack_weight(w.cuda(), K3, "dgrad", dt, 3, vox=10 ** 9)
    assert wp.code == 4
    yfwd = torch.randn((n,) + sp + (cout,), generator=g).to(dt).cuda()
    add = torch.randn((n,) + sp + (cout,), generator=g).to(dt).cuda()
    yf = yfwd.float()
    stats = torch.stack([yf.sum((1, 2, 3)).double(), (yf * yf).sum((1, 2, 3)).double()], -1).contiguous()
    gamma = (1 + 0.2 * torch.randn(cout, generator=g)).cuda()
    beta = (0.3 * torch.randn(cout, generator=g)).cuda()
    scale = (torch.rand((n, cout), generator=g) > 0.2).float().div(0.8).cuda()
    gn = (stats, gamma, beta, scale, sp[0] * sp[1] * sp[2], 8, 1e-5)
    g_ref = torch.empty((n,) + sp + (cout,), dtype=dt, device="cuda")
    be.conv(K3, 3, dy, wp, None, g_ref, None, add)
    sums_ref = torch.zeros(n, cout, 3, dtype=torch.float64, device="cuda")
    be.gn_bwd_reduce_gn(g_ref, yfwd, gn, sums_ref)
    g_out = torch.empty_like(g_ref)
    sums = torch.zeros(n, cout, 3, dtype=torch.float64, device="cuda")
    be.conv_bwdstats(K3, 3, dy, wp, g_out, add, yfwd, gn, sums)
    torch.cuda.synchronize()
    assert torch.equal(g_out, g_ref)
    # the conv itself against the emulation
    g_e = torch.zeros((n,) + sp + (cout,), dtype=dt)
    EMU.conv(K3, 3, dy.cpu(), EMU.pack_weight(w, K3, "dgrad", dt, 3), None, g_e, None, add.cpu())
    assert rel(g_out, g_e) < 6e-3, rel(g_out, g_e)
    scale_ = sums_ref[..., 0:2].abs().max(dim=0, keepdim=True).values + 1e-9
    assert ((sums[..., 0:2] - sums_ref[..., 0:2]).abs() / scale_).max() < 2e-5
    assert float(sums[..., 2].abs().max()) == 0.0
