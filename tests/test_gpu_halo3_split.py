"""conv_halo3_kernel at the VNet shapes and at shapes whose per-CTA ranges of output slice tiles start and end in
the middle of a column and cross from one sample into the next, against the emulated conv (statistics included),
and the fused GroupNorm-backward sums against conv + reduce.  `-m gpu`."""
import pytest
import torch

from emu_backend import EmuBackend, K3

pytestmark = pytest.mark.gpu
EMU = EmuBackend()


@pytest.fixture(scope="module")
def be():
    from pytorchdeeplearing_b200._abi import CudaBackend
    return CudaBackend()


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


CASES = [
    # n, spatial (d, h, w), cin, cout
    (2, (96, 96, 96), 16, 16),      # VNet level 1: 144 columns of 96 slices over the SMs
    (2, (48, 48, 48), 32, 32),      # VNet level 2
    (3, (50, 16, 8), 16, 16),       # one column per sample: most CTA ranges cross a sample boundary
    (2, (45, 20, 12), 32, 16),      # 2 x 2 ragged columns per sample, ranges of 2-3 tiles cross columns and samples
]


@pytest.mark.parametrize("n,sp,cin,cout", CASES)
@pytest.mark.parametrize("which", ["fwd", "dgrad"])
def test_halo3_split_matches_emulation(be, n, sp, cin, cout, which):
    g = torch.Generator().manual_seed(29)
    dt = torch.bfloat16
    w = torch.randn((cout, cin, 3, 3, 3), generator=g) * (2.0 / (cin * 27)) ** 0.5
    ci, co = (cin, cout) if which == "fwd" else (cout, cin)
    bias = torch.randn(co, generator=g) * 0.1
    x = torch.randn((n,) + sp + (ci,), generator=g).to(dt)
    add = torch.randn((n,) + sp + (co,), generator=g).to(dt)
    wp_c = be.pack_weight(w.cuda(), K3, which, dt, 3, vox=10 ** 9)
    assert wp_c.code == 3, "expected the halo layout"
    wp_e = EMU.pack_weight(w, K3, which, dt, 3)
    y_e = torch.zeros((n,) + sp + (co,), dtype=dt)
    st_e = torch.zeros(n, co, 2, dtype=torch.float64)
    EMU.conv(K3, 3, x, wp_e, bias, y_e, st_e, add)
    y_c = torch.zeros((n,) + sp + (co,), dtype=dt, device="cuda")
    st_c = torch.zeros(n, co, 2, dtype=torch.float64, device="cuda")
    be.conv(K3, 3, x.cuda(), wp_c, bias.cuda(), y_c, st_c, add.cuda())
    torch.cuda.synchronize()
    assert rel(y_c, y_e) < 6e-3, rel(y_c, y_e)
    # per sample, so that statistics flushed into the wrong sample show
    for s in range(n):
        assert rel(st_c[s], st_e[s]) < 1e-4, (s, rel(st_c[s], st_e[s]))


@pytest.mark.parametrize("n,sp,cin,cout", [(2, (48, 48, 48), 32, 32), (3, (50, 16, 8), 32, 32)])
def test_halo3_split_bwdstats(be, n, sp, cin, cout):
    g = torch.Generator().manual_seed(31)
    dt = torch.bfloat16
    w = torch.randn((cin, cout, 3, 3, 3), generator=g) * (2.0 / (cin * 27)) ** 0.5
    dy = torch.randn((n,) + sp + (cin,), generator=g).to(dt).cuda()
    wp = be.pack_weight(w.cuda(), K3, "dgrad", dt, 3, vox=10 ** 9)
    assert wp.code == 3
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
