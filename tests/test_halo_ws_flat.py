"""The flattened-padded-row tile geometry of conv_halows_kernel (64/128 input channels, streamed weights).

With P = W + 2, output (h, w) of a plane is anchor q = h * P + w of the zero-padded plane, and a tile is 128
consecutive anchors.  The host picks this geometry over the 8 x 16 column tile where it needs fewer tiles per plane
(conv_halows_geometry in csrc/conv_halo_ws.cu; b200seg_conv_halo_ws_geometry reports it).  The CPU part models the
rule and the work split and checks the model against the library's host query; the GPU part (marked `gpu`) runs the
flat kernels (64 input channels) at the VNet3d 24^3 level and at ragged planes: against the emulated conv, bit for
bit against fp64 on exactly representable operands (with channel-pitch guard bands), with the fused GroupNorm-backward sums, and
under graph replay."""
import ctypes as C

import pytest
import torch

from emu_backend import EmuBackend, K3
from test_gpu_conv_exact import (C as case, GUARD, IN_FILL, Q, Guarded, assert_bitwise, assert_guards, check_stats,
                                 conv_operands, exact_bound, ref_conv, stats_chain, _check_stats_guard, _run_conv)

EMU = EmuBackend()
NT, TW, TH, M = 64, 8, 16, 128
SMS = 132
MAX_POS = 184           # longest flat slice window (positions) the host accepts


# ---------------------------------------------------------------------------------------------------------- model
def geometry(h, w, cin=64):
    """"FLAT" or "COLUMN", as conv_halows_geometry decides: flat at 64 input channels where it needs fewer tiles per
    plane"""
    if cin != 64:
        return "COLUMN"
    col_tiles = -(-h // TH) * -(-w // TW)
    if M + 2 * (w + 2) + 2 > MAX_POS:
        return "COLUMN"
    return "FLAT" if flat_tiles(h, w) < col_tiles else "COLUMN"


def flat_tiles(h, w):
    return -(-((h - 1) * (w + 2) + w) // M)


def flat_units(n, sp, cout):
    d, h, w = sp
    return n * flat_tiles(h, w) * (cout // NT) * d


def flat_grid(units, sms=SMS):
    """CTAs of a flat launch: just enough for the largest share ceil(units / SMs)"""
    g = min(units, sms)
    share = -(-units // g)
    return -(-units // share)


def flat_segments(n, sp, cout, grid, b):
    """the segments (n, tile, g, d0, nd) of CTA b's range, units ordered (n, tile, group, d)"""
    d, h, w = sp
    nt, ng = flat_tiles(h, w), cout // NT
    t = flat_units(n, sp, cout)
    u, end = t * b // grid, t * (b + 1) // grid
    segs = []
    while u < end:
        d0, c = u % d, u // d
        g, c = c % ng, c // ng
        tile, s = c % nt, c // nt
        nd = min(d - d0, end - u)
        segs.append((s, tile, g, d0, nd))
        u += nd
    return segs


def row_output(h, w, q0, r):
    """(h, w) of tile row r, or None for a wrap-around anchor or one past the plane"""
    p = w + 2
    oh, ow = divmod(q0 + r, p)
    return (oh, ow) if oh < h and ow < w else None


# ---------------------------------------------------------------------------------------------------------- CPU part
def test_rule_picks_flat_at_vnet24_and_column_elsewhere():
    assert geometry(24, 24) == "FLAT"                                       # VNet3d 96^3, 64-channel level
    assert geometry(24, 24, cin=128) == "COLUMN"                            # 128 input channels keep the column
    # VNet3d's 12^3: two flat tiles (one of them a lower half) as against two column tiles, the same unit count
    assert flat_tiles(12, 12) == 2 and geometry(12, 12) == "COLUMN"
    assert geometry(32, 32) == "COLUMN" and geometry(16, 16) == "COLUMN"    # UNet3d 128^3: 32^3, 16^3
    assert geometry(16, 8) == "COLUMN"                                      # one column tile, exactly covered
    assert geometry(18, 10) == "FLAT" and geometry(20, 12) == "FLAT" and geometry(10, 20) == "FLAT"
    assert geometry(40, 40) == "COLUMN"                                     # slice window past the budget
    assert flat_tiles(24, 24) == 5                                          # 640 rows instead of 6 x 128


def _ws_desc(n, d, h, w, c):
    return _abi_mod().TensorDesc(0x100000, n, d, h, w, c, c, _abi_mod().BF16)


def _abi_mod():
    from pytorchdeeplearing_b200 import _abi
    return _abi


@pytest.mark.parametrize("hw", [(24, 24), (12, 12), (32, 32), (16, 16), (16, 8), (10, 14), (20, 12), (12, 20),
                                (24, 16), (40, 40), (25, 25), (26, 26), (1, 9), (7, 3)])
@pytest.mark.parametrize("cin", [64, 128])
def test_model_matches_library_query(hw, cin):
    """the library's host query (the value the launch switches on) agrees with the model"""
    _abi = _abi_mod()
    lib = _abi.load_library()
    h, w = hw
    x, y = _ws_desc(2, 6, h, w, cin), _ws_desc(2, 6, h, w, 64)
    rc = lib.b200seg_conv_halo_ws_geometry(K3, 3, C.byref(x), _abi.BF16_HALO_WS, C.byref(y), None)
    assert _abi.HALO_WS_GEOMS[rc] == geometry(h, w, cin)


def test_query_refuses_other_paths():
    _abi = _abi_mod()
    lib = _abi.load_library()
    x, y = _ws_desc(2, 6, 24, 24, 32), _ws_desc(2, 6, 24, 24, 32)      # 32 channels: not this kernel family
    assert lib.b200seg_conv_halo_ws_geometry(K3, 3, C.byref(x), _abi.BF16_HALO, C.byref(y), None) < 0


FLAT_CASES = [
    # n, spatial (d, h, w), cin, cout
    (2, (24, 24, 24), 64, 64),       # VNet 64-channel level: 240 units, two to each of 120 CTAs
    (3, (9, 18, 10), 64, 64),        # 18 x 10 plane: ranges of 2 cross d columns, tiles and samples
    (2, (13, 20, 12), 64, 128),      # 20 x 12 plane: a lower-half last tile; ranges cross groups and samples
    (2, (7, 10, 20), 64, 128),       # 10 x 20 plane, Cout > NT
]


@pytest.mark.parametrize("n,sp,cin,cout", FLAT_CASES)
@pytest.mark.parametrize("sms", [SMS, 7])
def test_flat_split_covers_every_output_once(n, sp, cin, cout, sms):
    """every valid (n, d, h, w, group) is owned by exactly one unit and tile row; wrap-around rows are never valid;
    per-CTA sizes differ by at most one"""
    d, h, w = sp
    assert geometry(h, w, cin) == "FLAT"
    nacc = 2
    units = flat_units(n, sp, cout)
    grid = flat_grid(units, sms)
    seen = set()
    sizes = []
    for b in range(grid):
        segs = flat_segments(n, sp, cout, grid, b)
        sizes.append(sum(s[4] for s in segs))
        for (s, tile, g, d0, nd) in segs:
            assert 1 <= nd and d0 + nd <= d
            items = [min(nacc, nd - o0) for o0 in range(0, nd, nacc)]
            assert sum(items) == nd and all(k == nacc for k in items[:-1])
            for dd in range(d0, d0 + nd):
                for r in range(M):
                    hw = row_output(h, w, tile * M, r)
                    if hw is None:
                        continue
                    assert hw[1] < w                      # a wrap-around anchor (w = W, W + 1) is never stored
                    key = (s, dd, hw[0], hw[1], g)
                    assert key not in seen
                    seen.add(key)
    assert len(seen) == n * d * h * w * (cout // NT)
    assert max(sizes) - min(sizes) <= 1


def test_wrap_around_rows_are_never_valid():
    for h, w in ((24, 24), (18, 10), (20, 12), (10, 20)):
        p = w + 2
        for tile in range(flat_tiles(h, w)):
            for r in range(M):
                q = tile * M + r
                if q % p >= w or q // p >= h:
                    assert row_output(h, w, tile * M, r) is None


@pytest.mark.parametrize("n,sp,cin,cout", FLAT_CASES)
def test_flat_split_keeps_the_statistics_chain_bound(n, sp, cin, cout):
    """no CTA owns more units than the column split would give it, so the HALO_WS statistics bound of
    test_gpu_conv_exact (counted with 8 x 16 tiles) holds"""
    d, h, w = sp
    col = n * d * -(-h // TH) * -(-w // TW) * (cout // NT)
    units = flat_units(n, sp, cout)
    assert -(-units // flat_grid(units)) <= -(-col // min(col, SMS))


def test_vnet24_pairs_are_single_items():
    """at 2 x 24^3 every CTA owns two slices of one column: one NACC = 2 item, one weight stream"""
    units = flat_units(2, (24, 24, 24), 64)
    grid = flat_grid(units)
    assert (units, grid) == (240, 120)
    for b in range(grid):
        segs = flat_segments(2, (24, 24, 24), 64, grid, b)
        assert len(segs) == 1 and segs[0][4] == 2


# ---------------------------------------------------------------------------------------------------------- GPU part
@pytest.fixture(scope="module")
def be():
    from pytorchdeeplearing_b200._abi import CudaBackend
    return CudaBackend()


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


@pytest.mark.gpu
@pytest.mark.parametrize("n,sp,cin,cout", FLAT_CASES)
@pytest.mark.parametrize("which", ["fwd", "dgrad"])
def test_flat_matches_emulation(be, n, sp, cin, cout, which):
    g = torch.Generator().manual_seed(53)
    dt = torch.bfloat16
    # (cin, cout) are the conv's own channels: the data-gradient form runs with the weights of a cout -> cin layer
    shape = (cout, cin) if which == "fwd" else (cin, cout)
    w = torch.randn(shape + (3, 3, 3), generator=g) * (2.0 / (cin * 27)) ** 0.5
    ci, co = cin, cout
    bias = torch.randn(co, generator=g) * 0.1
    x = torch.randn((n,) + sp + (ci,), generator=g).to(dt)
    add = torch.randn((n,) + sp + (co,), generator=g).to(dt)
    wp_c = be.pack_weight(w.cuda(), K3, which, dt, 3, vox=10 ** 9)
    assert wp_c.code == 4
    wp_e = EMU.pack_weight(w, K3, which, dt, 3)
    y_e = torch.zeros((n,) + sp + (co,), dtype=dt)
    st_e = torch.zeros(n, co, 2, dtype=torch.float64)
    EMU.conv(K3, 3, x, wp_e, bias, y_e, st_e, add)
    xc, ac = x.cuda(), add.cuda()
    outs = []
    for _ in range(2):
        y_c = torch.zeros((n,) + sp + (co,), dtype=dt, device="cuda")
        st_c = torch.zeros(n, co, 2, dtype=torch.float64, device="cuda")
        assert be.conv_path(K3, 3, xc, wp_c, y_c, ac) == "HALO_WS"
        assert be.conv_halo_ws_geometry(K3, 3, xc, wp_c, y_c, ac) == "FLAT"
        be.conv(K3, 3, xc, wp_c, bias.cuda(), y_c, st_c, ac)
        torch.cuda.synchronize()
        outs.append((y_c, st_c))
    y_c, st_c = outs[0]
    assert rel(y_c, y_e) < 6e-3, rel(y_c, y_e)
    for s in range(n):
        assert rel(st_c[s], st_e[s]) < 1e-4, (s, rel(st_c[s], st_e[s]))
    assert torch.equal(outs[1][0], y_c)
    assert torch.allclose(outs[1][1], st_c, rtol=1e-12, atol=0.0)


@pytest.mark.gpu
@pytest.mark.parametrize("n,sp,cin,cout", [(2, (24, 24, 24), 64, 64), (3, (9, 18, 10), 64, 64),
                                           (2, (13, 20, 12), 64, 128), (2, (7, 10, 20), 64, 64),
                                           (2, (9, 20, 12), 64, 128)])
def test_flat_bwdstats(be, n, sp, cin, cout):
    """the data gradient with an addend and the fused GroupNorm-backward sums against conv + gn_bwd_reduce_gn"""
    g = torch.Generator().manual_seed(59)
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
    assert be.conv_halo_ws_geometry(K3, 3, dy, wp, g_ref, add) == "FLAT"
    be.conv(K3, 3, dy, wp, None, g_ref, None, add)
    sums_ref = torch.zeros(n, cout, 3, dtype=torch.float64, device="cuda")
    be.gn_bwd_reduce_gn(g_ref, yfwd, gn, sums_ref)
    g_out = torch.empty_like(g_ref)
    sums = torch.zeros(n, cout, 3, dtype=torch.float64, device="cuda")
    assert be.conv_bwdstats_ok(K3, 3, dy, wp, g_out, add, yfwd)
    be.conv_bwdstats(K3, 3, dy, wp, g_out, add, yfwd, gn, sums)
    torch.cuda.synchronize()
    assert torch.equal(g_out, g_ref)
    g_e = torch.zeros((n,) + sp + (cout,), dtype=dt)
    EMU.conv(K3, 3, dy.cpu(), EMU.pack_weight(w, K3, "dgrad", dt, 3), None, g_e, None, add.cpu())
    assert rel(g_out, g_e) < 6e-3, rel(g_out, g_e)
    scale_ = sums_ref[..., 0:2].abs().max(dim=0, keepdim=True).values + 1e-9
    assert ((sums[..., 0:2] - sums_ref[..., 0:2]).abs() / scale_).max() < 2e-5
    assert float(sums[..., 2].abs().max()) == 0.0


EXACT_CASES = {
    "flat_vnet24": case("HALO_WS", K3, "fwd", 3, 2, (24, 24, 24), 64, 64, halo=True),
    "flat_vnet24_dgrad": case("HALO_WS", K3, "dgrad", 3, 2, (24, 24, 24), 64, 64, halo=True),
    "flat_18x10": case("HALO_WS", K3, "fwd", 3, 3, (9, 18, 10), 64, 64, halo=True),
    "flat_20x12": case("HALO_WS", K3, "fwd", 3, 2, (13, 20, 12), 64, 128, halo=True),
    "flat_20x12_dgrad": case("HALO_WS", K3, "dgrad", 3, 2, (13, 20, 12), 128, 64, halo=True),
    "flat_10x20_dgrad": case("HALO_WS", K3, "dgrad", 3, 2, (7, 10, 20), 128, 64, halo=True),
}


@pytest.mark.parametrize("name", sorted(EXACT_CASES))
def test_exact_case_sums_are_exact_in_fp32(name):
    cs = EXACT_CASES[name]
    x, w, bias, addend = conv_operands(cs)
    assert exact_bound(cs, x, w, bias, addend) < 2 ** 20 * Q
    assert geometry(*cs["sp"][1:], 64) == "FLAT" and (cs["cin"] if cs["which"] == "fwd" else cs["cout"]) == 64


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(EXACT_CASES))
def test_flat_exact(be, name):
    """outputs bit for bit against fp64, statistics within the HALO_WS chain bound, guard bands and pitch gaps
    (ld = C + 16) untouched: a stray store of a wrap-around row shows there"""
    cs = EXACT_CASES[name]
    x, w, bias, addend = conv_operands(cs)
    v, y = ref_conv(cs, x, w, bias, addend)
    gy, gx, ga, gs = _run_conv(be, cs, w, x, bias, addend, True)
    wp = be.pack_weight(w.float().cuda(), cs["kind"], cs["which"], torch.bfloat16, 3, vox=10 ** 9)
    assert be.conv_halo_ws_geometry(K3, 3, gx.view, wp, gy.view, ga.view) == "FLAT"
    assert_bitwise(gy.view.cpu(), y.float().bfloat16(), name)
    for gg, what in ((gy, ""), (gx, " input"), (ga, " addend")):
        assert_guards(gg, name + what)
    co = gy.view.shape[-1]
    _check_stats_guard(gs, name)
    chain = stats_chain("HALO_WS", cs["n"], cs["sp"], co)
    check_stats(gs[GUARD:-GUARD].view(cs["n"], co, 2).cpu(), v, chain, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["flat_vnet24_dgrad", "flat_20x12_dgrad", "flat_10x20_dgrad"])
def test_flat_bwdstats_exact(be, name):
    """the bwdstats form on guarded buffers: g bit for bit against fp64, every guard untouched (yfwd and the addend
    are read only at valid rows: their gaps hold a sentinel that would break the sums)"""
    cs = EXACT_CASES[name]
    x, w, _, addend = conv_operands(cs)
    _, gref = ref_conv(cs, x, w, None, addend)
    n, sp, co = cs["n"], cs["sp"], gref.shape[-1]
    gen = torch.Generator().manual_seed(7)
    yfwd = torch.randn((n,) + sp + (co,), generator=gen).bfloat16()
    yf = yfwd.double()
    stats = torch.stack([yf.sum((1, 2, 3)), (yf * yf).sum((1, 2, 3))], -1).contiguous()
    gamma = (1 + 0.2 * torch.randn(co, generator=gen)).float()
    beta = (0.3 * torch.randn(co, generator=gen)).float()
    scale = torch.ones((n, co))
    gx = Guarded((n,) + sp + (x.shape[-1],), torch.bfloat16, fill=IN_FILL, device="cuda")
    gx.view.copy_(x.bfloat16())
    ga = Guarded((n,) + sp + (co,), torch.bfloat16, fill=IN_FILL, device="cuda")
    ga.view.copy_(addend.bfloat16())
    gf = Guarded((n,) + sp + (co,), torch.bfloat16, fill=IN_FILL, device="cuda")
    gf.view.copy_(yfwd)
    gy = Guarded((n,) + sp + (co,), torch.bfloat16, device="cuda")
    wp = be.pack_weight(w.float().cuda(), K3, cs["which"], torch.bfloat16, 3, vox=10 ** 9)
    assert be.conv_halo_ws_geometry(K3, 3, gx.view, wp, gy.view, ga.view) == "FLAT"
    gn = (stats.cuda(), gamma.cuda(), beta.cuda(), scale.cuda(), sp[0] * sp[1] * sp[2], 8, 1e-5)
    sums = torch.zeros(n, co, 3, dtype=torch.float64, device="cuda")
    be.conv_bwdstats(K3, 3, gx.view, wp, gy.view, ga.view, gf.view, gn, sums)
    # the same sums from the separate reduce over the (exact) stored gradient
    sums_ref = torch.zeros(n, co, 3, dtype=torch.float64, device="cuda")
    be.gn_bwd_reduce_gn(gy.view, gf.view, gn, sums_ref)
    torch.cuda.synchronize()
    assert_bitwise(gy.view.cpu(), gref.float().bfloat16(), name)
    for gg, what in ((gy, "g"), (gx, "dy"), (ga, "addend"), (gf, "yfwd")):
        assert_guards(gg, f"{name} {what}")
    assert bool(torch.isfinite(sums).all())
    scale_ = sums_ref[..., 0:2].abs().max(dim=0, keepdim=True).values + 1e-9
    assert ((sums[..., 0:2] - sums_ref[..., 0:2]).abs() / scale_).max() < 2e-5
    assert float(sums[..., 2].abs().max()) == 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("n,sp,cin", [(2, (24, 24, 24), 64), (2, (13, 20, 12), 64)])
def test_flat_graph_replay_matches_eager(be, n, sp, cin):
    g = torch.Generator().manual_seed(61)
    dt = torch.bfloat16
    w = torch.randn((cin, cin, 3, 3, 3), generator=g) * (2.0 / (cin * 27)) ** 0.5
    wp = be.pack_weight(w.cuda(), K3, "fwd", dt, 3, vox=10 ** 9)
    x = torch.randn((n,) + sp + (cin,), generator=g).to(dt).cuda()
    add = torch.randn((n,) + sp + (cin,), generator=g).to(dt).cuda()
    bias = (torch.randn(cin, generator=g) * 0.1).cuda()
    y_e = torch.empty((n,) + sp + (cin,), dtype=dt, device="cuda")
    st_e = torch.zeros(n, cin, 2, dtype=torch.float64, device="cuda")
    assert be.conv_halo_ws_geometry(K3, 3, x, wp, y_e, add) == "FLAT"
    be.conv(K3, 3, x, wp, bias, y_e, st_e, add)
    torch.cuda.synchronize()
    y_g = torch.empty_like(y_e)
    st_g = torch.zeros_like(st_e)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        be.conv(K3, 3, x, wp, bias, y_g, st_g, add)        # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        st_g.zero_()
        be.conv(K3, 3, x, wp, bias, y_g, st_g, add)
    y_g.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(y_g, y_e)
    assert torch.allclose(st_g, st_e, rtol=1e-12, atol=0.0)
