"""Seg_Metirc3d / seg_metrics3d on the GPU (b200seg_segmetric3d, csrc/segmetric.cu): every fixture of the real
reference class (tests/golden/segmetric.npz), large cases against the fp64 scipy oracle (oracle/segmetric.py), NaN
guard bands around every output, run-to-run bit identity, CUDA-graph capture and predict_mask output as input."""
import numpy as np
import pytest
import torch

from oracle import segmetric as osm
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import runtime
from test_segmetric_cpu import GOLD, OK_CASES, masks, close, check_against_fixture

pytestmark = pytest.mark.gpu
GUARD = 64          # guard bytes before and after every output


def ellipsoid(shape, centre, radii):
    z, y, x = np.ogrid[tuple(slice(0, s) for s in shape)]
    return (((z - centre[0]) / radii[0]) ** 2 + ((y - centre[1]) / radii[1]) ** 2 +
            ((x - centre[2]) / radii[2]) ** 2) <= 1.0


def check_oracle(metrics, counts, r, p, sp):
    want, cnt = osm.seg_metrics(r, p, sp)
    assert counts.tolist() == list(cnt)
    got = metrics.cpu().numpy()
    assert got[:6].tobytes() == want[:6].tobytes(), (got[:6], want[:6])
    assert close(got[6:], want[6:]), (got[6:], want[6:])


# ------------------------------------------------------------------------------------------------ fixtures
@pytest.mark.parametrize("case", OK_CASES)
def test_class_matches_the_reference_fixture(case):
    r, p, sp = masks(case)
    m = b200.Seg_Metirc3d(r, p, sp)
    dice = m.get_dice_coefficient()
    vals = [dice[0], m.get_jaccard_index(), m.get_VOE(), m.get_RVD(), m.get_FNR(), m.get_FPR(), m.get_ASSD(),
            m.get_RMSD(), m.get_MSD()]
    assert [type(v) for v in vals] == [np.float64] * 3 + [float] + [np.float64] * 3 + [float, np.float64]
    assert type(dice[1]) is np.int64 and type(dice[2]) is np.int64
    check_against_fixture(case, vals, dice[1:], (len(m.real2pred_nn), len(m.pred2real_nn)),
                          (m.real_mask_surface_pts, m.pred_mask_surface_pts, m.real2pred_nn, m.pred2real_nn))
    if case == "dtype_uint8":       # documented divergence: the signed RVD, equal to the bool case's
        assert np.float64(m.get_RVD()).tobytes() == GOLD["dtype_bool_metrics"][3].tobytes()


def test_class_raises_on_the_empty_fixture_and_on_0_255_masks():
    r, p, sp = masks("empty")
    with pytest.raises(ValueError, match="empty"):
        b200.Seg_Metirc3d(r, p, sp)
    r, p, sp = masks("dtype_uint8")
    with pytest.raises(ValueError, match="binarise"):
        b200.Seg_Metirc3d(r, p * 255, sp)
    with pytest.raises(ValueError, match="binarise"):
        b200.Seg_Metirc3d(torch.from_numpy(r.astype(np.int32) * 2).cuda(), p, sp)


@pytest.mark.parametrize("dtype", [torch.bool, torch.uint8, torch.int32, torch.int64])
def test_every_mask_dtype_gives_the_same_bits(dtype):
    r, p, sp = masks("odd_extents")
    m, c = b200.seg_metrics3d(torch.from_numpy(r).to("cuda", dtype), torch.from_numpy(p).to("cuda", dtype), sp)
    m0, c0 = b200.seg_metrics3d(torch.from_numpy(r).cuda(), torch.from_numpy(p).cuda(), sp)
    assert torch.equal(c, c0) and m.cpu().numpy().tobytes() == m0.cpu().numpy().tobytes()
    check_against_fixture("odd_extents", m.cpu().numpy(), (2 * c[2].item(), c[0].item() + c[1].item()),
                          (c[4].item(), c[5].item()))


# ------------------------------------------------------------------------------------------------ large cases
@pytest.fixture(scope="module")
def ct_case():
    sh = (88, 410, 512)
    r = ellipsoid(sh, (44, 200, 250), (30, 150, 190))
    p = ellipsoid(sh, (47, 210, 262), (28, 140, 200))
    return r, p, (0.78, 0.78, 2.5)


def test_ct_sized_case_against_the_oracle_with_points(ct_case):
    r, p, sp = ct_case
    m = b200.Seg_Metirc3d(r, p, sp)
    want, cnt = osm.seg_metrics(r, p, sp)
    got = np.array([m.get_dice_coefficient()[0], m.get_jaccard_index(), m.get_VOE(), m.get_RVD(), m.get_FNR(),
                    m.get_FPR(), m.get_ASSD(), m.get_RMSD(), m.get_MSD()])
    assert got[:6].tobytes() == want[:6].tobytes()
    assert close(got[6:], want[6:]), (got[6:], want[6:])
    ri, pi, r2p, p2r = osm.surface_distances(r, p, sp)
    spz = np.array(sp[::-1]).reshape(1, 3)
    assert len(ri) > 100000
    assert np.array_equal(m.real_mask_surface_pts, ri * spz) and np.array_equal(m.pred_mask_surface_pts, pi * spz)
    assert close(m.real2pred_nn, r2p) and close(m.pred2real_nn, p2r)


def test_batch_of_two_with_a_spacing_per_volume():
    rng = np.random.RandomState(3)
    sh = (96, 96, 96)
    r = np.stack([ellipsoid(sh, (48, 45, 50), (30, 35, 25)), rng.rand(*sh) < 0.02])
    p = np.stack([ellipsoid(sh, (50, 50, 47), (28, 30, 33)), ellipsoid(sh, (20, 70, 30), (10, 15, 12))])
    sps = np.array([(0.8, 0.9, 1.7), (2.0, 0.5, 1.1)])
    m, c = b200.seg_metrics3d(torch.from_numpy(r).cuda(), torch.from_numpy(p).cuda(), sps)
    assert m.shape == (2, 9) and c.shape == (2, 6)
    for n in range(2):
        check_oracle(m[n], c[n], r[n], p[n], tuple(sps[n]))


def test_surfaces_as_far_apart_as_the_volume_allows():
    """one voxel in each of two opposite corners: almost every line of both transforms holds no seed"""
    sh = (40, 300, 301)
    r = np.zeros(sh, np.uint8)
    p = np.zeros(sh, np.uint8)
    r[0, 0, 0] = 1
    p[-1, -1, -1] = 1
    sp = (3.0, 0.7, 5.0)
    m, c = b200.seg_metrics3d(torch.from_numpy(r).cuda(), torch.from_numpy(p).cuda(), sp)
    diag = np.sqrt(((sh[0] - 1) * sp[2]) ** 2 + ((sh[1] - 1) * sp[1]) ** 2 + ((sh[2] - 1) * sp[0]) ** 2)
    assert close(m[6:].cpu().numpy(), np.array([diag, diag, diag]))
    check_oracle(m, c, r, p, sp)


def test_width_not_a_multiple_of_32():
    rng = np.random.RandomState(5)
    sh = (17, 45, 77)
    r = ndimage_blobs(rng, sh)
    p = ndimage_blobs(rng, sh)
    sp = (1.1, 0.6, 2.3)
    m, c = b200.seg_metrics3d(torch.from_numpy(r).cuda(), torch.from_numpy(p).cuda(), sp)
    check_oracle(m, c, r, p, sp)


def ndimage_blobs(rng, sh):
    from scipy import ndimage
    return ndimage.gaussian_filter(rng.rand(*sh), 2.0) > 0.52


# ------------------------------------------------------------------------------------------------ buffers and runs
def _guarded(n, dtype):
    """n elements of dtype inside a byte buffer whose other bytes hold 0xFF (a NaN / -1 pattern)"""
    item = torch.empty(0, dtype=dtype).element_size()
    buf = torch.full((GUARD + n * item + GUARD,), 0xFF, dtype=torch.uint8, device="cuda")
    return buf, buf[GUARD:GUARD + n * item].view(dtype)


def _guards_intact(buf):
    return bool((buf[:GUARD] == 0xFF).all()) and bool((buf[-GUARD:] == 0xFF).all())


def test_outputs_stay_inside_their_buffers():
    r, p, sp = masks("scattered")
    be = runtime.cuda_backend()
    rt, pt = torch.from_numpy(r).cuda()[None].contiguous(), torch.from_numpy(p).cuda()[None].contiguous()
    spt = torch.tensor([sp[::-1]], dtype=torch.float64, device="cuda")
    (bc, counts), (bm, metrics), (bf, flags) = _guarded(6, torch.int64), _guarded(9, torch.float64), _guarded(1, torch.int32)
    be.segmetric3d(rt, pt, spt, counts, metrics, flags)
    torch.cuda.synchronize()
    assert all(_guards_intact(b) for b in (bc, bm, bf))
    assert counts.tolist() == list(osm.counts(r, p)) and flags.item() == 0 and not metrics.isnan().any()
    Sr, Sp = counts[4].item(), counts[5].item()
    outs = [_guarded(Sr, torch.int64), _guarded(Sp, torch.int64), _guarded(Sr, torch.float64),
            _guarded(Sp, torch.float64)]
    be.segmetric3d_points(rt, pt, spt, *[v for _, v in outs])
    torch.cuda.synchronize()
    assert all(_guards_intact(b) for b, _ in outs)
    ri, pi, r2p, p2r = osm.surface_distances(r, p, sp)
    assert outs[0][1].tolist() == np.ravel_multi_index(ri.T, r.shape).tolist()
    assert outs[1][1].tolist() == np.ravel_multi_index(pi.T, r.shape).tolist()
    assert close(outs[2][1].cpu().numpy(), r2p) and close(outs[3][1].cpu().numpy(), p2r)


def test_two_runs_are_bit_identical(ct_case):
    r, p, sp = ct_case
    rt, pt = torch.from_numpy(r).cuda(), torch.from_numpy(p).cuda()
    a = [t.cpu().numpy().tobytes() for t in b200.seg_metrics3d(rt, pt, sp)]
    b = [t.cpu().numpy().tobytes() for t in b200.seg_metrics3d(rt, pt, sp)]
    assert a == b
    m1, m2 = b200.Seg_Metirc3d(rt, pt, sp), b200.Seg_Metirc3d(rt, pt, sp)
    assert m1.real2pred_nn.tobytes() == m2.real2pred_nn.tobytes()
    assert m1.pred2real_nn.tobytes() == m2.pred2real_nn.tobytes()


def test_graph_capture_and_replay_on_new_masks():
    rng = np.random.RandomState(11)
    sh = (2, 24, 40, 52)
    sps = np.array([(0.9, 1.0, 2.0), (1.5, 0.7, 0.8)])
    new = [(ndimage_blobs(rng, sh[1:]), ndimage_blobs(rng, sh[1:])) for _ in range(4)]
    r = torch.from_numpy(np.stack([new[0][0], new[1][0]])).cuda()
    p = torch.from_numpy(np.stack([new[0][1], new[1][1]])).cuda()
    b200.seg_metrics3d(r, p, sps)                                # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        m, c = b200.seg_metrics3d(r, p, sps)
    r.copy_(torch.from_numpy(np.stack([new[2][0], new[3][0]])))
    p.copy_(torch.from_numpy(np.stack([new[2][1], new[3][1]])))
    g.replay()
    torch.cuda.synchronize()
    m2, c2 = b200.seg_metrics3d(r, p, sps)
    assert torch.equal(c, c2) and m.cpu().numpy().tobytes() == m2.cpu().numpy().tobytes()
    for n in range(2):
        check_oracle(m[n], c[n], new[2 + n][0], new[2 + n][1], tuple(sps[n]))


def test_predict_mask_output_feeds_the_metrics_directly():
    import oracle
    from oracle import nets as onets
    prev = runtime.get_precision()
    b200.set_precision("bf16")
    try:
        sd = onets.init_state_dict(onets.vnet3d_state_spec(1, 2), seed=0, randomize_affine=True)
        model = b200.VNet3d(1, 2)
        model.load_state_dict(sd)
        model = model.cuda().eval()
        x, _ = oracle.make_inputs(2, 1, (32, 32, 32), 2)
        mask = b200.predict_mask(model, x.cuda())               # uint8 (2, 32, 32, 32) on the device, 0/1
    finally:
        b200.set_precision(prev)
    assert mask.dtype == torch.uint8 and mask.is_cuda
    label = torch.from_numpy(np.stack([ellipsoid((32, 32, 32), (16, 16, 16), (9, 11, 10))] * 2)).cuda()
    m, c = b200.seg_metrics3d(label, mask, (1.0, 1.0, 1.0))
    mh = mask.cpu().numpy()
    for n in range(2):
        assert c[n].tolist() == list(osm.counts(label[n].cpu().numpy(), mh[n]))
        if mh[n].any():
            check_oracle(m[n], c[n], label[n].cpu().numpy(), mh[n], (1.0, 1.0, 1.0))
        else:
            assert m[n, 6:].isnan().all()
