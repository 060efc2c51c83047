"""Seg_Metirc3d (reference model/metric.py:11-142) without a GPU: the fp64 scipy oracle against the fixtures the real
reference class produced (tests/golden/segmetric.npz), the drop-in class's refusals and return types, install() /
uninstall() of the name, and the class logic on an emulated backend."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import segmetric as osm
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import runtime
from conftest import GOLDEN
from emu_backend import EmuBackend

GOLD = dict(np.load(os.path.join(GOLDEN, "segmetric.npz")))
CASES = [str(c) for c in GOLD["cases"]]
OK_CASES = [c for c in CASES if c + "_raises" not in GOLD]


def masks(case):
    """-> (real, pred) numpy arrays in the case's dtype, spacing"""
    shape = tuple(int(s) for s in GOLD[case + "_shape"])
    n = int(np.prod(shape))
    dt = np.dtype(str(GOLD[case + "_dtype"]))
    r = np.unpackbits(GOLD[case + "_real"])[:n].reshape(shape).astype(dt)
    p = np.unpackbits(GOLD[case + "_pred"])[:n].reshape(shape).astype(dt)
    return r, p, tuple(float(s) for s in GOLD[case + "_spacing"])


def close(a, b, rel=1e-12):
    """elementwise |a - b| <= rel * |b|, or <= rel where b == 0"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and bool(np.all(np.abs(a - b) <= rel * np.where(b == 0, 1.0, np.abs(b))))


def check_against_fixture(case, metrics, dice_tuple, surf, pts=None):
    """metrics: nine values; dice_tuple: (2I, R + P); surf: (S_r, S_p); pts: (real pts, pred pts, real2pred,
    pred2real) or None"""
    want = GOLD[case + "_metrics"]
    assert [int(v) for v in dice_tuple] == GOLD[case + "_dice_tuple"].tolist()
    assert [int(v) for v in surf] == GOLD[case + "_S"].tolist()
    exact = [0, 1, 2, 4, 5] + ([] if case == "dtype_uint8" else [3])
    for k in exact:
        assert np.float64(metrics[k]).tobytes() == np.float64(want[k]).tobytes(), (case, osm.NAMES[k])
    assert close(metrics[6:], want[6:]), (case, list(metrics[6:]), list(want[6:]))
    if pts is not None and case + "_real_pts" in GOLD:
        for got, key in zip(pts[:2], ("_real_pts", "_pred_pts")):
            assert got.dtype == GOLD[case + key].dtype and np.array_equal(got, GOLD[case + key]), (case, key)
        for got, key in zip(pts[2:], ("_real2pred", "_pred2real")):
            assert got.dtype == np.float64 and close(got, GOLD[case + key]), (case, key)


@pytest.mark.parametrize("case", OK_CASES)
def test_oracle_reproduces_the_reference_fixture(case):
    r, p, sp = masks(case)
    m, cnt = osm.seg_metrics(r, p, sp)
    ri, pi, r2p, p2r = osm.surface_distances(r, p, sp)
    spz = np.array(sp[::-1]).reshape(1, 3)
    R, P, I, U, Sr, Sp = cnt
    check_against_fixture(case, m, (2 * I, R + P), (Sr, Sp), (ri * spz, pi * spz, r2p, p2r))


def test_uint8_fixture_shows_the_reference_rvd_wraparound():
    """the documented divergence: the reference's uint8 RVD wraps in unsigned arithmetic, bool gives the signed value"""
    assert GOLD["dtype_uint8_metrics"][3] > 1e15
    assert GOLD["dtype_bool_metrics"][3] < 0
    r, p, sp = masks("dtype_uint8")
    assert osm.seg_metrics(r, p, sp)[0][3] == GOLD["dtype_bool_metrics"][3]


def test_oracle_raises_on_the_empty_fixture():
    assert "empty_raises" in GOLD
    r, p, sp = masks("empty")
    with pytest.raises(ValueError):
        osm.seg_metrics(r, p, sp)


def test_block_touching_two_faces_has_44_surface_voxels():
    r, _, _ = masks("block_two_faces")
    assert int(r.sum()) == 48 and int(osm.surface(r).sum()) == 44
    assert osm.surface(np.ones((1, 4, 5), bool)).all()           # D == 1: every voxel is surface


# ------------------------------------------------------------------------------------------------ emulated backend
class _SegEmu(EmuBackend):
    """EmuBackend plus the segmentation-metric entry points, restated with the scipy oracle"""

    def upload_bytes(self, raw, device):
        return torch.frombuffer(bytearray(raw + bytes(-len(raw) % 16)), dtype=torch.uint8).to(device)

    @staticmethod
    def _volumes(real, pred, spacing_zyx):
        """the class places its masks on the current CUDA device when there is one"""
        sp = spacing_zyx.reshape(-1, 3).double().cpu().numpy()
        for n in range(real.shape[0]):
            yield real[n].cpu().numpy(), pred[n].cpu().numpy(), tuple(sp[n][::-1])

    def segmetric3d(self, real, pred, spacing_zyx, counts, metrics, flags):
        counts, metrics = counts.view(-1, 6), metrics.view(-1, 9)       # the buffers the C ABI reads as [N][6] / [N][9]
        for n, (r, p, sp) in enumerate(self._volumes(real, pred, spacing_zyx)):
            c = osm.counts(r, p)
            counts[n] = torch.tensor(c)
            flags[n] = int(not (np.isin(r, (0, 1)).all() and np.isin(p, (0, 1)).all()))
            if c[0] and c[1]:
                metrics[n] = torch.from_numpy(osm.seg_metrics(r, p, sp)[0])
            else:
                R, P, I, U = (np.float64(v) for v in c[:4])
                with np.errstate(divide="ignore", invalid="ignore"):
                    metrics[n] = torch.tensor([2 * I / (R + P), I / U, 1 - I / U, (P - R) / R, (R - I) / U,
                                               (P - I) / U, np.nan, np.nan, np.nan], dtype=torch.float64)

    def segmetric3d_points(self, real, pred, spacing_zyx, real_idx, pred_idx, real2pred, pred2real):
        out = [[], [], [], []]
        for r, p, sp in self._volumes(real, pred, spacing_zyx):
            ri, pi, r2p, p2r = osm.surface_distances(r, p, sp)
            out[0].append(np.ravel_multi_index(ri.T, r.shape))
            out[1].append(np.ravel_multi_index(pi.T, r.shape))
            out[2].append(r2p)
            out[3].append(p2r)
        for dst, parts in zip((real_idx, pred_idx, real2pred, pred2real), out):
            dst.copy_(torch.from_numpy(np.concatenate(parts)))


@pytest.fixture()
def emu():
    runtime._set_backend_for_testing(_SegEmu())
    yield
    runtime._set_backend_for_testing(None)


@pytest.mark.parametrize("case", OK_CASES)
def test_class_on_the_emulated_backend_matches_the_fixture_with_reference_types(emu, case):
    r, p, sp = masks(case)
    m = b200.Seg_Metirc3d(r, p, sp)
    assert m.real_mask is r and m.pred_mask is p and m.voxel_sapcing is sp
    dice = m.get_dice_coefficient()
    vals = [dice[0], m.get_jaccard_index(), m.get_VOE(), m.get_RVD(), m.get_FNR(), m.get_FPR(), m.get_ASSD(),
            m.get_RMSD(), m.get_MSD()]
    want_types = [str(t) for t in GOLD[case + "_types"]]
    if case != "dtype_uint8":       # the reference returns unsigned sums there; the drop-in keeps int64
        assert [type(v).__name__ for v in vals + list(dice[1:])] == want_types
    assert [type(v) for v in vals] == [np.float64] * 3 + [float] + [np.float64] * 3 + [float, np.float64]
    assert type(dice[1]) is np.int64 and type(dice[2]) is np.int64
    check_against_fixture(case, vals, dice[1:], (len(m.real2pred_nn), len(m.pred2real_nn)),
                          (m.real_mask_surface_pts, m.pred_mask_surface_pts, m.real2pred_nn, m.pred2real_nn))
    if case == "dtype_uint8":
        assert m.get_RVD() == float(GOLD["dtype_bool_metrics"][3])


def test_class_refuses_what_the_contract_excludes(emu):
    r, p, sp = masks("dtype_bool")
    with pytest.raises(ValueError, match="empty"):
        b200.Seg_Metirc3d(np.zeros_like(r), p, sp)
    with pytest.raises(ValueError, match="empty"):
        b200.Seg_Metirc3d(r, np.zeros_like(p), sp)
    with pytest.raises(ValueError, match="binarise"):
        b200.Seg_Metirc3d(r, p.astype(np.uint8) * 255, sp)
    with pytest.raises(ValueError, match="binarise"):
        b200.Seg_Metirc3d(r.astype(np.int64) * -1, p, sp)
    with pytest.raises(ValueError, match="3-D"):
        b200.Seg_Metirc3d(r[0], p[0], sp)
    with pytest.raises(ValueError, match="3-D"):
        b200.Seg_Metirc3d(r[None], p[None], sp)
    with pytest.raises(ValueError, match="3-D"):
        b200.Seg_Metirc3d(r, p[:-1], sp)
    for bad in ((1.0, 1.0), (1.0, 0.0, 1.0), (1.0, -2.0, 1.0), (1.0, float("nan"), 1.0), (float("inf"), 1.0, 1.0)):
        with pytest.raises(ValueError, match="voxel_spacing"):
            b200.Seg_Metirc3d(r, p, bad)
    with pytest.raises(TypeError):
        b200.Seg_Metirc3d(r.astype(np.float32), p, sp)


def test_functional_form_on_the_emulated_backend(emu):
    """(N, D, H, W) with one spacing per volume, and (D, H, W) -> (9,) / (6,)"""
    r1, p1, sp1 = masks("dtype_bool")
    r2, p2, sp2 = masks("identical")
    m, c = b200.seg_metrics3d(torch.from_numpy(r1), torch.from_numpy(p1), sp1)
    assert m.shape == (9,) and c.shape == (6,) and m.dtype == torch.float64 and c.dtype == torch.int64
    assert m.numpy().tobytes() == osm.seg_metrics(r1, p1, sp1)[0].tobytes()
    rr = torch.from_numpy(np.stack([r1, r1]))
    pp = torch.from_numpy(np.stack([p1, r1]))
    m, c = b200.seg_metrics3d(rr, pp, np.array([sp1, sp2]))
    assert m.shape == (2, 9) and c.shape == (2, 6)
    assert m[1, :6].tolist() == [1.0, 1.0, 0.0, 0.0, 0.0, 0.0] and m[1, 6:].tolist() == [0.0, 0.0, 0.0]
    assert c[0].tolist() == list(osm.counts(r1, p1))
    with pytest.raises(ValueError):
        b200.seg_metrics3d(rr, pp, np.ones((3, 3)))
    with pytest.raises(ValueError):
        b200.seg_metrics3d(rr[0, 0], pp[0, 0], sp1)


def test_install_rebinds_seg_metirc3d_and_uninstall_restores(monkeypatch):
    m = types.ModuleType("model.metric")
    orig = type("Seg_Metirc3d", (), {})
    m.Seg_Metirc3d = orig
    monkeypatch.setitem(sys.modules, "model.metric", m)
    try:
        assert b200.install() == 1
        assert m.Seg_Metirc3d is b200.Seg_Metirc3d
    finally:
        b200.uninstall()
    assert m.Seg_Metirc3d is orig
