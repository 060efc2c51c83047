"""Whole-volume 3-D inference (XModel.inference / inference_patch, reference model/modelVNet.py:678-698,
model/modelUnet.py:684-763) without a GPU: the fp64 oracle's normalize() against fixtures recorded from the reference
function, properties of the resample restatement, and the Python layer on an emulated backend (refusals, the
classifier TypeError, a stub-SimpleITK round trip)."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import nets as onets
from oracle import resample as R
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import inference as inf
from pytorchdeeplearing_b200 import runtime
from pytorchdeeplearing_b200._abi import NORM_MEANSTD, NORM_NONE
from conftest import GOLDEN
from emu_backend import EmuBackend

GOLD = dict(np.load(os.path.join(GOLDEN, "infer3d.npz")))
CASES = [str(c) for c in GOLD["cases"]]


@pytest.mark.parametrize("case", CASES)
def test_oracle_normalize_matches_the_reference_fixture_bit_for_bit(case):
    out = R.normalize(GOLD[case + "_input"])
    ref = GOLD[case + "_output"]
    assert out.dtype == np.float64 and out.shape == ref.shape
    assert np.array_equal(out.view(np.int64), ref.view(np.int64))


def test_fixture_cases_cover_both_early_returns_and_the_z_score():
    flags = {c: R.normalize_stats(GOLD[c + "_input"])[4] for c in CASES}
    assert flags["constant"] and flags["constant_zero"] and flags["nonzero_constant"]
    assert not flags["random"] and not flags["zero_heavy"] and not flags["ties"]


@pytest.mark.parametrize("dtype", [np.uint8, np.int16, np.int32, np.float32])
def test_equal_sizes_give_the_identity(dtype):
    rng = np.random.RandomState(0)
    v = (rng.rand(5, 7, 9) * 200).astype(dtype)
    out = R.resample_linear(v, v.shape, R.size_ratio(v.shape, v.shape))
    assert out.dtype == np.float32 and np.array_equal(out, v.astype(np.float32))


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_linear_ramps_are_reproduced_exactly(axis):
    shape = (13, 17, 19)
    ramp = np.indices(shape)[axis].astype(np.float32) * 4.0 - 7.0
    out_shape = (7, 11, 5)       # non-integer downsampling on every axis
    ratio = R.size_ratio(shape, out_shape)
    out = R.resample_linear(ramp, out_shape, ratio)
    u = np.arange(out_shape[axis]) * ratio[axis]
    want = (u * 4.0 - 7.0).astype(np.float32)
    idx = [None, None, None]
    idx[axis] = slice(None)
    assert np.array_equal(out, np.broadcast_to(want[tuple(idx)], out_shape))


def test_integer_cast_truncates_toward_zero_and_clamps():
    v = np.array([[[-3, 0]]], np.int16)                  # u = 0.5 * i: -1.5 truncates to -1
    out = R.resample_linear(v, (1, 1, 3), (1.0, 1.0, 0.5))
    assert out.tolist() == [[[-3.0, -1.0, 0.0]]]
    assert R.cast_pixel(np.array([300.7, -4.9]), np.uint8).tolist() == [255.0, 0.0]


def test_upsampling_beyond_two_gives_zeros_past_the_edge():
    v = np.full((4, 4, 4), 9.0, np.float32)
    out = R.resample_linear(v, (10, 4, 4), R.size_ratio((4, 4, 4), (10, 4, 4)))   # r = 0.4
    # u = 0.4 i < 3.5 for i <= 8; i = 9 gives u = 3.6 outside the buffer
    assert np.all(out[:9] == 9.0) and np.all(out[9] == 0.0)
    exact2 = R.resample_linear(v, (8, 4, 4), (0.5, 1.0, 1.0))
    assert np.all(exact2[7] == 0.0) and np.all(exact2[:7] == 9.0)     # u = 3.5 is outside too
    down = R.resample_linear(v, (3, 3, 3), R.size_ratio((4, 4, 4), (3, 3, 3)))
    assert np.all(down == 9.0)


def test_nearest_neighbour_ties_round_up_and_crop_pad():
    src = np.arange(4, dtype=np.uint8).reshape(1, 1, 4)
    out = R.resample_nearest(src, (1.0, 1.0, 0.5), (1, 1, 7), (1, 1, 7))
    assert out.tolist() == [[[0, 1, 1, 2, 2, 3, 3]]]        # u = 0.5, 1.5, 2.5 round up
    out = R.resample_nearest(src, (1.0, 1.0, 0.5), (1, 1, 8), (1, 1, 8))
    assert out[0, 0, 7] == 0                                 # u = 3.5: outside the buffer
    pad = R.resample_nearest(src, (1.0, 1.0, 1.0), (1, 1, 4), (2, 2, 6))
    assert pad[0, 0, :4].tolist() == [0, 1, 2, 3] and pad[0, 0, 4:].sum() == 0 and pad[1].sum() == 0
    crop = R.resample_nearest(src, (1.0, 1.0, 1.0), (1, 1, 4), (1, 1, 2))
    assert crop.tolist() == [[[0, 1]]]


@pytest.mark.parametrize("size,sp,nsp", [((512, 512, 300), (0.7, 0.7, 1.25), (1.0, 1.0, 1.0)),
                                         ((100, 90, 80), (1.0, 1.0, 1.0), (0.5, 0.5, 0.5)),
                                         ((64, 64, 33), (0.3, 0.3, 0.9), (0.7, 0.7, 0.7))])
def test_spacing_form_sizes_match_floor(size, sp, nsp):
    got = b200.spacing_size(size, sp, nsp)
    assert got == R.spacing_size(size, sp, nsp)
    assert got == tuple(int(np.floor(s * o / n + 1e-9)) for s, o, n in zip(size, sp, nsp))


@pytest.mark.parametrize("size,patch", [(96, 96), (100, 96), (200, 96), (9000, 96), (100, 8), (37, 4), (10, 2),
                                        (11, 3)])
def test_reference_window_walk_is_sliding_window_with_step_p_times_half_p(size, patch):
    assert inf._starts(size, patch, patch * (patch // 2)) == R.window_origins(size, patch)


# ---------------------------------------------------------------------------------------------- emulated backend
class EmuInfer(EmuBackend):
    """the new entry points, emulated through the oracle"""

    def resample_workspace(self, mode, out_zyx, device):
        return torch.zeros(256, dtype=torch.uint8, device=device)

    def resample_linear(self, src, ratio_zyx, out, mode=NORM_NONE, lower=0.0, upper=0.0, ws=None):
        if src.dtype not in (torch.uint8, torch.int16, torch.int32, torch.float32):
            raise TypeError(src.dtype)
        x = R.resample_linear(src.cpu().numpy(), tuple(out.shape), ratio_zyx)
        if mode == NORM_MEANSTD:
            x = R.truncate(x, lower, upper)
        out.copy_(torch.from_numpy(x))

    def normalize(self, mode, x, ws, out):
        xn = x.cpu().numpy()
        y = R.meanstd(xn) if mode == NORM_MEANSTD else R.normalize(xn).astype(np.float32)
        out.copy_(torch.from_numpy(y).reshape(out.shape))

    def resample_nearest_u8(self, src, ratio_zyx, valid_zyx, out):
        out.copy_(torch.from_numpy(R.resample_nearest(src.cpu().numpy(), ratio_zyx, valid_zyx, tuple(out.shape))))


@pytest.fixture
def emu():
    runtime._set_backend_for_testing(EmuInfer())
    prev = b200.get_precision()
    b200.set_precision("fp32")
    yield
    b200.set_precision(prev)
    runtime._set_backend_for_testing(None)


def _vnet(seed=0):
    model = b200.VNet3d(1, 2)
    model.load_state_dict(onets.init_state_dict(onets.vnet3d_state_spec(1, 2), seed=seed, randomize_affine=True))
    return model.eval()


def _volume(shape=(12, 20, 18), seed=3):
    return np.random.RandomState(seed).randint(-150, 150, size=shape).astype(np.int16)


def _oracle_chain(model, vol, new_size, intensity, window=(-100.0, 100.0)):
    out_zyx = tuple(reversed(new_size))
    x = R.resample_linear(vol, out_zyx, R.size_ratio(vol.shape, out_zyx))
    if intensity == "vnet":
        x = R.meanstd(R.truncate(x, *window))
    elif intensity == "unet":
        x = R.normalize(x).astype(np.float32)
    m = b200.predict(model, x[None])
    return R.resample_nearest(m, R.size_ratio(out_zyx, vol.shape), vol.shape, vol.shape)


@pytest.mark.parametrize("intensity", ["vnet", "unet", None])
def test_inference3d_on_the_emulated_backend_is_the_oracle_chain(emu, intensity):
    model, vol = _vnet(), _volume()
    got = b200.inference3d(model, vol, (16, 16, 16), intensity=intensity)
    assert got.dtype == np.uint8 and got.shape == vol.shape
    assert np.array_equal(got, _oracle_chain(model, vol, (16, 16, 16), intensity))


def test_inference_patch3d_on_the_emulated_backend(emu):
    model = _vnet()
    vol = np.random.RandomState(5).randint(-1100, -700, size=(14, 30, 26)).astype(np.int16)
    sp, nsp = (0.8, 0.8, 1.0), (1.2, 1.2, 0.75)
    got = b200.inference_patch3d(model, vol, sp, nsp, patch_size=(16, 16, 16))
    rs = R.spacing_size(tuple(reversed(vol.shape)), sp, nsp)
    rs_zyx = tuple(reversed(rs))
    x = R.resample_linear(vol, rs_zyx, tuple(n / o for n, o in zip(reversed(nsp), reversed(sp))))
    x = R.meanstd(R.truncate(x, -1024.0, -800.0))
    union = b200.sliding_window_mask(model, x[None], (16, 16, 16), step=(128, 128, 128))
    back = tuple(reversed(R.spacing_size(rs, nsp, sp)))
    want = R.resample_nearest(union, tuple(o / n for n, o in zip(reversed(nsp), reversed(sp))), back, vol.shape)
    assert got.dtype == np.uint8 and got.shape == vol.shape and np.array_equal(got, want)
    assert set(np.unique(got)) <= {0, 1}


def test_refusals(emu):
    model, vol = _vnet(), _volume()
    with pytest.raises(ValueError, match="intensity"):
        b200.inference3d(model, vol, intensity="ct")
    with pytest.raises(ValueError, match="newSize"):
        b200.inference3d(model, vol, (16, 16))
    with pytest.raises(ValueError, match="newSize"):
        b200.inference3d(model, vol, (16, 0, 16))
    with pytest.raises(ValueError, match=r"\(D, H, W\)"):
        b200.inference3d(model, vol[0])
    with pytest.raises(TypeError, match="int16"):
        b200.inference3d(model, vol.astype(np.int64))
    with pytest.raises(ValueError, match="spacing"):
        b200.inference_patch3d(model, vol, None, (1.0, 1.0, 1.0), patch_size=(16, 16, 16))
    with pytest.raises(ValueError, match="spacing"):
        b200.inference_patch3d(model, vol, (1.0, -1.0, 1.0), (1.0, 1.0, 1.0), patch_size=(16, 16, 16))
    with pytest.raises(ValueError, match="smaller than the patch"):
        b200.inference_patch3d(model, vol, (1.0, 1.0, 1.0), (1.0, 1.0, 1.0), patch_size=(32, 32, 32))
    with pytest.raises(ValueError, match="2-D"):
        b200.inference3d(b200.VNet2d(1, 2), vol)
    with pytest.raises(ValueError, match="interpolator"):
        b200.resample3d(torch.from_numpy(vol), (8, 8, 8), interpolator="cubic")
    with pytest.raises(TypeError, match="uint8"):
        b200.resample3d(torch.from_numpy(vol), (8, 8, 8), interpolator="nearest")
    with pytest.raises(ValueError, match="either newSize"):
        b200.resample3d(torch.from_numpy(vol))


def test_classifiers_raise_type_error(emu):
    vol = _volume()
    for model in (b200.ResNet3d(1, 2),):
        with pytest.raises(TypeError, match="classifier"):
            b200.inference3d(model, vol)
        with pytest.raises(TypeError, match="classifier"):
            b200.inference_patch3d(model, vol, (1.0, 1.0, 1.0), (1.0, 1.0, 1.0))


def test_resample3d_on_tensors_and_arrays(emu):
    vol = _volume()
    t = b200.resample3d(torch.from_numpy(vol), (9, 7, 5))
    assert isinstance(t, torch.Tensor) and t.dtype == torch.float32 and tuple(t.shape) == (5, 7, 9)
    a = b200.resample3d(vol, spacing=(1.0, 1.0, 1.0), newSpacing=(2.0, 2.0, 2.0), device="cpu")
    assert isinstance(a, np.ndarray) and a.shape == (6, 10, 9)
    assert np.array_equal(a, R.resample_linear(vol, (6, 10, 9), (2.0, 2.0, 2.0)))
    m = (vol > 0).astype(np.uint8)
    n = b200.resample3d(m, (9, 10, 6), interpolator="nearest", out_size=(20, 10, 6), device="cpu")
    assert n.shape == (6, 10, 20) and n[:, :, 9:].sum() == 0


class _StubImage:
    def __init__(self, arr):
        self.arr = arr
        self.origin, self.spacing, self.direction = (0.0, 0.0, 0.0), (1.0, 1.0, 1.0), (1.0, 0, 0, 0, 1.0, 0, 0, 0, 1.0)

    def GetSize(self):
        return tuple(reversed(self.arr.shape))

    def GetSpacing(self):
        return self.spacing

    def GetOrigin(self):
        return self.origin

    def GetDirection(self):
        return self.direction

    def SetSpacing(self, v):
        self.spacing = tuple(v)

    def SetOrigin(self, v):
        self.origin = tuple(v)

    def SetDirection(self, v):
        self.direction = tuple(v)


@pytest.fixture
def stub_sitk(monkeypatch):
    m = types.ModuleType("SimpleITK")
    m.GetArrayFromImage = lambda img: img.arr.copy()
    m.GetImageFromArray = lambda arr: _StubImage(np.asarray(arr))
    monkeypatch.setitem(sys.modules, "SimpleITK", m)
    return m


def test_simpleitk_round_trip_keeps_the_geometry(emu, stub_sitk):
    model, vol = _vnet(), _volume()
    img = _StubImage(vol)
    img.SetOrigin((-120.5, 33.25, 7.0))
    img.SetSpacing((0.7, 0.8, 2.5))
    img.SetDirection((0.0, 1.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, -1.0))
    out = b200.inference3d(model, img, (16, 16, 16))
    assert isinstance(out, _StubImage)
    assert out.GetOrigin() == img.GetOrigin() and out.GetSpacing() == img.GetSpacing()
    assert out.GetDirection() == img.GetDirection()
    assert out.arr.dtype == np.uint8 and np.array_equal(out.arr, _oracle_chain(model, vol, (16, 16, 16), "vnet"))
    # the patch form takes the image's own spacing
    p = b200.inference_patch3d(model, img, newSpacing=(0.7, 0.8, 1.25), patch_size=(16, 16, 16), intensity=None)
    assert isinstance(p, _StubImage) and p.GetSpacing() == img.GetSpacing() and p.arr.shape == vol.shape
