"""Mask post-processing (dataprocess/utils.py:7-66) without a GPU: the scipy oracle (oracle/postprocess.py) against
brute force (a BFS flood fill, literal loops over the ball), the ball sizes, and the host logic of the
reference-named wrappers through a stand-in backend and a stand-in SimpleITK module."""
import collections
import itertools
import sys
import types

import numpy as np
import pytest
import torch

from oracle import postprocess as opp
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import postprocess as pp, runtime


# ------------------------------------------------------------------------------------------------ brute force
def bfs_largest(mask):
    """flood fill over face neighbours, components numbered in C order of their first voxel"""
    fg = mask != 0
    lab = np.zeros(fg.shape, np.int64)
    sizes = []
    steps = [tuple(s * (a == k) for a in range(fg.ndim)) for k in range(fg.ndim) for s in (-1, 1)]
    for start in itertools.product(*(range(s) for s in fg.shape)):
        if not fg[start] or lab[start]:
            continue
        sizes.append(0)
        lab[start] = len(sizes)
        q = collections.deque([start])
        while q:
            p = q.popleft()
            sizes[-1] += 1
            for st in steps:
                nb = tuple(a + b for a, b in zip(p, st))
                if all(0 <= c < s for c, s in zip(nb, fg.shape)) and fg[nb] and not lab[nb]:
                    lab[nb] = len(sizes)
                    q.append(nb)
    if not sizes:
        return np.zeros(fg.shape, np.uint8), 0, 0
    best = max(range(len(sizes)), key=lambda k: (sizes[k], -k))
    return (lab == best + 1).astype(np.uint8), len(sizes), sizes[best]


def ball_offsets(r, dims):
    return [d for d in itertools.product(range(-r, r + 1), repeat=dims) if sum(v * v for v in d) <= r * r + r]


def brute_morph(mask, r, op):
    fg = mask != 0
    sh = fg.shape
    offs = ball_offsets(r, fg.ndim)

    def inside(q):
        return all(0 <= c < s for c, s in zip(q, sh))

    def dil(x, p):       # outside is background
        return any(inside(q) and x[q] for q in (tuple(a + b for a, b in zip(p, d)) for d in offs))

    def ero(x, p):       # outside is foreground
        return all(not inside(q) or x[q] for q in (tuple(a + b for a, b in zip(p, d)) for d in offs))

    def apply(f, x):
        out = np.zeros(sh, bool)
        for p in itertools.product(*(range(s) for s in sh)):
            out[p] = f(x, p)
        return out

    if op == "dilate":
        return apply(dil, fg).astype(np.uint8)
    if op == "erode":
        return apply(ero, fg).astype(np.uint8)
    if op == "open":
        return apply(dil, apply(ero, fg)).astype(np.uint8)
    # close on the mask extended by background to infinity: every ball point q of p lies in dilate(fg)
    out = np.zeros(sh, bool)
    for p in itertools.product(*(range(s) for s in sh)):
        out[p] = all(dil(fg, tuple(a + b for a, b in zip(p, d))) for d in offs)
    return out.astype(np.uint8)


def brute_bbox(mask):
    pts = [p[::-1] for p in itertools.product(*(range(s) for s in mask.shape)) if mask[p] == 1]
    if not pts:
        return np.zeros(2 * mask.ndim + 1, np.int64)
    lo = [min(p[a] for p in pts) for a in range(mask.ndim)]
    hi = [max(p[a] for p in pts) for a in range(mask.ndim)]
    return np.array(lo + [h - l + 1 for l, h in zip(lo, hi)] + [len(pts)], np.int64)


SHAPES = [(6, 7, 9), (1, 5, 8), (4, 1, 6), (9, 11), (1, 13), (5, 1)]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("density", [0.05, 0.3116, 0.6, 0.9])
def test_oracle_components_and_box_match_brute_force(shape, density):
    rng = np.random.default_rng([*shape, int(density * 1e4)])
    for _ in range(3):
        m = (rng.random(shape) < density).astype(np.int32) * rng.integers(1, 3, shape)
        got, want = opp.largest_component(m), bfs_largest(m)
        assert np.array_equal(got[0], want[0]) and got[1:] == want[1:]
        assert np.array_equal(opp.label_bbox(m), brute_bbox(m))


@pytest.mark.parametrize("shape", [(5, 6, 7), (1, 6, 7), (8, 9), (1, 7)])
@pytest.mark.parametrize("op", opp.OPS)
def test_oracle_morphology_matches_brute_force(shape, op):
    rng = np.random.default_rng(len(shape) * 100 + shape[-1])
    for r in (0, 1, 2, 3):
        m = (rng.random(shape) < 0.45).astype(np.uint8)
        assert np.array_equal(opp.morphology(m, r, op), brute_morph(m, r, op)), (r, op)


def test_ball_sizes():
    assert [int(opp.ball(r, 3).sum()) for r in range(4)] == [1, 19, 81, 179]
    assert [int(opp.ball(r, 2).sum()) for r in range(4)] == [1, 9, 21, 37]
    assert [len(ball_offsets(r, 3)) for r in range(4)] == [1, 19, 81, 179]


def test_oracle_checkerboard_ties_break_in_raster_order():
    m = (np.indices((4, 5, 6)).sum(axis=0) % 2).astype(np.uint8)
    out, n, big = opp.largest_component(m)
    assert n == int(m.sum()) and big == 1
    first = np.argwhere(m.ravel())[0, 0]
    assert np.flatnonzero(out.ravel()).tolist() == [first]


# ------------------------------------------------------------------------------------------------ stand-ins
class StandInBackend:
    """the backend's three post-processing methods on the oracle, recording each call"""

    def __init__(self):
        self.calls = []

    def largest_component(self, mask, out, stats):
        self.calls.append(("cc", mask.dtype, tuple(mask.shape)))
        m, n, big = opp.largest_component(mask.numpy())
        out.copy_(torch.from_numpy(m))
        stats.copy_(torch.tensor([n, big]))

    def morphology(self, mask, radius, op, out):
        self.calls.append(("morph", mask.dtype, tuple(mask.shape), radius, op))
        name = {v: k for k, v in b200._abi.MORPH_OPS.items()}[op]
        out.copy_(torch.from_numpy(opp.morphology(mask.numpy(), radius, name)))

    def label_bbox(self, mask, box):
        self.calls.append(("bbox", mask.dtype, tuple(mask.shape)))
        box.copy_(torch.from_numpy(opp.label_bbox(mask.numpy())))


class FakeImage:
    """records pixel type and geometry as SimpleITK's image does"""

    def __init__(self, arr):
        self.arr = np.asarray(arr)
        self.origin, self.spacing = (0.0,) * self.arr.ndim, (1.0,) * self.arr.ndim
        self.direction = tuple(np.eye(self.arr.ndim).ravel())

    def GetSize(self):
        return self.arr.shape[::-1]

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
def standin(monkeypatch):
    be = StandInBackend()
    runtime._set_backend_for_testing(be)
    monkeypatch.setattr(pp, "_device", lambda: torch.device("cpu"))
    yield be
    runtime._set_backend_for_testing(None)


@pytest.fixture
def fake_sitk(monkeypatch):
    m = types.ModuleType("SimpleITK")
    m.GetArrayFromImage = lambda img: img.arr.copy()
    m.GetImageFromArray = lambda arr: FakeImage(np.asarray(arr))
    monkeypatch.setitem(sys.modules, "SimpleITK", m)
    return m


def _image(arr):
    img = FakeImage(arr)
    img.SetOrigin((-12.5, 3.25, 7.0)[:arr.ndim])
    img.SetSpacing((0.7, 0.8, 2.5)[:arr.ndim])
    img.SetDirection(tuple(np.eye(arr.ndim)[::-1].ravel()))
    return img


def _two_blobs(shape=(6, 8, 9)):
    m = np.zeros(shape, np.int16)
    m[0:2, 0:2, 0:2] = 1
    m[3:6, 4:8, 3:9] = 1
    return m


def test_largest_component_numpy_and_sitk_paths(standin, fake_sitk):
    m = _two_blobs()
    want = opp.largest_component(m)[0]
    out = b200.GetLargestConnectedCompont(m)
    assert isinstance(out, np.ndarray) and out.dtype == np.uint32 and np.array_equal(out, want)
    img = _image(m)
    res = b200.GetLargestConnectedCompont(img)
    assert isinstance(res, FakeImage) and res.arr.dtype == np.uint32 and np.array_equal(res.arr, want)
    assert (res.GetOrigin(), res.GetSpacing(), res.GetDirection()) == (img.GetOrigin(), img.GetSpacing(),
                                                                      img.GetDirection())
    assert standin.calls[0] == ("cc", torch.int16, m.shape)


def test_largest_component_of_an_empty_mask_is_all_ones(standin):
    out = b200.GetLargestConnectedCompont(np.zeros((3, 4, 5), np.uint8))
    assert out.dtype == np.uint32 and (out == 1).all()
    # the device form has no quirk
    dev, stats = b200.largest_component(torch.zeros(3, 4, 5, dtype=torch.uint8))
    assert not dev.any() and stats.tolist() == [0, 0]


@pytest.mark.parametrize("name", ["open", "close", "dilate", "erode"])
def test_morphology_numpy_and_sitk_paths(standin, fake_sitk, name):
    m = _two_blobs().astype(np.float32)
    m[1, 1, 1] = np.nan                               # != 0 in ITK's test
    want = opp.morphology(m, 2, name)
    out = b200.MorphologicalOperation(m, 2, name)
    assert out.dtype == np.uint8 and np.array_equal(out, want)
    img = _image(m[2])
    res = b200.MorphologicalOperation(img, 1, name)
    assert isinstance(res, FakeImage) and res.arr.dtype == np.uint8
    assert np.array_equal(res.arr, opp.morphology(m[2], 1, name)) and res.GetSpacing() == img.GetSpacing()
    assert res.GetDirection() == img.GetDirection() and res.GetOrigin() == img.GetOrigin()


def test_morphology_default_name_unknown_names_and_float64(standin):
    m = _two_blobs()
    assert np.array_equal(b200.MorphologicalOperation(m, 1), opp.morphology(m, 1, "open"))
    assert b200.MorphologicalOperation(m, 1, "tophat") is None
    assert b200.MorphologicalOperation(m, 10 ** 6, "Open") is None        # the name is checked first
    f = m.astype(np.float64) * 0.5
    assert np.array_equal(b200.MorphologicalOperation(f, 1, "dilate"), opp.morphology(m, 1, "dilate"))
    assert standin.calls[-1][1] == torch.uint8


def test_bbox_numpy_sitk_and_missing_label(standin, fake_sitk):
    m = _two_blobs()
    m[0, 0, 0] = 2                                    # only voxels equal to 1 count
    box = b200.GetLargestConnectedCompontBoundingbox(m)
    assert box.dtype == np.int64 and box.tolist() == brute_bbox(m)[:-1].tolist()
    assert b200.GetLargestConnectedCompontBoundingbox(_image(m[4])).tolist() == brute_bbox(m[4])[:-1].tolist()
    assert len(b200.GetLargestConnectedCompontBoundingbox(m[4])) == 4
    with pytest.raises(RuntimeError, match="label 1"):
        b200.GetLargestConnectedCompontBoundingbox((m != 0).astype(np.uint8) * 255)


def test_unsigned_and_narrow_integer_masks_keep_zero_and_one(standin):
    m = _two_blobs()
    for dt in (np.int8, np.uint16, np.uint32, np.uint64):
        a = m.astype(dt)
        a[0, 0, 0] = np.iinfo(dt).max                  # nonzero, not 1, whatever the reinterpretation
        assert np.array_equal(b200.GetLargestConnectedCompont(a), opp.largest_component(a)[0].astype(np.uint32))
        assert b200.GetLargestConnectedCompontBoundingbox(a).tolist() == brute_bbox(a)[:-1].tolist()


def test_dtype_shape_and_radius_errors(standin):
    t = torch.zeros(4, 5, 6)
    with pytest.raises(TypeError, match="dtype"):
        b200.largest_component(t)
    with pytest.raises(TypeError, match="dtype"):
        b200.label_bbox(t.double())
    with pytest.raises(TypeError, match="dtype"):
        b200.binary_morphology(t.double(), 1, "open")
    b200.binary_morphology(t, 1, "open")              # float32 is a morphology dtype
    with pytest.raises(TypeError, match="pixel type"):
        b200.GetLargestConnectedCompont(np.zeros((3, 4), np.float32))
    with pytest.raises(ValueError, match="shape"):
        b200.largest_component(torch.zeros(2, 3, 4, 5, dtype=torch.uint8))
    with pytest.raises(ValueError, match="empty"):
        b200.label_bbox(torch.zeros(0, 4, dtype=torch.uint8))
    with pytest.raises(ValueError, match="op must be"):
        b200.binary_morphology(t, 1, "tophat")
    for r in (-1, 65):
        with pytest.raises(ValueError, match="radius"):
            b200.binary_morphology(t, r, "dilate")
        with pytest.raises(ValueError, match="radius"):
            b200.MorphologicalOperation(np.zeros((3, 4), np.uint8), r, "erode")
    with pytest.raises(TypeError, match="radius"):
        b200.binary_morphology(t, 1.5, "dilate")
    b200.binary_morphology(t, 64, "dilate")
    b200.binary_morphology(t, np.int64(3), "close")
    assert [c[3] for c in standin.calls if c[0] == "morph"] == [1, 64, 3]


def test_size_limits_raise_before_any_launch(standin):
    big = torch.zeros(1, 1, dtype=torch.uint8).expand(2 ** 16, 2 ** 15)       # 2^31 voxels, no storage
    with pytest.raises(ValueError, match="2\\^31"):
        b200.largest_component(big)
    near = torch.zeros(1, 1, dtype=torch.uint8).expand(2 ** 16, 2 ** 15 - 8)
    with pytest.raises(ValueError, match="padded"):
        b200.binary_morphology(near, 5, "close")
    assert standin.calls == []


def test_install_rebinds_dataprocess_utils(monkeypatch):
    mod = types.ModuleType("dataprocess.utils")
    orig = {n: object() for n in ("GetLargestConnectedCompont", "GetLargestConnectedCompontBoundingbox",
                                  "MorphologicalOperation")}
    for n, o in orig.items():
        setattr(mod, n, o)
    mod.file_name_path = object()
    monkeypatch.setitem(sys.modules, "dataprocess.utils", mod)
    try:
        assert b200.install() >= 3
        assert mod.GetLargestConnectedCompont is b200.GetLargestConnectedCompont
        assert mod.GetLargestConnectedCompontBoundingbox is b200.GetLargestConnectedCompontBoundingbox
        assert mod.MorphologicalOperation is b200.MorphologicalOperation
    finally:
        b200.uninstall()
    assert all(getattr(mod, n) is o for n, o in orig.items())
