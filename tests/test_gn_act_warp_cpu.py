"""Host-side checks of the LeakyReLU / InstanceNorm GroupNorm forms and the voxelmorph warp (no device needed): the
``b200seg_gn`` layout, the argument rules of the entry points (which all return before touching a device), and the
input checks of ``warp3d``."""
import ctypes as C
import os

import pytest
import torch

from pytorchdeeplearing_b200 import _abi, build

EINVAL = -1


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(_abi.LIB_PATH):
        build.build()
    return _abi.load_library()


def test_gn_struct_keeps_its_size_and_act_fills_the_padding():
    # 4 pointers, groups, (pad), vox, eps, act: the act field sits where eps's padding was
    assert C.sizeof(_abi.GnDesc) == 56
    assert _abi.GnDesc.act.offset == _abi.GnDesc.eps.offset + 4
    g = _abi.GnDesc(1, 2, 3, None, 8, 10, 1e-5)
    assert g.act == _abi.ACT_RELU


def test_version_is_bumped(lib):
    assert lib.b200seg_version() >= 201


def _desc(c=16, dtype=_abi.BF16, ptr=0x1000):
    return _abi.TensorDesc(ptr, 2, 4, 4, 4, c, c, dtype)


def _gn(act, groups=8, ptr=0x2000):
    return _abi.GnDesc(ptr, ptr, ptr, None, groups, 64, 1e-5, act)


def test_elementwise_entry_points_reject_bad_activation_and_groups(lib):
    y, out = _desc(), _desc()
    sums = C.c_void_p(0x3000)
    # an activation outside B200SEG_ACT_*
    assert lib.b200seg_apply_gn(C.byref(y), C.byref(_gn(2)), None, None, None, C.byref(out), 0, None) == EINVAL
    assert b"GroupNorm reference" in lib.b200seg_last_error()
    assert lib.b200seg_gn_bwd_reduce_gn(C.byref(y), C.byref(y), C.byref(_gn(-1)), sums, 0, None) == EINVAL
    # two branches of one apply share their activation
    y2 = _desc()
    assert lib.b200seg_apply_gn(C.byref(y), C.byref(_gn(1)), C.byref(y2), C.byref(_gn(0)), None, C.byref(out), 0,
                                None) == EINVAL
    # the ReLU kernels derive one group per thread: more than 256 groups only with the LeakyReLU tail (512 at most)
    y512 = _desc(512)
    assert lib.b200seg_apply_gn(C.byref(y512), C.byref(_gn(0, 512)), None, None, None, C.byref(y512), 0,
                                None) == EINVAL
    y1024 = _desc(1024)
    assert lib.b200seg_apply_gn(C.byref(y1024), C.byref(_gn(1, 1024)), None, None, None, C.byref(y1024), 0,
                                None) == EINVAL


def test_fused_families_refuse_leaky_relu(lib):
    x = _desc(1, _abi.F32)
    out = _desc(16)
    g = _desc(16)
    w = C.c_void_p(0x4000)
    b = C.c_void_p(0x5000)
    leaky = _gn(_abi.ACT_LEAKY)
    s = C.c_void_p(0x6000)
    assert lib.b200seg_stem_gn_apply(C.byref(x), w, b, w, b, C.byref(leaky), C.byref(leaky), C.byref(out), 0,
                                     None) == EINVAL
    assert b"ACT_RELU" in lib.b200seg_last_error()
    assert lib.b200seg_stem_gn_bwd_sums(C.byref(x), w, b, w, b, C.byref(leaky), C.byref(leaky), C.byref(g), s, s, 0,
                                        None) == EINVAL
    assert lib.b200seg_stem_gn_bwd(C.byref(x), w, b, w, b, C.byref(leaky), C.byref(leaky), C.byref(g), s, s, s, s, s,
                                   s, s, s, 0, None) == EINVAL
    x32 = _desc(32)
    assert lib.b200seg_up_gn_apply(C.byref(x32), w, b, C.byref(leaky), C.byref(out), 0, None) == EINVAL
    assert lib.b200seg_up_gn_bwd_sums(C.byref(x32), w, b, C.byref(leaky), C.byref(g), s, 0, None) == EINVAL
    assert lib.b200seg_up_gn_bwd(C.byref(x32), w, b, C.byref(leaky), C.byref(g), s, s, C.byref(x32), s, s, s, 0,
                                 None) == EINVAL
    assert b"ACT_RELU" in lib.b200seg_last_error()
    y = _desc(16)
    assert lib.b200seg_conv_bwdstats(0, 3, C.byref(y), w, _abi.BF16_HALO, C.byref(y), None, C.byref(y),
                                     C.byref(leaky), s, 0, None) == EINVAL
    assert b"ACT_RELU" in lib.b200seg_last_error()


def test_warp_entry_points_reject_bad_arguments(lib):
    p = C.c_void_p(0x1000)
    # extents of 1 (the normalisation divides by s - 1), nothing to warp, null pointers
    assert lib.b200seg_warp3d(p, p, 1, p, 1, 1, 1, 8, 8, p, p, 0, None) == EINVAL
    assert lib.b200seg_warp3d(p, None, 0, None, 0, 1, 8, 8, 8, None, None, 0, None) == EINVAL
    assert lib.b200seg_warp3d(p, None, 1, p, 1, 1, 8, 8, 8, p, p, 0, None) == EINVAL
    assert lib.b200seg_warp3d_bwd(p, None, 1, p, None, 1, 8, 8, 8, p, 0, None) == EINVAL
    assert lib.b200seg_warp3d_bwd(p, p, 0, p, None, 1, 8, 8, 8, p, 0, None) == EINVAL


def test_warp3d_input_checks():
    from pytorchdeeplearing_b200 import warp3d
    img = torch.zeros(1, 1, 4, 5, 6)
    lab = torch.zeros(1, 2, 4, 5, 6)
    ddf = torch.zeros(1, 3, 4, 5, 6)
    with pytest.raises(TypeError):
        warp3d(img.double(), lab, ddf)
    with pytest.raises(TypeError):
        warp3d(img, lab, ddf.half())
    with pytest.raises(ValueError, match="requires a gradient"):
        warp3d(img.clone().requires_grad_(), lab, ddf)
    with pytest.raises(ValueError, match="requires a gradient"):
        warp3d(img, lab.clone().requires_grad_(), ddf)
    with pytest.raises(ValueError, match="ddf must be"):
        warp3d(img, lab, torch.zeros(1, 2, 4, 5, 6))
    with pytest.raises(ValueError, match="moving_image must be"):
        warp3d(torch.zeros(1, 1, 4, 5, 7), lab, ddf)
    with pytest.raises(ValueError, match="at least 2"):
        warp3d(torch.zeros(1, 1, 1, 5, 6), None, torch.zeros(1, 3, 1, 5, 6))
    with pytest.raises(ValueError, match="nothing to warp"):
        warp3d(None, None, ddf)
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            warp3d(img, lab, ddf)
