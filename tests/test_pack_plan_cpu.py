"""Host-side operand layout plans (``_abi.CudaBackend._pack_plan``) checked on CPU: the (T, K, N2, N1, strides, flip)
descriptors that ``b200seg_pack_weights_multi`` executes on the device are run here by a numpy restatement of the
kernel's index rule

    dst[t'][k][n2][n1] = src[t*st + k*sk + n2*sn2 + n1*sn1],   t' = T-1-t if flip else t      (elementwise.cu)

and compared with the layout every packed-operand code promises (DESIGN.md section 3): the CUDA-core layouts against
the CPU emulation backend's own ``pack_weight``, the tensor-core layouts (K-major rows, 8-channel halo planes, 64-channel
weight-streaming groups) against direct permutations of the torch weight.  No GPU, no kernel launch: the library is
only asked which kernel family takes a shape (pure host functions)."""
import itertools

import numpy as np
import pytest
import torch

from pytorchdeeplearing_b200 import _abi
from pytorchdeeplearing_b200._abi import BF16, BF16_HALO, BF16_HALO_WS, BF16_TC, F32
from pytorchdeeplearing_b200.engine import DOWN, K1, K3, UP
from emu_backend import EmuBackend


def _backend():
    be = object.__new__(_abi.CudaBackend)            # no CUDA device here: only the planning half of the backend
    be.lib = _abi.load_library()
    return be


def _run_descs(w, shape, args):
    src = w.reshape(-1).numpy()
    out = np.full(int(np.prod(shape)), np.nan, dtype=np.float32)
    parts = args if isinstance(args, list) else [(0, 0, args)]
    for so, do, (T, K, N2, N1, s_t, s_k, s_n2, s_n1, flip) in parts:
        t, k, n2, n1 = np.meshgrid(np.arange(T), np.arange(K), np.arange(N2), np.arange(N1), indexing="ij")
        si = so + t * s_t + k * s_k + n2 * s_n2 + n1 * s_n1
        tt = (T - 1 - t) if flip else t
        di = do + ((tt * K + k) * N2 + n2) * N1 + n1
        assert np.isnan(out[di.reshape(-1)]).all()       # every destination element written once
        out[di.reshape(-1)] = src[si.reshape(-1)]
    assert not np.isnan(out).any()                       # ... and none left out
    return torch.from_numpy(out).view(shape)


def _weight(kind, cin, cout, dims):
    taps = {K3: 3, K1: 1, DOWN: 2, UP: 2}[kind] ** dims
    a, b = (cin, cout) if kind == UP else (cout, cin)    # ConvTranspose keeps (Ci, Co, taps)
    g = torch.Generator().manual_seed(cin * 1000 + cout * 10 + kind)
    return torch.randn((a, b) + (int(round(taps ** (1 / dims))),) * dims, generator=g), a, b, taps


@pytest.mark.parametrize("kind,which,dims", list(itertools.product((K3, K1, DOWN, UP), ("fwd", "dgrad"), (2, 3))))
def test_cuda_core_layouts_equal_the_emulation_backend(kind, which, dims):
    """fp32 (parity mode) plans and bf16 plans with the tensor-core paths disabled"""
    w, a, b, taps = _weight(kind, 24, 40, dims)
    ref = EmuBackend().pack_weight(w, kind, which, torch.float32, dims)
    be = _backend()
    for dtype, allow_tc in ((torch.float32, True), (torch.bfloat16, False)):
        shape, code, args = be._pack_plan(w, kind, which, dtype, dims, allow_tc, 10 ** 6)
        assert code == (F32 if dtype == torch.float32 else BF16)
        got = _run_descs(w, shape, args)
        assert got.shape == ref.shape and torch.equal(got, ref)


@pytest.mark.parametrize("cin,cout", [(16, 16), (16, 32), (32, 16), (32, 32)])
@pytest.mark.parametrize("which", ["fwd", "dgrad"])
def test_halo_planes_layout(cin, cout, which):
    """BF16_HALO (full-resolution 3x3x3 layers): [tap][K/8][N][K%8] with K = the contraction channel of the conv that
    consumes the operand (Cin forward, Cout for the data gradient, taps reversed)"""
    w, a, b, taps = _weight(K3, cin, cout, 3)
    shape, code, args = _backend()._pack_plan(w, K3, which, torch.bfloat16, 3, True, 96 ** 3)
    assert code == BF16_HALO
    got = _run_descs(w, shape, args)
    w3 = w.reshape(cout, cin, taps)
    if which == "fwd":
        want = w3.permute(2, 1, 0).reshape(taps, cin // 8, 8, cout).permute(0, 1, 3, 2)         # [t][ci/8][co][ci%8]
    else:
        want = w3.flip(2).permute(2, 0, 1).reshape(taps, cout // 8, 8, cin).permute(0, 1, 3, 2)  # [T-1-t][co/8][ci][co%8]
    assert tuple(got.shape) == tuple(want.shape) and torch.equal(got, want.contiguous())


@pytest.mark.parametrize("c", [64, 128])
@pytest.mark.parametrize("which", ["fwd", "dgrad"])
def test_weight_streaming_groups_layout(c, which):
    """BF16_HALO_WS (64/128-channel 3x3x3 levels): [N/NT][tap][K/8][N%NT][K%8], one contiguous block per group of NT
    output channels (what a CTA streams through its cp.async.bulk ring)"""
    w, a, b, taps = _weight(K3, c, c, 3)
    be = _backend()
    nt = be.lib.b200seg_conv_halo_ws_ntile(K3, c, c)
    assert nt > 0
    shape, code, args = be._pack_plan(w, K3, which, torch.bfloat16, 3, True, 24 ** 3)
    assert code == BF16_HALO_WS and isinstance(args, list) and len(args) == c // nt
    got = _run_descs(w, shape, args)
    w3 = w.reshape(c, c, taps)                         # (co, ci, t)
    src = w3 if which == "fwd" else w3.flip(2).permute(1, 0, 2)     # (n, k, t'): n = output channel of the consumer
    want = src.reshape(c // nt, nt, c // 8, 8, taps).permute(0, 4, 2, 1, 3)
    assert tuple(got.shape) == tuple(want.shape) and torch.equal(got, want.contiguous())


@pytest.mark.parametrize("kind,cin,cout,dims", [(K3, 256, 256, 3), (K1, 128, 64, 3), (DOWN, 16, 32, 3), (UP, 32, 16, 3),
                                                (DOWN, 32, 64, 2), (UP, 64, 32, 2), (K1, 64, 32, 2)])
@pytest.mark.parametrize("which", ["fwd", "dgrad"])
def test_kmajor_tensor_core_layout(kind, cin, cout, dims, which):
    """BF16_TC: [tap][N][K] rows, K = contraction channel contiguous (what the 2-D TMA descriptor of conv_tc.cu reads);
    the data gradient of a stride-1 conv reverses the taps, a transposed conv swaps the roles of its two channel axes"""
    w, a, b, taps = _weight(kind, cin, cout, dims)
    # small volumes: the halo kernels do not take the layer, the K-major plan is what remains
    shape, code, args = _backend()._pack_plan(w, kind, which, torch.bfloat16, dims, True, 6 ** 3)
    assert code == BF16_TC
    got = _run_descs(w, shape, args)
    w3 = w.reshape(a, b, taps)
    if which == "dgrad" and kind in (K3, K1):
        want = w3.flip(2).permute(2, 1, 0)             # [T-1-t][ci][co]: K = co
    elif (which == "fwd" and kind != UP) or (which == "dgrad" and kind == UP):
        want = w3.permute(2, 0, 1)                     # [t][A][B]: K = second torch axis
    else:
        want = w3.permute(2, 1, 0)                     # [t][B][A]
    assert tuple(got.shape) == tuple(want.shape) and torch.equal(got, want.contiguous())


# ------------------------------------------------------------------------------------------------ tensor descriptors
def test_tensor_descriptor_of_channel_pitch_views():
    """``_desc``: every kernel argument is an (N,D,H,W,C) view with unit channel stride and a channel pitch ld >= C
    (DESIGN.md section 3) -- the halves of a skip-concat buffer, unit-depth 2-D tensors, single-voxel levels."""
    cat = torch.zeros(2, 4, 6, 8, 32, dtype=torch.bfloat16)
    left, right = cat[..., :16], cat[..., 16:]
    for view, off in ((left, 0), (right, 16)):
        d = _abi._desc(view)
        assert (d.n, d.d, d.h, d.w, d.c, d.ld, d.dtype) == (2, 4, 6, 8, 16, 32, BF16)
        assert d.ptr == cat.data_ptr() + off * cat.element_size()
    d = _abi._desc(torch.zeros(3, 1, 5, 7, 4))                         # 2-D net: unit depth, fp32, dense
    assert (d.n, d.d, d.h, d.w, d.c, d.ld, d.dtype) == (3, 1, 5, 7, 4, 4, F32)
    d = _abi._desc(torch.zeros(2, 1, 1, 1, 64)[..., 32:])               # one voxel per sample: pitch from the batch stride
    assert (d.c, d.ld) == (32, 64)
    d = _abi._desc(torch.zeros(1, 1, 1, 1, 8))                          # nothing to infer a pitch from: dense
    assert (d.c, d.ld) == (8, 8)
    x = torch.zeros(2, 1, 4, 6, 8).permute(0, 2, 3, 4, 1)               # (N,1,D,H,W) network input read as NDHWC, C = 1
    d = _abi._desc(x)
    assert (d.n, d.d, d.h, d.w, d.c, d.ld) == (2, 4, 6, 8, 1, 1)
    assert _abi._desc(None) is None


def test_tensor_descriptor_rejects_what_the_kernels_cannot_address():
    ncdhw = torch.zeros(2, 8, 4, 4, 4).permute(0, 2, 3, 4, 1)[..., :8]
    assert ncdhw.stride(-1) != 1
    with pytest.raises(ValueError):
        _abi._desc(ncdhw)                                               # channel stride != 1
    with pytest.raises(ValueError):
        _abi._desc(torch.zeros(2, 4, 4, 4, 8)[:, :, ::2])               # strided rows
    with pytest.raises(ValueError):
        _abi._desc(torch.zeros(4, 4, 4, 8))                             # not 5-D
    with pytest.raises(TypeError):
        _abi._desc(torch.zeros(1, 2, 2, 2, 8, dtype=torch.float16))     # only fp32 / bf16 activations
