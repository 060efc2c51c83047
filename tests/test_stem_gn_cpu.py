"""The engine takes the fused input block (csrc/stem_gn.cu) only when the backend offers it and the layer fits: the
emulated CPU backend has no such method, and the fp32 parity mode keeps the per-branch calls."""
import torch

from pytorchdeeplearing_b200.engine import Engine
from emu_backend import EmuBackend


class _Probe(EmuBackend):
    def stem_gn_ok(self, x, cout, dims):
        return True


def _image():
    return torch.zeros((1, 8, 8, 16, 1))


def test_no_probe_no_fused_block():
    assert not Engine(EmuBackend(), torch.bfloat16, 3).stem_gn_ok(_image(), 16)


def test_probe_gates_on_precision_and_width():
    assert Engine(_Probe(), torch.bfloat16, 3).stem_gn_ok(_image(), 16)
    assert not Engine(_Probe(), torch.float32, 3).stem_gn_ok(_image(), 16)
    assert not Engine(_Probe(), torch.bfloat16, 3).stem_gn_ok(_image(), 32)


def test_vnet_forward_on_emulated_backend_uses_per_branch_calls():
    import pytorchdeeplearing_b200 as b200
    from pytorchdeeplearing_b200 import runtime
    calls = []

    class _Rec(EmuBackend):
        def conv(self, kind, dims, x, *a, **k):
            if x.shape[-1] == 1:
                calls.append(kind)
            return super().conv(kind, dims, x, *a, **k)

    runtime._set_backend_for_testing(_Rec())
    try:
        m = b200.VNet3d(1, 2).train()
        m(torch.randn(1, 1, 16, 16, 16))
    finally:
        runtime._set_backend_for_testing(None)
    assert sorted(calls) == [0, 1]          # both stems through backend.conv
