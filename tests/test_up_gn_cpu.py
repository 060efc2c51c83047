"""The engine takes the fused up_tr32 layer (csrc/up_gn.cu) only when the backend offers it and the layer fits: the
emulated CPU backend has no such method, and the fp32 parity mode and 2-D nets keep the per-layer calls."""
import torch

from pytorchdeeplearing_b200.engine import Engine, UP
from emu_backend import EmuBackend


class _Probe(EmuBackend):
    def up_gn_ok(self, x, wpk, cout, dims):
        return True


def _input():
    return torch.zeros((1, 8, 8, 16, 32))


def test_no_probe_no_fused_layer():
    assert not Engine(EmuBackend(), torch.bfloat16, 3).up_gn_ok(_input(), "up_tr32.up_conv.weight", 16)


def test_probe_gates_on_precision_and_dims():
    assert Engine(_Probe(), torch.bfloat16, 3).up_gn_ok(_input(), "up_tr32.up_conv.weight", 16)
    assert not Engine(_Probe(), torch.float32, 3).up_gn_ok(_input(), "up_tr32.up_conv.weight", 16)
    assert not Engine(_Probe(), torch.bfloat16, 2).up_gn_ok(_input(), "up_tr32.up_conv.weight", 16)


def test_vnet_on_emulated_backend_uses_per_layer_calls():
    import pytorchdeeplearing_b200 as b200
    from pytorchdeeplearing_b200 import runtime
    calls = []

    class _Rec(EmuBackend):
        def conv(self, kind, dims, x, *a, **k):
            if kind == UP:
                calls.append(x.shape[-1])
            return super().conv(kind, dims, x, *a, **k)

    runtime._set_backend_for_testing(_Rec())
    try:
        m = b200.VNet3d(1, 2).train()
        out = m(torch.randn(1, 1, 16, 16, 16))
        out[0].float().sum().backward()
    finally:
        runtime._set_backend_for_testing(None)
    assert 32 in calls                      # up_tr32's transposed conv (32 -> 16) through backend.conv
    assert all(p.grad is not None for p in m.parameters())
