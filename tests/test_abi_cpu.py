"""The C-ABI shared library loads without a GPU and exports every symbol include/b200seg.h declares
(no compute calls here).  Runs in the CPU suite."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    with open(os.path.join(ROOT, "include", "b200seg.h")) as f:
        src = f.read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200seg_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_expected_surface():
    syms = _declared_symbols()
    for must in ("b200seg_conv", "b200seg_wgrad", "b200seg_gn_finalize", "b200seg_apply", "b200seg_gn_bwd_reduce",
                 "b200seg_gn_bwd_finalize", "b200seg_gn_bwd_apply", "b200seg_loss_partials", "b200seg_loss_bwd",
                 "b200seg_pool_fwd", "b200seg_pool_bwd", "b200seg_head_probs", "b200seg_last_error"):
        assert must in syms


def test_library_loads_and_exports_every_declared_symbol():
    from pytorchdeeplearing_b200 import _abi, build
    if not os.path.exists(_abi.LIB_PATH):
        build.build()
    lib = _abi.load_library()
    assert lib.b200seg_version() >= 100
    declared = _declared_symbols()
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/b200seg.h but not exported"
    # the ctypes prototype table covers the whole header (and nothing else)
    assert sorted(_abi.EXPORTED_SYMBOLS) == declared
    assert lib.b200seg_last_error() is not None
    # pure host-side query, no device needed
    assert lib.b200seg_conv_tc_eligible(0, 32, 32) == 1
    assert lib.b200seg_conv_tc_eligible(0, 1, 16) == 0
    assert lib.b200seg_conv_tc_eligible(2, 32, 64) == 1       # k2s2 down conv runs on the tensor-core path too
    assert lib.b200seg_conv_tc_eligible(3, 32, 48) == 0       # transposed conv needs power-of-two Cout
    assert lib.b200seg_conv_halo_eligible(0, 16, 16) == 1 and lib.b200seg_conv_halo_eligible(0, 64, 64) == 0


def test_product_path_refuses_to_run_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from pytorchdeeplearing_b200 import _abi
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _abi.CudaBackend()
