"""Runtime switches of the drop-in: precision mode, backend lookup, data-parallel state.

There is exactly one product backend: the sm_90a CUDA library behind the C ABI of
``include/b200seg.h`` (``_abi.CudaBackend``).  There is NO CPU / eager / library fallback:
if the library is missing or the tensors are not on a CUDA device the call raises.
``_set_backend_for_testing`` exists so the CPU test-suite can drive the host-side layer
program with ``tests/emu_backend.py``; product code never calls it.
"""
from __future__ import annotations

import os
from typing import Optional

import torch

_PRECISION = os.environ.get("B200SEG_PRECISION", "bf16").lower()
_TEST_BACKEND = None
_CUDA_BACKEND = None


def set_precision(mode: str) -> None:
    """'bf16' (perf mode: bf16 activation/weight storage, fp32 accumulate) or
    'fp32' (parity mode: fp32 storage and FFMA arithmetic; SURVEY.md section 0.8)."""
    global _PRECISION
    mode = mode.lower()
    if mode not in ("bf16", "fp32"):
        raise ValueError("precision must be 'bf16' or 'fp32'")
    _PRECISION = mode


def get_precision() -> str:
    return _PRECISION


def act_dtype() -> torch.dtype:
    return torch.bfloat16 if _PRECISION == "bf16" else torch.float32


def _set_backend_for_testing(backend) -> None:
    """Instrumentation / test hook: route every op through ``backend`` (an object with the
    ``CudaBackend`` method set).  Used by the CPU test-suite (emulated ops) and by bench.py's per-kernel
    timing wrapper around the real ``CudaBackend``; ``None`` restores the product backend."""
    global _TEST_BACKEND
    _TEST_BACKEND = backend


def cuda_backend():
    """The process-wide ``CudaBackend`` (created on first use; raises without a CUDA device)."""
    global _CUDA_BACKEND
    if _CUDA_BACKEND is None:
        from . import _abi
        _CUDA_BACKEND = _abi.CudaBackend()
    return _CUDA_BACKEND


def get_backend(t: torch.Tensor):
    if _TEST_BACKEND is not None:
        return _TEST_BACKEND
    if not t.is_cuda:
        raise RuntimeError(
            "pytorchdeeplearing_b200 runs only on a CUDA (sm_90a) device: got a tensor on "
            f"'{t.device}'. There is no CPU fallback -- move the model and inputs to cuda.")
    return cuda_backend()


def is_capturing(device=None) -> bool:
    """True while the current CUDA stream is being captured into a graph (host-side checks that synchronise, and the
    torch generator bookkeeping of the dropout masks, are skipped then)."""
    if not torch.cuda.is_available():
        return False
    if device is not None and getattr(device, "type", "cuda") != "cuda":
        return False
    return torch.cuda.is_current_stream_capturing()


# ---------------------------------------------------------------------------- data parallel
_DP_GROUP = None
_DP_ENABLED = False


def enable_data_parallel(group=None) -> None:
    """Batch-sharded data parallelism (SURVEY.md section 8e): after this call the losses
    all-reduce their partial sums (global-batch-exact Dice) and the network backward
    SUM-all-reduces the flat gradient bucket over ``group`` (default: WORLD)."""
    global _DP_GROUP, _DP_ENABLED
    import torch.distributed as dist
    if not dist.is_initialized():
        raise RuntimeError("torch.distributed is not initialised")
    _DP_GROUP, _DP_ENABLED = group, True


def disable_data_parallel() -> None:
    global _DP_GROUP, _DP_ENABLED
    _DP_GROUP, _DP_ENABLED = None, False


def dp_state():
    return _DP_ENABLED, _DP_GROUP


def dp_rank_world():
    """(rank, world size) of the data-parallel group; (0, 1) when data parallelism is off."""
    if not _DP_ENABLED:
        return 0, 1
    import torch.distributed as dist
    return dist.get_rank(_DP_GROUP), dist.get_world_size(_DP_GROUP)
