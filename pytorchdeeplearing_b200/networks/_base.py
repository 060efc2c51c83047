"""Shared plumbing of the drop-in networks: one ``autograd.Function`` per forward that hands
the whole net to the layer program (``engine.Engine``), i.e. to the sm_90a kernels."""
from __future__ import annotations

import struct
from typing import List, Optional

import torch
import torch.nn as nn

from .. import runtime
from ..engine import Engine, P_DROP


class _SegNetFunction(torch.autograd.Function):
    """forward: (x, *params) -> (logits, probs); backward: d logits -> d params.
    Backward runs on the autograd thread; every kernel launch takes device+stream explicitly."""

    @staticmethod
    def forward(ctx, mod, need_grad, x, masks, *params):
        be = runtime.get_backend(x)
        eng = Engine(be, runtime.act_dtype(), mod._dims)
        P = dict(zip(mod._pnames, [p.detach() for p in params]))
        xx = x.detach()
        if xx.dtype != torch.float32:
            xx = xx.float()
        logits, probs = getattr(eng, mod._arch + "_forward")(P, xx, masks, need_grad)
        ctx.eng = eng if need_grad else None
        ctx.arch = mod._arch
        ctx.names = mod._pnames
        ctx.set_materialize_grads(False)
        return logits, probs

    @staticmethod
    def backward(ctx, g_logits, g_probs):
        if g_probs is not None:
            # the reference's second output carries grad through softmax/sigmoid; the drop-in computes parameter
            # gradients from d loss / d logits only (every hot-path loss takes logits, model/losses.py)
            raise RuntimeError("pytorchdeeplearing_b200: a gradient reached the network through its second output "
                               "(probs); losses must be computed on the logits (first output)")
        eng: Engine = ctx.eng
        if eng is None:
            raise RuntimeError("pytorchdeeplearing_b200: backward through the network a second time (the saved "
                               "activations are released after the first backward; retain_graph is not supported)")
        if g_logits is None:
            return (None, None, None, None) + (None,) * len(ctx.names)
        g = g_logits.permute(0, 2, 3, 4, 1) if g_logits.dim() == 5 else g_logits.permute(0, 2, 3, 1).unsqueeze(1)
        return _net_backward(ctx, eng, g)


def _net_backward(ctx, eng: Engine, g: torch.Tensor):
    """the engine's backward from d loss / d logits ``g`` (channels-last, or (N, numclass) for a classifier), with the
    gradient all-reduce of data-parallel runs; returns the autograd tuple of (mod, need_grad, x, masks, *params)"""
    if not g.is_contiguous():
        g = g.contiguous()
    if g.dtype != torch.float32:
        g = g.float()
    enabled, group = runtime.dp_state()
    works, split = [], [None]
    if enabled:
        import torch.distributed as dist

        def bucket_ready(flat_, off):
            # gradients flat[off:] (deepest encoder block .. head, ~96 % of the bytes) are final: their SUM
            # all-reduce starts now and overlaps the rest of backward (SURVEY.md section 8e, C1)
            split[0] = off
            works.append(dist.all_reduce(flat_[off:], op=dist.ReduceOp.SUM, group=group, async_op=True))
        eng.bucket_hook = bucket_ready
    flat = getattr(eng, ctx.arch + "_backward")(g)
    if enabled:
        if split[0] is None:
            dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        else:
            if split[0] > 0:
                dist.all_reduce(flat[:split[0]], op=dist.ReduceOp.SUM, group=group)
            for w in works:
                w.wait()
    grads = [eng.grads[n] for n in ctx.names]
    ctx.eng = None
    return (None, None, None, None) + tuple(grads)


class _ClsNetFunction(torch.autograd.Function):
    """Single-output form for the classifiers (ResNet2d / ResNet3d): forward (x, *params) -> (N, numclass) logits;
    backward: d logits -> d params."""

    @staticmethod
    def forward(ctx, mod, need_grad, x, masks, *params):
        be = runtime.get_backend(x)
        eng = Engine(be, runtime.act_dtype(), mod._dims)
        P = dict(zip(mod._pnames, [p.detach() for p in params]))
        xx = x.detach()
        if xx.dtype != torch.float32:
            xx = xx.float()
        logits = getattr(eng, mod._arch + "_forward")(P, xx, masks, need_grad)
        ctx.eng = eng if need_grad else None
        ctx.arch = mod._arch
        ctx.names = mod._pnames
        ctx.set_materialize_grads(False)
        return logits

    @staticmethod
    def backward(ctx, g_logits):
        eng: Engine = ctx.eng
        if eng is None:
            raise RuntimeError("pytorchdeeplearing_b200: backward through the network a second time (the saved "
                               "activations are released after the first backward; retain_graph is not supported)")
        if g_logits is None:
            return (None, None, None, None) + (None,) * len(ctx.names)
        return _net_backward(ctx, eng, g_logits)


class MaskPlan:
    """All dropout channel masks of one forward from ONE kernel launch (``b200seg_dropout_masks``) that reproduces the
    Philox stream of the reference's per-module ``bernoulli_`` draws on a CUDA generator (SURVEY.md 0.5), so
    ``torch.manual_seed(s); model(x)`` gives the masks the reference's own GPU run would draw.  Under data
    parallelism every rank takes ITS rows of the global-batch draw (SURVEY.md 8e): same seed on every rank."""

    def __init__(self, be, chans, n, device):
        self.be, self.n, self.device = be, n, device
        rank, world = runtime.dp_rank_world()
        first, rows = 0, []
        for c in chans:
            rows += [first, n * c, rank * n * c]
            first += n * c
        self.total, self.nmasks = first, len(chans)
        self.table = be.upload_bytes(struct.pack(f"{len(rows)}i", *rows), device)
        self.rng = torch.zeros(2, dtype=torch.int64, device=device)
        self.out = torch.empty(first, dtype=torch.float32, device=device)
        self.views, off = [], 0
        for c in chans:
            self.views.append(self.out[off:off + n * c].view(n, c))
            off += n * c

    def refresh(self):
        """Take {seed, offset} from the device's default generator, advance it by what the per-module draws would
        consume (4 per mask) and hand the pair to the device.  Never called during stream capture."""
        idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
        gen = torch.cuda.default_generators[idx]
        off = gen.get_offset()
        gen.set_offset(off + 4 * self.nmasks)
        self.be.upload_into(struct.pack("<Qq", gen.initial_seed() & 0xFFFFFFFFFFFFFFFF, off), self.rng)

    def launch(self):
        self.be.dropout_masks(self.rng, self.table, self.nmasks, self.total, P_DROP, self.out)
        return self.views


class SegNetBase(nn.Module):
    """Common forward of VNet3d / UNet3d / UNet2d.  Subclasses build the parameter tree with the
    reference's attribute names (so ``state_dict`` / ``load_state_dict`` / ``apply(initialize_weights)``
    behave identically) and set ``_arch`` / ``_dims`` / ``_mask_channels``."""

    _arch = ""
    _dims = 3
    _function = _SegNetFunction       # (logits, probs); the classifiers return logits only (_ClsNetFunction)
    dropout_masks: Optional[List[torch.Tensor]] = None     # test hook: inject (N,C) scales

    def _finish_init(self):
        self._pnames = [n for n, _ in self.named_parameters()]
        self._mask_plans = {}

    def _mask_channels(self) -> List[int]:
        raise NotImplementedError

    def mask_plan(self, n: int, device) -> "MaskPlan":
        key = (n, str(device), runtime.dp_rank_world())
        plan = self._mask_plans.get(key)
        if plan is None:
            plan = self._mask_plans[key] = MaskPlan(runtime.get_backend(torch.empty(0, device=device)),
                                                    self._mask_channels(), n, device)
        return plan

    def _draw_masks(self, x: torch.Tensor) -> Optional[List[torch.Tensor]]:
        """nn.Dropout3d/2d(p=0.2) contract (SURVEY.md section 0.5): per call, in module-call
        order, ``x.new_empty((N,C,1,1,1)).bernoulli_(1-p).div_(1-p)`` from the default generator."""
        if not self.training:
            return None
        if self.dropout_masks is not None:
            return [m.to(device=x.device, dtype=torch.float32) for m in self.dropout_masks]
        if x.is_cuda and runtime._TEST_BACKEND is None and not runtime.is_capturing(x.device):
            plan = self.mask_plan(x.shape[0], x.device)     # ONE launch instead of one bernoulli_ per layer
            plan.refresh()
            return plan.launch()
        # torch draws (CPU test backend, or inside a user's own stream capture where the generator state must stay
        # graph-safe): every mask by its own ``bernoulli_`` call on an (N,C,1,..) view of one flat buffer -- the same
        # generator consumption as the reference's per-module draws; under data parallelism the draw has the GLOBAL
        # batch and the rank keeps its rows.
        rank, world = runtime.dp_rank_world()
        n = x.shape[0]
        ng = n * world
        ones = (1,) * self._dims
        chans = self._mask_channels()
        flat = x.new_empty((ng * sum(chans),), dtype=torch.float32)
        masks, off = [], 0
        for c in chans:
            flat[off:off + ng * c].view((ng, c) + ones).bernoulli_(1 - P_DROP)
            masks.append(flat[off:off + ng * c].view(ng, c)[rank * n:(rank + 1) * n])
            off += ng * c
        flat.div_(1 - P_DROP)
        return masks

    def forward(self, x):
        if x.dim() != self._dims + 2:
            raise RuntimeError(f"expected a {self._dims + 2}-D input (N,C,{'D,' if self._dims == 3 else ''}H,W), "
                               f"got {tuple(x.shape)}")
        for s in x.shape[2:]:
            if s % 16 != 0:
                raise RuntimeError("spatial sizes must be multiples of 16 (four stride-2 stages), got "
                                   f"{tuple(x.shape[2:])}")
        params = [p for _, p in self.named_parameters()]
        for p in params:
            if p.dtype != torch.float32:
                raise RuntimeError("pytorchdeeplearing_b200 keeps parameters in fp32 (state_dict contract; bf16 / fp32 "
                                   f"compute is selected with set_precision): found {p.dtype} -- do not call .half()/"
                                   ".bfloat16() on the model")
        if x.requires_grad and torch.is_grad_enabled():
            raise RuntimeError("pytorchdeeplearing_b200 does not provide d/d(input) (the reference's training path never "
                               "asks for it); detach the input")
        masks = self._draw_masks(x)
        # (grad mode is always off inside Function.forward, so the decision is taken here)
        need_grad = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        return self._function.apply(self, need_grad, x, masks, *params)


class _Holder(nn.Module):
    """Parameter container with the reference's attribute names; never called directly."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("sub-blocks of the drop-in are parameter holders; call the network itself")
